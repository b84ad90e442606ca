"""The pose-only LM kernel (k_ba_pose, csrc/ba.cu) in the complete library built for the host (tests/emu_build.py, as in
test_full_library_emu.py) against the C oracle, in child processes (MVO_LIB points the wrapper at the emulated build; the
cluster size is read once per process).  The CPU-tier subset of test_ba_pose_gpu.py: the points next to a camera's principal
plane (chi2 beyond the float range), cluster sizes 1, 3 and 8, CH = 2 and the uncached kernel, and the frame-buffer variant
through mvo_test_ba_pose_store.  Cases and checks: tests/ba_pose_cases.py."""
import pytest

import ba_pose_cases as B


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    import emu_build
    return emu_build.build(tmp_path_factory.mktemp("poseemu"), emu_build.ALL_UNITS)


def _check_all(out, csize):
    for n, (r, dbg) in out.items():
        B.check(B.CASES[n](), r, dbg, csize)


NEAR = ["near_1e-12_huber", "near_1e-18_huber", "near_1e-18_plain", "near_1e-30_huber", "near_1e-30_plain", "near_1e-40_huber",
        "near_1e-40_plain", "refit_shape"]


def test_near_plane_points_match_the_oracle(emu_lib):
    """chi2 beyond FLT_MAX and a subnormal depth: the Huber weight, the depth reciprocal and the gain ratio must not go
    through their float seeds (rsqrtf(inf) = 0 made the edge subtract from chi2; a gain ratio of 0 ended the LM)."""
    _check_all(B.run_children(NEAR, lib=emu_lib), 8)


@pytest.mark.parametrize("cluster", [1, 3, 8])
def test_cluster_sizes(emu_lib, cluster):
    _check_all(B.run_children(["iters2", "many_small_frames", "store_basic"], cluster=cluster, lib=emu_lib), cluster)


def test_chunking_ch2_and_uncached(emu_lib):
    out = B.run_children(["c1_ch2", "c1_unc5"], cluster=1, lib=emu_lib)
    assert [out[n][1][0]["chunk"] for n in ("c1_ch2", "c1_unc5")] == [2, 5]
    _check_all(out, 1)


STORE = ["store_bad_ids", "store_cnt_over_cap", "store_min_links", "store_frame_all_dead", "store_all_dropped", "store_skip",
         "store_slot_order", "store_17_slots", "store_eu_over"]


def test_store_variant(emu_lib):
    _check_all(B.run_children(STORE, cluster=1, lib=emu_lib), 1)
