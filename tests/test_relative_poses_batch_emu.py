"""mvo_estimate_relative_poses_batch_dev EXECUTED ON THE CPU: the whole library built for the host (tests/emu_build.py, every
translation unit plus two_view_batch.cu, the combine step's own unit), so the essential and homography kernels
(csrc/epipolar_kernels.cuh) and the combine step (csrc/two_view_batch.cu) run through tests/cpp/cuda_emu.h, against the emulated mvo_estimate_relative_poses(calc_homo = 1) on the same points, record by
record and row by row, for both motion_cam2_to_cam1 values, with and without triangulation.  Small: 256 hypotheses, a few hundred
correspondences per pair (tests/test_relative_poses_batch_gpu.py is the full-size check on the hardware).  The emulation compiles
every device function with g++, so it cannot show a contraction difference between the device and the host: only the GPU tier can."""
import ctypes as C

import numpy as np
import pytest

import relative_poses_batch_cases as cases
import two_view_batch_cases as tvb

CAP = 320
HYP = 256


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import emu_build
    import mvo_b200
    so = emu_build.build(tmp_path_factory.mktemp("relposesbatchemu"), emu_build.ALL_UNITS + ["two_view_batch.cu"])
    lib = C.CDLL(str(so))
    for name in ("mvo_default_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_estimate_relative_poses",
                 "mvo_estimate_relative_poses_batch_dev", "mvo_kernel_launches"):
        res, args = mvo_b200.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def _ctx(lib, **kw):
    import mvo_b200
    p = mvo_b200.Params()
    lib.mvo_default_params(C.byref(p))
    p.epi_hypotheses = HYP
    for k, v in kw.items():
        setattr(p, k, v)
    h = C.c_void_p()
    assert lib.mvo_create(C.byref(h), 0, C.byref(p)) == 0
    return h


def _specs():
    """(specs, truths): truths[p] = (R, t) for the pairs whose true motion is known."""
    specs, truths = [], []

    def add(spec, truth=None):
        specs.append(spec)
        truths.append(truth)
    for s, n in ((0, 300), (1, 240)):
        add(("points",) + tvb.general_scene(s, n), cases.general_truth(s))
    for s, move in ((11, (0.4, 0.05, 0.05)), (12, (0.4, 0.05, 0.05)), (11, (0.1, 0.1, -0.4)), (12, (0.1, 0.1, -0.4))):
        p1, p2, R, t = cases.planar_scene(s, 200, move=move)                   # planar: H chosen, best = 1 for the sideways moves,
        add(("points", p1, p2), (R, t))                                        # 2 for the backward ones
    p1, p2, R, t = cases.rotation_scene(21, 200)
    add(("points", p1, p2), (R, t))                                            # homography of a pure rotation: num_h = 0
    clean = tvb.general_scene(4, CAP, noise=0.3, outliers=0.0)
    add(("points", clean[0][:8], clean[1][:8]))                                # n = 8
    add(("points",) + clean, cases.general_truth(4))                           # n = cap
    add(("points",) + tvb.random_pair(5, 60))                                  # all outliers
    g = tvb.general_scene(2, 180)
    add(("points", g[0][:5], g[1][:5]))                                        # n = 5: DEGENERATE
    for s in (("bad_frame",), ("count", -1), ("count", CAP + 1), ("bad_index",), ("bad_frame",)):
        add(s)
    add(("points",) + g, cases.general_truth(2))
    return specs, truths


def test_emulated_batch_equals_emulated_estimate_relative_poses(lib):
    """At eh_ratio_threshold 0.3 the general scenes still choose E and the planar ones choose H (the default 0.5 puts exactly
    planar scenes on the E side, DESIGN.md section 10)."""
    h = _ctx(lib, eh_ratio_threshold=0.3)
    try:
        specs, truths = _specs()
        b = tvb.Batch(specs, CAP, seed=1)
        for motion in (1, 0):
            refs = cases.references(lib, h, b, cases.K, motion)
            status = [rc for rc, _ in refs]
            assert [status[i] for i in (7, 9, 10)] == [cases.DEGENERATE] * 3 and status[11:16] == [cases.INVALID_ARG] * 5, status
            assert all(status[i] == 0 for i in (0, 1, 2, 3, 4, 5, 6, 8, 16)), status
            assert refs[6][1]["num"] == 1, refs[6][1]["num"]                    # the pure rotation's only solution is filtered out
            assert [refs[i][1]["best"] for i in (0, 1, 8, 16)] == [0] * 4       # E chosen
            assert [refs[i][1]["best"] for i in range(2, 6)] == [1, 1, 2, 2]    # H chosen, both homography slots
            for with_pts in (True, False):
                res, inl, pts = cases.call(lib, h, b, motion, with_pts)
                for p in range(b.n_pairs):
                    cases.check_pair(b, p, res, inl, pts, refs[p], with_pts)
                    if truths[p] is not None and res[p]["status"] == 0:
                        cases.check_truth(res[p], *truths[p], motion)
    finally:
        lib.mvo_destroy(h)
