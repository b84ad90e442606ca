"""mvo_vo_keyframe_points_batch_dev EXECUTED ON THE CPU: the whole library built for the host (tests/emu_build.py, every
translation unit plus vo_init_batch.cu), so the three kernels run through tests/cpp/cuda_emu.h and their device code is compiled by
g++: acos is glibc's there, and every pair's record, kept matches, points, angles, world positions and directions must be
BYTE-IDENTICAL to the host reference (tests/vo_keyframe_batch_cases.py: the state machine's keyframe branch over the library's host
entry points).  The emulation cannot show the device's acos or a contraction difference: tests/test_vo_keyframe_batch_gpu.py is
the check on the hardware."""
import ctypes as C

import numpy as np
import pytest

import vo_keyframe_batch_cases as cases

CAP = 320


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import emu_build
    import mvo_b200
    so = emu_build.build(tmp_path_factory.mktemp("vokfbatchemu"), emu_build.ALL_UNITS + ["vo_init_batch.cu"])
    lib = C.CDLL(str(so))
    for name in ("mvo_default_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_kernel_launches", "mvo_vo_default_params",
                 "mvo_retain_good_triangulation", "mvo_do_triangulation", "mvo_vo_keyframe_points_batch_dev"):
        res, args = mvo_b200.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def ctx(lib):
    import mvo_b200
    p = mvo_b200.Params()
    lib.mvo_default_params(C.byref(p))
    h = C.c_void_p()
    assert lib.mvo_create(C.byref(h), 0, C.byref(p)) == 0
    yield h
    lib.mvo_destroy(h)


def _run(lib, ctx, b, vp, outs=None):
    l0 = lib.mvo_kernel_launches(ctx)
    rc, got = cases.call(lib, ctx, b, vp, outs=outs)
    assert rc == 0, lib.mvo_last_error(ctx)
    assert lib.mvo_kernel_launches(ctx) - l0 == cases.LAUNCHES
    return got


@pytest.fixture(scope="module")
def mixed(lib, ctx):
    b = cases.Batch(cases.mixed_specs(CAP), CAP, seed=3)
    vp = cases.vi.vo_params(lib)
    refs = [cases.reference(lib, ctx, b, p, vp) for p in range(b.n_pairs)]
    return b, vp, refs


def test_emulated_batch_equals_the_state_machine(lib, ctx, mixed):
    b, vp, refs = mixed
    got = _run(lib, ctx, b, vp)
    for p in range(b.n_pairs):
        cases.check_exact(refs[p], got, p)
    recs = [r[1] for r in refs]
    # the batch reaches what it was built for
    assert recs[0]["n_kept"] == recs[0]["n_inliers"] == 300
    assert recs[1]["n_kept"] == 200
    assert recs[2]["usable"] == 1 and recs[2]["n_inliers"] == 0 and recs[2]["n_kept"] == 0 and recs[2]["median_angle"] == 0
    assert recs[3]["n_inliers"] == 1 and recs[3]["n_kept"] == 1
    assert 0 < recs[4]["n_kept"] <= 120 - 30
    assert recs[5]["n_kept"] == 120 - 3
    for i in (6, 7):
        ang, _ = cases.all_angles(lib, ctx, b, i)
        assert np.isnan(ang).any() and np.isnan(refs[i][4]).any(), i    # NaN angles are kept
    assert not np.isnan(recs[6]["median_angle"]) and np.isnan(recs[7]["median_angle"])
    assert recs[8]["t_curr_to_prev"].tolist() == [0.0, 0.0, 0.0]
    assert recs[9]["n_inliers"] == CAP
    assert refs[11][2].tobytes() == refs[4][2].tobytes() and refs[11][5].tobytes() == refs[4][5].tobytes()   # repeated pair
    assert recs[10]["n_kept"] > 0                                       # reversed pair
    assert recs[13]["usable"] == 0 and recs[13]["status"] == 0 and recs[13]["n_matches"] == 5
    assert [r[0] for r in refs[14:16]] == [cases.INVALID_ARG, cases.CUDA_ERR]
    assert [r[0] for r in refs[16:]] == [cases.INVALID_ARG] * len(cases.BAD_KINDS)


def test_emulated_optional_rows_may_be_null(lib, ctx, mixed):
    b, vp, refs = mixed
    for world, norm in ((False, True), (True, False), (False, False)):
        got = _run(lib, ctx, b, vp, outs=cases.outputs(b.n_pairs, b.cap, world, norm))
        for p in range(b.n_pairs):
            cases.check_exact(refs[p], got, p)


def test_emulated_thresholds_exactly_on_an_angle(lib, ctx):
    b = cases.Batch([dict(n=101, near=2)], CAP, seed=5)
    ang, med = cases.all_angles(lib, ctx, b, 0)
    srt = np.sort(ang)
    base = cases.reference(lib, ctx, b, 0, cases.vi.vo_params(lib))[1]["n_kept"]
    for vp, expect in ((cases.vi.vo_params(lib, min_triang_angle=float(srt[10])), base - 10),                # the angle at the minimum stays
                       (cases.vi.vo_params(lib, max_ratio_angle_to_median=float(srt[-2] / med)), 101 - 1)):  # the one above goes
        got = _run(lib, ctx, b, vp)
        ref = cases.reference(lib, ctx, b, 0, vp)
        cases.check_exact(ref, got, 0)
        assert ref[1]["n_kept"] == expect


def test_emulated_call_level_checks(lib, ctx):
    b = cases.Batch([dict(n=30)], CAP)
    vp = cases.vi.vo_params(lib)
    assert cases.call(lib, ctx, b, vp)[0] == 0
    for q in (np.nan, np.inf):
        for f in ("min_triang_angle", "max_ratio_angle_to_median"):
            assert cases.call(lib, ctx, b, cases.vi.vo_params(lib, **{f: q}))[0] == cases.INVALID_ARG, f
        for i in (0, 4):
            Kb = cases.K.copy()
            Kb.flat[i] = q
            assert cases.call(lib, ctx, b, vp, Kp=Kb)[0] == cases.INVALID_ARG
    for v in (0.0, -1.0):
        for i in (0, 4):
            Kb = cases.K.copy()
            Kb.flat[i] = v
            assert cases.call(lib, ctx, b, vp, Kp=Kb)[0] == cases.INVALID_ARG
