"""mvo_esti_motion_by_essential_batch_dev EXECUTED ON THE CPU: the whole library built for the host (tests/emu_build.py, every
translation unit), so the batched two-view kernels (csrc/epipolar_kernels.cuh: k_epi_gather ... k_triangulate_batch) run through
tests/cpp/cuda_emu.h, against the emulated mvo_estimate_relative_poses(calc_homo = 0) on the same points, byte for byte.
Small: 256 hypotheses, a few hundred correspondences per pair (tests/test_two_view_batch_gpu.py is the full-size check on the
hardware)."""
import ctypes as C

import numpy as np
import pytest

import two_view_batch_cases as cases

CAP = 320
HYP = 256


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import emu_build
    import mvo_b200
    so = emu_build.build(tmp_path_factory.mktemp("twoviewbatchemu"), emu_build.ALL_UNITS)
    lib = C.CDLL(str(so))
    for name in ("mvo_default_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_estimate_relative_poses",
                 "mvo_esti_motion_by_essential_batch_dev", "mvo_kernel_launches"):
        res, args = mvo_b200.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def ctx(lib):
    import mvo_b200
    p = mvo_b200.Params()
    lib.mvo_default_params(C.byref(p))
    p.epi_hypotheses = HYP
    h = C.c_void_p()
    assert lib.mvo_create(C.byref(h), 0, C.byref(p)) == 0
    yield h
    lib.mvo_destroy(h)


def _specs():
    g = [cases.general_scene(s, n) for s, n in ((0, 300), (1, 240), (2, 180))]
    planar = cases.general_scene(3, 200, outliers=0.1, planar=True)
    clean = cases.general_scene(4, CAP, noise=0.3, outliers=0.0)
    return [("points",) + g[0], ("points",) + g[1], ("points",) + planar,
            ("points", clean[0][:8], clean[1][:8]), ("points", clean[0][:9], clean[1][:9]), ("points",) + clean,
            ("points",) + cases.random_pair(5, 60),                          # all outliers: DEGENERATE
            ("points", g[2][0][:5], g[2][1][:5]),                             # n < 8: DEGENERATE
            ("bad_frame",), ("count", -1), ("count", CAP + 1), ("bad_index",), ("bad_frame",),
            ("points",) + g[2]]


def _call(lib, ctx, b, with_pts):
    res, inl, pts = cases.outputs(b.n_pairs, b.cap)
    Kc = np.ascontiguousarray(cases.K, np.float64)
    l0 = lib.mvo_kernel_launches(ctx)
    rc = lib.mvo_esti_motion_by_essential_batch_dev(ctx, b.kpts.ctypes.data, b.counts.ctypes.data, b.batch, b.cap, b.pairs.ctypes.data,
                                                    b.n_pairs, b.matches.ctypes.data, b.n_matches.ctypes.data, Kc.ctypes.data, 1.0,
                                                    res.ctypes.data, inl.ctypes.data, pts.ctypes.data if with_pts else None)
    assert rc == 0, lib.mvo_last_error(ctx)
    assert lib.mvo_kernel_launches(ctx) - l0 == cases.launches_per_call(with_pts)
    return res, inl, pts


def test_emulated_batch_equals_emulated_estimate_relative_poses(lib, ctx):
    b = cases.Batch(_specs(), CAP, seed=1)
    refs = cases.references(lib, ctx, b, cases.K)
    status = [rc for rc, _ in refs]
    assert [status[i] for i in (0, 1, 2, 5, 13)] == [0] * 5, status
    assert status[6] == status[7] == cases.DEGENERATE, status
    assert status[8:13] == [cases.INVALID_ARG] * 5, status
    for with_pts in (True, False):
        res, inl, pts = _call(lib, ctx, b, with_pts)
        for p in range(b.n_pairs):
            cases.check_pair(b, p, res, inl, pts, refs[p], with_pts)
