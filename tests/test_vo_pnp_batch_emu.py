"""mvo_vo_pnp_batch_dev EXECUTED ON THE CPU: the whole library built for the host (tests/emu_build.py, every translation unit), so
the batch forms of the PnP kernels (csrc/pnp_kernels.cuh: k_pnp_hypotheses / k_pnp_score / k_pnp_finish<true>), the per-job
refit (csrc/ba.cu: k_ba_pose<1, CACHED, false, true>) and the tail (csrc/pnp.cu: k_pnp_batch_tail) run through
tests/cpp/cuda_emu.h.  Every job's record, inlier list and kept matches must be BYTE-IDENTICAL to the emulated test entry
mvo_test_pnp_dev on the job's rows (tests/vo_pnp_batch_cases.py), with sentinels past every count and five launches.
tests/test_vo_pnp_batch_gpu.py is the check on the hardware."""
import ctypes as C
import os

import numpy as np
import pytest

import vo_pnp_batch_cases as cases

CAP, H = 64, 128


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import emu_build
    import mvo_b200
    so = emu_build.build(tmp_path_factory.mktemp("pnpbatchemu"), emu_build.ALL_UNITS)
    lib = C.CDLL(str(so))
    for name in ("mvo_default_params", "mvo_default_track_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_kernel_launches",
                 "mvo_solve_pnp_ransac", "mvo_vo_pnp_batch_dev", "mvo_set_params"):
        res, args = mvo_b200.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def ctx(lib):
    import mvo_b200
    p = mvo_b200.Params()
    lib.mvo_default_params(C.byref(p))
    p.pnp_hypotheses = H
    h = C.c_void_p()
    assert lib.mvo_create(C.byref(h), 0, C.byref(p)) == 0
    yield h
    lib.mvo_destroy(h)


@pytest.fixture(scope="module")
def scene():
    return cases.Scene(CAP, seed=3)


def _csize():
    v = int(os.environ.get("MVO_BA_CLUSTER", "8") or 8)
    return v if 1 <= v <= 8 else 8


def test_emulated_batch_equals_the_single_call(lib, ctx, scene):
    s = scene
    tp = cases.track_params(lib)
    refs = [cases.reference(lib, ctx, s, j, tp, H) for j in range(s.n_jobs)]
    l0 = lib.mvo_kernel_launches(ctx)
    rc, outs = cases.call(lib, ctx, s, tp)
    assert rc == 0, lib.mvo_last_error(ctx)
    assert lib.mvo_kernel_launches(ctx) - l0 == cases.LAUNCHES
    cases.check_coverage(outs, s)
    for j in range(s.n_jobs):
        cases.check_exact(refs[j], outs, s, j)
        cases.check_host(lib, ctx, s, j, tp, outs, _csize())
    # repeated jobs give the same rows
    out = outs[0]
    assert out[s.kinds.index("repeat")].tobytes() == out[s.kinds.index("full")].tobytes()


def test_emulated_without_kept_rows_and_at_the_threshold(lib, ctx, scene):
    s = scene.subset([1, 3, 4, 9, 12])
    tp = cases.track_params(lib)
    refs = [cases.reference(lib, ctx, s, j, tp, H) for j in range(s.n_jobs)]
    rc, outs = cases.call(lib, ctx, s, tp, outs=cases.outputs(s.n_jobs, CAP, kept=False))
    assert rc == 0, lib.mvo_last_error(ctx)
    for j in range(s.n_jobs):
        cases.check_exact(refs[j], outs, s, j)
    cases.check_threshold(lib, ctx, scene, tp)


def test_emulated_call_level_checks(lib, ctx, scene):
    s = scene
    tp = cases.track_params(lib)
    kinds = cases.call_level_kinds(s) + [(dict(n_jobs=32769), cases.UNSUPPORTED)]     # n_jobs x 128 hypotheses > 2^22
    for kw, want in kinds:
        outs = cases.outputs(s.n_jobs, CAP)
        l0 = lib.mvo_kernel_launches(ctx)
        rc, got = cases.call(lib, ctx, s, tp, outs=outs, **kw)
        assert rc == want, (kw, rc)
        assert lib.mvo_kernel_launches(ctx) == l0
        assert all((a.view(np.uint8) == cases.SENTINEL).all() for a in got), kw
    # a non-finite max_dist_to_prev
    for v in (np.nan, np.inf):
        assert cases.call(lib, ctx, s, cases.track_params(lib, max_dist=v))[0] == cases.INVALID_ARG
    # null required pointers (d_kept is optional)
    for name in ("mm", "matches", "p3", "p2", "T_prev", "out", "inl"):
        outs = cases.outputs(s.n_jobs, CAP)
        target = {"mm": s.mm, "matches": s.matches, "p3": s.p3, "p2": s.p2, "T_prev": s.T_prev, "out": outs[0], "inl": outs[1]}[name]
        rc, _ = cases.call(lib, ctx, s, tp, outs=outs, ptr=lambda a: None if a is target else a.ctypes.data)
        assert rc == cases.INVALID_ARG, name
    assert cases.call(lib, ctx, s, None)[0] == cases.INVALID_ARG
    # pnp_mode 1 has no batch form
    import mvo_b200
    p = mvo_b200.Params()
    lib.mvo_default_params(C.byref(p))
    p.pnp_hypotheses, p.pnp_mode = H, 1
    assert lib.mvo_set_params(ctx, C.byref(p)) == 0
    try:
        assert cases.call(lib, ctx, s, tp)[0] == cases.UNSUPPORTED
    finally:
        p.pnp_mode = 0
        assert lib.mvo_set_params(ctx, C.byref(p)) == 0
    # zero jobs: nothing launched
    l0 = lib.mvo_kernel_launches(ctx)
    assert cases.call(lib, ctx, s, tp, n_jobs=0)[0] == 0 and lib.mvo_kernel_launches(ctx) == l0
