"""mvo_vo_map_matches_batch_dev EXECUTED ON THE CPU: the whole library built for the host (tests/emu_build.py, every translation
unit), so the map-query matcher (csrc/match.cu: match_batch_kernel<MODE, true>), the projection (k_project_map_batch) and the
filter (csrc/track_filter.cuh: k_map_match_filter) run through tests/cpp/cuda_emu.h.  Every job's record, candidate rows, match
list and PnP inputs must be BYTE-IDENTICAL to the host reference of tests/map_matches_batch_cases.py (the state machine's
projection restated over Python floats, the emulated mvo_match_features on the candidate arrays), with sentinels past every count
and the documented number of launches.  tests/test_map_matches_batch_gpu.py is the check on the hardware."""
import ctypes as C

import numpy as np
import pytest

import map_matches_batch_cases as cases

CAP = 320


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import emu_build
    import mvo_b200
    so = emu_build.build(tmp_path_factory.mktemp("mapmatchemu"), emu_build.ALL_UNITS)
    lib = C.CDLL(str(so))
    for name in ("mvo_default_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_kernel_launches", "mvo_match_features",
                 "mvo_vo_map_matches_batch_dev"):
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


@pytest.fixture(scope="module")
def scene():
    return cases.Scene(CAP, n_map=400, seed=1)


@pytest.mark.parametrize("method", [1, 2, 3])
def test_emulated_batch_equals_the_state_machine(lib, ctx, scene, method):
    s = scene
    refs = [cases.reference(lib, ctx, s, j, method) for j in range(s.n_jobs)]
    cases.check_scene_coverage(lib, ctx, s, refs, method)
    l0 = lib.mvo_kernel_launches(ctx)
    rc, got = cases.call(lib, ctx, s, method)
    assert rc == 0, lib.mvo_last_error(ctx)
    assert lib.mvo_kernel_launches(ctx) - l0 == cases.launches(method)
    for j in range(s.n_jobs):
        cases.check_exact(refs[j], got, j, s.n_map, CAP)


def test_emulated_null_optional_rows_and_empty_map(lib, ctx, scene):
    s = scene
    refs = [cases.reference(lib, ctx, s, j, 3) for j in range(s.n_jobs)]
    outs = cases.outputs(s.n_jobs, s.n_map, CAP, xy=False, pnp=False)
    rc, got = cases.call(lib, ctx, s, 3, outs=outs)
    assert rc == 0, lib.mvo_last_error(ctx)
    for j in range(s.n_jobs):
        cases.check_exact(refs[j], got, j, s.n_map, CAP)
    # n_map = 0: one launch, every valid job has no candidates and no matches
    l0 = lib.mvo_kernel_launches(ctx)
    rc, got = cases.call(lib, ctx, s, 1, n_map=0)
    assert rc == 0 and lib.mvo_kernel_launches(ctx) - l0 == cases.launches(1, 0)
    out, m = got[0], got[3].reshape(s.n_jobs, CAP)
    for j in range(s.n_jobs - s.n_bad):
        assert out[j]["status"] == 0 and out[j]["n_candidates"] == 0 and out[j]["n_matches"] == 0, j
        assert (m[j].view(np.uint8) == cases.SENTINEL).all()
    assert (got[1].view(np.uint8) == cases.SENTINEL).all()
    assert out[s.n_jobs - s.n_bad:]["status"].tolist() == [cases.INVALID_ARG] * s.n_bad


def test_emulated_call_level_checks(lib, ctx, scene):
    s = scene
    bad_K = np.array(cases.K)
    bad_K[0, 0] = np.nan
    neg_K = np.array(cases.K)
    neg_K[1, 1] = -500.0
    INV, UNS = cases.INVALID_ARG, cases.UNSUPPORTED
    kinds = [
        (dict(method=0), INV), (dict(method=4), INV), (dict(batch=0), INV), (dict(cap=0), INV), (dict(n_jobs=-1), INV),
        (dict(n_map=-1), INV), (dict(rows=0), INV), (dict(cols=0), INV), (dict(Kp=bad_K), INV), (dict(Kp=neg_K), INV),
        (dict(cap=8193), UNS), (dict(n_map=65536), UNS), (dict(n_jobs=65536), UNS), (dict(n_jobs=1025, n_map=65535), UNS),
    ]
    for kw, want in kinds:
        kw = dict(kw)
        method = kw.pop("method", 1)
        outs = cases.outputs(s.n_jobs, s.n_map, CAP)
        l0 = lib.mvo_kernel_launches(ctx)
        rc, got = cases.call(lib, ctx, s, method, outs=outs, **kw)
        assert rc == want, (kw, rc)
        assert lib.mvo_kernel_launches(ctx) == l0
        assert all((a.view(np.uint8) == cases.SENTINEL).all() for a in got if a is not None), kw
    # null required pointers (and only one of the PnP rows)
    names = ["kpts", "desc", "counts", "frames", "T", "map_pts", "map_desc", "out", "cand", "m", "p3"]
    for name in names:
        outs = list(cases.outputs(s.n_jobs, s.n_map, CAP))
        arrays = {"kpts": s.kpts, "desc": s.desc, "counts": s.counts, "frames": s.frames, "T": s.T, "map_pts": s.map_pts,
                  "map_desc": s.map_desc, "out": outs[0], "cand": outs[1], "m": outs[3], "p3": outs[4]}
        target = arrays[name]
        rc, _ = cases.call(lib, ctx, s, 3, outs=tuple(outs), ptr=lambda a: None if a is target else a.ctypes.data)
        assert rc == INV, name
    # method 1 needs no keypoints without the PnP rows; a zero-job call does nothing
    outs = cases.outputs(s.n_jobs, s.n_map, CAP, pnp=False)
    rc, _ = cases.call(lib, ctx, s, 1, outs=outs, ptr=lambda a: None if a is s.kpts else a.ctypes.data)
    assert rc == 0
    l0 = lib.mvo_kernel_launches(ctx)
    assert cases.call(lib, ctx, s, 1, n_jobs=0)[0] == 0 and lib.mvo_kernel_launches(ctx) == l0
