"""mvo_match_features_batch_dev EXECUTED ON THE CPU: the whole library built for the host (tests/emu_build.py, every translation
unit), so the batched all-pairs kernel (csrc/match.cu: match_batch_kernel) and the batched matchFeatures tail
(csrc/track_filter.cuh: k_match_filter_batch) run through tests/cpp/cuda_emu.h, against the emulated mvo_match_features on the
same descriptors.  Small: five frames of a few hundred keypoints, four pairs, all three methods (tests/test_match_batch_gpu.py
is the full-size check on the hardware)."""
import ctypes as C

import numpy as np
import pytest

import mvo_synth

CAP = 300


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import emu_build
    import mvo_b200
    so = emu_build.build(tmp_path_factory.mktemp("matchbatchemu"), emu_build.ALL_UNITS)
    lib = C.CDLL(str(so))
    for name in ("mvo_default_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_match_features", "mvo_match_features_batch_dev",
                 "mvo_kernel_launches"):
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


def _frames():
    """Five frames in the layout of mvo_orb_extract_batch_dev: descriptors with duplicated rows (distance ties), keypoints
    clustered so that a 50 px radius keeps some trains and drops others, counts 300 / 257 / 0 / 1 / 280."""
    import mvo_b200
    rng = np.random.default_rng(7)
    counts = np.array([300, 257, 0, 1, 280], np.int32)
    desc = np.zeros((len(counts), CAP, 32), np.uint8)
    kpts = np.zeros((len(counts), CAP), mvo_b200.KEYPOINT_DTYPE)
    base = rng.uniform([0, 0], [640, 480], (CAP, 2)).astype(np.float32)
    for f, n in enumerate(counts):
        desc[f] = mvo_synth.random_descriptors(10 + f, CAP, dup_every=5 + f)
        xy = base[rng.permutation(CAP)] + rng.normal(0, 15, (CAP, 2)).astype(np.float32)
        kpts[f]["x"], kpts[f]["y"] = xy[:, 0], xy[:, 1]
        kpts[f]["class_id"] = -1
        desc[f, n:] = 0xA5                                 # rows beyond the count must not be read
    return desc, kpts, counts


def _host(lib, ctx, desc, kpts, counts, q, t, method, radius):
    import mvo_b200
    n1, n2 = int(counts[q]), int(counts[t])
    d1, d2 = np.ascontiguousarray(desc[q, :n1]), np.ascontiguousarray(desc[t, :n2])
    xy1 = np.ascontiguousarray(np.stack([kpts[q]["x"], kpts[q]["y"]], 1)[:n1], np.float32)
    xy2 = np.ascontiguousarray(np.stack([kpts[t]["x"], kpts[t]["y"]], 1)[:n2], np.float32)
    out, n = np.zeros(max(n1, 1), mvo_b200.DMATCH_DTYPE), C.c_int(0)
    rc = lib.mvo_match_features(ctx, d1.ctypes.data, n1, d2.ctypes.data, n2, method, xy1.ctypes.data, xy2.ctypes.data, radius,
                                out.ctypes.data, C.byref(n))
    return rc, out[: n.value]


@pytest.mark.parametrize("method,radius", [(1, 0.0), (2, 0.0), (3, 50.0)])
def test_emulated_batch_equals_emulated_match_features(lib, ctx, method, radius):
    import mvo_b200
    desc, kpts, counts = _frames()
    pairs = np.array([[0, 1], [4, 0], [1, 1], [0, 3]], np.int32)   # consecutive-like, reversed, a frame with itself, a 1-keypoint train
    out = np.zeros((len(pairs), CAP), mvo_b200.DMATCH_DTYPE)
    n_out = np.full(len(pairs), 12345, np.int32)
    l0 = lib.mvo_kernel_launches(ctx)
    rc = lib.mvo_match_features_batch_dev(ctx, kpts.ctypes.data, desc.ctypes.data, counts.ctypes.data, len(counts), CAP, pairs.ctypes.data,
                                          len(pairs), method, radius, out.ctypes.data, n_out.ctypes.data)
    assert rc == 0, lib.mvo_last_error(ctx)
    assert lib.mvo_kernel_launches(ctx) - l0 == 2
    for p, (q, t) in enumerate(pairs):
        rc_h, ref = _host(lib, ctx, desc, kpts, counts, q, t, method, radius)
        if rc_h != 0:
            assert method == 2 and counts[t] < 2 and n_out[p] == rc_h == -1, (p, rc_h, n_out[p])
            assert not np.frombuffer(out[p].tobytes(), np.uint8).any()     # nothing written for a pair that fails
            continue
        assert n_out[p] == len(ref), (p, n_out[p], len(ref))
        assert out[p, : n_out[p]].tobytes() == ref.tobytes(), p
    assert (n_out[:3] > 0).all()
