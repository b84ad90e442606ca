"""mvo_match_features_batch_dev (csrc/match.cu: match_batch_kernel, csrc/track_filter.cuh: k_match_filter_batch) — geometry::
matchFeatures for a batch of frame pairs, on the device — against mvo_match_features on host copies of the same frames, byte for
byte (query_idx, train_idx, img_idx, distance, list order), and against cv2.BFMatcher for methods 1 / 2.

Frames come from mvo_orb_extract_batch_dev over mvo_synth scenes (the bench's room sequence, dense scenes above the keypoint cap,
a blank frame), with two counts overwritten to 1 and 2 (the counts are inputs).  Adversarial lists put the train-index patterns
of tests/test_track_filter_gpu.py (duplicates, organ pipe, sawtooth ... — the ones that take libstdc++'s introsort to its depth
limit) and duplicated descriptor rows (distance ties) into synthetic frames of the same layout."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CAP = 2001
H, W = 480, 640


@pytest.fixture(scope="module")
def mctx(built):
    import mvo_b200
    c = mvo_b200.Context(0, max_keypoints=2000)
    yield c
    c.close()


class Dev:
    """A batch in the layout of mvo_orb_extract_batch_dev, on the device (torch) and as host copies."""

    def __init__(self, kpts, desc, counts):
        import torch
        import mvo_b200
        self.cap = kpts.shape[1]
        self.batch = len(counts)
        self.kpts_h, self.desc_h, self.counts_h = kpts, desc, np.asarray(counts, np.int32)
        self.k = torch.from_numpy(np.ascontiguousarray(kpts).view(np.uint8).reshape(-1).copy()).cuda()
        self.d = torch.from_numpy(np.ascontiguousarray(desc, np.uint8).reshape(-1).copy()).cuda()
        self.c = torch.from_numpy(self.counts_h.copy()).cuda()
        assert kpts.dtype == mvo_b200.KEYPOINT_DTYPE
        torch.cuda.synchronize()

    def frame(self, f):
        n = int(self.counts_h[f]) if 0 <= f < self.batch else 0
        k = self.kpts_h[f, :n]
        return np.ascontiguousarray(self.desc_h[f, :n]), np.ascontiguousarray(np.stack([k["x"], k["y"]], 1), np.float32)


def _extracted(mctx):
    """Ten extracted frames: six of the bench's room sequence, three dense scenes (far more candidates than the cap), a blank
    frame; frame 4's count is then set to 1 and frame 5's to 2."""
    import torch
    import mvo_b200
    import mvo_synth
    room, _ = mvo_synth.room_loop_sequence(0, n_frames=6)
    gray = list(room) + [mvo_synth.rect_scene(3, W, H), mvo_synth.noise_scene(1, W, H)]
    imgs = [mvo_synth.gray_to_bgr(g) for g in gray] + [mvo_synth.color_scene(2, W, H), np.zeros((H, W, 3), np.uint8)]
    B = len(imgs)
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack(imgs))).cuda()
    d_k = torch.zeros(B * CAP * 28, dtype=torch.uint8, device="cuda")
    d_d = torch.zeros(B * CAP * 32, dtype=torch.uint8, device="cuda")
    d_c = torch.zeros(B, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mctx.orb_extract_batch_dev(d_img.data_ptr(), B, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), CAP)
    mctx.synchronize()
    counts = d_c.cpu().numpy().copy()
    assert counts[9] == 0 and counts[:9].min() > 50, counts
    counts[4], counts[5] = 1, 2
    kp = d_k.cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE).reshape(B, CAP)
    return Dev(kp, d_d.cpu().numpy().reshape(B, CAP, 32), counts)


@pytest.fixture(scope="module")
def extracted(mctx):
    return _extracted(mctx)


def _run(ctx, dev, pairs, method, radius):
    import torch
    import mvo_b200
    pairs = np.asarray(pairs, np.int32).reshape(-1, 2)
    n = len(pairs)
    d_p = torch.from_numpy(pairs.copy()).cuda()
    d_out = torch.zeros(max(n, 1) * dev.cap * 16, dtype=torch.uint8, device="cuda")
    d_n = torch.full((max(n, 1),), 12345, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.match_features_batch_dev(dev.k.data_ptr(), dev.d.data_ptr(), dev.c.data_ptr(), dev.batch, dev.cap, d_p.data_ptr(), n, method,
                                 radius, d_out.data_ptr(), d_n.data_ptr())
    ctx.synchronize()
    return d_out.cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(max(n, 1), dev.cap)[:n], d_n.cpu().numpy()[:n]


def _host(ctx, dev, q, t, method, radius):
    """mvo_match_features(query frame, train frame) on the host copies: (status, matches)."""
    import mvo_b200
    d1, xy1 = dev.frame(q)
    d2, xy2 = dev.frame(t)
    try:
        return 0, ctx.match_features(d1, d2, method, xy1, xy2, radius)
    except mvo_b200.MvoError as e:
        return e.code, None


def _check(ctx, dev, pairs, method, radius, out, n_out):
    nonzero = 0
    for p, (q, t) in enumerate(pairs):
        if not (0 <= q < dev.batch and 0 <= t < dev.batch):
            assert n_out[p] == -1, (p, q, t, n_out[p])
            assert not np.frombuffer(out[p].tobytes(), np.uint8).any()
            continue
        rc, ref = _host(ctx, dev, q, t, method, radius)
        if rc != 0:
            assert rc == -1 and method == 2 and dev.counts_h[t] < 2 and n_out[p] == -1, (p, q, t, rc, n_out[p])
            assert not np.frombuffer(out[p].tobytes(), np.uint8).any()
            continue
        assert n_out[p] == len(ref), (method, radius, p, q, t, n_out[p], len(ref))
        assert out[p, : len(ref)].tobytes() == ref.tobytes(), (method, radius, p, q, t)
        nonzero += len(ref) > 0
    return nonzero


BLANK, ONE, TWO = 9, 4, 5
PAIRS = ([(i, i + 1) for i in range(9)] + [(i + 1, i) for i in range(9)]                       # consecutive, reversed
         + [(0, 1), (0, 1), (6, 6), (7, 7), (0, 0)]                                            # repeated, a frame with itself
         + [(BLANK, 0), (0, BLANK), (BLANK, BLANK), (ONE, 0), (0, ONE), (TWO, 0), (0, TWO), (ONE, ONE), (ONE, TWO), (TWO, ONE)]
         + [(0, 10), (-1, 3), (3, 99999), (10, 10)])                                           # frame indices out of range


@pytest.mark.parametrize("method,radius", [(1, 0.0), (2, 0.0), (3, 0.0), (3, 50.0), (3, 100.0), (3, 1e4)])
def test_batch_equals_match_features_on_extracted_frames(mctx, extracted, method, radius):
    out, n_out = _run(mctx, extracted, PAIRS, method, radius)
    nonzero = _check(mctx, extracted, PAIRS, method, radius, out, n_out)
    assert nonzero >= (0 if (method, radius) == (3, 0.0) else 10), nonzero
    if method == 2:                                   # a 1-keypoint train fails, a 2-keypoint train does not
        assert n_out[PAIRS.index((3, ONE))] == -1 and n_out[PAIRS.index((ONE, TWO))] >= 0


def test_lowe_ratio_and_xiang_gao_ratio_from_the_context(mctx, extracted):
    """The thresholds are the context's parameters, as for mvo_match_features."""
    pairs = [(i, i + 1) for i in range(8)]
    mctx.set_params(lowe_ratio=0.8, xiang_gao_ratio=3.0)
    try:
        for method in (1, 2):
            out, n_out = _run(mctx, extracted, pairs, method, 0.0)
            _check(mctx, extracted, pairs, method, 0.0, out, n_out)
    finally:
        mctx.set_params(lowe_ratio=1.0, xiang_gao_ratio=2.0)


def _cv2_reference(d1, d2, method):
    """matchFeatures' tail (feature_match.cpp:179-217, 229) over cv2.BFMatcher's own matches; removeDuplicatedMatches through the
    oracle's libstdc++ std::sort."""
    import cv2
    import mvo_b200
    from oracle import oracle_lib
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    rows = []
    if method == 1:
        ms = bf.match(d1, d2)
        min_dis = min([m.distance for m in ms], default=9999999.0)
        thr = max(float(np.float32(min_dis * 2.0)), 30.0)
        rows = [(m.queryIdx, m.trainIdx, m.imgIdx, m.distance) for m in ms if m.distance < thr]
    else:
        for k in bf.knnMatch(d1, d2, k=2):
            if k[0].distance < 1.0 * k[1].distance:
                rows.append((k[0].queryIdx, k[0].trainIdx, k[0].imgIdx, k[0].distance))
    return oracle_lib.remove_duplicated_matches(np.array(rows, mvo_b200.DMATCH_DTYPE))


def test_methods_1_and_2_agree_with_cv2_bfmatcher(mctx, extracted):
    from conftest import have_cv2
    if not have_cv2():
        pytest.skip("cv2 not importable")
    pairs = [(0, 1), (2, 3), (6, 7), (8, 0), (7, 6)]
    for method in (1, 2):
        out, n_out = _run(mctx, extracted, pairs, method, 0.0)
        for p, (q, t) in enumerate(pairs):
            ref = _cv2_reference(extracted.frame(q)[0], extracted.frame(t)[0], method)
            assert n_out[p] == len(ref) > 0 and out[p, : len(ref)].tobytes() == ref.tobytes(), (method, q, t)


def _synthetic(rng, n, nk, patterns, cap, dup_train=False):
    """Frame 0: nk train descriptors (distinct rows, or with duplicated rows when dup_train), frame 1 + i: n queries whose row j is
    train row patterns[i][j] with a few bits flipped — query j's nearest train is that row (the lowest index of its copies) — so
    the match list carries the train-index pattern into removeDuplicatedMatches.  All keypoints in a 200 px square."""
    import mvo_b200
    B = 1 + len(patterns)
    desc = np.zeros((B, cap, 32), np.uint8)
    tr = rng.integers(0, 256, (nk, 32), dtype=np.uint8)
    if dup_train:
        tr[1::3] = tr[0::3][: len(tr[1::3])]
    desc[0, :nk] = tr
    for i, pat in enumerate(patterns):
        rows = tr[np.asarray(pat) % nk].copy()
        flip = rng.integers(0, 256, (len(rows), 32), dtype=np.uint8) * (rng.random((len(rows), 32)) < 0.02)
        desc[1 + i, : len(rows)] = rows ^ flip.astype(np.uint8)
    kp = np.zeros((B, cap), mvo_b200.KEYPOINT_DTYPE)
    kp["x"] = rng.uniform(100, 300, (B, cap))
    kp["y"] = rng.uniform(100, 300, (B, cap))
    kp["class_id"] = -1
    counts = [nk] + [len(p) for p in patterns]
    return Dev(kp, desc, counts)


@pytest.mark.parametrize("n,nk,dup", [(2001, 1003, False), (2001, 2001, True), (517, 300, False), (33, 17, True)])
def test_adversarial_train_patterns_equal_host_std_sort(mctx, n, nk, dup):
    from test_track_filter_gpu import _train_patterns
    rng = np.random.default_rng(n + nk)
    pats = [p for _, p in _train_patterns(rng, n, nk)]
    dev = _synthetic(rng, n, nk, pats, CAP, dup)
    pairs = [(1 + i, 0) for i in range(len(pats))] + [(0, 1 + i) for i in range(len(pats))]
    for method, radius in ((1, 0.0), (2, 0.0), (3, 1e4)):
        out, n_out = _run(mctx, dev, pairs, method, radius)
        assert _check(mctx, dev, pairs, method, radius, out, n_out) >= len(pats)


def test_cap_limit(mctx):
    import mvo_b200
    from test_track_filter_gpu import _train_patterns
    rng = np.random.default_rng(8192)
    n = 8192
    pats = [p for name, p in _train_patterns(rng, n, n) if name in ("random", "organ-pipe", "heavy-dup")]
    dev = _synthetic(rng, n, n, pats, 8192)
    pairs = [(1, 0), (2, 0), (3, 0), (0, 1)]
    for method, radius in ((1, 0.0), (2, 0.0), (3, 1e4)):
        out, n_out = _run(mctx, dev, pairs, method, radius)
        assert _check(mctx, dev, pairs, method, radius, out, n_out) >= 3
    big = Dev(np.zeros((1, 8193), mvo_b200.KEYPOINT_DTYPE), np.zeros((1, 8193, 32), np.uint8), [0])
    with pytest.raises(mvo_b200.MvoError) as e:
        _run(mctx, big, [(0, 0)], 1, 0.0)
    assert e.value.code == -5


def test_argument_errors(mctx, extracted):
    lib, h, dv = mctx.lib, mctx.h, extracted
    p = np.zeros(2, np.int32)
    args = lambda **kw: dict(dict(k=dv.k.data_ptr(), d=dv.d.data_ptr(), c=dv.c.data_ptr(), b=dv.batch, cap=dv.cap, p=p.ctypes.data, n=1, m=1,
                                  r=0.0, o=dv.d.data_ptr(), no=dv.c.data_ptr()), **kw)

    def call(a):
        return lib.mvo_match_features_batch_dev(h, C.c_void_p(a["k"]), C.c_void_p(a["d"]), C.c_void_p(a["c"]), a["b"], a["cap"],
                                                C.c_void_p(a["p"]), a["n"], a["m"], C.c_float(a["r"]), C.c_void_p(a["o"]),
                                                C.c_void_p(a["no"]))
    for bad in (dict(m=0), dict(m=4), dict(n=-1), dict(d=None), dict(c=None), dict(p=None), dict(o=None), dict(no=None),
                dict(m=3, k=None), dict(b=0), dict(cap=0)):
        assert call(args(**bad)) == -1, bad
    assert call(args(cap=8193)) == -5
    assert call(args(n=0)) == 0                       # nothing to do, nothing launched or read


def test_deterministic_and_launch_count_independent_of_pairs(mctx, extracted):
    pairs64 = [(i % 9, (i + 1) % 9) for i in range(64)]
    for method, radius in ((1, 0.0), (2, 0.0), (3, 100.0)):
        a = _run(mctx, extracted, pairs64, method, radius)
        b = _run(mctx, extracted, pairs64, method, radius)
        assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
        deltas = []
        for pairs in ([(0, 1)], pairs64):
            _run(mctx, extracted, pairs, method, radius)             # scratch buffers at their size
            l0 = mctx.kernel_launches
            _run(mctx, extracted, pairs, method, radius)
            deltas.append(mctx.kernel_launches - l0)
        assert deltas[0] == deltas[1] == 2, deltas
