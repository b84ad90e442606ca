"""mvo_estimate_relative_poses_batch_dev on the hardware: every pair of a batch byte-identical to
mvo_estimate_relative_poses(calc_homo = 1) on the same points (record, inlier rows, triangulated rows), for both
motion_cam2_to_cam1 values.  This is the tier that sees the device's arithmetic: the combine step (csrc/two_view_batch.cu) must round
as the host code does, which the emulated build cannot show.

- Synthetic batches (tests/relative_poses_batch_cases.py) at full size: 1 / 4096 / 10000 hypotheses, another seed, essential
  thresholds 0.5 / 1 / 3, homography thresholds 1 / 3, eh_ratio_threshold 0.5 and 0.3, fx != fy, n = 6400; general scenes (E),
  planar ones (H, best 1 and 2), a pure rotation for the homography, all-outlier pairs, every invalid-input kind.  Every MVO_OK
  pair with a known motion is checked against it.
- Pairs whose two scores are both 0, so that ratio = 0 / 0.
- The real chain on 16 frames of the bench's room sequence: extract -> match -> relative poses against the per-pair host path on
  the downloaded keypoints and matches.
- Determinism, the launch count for 1, 63 and 500 pairs, and every call-level limit."""
from types import SimpleNamespace

import numpy as np
import pytest

import relative_poses_batch_cases as cases
import two_view_batch_cases as tvb

pytestmark = pytest.mark.gpu

H, W = 480, 640


@pytest.fixture(scope="module")
def gctx(built):
    import mvo_b200
    c = mvo_b200.Context(0, max_keypoints=2000)
    yield c
    c.close()


def _up(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


class DevBatch:
    """A Batch's arrays on the device (torch)."""

    def __init__(self, b):
        import torch
        self.b = b
        self.k, self.c, self.p, self.m, self.n = _up(b.kpts), _up(b.counts), _up(b.pairs), _up(b.matches), _up(b.n_matches)
        torch.cuda.synchronize()


def _run(ctx, d, Km, motion=1, with_pts=True, n_pairs=None):
    """One batch call on sentinel-filled device outputs: (res, inliers, pts3d) as host arrays, launches of the call."""
    import torch
    b = d.b
    n_pairs = b.n_pairs if n_pairs is None else n_pairs
    res, inl, pts = cases.outputs(n_pairs, b.cap)
    d_res, d_inl, d_pts = _up(res), _up(inl), _up(pts)
    torch.cuda.synchronize()
    l0 = ctx.lib.mvo_kernel_launches(ctx.h)
    ctx.estimate_relative_poses_batch_dev(d.k.data_ptr(), d.c.data_ptr(), b.batch, b.cap, d.p.data_ptr(), n_pairs, d.m.data_ptr(),
                                          d.n.data_ptr(), Km, d_res.data_ptr(), d_inl.data_ptr(), d_pts.data_ptr() if with_pts else None,
                                          motion_cam2_to_cam1=motion)
    launches = ctx.lib.mvo_kernel_launches(ctx.h) - l0
    ctx.synchronize()
    out = tuple(t.cpu().numpy().view(a.dtype).reshape(a.shape) for t, a in ((d_res, res), (d_inl, inl), (d_pts, pts)))
    return out, launches


def _mixed(cap, Km, n_big):
    """(specs, truths): general scenes, planar scenes (sideways and backward moves), the pure-rotation scene, a large pair,
    small and all-outlier pairs, every invalid-input kind."""
    specs, truths = [], []

    def add(spec, truth=None):
        specs.append(spec)
        truths.append(truth)
    for s, n in ((10, 1500), (11, 800), (12, 400)):
        add(("points",) + tvb.general_scene(s, n, Km=Km), cases.general_truth(s))
    for s, move in ((11, (0.4, 0.05, 0.05)), (12, (0.4, 0.05, 0.05)), (11, (0.1, 0.1, -0.4)), (12, (0.1, 0.1, -0.4))):
        p1, p2, R, t = cases.planar_scene(s, 900, move=move, Km=Km)
        add(("points", p1, p2), (R, t))
    p1, p2, R, t = cases.rotation_scene(21, 600, Km=Km)
    add(("points", p1, p2), (R, t))
    add(("points",) + tvb.general_scene(14, n_big, noise=0.3, outliers=0.2, Km=Km), cases.general_truth(14))
    g = tvb.general_scene(12, 400, Km=Km)
    add(("points", g[0][:8], g[1][:8]))
    add(("points", g[0][:5], g[1][:5]))
    add(("points",) + tvb.random_pair(15, 300))
    for s in (("bad_frame",), ("count", -1), ("count", cap + 1), ("bad_index",), ("bad_frame",)):
        add(s)
    return specs, truths


FX_FY = np.array([[520.0, 0, 325.1], [0, 480.5, 249.7], [0, 0, 1]])
CONFIGS = [  # (epi_hypotheses, pnp_seed or None, essential threshold, homography threshold, eh_ratio_threshold, K, cap, n of the large pair)
    (4096, None, 1.0, 3.0, 0.5, cases.K, 2000, 2000),
    (4096, None, 1.0, 3.0, 0.3, cases.K, 6400, 6400),
    (1, None, 1.0, 3.0, 0.3, cases.K, 2000, 1200),
    (10000, None, 1.0, 3.0, 0.3, cases.K, 2000, 1200),
    (4096, 0x1234567887654321, 1.0, 3.0, 0.3, cases.K, 2000, 1200),
    (4096, None, 0.5, 1.0, 0.3, cases.K, 2000, 1200),
    (4096, None, 3.0, 1.0, 0.5, cases.K, 2000, 1200),
    (4096, None, 1.0, 3.0, 0.3, FX_FY, 2000, 1200),
]
IDS = ["default", "cap6400", "hyp1", "hyp10000", "seed", "thr0.5-h1", "thr3-h1", "fx!=fy"]


def _set(gctx, **kw):
    import mvo_b200
    default = mvo_b200.default_params()
    keys = ("epi_hypotheses", "pnp_seed", "essential_threshold", "homography_threshold", "eh_ratio_threshold")
    gctx.set_params(**{k: kw.get(k, getattr(default, k)) for k in keys})


@pytest.mark.parametrize("hyp,seed,thr,hthr,eh,Km,cap,n_big", CONFIGS, ids=IDS)
def test_batch_equals_estimate_relative_poses(gctx, hyp, seed, thr, hthr, eh, Km, cap, n_big):
    kw = dict(epi_hypotheses=hyp, essential_threshold=thr, homography_threshold=hthr, eh_ratio_threshold=eh)
    if seed is not None:
        kw["pnp_seed"] = seed
    _set(gctx, **kw)
    try:
        specs, truths = _mixed(cap, Km, n_big)
        b = tvb.Batch(specs, cap, seed=hyp)
        d = DevBatch(b)
        chosen = set()
        for motion in (1, 0):
            refs = cases.references(gctx.lib, gctx.h, b, Km, motion)
            status = [rc for rc, _ in refs]
            assert status[-5:] == [cases.INVALID_ARG] * 5 and status[10] == cases.DEGENERATE, status
            if hyp > 1:
                assert all(rc == 0 for rc in status[:9]), status
                assert refs[7][1]["num"] == 1                       # the pure rotation: no homography solution survives
            for with_pts in (True, False):
                (res, inl, pts), launches = _run(gctx, d, Km, motion, with_pts)
                assert launches == cases.launches_per_call(with_pts)
                for p in range(b.n_pairs):
                    cases.check_pair(b, p, res, inl, pts, refs[p], with_pts)
                    if truths[p] is not None and res[p]["status"] == 0 and hyp > 1 and Km is cases.K:     # E assumes fx = fy
                        planar = 3 <= p <= 6
                        if not planar or res[p]["best"] > 0:        # E on a planar scene is not determined by it
                            cases.check_truth(res[p], *truths[p], motion, dir_tol=0.2 if planar else 0.1)
                        chosen.add((planar, int(res[p]["best"])))
        if hyp > 1 and Km is cases.K:
            assert (False, 0) in chosen, chosen
            if eh < 0.5:
                assert {(True, 1), (True, 2)} <= chosen, chosen
    finally:
        _set(gctx)


def test_nan_ratio_is_the_host_nan(gctx):
    """All-outlier pairs at large thresholds: every essential and homography inlier fails its chi-square test in both
    directions on some pairs, so score_e = score_h = 0 and ratio = 0 / 0; the batch record has the host's NaN bits."""
    _set(gctx, essential_threshold=60.0, homography_threshold=200.0)
    try:
        specs = [("points",) + tvb.random_pair(100 + s, 14) for s in range(256)]
        b = tvb.Batch(specs, 64, seed=2)
        refs = cases.references(gctx.lib, gctx.h, b, cases.K, 1)
        nan = [p for p, (rc, w) in enumerate(refs) if rc == 0 and np.isnan(w["ratio"])]
        assert nan, "no pair with both scores 0"
        for p in nan:
            assert np.frombuffer(refs[p][1]["sol"][-8:], np.uint64)[0] == cases.X86_DEFAULT_NAN
        (res, inl, pts), _ = _run(gctx, DevBatch(b), cases.K)
        for p in range(b.n_pairs):
            cases.check_pair(b, p, res, inl, pts, refs[p])
        assert all(res[p]["ratio"].view(np.uint64) == cases.X86_DEFAULT_NAN for p in nan)
    finally:
        _set(gctx)


CAP = 2001
NF = 16


@pytest.fixture(scope="module")
def chain(gctx):
    """16 frames of the bench's room sequence extracted in one call: device keypoints / counts and their host copies."""
    import torch
    import mvo_b200
    import mvo_synth
    frames, _ = mvo_synth.room_loop_sequence(0, n_frames=NF)
    imgs = np.ascontiguousarray(np.stack([mvo_synth.gray_to_bgr(f) for f in frames]))
    d_img = torch.from_numpy(imgs).cuda()
    d_k = torch.zeros(NF * CAP * 28, dtype=torch.uint8, device="cuda")
    d_d = torch.zeros(NF * CAP * 32, dtype=torch.uint8, device="cuda")
    d_c = torch.zeros(NF, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    gctx.orb_extract_batch_dev(d_img.data_ptr(), NF, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), CAP)
    gctx.synchronize()
    kp = d_k.cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE).reshape(NF, CAP)
    return dict(k=d_k, d=d_d, c=d_c, kp=kp, counts=d_c.cpu().numpy())


def _match(gctx, chain, pairs, method, radius):
    import torch
    n = len(pairs)
    d_p = torch.from_numpy(np.asarray(pairs, np.int32).reshape(-1)).cuda()
    d_m = torch.zeros(n * CAP * 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    gctx.match_features_batch_dev(chain["k"].data_ptr(), chain["d"].data_ptr(), chain["c"].data_ptr(), NF, CAP, d_p.data_ptr(), n, method,
                                  radius, d_m.data_ptr(), d_n.data_ptr())
    return d_p, d_m, d_n


CHAIN_PAIRS = [(i, i + 1) for i in range(NF - 1)] + [(i, i + 4) for i in range(NF - 4)] + [(5, 5), (0, 0)]


@pytest.mark.parametrize("method,radius", [(1, 0.0), (3, 50.0)])
def test_real_chain_equals_per_pair_host_path(gctx, chain, method, radius):
    """What a caller does today: download keypoints and match lists, mvo_estimate_relative_poses(calc_homo = 1) per pair."""
    d_p, d_m, d_n = _match(gctx, chain, CHAIN_PAIRS, method, radius)
    gctx.synchronize()
    n = len(CHAIN_PAIRS)
    d = SimpleNamespace(k=chain["k"], c=chain["c"], p=d_p, m=d_m, n=d_n, b=SimpleNamespace(batch=NF, cap=CAP, n_pairs=n))
    import mvo_b200
    matches = d_m.cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(n, CAP)
    n_m = d_n.cpu().numpy()
    kp = chain["kp"]
    pts_of = lambda q, t, m: (np.stack([kp[q]["x"][m["query_idx"]], kp[q]["y"][m["query_idx"]]], 1).astype(np.float32),
                              np.stack([kp[t]["x"][m["train_idx"]], kp[t]["y"][m["train_idx"]]], 1).astype(np.float32))
    points = [pts_of(q, t, matches[p, :n_m[p]]) for p, (q, t) in enumerate(CHAIN_PAIRS)]
    b = SimpleNamespace(cap=CAP, n_matches=n_m, points=points)          # what check_pair reads of a batch
    for motion in (1, 0):
        (res, inl, pts), _ = _run(gctx, d, cases.K, motion)
        ok = 0
        for p in range(n):
            ref = cases.reference(gctx.lib, gctx.h, points[p][0], points[p][1], cases.K, motion)
            cases.check_pair(b, p, res, inl, pts, ref)
            ok += ref[0] == 0
        assert ok >= n // 2, ok


def test_deterministic_and_constant_launch_count(gctx, chain):
    pairs = [(i % NF, (i * 7 + 1) % NF) for i in range(500)]
    d_p, d_m, d_n = _match(gctx, chain, pairs, 1, 0.0)
    d = SimpleNamespace(k=chain["k"], c=chain["c"], p=d_p, m=d_m, n=d_n, b=SimpleNamespace(batch=NF, cap=CAP, n_pairs=len(pairs)))
    first, l1 = _run(gctx, d, cases.K)
    again, l2 = _run(gctx, d, cases.K)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(first, again))
    assert (first[0]["status"] == 0).sum() > 400
    counts = {l1, l2}
    for n_pairs in (1, 63):
        _, l = _run(gctx, d, cases.K, n_pairs=n_pairs)
        counts.add(l)
        _, l = _run(gctx, d, cases.K, with_pts=False, n_pairs=n_pairs)
        assert l == cases.launches_per_call(False)
    assert counts == {cases.launches_per_call(True)}
    sub, _ = _run(gctx, d, cases.K, n_pairs=63)                         # a prefix of the batch is the same computation
    assert all(s.tobytes() == f[:63].tobytes() for s, f in zip(sub, first))


def test_call_level_limits(gctx):
    import torch
    lib, h = gctx.lib, gctx.h
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    a = buf.data_ptr()
    K = np.ascontiguousarray(cases.K, np.float64)

    def call(kpts=a, counts=a, batch=2, cap=100, pairs=a, n_pairs=1, matches=a, n_matches=a, Km=K, res=a, inl=a, pts=None):
        Kp = None if Km is None else np.ascontiguousarray(Km, np.float64).ctypes.data
        return lib.mvo_estimate_relative_poses_batch_dev(h, kpts, counts, batch, cap, pairs, n_pairs, matches, n_matches, Kp, 1, res, inl, pts)

    for kw in ("kpts", "counts", "pairs", "matches", "n_matches", "res", "inl"):
        assert call(**{kw: None}) == cases.INVALID_ARG, kw
    assert call(Km=None) == cases.INVALID_ARG
    for ij, v in (((0, 0), 0.0), ((1, 1), -1.0), ((2, 2), 0.0)):            # a focal length <= 0, a singular K
        Kb = K.copy()
        Kb[ij] = v
        assert call(Km=Kb) == cases.INVALID_ARG, ij
    assert call(n_pairs=-1) == cases.INVALID_ARG and call(batch=0) == cases.INVALID_ARG and call(cap=0) == cases.INVALID_ARG
    UNSUPPORTED = -5
    assert call(cap=6401) == UNSUPPORTED
    assert call(cap=6400, n_pairs=0) == 0
    assert call(n_pairs=65536) == UNSUPPORTED
    Hy = gctx.params.epi_hypotheses
    assert call(n_pairs=(1 << 22) // Hy + 1) == UNSUPPORTED
    l0 = lib.mvo_kernel_launches(h)
    assert call(n_pairs=0) == 0 and lib.mvo_kernel_launches(h) == l0
    gctx.set_params(epi_hypotheses=1)
    try:
        assert call(n_pairs=65536) == UNSUPPORTED
    finally:
        gctx.set_params(epi_hypotheses=Hy)
    gctx.synchronize()
