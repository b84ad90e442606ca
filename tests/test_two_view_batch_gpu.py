"""mvo_esti_motion_by_essential_batch_dev (csrc/epipolar_kernels.cuh: k_epi_gather ... k_triangulate_batch) on the hardware:
every pair of a batch byte-identical to the per-pair path on the same points.

- Synthetic batches (tests/two_view_batch_cases.py) at full size against mvo_estimate_relative_poses(calc_homo = 0): the default
  4096 hypotheses, 1 and 10000, a non-default seed, thresholds 0.5 / 1 / 3, fx != fy, n up to 6400 (the consensus kernel's
  shared-memory opt-in), failed pairs that must leave their output slots alone.
- The real chain: 16 frames of the bench's room sequence through mvo_orb_extract_batch_dev and mvo_match_features_batch_dev
  (methods 1 and 3), pairs (i, i+1), (i, i+4) and a frame with itself, against mvo_esti_motion_by_essential followed by
  mvo_do_triangulation on the downloaded keypoints and matches.
- Determinism, the launch count, and every call-level limit."""
from types import SimpleNamespace

import numpy as np
import pytest

import two_view_batch_cases as cases

pytestmark = pytest.mark.gpu

H, W = 480, 640


@pytest.fixture(scope="module")
def gctx(built):
    import mvo_b200
    c = mvo_b200.Context(0, max_keypoints=2000)
    yield c
    c.close()


class DevBatch:
    """A Batch's arrays on the device (torch)."""

    def __init__(self, b):
        import torch
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
        self.b = b
        self.k, self.c, self.p, self.m, self.n = up(b.kpts), up(b.counts), up(b.pairs), up(b.matches), up(b.n_matches)
        torch.cuda.synchronize()


def _run(ctx, d, Km, threshold, with_pts=True, n_pairs=None):
    """One batch call on sentinel-filled device outputs: (res, inliers, pts3d) as host arrays, launches of the call."""
    import torch
    b = d.b
    n_pairs = b.n_pairs if n_pairs is None else n_pairs
    res, inl, pts = cases.outputs(n_pairs, b.cap)
    d_res, d_inl, d_pts = (torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda() for a in (res, inl, pts))
    torch.cuda.synchronize()
    l0 = ctx.lib.mvo_kernel_launches(ctx.h)
    ctx.esti_motion_by_essential_batch_dev(d.k.data_ptr(), d.c.data_ptr(), b.batch, b.cap, d.p.data_ptr(), n_pairs, d.m.data_ptr(),
                                           d.n.data_ptr(), Km, threshold, d_res.data_ptr(), d_inl.data_ptr(),
                                           d_pts.data_ptr() if with_pts else None)
    launches = ctx.lib.mvo_kernel_launches(ctx.h) - l0
    ctx.synchronize()
    out = tuple(t.cpu().numpy().view(a.dtype).reshape(a.shape) for t, a in ((d_res, res), (d_inl, inl), (d_pts, pts)))
    return out, launches


def _mixed(cap, Km, n_big):
    g = [cases.general_scene(s, n, Km=Km) for s, n in ((10, 1500), (11, 800), (12, 400))]
    planar = cases.general_scene(13, 900, outliers=0.1, planar=True, Km=Km)
    clean = cases.general_scene(14, n_big, noise=0.3, outliers=0.2, Km=Km)
    return [("points",) + g[0], ("points",) + g[1], ("points",) + planar, ("points",) + clean,
            ("points", g[2][0][:8], g[2][1][:8]), ("points", g[2][0][:9], g[2][1][:9]),
            ("points",) + cases.random_pair(15, 300), ("points", g[2][0][:7], g[2][1][:7]),
            ("bad_frame",), ("count", -1), ("count", cap + 1), ("bad_index",), ("bad_frame",), ("points",) + g[2]]


FX_FY = np.array([[520.0, 0, 325.1], [0, 480.5, 249.7], [0, 0, 1]])
CONFIGS = [  # (epi_hypotheses, pnp_seed or None, threshold, K, cap, n of the large pair)
    (4096, None, 1.0, cases.K, 2000, 2000),
    (4096, None, 1.0, cases.K, 6400, 6400),
    (1, None, 1.0, cases.K, 2000, 1200),
    (10000, None, 1.0, cases.K, 2000, 1200),
    (4096, 0x1234567887654321, 1.0, cases.K, 2000, 1200),
    (4096, None, 0.5, cases.K, 2000, 1200),
    (4096, None, 3.0, cases.K, 2000, 1200),
    (4096, None, 1.0, FX_FY, 2000, 1200),
]


@pytest.mark.parametrize("hyp,seed,thr,Km,cap,n_big", CONFIGS, ids=["default", "cap6400", "hyp1", "hyp10000", "seed", "thr0.5", "thr3", "fx!=fy"])
def test_batch_equals_estimate_relative_poses(gctx, hyp, seed, thr, Km, cap, n_big):
    import mvo_b200
    default = mvo_b200.default_params()
    gctx.set_params(epi_hypotheses=hyp, pnp_seed=default.pnp_seed if seed is None else seed, essential_threshold=thr)
    try:
        b = cases.Batch(_mixed(cap, Km, n_big), cap, seed=hyp)
        refs = cases.references(gctx.lib, gctx.h, b, Km)
        assert sum(rc == 0 for rc, _ in refs) >= (3 if hyp == 1 else 6), [rc for rc, _ in refs]
        assert [rc for rc, _ in refs[8:13]] == [cases.INVALID_ARG] * 5
        d = DevBatch(b)
        for with_pts in (True, False):
            (res, inl, pts), launches = _run(gctx, d, Km, thr, with_pts)
            assert launches == cases.launches_per_call(with_pts)
            for p in range(b.n_pairs):
                cases.check_pair(b, p, res, inl, pts, refs[p], with_pts)
    finally:
        gctx.set_params(epi_hypotheses=default.epi_hypotheses, pnp_seed=default.pnp_seed, essential_threshold=default.essential_threshold)


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


def _per_pair(gctx, kp, counts, q, t, m):
    """The host path a caller has today: pts from the downloaded keypoints and matches, mvo_esti_motion_by_essential, then
    mvo_do_triangulation on pixel2CamNormPlane points."""
    import mvo_b200
    K = cases.K
    p1 = np.ascontiguousarray(np.stack([kp[q]["x"][m["query_idx"]], kp[q]["y"][m["query_idx"]]], 1), np.float32)
    p2 = np.ascontiguousarray(np.stack([kp[t]["x"][m["train_idx"]], kp[t]["y"][m["train_idx"]]], 1), np.float32)
    try:
        E, R, t_, inl = gctx.esti_motion_by_essential(p1, p2, K, 1.0)
    except mvo_b200.MvoError as e:
        return e.code, None
    norm = lambda p: np.stack([((p[:, 0].astype(np.float64) - K[0, 2]) / K[0, 0]).astype(np.float32),
                               ((p[:, 1].astype(np.float64) - K[1, 2]) / K[1, 1]).astype(np.float32)], 1)
    pts = gctx.do_triangulation(norm(p1), norm(p2), R, t_, inl)
    return 0, dict(n_inliers=len(inl), E=np.ascontiguousarray(E, np.float64).reshape(-1), R=np.ascontiguousarray(R, np.float64).reshape(-1),
                   t=np.ascontiguousarray(t_, np.float64).reshape(-1), inliers=np.asarray(inl, np.int32), pts3d=np.asarray(pts, np.float32))


CHAIN_PAIRS = [(i, i + 1) for i in range(NF - 1)] + [(i, i + 4) for i in range(NF - 4)] + [(5, 5), (0, 0)]


@pytest.mark.parametrize("method,radius", [(1, 0.0), (3, 50.0)])
def test_real_chain_equals_per_pair_host_path(gctx, chain, method, radius):
    import torch
    import mvo_b200
    d_p, d_m, d_n = _match(gctx, chain, CHAIN_PAIRS, method, radius)
    n = len(CHAIN_PAIRS)
    res, inl, pts = cases.outputs(n, CAP)
    d_res, d_inl, d_pts = (torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda() for a in (res, inl, pts))
    torch.cuda.synchronize()
    gctx.esti_motion_by_essential_batch_dev(chain["k"].data_ptr(), chain["c"].data_ptr(), NF, CAP, d_p.data_ptr(), n, d_m.data_ptr(),
                                            d_n.data_ptr(), cases.K, 1.0, d_res.data_ptr(), d_inl.data_ptr(), d_pts.data_ptr())
    gctx.synchronize()
    res = d_res.cpu().numpy().view(mvo_b200.TWO_VIEW_RESULT_DTYPE)
    inl = d_inl.cpu().numpy().view(np.int32).reshape(n, CAP)
    pts = d_pts.cpu().numpy().view(np.float32).reshape(n, CAP, 3)
    matches = d_m.cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(n, CAP)
    n_m = d_n.cpu().numpy()
    ok = 0
    b = SimpleNamespace(cap=CAP, n_matches=n_m)           # what check_pair reads of a batch
    for p, (q, t) in enumerate(CHAIN_PAIRS):
        ref = _per_pair(gctx, chain["kp"], chain["counts"], q, t, matches[p, :n_m[p]])
        cases.check_pair(b, p, res, inl, pts, ref)
        ok += ref[0] == 0
    assert ok >= len(CHAIN_PAIRS) // 2, ok


def test_deterministic_and_constant_launch_count(gctx, chain):
    import torch
    pairs = [(i % NF, (i * 7 + 1) % NF) for i in range(500)]
    d_p, d_m, d_n = _match(gctx, chain, pairs, 1, 0.0)
    _Dev = SimpleNamespace(k=chain["k"], c=chain["c"], p=d_p, m=d_m, n=d_n, b=SimpleNamespace(batch=NF, cap=CAP, n_pairs=len(pairs)))
    first, l1 = _run(gctx, _Dev, cases.K, 1.0)
    again, l2 = _run(gctx, _Dev, cases.K, 1.0)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(first, again))
    assert (first[0]["status"] == 0).sum() > 400
    counts = {l1, l2}
    for n_pairs in (1, 63):
        _, l = _run(gctx, _Dev, cases.K, 1.0, n_pairs=n_pairs)
        counts.add(l)
        _, l = _run(gctx, _Dev, cases.K, 1.0, with_pts=False, n_pairs=n_pairs)
        assert l == cases.launches_per_call(False)
    assert counts == {cases.launches_per_call(True)}
    # a prefix of the batch is the same computation
    sub, _ = _run(gctx, _Dev, cases.K, 1.0, n_pairs=63)
    assert sub[0].tobytes() == first[0][:63].tobytes() and sub[1].tobytes() == first[1][:63].tobytes()
    torch.cuda.synchronize()


def test_call_level_limits(gctx):
    import torch
    lib, h = gctx.lib, gctx.h
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    a = buf.data_ptr()
    K = np.ascontiguousarray(cases.K, np.float64)

    def call(kpts=a, counts=a, batch=2, cap=100, pairs=a, n_pairs=1, matches=a, n_matches=a, Km=K, thr=1.0, res=a, inl=a, pts=None):
        Kp = None if Km is None else np.ascontiguousarray(Km, np.float64).ctypes.data
        return lib.mvo_esti_motion_by_essential_batch_dev(h, kpts, counts, batch, cap, pairs, n_pairs, matches, n_matches, Kp, thr, res, inl, pts)

    for kw in ("kpts", "counts", "pairs", "matches", "n_matches", "res", "inl"):
        assert call(**{kw: None}) == cases.INVALID_ARG, kw
    assert call(Km=None) == cases.INVALID_ARG
    for ij, v in (((0, 0), 0.0), ((1, 1), -1.0)):
        Kb = K.copy()
        Kb[ij] = v
        assert call(Km=Kb) == cases.INVALID_ARG, ij
    assert call(thr=0.0) == cases.INVALID_ARG and call(thr=-1.0) == cases.INVALID_ARG and call(thr=float("nan")) == cases.INVALID_ARG
    assert call(n_pairs=-1) == cases.INVALID_ARG and call(batch=0) == cases.INVALID_ARG and call(cap=0) == cases.INVALID_ARG
    UNSUPPORTED = -5
    assert call(cap=6401) == UNSUPPORTED
    assert call(cap=6400, n_pairs=0) == 0
    assert call(n_pairs=65536) == UNSUPPORTED
    H = gctx.params.epi_hypotheses
    assert call(n_pairs=(1 << 22) // H + 1) == UNSUPPORTED
    l0 = lib.mvo_kernel_launches(h)
    assert call(n_pairs=0) == 0 and lib.mvo_kernel_launches(h) == l0
    gctx.set_params(epi_hypotheses=1)
    try:
        assert call(n_pairs=65536) == UNSUPPORTED
    finally:
        gctx.set_params(epi_hypotheses=H)
    gctx.synchronize()
