"""TEST INFRASTRUCTURE: fabricated jobs for mvo_vo_pnp_batch_dev, written directly in mvo_vo_map_matches_batch_dev's row layout
(job j's matches, 3D points and pixels at + j * cap), and the references the batch is held to.

Per job the batch must return:
- best, n_inliers, the inlier list and Rt BYTE-IDENTICAL to the test entry mvo_test_pnp_dev (the tracker's device-resident PnP)
  on the job's cap rows with the job's count (0 below min_pnp_points);
- the consensus set of mvo_solve_pnp_ransac on the job's pairs alone, and its pose within 1e-12 (bit-identical when the single
  call's refit launches the same k_ba_pose kernel as the batch's, which runs on cap edge slots);
- pnp_ok of the state machine's composition (rvec -> R -> inverse -> jump rule, vo_pipeline.cpp), with the margin of the jump
  distance to max_dist_to_prev asserted, and its T_w_c within 1e-10 (the Rodrigues round trip re-orthonormalises R);
- T_w_c byte-identical to the tail restated here over Python floats from Rt (host operation order), d_kept = the matches at
  the inlier indices, and sentinel bytes past every count.  A failed job writes its status only."""
import ctypes as C
import math
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "monocular-visual-odometry_b200" / "python"))
import mvo_b200  # noqa: E402

OK, INVALID_ARG, UNSUPPORTED, DEGENERATE = 0, -1, -5, -6
SENTINEL = 0xA7
K = np.array([[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1.0]])
MIN_PTS = 8                                  # min_pnp_points of every case: 4, 7 and 8 pairs are then three different cases
MAX_DIST = 0.3
MM = mvo_b200.MAP_MATCHES_RESULT_DTYPE
OUT = mvo_b200.VO_PNP_RESULT_DTYPE
DM = mvo_b200.DMATCH_DTYPE
PF_T = 512
LAUNCHES = 5


def refit_kernel(n_upper, csize):
    """The pose LM the refit launches for n_upper edge slots: cached while n_upper <= cluster x 512 threads."""
    return "cached" if n_upper <= csize * PF_T else "uncached"


def rod(w):
    w = np.asarray(w, np.float64)
    th = np.linalg.norm(w)
    if th < 1e-15:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * Kx + (1 - math.cos(th)) * Kx @ Kx


def T_w_c_of(R, t):
    T = np.eye(4)
    T[:3, :3] = R.T
    T[:3, 3] = -R.T @ t
    return T


def track_params(lib, min_pts=MIN_PTS, max_dist=MAX_DIST):
    tp = mvo_b200.TrackParams()
    lib.mvo_default_track_params(C.byref(tp))
    tp.min_pnp_points, tp.max_dist_to_prev = min_pts, max_dist
    return tp


class Scene:
    """Jobs of one batch.  kinds: the case each job covers; n_bad failed jobs at the end."""

    def __init__(self, cap, seed=0):
        assert cap >= 64
        self.cap = cap
        rng = np.random.default_rng(seed)
        kinds = [("empty", 0), ("four", 4), ("below_min", MIN_PTS - 1), ("at_min", MIN_PTS), ("full", cap), ("half", cap // 2 + 3),
                 ("outliers", min(cap, 40)), ("coincident", 20), ("planar", cap // 2), ("jump", cap // 3), ("repeat", cap),
                 ("status", 30), ("n_neg", -1), ("n_over", cap + 1), ("prev_nan", 30), ("prev_inf", 30)]
        self.kinds = [k for k, _ in kinds]
        self.n_bad = 5
        n_jobs = len(kinds)
        self.n_jobs = n_jobs
        self.mm = np.zeros(n_jobs, MM)
        self.matches = np.full(n_jobs * cap * DM.itemsize, SENTINEL, np.uint8).view(DM).reshape(n_jobs, cap)
        self.p3 = np.full(n_jobs * cap * 12, SENTINEL, np.uint8).view(np.float32).reshape(n_jobs, cap, 3)
        self.p2 = np.full(n_jobs * cap * 8, SENTINEL, np.uint8).view(np.float32).reshape(n_jobs, cap, 2)
        self.T_prev = np.zeros((n_jobs, 16))
        for j, (kind, n) in enumerate(kinds):
            if kind == "repeat":
                src = self.kinds.index("full")
                self.mm[j], self.matches[j], self.p3[j], self.p2[j], self.T_prev[j] = (self.mm[src], self.matches[src], self.p3[src],
                                                                                       self.p2[src], self.T_prev[src])
                continue
            R = rod(rng.normal(0, 0.3, 3))
            t = rng.normal(0, 0.3, 3)
            m = max(0, min(n, cap))
            if kind == "planar":                                       # world points on the plane z = 0, seen from 5 units away
                R, t = rod(rng.normal(0, 0.1, 3)), np.array([0.1, -0.1, 5.0])
                P = np.stack([rng.uniform(-3, 3, m), rng.uniform(-2, 2, m), np.zeros(m)], 1)
            else:
                pc = np.stack([rng.uniform(-2, 2, m), rng.uniform(-1.5, 1.5, m), rng.uniform(2, 8, m)], 1)
                P = (pc - t) @ R
            if kind == "coincident":
                P[:] = P[0]
            P = P.astype(np.float32)
            pc = P.astype(np.float64) @ R.T + t
            uv = np.stack([K[0, 0] * pc[:, 0] / pc[:, 2] + K[0, 2], K[1, 1] * pc[:, 1] / pc[:, 2] + K[1, 2]], 1)
            uv += rng.normal(0, 0.5, uv.shape)
            outl = {"outliers": 1.0, "full": 0.3, "half": 0.2, "jump": 0.25}.get(kind, 0.0)
            bad = rng.random(m) < outl
            uv[bad] = np.stack([rng.uniform(0, 640, bad.sum()), rng.uniform(0, 480, bad.sum())], 1)
            self.p3[j, :m], self.p2[j, :m] = P, uv.astype(np.float32)
            mt = self.matches[j, :m]
            mt["query_idx"], mt["train_idx"] = rng.permutation(max(m, 1))[:m], rng.integers(0, 2000, m)
            mt["img_idx"], mt["distance"] = 0, rng.integers(0, 64, m).astype(np.float32)
            Tp = T_w_c_of(R, t)
            Tp[:3, 3] += (1.0, 0.0, 0.0) if kind == "jump" else rng.normal(0, 0.03, 3)
            self.T_prev[j] = Tp.ravel()
            self.mm[j] = (OK, m + 5, n, 0)
        self.mm[self.kinds.index("status")]["status"] = UNSUPPORTED
        self.T_prev[self.kinds.index("prev_nan"), 7] = np.nan
        self.T_prev[self.kinds.index("prev_inf"), 15] = -np.inf
        assert self.kinds[-self.n_bad:] == ["status", "n_neg", "n_over", "prev_nan", "prev_inf"]
        self.want_status = [OK] * (n_jobs - self.n_bad) + [UNSUPPORTED, INVALID_ARG, INVALID_ARG, INVALID_ARG, INVALID_ARG]

    def subset(self, idx):
        """The jobs idx (repeats allowed) as a new batch of the same cap."""
        s = object.__new__(Scene)
        s.cap, idx = self.cap, np.asarray(idx)
        s.kinds = [self.kinds[i] for i in idx]
        s.n_jobs = len(idx)
        s.mm, s.matches, s.p3, s.p2 = (np.ascontiguousarray(a[idx]) for a in (self.mm, self.matches, self.p3, self.p2))
        s.T_prev = np.ascontiguousarray(self.T_prev[idx])
        s.want_status = [self.want_status[i] for i in idx]
        s.n_bad = sum(st != OK for st in s.want_status)
        return s


def outputs(n_jobs, cap, kept=True):
    out = np.full(max(n_jobs, 1) * OUT.itemsize, SENTINEL, np.uint8).view(OUT)
    inl = np.full(max(n_jobs, 1) * cap, SENTINEL * 0x01010101 - (1 << 32), np.int32)
    kp = np.full(max(n_jobs, 1) * cap * DM.itemsize, SENTINEL, np.uint8).view(DM) if kept else None
    return out, inl, kp


def call(lib, h, s, tp, ptr=lambda a: a.ctypes.data, outs=None, n_jobs=None, cap=None, Kp=None):
    """One mvo_vo_pnp_batch_dev call on the scene's rows (ptr maps a host array to the pointer the call gets)."""
    n_jobs = s.n_jobs if n_jobs is None else n_jobs
    cap = s.cap if cap is None else cap
    outs = outputs(s.n_jobs, s.cap) if outs is None else outs
    out, inl, kp = outs
    Kh = np.ascontiguousarray(K if Kp is None else Kp, np.float64)
    opt = lambda a: None if a is None else ptr(a)                    # noqa: E731
    rc = lib.mvo_vo_pnp_batch_dev(h, opt(s.mm), opt(s.matches), opt(s.p3), opt(s.p2), n_jobs, cap, opt(s.T_prev), Kh.ctypes.data,
                                  C.byref(tp) if tp is not None else None, opt(out), opt(inl), opt(kp))
    return rc, outs


# ---- references --------------------------------------------------------------------------------------------------------------
def _test_entry(lib):
    f = lib.mvo_test_pnp_dev
    vp = C.c_void_p
    f.restype = C.c_int
    f.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    return f


def count_of(s, j, tp):
    n = int(s.mm[j]["n_matches"])
    return n if n >= tp.min_pnp_points else 0


def single_dev(lib, h, s, j, count, H):
    """mvo_test_pnp_dev on job j's cap rows with the given count: pose_io, out_i and the inlier list."""
    pose_io, out_i = np.full(12, np.nan), np.full(4, -7, np.int32)
    inl, counts = np.full(s.cap, -7, np.int32), np.full(H, -7, np.int32)
    p3, p2 = np.ascontiguousarray(s.p3[j]), np.ascontiguousarray(s.p2[j])
    Kh = np.ascontiguousarray(K)
    rc = _test_entry(lib)(h, p3.ctypes.data, p2.ctypes.data, s.cap, count, Kh.ctypes.data, None, None, pose_io.ctypes.data,
                          out_i.ctypes.data, inl.ctypes.data, counts.ctypes.data)
    assert rc == OK, rc
    return dict(pose_io=pose_io, out_i=out_i, inl=inl[: max(int(out_i[0]), 0)].copy())


def single_host(lib, h, s, j, n):
    """mvo_solve_pnp_ransac on job j's n pairs alone."""
    p3, p2 = np.ascontiguousarray(s.p3[j, :n]), np.ascontiguousarray(s.p2[j, :n])
    rvec, tvec, inl = np.full(3, np.nan), np.full(3, np.nan), np.full(n, -7, np.int32)
    ni = C.c_int(n)
    Kh = np.ascontiguousarray(K)
    rc = lib.mvo_solve_pnp_ransac(h, p3.ctypes.data, p2.ctypes.data, n, Kh.ctypes.data, rvec.ctypes.data, tvec.ctypes.data,
                                  inl.ctypes.data, C.byref(ni))
    return dict(rc=rc, rvec=rvec, tvec=tvec, inl=inl[: ni.value].copy() if rc == OK else inl[:0])


def tail(Rt, T_prev, max_dist, model):
    """k_pnp_batch_tail over Python floats: T_w_c = [R|t]^-1 in inv_rigid's operation order, trans_dist, the jump rule."""
    P, Tp = [float(x) for x in Rt], [float(x) for x in T_prev]
    if not model:
        return 0, np.array(Tp), None
    T = [0.0] * 16
    for i in range(3):
        for c in range(3):
            T[i * 4 + c] = P[c * 3 + i]
        T[i * 4 + 3] = -((P[i] * P[9] + P[3 + i] * P[10]) + P[6 + i] * P[11])
    T[15] = 1.0
    dx, dy, dz = T[3] - Tp[3], T[7] - Tp[7], T[11] - Tp[11]
    d = math.sqrt((dx * dx + dy * dy) + dz * dz)
    ok = 0 if d >= max_dist else 1
    return ok, (np.array(T) if ok else np.array(Tp)), d


def reference(lib, h, s, j, tp, H):
    """The record, inlier list and kept matches job j must get (None for a failed job), from mvo_test_pnp_dev."""
    if s.want_status[j] != OK:
        return None
    d = single_dev(lib, h, s, j, count_of(s, j, tp), H)
    rec = np.zeros(1, OUT)[0]
    rec["status"], rec["n_matches"] = OK, s.mm[j]["n_matches"]
    rec["n_inliers"], rec["best"], rec["Rt"] = d["out_i"][0], d["out_i"][1], d["pose_io"]
    ok, T, dist = tail(d["pose_io"], s.T_prev[j], tp.max_dist_to_prev, d["out_i"][1] >= 0)
    rec["pnp_ok"], rec["T_w_c"] = ok, T
    return dict(rec=rec, inl=d["inl"], kept=s.matches[j][d["inl"]], dist=dist)


def views(outs, n_jobs, cap):
    out, inl, kp = outs
    return out, inl.reshape(-1, cap), None if kp is None else kp.reshape(-1, cap)


def check_exact(ref, outs, s, j):
    out, inl, kp = views(outs, s.n_jobs, s.cap)
    o = out[j]
    if ref is None:                                                  # status only
        assert o["status"] == s.want_status[j], (j, s.kinds[j], o["status"])
        assert (o.tobytes()[4:] == bytes([SENTINEL]) * (OUT.itemsize - 4)), (j, s.kinds[j])
        assert (inl[j].view(np.uint8) == SENTINEL).all() and (kp is None or (kp[j].view(np.uint8) == SENTINEL).all()), j
        return
    assert o.tobytes() == ref["rec"].tobytes(), (j, s.kinds[j], o, ref["rec"])
    ni = int(ref["rec"]["n_inliers"])
    assert inl[j, :ni].tobytes() == ref["inl"].tobytes(), (j, s.kinds[j])
    assert (inl[j, ni:].view(np.uint8) == SENTINEL).all(), (j, s.kinds[j])
    if kp is not None:
        assert kp[j, :ni].tobytes() == ref["kept"].tobytes(), (j, s.kinds[j])
        assert (kp[j, ni:].view(np.uint8) == SENTINEL).all(), (j, s.kinds[j])


def check_host(lib, h, s, j, tp, outs, csize):
    """Job j against mvo_solve_pnp_ransac on its pairs alone and the state machine's pose composition."""
    from oracle import pnp_oracle as po
    if s.want_status[j] != OK:
        return
    o = views(outs, s.n_jobs, s.cap)[0][j]
    n = count_of(s, j, tp)
    if n < 4:
        assert o["best"] == -1 and o["n_inliers"] == 0 and o["pnp_ok"] == 0, (j, s.kinds[j])
        assert o["T_w_c"].tobytes() == s.T_prev[j].tobytes()
        return
    r = single_host(lib, h, s, j, n)
    if r["rc"] == DEGENERATE:
        assert o["best"] == -1 and o["n_inliers"] == 0 and o["pnp_ok"] == 0 and o["T_w_c"].tobytes() == s.T_prev[j].tobytes()
        return
    assert r["rc"] == OK, r["rc"]
    ni = int(o["n_inliers"])
    assert np.array_equal(views(outs, s.n_jobs, s.cap)[1][j, :ni], r["inl"]), (j, s.kinds[j])
    R = po.rodrigues(r["rvec"])
    assert np.abs(o["Rt"][:9] - R.ravel()).max() < 1e-10
    dt = np.abs(o["Rt"][9:] - r["tvec"]).max()
    same = refit_kernel(n, csize) == refit_kernel(s.cap, csize)
    assert (dt == 0) if same else (dt < 1e-12), (j, s.kinds[j], dt)
    # the state machine's composition: rvec -> R -> T -> inverse -> trans_dist >= max_dist_to_prev
    Tc = np.eye(4)
    Tc[:3, :3], Tc[:3, 3] = R, r["tvec"]
    T = np.linalg.inv(Tc)
    Tp = s.T_prev[j].reshape(4, 4)
    dist = float(np.linalg.norm(T[:3, 3] - Tp[:3, 3]))
    assert abs(dist - tp.max_dist_to_prev) > 1e-9, (j, dist)                    # far enough from the threshold to decide
    ok = int(dist < tp.max_dist_to_prev)
    assert o["pnp_ok"] == ok, (j, s.kinds[j], dist)
    want = T.ravel() if ok else s.T_prev[j]
    # the state machine's R comes back through rvec, which re-orthonormalises it (~1e-12 off after the LM, as in pnp_cases): the
    # rotation part and -R^T t carry that difference
    assert np.abs(o["T_w_c"] - want).max() < 1e-10, (j, s.kinds[j], np.abs(o["T_w_c"] - want).max())


def check_coverage(outs, s):
    """The scene reaches what it is meant to: a model, no model with enough pairs, a rejected jump, an accepted pose."""
    out = outs[0]
    kind = {k: out[s.kinds.index(k)] for k in s.kinds}
    assert kind["full"]["best"] >= 0 and kind["full"]["pnp_ok"] == 1 and kind["full"]["n_inliers"] > s.cap // 2
    assert kind["at_min"]["best"] >= 0 and kind["planar"]["best"] >= 0 and kind["planar"]["pnp_ok"] == 1
    assert kind["coincident"]["best"] == -1 and kind["coincident"]["pnp_ok"] == 0
    assert kind["jump"]["best"] >= 0 and kind["jump"]["pnp_ok"] == 0 and kind["jump"]["n_inliers"] > 0
    assert kind["four"]["best"] == -1 and kind["below_min"]["best"] == -1


def check_threshold(lib, h, s, tp, ptr=lambda a: a.ctypes.data, run=None):
    """max_dist_to_prev set to exactly the distance of the tail's host-order restatement: >= rejects it; one ulp above accepts."""
    j = s.kinds.index("full")
    t = s.subset([j])
    outs = outputs(1, s.cap)
    rc, outs = run(t, tp, outs) if run else call(lib, h, t, tp, ptr, outs)
    assert rc == OK
    o = outs[0][0]
    _, _, d = tail(o["Rt"], t.T_prev[0], 0.0, True)
    for max_dist, ok in ((d, 0), (float(np.nextafter(d, np.inf)), 1)):
        tq = track_params(lib, tp.min_pnp_points, max_dist)
        outs = outputs(1, s.cap)
        rc, outs = run(t, tq, outs) if run else call(lib, h, t, tq, ptr, outs)
        assert rc == OK
        o = outs[0][0]
        assert o["pnp_ok"] == ok, (d, max_dist)
        want = t.T_prev[0] if not ok else tail(o["Rt"], t.T_prev[0], max_dist, True)[1]
        assert o["T_w_c"].tobytes() == np.asarray(want, np.float64).tobytes()


def call_level_kinds(s):
    """(keyword arguments of call, expected return code) for every call-level check."""
    bad_K, neg_K, inf_K = np.array(K), np.array(K), np.array(K)
    bad_K[0, 0], neg_K[1, 1], inf_K[1, 1] = np.nan, -615.0, np.inf
    return [(dict(cap=0), INVALID_ARG), (dict(n_jobs=-1), INVALID_ARG), (dict(Kp=bad_K), INVALID_ARG), (dict(Kp=neg_K), INVALID_ARG),
            (dict(Kp=inf_K), INVALID_ARG), (dict(cap=8193), UNSUPPORTED), (dict(n_jobs=65536), UNSUPPORTED)]


# ---- the state machine end to end (GPU) ------------------------------------------------------------------------------------------
ROWS, COLS, KCAP = 480, 640, 2008


def record_tracking(imgs, K_cam):
    """The state machine in host-array mode over imgs: for every tracked frame, the map before it (container order), the reference
    keyframe's pose (the guess) and the previous frame's pose (frame_pose(0)) before add_frame, and after it the PnP outcome:
    n_matches, pnp_ok, n_inliers, matches_with_map and T_w_c_pnp.  Returns (events, vo params)."""
    ctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    vo = mvo_b200.VisualOdometry(ctx, K_cam, ROWS, COLS, track={"device_resident": 0})
    ev, last_kf, added = [], None, 0
    for i, im in enumerate(imgs):
        before = None
        if vo.is_initialized() and last_kf is not None:
            ids, pts, desc, _ = vo.get_map()
            before = (ids.copy(), pts.copy(), desc.copy(), vo.frame_pose(added - 1 - last_kf), vo.frame_pose(0))
        _, info = vo.add_frame(im)
        added += 1
        if info.state_in == 2 and before is not None:
            ev.append(dict(i=i, n_matches=info.n_matches, pnp_ok=info.pnp_ok, n_inliers=info.n_inliers,
                           mwm=vo.frame_data("matches_with_map", 0).copy(), T_pnp=np.array(info.T_w_c_pnp[:]), before=before))
        if info.keyframe:
            last_kf = info.frame_id
    vp = vo.params
    vo.close()
    ctx.close()
    return ev, vp


class Replay:
    """One extraction over the tracked frames, then per map version one mvo_vo_map_matches_batch_dev and its rows ready for
    mvo_vo_pnp_batch_dev (groups: the frames of each version, with their device rows)."""

    def __init__(self, bctx, ev, imgs, vp, K_cam):
        import torch
        self.bctx, self.ev, self.vp, self.K = bctx, ev, vp, np.asarray(K_cam, np.float64)
        z = lambda nbytes: torch.zeros(max(nbytes, 1), dtype=torch.uint8, device="cuda")     # noqa: E731
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()  # noqa: E731
        NF = len(ev)
        d_img = torch.from_numpy(np.ascontiguousarray(np.stack([imgs[e["i"]] for e in ev]))).cuda()
        self.d_k, self.d_d, self.d_c = z(NF * KCAP * 28), z(NF * KCAP * 32), torch.zeros(NF, dtype=torch.int32, device="cuda")
        bctx.orb_extract_batch_dev(d_img.data_ptr(), NF, ROWS, COLS, 3, COLS * 3, ROWS * COLS * 3, self.d_k.data_ptr(), self.d_d.data_ptr(),
                                   self.d_c.data_ptr(), KCAP)
        versions = {}
        for f, e in enumerate(ev):
            ids, pts, desc = e["before"][:3]
            versions.setdefault(ids.tobytes() + pts.tobytes() + desc.tobytes(), []).append(f)
        self.groups = []
        for fs in versions.values():
            ids, pts, desc = ev[fs[0]]["before"][:3]
            n_map, n_jobs = len(ids), len(fs)
            g = dict(fs=fs, n_jobs=n_jobs, d_map_p=dev(np.ascontiguousarray(pts, np.float32)), d_map_d=dev(np.ascontiguousarray(desc, np.uint8)),
                     d_fr=dev(np.array(fs, np.int32)), d_T=dev(np.stack([ev[f]["before"][3] for f in fs]).astype(np.float64)),
                     d_prev=dev(np.stack([ev[f]["before"][4] for f in fs]).astype(np.float64)),
                     d_mm=z(n_jobs * 16), d_cand=z(n_jobs * n_map * 4), d_m=z(n_jobs * KCAP * 16), d_p3=z(n_jobs * KCAP * 12),
                     d_p2=z(n_jobs * KCAP * 8), d_out=z(n_jobs * 256), d_inl=z(n_jobs * KCAP * 4), d_kept=z(n_jobs * KCAP * 16))
            bctx.vo_map_matches_batch_dev(self.d_k.data_ptr(), self.d_d.data_ptr(), self.d_c.data_ptr(), NF, KCAP, g["d_fr"].data_ptr(),
                                          g["d_T"].data_ptr(), n_jobs, g["d_map_p"].data_ptr(), g["d_map_d"].data_ptr(), n_map, self.K, ROWS,
                                          COLS, vp.track.match_method, vp.track.match_radius, g["d_mm"].data_ptr(), g["d_cand"].data_ptr(),
                                          g["d_m"].data_ptr(), d_pts3d=g["d_p3"].data_ptr(), d_pts2d=g["d_p2"].data_ptr())
            self.groups.append(g)
        bctx.synchronize()

    def pnp(self, g):
        """The batch PnP of one map version (asynchronous)."""
        self.bctx.vo_pnp_batch_dev(g["d_mm"].data_ptr(), g["d_m"].data_ptr(), g["d_p3"].data_ptr(), g["d_p2"].data_ptr(), g["n_jobs"], KCAP,
                                   g["d_prev"].data_ptr(), self.K, self.vp.track, g["d_out"].data_ptr(), g["d_inl"].data_ptr(),
                                   g["d_kept"].data_ptr())

    def host_pnp(self, g, j):
        """The per-frame host composition: job j's pairs downloaded, then mvo_solve_pnp_ransac on them."""
        n = int(g["d_mm"][j * 16 + 8:j * 16 + 12].cpu().numpy().view(np.int32)[0])
        p3 = g["d_p3"][j * KCAP * 12:(j * KCAP + n) * 12].cpu().numpy().view(np.float32)
        p2 = g["d_p2"][j * KCAP * 8:(j * KCAP + n) * 8].cpu().numpy().view(np.float32)
        if n < self.vp.track.min_pnp_points:
            return None
        rvec, tvec, inl = np.zeros(3), np.zeros(3), np.zeros(max(n, 1), np.int32)
        ni = C.c_int(n)
        rc = self.bctx.lib.mvo_solve_pnp_ransac(self.bctx.h, p3.ctypes.data, p2.ctypes.data, n, self.K.ctypes.data, rvec.ctypes.data,
                                                tvec.ctypes.data, inl.ctypes.data, C.byref(ni))
        return rc, rvec, tvec, inl[: ni.value]

    def results(self, g):
        n_jobs = g["n_jobs"]
        out = g["d_out"].cpu().numpy().view(OUT)
        m = g["d_m"].cpu().numpy().view(DM).reshape(n_jobs, KCAP)
        kept = g["d_kept"].cpu().numpy().view(DM).reshape(n_jobs, KCAP)
        mm = g["d_mm"].cpu().numpy().view(MM)
        return out, m, kept, mm


def check_replay(rp):
    """Every tracked frame: pnp_ok, n_inliers and matches_with_map after PnP byte-identical to the state machine's, T_w_c_pnp
    within 1e-10 (its R came through rvec).  Returns the largest T_w_c_pnp difference."""
    worst = 0.0
    for g in rp.groups:
        rp.pnp(g)
        rp.bctx.synchronize()
        out, m, kept, mm = rp.results(g)
        for j, f in enumerate(g["fs"]):
            e, o = rp.ev[f], out[j]
            assert o["status"] == OK and mm[j]["n_matches"] == e["n_matches"] == o["n_matches"], (e["i"], o)
            assert o["pnp_ok"] == e["pnp_ok"], (e["i"], o["pnp_ok"], e["pnp_ok"])
            if o["best"] >= 0:
                assert o["n_inliers"] == e["n_inliers"], (e["i"], o["n_inliers"], e["n_inliers"])
                assert kept[j, :o["n_inliers"]].tobytes() == e["mwm"].tobytes(), e["i"]
            else:
                assert m[j, :o["n_matches"]].tobytes() == e["mwm"].tobytes(), e["i"]
            d = float(np.abs(o["T_w_c"] - e["T_pnp"]).max())
            assert d < 1e-10, (e["i"], d)
            worst = max(worst, d)
    return worst
