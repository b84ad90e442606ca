"""Batches for mvo_vo_init_candidates_batch_dev (tests/test_vo_init_batch_emu.py, tests/test_vo_init_batch_gpu.py).

The call reads device buffers, so most pairs are FABRICATED: a relative-poses record with its inlier and triangulated rows, the
match list and both frames' keypoints, built from a known scene instead of hoping that RANSAC produces them.  The HOST REFERENCE of
a pair is the state machine's own sequence (vo_pipeline.cpp: estimate_motion_and_3d_points + is_vo_good_to_init) composed from
public pieces: the record and rows, transCoord / convertRt2T / the rigid inverse / the 4x4 product restated over Python floats in
vo_pipeline.cpp's order of operations, and the library's mvo_retain_good_triangulation, mvo_normalize_init_depth and
mvo_is_vo_good_to_init."""
import ctypes as C

import numpy as np

import mvo_b200

INVALID_ARG, DEGENERATE = -1, -6
RP = mvo_b200.RELATIVE_POSES_RESULT_DTYPE
OUT = mvo_b200.INIT_CANDIDATE_RESULT_DTYPE
KP, DM = mvo_b200.KEYPOINT_DTYPE, mvo_b200.DMATCH_DTYPE
K = np.array([[520.9, 0, 325.1], [0, 521.0, 249.7], [0, 0, 1]])
SENTINEL = 0xA5

# a reference keyframe that is not at the origin
T_REF = np.array([[0.9362934, -0.2896295, 0.1986693, 0.7], [0.3129918, 0.9447025, -0.0978434, -0.3],
                  [-0.1593451, 0.1537935, 0.9751703, 1.25], [0, 0, 0, 1.0]])


def rot(w):
    w = np.asarray(w, np.float64)
    th = np.linalg.norm(w)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def vo_params(lib, **kw):
    vp = mvo_b200.VoParams()
    lib.mvo_vo_default_params(C.byref(vp))
    for k, v in kw.items():
        setattr(vp, k, v)
    return vp


# ---- the state machine's host arithmetic over Python floats (vo_pipeline.cpp, mvo_internal.h) ----
def trans_coord(p, R, t):
    return np.array([R[3 * r] * float(p[0]) + R[3 * r + 1] * float(p[1]) + R[3 * r + 2] * float(p[2]) + t[r] for r in range(3)]).astype(np.float32)


def rt_to_T(R, t):
    T = [0.0] * 16
    for i in range(3):
        for j in range(3):
            T[i * 4 + j] = R[i * 3 + j]
        T[i * 4 + 3] = t[i]
    T[15] = 1.0
    return T


def inv_rigid(T):
    r = [0.0] * 16
    for i in range(3):
        for j in range(3):
            r[i * 4 + j] = T[j * 4 + i]
    for i in range(3):
        r[i * 4 + 3] = -(r[i * 4] * T[3] + r[i * 4 + 1] * T[7] + r[i * 4 + 2] * T[11])
    r[15] = 1.0
    return r


def mul44(A, B):
    out = [0.0] * 16
    for i in range(4):
        for j in range(4):
            a = 0.0
            for k in range(4):
                a += A[i * 4 + k] * B[k * 4 + j]
            out[i * 4 + j] = a
    return out


def pose(T_ref, R, t):
    return mul44([float(x) for x in np.ravel(T_ref)], inv_rigid(rt_to_T(R, t)))


class Batch:
    """Pair p = (frame 2p, frame 2p + 1).  specs: dicts of scene() keywords, or {"status": s} for a propagated status; "bad" names
    an invalid-input kind applied after the pair is built."""

    def __init__(self, specs, cap, seed=0):
        self.cap, self.n_pairs, self.batch = cap, len(specs), 2 * len(specs)
        rng = np.random.default_rng(seed)
        self.kpts = np.zeros((self.batch, cap), KP)
        self.counts = np.zeros(self.batch, np.int32)
        self.pairs = np.arange(self.batch, dtype=np.int32).reshape(-1, 2).copy()
        self.matches = np.zeros((self.n_pairs, cap), DM)
        self.n_matches = np.zeros(self.n_pairs, np.int32)
        self.rp = np.zeros(self.n_pairs, RP)
        self.rp_inl = np.zeros((self.n_pairs, 5, cap), np.int32)
        self.rp_pts = rng.normal(0, 3, (self.n_pairs, 5, cap, 3)).astype(np.float32)
        for p, spec in enumerate(specs):
            spec = dict(spec)
            bad = spec.pop("bad", None)
            if "status" in spec:
                self.rp[p]["status"] = spec["status"]
                self.rp[p]["n_matches"] = self.n_matches[p] = spec.get("n", 30)
                self.rp[p]["num_solutions"], self.rp[p]["best"] = 5, 7
                continue
            self._scene(p, rng, **spec)
            if bad:
                self._break(p, bad)

    def _scene(self, p, rng, n, ni=None, best=0, num=1, far=0, inf=0, near=0, depth=1.0, motion=((0.02, -0.05, 0.03), (1.0, 0.1, 0.05))):
        cap = self.cap
        ni = n if ni is None else ni
        R = rot(motion[0])
        t = np.asarray(motion[1], np.float64)
        t = t / np.linalg.norm(t)
        Xr = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 7, n)], 1)
        Xr *= depth
        idx = rng.permutation(n)
        Xr[idx[:far]] *= 400.0                                        # far: angles below 1 degree
        Xr[idx[far:far + near]] *= 0.01                               # near: far above the median
        Xc = Xr @ R.T + t
        proj = lambda X: (X[:, :2] / np.maximum(np.abs(X[:, 2:]), 1e-3)) * [K[0, 0], K[1, 1]] + [K[0, 2], K[1, 2]]
        perm = rng.permutation(n)
        q, tr = 2 * p, 2 * p + 1
        self.counts[q] = self.counts[tr] = n
        self.kpts[q]["x"][:n], self.kpts[q]["y"][:n] = proj(Xr).T.astype(np.float32)
        self.kpts[tr]["x"][perm], self.kpts[tr]["y"][perm] = proj(Xc).T.astype(np.float32)
        self.matches[p, :n]["query_idx"] = np.arange(n)
        self.matches[p, :n]["train_idx"] = perm
        self.matches[p, :n]["img_idx"] = 3
        self.matches[p, :n]["distance"] = rng.integers(0, 64, n).astype(np.float32)
        self.n_matches[p] = n
        r = self.rp[p]
        r["n_matches"], r["num_solutions"], r["best"] = n, num, best
        for s in range(num):
            k = ni if s == best else int(rng.integers(0, n + 1))
            r["n_inliers"][s] = k
            self.rp_inl[p, s, :k] = np.sort(rng.choice(n, k, replace=False))
            r["R"][s] = rot(rng.normal(0, 0.1, 3)).ravel()
            r["t"][s] = rng.normal(0, 1, 3)
        r["R"][best], r["t"][best] = R.ravel(), t
        inl = self.rp_inl[p, best, :ni]
        pts = Xr[inl].astype(np.float32)
        if inf:                                                       # points at infinity: NaN angles, kept
            at = rng.choice(ni, min(inf, ni), replace=False)
            pts[at] = np.array([0.0, 0.0, np.inf], np.float32)
        self.rp_pts[p, best, :ni] = pts

    def _break(self, p, bad):
        r = self.rp[p]
        best = int(r["best"])
        nm = int(self.n_matches[p])
        ni = int(r["n_inliers"][best])
        if bad == "best_neg":
            r["best"] = -1
        elif bad == "best_past":
            r["best"] = r["num_solutions"]
        elif bad == "num_zero":
            r["num_solutions"], r["best"] = 0, 0
        elif bad == "num_six":
            r["num_solutions"] = 6
        elif bad == "ni_neg":
            r["n_inliers"][best] = -1
        elif bad == "ni_past":
            r["n_inliers"][best] = nm + 1
        elif bad == "inl_neg":
            self.rp_inl[p, best, ni // 2] = -1
        elif bad == "inl_past":
            self.rp_inl[p, best, ni - 1] = nm
        elif bad == "frame_neg":
            self.pairs[p, 0] = -1
        elif bad == "frame_past":
            self.pairs[p, 1] = self.batch
        elif bad == "nm_past":
            self.n_matches[p] = self.cap + 1
        elif bad == "query_kp":
            self.matches[p, int(self.rp_inl[p, best, 0])]["query_idx"] = self.counts[2 * p]
        elif bad == "train_kp":
            self.matches[p, int(self.rp_inl[p, best, ni - 1])]["train_idx"] = -1
        else:
            raise ValueError(bad)


BAD_KINDS = ("best_neg", "best_past", "num_zero", "num_six", "ni_neg", "ni_past", "inl_neg", "inl_past", "frame_neg", "frame_past",
             "nm_past", "query_kp", "train_kp")


def reference(lib, b, p, T_ref, vp):
    """(status, record or None, kept matches, kept points, kept angles) of pair p as the state machine computes it."""
    r = b.rp[p]
    st = int(r["status"])
    rec = np.zeros(1, OUT)[0]
    empty = (np.zeros(0, DM), np.zeros((0, 3), np.float32), np.zeros(0))
    if st == DEGENERATE:
        rec["best_sol"] = -1
        rec["T_w_c"] = np.ravel(T_ref)
        return (0, rec) + empty
    if st != 0:
        return (st, None) + empty
    q, tr = (int(x) for x in b.pairs[p])
    nm, ns, best = int(b.n_matches[p]), int(r["num_solutions"]), int(r["best"])
    if not (0 <= q < b.batch and 0 <= tr < b.batch and 0 <= nm <= b.cap and 1 <= ns <= 5 and 0 <= best < ns):
        return (INVALID_ARG, None) + empty
    ni = int(r["n_inliers"][best])
    if not 0 <= ni <= nm:
        return (INVALID_ARG, None) + empty
    inl = b.rp_inl[p, best, :ni]
    if ni and (inl.min() < 0 or inl.max() >= nm):
        return (INVALID_ARG, None) + empty
    m = b.matches[p, inl].copy()
    cq, ct = (min(max(int(b.counts[f]), 0), b.cap) for f in (q, tr))
    if ni and (m["query_idx"].min() < 0 or m["query_idx"].max() >= cq or m["train_idx"].min() < 0 or m["train_idx"].max() >= ct):
        return (INVALID_ARG, None) + empty
    m["img_idx"] = -1
    R = [float(x) for x in r["R"][best]]
    t = [float(x) for x in r["t"][best]]
    with np.errstate(all="ignore"):
        pts = np.array([trans_coord(x, R, t) for x in b.rp_pts[p, best, :ni]], np.float32).reshape(-1, 3)
    Tr = np.ascontiguousarray(np.ravel(T_ref), np.float64)
    Tc = np.array(pose(T_ref, R, t))
    keep = np.zeros(max(ni, 1), np.int32)
    ang = np.zeros(max(ni, 1))
    nk = C.c_int(0)
    assert lib.mvo_retain_good_triangulation(pts.ctypes.data, ni, Tc.ctypes.data, Tr.ctypes.data, vp.min_triang_angle,
                                             vp.max_ratio_angle_to_median, keep.ctypes.data, ang.ctypes.data, C.byref(nk)) == 0
    nk = nk.value
    keep, ang = keep[:nk], ang[:nk].copy()
    kept_m, kept_p = m[keep], np.ascontiguousarray(pts[keep])
    tt = np.array(t)
    scale = C.c_double(0)
    if nk >= 20:
        assert lib.mvo_normalize_init_depth(kept_p.ctypes.data, nk, tt.ctypes.data, vp.assumed_mean_depth_init, C.byref(scale)) == 0
        Tc = np.array(pose(T_ref, R, [float(x) for x in tt]))
        rec["normalized"], rec["scale"] = 1, scale.value
    p1 = np.ascontiguousarray(np.stack([b.kpts[q]["x"][kept_m["query_idx"]], b.kpts[q]["y"][kept_m["query_idx"]]], 1), np.float32)
    p2 = np.ascontiguousarray(np.stack([b.kpts[tr]["x"][kept_m["train_idx"]], b.kpts[tr]["y"][kept_m["train_idx"]]], 1), np.float32)
    good, mean, med = C.c_int(0), C.c_double(0), C.c_double(0)
    assert lib.mvo_is_vo_good_to_init(p1.ctypes.data, p2.ctypes.data, nk, ang.ctypes.data if nk else None, nk, vp.min_inlier_matches,
                                      vp.min_pixel_dist, vp.min_median_triangulation_angle, C.byref(good), C.byref(mean), C.byref(med)) == 0
    rec["usable"], rec["good"], rec["best_sol"], rec["n_inliers"], rec["n_kept"] = 1, good.value, best, ni, nk
    rec["mean_pixel_dist"], rec["median_angle"] = mean.value, med.value
    rec["t_curr_to_prev"] = tt
    rec["T_w_c"] = Tc
    return 0, rec, kept_m, kept_p, ang


def outputs(n_pairs, cap):
    out = np.full(n_pairs * OUT.itemsize, SENTINEL, np.uint8).view(OUT)
    kept = np.full(n_pairs * cap * DM.itemsize, SENTINEL, np.uint8).view(DM).reshape(n_pairs, cap)
    kpts = np.full(n_pairs * cap * 12, SENTINEL, np.uint8).view(np.float32).reshape(n_pairs, cap, 3)
    kang = np.full(n_pairs * cap * 8, SENTINEL, np.uint8).view(np.float64).reshape(n_pairs, cap)
    return out, kept, kpts, kang


def call(lib, ctx, b, T_ref, vp, ptr=lambda a: a.ctypes.data, outs=None):
    """The call over host arrays (the emulated library) or, with ptr / outs, over device copies."""
    out, kept, kpts, kang = outs or outputs(b.n_pairs, b.cap)
    T = np.ascontiguousarray(np.ravel(T_ref), np.float64)
    rc = lib.mvo_vo_init_candidates_batch_dev(ctx, ptr(b.kpts), ptr(b.counts), b.batch, b.cap, ptr(b.pairs), b.n_pairs, ptr(b.matches),
                                              ptr(b.n_matches), ptr(b.rp), ptr(b.rp_inl), ptr(b.rp_pts), T.ctypes.data, C.byref(vp),
                                              ptr(out), ptr(kept), ptr(kpts), ptr(kang))
    return rc, (out, kept, kpts, kang)


def check_failed(out, kept, p, status):
    """A failed pair writes its status and nothing else."""
    assert out[p]["status"] == status, (p, out[p]["status"], status)
    assert (out[p:p + 1].view(np.uint8)[4:] == SENTINEL).all(), p
    assert (kept[p].view(np.uint8) == SENTINEL).all(), p


def check_exact(ref, got, p):
    """Emulated tier: every byte of the record and of the kept rows."""
    out, kept, kpts, kang = got
    st, rec, km, kp, ka = ref
    if rec is None:
        check_failed(out, kept, p, st)
        return
    assert out[p:p + 1].tobytes() == rec.tobytes(), (p, out[p], rec)
    nk = int(rec["n_kept"])
    assert kept[p, :nk].tobytes() == km.tobytes(), p
    assert kpts[p, :nk].tobytes() == kp.tobytes(), p
    assert kang[p, :nk].tobytes() == ka.tobytes(), p
    check_untouched_past(got, p, nk)


def check_untouched_past(got, p, nk):
    """Nothing past n_kept is written in the three rows."""
    _, kept, kpts, kang = got
    for row in (kept[p, nk:], kpts[p, nk:], kang[p, nk:]):
        assert (row.view(np.uint8) == SENTINEL).all(), p


def ulp_diff(a, b):
    """|a - b| in units in the last place of doubles (same-sign finite values; equal NaN bits count 0)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ia, ib = a.view(np.int64), b.view(np.int64)
    both_nan = np.isnan(a) & np.isnan(b)
    d = np.where(both_nan & (ia == ib), 0, np.abs(ia.astype(object) - ib.astype(object)) if a.size else 0)
    return np.asarray(d, dtype=object)


def margin_failures(ang, med_retain, vp, med_init, ulps=4):
    """The decisions of the pair that lie too close to their threshold for the GPU tier's exact check, one line each (empty: none).
    Each angle and the median are within `ulps` of the host's on the device, so an angle is compared with min_triang_angle and the
    kept median with min_median_triangulation_angle at that margin; the ratio test compares the quotient angle / median, which
    can then move by about 2 x ulps + 1, so the quotient is held to 4 x ulps of margin."""
    a = np.asarray(ang, np.float64)
    a = a[~np.isnan(a)]

    def near(x, bound, n):
        if not np.isfinite(bound) or x.size == 0:
            return np.zeros(x.shape, bool)
        lo, hi = bound, bound
        for _ in range(n):
            lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        return (x >= lo) & (x <= hi)
    out = []
    if near(a, vp.min_triang_angle, ulps).any():
        out.append(f"{int(near(a, vp.min_triang_angle, ulps).sum())} angle(s) within {ulps} ulp of min_triang_angle")
    if np.isfinite(med_retain) and med_retain > 0:
        with np.errstate(all="ignore"):
            q = a / med_retain
        m = near(q, vp.max_ratio_angle_to_median, 4 * ulps)
        if m.any():
            out.append(f"{int(m.sum())} angle / median quotient(s) within {4 * ulps} ulp of max_ratio_angle_to_median")
    if near(np.array([med_init]), vp.min_median_triangulation_angle, ulps).any():
        out.append(f"the median angle within {ulps} ulp of min_median_triangulation_angle")
    return out


def all_angles(lib, b, p, T_ref):
    """Every inlier's angle and the retain median of pair p (host), for the margin check."""
    r = b.rp[p]
    best, ni = int(r["best"]), int(r["n_inliers"][int(r["best"])])
    R, t = [float(x) for x in r["R"][best]], [float(x) for x in r["t"][best]]
    with np.errstate(all="ignore"):
        pts = np.array([trans_coord(x, R, t) for x in b.rp_pts[p, best, :ni]], np.float32).reshape(-1, 3)
    Tc = np.array(pose(T_ref, R, t))
    Tr = np.ascontiguousarray(np.ravel(T_ref), np.float64)
    keep, ang, nk = np.zeros(max(ni, 1), np.int32), np.zeros(max(ni, 1)), C.c_int(0)
    lib.mvo_retain_good_triangulation(pts.ctypes.data, ni, Tc.ctypes.data, Tr.ctypes.data, -np.inf, np.inf, keep.ctypes.data,
                                      ang.ctypes.data, C.byref(nk))
    ang = ang[:ni]
    med = np.sort(ang)[ni // 2] if ni and not np.isnan(ang).any() else np.nan
    return ang, med


def mixed_specs(cap, big):
    """The fabricated pairs of one call: E / H choices, the n_inliers / n_kept edges, points at infinity, every invalid kind and
    the propagated statuses."""
    specs = [
        dict(n=300),                                                        # E chosen, normalised
        dict(n=200, num=3, best=1),                                         # H chosen, best 1
        dict(n=200, num=3, best=2, motion=((0.01, 0.04, -0.02), (-0.3, 0.2, -1.0))),     # best 2, moving backwards
        dict(n=60, ni=0),                                                   # n_inliers[best] = 0: no median
        dict(n=40, far=40),                                                 # n_kept = 0 after the angle test
        dict(n=30, far=11),                                                 # n_kept = 19: not normalised
        dict(n=30, far=10),                                                 # n_kept = 20: normalised
        dict(n=120, near=3, depth=5.0),                                     # three dropped above max_ratio x median
        dict(n=41, inf=15),                                                 # NaN angles, kept
        dict(n=41, inf=30),                                                 # NaN at the median position
        dict(n=25, inf=5, far=8),                                           # NaN angles, fewer than 20 kept
        dict(n=12),                                                         # too few to initialise
        dict(n=big, far=big // 10, near=5),                                 # n = cap
        {"status": DEGENERATE, "n": 5},
        {"status": INVALID_ARG, "n": 7},
    ]
    specs += [dict(n=50, bad=k) for k in BAD_KINDS]
    return specs


def boundary_batches(lib, cap):
    """Calls whose thresholds sit exactly on an angle of their pair: (batch, vp) with the angle at min_triang_angle, and at
    max_ratio x median."""
    b = Batch([dict(n=101, near=2)], cap, seed=5)
    ang, med = all_angles(lib, b, 0, T_REF)
    srt = np.sort(ang)
    out = [(b, vo_params(lib, min_triang_angle=float(srt[10])))]                       # exactly at the minimum: kept
    out.append((b, vo_params(lib, max_ratio_angle_to_median=float(srt[-2] / med))))   # exactly at the ratio: kept, the largest dropped
    rec = reference(lib, b, 0, T_REF, vo_params(lib))[1]
    out.append((b, vo_params(lib, min_median_triangulation_angle=float(rec["median_angle"]))))      # median not above it: not good
    return out
