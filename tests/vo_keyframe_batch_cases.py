"""Batches for mvo_vo_keyframe_points_batch_dev (tests/test_vo_keyframe_batch_emu.py, tests/test_vo_keyframe_batch_gpu.py).

The call reads device buffers, so the pairs are FABRICATED: a known scene seen by two posed frames, the match list between them,
and an essential record with its inlier row, instead of hoping that RANSAC produces the case.  The HOST REFERENCE of a pair is the
state machine's own keyframe branch (vo_pipeline.cpp: insert_keyframe) composed from public pieces: the known motion
T_w_c_curr^-1 * T_w_c_ref, pixel2CamNormPlane and transCoord restated over Python floats in vo_pipeline.cpp's order of
operations, the library's mvo_do_triangulation and mvo_retain_good_triangulation, std::nth_element for the median, and
preTranslatePoint3f with the viewing direction of push_curr_points_to_map.

The pairs cover n_inliers 0, 1 and cap, drops by the angle and by the ratio to the median, points at infinity with one at the
median, pure rotation, a frame with itself, reversed and repeated pairs, identity and general reference poses, the propagated
statuses, every invalid input and call-level limit, NULL optional rows and sentinel bytes past n_kept.  The emulated tier expects
every byte; the GPU tier allows 4 ulp on the angles and the median (the device's acos) and replays every keyframe insertion of the
bench sequence through the batch chain."""
import ctypes as C
import math
import subprocess
import tempfile
from pathlib import Path

import numpy as np

import mvo_b200
import vo_init_batch_cases as vi

INVALID_ARG, CUDA_ERR, DEGENERATE = -1, -3, -6
ESS = mvo_b200.TWO_VIEW_RESULT_DTYPE
OUT = mvo_b200.KEYFRAME_POINTS_RESULT_DTYPE
KP, DM = mvo_b200.KEYPOINT_DTYPE, mvo_b200.DMATCH_DTYPE
# principal point exactly representable in float: a keypoint there is exactly on the optical axis (see Batch._scene, inf)
K = np.array([[520.9, 0, 325.0], [0, 521.0, 249.5], [0, 0, 1]])
T_REF = vi.T_REF
SENTINEL = vi.SENTINEL
LAUNCHES = 3
HOST_NAN = np.frombuffer(np.uint64(0xFFF8000000000000).tobytes(), np.float64)[0]

_NTH = []


def nth_median(a):
    """std::nth_element(v, v + n / 2, v + n) of libstdc++, then v[n / 2]: retainGoodTriangulationResult_'s median."""
    if not _NTH:
        d = Path(tempfile.mkdtemp(prefix="nth_median"))
        (d / "nth.cpp").write_text('#include <algorithm>\nextern "C" double nth_median(double *v, int n) '
                                   '{ std::nth_element(v, v + n / 2, v + n); return v[n / 2]; }\n')
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", str(d / "nth.cpp"), "-o", str(d / "nth.so")], check=True)
        lib = C.CDLL(str(d / "nth.so"))
        lib.nth_median.restype, lib.nth_median.argtypes = C.c_double, [C.c_void_p, C.c_int]
        _NTH.append(lib)
    v = np.ascontiguousarray(a, np.float64).copy()
    return _NTH[0].nth_median(v.ctypes.data, len(v))


def host_nan(x):
    return HOST_NAN if x != x else x


# ---- the state machine's host arithmetic over Python floats (vo_pipeline.cpp, mvo_internal.h) ----
def known_motion(T_curr, T_ref):
    T = vi.mul44(vi.inv_rigid([float(x) for x in np.ravel(T_curr)]), [float(x) for x in np.ravel(T_ref)])
    return [T[i * 4 + j] for i in range(3) for j in range(3)], [T[i * 4 + 3] for i in range(3)]


def to_norm_plane(x, y):
    return np.float32((float(x) - K[0, 2]) / K[0, 0]), np.float32((float(y) - K[1, 2]) / K[1, 1])


def pre_translate(p, T):
    out = []
    for r in range(3):
        a = 0.0
        a += T[r * 4] * float(p[0])
        a += T[r * 4 + 1] * float(p[1])
        a += T[r * 4 + 2] * float(p[2])
        a += T[r * 4 + 3] * 1.0
        out.append(a)
    return np.array(out).astype(np.float32)


def direction(pos, cam):
    d = [float(pos[q]) - cam[q] for q in range(3)]
    n = np.float64(math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])) if all(x == x for x in d) else np.float64(np.nan)
    with np.errstate(all="ignore"):
        return [host_nan(float(np.float64(x) / n)) for x in d]


def pose_of(rel, T_ref):
    """T_w_c of a frame whose pose relative to T_ref is rotation w, centre c (in the reference camera)."""
    w, c = rel
    Tr = np.eye(4)
    Tr[:3, :3] = vi.rot(w) if np.linalg.norm(w) > 0 else np.eye(3)
    Tr[:3, 3] = c
    return np.asarray(T_ref, np.float64) @ Tr


class Batch:
    """Every spec owns frames 2s and 2s + 1 and pair s = (2s, 2s + 1) by default.  Spec kinds:
      scene keywords (n, ni, far, near, inf, rel, ref): a scene seen from both frames, matched, with an essential record;
      {"status": s, "n": n}: a record with that essential status;
      {"of": q, "how": "reversed" | "repeated" | "self"}: a pair over the frames of scene q (its own frames stay empty).
    "bad" names an invalid-input kind applied after the pair is built."""

    def __init__(self, specs, cap, seed=0):
        self.cap, self.n_pairs, self.batch = cap, len(specs), 2 * len(specs)
        rng = np.random.default_rng(seed)
        self.kpts = np.zeros((self.batch, cap), KP)
        self.counts = np.zeros(self.batch, np.int32)
        self.pairs = np.arange(self.batch, dtype=np.int32).reshape(-1, 2).copy()
        self.matches = np.zeros((self.n_pairs, cap), DM)
        self.n_matches = np.zeros(self.n_pairs, np.int32)
        self.ess = np.zeros(self.n_pairs, ESS)
        self.inl = np.zeros((self.n_pairs, cap), np.int32)
        self.T = np.tile(np.eye(4), (self.batch, 1, 1))
        for p, spec in enumerate(specs):
            spec = dict(spec)
            bad = spec.pop("bad", None)
            if "status" in spec:
                self.ess[p]["status"] = spec["status"]
                self.n_matches[p] = spec.get("n", 30)
                self.ess[p]["n_inliers"] = 7 * cap
            elif "of" in spec:
                self._derived(p, rng, spec["of"], spec["how"])
            else:
                self._scene(p, rng, **spec)
            if bad:
                self._break(p, bad)

    def _record(self, p, rng, n, ni):
        e = self.ess[p]
        e["status"], e["n_matches"], e["n_inliers"], e["votes"] = 0, n, ni, ni
        e["E"], e["R"], e["t"] = rng.normal(0, 1, 9), rng.normal(0, 1, 9), rng.normal(0, 1, 3)
        self.inl[p, :ni] = np.sort(rng.choice(n, ni, replace=False))

    def _scene(self, p, rng, n, ni=None, far=0, near=0, inf=0, rel=((0.02, -0.05, 0.03), (0.6, 0.05, 0.1)), ref="general"):
        cap = self.cap
        ni = n if ni is None else ni
        T_ref = T_REF if ref == "general" else np.eye(4)
        q, tr = 2 * p, 2 * p + 1
        self.T[q], self.T[tr] = T_ref, pose_of(rel, T_ref)
        Xr = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 7, n)], 1)
        idx = rng.permutation(n)
        Xr[idx[:far]] *= 400.0                                        # far: angles below 1 degree
        near_at = idx[far:far + near]                                 # near: between the camera centres, far above the median
        Xr[near_at] = 0.5 * np.asarray(rel[1], np.float64) + np.stack([rng.uniform(-0.02, 0.02, near), rng.uniform(-0.02, 0.02, near),
                                                                       np.full(near, 0.05)], 1)
        Rrel = self.T[tr][:3, :3].T @ self.T[q][:3, :3]               # reference camera -> current camera
        Xc = (Xr - np.asarray(rel[1], np.float64)) @ Rrel.T
        # points at infinity: on the optical axis of both cameras, which a pair moving straight forward (rel = (0, 0, 0), (0, 0, z))
        # from the identity pose shares; both keypoints sit exactly on the principal point, the DLT's last column is exactly 0
        # and the point comes out with w = 0 (a NaN angle)
        at = idx[far + near:far + near + inf]
        Xr[at] = [0.0, 0.0, 5.0]
        Xc[at] = (Xr[at] - np.asarray(rel[1], np.float64)) @ Rrel.T
        proj = lambda X: (X[:, :2] / np.maximum(np.abs(X[:, 2:]), 1e-3)) * [K[0, 0], K[1, 1]] + [K[0, 2], K[1, 2]]
        perm = rng.permutation(n)
        self.counts[q] = self.counts[tr] = n
        self.kpts[q]["x"][:n], self.kpts[q]["y"][:n] = proj(Xr).T.astype(np.float32)
        self.kpts[tr]["x"][perm], self.kpts[tr]["y"][perm] = proj(Xc).T.astype(np.float32)
        order = rng.permutation(n)                                    # match list order is not keypoint order
        self.matches[p, :n]["query_idx"] = order
        self.matches[p, :n]["train_idx"] = perm[order]
        self.matches[p, :n]["img_idx"] = 3
        self.matches[p, :n]["distance"] = rng.integers(0, 64, n).astype(np.float32)
        self.n_matches[p] = n
        self._record(p, rng, n, ni)

    def _derived(self, p, rng, of, how):
        q, tr = (int(x) for x in self.pairs[of])
        n = int(self.n_matches[of])
        m = self.matches[of, :n].copy()
        if how == "reversed":
            self.pairs[p] = (tr, q)
            m["query_idx"], m["train_idx"] = m["train_idx"].copy(), m["query_idx"].copy()
        elif how == "repeated":
            self.pairs[p] = (q, tr)
        elif how == "self":
            self.pairs[p] = (tr, tr)
            m["query_idx"] = m["train_idx"]
        else:
            raise ValueError(how)
        self.matches[p, :n] = m
        self.n_matches[p] = n
        self._record(p, rng, n, n if how == "self" else int(self.ess[of]["n_inliers"]))
        if how == "repeated":
            self.inl[p] = self.inl[of]

    def _break(self, p, bad):
        e = self.ess[p]
        nm, ni = int(self.n_matches[p]), int(e["n_inliers"])
        q, tr = (int(x) for x in self.pairs[p])
        if bad == "frame_neg":
            self.pairs[p, 0] = -1
        elif bad == "frame_past":
            self.pairs[p, 1] = self.batch
        elif bad == "nm_neg":
            self.n_matches[p] = -1
        elif bad == "nm_past":
            self.n_matches[p] = self.cap + 1
        elif bad == "ni_neg":
            e["n_inliers"] = -1
        elif bad == "ni_past":
            e["n_inliers"] = nm + 1
        elif bad == "inl_neg":
            self.inl[p, ni // 2] = -1
        elif bad == "inl_past":
            self.inl[p, ni - 1] = nm
        elif bad == "query_kp":
            self.matches[p, int(self.inl[p, 0])]["query_idx"] = self.counts[q]
        elif bad == "train_kp":
            self.matches[p, int(self.inl[p, ni - 1])]["train_idx"] = -1
        elif bad == "ref_pose_nan":
            self.T[q][1, 3] = np.nan
        elif bad == "curr_pose_inf":
            self.T[tr][2, 1] = np.inf
        else:
            raise ValueError(bad)


BAD_KINDS = ("frame_neg", "frame_past", "nm_neg", "nm_past", "ni_neg", "ni_past", "inl_neg", "inl_past", "query_kp", "train_kp",
             "ref_pose_nan", "curr_pose_inf")


def _triangulate(lib, ctx, b, p, inl, R, t):
    """mvo_do_triangulation on pixel2CamNormPlane points of the inlier matches (the host path of insert_keyframe)."""
    q, tr = (int(x) for x in b.pairs[p])
    ni = len(inl)
    m = b.matches[p, inl]
    np1 = np.zeros((max(ni, 1), 2), np.float32)
    np2 = np.zeros((max(ni, 1), 2), np.float32)
    for i in range(ni):
        np1[i] = to_norm_plane(b.kpts[q]["x"][m[i]["query_idx"]], b.kpts[q]["y"][m[i]["query_idx"]])
        np2[i] = to_norm_plane(b.kpts[tr]["x"][m[i]["train_idx"]], b.kpts[tr]["y"][m[i]["train_idx"]])
    out = np.zeros((max(ni, 1), 3), np.float32)
    if ni:
        Ra, ta = np.array(R), np.array(t)
        rng = np.arange(ni, dtype=np.int32)
        assert lib.mvo_do_triangulation(ctx, np1.ctypes.data, np2.ctypes.data, ni, Ra.ctypes.data, ta.ctypes.data, rng.ctypes.data, ni,
                                        out.ctypes.data) == 0
    return out[:ni]


def current_points(lib, ctx, b, p):
    """(points in the current camera, T_w_c_curr, T_w_c_ref, R, t) of a well-formed usable pair."""
    q, tr = (int(x) for x in b.pairs[p])
    ni = int(b.ess[p]["n_inliers"])
    R, t = known_motion(b.T[tr], b.T[q])
    tri = _triangulate(lib, ctx, b, p, b.inl[p, :ni], R, t)
    with np.errstate(all="ignore"):
        pts = np.array([vi.trans_coord(x, R, t) for x in tri], np.float32).reshape(-1, 3)
    return pts, np.ascontiguousarray(b.T[tr].ravel()), np.ascontiguousarray(b.T[q].ravel()), R, t


def all_angles(lib, ctx, b, p):
    """Every inlier's angle and the retain median of pair p (host), for the margin check."""
    pts, Tc, Tr, _, _ = current_points(lib, ctx, b, p)
    ni = len(pts)
    keep, ang, nk = np.zeros(max(ni, 1), np.int32), np.zeros(max(ni, 1)), C.c_int(0)
    lib.mvo_retain_good_triangulation(pts.ctypes.data, ni, Tc.ctypes.data, Tr.ctypes.data, -np.inf, np.inf, keep.ctypes.data,
                                      ang.ctypes.data, C.byref(nk))
    ang = ang[:ni]
    return ang, (nth_median(ang) if ni else 0.0)


def reference(lib, ctx, b, p, vp):
    """(status, record or None, kept matches, kept points, kept angles, world positions, directions) of pair p as the state
    machine computes it."""
    e = b.ess[p]
    st = int(e["status"])
    rec = np.zeros(1, OUT)[0]
    empty = (np.zeros(0, DM), np.zeros((0, 3), np.float32), np.zeros(0), np.zeros((0, 3), np.float32), np.zeros((0, 3)))
    if st not in (0, DEGENERATE):
        return (st, None) + empty
    q, tr = (int(x) for x in b.pairs[p])
    nm = int(b.n_matches[p])
    if not (0 <= q < b.batch and 0 <= tr < b.batch and 0 <= nm <= b.cap):
        return (INVALID_ARG, None) + empty
    rec["n_matches"] = nm
    if st == DEGENERATE:                                              # insert_keyframe returns: no keyframe
        return (0, rec) + empty
    ni = int(e["n_inliers"])
    if not 0 <= ni <= nm:
        return (INVALID_ARG, None) + empty
    inl = b.inl[p, :ni]
    if ni and (inl.min() < 0 or inl.max() >= nm):
        return (INVALID_ARG, None) + empty
    m = b.matches[p, inl].copy()
    cq, ct = (min(max(int(b.counts[f]), 0), b.cap) for f in (q, tr))
    if ni and (m["query_idx"].min() < 0 or m["query_idx"].max() >= cq or m["train_idx"].min() < 0 or m["train_idx"].max() >= ct):
        return (INVALID_ARG, None) + empty
    if not (np.isfinite(b.T[q]).all() and np.isfinite(b.T[tr]).all()):
        return (INVALID_ARG, None) + empty
    m["img_idx"] = -1
    pts, Tc, Tr, R, t = current_points(lib, ctx, b, p)
    keep = np.zeros(max(ni, 1), np.int32)
    ang = np.zeros(max(ni, 1))
    nk = C.c_int(0)
    assert lib.mvo_retain_good_triangulation(pts.ctypes.data, ni, Tc.ctypes.data, Tr.ctypes.data, vp.min_triang_angle,
                                             vp.max_ratio_angle_to_median, keep.ctypes.data, ang.ctypes.data, C.byref(nk)) == 0
    nk = nk.value
    keep, ang = keep[:nk], np.array([host_nan(x) for x in ang[:nk]])
    kept_m, kept_p = m[keep], np.ascontiguousarray(pts[keep]).reshape(-1, 3)
    Tcl = [float(x) for x in Tc]
    cam = [Tcl[3], Tcl[7], Tcl[11]]
    with np.errstate(all="ignore"):
        world = np.array([pre_translate(x, Tcl) for x in kept_p], np.float32).reshape(-1, 3)
    norm = np.array([direction(x, cam) for x in world]).reshape(-1, 3)
    _, med = all_angles(lib, ctx, b, p)
    rec["usable"], rec["n_inliers"], rec["n_kept"] = 1, ni, nk
    rec["median_angle"] = host_nan(med)
    rec["R_curr_to_prev"], rec["t_curr_to_prev"] = R, t
    return 0, rec, kept_m, kept_p, ang, world, norm


def outputs(n_pairs, cap, world=True, norm=True):
    out = np.full(n_pairs * OUT.itemsize, SENTINEL, np.uint8).view(OUT)
    kept = np.full(n_pairs * cap * DM.itemsize, SENTINEL, np.uint8).view(DM).reshape(n_pairs, cap)
    kpts = np.full(n_pairs * cap * 12, SENTINEL, np.uint8).view(np.float32).reshape(n_pairs, cap, 3)
    kang = np.full(n_pairs * cap * 8, SENTINEL, np.uint8).view(np.float64).reshape(n_pairs, cap)
    kw = np.full(n_pairs * cap * 12, SENTINEL, np.uint8).view(np.float32).reshape(n_pairs, cap, 3) if world else None
    kn = np.full(n_pairs * cap * 24, SENTINEL, np.uint8).view(np.float64).reshape(n_pairs, cap, 3) if norm else None
    return out, kept, kpts, kang, kw, kn


def call(lib, ctx, b, vp, ptr=lambda a: a.ctypes.data, outs=None, n_pairs=None, Kp=None):
    """The call over host arrays (the emulated library) or, with ptr / outs, over device copies."""
    out, kept, kpts, kang, kw, kn = outs or outputs(b.n_pairs, b.cap)
    Kh = np.ascontiguousarray(K if Kp is None else Kp, np.float64)
    rc = lib.mvo_vo_keyframe_points_batch_dev(ctx, ptr(b.kpts), ptr(b.counts), b.batch, b.cap, ptr(b.pairs),
                                              b.n_pairs if n_pairs is None else n_pairs, ptr(b.matches), ptr(b.n_matches), ptr(b.ess),
                                              ptr(b.inl), ptr(b.T), Kh.ctypes.data, C.byref(vp), ptr(out), ptr(kept), ptr(kpts),
                                              ptr(kang), None if kw is None else ptr(kw), None if kn is None else ptr(kn))
    return rc, (out, kept, kpts, kang, kw, kn)


def check_failed(got, p, status):
    """A failed pair writes its status and nothing else."""
    out = got[0]
    assert out[p]["status"] == status, (p, out[p]["status"], status)
    assert (out[p:p + 1].view(np.uint8)[4:] == SENTINEL).all(), p
    check_untouched_past(got, p, 0)


def check_untouched_past(got, p, nk, ni=0):
    """Nothing past n_kept is written in any row, except in the point row: it holds the triangulated inliers between the second
    and the third launch, so its entries up to n_inliers are unspecified."""
    for i, a in enumerate(got[1:]):
        if a is not None:
            assert (a[p, max(nk, ni) if i == 1 else nk:].view(np.uint8) == SENTINEL).all(), (p, i)


def check_exact(ref, got, p):
    """Emulated tier: every byte of the record and of the kept rows."""
    st, rec, km, kp, ka, kw, kn = ref
    if rec is None:
        check_failed(got, p, st)
        return
    out, kept, kpts, kang, gw, gn = got
    assert out[p:p + 1].tobytes() == rec.tobytes(), (p, out[p], rec)
    nk = int(rec["n_kept"])
    assert kept[p, :nk].tobytes() == km.tobytes(), p
    assert kpts[p, :nk].tobytes() == kp.tobytes(), p
    assert kang[p, :nk].tobytes() == ka.tobytes(), p
    if gw is not None:
        assert gw[p, :nk].tobytes() == kw.tobytes(), p
    if gn is not None:
        assert gn[p, :nk].tobytes() == np.ascontiguousarray(kn).tobytes(), p
    check_untouched_past(got, p, nk, int(rec["n_inliers"]) if rec["usable"] else 0)


FORWARD = ((0.0, 0.0, 0.0), (0.0, 0.0, 0.5))


def mixed_specs(cap):
    """The fabricated pairs of one call."""
    specs = [
        dict(n=300),                                                        # general reference pose, every point kept
        dict(n=200, ref="identity"),                                        # identity reference pose
        dict(n=60, ni=0),                                                   # n_inliers = 0: no median
        dict(n=40, ni=1),                                                   # n_inliers = 1
        dict(n=120, far=30),                                                # drops by min_triang_angle
        dict(n=120, near=3),                                                # drops by the ratio to the median
        dict(n=41, inf=15, rel=FORWARD, ref="identity"),                    # points at infinity
        dict(n=41, inf=30, rel=FORWARD, ref="identity"),                    # ... at the median position
        dict(n=50, rel=((0.03, 0.01, -0.02), (0.0, 0.0, 0.0))),             # pure rotation, t = 0
        dict(n=cap, far=cap // 10, near=5),                                 # n_inliers = cap
        {"of": 0, "how": "reversed"},
        {"of": 4, "how": "repeated"},
        {"of": 1, "how": "self"},                                           # a frame with itself
        {"status": DEGENERATE, "n": 5},
        {"status": INVALID_ARG, "n": 7},
        {"status": CUDA_ERR, "n": 9},
    ]
    specs += [dict(n=50, bad=k) for k in BAD_KINDS]
    return specs
