"""Batches for mvo_vo_map_matches_batch_dev (tests/test_map_matches_batch_emu.py, tests/test_map_matches_batch_gpu.py).

A fabricated scene in the layout of mvo_orb_extract_batch_dev: one map, frames whose keypoints are noisy projections of map points
(descriptors with a few flipped bits) among unrelated keypoints, and (frame, guess pose) jobs.  The HOST REFERENCE of a job is
what the state machine's pose_estimation_pnp computes before solvePnPRansac: inv_rigid, preTranslatePoint3f, the z < 0 test,
cam2pixel and the strict inside test restated over Python floats in vo_pipeline.cpp's order of operations, then the library's
mvo_match_features on the candidate arrays with match_into's skip rules, then the 3D-2D pairs in match order.

The scene covers points behind the camera, at camera z = +0.0 and -0.0, pixels exactly on 0 / cols / rows, a keypoint exactly at
the radius, duplicated map descriptors (removeDuplicatedMatches ties), frames with 0, 1, a negative and an over-cap keypoint count,
identity and general guesses, a frame under two guesses, a repeated job, a guess that sees nothing, every per-job invalid input,
and sentinels past every count."""
import ctypes as C

import numpy as np

import mvo_b200
import vo_init_batch_cases as vi

INVALID_ARG, UNSUPPORTED = -1, -5
OUT = mvo_b200.MAP_MATCHES_RESULT_DTYPE
KP, DM = mvo_b200.KEYPOINT_DTYPE, mvo_b200.DMATCH_DTYPE
K = np.array([[500.0, 0, 320.0], [0, 500.0, 240.0], [0, 0, 1]])
ROWS, COLS = 480, 640
RADIUS = 5.0
SENTINEL = vi.SENTINEL
T_GEN = vi.T_REF


def launches(method, n_map=1):
    return 0 if n_map < 0 else (1 if n_map == 0 else (3 if method == 3 else 2))


def rot(w):
    return vi.rot(w)


def pose(w, c, base=None):
    T = np.eye(4)
    T[:3, :3] = rot(w) if np.linalg.norm(w) > 0 else np.eye(3)
    T[:3, 3] = c
    return T if base is None else np.asarray(base) @ T


# ---- the state machine's host arithmetic (vo_pipeline.cpp: project_in_frame, mvo_internal.h: inv_rigid / pre_translate) ----
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


def candidates(map_pts, T_w_c, Kc=K, rows=ROWS, cols=COLS):
    """getMappointsInCurrentView_: map indices and pixels of the points in view, in map order.  numpy's elementwise float64
    products and sums round one by one, in the order written, as pre_translate / project_in_frame do."""
    Tcw = vi.inv_rigid([float(x) for x in np.ravel(T_w_c)])
    P = np.asarray(map_pts, np.float32).astype(np.float64).reshape(-1, 3)
    pc = []
    for r in range(3):
        a = np.zeros(len(P))
        a = a + Tcw[r * 4] * P[:, 0]
        a = a + Tcw[r * 4 + 1] * P[:, 1]
        a = a + Tcw[r * 4 + 2] * P[:, 2]
        a = a + Tcw[r * 4 + 3] * 1.0
        pc.append(a.astype(np.float32).astype(np.float64))
    with np.errstate(all="ignore"):
        u = (Kc[0, 0] * pc[0] / pc[2] + Kc[0, 2]).astype(np.float32)
        w = (Kc[1, 1] * pc[1] / pc[2] + Kc[1, 2]).astype(np.float32)
        keep = ~(pc[2] < 0) & (u > 0) & (w > 0) & (u < np.float32(cols)) & (w < np.float32(rows))
    idx = np.nonzero(keep)[0].astype(np.int32)
    return idx, np.ascontiguousarray(np.stack([u[idx], w[idx]], 1), np.float32).reshape(-1, 2)


def with_jobs(s, idx):
    """A shallow copy of scene s whose jobs are s's jobs idx (repeats allowed)."""
    import copy
    t = copy.copy(s)
    idx = np.asarray(idx)
    t.frames, t.T, t.n_jobs = np.ascontiguousarray(s.frames[idx]), np.ascontiguousarray(s.T[idx]), len(idx)
    t.n_bad = int(sum(1 for i in idx if i >= s.n_jobs - s.n_bad))
    return t


def project(T_w_c, X):
    """Pixels of world points X (float64, for building scenes only)."""
    Tcw = np.linalg.inv(np.asarray(T_w_c))
    Xc = X @ Tcw[:3, :3].T + Tcw[:3, 3]
    return np.stack([K[0, 0] * Xc[:, 0] / Xc[:, 2] + K[0, 2], K[1, 1] * Xc[:, 1] / Xc[:, 2] + K[1, 2]], 1), Xc[:, 2]


class Scene:
    """A map of n_map points and the frames / jobs of one call (see the module docstring)."""

    def __init__(self, cap, n_map=400, seed=0, dup_every=9):
        rng = np.random.default_rng(seed)
        self.cap = cap
        T_id = np.eye(4)
        self.T_gen, self.T_id = T_GEN, T_id
        pts = []
        # half the map in front of the general pose, half in front of the identity pose, some behind both
        n_gen, n_id = n_map // 2 - 20, n_map // 2 - 20
        for T, n in ((T_GEN, n_gen), (T_id, n_id)):
            Xc = np.stack([rng.uniform(-2.5, 2.5, n), rng.uniform(-1.8, 1.8, n), rng.uniform(3, 7, n)], 1)
            pts.append(Xc @ np.asarray(T)[:3, :3].T + np.asarray(T)[:3, 3])
        pts.append(np.stack([rng.uniform(-2, 2, 8), rng.uniform(-2, 2, 8), rng.uniform(-6, -1, 8)], 1))       # behind both
        # exact points seen by the identity guess (T_c_w = identity, t = -0.0): camera z = +0.0 / -0.0, pixels on the borders
        special = [(-1.0, -1.0, 0.0), (1.0, 0.5, -0.0), (-1.0, -1.0, -0.0), (0.0, 0.0, 0.0),
                   (-320.0, 10.0, 500.0), (320.0, 10.0, 500.0), (10.0, -240.0, 500.0), (10.0, 240.0, 500.0),   # u = 0 / cols, v = 0 / rows
                   (-319.0, 10.0, 500.0), (319.0, -239.0, 500.0),                                              # just inside
                   (20.0, 30.0, 500.0), (40.0, -30.0, 500.0)]                                                  # radius cases
        pts.append(np.array(special))
        X = np.concatenate(pts)
        n_map = len(X) if n_map >= len(X) else n_map
        X = X[:n_map] if len(X) > n_map else X
        rest = n_map - len(X)
        if rest > 0:
            X = np.concatenate([X, np.stack([rng.uniform(-2, 2, rest), rng.uniform(-1, 1, rest), rng.uniform(3, 7, rest)], 1)])
        self.map_pts = np.ascontiguousarray(X, np.float32)
        self.n_map = len(self.map_pts)
        self.map_desc = np.ascontiguousarray(rng.integers(0, 256, (self.n_map, 32), dtype=np.uint8))
        if dup_every:
            for i in range(dup_every, self.n_map, dup_every):
                self.map_desc[i] = self.map_desc[i - dup_every]        # exact duplicates: removeDuplicatedMatches ties
        self.special0 = n_gen + n_id + 8

        # frames: 0 sees the map from the general pose, 1 from the identity pose, 2 has no keypoints, 3 one keypoint,
        # 4 a negative count, 5 a count past cap (frame 0's keypoints and more)
        f0, f1 = self._frame(rng, T_GEN, 0.8 * cap), self._frame(rng, T_id, 0.7 * cap, radius_cases=True)
        frames = [(f0, len(f0[0])), (f1, len(f1[0])), (None, 0), (self._frame(rng, T_id, 0.7 * cap), 1), (None, -5),
                  (self._frame(rng, T_GEN, cap), cap + 37)]
        self.batch = len(frames)
        self.kpts = np.zeros((self.batch, cap), KP)
        self.desc = np.full((self.batch, cap, 32), SENTINEL, np.uint8)
        self.counts = np.zeros(self.batch, np.int32)
        for f, (fr, n) in enumerate(frames):
            self.counts[f] = n
            if fr is not None:
                kp, d = fr
                m = len(kp)
                self.kpts[f, :m], self.desc[f, :m] = kp, d
        self.kpts["class_id"] = -1
        self.kpts = np.ascontiguousarray(self.kpts)

        away = pose((0.0, 0.0, 0.0), (0.0, 0.0, 1000.0))                     # the whole map is behind it
        moved = pose((0.01, -0.02, 0.015), (0.05, -0.02, 0.03), T_GEN)
        jobs = [(0, T_GEN), (1, T_id), (0, moved), (2, T_GEN), (3, T_id), (4, T_id), (5, T_GEN), (0, T_GEN),   # 7 repeats 0
                (1, away), (3, T_id)]
        bad = []
        nanpose = T_GEN.copy(); nanpose[1, 2] = np.nan
        infpose = T_GEN.copy(); infpose[3, 3] = np.inf
        inftr = T_GEN.copy(); inftr[0, 3] = -np.inf
        bad = [(-1, T_GEN), (self.batch, T_GEN), (0, nanpose), (0, infpose), (1, inftr)]
        jobs += bad
        self.n_bad = len(bad)
        self.frames = np.array([j[0] for j in jobs], np.int32)
        self.T = np.ascontiguousarray(np.stack([np.asarray(j[1], np.float64) for j in jobs]))
        self.n_jobs = len(jobs)

    def _frame(self, rng, T, n, radius_cases=False):
        """Keypoints: noisy projections of the map points this pose sees (descriptors with 0..12 flipped bits), then unrelated ones."""
        n = int(n)
        with np.errstate(all="ignore"):
            uv, z = project(T, self.map_pts.astype(np.float64))
        vis = np.where((z > 0) & (uv[:, 0] > 2) & (uv[:, 1] > 2) & (uv[:, 0] < COLS - 2) & (uv[:, 1] < ROWS - 2))[0]
        vis = rng.permutation(vis)[: int(0.7 * n)]
        xy = uv[vis] + rng.normal(0, 1.5, (len(vis), 2))
        d = self.map_desc[vis].copy()
        for r in range(len(d)):
            for b in rng.choice(256, rng.integers(0, 13), replace=False):
                d[r, b // 8] ^= np.uint8(1 << (b % 8))
        if radius_cases:                                                       # map points special0 + 10 / 11 at (340, 270) / (360, 210)
            s = self.special0
            xy = np.concatenate([xy, [[340.0 + RADIUS, 270.0], [360.0, 210.0 + RADIUS + 0.5]]])
            d = np.concatenate([d, self.map_desc[[s + 10, s + 11]]])
        m = n - len(xy)
        xy = np.concatenate([xy, rng.uniform([0, 0], [COLS, ROWS], (max(m, 0), 2))])[:n]
        d = np.concatenate([d, rng.integers(0, 256, (max(m, 0), 32), dtype=np.uint8)])[:n]
        order = rng.permutation(n)
        kp = np.zeros(n, KP)
        kp["x"], kp["y"] = xy[order, 0], xy[order, 1]
        kp["size"], kp["angle"], kp["response"] = 31.0, rng.uniform(0, 360, n), rng.uniform(0, 1, n)
        return kp, np.ascontiguousarray(d[order])


def reference(lib, ctx, s, j, method, radius=RADIUS):
    """(status, record, candidate indices, candidate pixels, matches, pts3d, pts2d) of job j."""
    f, T = int(s.frames[j]), s.T[j]
    if f < 0 or f >= s.batch or not np.isfinite(T).all():
        return INVALID_ARG, None, None, None, None, None, None
    cand, cxy = candidates(s.map_pts, T)
    n1, n2 = len(cand), min(max(int(s.counts[f]), 0), s.cap)
    out = np.zeros(max(n1, 1), DM)
    nm = C.c_int(0)
    if n1 > 0 and n2 > 0 and not (method == 2 and n2 < 2):                   # match_into
        cd = np.ascontiguousarray(s.map_desc[cand])
        kxy = np.ascontiguousarray(np.stack([s.kpts[f, :n2]["x"], s.kpts[f, :n2]["y"]], 1).astype(np.float32))
        rc = lib.mvo_match_features(ctx, cd.ctypes.data, n1, np.ascontiguousarray(s.desc[f, :n2]).ctypes.data, n2, method,
                                    np.ascontiguousarray(cxy).ctypes.data, kxy.ctypes.data, C.c_float(radius), out.ctypes.data,
                                    C.byref(nm))
        assert rc == 0, rc
    m = out[: nm.value].copy()
    p3 = np.ascontiguousarray(s.map_pts[cand[m["query_idx"]]]) if len(m) else np.zeros((0, 3), np.float32)
    p2 = np.stack([s.kpts[f]["x"][m["train_idx"]], s.kpts[f]["y"][m["train_idx"]]], 1).astype(np.float32)
    rec = np.zeros(1, OUT)[0]
    rec["status"], rec["n_candidates"], rec["n_matches"] = 0, n1, len(m)
    return 0, rec, cand, cxy, m, p3, p2


def outputs(n_jobs, n_map, cap, xy=True, pnp=True):
    def buf(n, dt):
        return np.full(max(n, 1) * np.dtype(dt).itemsize, SENTINEL, np.uint8).view(dt)
    out = buf(n_jobs, OUT)
    cand = buf(n_jobs * n_map, np.int32).reshape(-1)
    cxy = buf(n_jobs * n_map * 2, np.float32) if xy else None
    m = buf(n_jobs * cap, DM)
    p3 = buf(n_jobs * cap * 3, np.float32) if pnp else None
    p2 = buf(n_jobs * cap * 2, np.float32) if pnp else None
    return out, cand, cxy, m, p3, p2


def call(lib, ctx, s, method, ptr=lambda a: a.ctypes.data, outs=None, n_jobs=None, n_map=None, Kp=None, rows=ROWS, cols=COLS, cap=None,
         batch=None, radius=RADIUS, frames=None):
    """The call over host arrays (the emulated library) or, with ptr / outs, over device copies."""
    n_map = s.n_map if n_map is None else n_map
    outs = outs or outputs(s.n_jobs, max(n_map, 0), s.cap)
    out, cand, cxy, m, p3, p2 = outs
    Kh = np.ascontiguousarray(K if Kp is None else Kp, np.float64)
    opt = (lambda a: None if a is None else ptr(a))
    rc = lib.mvo_vo_map_matches_batch_dev(ctx, ptr(s.kpts), ptr(s.desc), ptr(s.counts), s.batch if batch is None else batch,
                                          s.cap if cap is None else cap, ptr(s.frames if frames is None else frames), ptr(s.T),
                                          s.n_jobs if n_jobs is None else n_jobs, ptr(s.map_pts), ptr(s.map_desc), n_map,
                                          Kh.ctypes.data, rows, cols, method, C.c_float(radius), ptr(out), ptr(cand), opt(cxy), ptr(m),
                                          opt(p3), opt(p2))
    return rc, outs


def views(got, n_jobs, n_map, cap):
    out, cand, cxy, m, p3, p2 = got
    return (out, cand.reshape(n_jobs, max(n_map, 0)) if n_map else cand, None if cxy is None else cxy.reshape(n_jobs, n_map, 2),
            m.reshape(n_jobs, cap), None if p3 is None else p3.reshape(n_jobs, cap, 3), None if p2 is None else p2.reshape(n_jobs, cap, 2))


def check_failed(got, j, status, n_map, cap):
    """A failed job writes its status and nothing else."""
    out, cand, cxy, m, p3, p2 = views(got, len(got[0]), n_map, cap)
    assert out[j]["status"] == status, (j, out[j]["status"], status)
    assert (out[j:j + 1].view(np.uint8)[4:] == SENTINEL).all(), j
    for a in (cand, cxy, m, p3, p2):
        if a is not None and a.size:
            assert (a[j].view(np.uint8) == SENTINEL).all(), j


def check_exact(ref, got, j, n_map, cap):
    """Every byte of the record and of the rows, and sentinels past every count."""
    st, rec, cand, cxy, m, p3, p2 = ref
    if rec is None:
        check_failed(got, j, st, n_map, cap)
        return
    gout, gcand, gcxy, gm, gp3, gp2 = views(got, len(got[0]), n_map, cap)
    assert gout[j:j + 1].tobytes() == rec.tobytes(), (j, gout[j], rec)
    nc, nm = len(cand), len(m)
    if n_map:
        assert gcand[j, :nc].tobytes() == cand.tobytes(), j
        assert (gcand[j, nc:].view(np.uint8) == SENTINEL).all(), j
        if gcxy is not None:
            assert gcxy[j, :nc].tobytes() == np.ascontiguousarray(cxy).tobytes(), j
            assert (gcxy[j, nc:].view(np.uint8) == SENTINEL).all(), j
    assert gm[j, :nm].tobytes() == m.tobytes(), (j, gm[j, :nm][:5], m[:5])
    assert (gm[j, nm:].view(np.uint8) == SENTINEL).all(), j
    if gp3 is not None:
        assert gp3[j, :nm].tobytes() == np.ascontiguousarray(p3, np.float32).tobytes(), j
        assert gp2[j, :nm].tobytes() == np.ascontiguousarray(p2, np.float32).tobytes(), j
        assert (gp3[j, nm:].view(np.uint8) == SENTINEL).all() and (gp2[j, nm:].view(np.uint8) == SENTINEL).all(), j


def check_scene_coverage(lib, ctx, s, refs, method):
    """The fabricated batch reaches what it was built for."""
    recs = [r[1] for r in refs]
    assert recs[0]["n_candidates"] > 50 and recs[0]["n_matches"] > 20, recs[0]
    assert recs[1]["n_candidates"] > 50 and recs[1]["n_matches"] > 20, recs[1]
    assert recs[2]["n_candidates"] != recs[0]["n_candidates"] or refs[2][2].tobytes() != refs[0][2].tobytes()
    assert recs[3]["n_matches"] == 0 and recs[3]["n_candidates"] > 0            # no keypoints
    assert recs[5]["n_matches"] == 0                                            # negative count
    assert recs[7].tobytes() == recs[0].tobytes()                               # repeated job
    assert recs[8]["n_candidates"] == 0 and recs[8]["n_matches"] == 0           # nothing in view
    if method == 2:
        assert recs[4]["n_matches"] == 0 and recs[4]["n_candidates"] > 0        # one keypoint: knnMatch needs two
    else:
        assert recs[4]["n_matches"] <= 1
    assert [r[0] for r in refs[-s.n_bad:]] == [INVALID_ARG] * s.n_bad
    sp = s.special0
    c1 = set(refs[1][2].tolist())
    assert not any(sp + k in c1 for k in range(8)), "z = 0 / -0 and border pixels are out of view"
    assert sp + 8 in c1 and sp + 9 in c1 and sp + 10 in c1 and sp + 11 in c1
    if method == 3:
        # the keypoint exactly at the radius from point sp + 10 is matched (by it, or by a point with the same descriptor that
        # removeDuplicatedMatches keeps); the one just beyond the radius from sp + 11 is not matched to sp + 11
        m, cand = refs[1][4], refs[1][2]
        kx, ky = s.kpts[1]["x"], s.kpts[1]["y"]
        at = int(np.nonzero((kx == np.float32(340.0 + RADIUS)) & (ky == np.float32(270.0)))[0][0])
        beyond = int(np.nonzero((kx == np.float32(360.0)) & (ky == np.float32(210.0 + RADIUS + 0.5)))[0][0])
        assert at in set(m["train_idx"].tolist())
        assert not any(int(cand[q]) == sp + 11 and t == beyond for q, t in zip(m["query_idx"], m["train_idx"]))
