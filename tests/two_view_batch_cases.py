"""Batches for mvo_esti_motion_by_essential_batch_dev (tests/test_two_view_batch_emu.py, tests/test_two_view_batch_gpu.py): frames in the
layout of mvo_orb_extract_batch_dev with match lists in the layout of mvo_match_features_batch_dev, built from known
correspondences, and the per-pair reference (mvo_estimate_relative_poses with calc_homo = 0 on the same points, through the same
library) that every pair of a batch must reproduce byte for byte.

A pair spec is one of
  ("points", pts1, pts2)   a valid pair whose correspondences are pts1[i] <-> pts2[i]
  ("bad_frame",)           a frame index outside [0, batch)
  ("count", c)             valid frames, match count c (negative, or above cap)
  ("bad_index",)           valid frames, one train_idx equal to its frame's count
Every "points" pair gets two frames of its own; its keypoints sit at shuffled rows among a few unmatched ones, the rows past a
frame's count and the match rows past a pair's count hold values that must never be read."""
import ctypes as C

import numpy as np

import mvo_synth

K = mvo_synth.K_DEFAULT
INVALID_ARG, DEGENERATE = -1, -6
SENTINEL = 0x5A                     # byte fill of every output slot before a call: failed pairs must leave it in place


def rodrigues(r):
    th = np.linalg.norm(r)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def general_scene(seed, n, noise=0.5, outliers=0.2, Km=K, planar=False):
    """Points in front of both cameras (on a plane 4 m away with 2 cm of relief when planar), projected with Km, Gaussian
    pixel noise, a fraction of the second view's points replaced by uniform ones."""
    rng = np.random.default_rng(seed)
    R = rodrigues(rng.normal(0, 0.06, 3) + 1e-9)
    t = np.array([0.25, 0.02, 0.05]) + rng.normal(0, 0.02, 3)
    z = 4.0 + rng.normal(0, 0.02, n) if planar else rng.uniform(2.5, 9, n)
    X1 = np.stack([rng.uniform(-0.45, 0.45, n) * z, rng.uniform(-0.35, 0.35, n) * z, z], 1)
    X2 = X1 @ R.T + t
    f, c = np.array([Km[0, 0], Km[1, 1]]), Km[:2, 2]
    p1 = X1[:, :2] / X1[:, 2:3] * f + c + rng.normal(0, noise, (n, 2))
    p2 = X2[:, :2] / X2[:, 2:3] * f + c + rng.normal(0, noise, (n, 2))
    bad = rng.random(n) < outliers
    p2[bad] = rng.uniform([0, 0], [640, 480], (bad.sum(), 2))
    return p1.astype(np.float32), p2.astype(np.float32)


def random_pair(seed, n):
    """No geometry at all: every correspondence is an outlier."""
    rng = np.random.default_rng(seed)
    return rng.uniform([0, 0], [640, 480], (n, 2)).astype(np.float32), rng.uniform([0, 0], [640, 480], (n, 2)).astype(np.float32)


class Batch:
    """kpts [batch][cap], counts [batch], pairs [n_pairs][2], matches [n_pairs][cap], n_matches [n_pairs] (host arrays) and, per
    pair, its points or None (an invalid pair)."""

    def __init__(self, specs, cap, seed=0):
        import mvo_b200
        rng = np.random.default_rng(seed)
        n_frames = max(2, 2 * sum(s[0] == "points" for s in specs))
        self.cap = cap
        self.kpts = np.zeros((n_frames, cap), mvo_b200.KEYPOINT_DTYPE)
        self.kpts["x"], self.kpts["y"], self.kpts["class_id"] = 1e30, -1e30, -1          # rows past a count: never read
        self.counts = np.full(n_frames, 3, np.int32)
        self.pairs = np.zeros((len(specs), 2), np.int32)
        self.matches = np.zeros((len(specs), cap), mvo_b200.DMATCH_DTYPE)
        self.matches["query_idx"], self.matches["train_idx"] = -7, cap + 7                 # rows past a pair's count: never read
        self.n_matches = np.zeros(len(specs), np.int32)
        self.points = []
        f = 0
        for p, s in enumerate(specs):
            if s[0] != "points":
                self.points.append(None)
                continue
            p1, p2 = s[1], s[2]
            n = len(p1)
            extra = min(cap - n, int(rng.integers(0, 20)))
            for fr, pts in ((f, p1), (f + 1, p2)):
                rows = rng.permutation(n + extra)
                self.kpts["x"][fr, rows[:n]] = pts[:, 0]
                self.kpts["y"][fr, rows[:n]] = pts[:, 1]
                self.kpts["x"][fr, rows[n:]] = rng.uniform(0, 640, extra)
                self.kpts["y"][fr, rows[n:]] = rng.uniform(0, 480, extra)
                self.counts[fr] = n + extra
                self.matches[p, :n]["query_idx" if fr == f else "train_idx"] = rows[:n]
            self.matches[p, :n]["img_idx"] = 0
            self.matches[p, :n]["distance"] = rng.integers(0, 60, n)
            self.pairs[p] = (f, f + 1)
            self.n_matches[p] = n
            self.points.append((p1, p2))
            f += 2
        if f == 0:
            self.counts[:] = 0
        for p, s in enumerate(specs):
            if s[0] == "bad_frame":
                self.pairs[p] = (0, n_frames + 3) if p % 2 else (-1, 0)
                self.n_matches[p] = min(10, self.counts[0])
                self.matches[p, :self.n_matches[p]]["query_idx"] = 0
                self.matches[p, :self.n_matches[p]]["train_idx"] = 0
            elif s[0] == "count":
                self.pairs[p] = (0, 1)
                self.n_matches[p] = s[1]
            elif s[0] == "bad_index":
                self.pairs[p] = (0, 1)
                n = int(min(self.counts[0], self.counts[1]))
                self.n_matches[p] = n
                self.matches[p, :n]["query_idx"] = np.arange(n)
                self.matches[p, :n]["train_idx"] = np.arange(n)
                self.matches["train_idx"][p, n // 2] = self.counts[1]
        self.batch = n_frames

    @property
    def n_pairs(self):
        return len(self.pairs)


def outputs(n_pairs, cap):
    """Sentinel-filled output arrays: results, inlier rows, triangulated points."""
    import mvo_b200
    res = np.frombuffer(bytearray([SENTINEL]) * (n_pairs * mvo_b200.TWO_VIEW_RESULT_DTYPE.itemsize), mvo_b200.TWO_VIEW_RESULT_DTYPE).copy()
    inl = np.frombuffer(bytearray([SENTINEL]) * (n_pairs * cap * 4), np.int32).reshape(n_pairs, cap).copy()
    pts = np.frombuffer(bytearray([SENTINEL]) * (n_pairs * cap * 12), np.float32).reshape(n_pairs, cap, 3).copy()
    return res, inl, pts


def reference(lib, h, p1, p2, Km):
    """mvo_estimate_relative_poses(calc_homo = 0, motion_cam2_to_cam1 = 1) on one pair: (status, E, R, t, inliers, pts3d) of its
    solution 0.  The context's essential_threshold is the batch call's threshold."""
    import mvo_b200
    n = len(p1)
    p1, p2 = np.ascontiguousarray(p1, np.float32), np.ascontiguousarray(p2, np.float32)
    Kc = np.ascontiguousarray(Km, np.float64)
    sol = mvo_b200.TwoViewSolutions()
    inl = np.zeros(max(n, 1), np.int32)
    pts = np.zeros((max(n, 1), 3), np.float32)
    rc = lib.mvo_estimate_relative_poses(h, p1.ctypes.data, p2.ctypes.data, n, Kc.ctypes.data, 0, 1, C.byref(sol), inl.ctypes.data,
                                         pts.ctypes.data)
    if rc != 0:
        return rc, None
    ni = sol.n_inliers[0]
    return 0, dict(n_inliers=ni, E=np.array(sol.E[:]), R=np.array(sol.R[0][:]), t=np.array(sol.t[0][:]), inliers=inl[:ni].copy(),
                   pts3d=pts[:ni].copy())


def check_pair(batch, p, res, inl, pts, ref, with_pts=True):
    """Pair p of a batch call against its reference (status, dict); failed pairs must have written their status only."""
    import mvo_b200
    r = res[p]
    rc, want = ref
    sentinel_rec = np.frombuffer(bytes([SENTINEL]) * mvo_b200.TWO_VIEW_RESULT_DTYPE.itemsize, mvo_b200.TWO_VIEW_RESULT_DTYPE)[0]
    cap = batch.cap
    if rc != 0:
        assert r["status"] == rc, (p, r["status"], rc)
        assert r.tobytes()[4:] == sentinel_rec.tobytes()[4:], p          # nothing but the status written
        assert (inl[p].view(np.uint8) == SENTINEL).all(), p
        assert (pts[p].view(np.uint8) == SENTINEL).all(), p
        return
    assert r["status"] == 0, (p, r["status"])
    ni = want["n_inliers"]
    assert r["n_matches"] == batch.n_matches[p] and r["n_inliers"] == ni, (p, r["n_matches"], r["n_inliers"], ni)
    assert 0 <= r["votes"] <= ni, (p, r["votes"], ni)          # 0: no candidate puts a point within 50 depth units (little parallax)
    assert r["E"].tobytes() == want["E"].tobytes(), p
    assert r["R"].tobytes() == want["R"].tobytes(), p
    assert r["t"].tobytes() == want["t"].tobytes(), (p, r["t"], want["t"])
    assert inl[p, :ni].tobytes() == want["inliers"].tobytes(), p
    assert (inl[p, ni:].view(np.uint8) == SENTINEL).all(), p
    if with_pts:
        assert pts[p, :ni].tobytes() == want["pts3d"].tobytes(), p
        assert (pts[p, ni:].view(np.uint8) == SENTINEL).all(), p
    else:
        assert (pts[p].view(np.uint8) == SENTINEL).all(), p
    assert cap >= ni


def references(lib, h, batch, Km):
    return [reference(lib, h, pp[0], pp[1], Km) if pp is not None else (INVALID_ARG, None) for pp in batch.points]


def launches_per_call(with_pts):
    """The constant of include/mvo.h: gather, hypotheses, scoring, finish, vote, pick (+ triangulation)."""
    return 7 if with_pts else 6
