"""Batches for mvo_estimate_relative_poses_batch_dev (tests/test_relative_poses_batch_emu.py, tests/test_relative_poses_batch_gpu.py).
The frame / match layouts, the scene builders and the sentinel fill are those of two_view_batch_cases.py; this module adds the scenes
whose true motion is known (for the check against the truth), the per-pair reference (mvo_estimate_relative_poses with calc_homo = 1
on the same points, through the same library) and the record-by-record, row-by-row comparison."""
import ctypes as C

import numpy as np

import two_view_batch_cases as tvb

K = tvb.K
SENTINEL = tvb.SENTINEL
INVALID_ARG, DEGENERATE = tvb.INVALID_ARG, tvb.DEGENERATE
X86_DEFAULT_NAN = 0xFFF8000000000000          # what 0 / 0 gives on the host (mvo.h): the device writes these bits for a NaN


def general_truth(seed):
    """(R, t) of tvb.general_scene(seed, ...): its first two draws, x2 ~ R x1 + t."""
    rng = np.random.default_rng(seed)
    R = tvb.rodrigues(rng.normal(0, 0.06, 3) + 1e-9)
    t = np.array([0.25, 0.02, 0.05]) + rng.normal(0, 0.02, 3)
    return R, t


def project(X, Km):
    f, c = np.array([Km[0, 0], Km[1, 1]]), Km[:2, 2]
    return X[:, :2] / X[:, 2:3] * f + c


def planar_scene(seed, n, noise=0.3, tilt=0.3, move=(0.4, 0.05, 0.05), Km=K):
    """Points on a tilted plane about 4 m in front of camera 1, seen after a move of about `move`: (p1, p2, R, t)."""
    rng = np.random.default_rng(seed)
    R = tvb.rodrigues(rng.normal(0, 0.05, 3) + 1e-9)
    t = np.array(move) + rng.normal(0, 0.03, 3)
    nrm = np.array([rng.uniform(-tilt, tilt), rng.uniform(-tilt, tilt), 1.0])
    nrm /= np.linalg.norm(nrm)
    rays = np.stack([rng.uniform(-0.45, 0.45, n), rng.uniform(-0.35, 0.35, n), np.ones(n)], 1)
    X1 = rays * (4.0 / (rays @ nrm))[:, None]
    X2 = X1 @ R.T + t
    p1 = project(X1, Km) + rng.normal(0, noise, (n, 2))
    p2 = project(X2, Km) + rng.normal(0, noise, (n, 2))
    return p1.astype(np.float32), p2.astype(np.float32), R, t


def rotation_scene(seed, n, far=0.6, Km=K):
    """A camera that moves sideways without turning in front of a scene whose points are mostly at infinity: those appear at
    the same pixel in both views (a pure rotation, R = I, for the homography: decompose_homography returns its single t = n = 0
    solution, which the visibility filter removes), the near ones carry the translation.  (p1, p2, R, t)."""
    rng = np.random.default_rng(seed)
    R, t = np.eye(3), np.array([0.3, 0.0, 0.02])
    p1 = np.stack([rng.uniform(20, 620, n), rng.uniform(20, 460, n)], 1).astype(np.float32)
    p2 = p1.copy()
    near = rng.random(n) >= far
    z = rng.uniform(2.5, 9, near.sum())
    X1 = np.concatenate([(p1[near] - Km[:2, 2]) / np.array([Km[0, 0], Km[1, 1]]), np.ones((near.sum(), 1))], 1) * z[:, None]
    p2[near] = (project(X1 @ R.T + t, Km) + rng.normal(0, 0.3, (near.sum(), 2))).astype(np.float32)
    return p1, p2, R, t


def outputs(n_pairs, cap):
    """Sentinel-filled output arrays: records, inlier rows [pair][5][cap], triangulated points [pair][5][cap][3]."""
    import mvo_b200
    res = np.frombuffer(bytearray([SENTINEL]) * (n_pairs * mvo_b200.RELATIVE_POSES_RESULT_DTYPE.itemsize),
                        mvo_b200.RELATIVE_POSES_RESULT_DTYPE).copy()
    inl = np.frombuffer(bytearray([SENTINEL]) * (n_pairs * 5 * cap * 4), np.int32).reshape(n_pairs, 5, cap).copy()
    pts = np.frombuffer(bytearray([SENTINEL]) * (n_pairs * 5 * cap * 12), np.float32).reshape(n_pairs, 5, cap, 3).copy()
    return res, inl, pts


def reference(lib, h, p1, p2, Km, motion_cam2_to_cam1):
    """mvo_estimate_relative_poses(calc_homo = 1) on one pair: (status, dict(sol = the struct's bytes, inliers, pts3d))."""
    import mvo_b200
    n = len(p1)
    p1, p2 = np.ascontiguousarray(p1, np.float32), np.ascontiguousarray(p2, np.float32)
    Kc = np.ascontiguousarray(Km, np.float64)
    sol = mvo_b200.TwoViewSolutions()
    inl = np.zeros((5, max(n, 1)), np.int32)
    pts = np.zeros((5, max(n, 1), 3), np.float32)
    rc = lib.mvo_estimate_relative_poses(h, p1.ctypes.data, p2.ctypes.data, n, Kc.ctypes.data, 1, int(motion_cam2_to_cam1), C.byref(sol),
                                         inl.ctypes.data, pts.ctypes.data)
    if rc != 0:
        return rc, None
    return 0, dict(sol=bytes(sol), num=sol.num_solutions, n_inliers=list(sol.n_inliers), best=sol.best, ratio=sol.ratio,
                   inliers=inl.copy(), pts3d=pts.copy())


def references(lib, h, batch, Km, motion_cam2_to_cam1):
    return [reference(lib, h, pp[0], pp[1], Km, motion_cam2_to_cam1) if pp is not None else (INVALID_ARG, None) for pp in batch.points]


def check_pair(batch, p, res, inl, pts, ref, with_pts=True):
    """Pair p of a batch call against its reference: every byte of the record, every inlier row and triangulated row; a failed pair
    must have written its status and match count only, unused rows must still hold the sentinel."""
    import mvo_b200
    r = res[p]
    rc, want = ref
    itemsize = mvo_b200.RELATIVE_POSES_RESULT_DTYPE.itemsize
    assert r["n_matches"] == batch.n_matches[p], (p, r["n_matches"], batch.n_matches[p])
    if rc != 0:
        assert r["status"] == rc, (p, r["status"], rc)
        assert r.tobytes()[8:] == bytes([SENTINEL]) * (itemsize - 8), p
        assert (inl[p].view(np.uint8) == SENTINEL).all(), p
        assert (pts[p].view(np.uint8) == SENTINEL).all(), p
        return
    assert r["status"] == 0, (p, r["status"])
    assert r.tobytes()[8:] == want["sol"], (p, diff_fields(r, want["sol"]))
    n = len(batch.points[p][0])
    for s in range(5):
        ni = want["n_inliers"][s] if s < want["num"] else 0
        assert inl[p, s, :ni].tobytes() == want["inliers"][s, :ni].tobytes(), (p, s)
        assert (inl[p, s, ni:].view(np.uint8) == SENTINEL).all(), (p, s)
        if with_pts:
            assert pts[p, s, :ni].tobytes() == want["pts3d"][s, :ni].tobytes(), (p, s)
            assert (pts[p, s, ni:].view(np.uint8) == SENTINEL).all(), (p, s)
        else:
            assert (pts[p, s].view(np.uint8) == SENTINEL).all(), (p, s)
    assert max(want["n_inliers"]) <= min(n, batch.cap)


def diff_fields(rec, want_bytes):
    """Names of the fields of a record whose bytes differ from a TwoViewSolutions' bytes (for the assertion message)."""
    import mvo_b200
    w = np.frombuffer(bytes(8) + want_bytes, mvo_b200.RELATIVE_POSES_RESULT_DTYPE)[0]
    return [f for f in mvo_b200.RELATIVE_POSES_RESULT_DTYPE.names[2:] if rec[f].tobytes() != w[f].tobytes()]


def rotation_angle(Ra, Rb):
    c = (np.trace(Ra.T @ Rb) - 1) / 2
    return float(np.arccos(np.clip(c, -1, 1)))


def check_truth(rec, R_true, t_true, motion_cam2_to_cam1, rot_tol=0.02, dir_tol=0.2):
    """The chosen solution of an MVO_OK record against the scene's true motion (x2 ~ R x1 + t), t up to scale."""
    b = int(rec["best"])
    R, t = rec["R"][b].reshape(3, 3), rec["t"][b]
    if not motion_cam2_to_cam1:                    # the record holds the inverse motion
        R, t = R.T, -R.T @ t
    assert rotation_angle(R, R_true) < rot_tol, (b, rotation_angle(R, R_true))
    cosang = float(t @ t_true) / (np.linalg.norm(t) * np.linalg.norm(t_true))
    assert np.arccos(np.clip(cosang, -1, 1)) < dir_tol, (b, t, t_true)


def launches_per_call(with_pts):
    """The constant of include/mvo.h: the essential half (6), the homography half (3), the combine step (+ triangulation)."""
    return 11 if with_pts else 10


def call(lib, ctx, b, motion_cam2_to_cam1, with_pts, Km=K):
    res, inl, pts = outputs(b.n_pairs, b.cap)
    Kc = np.ascontiguousarray(Km, np.float64)
    l0 = lib.mvo_kernel_launches(ctx)
    rc = lib.mvo_estimate_relative_poses_batch_dev(ctx, b.kpts.ctypes.data, b.counts.ctypes.data, b.batch, b.cap, b.pairs.ctypes.data,
                                                   b.n_pairs, b.matches.ctypes.data, b.n_matches.ctypes.data, Kc.ctypes.data,
                                                   int(motion_cam2_to_cam1), res.ctypes.data, inl.ctypes.data,
                                                   pts.ctypes.data if with_pts else None)
    assert rc == 0, lib.mvo_last_error(ctx)
    assert lib.mvo_kernel_launches(ctx) - l0 == launches_per_call(with_pts)
    return res, inl, pts
