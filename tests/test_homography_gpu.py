"""GPU check of the homography half of the two-view stage (mvo_esti_motion_by_homography,
mvo_remove_wrong_rt_of_homography; reference src/geometry/epipolar_geometry.cpp:59-128) against the reference's
arithmetic (oracle/epipolar_oracle.py = cv2.findHomography + decomposeHomographyMat + filterHomographyDecompByVisibleRefpoints).

The check runs in a CHILD process so that a faulting kernel
cannot take the rest of the suite with it."""
import subprocess
import sys
from pathlib import Path

import pytest

import os as _os
_TIMEOUT_SCALE = float(_os.environ.get("MVO_TEST_TIMEOUT_SCALE", "1"))      # > 1 when the library under test is the CPU emulation (MVO_LIB)
from conftest import have_cv2

ROOT = Path(__file__).resolve().parent.parent
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_cv2(), reason="cv2 not importable")]

CHILD = r'''
import sys
import numpy as np
sys.path.insert(0, r"{root}"); sys.path.insert(0, r"{root}/monocular-visual-odometry_b200/python")
import mvo_b200, mvo_synth
from oracle import epipolar_oracle
K = mvo_synth.K_DEFAULT

def rod(r):
    th = np.linalg.norm(r); k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx

ctx = mvo_b200.Context(0)
for seed in range(3):
    rng = np.random.default_rng(seed)
    n = 1200
    R = rod(rng.normal(0, 0.05, 3) + 1e-9)
    t = np.array([0.3, 0.03, 0.08]) + rng.normal(0, 0.02, 3)
    nrm = np.array([rng.normal(0, 0.15), rng.normal(0, 0.15), 1.0]); nrm /= np.linalg.norm(nrm)
    d = 4.0
    P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), np.zeros(n)], 1)
    P[:, 2] = (d - P[:, :2] @ nrm[:2]) / nrm[2]
    P2 = P @ R.T + t
    p1 = P[:, :2] / P[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, 0.4, (n, 2))
    p2 = P2[:, :2] / P2[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, 0.4, (n, 2))
    bad = rng.random(n) < 0.2
    p2[bad] = rng.uniform([0, 0], [640, 480], (bad.sum(), 2))
    p1, p2 = p1.astype(np.float32), p2.astype(np.float32)
    H, Rs, ts, ns, inl = ctx.esti_motion_by_homography(p1, p2, K, 3.0)
    Ho, Rso, tso, nso, inlo = epipolar_oracle.esti_motion_by_homography(p1, p2, K, 3.0)
    assert abs(H[2, 2] - 1) < 1e-12 and len(Rs) == 4
    # the homography itself: transfer error of the noise-free plane points no worse than OpenCV's (+0.1 px)
    def terr(Hm):
        q1 = np.c_[P[:, :2] / P[:, 2:3] * K[0, 0] + K[:2, 2], np.ones(n)]
        q2 = P2[:, :2] / P2[:, 2:3] * K[0, 0] + K[:2, 2]
        m = q1 @ Hm.T
        return np.sqrt(np.mean(np.sum((m[:, :2] / m[:, 2:3] - q2) ** 2, 1)))
    assert terr(H) < terr(Ho) + 0.1, (terr(H), terr(Ho))
    a, b = set(inl.tolist()), set(inlo.tolist())
    assert np.all(np.diff(inl) > 0) and len(a & b) / len(b) > 0.9 and (~bad)[inl].mean() > 0.97
    # decomposition: the true motion is among the solutions, |t| = 1, proper rotations, pairs (a, -a, b, -b)
    td = t / np.linalg.norm(t)
    err = [max(np.abs(Rs[i] - R).max(), np.abs(ts[i] - td).max(), np.abs(ns[i] - nrm).max()) for i in range(4)]
    assert min(err) < 0.02, err
    for i in range(4):
        assert abs(np.linalg.det(Rs[i]) - 1) < 1e-8 and abs(np.linalg.norm(ts[i]) - 1) < 1e-9
    assert np.allclose(ts[0], -ts[1]) and np.allclose(ns[2], -ns[3])
    # removeWrongRtOfHomography: same survivors as OpenCV's filter given the same solutions
    Ki = np.linalg.inv(K)
    np1 = ((np.c_[p1, np.ones(n)] @ Ki.T)[:, :2]).astype(np.float32)
    np2 = ((np.c_[p2, np.ones(n)] @ Ki.T)[:, :2]).astype(np.float32)
    keep = epipolar_oracle.remove_wrong_rt_of_homography(np1, np2, inl, list(Rs), list(ts), list(ns))
    R2, t2, n2 = ctx.remove_wrong_rt_of_homography(np1, np2, inl, Rs, ts, ns)
    assert len(R2) == len(keep) and all(np.array_equal(R2[j], Rs[k]) and np.array_equal(n2[j], ns[k]) for j, k in enumerate(keep))
    assert len(keep) >= 1 and int(np.argmin(err)) in keep
# ---- the assembled initialisation helper (motion_estimation.cpp:10-158) on a general scene and on a plane ----
for planar in (False, True):
    rng = np.random.default_rng(40 + planar)
    n = 900
    R = rod(rng.normal(0, 0.05, 3) + 1e-9)
    t = np.array([0.3, 0.02, 0.06])
    nrm = np.array([0.05, -0.08, 1.0]); nrm /= np.linalg.norm(nrm)
    P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2.5, 8, n)], 1)
    if planar:
        P[:, 2] = (4.0 - P[:, :2] @ nrm[:2]) / nrm[2]
    P2 = P @ R.T + t
    p1 = (P[:, :2] / P[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, 0.4, (n, 2))).astype(np.float32)
    p2 = (P2[:, :2] / P2[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, 0.4, (n, 2))).astype(np.float32)
    sols, best, info = ctx.estimate_relative_poses(p1, p2, K)
    assert 1 <= len(sols) <= 5 and 0 <= best < len(sols)
    td = t / np.linalg.norm(t)
    if not planar:
        assert best == 0, (best, info)
        s0 = sols[0]
        assert np.abs(s0["R"] - R).max() < 5e-3 and np.arccos(np.clip(s0["t"] @ td, -1, 1)) < 0.05
        X = s0["pts3d"] * np.linalg.norm(t)                        # unit baseline -> true scale
        assert np.median(np.linalg.norm(X - P[s0["inliers"]], axis=1) / np.linalg.norm(P[s0["inliers"]], axis=1)) < 0.05
    else:
        assert len(sols) >= 2 and np.allclose(sols[0]["normal"], 0)
        errs = [max(np.abs(s["R"] - R).max(), np.abs(s["t"] - td).max()) for s in sols[1:]]
        assert min(errs) < 0.03, errs                              # the true motion is among the surviving homography solutions
    sols_inv, _, _ = ctx.estimate_relative_poses(p1, p2, K, motion_cam2_to_cam1=False)
    assert np.allclose(sols_inv[0]["R"], sols[0]["R"].T, atol=1e-12) and np.allclose(sols_inv[0]["t"], -sols[0]["R"].T @ sols[0]["t"], atol=1e-12)
# six correspondences of an exactly planar scene: fewer than the essential matrix needs, enough for a homography
rng = np.random.default_rng(6)
n = 6
R, t = rod(np.array([0.02, -0.03, 0.01])), np.array([0.3, 0.02, 0.05])
nrm = np.array([0.1, -0.05, 1.0]) / np.linalg.norm([0.1, -0.05, 1.0])
P = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), np.zeros(n)], 1)
P[:, 2] = (4.0 - P[:, :2] @ nrm[:2]) / nrm[2]
P2 = P @ R.T + t
p1 = (P[:, :2] / P[:, 2:3] * K[0, 0] + K[:2, 2]).astype(np.float32)
p2 = (P2[:, :2] / P2[:, 2:3] * K[0, 0] + K[:2, 2]).astype(np.float32)
H, Rs, ts, ns, inl = ctx.esti_motion_by_homography(p1, p2, K, 3.0)          # raises unless the call returns MVO_OK
assert len(inl) >= 4
assert inl.tolist() == list(range(6)) and abs(H[2, 2] - 1) < 1e-12, (inl, H)
m = np.c_[p1.astype(np.float64), np.ones(n)] @ H.T
assert np.abs(m[:, :2] / m[:, 2:3] - p2).max() < 1e-3
try:
    ctx.esti_motion_by_homography(np.zeros((3, 2), np.float32), np.zeros((3, 2), np.float32), K)
    raise SystemExit("n < 4 was accepted")
except mvo_b200.MvoError as e:
    assert e.code == -6
print("homography child ok")
'''


def test_homography_path_in_child_process(built):
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=str(ROOT))], capture_output=True, text=True, timeout=180 * _TIMEOUT_SCALE)
    assert r.returncode == 0 and "homography child ok" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
