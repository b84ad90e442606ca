"""Cases of the RANSAC PnP (csrc/pnp.cu, pnp_kernels.cuh, pnp_cv_kernels.cuh) and their checks against the fp64 oracle
(oracle/pnp_oracle.py, p3p_oracle.py) and the float-rule restatement of cv::solvePnPRansac (oracle/pnp_cv_oracle.py), shared by
test_pnp_cases_gpu.py (the H100) and test_pnp_cases_emu.py (the emulated library on the CPU).

A case runs through the test entry mvo_test_pnp_dev, which runs the device-resident sequence of the tracker (the correspondence
count read on the device, n_upper an upper bound), optionally on caller-supplied hypotheses.  `run_case` runs it in the calling
process, `run_children` in a child process on the library MVO_LIB names.  `check` compares the result with the oracle and
with the host path mvo_solve_pnp_ransac; `config` restates the host's launch rules and says which configuration a case reaches.

Tolerances:
  * batched mode: every hypothesis's inlier count equals the fp64 oracle's exactly; a point is left undecided only where
    |err^2 - thr^2| is within 1e-10 px^2 plus the fp64 rounding bound of its projection (which exceeds 1e-10 only at large
    coordinates), or its depth is within rounding of the 1e-9 cut.  Each sample reprojects onto its pixels to 1e-6 px, the
    best hypothesis is the lowest index of the maximum count, the inlier list is its fp64 consensus set, and the refit is the
    least-squares optimum of that set to 1e-8 (times 3 |t| where the translation is large);
  * pnp_mode = 1: counts equal the float rule on the device's own poses except points within 2 float ulps of thr^2, the
    chosen iteration and the iterations run equal a replay of RANSACUpdateNumIters over the device's counts;
  * device count: hypotheses, counts and inlier list bit-identical to mvo_solve_pnp_ransac on the first min(count, n_upper)
    correspondences, the pose within 1e-12 (bit-identical where both refits launch the same k_ba_pose kernel)."""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np

import ba_pose_cases as B

ROOT = Path(__file__).resolve().parent.parent
PY = ROOT / "monocular-visual-odometry_b200" / "python"
SM_H100 = 132                     # H100 SXM; the emulated runtime reports the same
FIN_T, FIN_MAXPER = 1024, 4
SMEM_DEFAULT = 48 * 1024
N_MAX = 200 * 1024 // 20
MVO_ERR_UNSUPPORTED, MVO_ERR_DEGENERATE = -5, -6
EPS64 = np.finfo(np.float64).eps
K0 = np.array([[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1.0]])
K_FXFY = np.array([[1800.0, 0, 330.0], [0, 1750.0, 250.0], [0, 0, 1.0]])
K_OFF = np.array([[615.0, 0, 1400.0], [0, 615.0, -900.0], [0, 0, 1.0]])


# ---- the host's launch rules, restated ----------------------------------------------------------------------------------
def score_passes(H, sm=SM_H100):
    """pnp_score_finish: grid = min((H + 7) / 8, 4 SMs) CTAs of 8 warps, one hypothesis per warp per pass."""
    grid = min((H + 7) // 8, 4 * sm)
    return -(-H // (grid * 8))


def smem_optin(n_upper):
    """k_pnp_score stages the n_upper correspondences (20 B each) next to its 32 B of static shared memory; above 48 KB in
    all the launch opts in (from n = 2457 on)."""
    return n_upper * 20 + 32 > SMEM_DEFAULT


def finish_reread(n_eff):
    """k_pnp_finish keeps each thread's ceil(n / 1024) points in registers up to 4 of them, and re-reads them beyond."""
    return -(-n_eff // FIN_T) > FIN_MAXPER


def refit_kernel(n_upper, csize=8):
    """pnp_refit launches the pose LM for E = n_upper edge slots with chunk 1 (not run_ba's chunk rule): cached while
    E <= cluster x 512 threads, the uncached strided kernel beyond."""
    return "<1,true,false>" if n_upper <= csize * B.PF_T else "<1,false,false>"


def config(c, sm=SM_H100):
    """The configuration a case reaches: (mode, score passes >= 2, opt-in, finish re-read, device count)."""
    n_eff = min(c["n_upper"], max(c["count"], 0))
    if c["mode"] == 1:
        return (1, None, None, finish_reread(n_eff), c["path"] == "dev")
    return (0, score_passes(c["H"], sm) >= 2, smem_optin(c["n_upper"]), finish_reread(n_eff), c["path"] == "dev")


def feasible_cells():
    """Every cell of the matrix that exists: a re-read needs more than 4096 points, hence the opt-in; pnp_mode = 1 has neither
    a grid-stride scoring loop nor staged points."""
    cells = set()
    for dev in (False, True):
        for passes in (False, True):
            for optin, reread in ((False, False), (True, False), (True, True)):
                cells.add((0, passes, optin, reread, dev))
        for reread in (False, True):
            cells.add((1, None, None, reread, dev))
    return cells


# ---- scenes and hypotheses -------------------------------------------------------------------------------------------------
def rod(r):
    return B._rod(np.asarray(r, np.float64))


def scene(seed, n, K=K0, outl=0.3, noise=0.5, t_scale=None):
    """n correspondences of a pose (R, t): camera-frame points in a 4 x 3 x 6 box at depth 2..8, world points float32,
    pixels their projections plus noise, a fraction outl moved anywhere in a 640 x 480 image around the principal point.
    t_scale: translation components of that size (world coordinates of the same size)."""
    rng = np.random.default_rng(seed)
    R = rod(rng.normal(0, 0.3, 3))
    t = rng.uniform(-t_scale, t_scale, 3) if t_scale else rng.normal(0, 0.3, 3)
    pc = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2, 8, n)], 1)
    P = ((pc - t) @ R).astype(np.float32)
    uv, _ = project(P, R, t, K)
    uv += rng.normal(0, noise, uv.shape)
    bad = rng.random(n) < outl
    uv[bad] = np.stack([rng.uniform(-320, 320, bad.sum()), rng.uniform(-240, 240, bad.sum())], 1) + K[:2, 2]
    return P, uv.astype(np.float32), R, t


def project(P, R, t, K):
    from oracle import pnp_oracle as po
    return po.project(P, R, t, K)


def pose12(R, t):
    return np.concatenate([np.asarray(R).ravel(), np.asarray(t).ravel()])


def perturbed(rng, R, t, H, sig_r=(1e-4, 3e-2), sig_t=(1e-4, 5e-2)):
    """H poses around (R, t), each with its own perturbation size (log-uniform in the given ranges)."""
    out = np.zeros((H, 12))
    for h in range(H):
        sr = np.exp(rng.uniform(*np.log(sig_r)))
        st = np.exp(rng.uniform(*np.log(sig_t))) * max(1.0, np.abs(t).max())
        out[h] = pose12(rod(rng.normal(0, sr, 3)) @ R, t + rng.normal(0, st, 3))
    return out


def pin_to_threshold(pose, P, uv, K, i, thr, off):
    """pose with t_y moved so that point i projects onto its observation's row, and t_x so that it lies at pixel distance
    thr + off from it (in the fp64 of the oracle); None when the point is behind the camera."""
    R, t = pose[:9].reshape(3, 3), pose[9:].copy()
    pc = R @ P[i].astype(np.float64) + t
    if not pc[2] > 1e-3:
        return None
    du0 = K[0, 0] * pc[0] / pc[2] + K[0, 2] - uv[i, 0]
    dv = K[1, 1] * pc[1] / pc[2] + K[1, 2] - uv[i, 1]
    t[1] -= dv * pc[2] / K[1, 1]
    t[0] += (np.copysign(thr + off, du0) - du0) * pc[2] / K[0, 0]
    return pose12(R, t)


# ---- the oracle's counts, with the undecidable points set apart -------------------------------------------------------------
def fp64_errors(P, uv, K, poses):
    """err^2 of every (hypothesis, point) as pnp_oracle.reproj_err2 computes it (inf where z <= 1e-9), and a bound on the
    difference between two fp64 evaluations of the same expression in different operation orders: (err2, tol, z_amb)."""
    Pd = np.asarray(P, np.float64)
    uvd = np.asarray(uv, np.float64)
    R = poses[:, :9].reshape(-1, 3, 3)
    t = poses[:, 9:]
    pc = np.einsum("hij,nj->hni", R, Pd) + t[:, None, :]
    mag = np.einsum("hij,nj->hni", np.abs(R), np.abs(Pd)) + np.abs(t)[:, None, :]      # size of the terms of each coordinate
    a = 4 * EPS64 * mag
    z = pc[..., 2]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        xz, yz = pc[..., 0] / z, pc[..., 1] / z
        pu, pv = K[0, 0] * xz + K[0, 2], K[1, 1] * yz + K[1, 2]
        du, dv = pu - uvd[:, 0], pv - uvd[:, 1]
        e = du * du + dv * dv
        az = np.abs(z)
        d_u = K[0, 0] * (a[..., 0] + np.abs(xz) * a[..., 2]) / az + 4 * EPS64 * (np.abs(pu) + abs(K[0, 2]))
        d_v = K[1, 1] * (a[..., 1] + np.abs(yz) * a[..., 2]) / az + 4 * EPS64 * (np.abs(pv) + abs(K[1, 2]))
        tol = 1e-10 + 2 * (np.abs(du) * d_u + np.abs(dv) * d_v) + d_u * d_u + d_v * d_v
    z_amb = np.abs(z - 1e-9) <= a[..., 2]
    e = np.where(z > 1e-9, e, np.inf)
    return e, tol, z_amb


def oracle_counts(P, uv, K, poses, thr):
    """(sure inliers, undecided points) per hypothesis."""
    thr2 = thr * thr
    chunk = max(1, 1_000_000 // max(len(P), 1))
    sure = np.zeros(len(poses), np.int64)
    amb = np.zeros(len(poses), np.int64)
    for s in range(0, len(poses), chunk):
        e, tol, z_amb = fp64_errors(P, uv, K, poses[s:s + chunk])
        close = np.abs(e - thr2) <= tol
        und = (close & np.isfinite(e)) | (z_amb & ~(np.abs(np.where(np.isfinite(e), e, 0.0)) > thr2 + tol))
        sure[s:s + chunk] = ((e <= thr2) & ~und).sum(1)
        amb[s:s + chunk] = und.sum(1)
    return sure, amb


def consensus(P, uv, K, pose, thr):
    """(sure consensus set, undecided points) of one pose, ascending indices."""
    e, tol, z_amb = fp64_errors(P, uv, K, pose[None])
    e, tol, z_amb = e[0], tol[0], z_amb[0]
    und = (np.isfinite(e) & (np.abs(e - thr * thr) <= tol)) | z_amb
    return np.flatnonzero((e <= thr * thr) & ~und), np.flatnonzero(und)


# ---- the cases ----------------------------------------------------------------------------------------------------------------
def _case(P, uv, K, H=4096, thr=2.0, mode=0, count=None, path="dev", poses=None, valid=None, seed=0x9E3779B97F4A7C15, tie=None):
    n_upper = len(P)
    thr = float(np.float32(thr))             # mvo_params::pnp_reproj_error is a float: the device squares float(thr) in fp64
    return dict(P=np.ascontiguousarray(P, np.float32), uv=np.ascontiguousarray(uv, np.float32), K=np.asarray(K, np.float64), H=H, thr=thr,
                mode=mode, n_upper=n_upper, count=n_upper if count is None else count, path=path, poses=poses, valid=valid,
                seed=seed, tie=tie)


def batch(seed, H, n, thr=2.0, K=K0, path="dev", outl=0.3, noise=0.5):
    P, uv, _, _ = scene(seed, n, K, outl=outl, noise=noise)
    return _case(P, uv, K, H=H, thr=thr, path=path)


def dev_count(seed, n_upper, count, mode=0, H=512):
    """n_upper slots, the first `count` of a scene, the slots past the count filled with copies of its inliers (a kernel that
    scores them finds more inliers; one that gathers them returns indices past the count)."""
    P, uv, R, t = scene(seed, n_upper, outl=0.25, noise=0.3)
    m = min(max(count, 0), n_upper)
    if m < n_upper:
        src = np.arange(max(m, 1))
        e, _, _ = fp64_errors(P[src], uv[src], K0, pose12(R, t)[None])
        good = src[e[0] < 1.0] if m >= 1 else src[:0]
        if len(good) == 0:
            Pp, uvp, _, _ = scene(seed + 1, 64, outl=0.0, noise=0.3)
            R, t = None, None
            P[m:], uv[m:] = Pp[np.arange(n_upper - m) % 64], uvp[np.arange(n_upper - m) % 64]
        else:
            j = good[np.arange(n_upper - m) % len(good)]
            P[m:], uv[m:] = P[j], uv[j]
    return _case(P, uv, K0, H=H if mode == 0 else 100, mode=mode, count=count)


def adversarial(seed, H=4096, thr=2.0, K=K0, t_scale=None):
    thr = float(np.float32(thr))
    """Supplied hypotheses around the true pose.  Point p is pinned at pixel distance thr +- d from its observation under
    hypothesis p (d log-uniform in 1e-9 .. 1e-1 px); a few hypotheses put a point on their optical axis at depth
    +-{1e-9, 1e-6, 1e-3} with its pixel 0.36 px from the principal point; a tenth of the points are the mirror images of
    inliers behind the camera, observed at their twin's pixel (zero error, but behind)."""
    rng = np.random.default_rng(seed)
    n = 1500
    P, uv, R, t = scene(seed, n, K, outl=0.2, noise=0.4, t_scale=t_scale)
    nm = n // 10
    pc = P[:nm].astype(np.float64) @ R.T + t
    P[n - nm:] = ((-pc - t) @ R).astype(np.float32)
    uv[n - nm:] = uv[:nm]
    poses = perturbed(rng, R, t, H, sig_r=(1e-6, 1e-2), sig_t=(1e-6, 1e-2))
    poses[0] = pose12(R, t)
    near = [n - nm - 1 - k for k in range(6)]
    uv[near] = (K[0, 2] + 0.3, K[1, 2] - 0.2)
    n_pin = 0
    for h in range(1, H - 12):
        d = np.exp(rng.uniform(np.log(1e-9), np.log(1e-1)))
        q = pin_to_threshold(poses[h], P, uv, K, h % (n - nm), thr, d if h % 2 else -d)
        if q is not None:
            poses[h] = q
            n_pin += 1
    for k, zt in enumerate([1e-9, -1e-9, 1e-6, -1e-6, 1e-3, -1e-3]):
        i = near[k]
        for rep in range(2):
            h = H - 12 + 2 * k + rep
            Rh = rod(rng.normal(0, 1e-3, 3)) @ R
            X = P[i].astype(np.float64)
            th = np.array([0.0, 0.0, zt]) - Rh @ X
            poses[h] = pose12(Rh, th)
    valid = np.ones(H, np.int32)
    return _case(P, uv, K, H=H, thr=thr, poses=poses, valid=valid, tie=dict(pinned=n_pin))


def ties(seed, winners, H=65535, n=200):
    """Supplied hypotheses: `winners` are the true pose; every other hypothesis is a perturbation of it (or invalid) whose
    count, undecided points included, stays below the winners'."""
    from oracle import pnp_oracle as po
    rng = np.random.default_rng(seed)
    P, uv, R, t = scene(seed, n, outl=0.3, noise=0.3)
    poses = perturbed(rng, R, t, H, sig_r=(1e-3, 3e-2), sig_t=(1e-3, 5e-2))
    valid = (rng.random(H) > 0.05).astype(np.int32)
    best = pose12(R, t)
    c_best = int((po.reproj_err2(P, uv, K0, R, t) <= 4.0).sum())
    sure, amb = oracle_counts(P, uv, K0, poses, 2.0)
    valid[sure + amb >= c_best] = 0
    for w in winners:
        poses[w], valid[w] = best, 1
    return _case(P, uv, K0, H=H, poses=poses, valid=valid, tie=dict(winners=list(winners), count=c_best))


def degenerate(kind, H=64):
    """All hypotheses invalid, or every valid one below 4 inliers (each hypothesis fits three points: of a scene of
    unrelated points no fourth one lands within the threshold)."""
    rng = np.random.default_rng(77)
    P, uv, R, t = scene(77, 300, outl=1.0)
    if kind == "invalid":
        return _case(P, uv, K0, H=H, poses=np.zeros((H, 12)), valid=np.zeros(H, np.int32))
    poses = perturbed(rng, R, t, H)
    sure, amb = oracle_counts(P, uv, K0, poses, 2.0)
    assert (sure + amb).max() < 4, (sure + amb).max()
    return _case(P, uv, K0, H=H, poses=poses, valid=np.ones(H, np.int32))


def cv(seed, n, thr=2.0, noise=0.5, count=None):
    P, uv, _, _ = scene(seed, n, outl=0.3, noise=noise)
    return _case(P, uv, K0, H=100, thr=thr, mode=1, count=count)


CASES = {
    # batched mode over the launch matrix: (H, n) on each side of the rules' boundaries; K and threshold varied
    "b_h1_n33": lambda: batch(1, 1, 33, outl=0.0, noise=0.3),
    "b_h7_n4": lambda: batch(2, 7, 4, outl=0.0),
    "b_h8_n5_thr05": lambda: batch(3, 8, 5, thr=0.5, outl=0.0, noise=0.1),
    "b_h9_n1024_fxfy": lambda: batch(4, 9, 1024, K=K_FXFY),
    "b_h129_n1025_off_thr37": lambda: batch(5, 129, 1025, thr=3.7, K=K_OFF),
    "b_h4096_n2456": lambda: batch(22, 4096, 2456),
    # 2457 points: 49140 B of staged points fit 48 KB, with the kernel's static 32 B they did not (the launch failed)
    "b_h4096_n2457": lambda: batch(6, 4096, 2457),
    "b_h4224_n2458_fxfy": lambda: batch(7, 4224, 2458, K=K_FXFY),
    "b_h4225_n1025": lambda: batch(8, 4225, 1025),
    "b_h4225_n2458_thr05": lambda: batch(9, 4225, 2458, thr=0.5),
    "b_h8192_n4096": lambda: batch(10, 8192, 4096),
    "b_h512_n4097_off": lambda: batch(11, 512, 4097, K=K_OFF),
    "b_h8192_n4097_thr37": lambda: batch(12, 8192, 4097, thr=3.7),
    "b_h65535_n33": lambda: batch(13, 65535, 33),
    "b_h1024_n8000_fxfy_thr05": lambda: batch(14, 1024, 8000, thr=0.5, K=K_FXFY),
    "b_h4096_n10240_off": lambda: batch(15, 4096, 10240, K=K_OFF),
    # the host path (mvo_solve_pnp_ransac, no device count) in the same cells
    "h_h129_n1025": lambda: batch(16, 129, 1025, path="host"),
    "h_h4225_n1025": lambda: batch(17, 4225, 1025, path="host"),
    "h_h4096_n2458": lambda: batch(18, 4096, 2458, path="host"),
    "h_h4225_n2458": lambda: batch(19, 4225, 2458, path="host"),
    "h_h512_n4097": lambda: batch(20, 512, 4097, path="host"),
    "h_h4225_n4097": lambda: batch(21, 4225, 4097, path="host"),
    # scoring at the edges of the fp32 bound
    "adv_default": lambda: adversarial(30),
    "adv_fxfy_thr05": lambda: adversarial(31, thr=0.5, K=K_FXFY),
    "adv_off_thr37": lambda: adversarial(32, thr=3.7, K=K_OFF),
    "adv_world_1e3": lambda: adversarial(33, t_scale=1e3),
    "adv_world_1e3_fxfy": lambda: adversarial(34, H=4225, K=K_FXFY, t_scale=1e3),
    # the arg-max
    "tie_1500_3000_65534": lambda: ties(40, [1500, 3000, 65534]),
    "sole_65534": lambda: ties(41, [65534]),
    "none_valid": lambda: degenerate("invalid"),
    "none_4_inliers": lambda: degenerate("below4"),
    # pnp_mode = 1
    "cv_n6": lambda: cv(50, 6, noise=0.3),
    "cv_n40": lambda: cv(51, 40),
    "cv_n2000": lambda: cv(52, 2000),
    "cv_n2000_noisefree": lambda: cv(53, 2000, noise=0.0),
    "cv_n2000_thr37": lambda: cv(54, 2000, thr=3.7),
    "cv_n4097": lambda: cv(55, 4097),
    "cv_n10240": lambda: cv(56, 10240, thr=1.3),
    "cv_host_n2000": lambda: dict(cv(57, 2000), path="host"),
    "cv_host_n4097": lambda: dict(cv(58, 4097), path="host"),
}


def _add_count_cases(prefix, n_upper, mode, seed):
    for cnt in (0, 3, 4, 5, 6, n_upper - 1, n_upper, n_upper + 7):
        CASES[f"{prefix}_c{cnt}"] = lambda cnt=cnt: dev_count(seed, n_upper, cnt, mode=mode)


_add_count_cases("cnt_b300", 300, 0, 60)
_add_count_cases("cnt_cv300", 300, 1, 61)
for _m, _s in ((0, 62), (1, 63)):
    CASES[f"cnt_{'cv' if _m else 'b'}4500_c4097"] = lambda m=_m, s=_s: dev_count(s, 4500, 4097, mode=m)
    CASES[f"cnt_{'cv' if _m else 'b'}4500_c4000"] = lambda m=_m, s=_s: dev_count(s, 4500, 4000, mode=m)

# the configuration each case is written for: (mode, passes >= 2, opt-in, re-read, device count)
EXPECT = {
    "b_h1_n33": (0, False, False, False, True), "b_h4224_n2458_fxfy": (0, False, True, False, True),
    "b_h4225_n1025": (0, True, False, False, True), "b_h4225_n2458_thr05": (0, True, True, False, True),
    "b_h8192_n4096": (0, True, True, False, True), "b_h512_n4097_off": (0, False, True, True, True),
    "b_h8192_n4097_thr37": (0, True, True, True, True), "b_h65535_n33": (0, True, False, False, True),
    "b_h4096_n2456": (0, False, False, False, True), "b_h4096_n2457": (0, False, True, False, True), "b_h4096_n10240_off": (0, False, True, True, True),
    "h_h129_n1025": (0, False, False, False, False), "h_h4225_n1025": (0, True, False, False, False),
    "h_h4096_n2458": (0, False, True, False, False), "h_h4225_n2458": (0, True, True, False, False),
    "h_h512_n4097": (0, False, True, True, False), "h_h4225_n4097": (0, True, True, True, False),
    "cv_n4097": (1, None, None, True, True), "cv_n2000": (1, None, None, False, True),
    "cv_host_n2000": (1, None, None, False, False), "cv_host_n4097": (1, None, None, True, False),
    "cnt_b4500_c4097": (0, False, True, True, True), "cnt_b4500_c4000": (0, False, True, False, True),
    "adv_world_1e3_fxfy": (0, True, False, False, True),
}


# ---- running --------------------------------------------------------------------------------------------------------------------
def _entry(lib):
    f = lib.mvo_test_pnp_dev
    vp = C.c_void_p
    f.restype = C.c_int
    f.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    return f


def _params(c):
    p = dict(pnp_mode=c["mode"], pnp_reproj_error=c["thr"], pnp_seed=c["seed"])
    if c["mode"] == 0:
        p["pnp_hypotheses"] = c["H"]
    return p


def run_dev(ctx, c, n_upper=None, count=None):
    """mvo_test_pnp_dev on the case (or on its first n_upper correspondences with the given count)."""
    n_upper = c["n_upper"] if n_upper is None else n_upper
    count = c["count"] if count is None else count
    P, uv, K = np.ascontiguousarray(c["P"][:n_upper]), np.ascontiguousarray(c["uv"][:n_upper]), np.ascontiguousarray(c["K"])
    H = int(ctx.params.pnp_hypotheses) if ctx.params.pnp_mode == 0 else 100      # what the entry returns counts of
    pose_io, out_i = np.full(12, np.nan), np.full(4, -7, np.int32)
    inl, counts = np.full(n_upper, -7, np.int32), np.full(H, -7, np.int32)
    poses = None if c["poses"] is None else np.ascontiguousarray(c["poses"], np.float64)
    valid = None if c["valid"] is None else np.ascontiguousarray(c["valid"], np.int32)
    rc = _entry(ctx.lib)(ctx.h, P.ctypes.data, uv.ctypes.data, n_upper, count, K.ctypes.data, None if poses is None else poses.ctypes.data,
                         None if valid is None else valid.ctypes.data, pose_io.ctypes.data, out_i.ctypes.data, inl.ctypes.data, counts.ctypes.data)
    r = dict(rc=rc, pose_io=pose_io, out_i=out_i, inl=inl[: max(int(out_i[0]), 0)], counts=counts)
    if rc == 0:
        r["hyp"], hc = ctx.pnp_last_hypotheses()
        assert np.array_equal(hc, counts)
    return r


def run_host(ctx, P, uv, K):
    """mvo_solve_pnp_ransac (no device count): rc, rvec, tvec, inliers, hypotheses and counts."""
    p3, p2, K = np.ascontiguousarray(P, np.float32), np.ascontiguousarray(uv, np.float32), np.ascontiguousarray(K, np.float64)
    rvec, tvec = np.full(3, np.nan), np.full(3, np.nan)
    inl = np.full(max(len(p3), 1), -7, np.int32)
    n = C.c_int(len(p3))
    rc = ctx.lib.mvo_solve_pnp_ransac(ctx.h, p3.ctypes.data, p2.ctypes.data, len(p3), K.ctypes.data, rvec.ctypes.data, tvec.ctypes.data,
                                      inl.ctypes.data, C.byref(n))
    r = dict(rc=rc, rvec=rvec, tvec=tvec, n_inliers=n.value, inl=inl[: max(n.value, 0)] if rc == 0 else inl)
    if len(p3) >= 4 and rc in (0, MVO_ERR_DEGENERATE):
        r["hyp"], r["counts"] = ctx.pnp_last_hypotheses()
    return r


def run_case(ctx, c, compare=True):
    """Runs case c on the library behind ctx: the device path, the host path, and for device-count cases (compare) also the
    host path on the correspondences the count selects and the device path with n_upper = count.  Restores the defaults."""
    ctx.set_params(**_params(c))
    try:
        out = {}
        if c["path"] == "host":
            out["host"] = run_host(ctx, c["P"], c["uv"], c["K"])
        out["dev"] = run_dev(ctx, c)
        m = min(max(c["count"], 0), c["n_upper"])
        if compare and c["poses"] is None and c["count"] != c["n_upper"]:
            if m >= 4:
                out["host_m"] = run_host(ctx, c["P"][:m], c["uv"][:m], c["K"])
                out["dev_m"] = run_dev(ctx, c, n_upper=m, count=m)
        return out
    finally:
        ctx.set_params(pnp_mode=0, pnp_reproj_error=2.0, pnp_hypotheses=4096, pnp_seed=0x9E3779B97F4A7C15)


CHILD = r'''
import sys
sys.path[:0] = [{root!r}, {tests!r}, {py!r}]
import numpy as np, mvo_b200, pnp_cases as PC
ctx = mvo_b200.Context(0)
for name in {names!r}:
    sys.stderr.write("@case " + name + "\n"); sys.stderr.flush()
    out = PC.run_case(ctx, PC.CASES[name](), compare=name not in {light!r})
    np.savez({out!r} + "/" + name + ".npz", **{{k + "." + f: v for k, r in out.items() for f, v in r.items()}})
ctx.close()
print("child ok")
'''


def run_children(groups, out_dir, lib=None, light=(), timeout=1800):
    """Runs each group of named cases in its own child process, the groups concurrently (MVO_LIB = lib when given; the cases
    in `light` without the comparison runs); returns {name: result of run_case}."""
    env = dict(os.environ)
    if lib is not None:
        env["MVO_LIB"] = str(lib)
    procs = []
    for names in groups:
        code = CHILD.format(root=str(ROOT), tests=str(ROOT / "tests"), py=str(PY), names=list(names), out=str(out_dir), light=list(light))
        procs.append(subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env))
    for p in procs:
        so, se = p.communicate(timeout=timeout)
        assert p.returncode == 0 and "child ok" in so, (so[-1500:], se[-2500:])
    res = {}
    for n in [n for g in groups for n in g]:
        z = np.load(Path(out_dir) / (n + ".npz"))
        d = {}
        for k in z.files:
            a, f = k.split(".", 1)
            d.setdefault(a, {})[f] = z[k][()] if z[k].shape == () else z[k]
        res[n] = d
    return res


# ---- checks -------------------------------------------------------------------------------------------------------------------
def _pose_tol(t):
    """1e-8, times 3 |t| where the translation is large: the LM's increment acts on the left, so an angle within its step
    tolerance of the optimum moves t by that angle times |t| (at |t| = 1.4e3 the refit ends 2e-8 rad from it)."""
    return 1e-8 * max(1.0, 3.0 * float(np.linalg.norm(t)))


def cv_replay(counts, n, H=100, confidence=0.999):
    """RANSACPointSetRegistrator::run's sequential part over the counts of the evaluated iterations: (best, iterations run)."""
    from oracle import pnp_cv_oracle as pc
    niters, best, max_good, it = H, -1, 0, 0
    while it < niters:
        good = int(counts[it])
        if good > max(max_good, 4):
            best, max_good = it, good
            niters = pc.ransac_update_num_iters(confidence, (n - good) / n, 5, niters)
        it += 1
    return best, it


def check_refit(c, P, uv, inl, start, got):
    """The refit pose is the least-squares optimum of the consensus set it was run on."""
    from oracle import pnp_oracle as po
    ro, to = po.refine(P[inl], uv[inl], c["K"], po.rvec_from_R(start[:9].reshape(3, 3)), start[9:])
    Rg = got[:9].reshape(3, 3)
    tol = _pose_tol(to)
    assert np.abs(Rg - po.rodrigues(ro)).max() < tol and np.abs(got[9:] - to).max() < tol, (np.abs(Rg - po.rodrigues(ro)).max(),
                                                                                              np.abs(got[9:] - to).max())


def check_batch(c, r, report):
    """The device result r (run_dev) of a batched-mode case against the fp64 oracle."""
    from oracle import p3p_oracle as p3
    assert r["rc"] == 0, r["rc"]
    n_eff = min(c["n_upper"], max(c["count"], 0))
    P, uv, K, thr, H = c["P"][:n_eff], c["uv"][:n_eff], c["K"], c["thr"], c["H"]
    counts, hyp = r["counts"], r["hyp"]
    assert len(counts) == H
    if c["poses"] is not None:
        assert np.array_equal(hyp, c["poses"])                    # the scoring read the supplied hypotheses
        assert np.array_equal(counts < 0, c["valid"] == 0)
    valid = counts >= 0
    if n_eff < 4:
        assert not valid.any()
    else:
        sure, amb = oracle_counts(P, uv, K, hyp[valid], thr)
        got = counts[valid]
        bad = np.flatnonzero((got < sure) | (got > sure + amb))
        assert len(bad) == 0, [(int(np.flatnonzero(valid)[b]), int(got[b]), int(sure[b]), int(amb[b])) for b in bad[:10]]
        report["undecided"] = report.get("undecided", 0) + int(amb.sum())
        report["pairs"] = report.get("pairs", 0) + int(valid.sum()) * n_eff
        if c["poses"] is None:                                    # the product's samples: P3P exact on its three points
            vh = np.flatnonzero(valid)
            step = max(1, len(vh) // 4096)
            for h in vh[::step]:
                idx = p3.sample_indices(c["seed"], int(h), n_eff)[:3]
                px, z = project(P[idx], hyp[h, :9].reshape(3, 3), hyp[h, 9:], K)
                assert (z > 0).all() and np.abs(px - uv[idx].astype(np.float64)).max() < 1e-6, (h, px, uv[idx])
    n_in, best = int(r["out_i"][0]), int(r["out_i"][1])
    if not valid.any() or counts.max() < 4:
        assert (n_in, best) == (0, -1), r["out_i"]
        assert np.array_equal(r["pose_io"], pose12(np.eye(3), np.zeros(3)))       # nothing of an earlier call
        return
    assert best == int(np.flatnonzero(counts == counts.max())[0]), (best, counts.max())
    sure_set, und = consensus(P, uv, K, hyp[best], thr)
    inl = r["inl"]
    assert n_in == counts[best] == len(inl) and np.all(np.diff(inl) > 0)
    assert set(sure_set) <= set(inl) <= set(sure_set) | set(und), (len(sure_set), len(und), len(inl))
    check_refit(c, P, uv, inl, hyp[best], r["pose_io"])


def check_cv(c, r, report):
    """The device result of a pnp_mode = 1 case against the float rule and the replayed adaptive stop."""
    from oracle import pnp_cv_oracle as pc
    assert r["rc"] == 0, r["rc"]
    n_eff = min(c["n_upper"], max(c["count"], 0))
    P, uv, K = c["P"][:n_eff], c["uv"][:n_eff], c["K"]
    counts, hyp = r["counts"], r["hyp"]
    assert len(counts) == 100
    thr2f = np.float32(c["thr"] * c["thr"])
    ulp2 = 2 * float(np.spacing(thr2f))
    if n_eff < 6:
        assert (counts == -1).all()
    for h in np.flatnonzero(counts >= 0):
        e = pc.float_errors(P, uv, K, hyp[h, :9].reshape(3, 3), hyp[h, 9:])
        und = np.abs(e.astype(np.float64) - float(thr2f)) <= ulp2
        sure = int(((e <= thr2f) & ~und).sum())
        assert sure <= counts[h] <= sure + und.sum(), (h, counts[h], sure, und.sum())
        report["undecided"] = report.get("undecided", 0) + int(und.sum())
        report["pairs"] = report.get("pairs", 0) + n_eff
    best, iters = cv_replay(counts, n_eff)
    assert (int(r["out_i"][1]), int(r["out_i"][3])) == (best, iters), (r["out_i"], best, iters)
    if best < 0:
        assert int(r["out_i"][0]) == 0
        return
    e = pc.float_errors(P, uv, K, hyp[best, :9].reshape(3, 3), hyp[best, 9:])
    und = np.abs(e.astype(np.float64) - float(thr2f)) <= ulp2
    inl = r["inl"]
    assert int(r["out_i"][0]) == len(inl) == counts[best] and np.all(np.diff(inl) > 0)
    assert set(np.flatnonzero((e <= thr2f) & ~und)) <= set(inl) <= set(np.flatnonzero((e <= thr2f) | und))
    check_refit(c, P, uv, inl, r["pose_io"], r["pose_io"])


def check_same_run(a, b, csize=8, n_a=None, n_b=None):
    """Two runs that must compute the same thing: the device path against the host path (or a device run with the clamped
    count as its bound).  Hypotheses, counts and inliers bit-identical; the pose within 1e-12, bit-identical when both refits
    launch the same k_ba_pose kernel."""
    from oracle import pnp_oracle as po
    assert np.array_equal(a["hyp"], b["hyp"]) and np.array_equal(a["counts"], b["counts"])
    assert np.array_equal(a["inl"], b["inl"]), (len(a["inl"]), len(b["inl"]))
    same_kernel = refit_kernel(n_a, csize) == refit_kernel(n_b, csize)
    if "pose_io" in b:
        d = np.abs(a["pose_io"] - b["pose_io"]).max()
        assert d == 0 if same_kernel else d < 1e-12, d
    else:                       # the host path returns rvec / tvec; the rvec round trip re-orthonormalises R (~1e-12 off after the LM)
        assert np.abs(a["pose_io"][:9] - po.rodrigues(b["rvec"]).ravel()).max() < 1e-10
        d = np.abs(a["pose_io"][9:] - b["tvec"]).max()
        assert d == 0 if same_kernel else d < 1e-12, d


def check(c, out, report=None, csize=8):
    """Checks one case's results (run_case / run_children); returns the configuration it reached."""
    report = {} if report is None else report
    r = out["dev"]
    (check_cv if c["mode"] == 1 else check_batch)(c, r, report)
    n_eff = min(c["n_upper"], max(c["count"], 0))
    if "host" in out:
        h = out["host"]
        if int(r["out_i"][0]) == 0:
            assert h["rc"] == MVO_ERR_DEGENERATE and h["n_inliers"] == 0
        else:
            assert h["rc"] == 0
            check_same_run(r, h, csize, c["n_upper"], c["n_upper"])
    if "host_m" in out:                                           # the device count against the host path on the first n_eff
        h, dm = out["host_m"], out["dev_m"]
        if int(r["out_i"][0]) == 0:
            assert h["rc"] == MVO_ERR_DEGENERATE and int(dm["out_i"][0]) == 0
            assert np.array_equal(h["counts"], r["counts"])
        else:
            assert h["rc"] == 0
            check_same_run(r, h, csize, c["n_upper"], n_eff)
            check_same_run(r, dm, csize, c["n_upper"], n_eff)
    elif c["poses"] is None and n_eff < (6 if c["mode"] == 1 else 4):
        assert int(r["out_i"][0]) == 0                            # below the minimal set: no model
    if c["tie"] and "winners" in c["tie"]:
        assert int(r["out_i"][1]) == c["tie"]["winners"][0] and int(r["out_i"][0]) == c["tie"]["count"], (r["out_i"], c["tie"])
        assert (r["counts"] == c["tie"]["count"]).sum() == len(c["tie"]["winners"])
    return config(c)
