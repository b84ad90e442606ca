"""Cases of the free-points Schur bundle adjustment (k_ba, csrc/ba.cu) and their checks against the C oracle
(oracle/ba_oracle.c), shared by test_ba_schur_gpu.py (the H100) and test_ba_schur_emu.py (the emulated library on the CPU).

k_ba runs as one cluster of 8 CTAs.  Rank r owns the points [r per, (r + 1) per) with per = ceil(P / 8) and linearises them
in rounds of 256 threads; the Schur products stage pc points at a time in shared memory; the pose system has n = 6 nact rows.
`launch` restates how the host chooses these values, and every case checks them against the MVO_BA_DEBUG line of its call
(pc, per, nact, dynamic shared memory, LM iterations, trials and rejected trials).  `configs` names the configurations a case
reaches; test_ba_schur_gpu.py checks that the cases together reach all of REQUIRED.

Bars (fp64 on both sides, different summation order), as in test_ba_gpu.py:
  * chi2 relative 1e-9, poses 1e-8, points 1e-6, iterations, trials and rejections equal while `decisive` holds;
  * no pose fixed and F >= 2, or one free frame: the solution is defined up to a similarity (the gauge), which only the damping
    holds, so the bars are the gauge-invariant ones of test_ba_free_points_gauge_invariants: chi2 1e-5 relative, reprojections
    1e-2 px;
  * a point with one observation moves along its ray at the rate lambda allows: its reprojection is compared, within 1e-6 px
    plus what rounding the point to float32 (as the C ABI returns it) can move it;
  * a final chi2 below 1e-12 of the initial one (an exact fit: one frame, or points seen once, residuals of nanopixels that
    rounding decides) is not compared relatively but must be as small on both sides, and its iteration count may differ by 3;
  * a point without edges, the fixed first pose of a structure-only problem at the identity, and the points of an
    update_points = 0 call come back bit for bit."""
import re

import numpy as np

from ba_pose_cases import K, _rel, _rod, _trace_counts, decisive

BA_T, BA_CLUSTER, BA_NW = 256, 8, 8
DEBUG = re.compile(r"k_ba: F=(\d+) P=(\d+) E=(\d+) pc=(\d+) per=(\d+) nact=(\d+) smem=(\d+) it=(\d+) trials=(\d+) rejected=(\d+)")
DBL_MAX = np.finfo(np.float64).max


# ---- the host's launch rules, restated (run_ba) -----------------------------------------------------------------------------
def pc_rule(F):
    """Points per staging chunk of the Schur products: <= 64 KB of shared memory, 1..64."""
    return max(1, min(65536 // (F * 36 * 8 + 24), 64))


def per_rule(P):
    return -(-P // BA_CLUSTER)


def rank_points(P):
    """How many points each CTA owns."""
    per = per_rule(P)
    return [min(r * per + per, P) - min(r * per, P) for r in range(BA_CLUSTER)]


def rounds(P):
    """Linearisation rounds of 256 threads per CTA."""
    return [-(-n // BA_T) for n in rank_points(P)]


def tails(P, F):
    """Points in the last staging chunk of each CTA (0: no points, or only full chunks)."""
    return [n % pc_rule(F) for n in rank_points(P)]


def smem_doubles(F, nact, pc):
    """ba_smem_doubles: the dynamic shared memory of k_ba in doubles."""
    n, NA = 6 * nact, F * 27 + 2
    NC = n * n + n
    u = max(BA_NW * NA, n * n + n + 8, pc * F * 36 + pc * 3 + 8)
    return F * 24 + 2 * NA + 4 + ((n + 3) & ~3) + 4 + ((NC + 3) & ~3) + u + 16


def launch(F, P, fix_first):
    nact = F - int(bool(fix_first))
    pc = pc_rule(F)
    return dict(pc=pc, per=per_rule(P), nact=nact, smem=8 * smem_doubles(F, nact, pc))


def configs(c):
    """The launch configurations case c reaches (by the rules above; each case checks them against the library)."""
    pb = c["pb"]
    F, P = len(pb["T_w_c"]), len(pb["points"])
    if c["iters"] == 0 or len(pb["obs"]) == 0:
        return set()
    L = launch(F, P, c["fix_first"])
    pc, per = L["pc"], L["per"]
    out = {f"rounds={max(rounds(P))}", f"n={6 * L['nact']}"}
    if min(rank_points(P)) == 0:
        out.add("cta_without_points")
    if sorted(set(rounds(P))) == [1, 2]:
        out.add("rounds=2_and_1")
    for name, v in (("pc-1", pc - 1), ("pc", pc), ("pc+1", pc + 1), ("2pc+1", 2 * pc + 1)):
        if per == v:
            out.add(f"F={F}:per={name}")
    if per > pc and 1 in tails(P, F):
        out.add("one_point_tail")
    return out


REQUIRED = ({"rounds=1", "rounds=2", "rounds=3", "rounds=10", "rounds=2_and_1", "cta_without_points", "one_point_tail",
             "n=96", "n=90", "n=6", "n=0"}
            | {f"F={F}:per={v}" for F in (1, 4, 5, 8, 16) for v in ("pc-1", "pc", "pc+1", "2pc+1")})


# ---- problems -------------------------------------------------------------------------------------------------------------------
def make_problem(seed, F, P, n_obs=None, only0=(), empty=(), dup=0, shuffle=False, pose_pert=1e-2, point_pert=1e-2, noise=0.5,
                 outlier_frac=0.05):
    """Poses on a smooth arc (as mvo_synth.ba_problem) and P points in front of them.  Point l is observed by n_obs[l] frames
    (0, 1, 2, ... or F: every frame not in empty; default F), chosen at random among the frames not in empty; the points in
    only0 by frame 0 alone.  dup observations are repeated (same point and frame, the pixel 0.25 off).  Edges are frame-major
    unless shuffled."""
    rng = np.random.default_rng(seed)
    only0 = set(only0)
    X = np.stack([rng.uniform(-2, 2, P), rng.uniform(-1.5, 1.5, P), rng.uniform(2, 8, P)], 1)
    allowed = np.array([f for f in range(F) if f not in set(empty)], np.int64)
    n_obs = np.full(P, len(allowed)) if n_obs is None else np.minimum(np.asarray(n_obs), len(allowed))
    seen = np.zeros((F, P), bool)
    for l in range(P):
        if l in only0:
            seen[0, l] = True
        elif n_obs[l]:
            seen[rng.choice(allowed, int(n_obs[l]), replace=False), l] = True
    T_init, ef, ep, obs = [], [], [], []
    for f in range(F):
        Tcw = np.eye(4)
        Tcw[:3, :3], Tcw[:3, 3] = _rod(np.array([0.01, -0.02, 0.005]) * f), [0.05 * f, 0.01 * f, 0.004 * f * f]
        Tp = np.eye(4)
        Tp[:3, :3], Tp[:3, 3] = _rod(rng.normal(0, pose_pert, 3)), rng.normal(0, pose_pert, 3)
        T_init.append(np.linalg.inv(Tp @ Tcw))
        idx = np.flatnonzero(seen[f])
        pc = X[idx] @ Tcw[:3, :3].T + Tcw[:3, 3]
        uv = pc[:, :2] / pc[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, noise, (len(idx), 2))
        bad = rng.random(len(idx)) < outlier_frac
        uv[bad] += rng.uniform(-30, 30, (int(bad.sum()), 2))
        ef.append(np.full(len(idx), f, np.int32))
        ep.append(idx.astype(np.int32))
        obs.append(uv)
    pb = dict(T_w_c=np.array(T_init), points=(X + rng.normal(0, point_pert, X.shape)).astype(np.float32),
              edge_frame=np.concatenate(ef), edge_point=np.concatenate(ep), obs=np.concatenate(obs).astype(np.float32))
    if dup:
        j = rng.choice(len(pb["obs"]), dup, replace=False)
        for k in ("edge_frame", "edge_point", "obs"):
            pb[k] = np.concatenate([pb[k], pb[k][j] + (0.25 if k == "obs" else 0)]).astype(pb[k].dtype)
    if shuffle:
        p = rng.permutation(len(pb["obs"]))
        for k in ("edge_frame", "edge_point", "obs"):
            pb[k] = pb[k][p]
    return pb


def zero_depth(pb, l):
    """Frame 0 at the identity and point l at (1, 0.5, 0): its depth in frame 0 is exactly 0, its Hll block NaN."""
    pb["T_w_c"][0] = np.eye(4)
    pb["points"][l] = np.array([1.0, 0.5, 0.0], np.float32)
    return pb


def near_plane(z_c, F=2):
    """Frame 0 at the identity and point 0 at (1, 0.5, z_c): its camera depth is exactly z_c (float32 of it)."""
    pb = make_problem(3, F, 60)
    pb["T_w_c"][0] = np.eye(4)
    pb["points"][0] = np.array([1.0, 0.5, z_c], np.float32)
    return pb


def _ba(pb, iters=5, huber=1.0, info=None, fix_first=0, update=1, single=False):
    return dict(kind="single" if single else "ba", pb=pb, iters=iters, huber=huber, info=info, fix_first=fix_first, update=update)


# ---- running ------------------------------------------------------------------------------------------------------------------
def run_case(ctx, c):
    """Runs case c on the library behind ctx; returns a JSON-able dict."""
    pb = c["pb"]
    ctx.set_params(ba_iterations=c["iters"], ba_huber_delta=c["huber"], ba_fix_first_pose=c["fix_first"], ba_step_tol=0.0)
    try:
        if c["kind"] == "single":
            gp, gx = ctx.optimize_single_frame(pb["T_w_c"][0], pb["points"], pb["obs"], K, fix_points=False, update_points=True)
            gp, gs = gp[None], [0.0] * 4
        else:
            gp, gx, gs = ctx.bundle_adjustment(pb["T_w_c"], pb["points"], pb["edge_frame"], pb["edge_point"], pb["obs"], K,
                                               information=c["info"], fix_points=False, update_points=bool(c["update"]))
    finally:
        ctx.set_params(ba_iterations=50, ba_huber_delta=1.0, ba_fix_first_pose=0, ba_step_tol=0.0)
    return dict(pose=np.asarray(gp).tolist(), points=np.asarray(gx, np.float64).tolist(), stats=list(map(float, gs)))


def parse_debug(text):
    """The MVO_BA_DEBUG lines of k_ba in text, as dicts."""
    keys = ("F", "P", "E", "pc", "per", "nact", "smem", "it", "trials", "rejected")
    return [dict(zip(keys, map(int, m.groups()))) for m in DEBUG.finditer(text)]


def run_children(names, lib=None, timeout=1800):
    """The cases in one child process (ba_pose_cases.run_children); {name: (result, [debug records])}."""
    import ba_pose_cases
    return ba_pose_cases.run_children(names, lib=lib, timeout=timeout, module="ba_schur_cases")


# ---- checks ---------------------------------------------------------------------------------------------------------------------
def oracle(c):
    from oracle import oracle_lib
    pb = c["pb"]
    single = c["kind"] == "single"
    return oracle_lib.bundle_adjustment_with_trace(pb["T_w_c"][:1] if single else pb["T_w_c"], pb["points"], pb["edge_frame"],
                                                   pb["edge_point"], pb["obs"], K, information=None if single else c["info"],
                                                   fix_points=False, update_points=True if single else bool(c["update"]),
                                                   iterations=c["iters"], huber_delta=0.0 if single else c["huber"],
                                                   fix_first_pose=bool(c["fix_first"]))


def _close(a, b, tol):
    return a == b or _rel(a, b) < tol


def _decisive(os_, trace):
    """decisive(), and every run that starts from a non-finite chi2 (its decisions compare inf and DBL_MAX, not rounding)."""
    return not np.isfinite(os_[0]) or decisive(os_[0], trace)


def _pixels_agree(ug, uo, tol):
    """Pixels of the two sides within tol where they are finite; non-finite (a point at zero depth) on the same edges."""
    fin = np.isfinite(ug).all(1)
    assert np.array_equal(fin, np.isfinite(uo).all(1))
    tol = tol[fin] if np.ndim(tol) else tol
    assert (np.abs(ug[fin] - uo[fin]).max(1, initial=0) < tol).all(), np.abs(ug[fin] - uo[fin]).max(initial=0)


def _project(T_w_c, X, ef, ep):
    """Pixel of each edge's point in its frame (fp64), and the pixel's largest change per unit of each point coordinate."""
    Tcw = np.linalg.inv(T_w_c)
    R, t = Tcw[ef, :3, :3], Tcw[ef, :3, 3]
    pc = np.einsum("eij,ej->ei", R, X[ep].astype(np.float64)) + t
    z = pc[:, 2:3]
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = pc[:, :2] / z * K[0, 0] + K[:2, 2]
        # d(u, v) / dX = f / z (R_01 - (x, y) / z R_2)
        J = K[0, 0] / z[:, :, None] * (R[:, :2, :] - pc[:, :2, None] / z[:, :, None] * R[:, 2:3, :])
    return uv, np.abs(J).max(1)


def gauge(c):
    """Whether the solution is only defined up to the gauge: no pose fixed (with free points every frame can move)."""
    return not c["fix_first"]


def check(c, r, debug):
    """Checks one case's result (run_case / run_children) against the oracle; returns the configurations it reached."""
    pb = c["pb"]
    single = c["kind"] == "single"
    F, P, E = (1 if single else len(pb["T_w_c"])), len(pb["points"]), len(pb["obs"])
    T0, X0 = (pb["T_w_c"][:1] if single else pb["T_w_c"]), np.asarray(pb["points"], np.float32)
    gp = np.asarray(r["pose"]).reshape(-1, 4, 4)
    gx = np.asarray(r["points"]).astype(np.float32).reshape(-1, 3)
    gs = r["stats"]
    if c["iters"] == 0 or E == 0:          # nothing to optimise: run_ba returns before the kernel
        assert debug == [] and np.array_equal(gp, T0) and np.array_equal(gx, X0) and gs == [0.0] * 4
        return set()
    op, ox, os_, trace = oracle(c)
    assert len(debug) == 1, debug
    d = debug[0]
    assert {k: d[k] for k in ("F", "P", "E", "pc", "per", "nact", "smem")} == dict(F=F, P=P, E=E, **launch(F, P, c["fix_first"])), d
    assert np.isfinite(gp).all() and np.isfinite(gx).all()
    ef, ep = pb["edge_frame"], pb["edge_point"]
    cnt = np.bincount(ep, minlength=P)
    floor = os_[1] <= 1e-12 * os_[0]
    if not single:
        assert d["it"] == gs[2]
        assert _close(gs[0], os_[0], 1e-9), (gs, list(os_))
        if floor:
            assert gs[1] <= 1e-12 * gs[0] and abs(gs[2] - os_[2]) <= 3, (gs, list(os_))
        elif gauge(c) and F >= 2:
            assert gs[1] == os_[1] or abs(gs[1] - os_[1]) < 1e-5 * os_[1] + 1e-9, (gs, list(os_))
        else:
            assert _close(gs[1], os_[1], 1e-9), (gs, list(os_))
        assert np.isfinite(gs[3]) and (_close(gs[3], os_[3], 1e-6) or not _decisive(os_, trace)), (gs, list(os_))
    if _decisive(os_, trace) and not floor:
        assert (d["it"], d["trials"], d["rejected"]) == (os_[2],) + _trace_counts(trace), (d, list(os_), _trace_counts(trace))
    if not c["update"]:
        assert np.array_equal(gx, X0)                            # g2o_ba.cpp:308: the points are not written back
        ox = X0
    assert np.array_equal(gx[cnt == 0], X0[cnt == 0]) and np.array_equal(ox[cnt == 0], X0[cnt == 0])
    if gauge(c):
        _pixels_agree(_project(gp, gx, ef, ep)[0], _project(op, ox, ef, ep)[0], 1e-2)
        return configs(c)
    assert np.abs(gp - op).max() < 1e-8, np.abs(gp - op).max()
    assert np.abs(gp[0] - T0[0]).max() < 1e-12                   # the fixed pose only goes through the host's conversions
    if not (T0[0] - np.eye(4)).any():
        assert np.array_equal(gp[0], T0[0])                      # at the identity they are exact
    multi = cnt >= 2
    if c["update"]:
        assert np.abs(gx[multi] - ox[multi]).max(initial=0) < 1e-6, np.abs(gx[multi] - ox[multi]).max()
    once = np.isin(ep, np.flatnonzero(cnt == 1))
    if once.any():
        ug, J = _project(gp, gx, ef[once], ep[once])
        uo, _ = _project(op, ox, ef[once], ep[once])
        ulp = np.spacing(np.maximum(np.abs(gx[ep[once]]), np.abs(ox[ep[once]])))      # one float32 step of each coordinate
        _pixels_agree(ug, uo, 1e-6 + (J * ulp).sum(1))
    return configs(c)


# ---- the cases ------------------------------------------------------------------------------------------------------------------
def _per_case(F, per, fix_first=0, seed=0):
    """F frames and a point count that gives every CTA but the last `per` points."""
    return _ba(make_problem(100 + seed + F * 7 + per, F, 8 * per - 3), iters=3, fix_first=fix_first)


def _lm_reject():
    # a start 0.8 rad / 0.8 from the arc, no robust kernel: the undamped first steps overshoot and trials are rejected far above
    # rounding (as ba_pose_cases._lm_reject)
    return _ba(make_problem(22, 2, 300, pose_pert=0.8, outlier_frac=0.0), iters=8, huber=0.0, fix_first=1)


def _zero_info():
    # all-zero information: chi2 = 0, lambda_0 = 0, every Hll + lambda I singular on every CTA; ten rejected trials end the LM
    return _ba(make_problem(23, 3, 200), iters=5, info=np.zeros((2, 2)))


def _zero_depth_on(rank, fix_first):
    # one point at zero depth in frame 0, in rank's range: only that CTA sees its Hll + lambda I fail, the others must learn it
    # through the cluster-wide flag (with frame 0 free its NaN b reaches every CTA anyway).  The information has an
    # off-diagonal term so that the point's chi2 is inf, not NaN: every trial is then accepted at DBL_MAX, where a CTA that
    # went on with the solve would reject it (inf - inf)
    P = 200
    l = rank * per_rule(P) + 5
    return _ba(zero_depth(make_problem(24 + rank, 2, P), l), iters=3, info=np.array([[2.0, 0.3], [0.3, 0.5]]), fix_first=fix_first)


def _divergence():
    # F = 2, nothing fixed, information [[2, 0.3], [0.3, 0.5]], point 0 at zero depth in frame 0: both sides start from
    # chi2 = inf and every solve fails; the gain denominator must not take frame 0's NaN b (the oracle accepts each trial with
    # chi2 = DBL_MAX)
    return _ba(zero_depth(make_problem(25, 2, 100), 0), iters=4, info=np.array([[2.0, 0.3], [0.3, 0.5]]))


def _no_edge_points():
    P = 800                      # per = 100: rank 3 owns [300, 400)
    n = np.full(P, 3)
    n[::2] = 0
    n[300:400] = 0
    return _ba(make_problem(26, 3, P, n_obs=n), iters=4, fix_first=1)


def _single_obs():
    P = 600
    n = np.where(np.arange(P) % 3 == 0, 1, 3)
    return _ba(make_problem(27, 3, P, n_obs=n), iters=5, fix_first=1)


CASES = {
    # points per CTA (F = 3, first pose fixed): CTAs without points, one and several linearisation rounds
    "P1": lambda: _ba(make_problem(1, 3, 1), iters=3, fix_first=1),
    "P7": lambda: _ba(make_problem(2, 3, 7), iters=3, fix_first=1),
    "P8": lambda: _ba(make_problem(3, 3, 8), iters=3, fix_first=1),
    "P2047": lambda: _ba(make_problem(4, 3, 2047), iters=3, fix_first=1),
    "P2048": lambda: _ba(make_problem(5, 3, 2048), iters=3, fix_first=1),
    "P2049": lambda: _ba(make_problem(6, 3, 2049), iters=3, fix_first=1),
    "P4097": lambda: _ba(make_problem(7, 3, 4097), iters=3, fix_first=1),
    "P20000_F5": lambda: _ba(make_problem(8, 5, 20000), iters=3, fix_first=1),
    # active poses
    "F16_free": lambda: _ba(make_problem(9, 16, 200), iters=4),
    "F16_fix": lambda: _ba(make_problem(10, 16, 200), iters=4, fix_first=1),
    "F16_fix_small": lambda: _ba(make_problem(11, 16, 60), iters=3, fix_first=1),
    "F2_fix": lambda: _ba(make_problem(12, 2, 300), iters=5, fix_first=1),
    "structure_only": lambda: _ba(dict(make_problem(13, 1, 300), T_w_c=np.eye(4)[None]), iters=5, fix_first=1),
    "structure_only_P7": lambda: _ba(dict(make_problem(14, 1, 7), T_w_c=np.eye(4)[None]), iters=3, fix_first=1),
    # layout
    "no_edge_points": _no_edge_points,
    "frame0_only_points": lambda: _ba(make_problem(28, 3, 400, only0=range(0, 400, 4)), iters=4, fix_first=1),
    "single_obs_points": _single_obs,
    "empty_active_frame": lambda: _ba(make_problem(29, 4, 300, empty=(2,)), iters=4, fix_first=1),
    "duplicates": lambda: _ba(make_problem(30, 4, 250, dup=60), iters=6, info=np.array([[2.0, 0.3], [0.3, 0.5]]), fix_first=1),
    "shuffled": lambda: _ba(make_problem(31, 4, 500, shuffle=True), iters=5, fix_first=1),
    "one_frame_edges": lambda: _ba(make_problem(32, 4, 300, n_obs=np.ones(300, int), empty=(0, 1, 3)), iters=4, fix_first=1),
    "no_pose_fixed": lambda: _ba(make_problem(33, 5, 400), iters=6),
    # LM control
    "huber_off": lambda: _ba(make_problem(15, 3, 500), iters=4, huber=0.0, fix_first=1),
    "info_nondiag": lambda: _ba(make_problem(16, 3, 500), iters=8, info=np.array([[2.0, 0.3], [0.3, 0.5]]), fix_first=1),
    "iters1": lambda: _ba(make_problem(17, 2, 300), iters=1, fix_first=1),
    "iters2": lambda: _ba(make_problem(18, 2, 300), iters=2, fix_first=1),
    "rejections": _lm_reject,
    "converge50": lambda: _ba(make_problem(19, 4, 400, outlier_frac=0.0), iters=50, fix_first=1),
    "no_update": lambda: _ba(make_problem(20, 3, 400), iters=5, update=0, fix_first=1),
    "iters0": lambda: _ba(make_problem(21, 3, 100), iters=0, fix_first=1),
    # solve failure
    "zero_info": _zero_info,
    "divergence": _divergence,
    # range: a point near frame 0's principal plane
    "near_1e-12_huber": lambda: _ba(near_plane(1e-12), fix_first=1),
    "near_1e-12_plain": lambda: _ba(near_plane(1e-12), huber=0.0, fix_first=1),
    "near_1e-18_huber": lambda: _ba(near_plane(1e-18), fix_first=1),
    "near_1e-18_plain": lambda: _ba(near_plane(1e-18), huber=0.0, fix_first=1),
    # optimizeSingleFrame with free points (no robust kernel) at P above 2048
    "single_frame_P2500": lambda: _ba(make_problem(34, 1, 2500, outlier_frac=0.0), iters=8, huber=0.0, single=True),
}
for _r in range(BA_CLUSTER):
    CASES[f"zero_depth_rank{_r}_fix"] = (lambda r: lambda: _zero_depth_on(r, 1))(_r)
    CASES[f"zero_depth_rank{_r}_free"] = (lambda r: lambda: _zero_depth_on(r, 0))(_r)
# staging chunk: per = pc - 1, pc, pc + 1 (a one-point tail) and 2 pc + 1, for F = 1, 4, 5, 8 and 16 (first pose fixed: F = 1 is
# then structure-only)
for _F in (1, 4, 5, 8, 16):
    _pc = pc_rule(_F)
    for _name, _per in (("pc-1", _pc - 1), ("pc", _pc), ("pc+1", _pc + 1), ("2pc+1", 2 * _pc + 1)):
        CASES[f"stage_F{_F}_{_name}"] = (lambda F, per: lambda: _per_case(F, per, fix_first=1))(_F, _per)
