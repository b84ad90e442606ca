"""Cases of the pose-only Levenberg-Marquardt kernel (k_ba_pose, csrc/ba.cu) and their checks against the C oracle
(oracle/ba_oracle.c), shared by test_ba_pose_gpu.py (the H100) and test_ba_pose_emu.py (the emulated library on the CPU).

A case is built by a function of CASES and runs either in the calling process (`run_case`) or in a child process
(`run_children`: the kernel's cluster size is read once per process, and the emulated library is loaded through MVO_LIB).
Each run reports the kernel's result and, for the mvo_bundle_adjustment path, the MVO_BA_DEBUG line of the call (padded edge
count, chunk, cluster size, trials, rejected trials); `check` compares that with the oracle's trace and with the host's chunk
rule restated below, and returns the k_ba_pose instantiation the case reached.

Tolerances are those of test_ba_gpu.py: chi2 relative 1e-9, poses 1e-8, equal LM iteration counts while chi2 is above the
rounding floor; here also equal trial and rejection counts."""
import ctypes as C
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
PY = ROOT / "monocular-visual-odometry_b200" / "python"
PF_T, PF_MAXC, BA_MAXF = 512, 8, 16
MVO_ERR_UNSUPPORTED = -5
K = np.array([[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1.0]])
DEBUG = re.compile(r"k_ba_pose: F=(\d+) E=(\d+) Ep=(\d+) chunk=(\d+) cluster=(\d+) it=(\d+) trials=(\d+) rejected=(\d+)")


# ---- the host's launch rules, restated ----------------------------------------------------------------------------------
def cluster_size(env=None):
    """pose_cluster_size(): MVO_BA_CLUSTER in 1..8, anything else 8."""
    try:
        v = int(env) if env is not None else 8
    except ValueError:
        v = 0
    return v if 1 <= v <= PF_MAXC else 8


def chunk_rule(counts, csize):
    """run_ba + mvo_ba_pose_launch: edges per thread, padded edge count, and the instantiation."""
    E, F = int(sum(counts)), len(counts)
    chunk = 1
    while E + F * (chunk - 1) > chunk * csize * PF_T and chunk < 64:
        chunk += 1
    Ep = sum(-(-int(n) // chunk) * chunk for n in counts)
    cached = chunk <= 4 and Ep // chunk <= csize * PF_T
    return chunk, Ep, f"<{chunk if cached else 1},{'true' if cached else 'false'},false>"


def store_chunk(e_upper, nslots, csize):
    """mvo_ba_pose_store_launch: CH of k_ba_pose<CH,true,true>, None when the edges exceed the device-resident path."""
    chunk = 1
    while e_upper + nslots * (chunk - 1) > chunk * csize * PF_T and chunk <= 4:
        chunk += 1
    return chunk if chunk <= 4 else None


# ---- problems -------------------------------------------------------------------------------------------------------------
def _rod(r):
    th = np.linalg.norm(r)
    if th < 1e-300:
        return np.eye(3)
    k = r / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def make_problem(seed, counts, n_points=None, pose_pert=1e-2, noise=0.5, outlier_frac=0.05, shuffle=False):
    """Poses on a smooth arc (as mvo_synth.ba_problem), frame f observing counts[f] points; edges frame-major unless shuffled."""
    rng = np.random.default_rng(seed)
    F = len(counts)
    P = n_points or max(1, max(counts))
    X = np.stack([rng.uniform(-2, 2, P), rng.uniform(-1.5, 1.5, P), rng.uniform(2, 8, P)], 1)
    T_init, ef, ep, obs = [], [], [], []
    for f in range(F):
        Tcw = np.eye(4)
        Tcw[:3, :3], Tcw[:3, 3] = _rod(np.array([0.01, -0.02, 0.005]) * f), [0.05 * f, 0.01 * f, 0.004 * f * f]
        Tp = np.eye(4)
        Tp[:3, :3], Tp[:3, 3] = _rod(rng.normal(0, pose_pert, 3)), rng.normal(0, pose_pert, 3)
        T_init.append(np.linalg.inv(Tp @ Tcw))
        idx = rng.permutation(P)[: counts[f]] if counts[f] <= P else rng.integers(0, P, counts[f])
        pc = X[idx] @ Tcw[:3, :3].T + Tcw[:3, 3]
        uv = pc[:, :2] / pc[:, 2:3] * K[0, 0] + K[:2, 2] + rng.normal(0, noise, (len(idx), 2))
        bad = rng.random(len(idx)) < outlier_frac
        uv[bad] += rng.uniform(-30, 30, (int(bad.sum()), 2))
        ef.append(np.full(len(idx), f, np.int32))
        ep.append(idx.astype(np.int32))
        obs.append(uv)
    pb = dict(T_w_c=np.array(T_init), points=(X + rng.normal(0, 1e-2, X.shape)).astype(np.float32),
              edge_frame=np.concatenate(ef), edge_point=np.concatenate(ep), obs=np.concatenate(obs).astype(np.float32))
    if shuffle:
        p = rng.permutation(len(pb["edge_frame"]))
        for k in ("edge_frame", "edge_point", "obs"):
            pb[k] = pb[k][p]
    return pb


def near_plane(z_c, F=2):
    """Frame 0 at the identity and point 0 at (1, 0.5, z_c): its camera depth is exactly z_c (float32 of it), its residual
    about f / z_c pixels."""
    pb = make_problem(3, [60] * F, n_points=60)
    pb["T_w_c"][0] = np.eye(4)
    pb["points"][0] = np.array([1.0, 0.5, z_c], np.float32)
    return pb


def _ba(pb, iters=5, huber=1.0, info=None, fix_first=0, step_tol=0.0, single=False):
    if single:      # optimizeSingleFrame: observation i is of point i
        pb = dict(pb, points=pb["points"][pb["edge_point"]], edge_point=np.arange(len(pb["obs"]), dtype=np.int32))
    return dict(kind="single" if single else "ba", pb=pb, iters=iters, huber=huber, info=info, fix_first=fix_first, step_tol=step_tol)


# ---- the frame-buffer (STORE) variant ---------------------------------------------------------------------------------------
def make_store(seed, counts, ring=8, cap=None, slots=None, min_links=3, dead=0.0, bad_ids=0, cnt_over=None, all_dead=(),
               skip=0, e_upper=None, iters=6, huber=1.0, step_tol=0.0):
    """A frame ring as the tracker keeps it: slots[f] holds frame f of a problem with counts[f] observations (their map point
    ids, pixels and count), the other slots hold garbage that the kernel must not touch.  dead: fraction of observed points
    that left the map; bad_ids: observations whose id is negative or >= n_ids; cnt_over: {frame: extra} counts beyond cap;
    all_dead: frames whose every point is dead."""
    rng = np.random.default_rng(seed + 1000)
    pb = make_problem(seed, counts, n_points=max(64, max(counts)))
    F = len(counts)
    slots = list(range(F)) if slots is None else list(slots)
    cap = cap or max(counts)
    n_ids = len(pb["points"])
    alive = (rng.random(n_ids) >= dead).astype(np.uint8)
    for f in all_dead:
        alive[pb["edge_point"][pb["edge_frame"] == f]] = 0
    edge_map = rng.integers(-5, 2 * n_ids, (ring, cap)).astype(np.int32)      # garbage beyond the counts
    edge_obs = rng.uniform(-1e3, 1e3, (ring, cap, 2)).astype(np.float32)
    cnt = rng.integers(0, cap + 1, ring).astype(np.int32)
    pose = rng.normal(0, 1, (ring, 12))
    for f, s in enumerate(slots):
        m = pb["edge_frame"] == f
        ids, ob = pb["edge_point"][m].copy(), pb["obs"][m]
        n = min(len(ids), cap)
        if bad_ids:
            j = rng.choice(n, min(bad_ids, n), replace=False)
            ids[j] = np.where(rng.random(len(j)) < 0.5, -1 - rng.integers(0, 3, len(j)), n_ids + rng.integers(0, 3, len(j)))
        edge_map[s, :n], edge_obs[s, :n] = ids[:n], ob[:n]
        cnt[s] = len(ids) + (cnt_over or {}).get(f, 0)
        Tcw = np.linalg.inv(pb["T_w_c"][f])
        pose[s, :9], pose[s, 9:] = Tcw[:3, :3].ravel(), Tcw[:3, 3]
    return dict(kind="store", map_pts=pb["points"], alive=alive, edge_map=edge_map, edge_obs=edge_obs, cnt=cnt, pose=pose, cap=cap,
                slots=slots, min_links=min_links, skip=skip, e_upper=int(e_upper if e_upper is not None else sum(counts)),
                iters=iters, huber=huber, step_tol=step_tol)


def store_graph(c):
    """The graph the kernel has to build (vo.cpp:417-440): listed slots in listing order whose min(cnt, cap) >= min_links,
    and of their observations those whose id is in [0, n_ids) and alive."""
    n_ids = len(c["alive"])
    fr, ef, ep, ob = [], [], [], []
    if not c["skip"]:
        for s in c["slots"][:BA_MAXF]:
            n = min(int(c["cnt"][s]), c["cap"])
            if n < c["min_links"]:
                continue
            for j in range(n):
                i = int(c["edge_map"][s, j])
                if 0 <= i < n_ids and c["alive"][i]:
                    ef.append(len(fr))
                    ep.append(i)
                    ob.append(c["edge_obs"][s, j])
            fr.append(s)
    return fr, np.array(ef, np.int32), np.array(ep, np.int32), np.array(ob, np.float32).reshape(-1, 2)


def _Rt_to_T(p):
    T = np.eye(4)
    T[:3, :3] = p[:9].reshape(3, 3).T
    T[:3, 3] = -T[:3, :3] @ p[9:]
    return T


# ---- running ------------------------------------------------------------------------------------------------------------------
def run_case(ctx, c):
    """Runs case c on the library behind ctx; returns a JSON-able dict."""
    if c["kind"] == "store":
        lib = ctx.lib
        f = lib.mvo_test_ba_pose_store
        f.restype = C.c_int
        vp, i, d = C.c_void_p, C.c_int, C.c_double
        f.argtypes = [vp, vp, vp, i, vp, vp, vp, vp, i, i, vp, i, i, i, i, vp, vp, i, i, d, d, vp, vp]
        pose = np.ascontiguousarray(c["pose"], np.float64).copy()
        slots = np.zeros(max(17, len(c["slots"])), np.int32)
        slots[: len(c["slots"])] = c["slots"]
        info = np.full(18, -7, np.int32)
        stats = np.full(16, -7.0)
        arr = [np.ascontiguousarray(c[k]) for k in ("map_pts", "alive", "edge_map", "edge_obs", "cnt")]
        I2 = np.ascontiguousarray(np.eye(2))
        rc = f(ctx.h, arr[0].ctypes.data, arr[1].ctypes.data, len(c["alive"]), arr[2].ctypes.data, arr[3].ctypes.data, arr[4].ctypes.data,
               pose.ctypes.data, len(pose), c["cap"], slots.ctypes.data, len(c["slots"]), c["min_links"], c["skip"], c["e_upper"],
               np.ascontiguousarray(K).ctypes.data, I2.ctypes.data, c["iters"], int(c["huber"] > 0), c["huber"], c["step_tol"],
               info.ctypes.data, stats.ctypes.data)
        return dict(rc=rc, pose=pose.tolist(), info=info.tolist(), stats=stats.tolist())
    pb = c["pb"]
    ctx.set_params(ba_iterations=c["iters"], ba_huber_delta=c["huber"], ba_fix_first_pose=c["fix_first"], ba_step_tol=c["step_tol"])
    try:
        if c["kind"] == "single":
            gp, _ = ctx.optimize_single_frame(pb["T_w_c"][0], pb["points"], pb["obs"], K, fix_points=True, update_points=False)
            gp, gs = gp[None], [0.0] * 4
        else:
            gp, _, gs = ctx.bundle_adjustment(pb["T_w_c"], pb["points"], pb["edge_frame"], pb["edge_point"], pb["obs"], K,
                                              information=c["info"], fix_points=True, update_points=False)
    finally:
        ctx.set_params(ba_iterations=50, ba_huber_delta=1.0, ba_fix_first_pose=0, ba_step_tol=0.0)
    return dict(pose=np.asarray(gp).tolist(), stats=list(map(float, gs)))


def parse_debug(text):
    """The MVO_BA_DEBUG lines of k_ba_pose in text, as dicts."""
    keys = ("F", "E", "Ep", "chunk", "cluster", "it", "trials", "rejected")
    return [dict(zip(keys, map(int, m.groups()))) for m in DEBUG.finditer(text)]


CHILD = r'''
import json, sys
sys.path[:0] = [{root!r}, {tests!r}, {py!r}]
import mvo_b200, {module} as B
ctx = mvo_b200.Context(0)
for name in {names!r}:
    sys.stderr.write("@case " + name + "\n"); sys.stderr.flush()
    print(json.dumps(dict(name=name, **B.run_case(ctx, B.CASES[name]()))), flush=True)
ctx.close()
print("child ok")
'''


def run_children(names, cluster=None, lib=None, timeout=1800, module="ba_pose_cases"):
    """Runs the named cases of module (its CASES, run_case and parse_debug) in one child process (MVO_BA_CLUSTER = cluster,
    MVO_LIB = lib when given, MVO_BA_DEBUG on); returns {name: (result, [debug records])}."""
    import importlib
    parse = importlib.import_module(module).parse_debug
    env = dict(os.environ, MVO_BA_DEBUG="1")
    env.pop("MVO_BA_CLUSTER", None)
    if cluster is not None:
        env["MVO_BA_CLUSTER"] = str(cluster)
    if lib is not None:
        env["MVO_LIB"] = str(lib)
    code = CHILD.format(root=str(ROOT), tests=str(ROOT / "tests"), py=str(PY), names=list(names), module=module)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0 and "child ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])
    res = {}
    for line in r.stdout.splitlines():
        if line.startswith("{"):
            d = json.loads(line)
            res[d.pop("name")] = d
    dbg = {}
    for part in r.stderr.split("@case ")[1:]:
        name, _, rest = part.partition("\n")
        dbg[name] = parse(rest)
    return {n: (res[n], dbg.get(n, [])) for n in names}


# ---- checks ---------------------------------------------------------------------------------------------------------------------
def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


def _trace_counts(trace):
    return len(trace), int((trace[:, 4] == 0).sum())


def oracle(c):
    from oracle import oracle_lib
    if c["kind"] == "store":
        fr, ef, ep, ob = store_graph(c)
        T = np.array([_Rt_to_T(c["pose"][s]) for s in fr]).reshape(-1, 4, 4)
        if not fr:
            return fr, ef, None
        out = oracle_lib.bundle_adjustment_with_trace(T, c["map_pts"], ef, ep, ob, K, fix_points=True, update_points=False,
                                                      iterations=c["iters"], huber_delta=c["huber"])
        return fr, ef, out
    pb = c["pb"]
    ef = pb["edge_frame"] if c["kind"] == "ba" else np.zeros(len(pb["obs"]), np.int32)
    ep = pb["edge_point"] if c["kind"] == "ba" else np.arange(len(pb["obs"]), dtype=np.int32)
    T = pb["T_w_c"] if c["kind"] == "ba" else pb["T_w_c"][:1]
    return oracle_lib.bundle_adjustment_with_trace(T, pb["points"], ef, ep, pb["obs"], K, information=c["info"], fix_points=True,
                                                   update_points=False, iterations=c["iters"],
                                                   huber_delta=0.0 if c["kind"] == "single" else c["huber"],
                                                   fix_first_pose=bool(c["fix_first"]))


def check_lm(gp, gs, op, os_, trace, trials=None, rejected=None, exact_iters=True):
    """Kernel result against the oracle's: chi2 (initial, final) relative 1e-9, poses 1e-8, iterations, trials, rejections."""
    gp, op = np.asarray(gp).reshape(-1, 4, 4), np.asarray(op).reshape(-1, 4, 4)
    assert np.isfinite(gp).all(), gp
    assert _rel(gs[0], os_[0]) < 1e-9 and _rel(gs[1], os_[1]) < 1e-9, (gs, list(os_))
    assert np.abs(gp - op).max() < 1e-8, np.abs(gp - op).max()
    if exact_iters and decisive(os_[0], trace):
        assert gs[2] == os_[2], (gs, list(os_))
        nt, nr = _trace_counts(trace)
        if trials is not None:
            assert (trials, rejected) == (nt, nr), ((trials, rejected), (nt, nr))


def decisive(chi0, trace, margin=1e-11):
    """Whether every trial of the oracle's LM changed chi2 by more than the rounding of the two sums (relative margin): then
    both sides take the same accept / reject decisions.  Once chi2 sits at the optimum, they are rounding-driven (as in
    test_ba_gpu.py::test_converged_fixed_points_50_iterations) and only chi2 and the poses are compared."""
    cur = chi0
    for r in trace:
        if np.isfinite(r[2]) and abs(r[2] - cur) <= margin * abs(cur):
            return False
        if r[4]:
            cur = r[2]
    return True


def check(c, result, debug, csize):
    """Checks one case's result (run_case / run_children) against the oracle; returns the instantiation it reached."""
    if c["kind"] == "store":
        return check_store(c, result, csize)
    pb = c["pb"]
    op, _, os_, trace = oracle(c)
    if c["kind"] == "single":
        assert len(debug) == 1, debug
        d = debug[0]
        counts = [len(pb["obs"])]
        assert np.isfinite(np.asarray(result["pose"])).all()
        # step_tol > 0 ends the LM once a trial step is below it: the pose is final to within that bound
        assert np.abs(np.asarray(result["pose"]).reshape(4, 4) - op[0]).max() < 1e-8
        assert d["it"] <= os_[2] and d["trials"] <= len(trace)
    else:
        F = len(pb["T_w_c"])
        counts = np.bincount(pb["edge_frame"], minlength=F).tolist()
        if c["fix_first"] and F == 1:        # nothing to optimise: the call returns before the kernel, the pose is untouched
            assert debug == [] and np.array_equal(np.asarray(result["pose"]).reshape(-1, 4, 4), pb["T_w_c"])
            assert result["stats"] == [0.0] * 4
            return None
        assert len(debug) == 1, debug
        d = debug[0]
        check_lm(result["pose"], result["stats"], op, os_, trace, d["trials"], d["rejected"])
        assert d["it"] == result["stats"][2]
    chunk, Ep, inst = chunk_rule(counts, csize)
    assert (d["cluster"], d["chunk"], d["Ep"], d["E"]) == (csize, chunk, Ep, sum(counts)), (d, csize, chunk, Ep)
    return inst


def check_store(c, result, csize):
    ring = np.asarray(c["pose"])
    got = np.asarray(result["pose"])
    chunk = store_chunk(c["e_upper"], len(c["slots"]), csize)
    if len(c["slots"]) > BA_MAXF or chunk is None:
        assert result["rc"] == MVO_ERR_UNSUPPORTED, result["rc"]
        return None
    assert result["rc"] == 0, result["rc"]
    fr, ef, out = oracle(c)
    info = result["info"]
    assert info[0] == len(fr), (info[:2], fr)
    assert info[1] == len(ef), (info[1], len(ef))                     # the surviving edges, exactly
    assert info[2:2 + len(fr)] == fr, (info, fr)                       # the slots of the graph in listing order
    assert info[2 + len(fr):] == [-7] * (16 - len(fr)), info           # nothing beyond them
    others = [s for s in range(len(ring)) if s not in fr]
    assert np.array_equal(got[others], ring[others])                    # every slot outside the graph untouched, bit for bit
    if not fr:
        assert result["stats"][:4] == [0.0] * 4 and result["stats"][15] == 0
        return f"<{chunk},true,true>"
    op, _, os_, trace = out
    gp = np.array([_Rt_to_T(got[s]) for s in fr])
    st = result["stats"]
    check_lm(gp, st, op, os_, trace, int(st[15]), int(st[7]), exact_iters=c["step_tol"] == 0)
    return f"<{chunk},true,true>"


# ---- the cases ------------------------------------------------------------------------------------------------------------------
def _lm_reject():
    # a start 0.8 rad / 0.8 from the arc, no robust kernel: the undamped first steps overshoot, and 7 of 15 trials are rejected
    # with chi2 at least 0.2 % above the current one (decided far above rounding)
    return _ba(make_problem(22, [300] * 2, n_points=300, pose_pert=0.8, outlier_frac=0.0), iters=8, huber=0.0)


def _qmax10():
    # frame 0 fixed and frame 1 without edges: the initial damping is 0 (no active diagonal), every solve fails, and the tenth
    # rejected trial ends the LM (qmax == 10) after one iteration
    return _ba(make_problem(23, [200, 0], n_points=200), iters=5, fix_first=1)


CASES = {
    # chunking, at the default cluster of 8 (4096 threads): CH = 1..4 cached, then the uncached kernel
    "ch1": lambda: _ba(make_problem(1, [800] * 5), iters=6),
    "ch2": lambda: _ba(make_problem(2, [1000] * 5), iters=6),
    "ch3": lambda: _ba(make_problem(3, [2500] * 4, n_points=2500), iters=5),
    "ch4": lambda: _ba(make_problem(4, [3500] * 4, n_points=3500), iters=5),
    "unc5": lambda: _ba(make_problem(5, [4200] * 4, n_points=4200), iters=4),
    "unc23": lambda: _ba(make_problem(6, [18500] * 5, n_points=18500), iters=3),
    "unc64": lambda: _ba(make_problem(7, [53000] * 5, n_points=53000), iters=3),
    # the same two rules at a cluster of 1 (512 threads): CH = 2 from 513 edges, uncached from 2049
    "c1_ch2": lambda: _ba(make_problem(24, [300, 300], n_points=300), iters=4),
    "c1_unc5": lambda: _ba(make_problem(25, [1100, 1100], n_points=1100), iters=3),
    # layout
    "many_small_frames": lambda: _ba(make_problem(8, [1, 2, 3, 4, 5, 1, 2, 3, 4, 5, 1, 2, 3, 4, 5, 3], n_points=40), iters=5),
    "empty_frames": lambda: _ba(make_problem(9, [300, 0, 200, 0, 250], n_points=300), iters=6),
    "ragged_ch2": lambda: _ba(make_problem(10, [2 * 701 - 1, 2 * 700 + 1, 2 * 650 - 1, 2 * 600 + 1, 2 * 451], n_points=1500), iters=5),
    "ragged_ch3": lambda: _ba(make_problem(11, [3 * 900 - 1, 3 * 900 + 1, 3 * 800 + 1, 3 * 700 - 1], n_points=2800), iters=5),
    "shuffled": lambda: _ba(make_problem(12, [1200] * 4, n_points=1200, shuffle=True), iters=6),
    "fix_first_f1": lambda: _ba(make_problem(13, [200], n_points=200), iters=5, fix_first=1),
    "fix_first_f2": lambda: _ba(make_problem(14, [200, 300], n_points=300), iters=5, fix_first=1),
    # LM control
    "huber_off": lambda: _ba(make_problem(15, [500] * 3, n_points=500), iters=4, huber=0.0),
    "info_nondiag": lambda: _ba(make_problem(16, [500] * 3, n_points=500), iters=8, info=np.array([[2.0, 0.3], [0.3, 0.5]])),
    "iters1": lambda: _ba(make_problem(17, [300] * 2, n_points=300), iters=1),
    "iters2": lambda: _ba(make_problem(18, [300] * 2, n_points=300), iters=2),
    "rejections": _lm_reject,
    "qmax10": _qmax10,
    # float range: a point next to frame 0's principal plane (residual ~ f / z_c pixels)
    "near_1e-12_huber": lambda: _ba(near_plane(1e-12), huber=1.0),
    "near_1e-18_huber": lambda: _ba(near_plane(1e-18), huber=1.0),
    "near_1e-18_plain": lambda: _ba(near_plane(1e-18), huber=0.0),
    "near_1e-30_huber": lambda: _ba(near_plane(1e-30), huber=1.0),
    "near_1e-30_plain": lambda: _ba(near_plane(1e-30), huber=0.0),
    "near_1e-40_huber": lambda: _ba(near_plane(1e-40), huber=1.0),
    "near_1e-40_plain": lambda: _ba(near_plane(1e-40), huber=0.0),
    "refit_shape": lambda: _ba(near_plane(1e-18, F=1), iters=10, huber=0.0, step_tol=1e-10, single=True),
    # the frame-buffer variant: 5-frame windows in a ring of 8
    "store_basic": lambda: make_store(30, [300, 280, 260, 240, 220], slots=[4, 3, 2, 1, 0]),
    "store_bad_ids": lambda: make_store(31, [300, 280, 260, 240, 220], slots=[6, 1, 3, 0, 5], dead=0.2, bad_ids=25),
    "store_cnt_over_cap": lambda: make_store(32, [300, 280, 260, 240, 220], cap=250, cnt_over={1: 40, 3: 500}),
    "store_min_links": lambda: make_store(33, [300, 2, 260, 3, 1], min_links=3),
    "store_frame_all_dead": lambda: make_store(34, [300, 280, 260, 240, 220], all_dead=(2,)),
    "store_all_dropped": lambda: make_store(35, [2, 1, 0, 2, 1], min_links=3),
    "store_skip": lambda: make_store(36, [300, 280, 260, 240, 220], skip=1),
    "store_slot_order": lambda: make_store(37, [300, 280, 260, 240, 220], slots=[2, 7, 0, 5, 3]),
    "store_16_frames": lambda: make_store(38, [60 + 7 * f for f in range(16)], ring=20, slots=list(range(19, 3, -1)), iters=5),
    "store_17_slots": lambda: make_store(39, [40] * 17, ring=20),
    "store_step_tol": lambda: make_store(40, [300, 280, 260, 240, 220], step_tol=1e-9, iters=10),
    "store_step_tol_ref": lambda: make_store(40, [300, 280, 260, 240, 220], step_tol=0.0, iters=10),
}


def _store_eu(name, seed, e_upper):
    CASES[name] = lambda: make_store(seed, [300, 280, 260, 240, 220], slots=[3, 1, 4, 0, 2], e_upper=e_upper)


# e_upper on each side of each CH boundary of the cluster of 8 (5 slots): CH = ceil((e_upper + 5 (CH - 1)) / 4096)
for _n, _eu in (("eu_ch1", 4096), ("eu_ch2_lo", 4097), ("eu_ch2_hi", 8192 - 5), ("eu_ch3_lo", 8192 - 4), ("eu_ch3_hi", 12288 - 10),
                ("eu_ch4_lo", 12288 - 9), ("eu_ch4_hi", 16384 - 15), ("eu_over", 16384 - 14)):
    _store_eu("store_" + _n, 41, _eu)
