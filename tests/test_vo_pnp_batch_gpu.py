"""mvo_vo_pnp_batch_dev on the hardware.

- The fabricated jobs of tests/vo_pnp_batch_cases.py at cap 2008 (the bench's), 2456 / 2457 (the scoring kernel's shared memory
  either side of the 48 KB opt-in), 4096, 4097 (the uncached refit, the finish kernel's re-read path) and 8192: records, inlier
  lists and Rt byte for byte against the single device call mvo_test_pnp_dev, consensus sets and poses against
  mvo_solve_pnp_ransac, T_w_c and pnp_ok against the state machine's composition, sentinels past every count.
- d_kept = NULL, max_dist_to_prev at exactly the distance, every call-level check.
- Determinism and five launches for 1, 63 and 500 jobs.
- Cluster sizes 1 and 8 of the refit (MVO_BA_CLUSTER, read once per process: child processes), each bit-identical to the single
  device call at that size.
- The state machine end to end on the bench's room sequence: every tracked frame replayed through one extraction, one map-matches
  call and one PnP call per map version."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import vo_pnp_batch_cases as cases

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def gctx(built):
    import mvo_b200
    c = mvo_b200.Context(0)
    yield c
    c.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _runner(gctx):
    """call() on device copies of the scene and outputs; returns (rc, outputs back on the host) and records the launches."""
    import torch

    def run(s, tp, outs, **kw):
        keep = {id(a): _dev(a) for a in (s.mm, s.matches, s.p3, s.p2, s.T_prev) + tuple(o for o in outs if o is not None)}
        torch.cuda.synchronize()
        l0 = gctx.kernel_launches
        rc, _ = cases.call(gctx.lib, gctx.h, s, tp, ptr=lambda a: keep[id(a)].data_ptr(), outs=outs, **kw)
        run.launches = gctx.kernel_launches - l0
        gctx.synchronize()
        got = tuple(None if o is None else keep[id(o)].cpu().numpy().view(o.dtype).reshape(o.shape) for o in outs)
        return rc, got
    return run


@pytest.mark.parametrize("cap", [2008, 2456, 2457, 4096, 4097, 8192])
def test_cases_equal_the_single_calls(gctx, cap):
    s = cases.Scene(cap, seed=cap)
    tp = cases.track_params(gctx.lib)
    H = gctx.params.pnp_hypotheses
    refs = [cases.reference(gctx.lib, gctx.h, s, j, tp, H) for j in range(s.n_jobs)]
    run = _runner(gctx)
    rc, outs = run(s, tp, cases.outputs(s.n_jobs, cap))
    assert rc == 0 and run.launches == cases.LAUNCHES
    cases.check_coverage(outs, s)
    for j in range(s.n_jobs):
        cases.check_exact(refs[j], outs, s, j)
        cases.check_host(gctx.lib, gctx.h, s, j, tp, outs, 8)


def test_without_kept_rows_at_the_threshold_and_call_checks(gctx):
    s = cases.Scene(cases.KCAP, seed=7)
    tp = cases.track_params(gctx.lib)
    H = gctx.params.pnp_hypotheses
    run = _runner(gctx)
    t = s.subset([1, 3, 4, 8, 9, 13])
    refs = [cases.reference(gctx.lib, gctx.h, t, j, tp, H) for j in range(t.n_jobs)]
    rc, outs = run(t, tp, cases.outputs(t.n_jobs, s.cap, kept=False))
    assert rc == 0
    for j in range(t.n_jobs):
        cases.check_exact(refs[j], outs, t, j)
    cases.check_threshold(gctx.lib, gctx.h, s, tp, run=run)
    for kw, want in cases.call_level_kinds(s) + [(dict(n_jobs=1025), cases.UNSUPPORTED)]:     # 1025 x 4096 hypotheses > 2^22
        outs = cases.outputs(s.n_jobs, s.cap)
        rc, got = run(s, tp, outs, **kw)
        assert rc == want and run.launches == 0, (kw, rc)
        assert all((a.view(np.uint8) == cases.SENTINEL).all() for a in got), kw


@pytest.mark.parametrize("n_jobs", [1, 63, 500])
def test_determinism_and_launches(gctx, n_jobs):
    s = cases.Scene(cases.KCAP, seed=4)
    tp = cases.track_params(gctx.lib)
    valid = s.n_jobs - s.n_bad
    t = s.subset(np.arange(n_jobs) % s.n_jobs)
    run = _runner(gctx)
    rc, a = run(t, tp, cases.outputs(n_jobs, s.cap))
    la = run.launches
    rc2, b = run(t, tp, cases.outputs(n_jobs, s.cap))
    assert rc == rc2 == 0 and la == run.launches == cases.LAUNCHES
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    out, inl, kept = cases.views(a, n_jobs, s.cap)
    for j in range(n_jobs):                                          # a repeated job gives the same rows
        k = j % s.n_jobs
        assert out[j].tobytes() == out[k].tobytes() and inl[j].tobytes() == inl[k].tobytes() and kept[j].tobytes() == kept[k].tobytes()
    assert valid > 0


@pytest.mark.parametrize("csize", [1, 8])
def test_cluster_sizes_in_child_processes(built, csize, tmp_path):
    """The refit at cluster size 1 (cap 2008 > 512 edge slots: the uncached kernel) and 8 (cached), each in its own process."""
    script = tmp_path / "child.py"
    script.write_text('''
import sys
sys.path[:0] = [sys.argv[1], sys.argv[2], sys.argv[3]]
import numpy as np, torch, mvo_b200, vo_pnp_batch_cases as cases
csize, cap = int(sys.argv[4]), int(sys.argv[5])
ctx = mvo_b200.Context(0)
s = cases.Scene(cap, seed=11)
tp = cases.track_params(ctx.lib)
H = ctx.params.pnp_hypotheses
refs = [cases.reference(ctx.lib, ctx.h, s, j, tp, H) for j in range(s.n_jobs)]
outs = cases.outputs(s.n_jobs, cap)
keep = {id(a): torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
        for a in (s.mm, s.matches, s.p3, s.p2, s.T_prev) + outs}
rc, _ = cases.call(ctx.lib, ctx.h, s, tp, ptr=lambda a: keep[id(a)].data_ptr(), outs=outs)
assert rc == 0
ctx.synchronize()
got = tuple(keep[id(o)].cpu().numpy().view(o.dtype).reshape(o.shape) for o in outs)
cases.check_coverage(got, s)
for j in range(s.n_jobs):
    cases.check_exact(refs[j], got, s, j)
    cases.check_host(ctx.lib, ctx.h, s, j, tp, got, csize)
ctx.close()
print("ok", csize)
''')
    env = dict(os.environ, MVO_BA_CLUSTER=str(csize))
    r = subprocess.run([sys.executable, str(script), str(ROOT), str(ROOT / "monocular-visual-odometry_b200" / "python"), str(ROOT / "tests"),
                        str(csize), str(cases.KCAP)], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_state_machine_tracking_end_to_end(built):
    """Every tracked frame of the state machine on the bench's room sequence (host-array mode), replayed through one extraction,
    one map-matches call and one PnP call per map version."""
    import mvo_b200
    import mvo_synth
    imgs = [mvo_synth.gray_to_bgr(f) for f in mvo_synth.cached_room_loop_sequence(seed=0)[0]]
    ev, vp = cases.record_tracking(imgs, mvo_synth.K_DEFAULT)
    assert len(ev) > 50, len(ev)
    assert any(e["pnp_ok"] for e in ev)
    bctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    try:
        rp = cases.Replay(bctx, ev, imgs, vp, mvo_synth.K_DEFAULT)
        worst = cases.check_replay(rp)
        print(f"{len(ev)} tracked frames replayed in {len(rp.groups)} PnP calls; largest T_w_c_pnp difference {worst:.3g}")
    finally:
        bctx.close()
