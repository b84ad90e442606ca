"""The pose-only LM kernel (k_ba_pose, csrc/ba.cu) on the H100 against the C oracle, in every launch configuration: the
instantiations <CH,true,false> (CH = 1..4 edges per thread, cached in shared memory), <1,false,false> (uncached, runtime chunk
up to 64, strided sweeps), the frame-buffer variant <CH,true,true> through the test entry mvo_test_ba_pose_store, and cluster
sizes 1..8 (MVO_BA_CLUSTER, out-of-range values fall back to 8).  Cases, rules and checks: tests/ba_pose_cases.py."""
import os

import numpy as np
import pytest

import ba_pose_cases as B

pytestmark = pytest.mark.gpu

CSIZE = B.cluster_size(os.environ.get("MVO_BA_CLUSTER"))
BA_NAMES = [n for n in B.CASES if not n.startswith("store")]
STORE_NAMES = [n for n in B.CASES if n.startswith("store")]
# at the default cluster of 8: what the host's chunk rule must pick for these cases
EXPECTED_CHUNK = {"ch1": 1, "ch2": 2, "ch3": 3, "ch4": 4, "unc5": 5, "unc23": 23, "unc64": 64, "ragged_ch2": 2, "ragged_ch3": 3}


def _run_inproc(ctx, name, monkeypatch, capfd):
    monkeypatch.setenv("MVO_BA_DEBUG", "1")         # read at every call
    c = B.CASES[name]()
    capfd.readouterr()
    r = B.run_case(ctx, c)
    return c, r, B.parse_debug(capfd.readouterr().err)


@pytest.mark.parametrize("name", BA_NAMES)
def test_pose_lm_vs_oracle(ctx, name, monkeypatch, capfd):
    c, r, dbg = _run_inproc(ctx, name, monkeypatch, capfd)
    inst = B.check(c, r, dbg, CSIZE)
    if CSIZE == 8 and name in EXPECTED_CHUNK:
        assert dbg[0]["chunk"] == EXPECTED_CHUNK[name]
        assert inst == (f"<{EXPECTED_CHUNK[name]},true,false>" if EXPECTED_CHUNK[name] <= 4 else "<1,false,false>")
    if name == "unc64" and CSIZE == 8:
        assert dbg[0]["Ep"] // 64 > 8 * B.PF_T           # more chunks than threads: rank 0 sweeps twice
    if name in ("rejections", "qmax10", "iters1", "iters2", "info_nondiag", "many_small_frames", "empty_frames"):
        _, _, os_, trace = B.oracle(c)
        assert B.decisive(os_[0], trace)             # so check() compared iterations, trials and rejections exactly
    if name in ("rejections", "qmax10"):
        assert dbg[0]["rejected"] >= 7
        if name == "qmax10":
            assert len(trace) == 10 and (trace[:, 4] == 0).all() and os_[2] == 1 < c["iters"]


@pytest.mark.parametrize("name", STORE_NAMES)
def test_pose_lm_store_vs_oracle(ctx, name):
    c = B.CASES[name]()
    B.check(c, B.run_case(ctx, c), [], CSIZE)


def test_store_step_tol_only_skips_negligible_trials(ctx):
    """The tracker's ba_step_tol = 1e-9 against the same call with step_tol = 0: poses within 1e-8 (the bound of
    test_tracker_gpu.py::test_ba_step_tolerance_only_skips_negligible_trials), never more trials."""
    a, b = B.run_case(ctx, B.CASES["store_step_tol"]()), B.run_case(ctx, B.CASES["store_step_tol_ref"]())
    assert a["rc"] == b["rc"] == 0 and a["info"] == b["info"]
    assert np.abs(np.asarray(a["pose"]) - np.asarray(b["pose"])).max() < 1e-8
    assert a["stats"][15] <= b["stats"][15]


def test_debug_line_matches_chunk_rule_in_a_child():
    """The chunk rule restated in ba_pose_cases against the padded edge count the library prints, in a fresh process."""
    out = B.run_children(["ragged_ch3", "empty_frames", "unc5"])
    for n, (r, dbg) in out.items():
        counts = np.bincount(B.CASES[n]()["pb"]["edge_frame"], minlength=len(r["pose"])).tolist()
        chunk, Ep, _ = B.chunk_rule(counts, 8)
        assert len(dbg) == 1 and (dbg[0]["chunk"], dbg[0]["Ep"], dbg[0]["cluster"]) == (chunk, Ep, 8), (n, dbg)


CLUSTER_CASES = ["ch1", "ch2", "unc5", "many_small_frames", "empty_frames", "rejections", "near_1e-18_huber",
                 "store_basic", "store_bad_ids", "store_16_frames", "store_eu_ch1"]
_by_cluster = {}


def _cluster_run(cluster):
    if cluster not in _by_cluster:
        _by_cluster[cluster] = B.run_children(CLUSTER_CASES, cluster=cluster)
    return _by_cluster[cluster]


@pytest.mark.parametrize("cluster", [1, 2, 3, 5, 7, 8, 9, 0])
def test_cluster_sizes(built, cluster):
    """Every case at every cluster size against the oracle; two runs bit-identical; 9 and 0 exactly like 8."""
    csize = B.cluster_size(cluster)
    first = _cluster_run(cluster)
    second = B.run_children(CLUSTER_CASES, cluster=cluster)
    for n in CLUSTER_CASES:
        (r, dbg), (r2, _) = first[n], second[n]
        B.check(B.CASES[n](), r, dbg, csize)
        assert _results(r) == _results(r2), n
    if csize != cluster:
        ref = _cluster_run(8)
        for n in CLUSTER_CASES:
            assert _results(first[n][0]) == _results(ref[n][0]), n


def _results(r):
    """What a run computes: everything but the clock64 cycle counts of the frame-buffer entry's stats (4..6, 8..13)."""
    st = r["stats"]
    return dict(r, stats=st[:4] + st[7:8] + st[15:] if len(st) == 16 else st)


def test_every_instantiation_is_reached():
    """The cases above, by the host's rules (which each case checks against the library), reach all nine k_ba_pose kernels."""
    got = set()
    for cs in (1, 2, 3, 5, 7, 8):
        for n in BA_NAMES if cs == CSIZE else [n for n in CLUSTER_CASES if not n.startswith("store")]:
            pb = B.CASES[n]()["pb"]
            got.add(B.chunk_rule(np.bincount(pb["edge_frame"], minlength=len(pb["T_w_c"])).tolist(), cs)[2])
        for n in STORE_NAMES if cs == CSIZE else [n for n in CLUSTER_CASES if n.startswith("store")]:
            c = B.CASES[n]()
            ch = B.store_chunk(c["e_upper"], len(c["slots"]), cs)
            if ch and len(c["slots"]) <= 16:
                got.add(f"<{ch},true,true>")
    want = {f"<{k},true,{s}>" for k in (1, 2, 3, 4) for s in ("false", "true")} | {"<1,false,false>"}
    assert got == want, sorted(got)
