"""The RANSAC PnP on the H100 in every launch configuration, against the fp64 oracle (pnp_mode = 0) and the float rule of
cv::solvePnPRansac (pnp_mode = 1): the scoring grid with one and several passes, the staged points below and above 48 KB, the
consensus kernel's register path and its re-read path, the host count and the device count, adversarial scoring inputs, ties
and winners near H = 65535.  Cases, restated launch rules and checks: tests/pnp_cases.py."""
import ctypes as C

import numpy as np
import pytest

import pnp_cases as PC

pytestmark = pytest.mark.gpu
_report = {}


@pytest.mark.parametrize("name", list(PC.CASES))
def test_pnp_case(ctx, name):
    c = PC.CASES[name]()
    cfg = PC.check(c, PC.run_case(ctx, c), _report)
    if name in PC.EXPECT:
        assert cfg == PC.EXPECT[name], (cfg, PC.EXPECT[name])
    if c["tie"] and "pinned" in c["tie"]:
        assert c["tie"]["pinned"] > 0.7 * c["H"]


def test_undecided_fraction():
    """The points the oracle leaves undecided (a few fp64 roundings from the threshold) are a vanishing fraction."""
    assert _report.get("pairs", 0) > 1e8, _report
    frac = _report["undecided"] / _report["pairs"]
    print(f"undecided (hypothesis, point) pairs: {_report['undecided']} of {_report['pairs']} ({frac:.2e})")
    assert frac < 1e-6


def test_every_cell_is_reached():
    """The cases reach every configuration of the launch matrix that exists (pnp_cases.feasible_cells), by the host's rules
    restated with this device's SM count."""
    import subprocess
    import sys
    sm = int(subprocess.run([sys.executable, "-c", "import torch; print(torch.cuda.get_device_properties(0).multi_processor_count)"],
                            capture_output=True, text=True, check=True).stdout)
    got = {PC.config(PC.CASES[n](), sm) for n in PC.CASES}
    assert PC.feasible_cells() <= got, sorted(PC.feasible_cells() - got, key=str)


def test_more_than_10240_correspondences_are_unsupported(ctx):
    import mvo_b200
    P, uv, _, _ = PC.scene(3, 10241)
    for mode in (0, 1):
        ctx.set_params(pnp_mode=mode)
        try:
            with pytest.raises(mvo_b200.MvoError) as e:
                ctx.solve_pnp_ransac(P, uv, PC.K0)
            assert e.value.code == PC.MVO_ERR_UNSUPPORTED
        finally:
            ctx.set_params(pnp_mode=0)
    assert PC.run_dev(ctx, PC._case(P, uv, PC.K0))["rc"] == PC.MVO_ERR_UNSUPPORTED


def test_degenerate_after_a_successful_call(ctx):
    """No model leaves nothing of the previous call on the same context: consensus size 0, no best hypothesis, the identity
    pose, and mvo_solve_pnp_ransac returns MVO_ERR_DEGENERATE with 0 inliers and the output array untouched."""
    assert PC.run_case(ctx, PC.CASES["b_h129_n1025_off_thr37"]())["dev"]["out_i"][0] > 500
    for name in ("none_valid", "none_4_inliers"):
        c = PC.CASES[name]()
        PC.check(c, PC.run_case(ctx, c))
    P, uv, R, t = PC.scene(5, 300)
    assert ctx.solve_pnp_ransac(P, uv, PC.K0)[2].size > 150
    rng = np.random.default_rng(9)
    P4 = rng.uniform(-2, 2, (4, 3)).astype(np.float32) + np.float32([0, 0, 5])
    uv4 = rng.uniform(0, 640, (4, 2)).astype(np.float32)
    h = PC.run_host(ctx, P4, uv4, PC.K0)
    assert h["rc"] == PC.MVO_ERR_DEGENERATE and h["n_inliers"] == 0 and (h["inl"] == -7).all()
    sure, amb = PC.oracle_counts(P4, uv4, PC.K0, h["hyp"][h["counts"] >= 0], 2.0)
    assert (sure + amb).max() < 4 and h["counts"].max() < 4


@pytest.mark.parametrize("mode", [0, 1])
def test_launch_count(ctx, mode):
    """mvo_solve_pnp_ransac and the device path launch four kernels in either mode (hypotheses, scoring, consensus, refit);
    supplied hypotheses skip the first."""
    P, uv, _, _ = PC.scene(4, 500)
    ctx.set_params(pnp_mode=mode)
    try:
        n0 = ctx.kernel_launches
        ctx.solve_pnp_ransac(P, uv, PC.K0)
        n1 = ctx.kernel_launches
        assert PC.run_dev(ctx, PC._case(P, uv, PC.K0, mode=mode))["rc"] == 0
        n2 = ctx.kernel_launches
        assert (n1 - n0, n2 - n1) == (4, 4)
    finally:
        ctx.set_params(pnp_mode=0)
    c = PC.CASES["none_valid"]()
    n2 = ctx.kernel_launches
    PC.run_case(ctx, c)
    assert ctx.kernel_launches - n2 == 3
