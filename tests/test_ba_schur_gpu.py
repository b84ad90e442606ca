"""The free-points Schur bundle adjustment (k_ba, csrc/ba.cu) on the H100 against the C oracle, in every launch configuration:
CTAs without points, one to ten linearisation rounds per CTA, staging chunks with a one-point tail, fewer points than a chunk
and exactly one or two chunks for F = 1, 4, 5, 8 and 16, pose systems of n = 0, 6, 90 and 96 rows, graph layouts (points
without edges, points seen once or by the fixed frame only, frames without edges, duplicated and shuffled edges), the LM
control against the oracle's trace (trials and rejections), both ways the Schur solve fails (every Hll singular, one CTA's
block singular) and points at depths down to 1e-18.  Cases, rules and checks: tests/ba_schur_cases.py."""
import numpy as np
import pytest

import ba_schur_cases as S

pytestmark = pytest.mark.gpu

ZERO_DEPTH = [n for n in S.CASES if n.startswith("zero_depth")]
# cases whose LM decisions are all taken far above rounding: check() compared iterations, trials and rejections exactly
DECISIVE = ["rejections", "zero_info", "divergence", "iters1", "iters2", "info_nondiag", "huber_off", "duplicates", "shuffled",
            "P2049", "P4097", "F16_fix", "empty_active_frame"] + ZERO_DEPTH


def _run(ctx, name, monkeypatch, capfd):
    monkeypatch.setenv("MVO_BA_DEBUG", "1")         # read at every call
    c = S.CASES[name]()
    capfd.readouterr()
    r = S.run_case(ctx, c)
    return c, r, S.parse_debug(capfd.readouterr().err)


@pytest.mark.parametrize("name", list(S.CASES))
def test_schur_ba_vs_oracle(ctx, name, monkeypatch, capfd):
    c, r, dbg = _run(ctx, name, monkeypatch, capfd)
    S.check(c, r, dbg)
    _, r2, dbg2 = _run(ctx, name, monkeypatch, capfd)
    assert r2 == r                                  # poses, points and stats 0..3 bit for bit
    assert [(d["it"], d["trials"], d["rejected"]) for d in dbg2] == [(d["it"], d["trials"], d["rejected"]) for d in dbg]
    if name in DECISIVE:
        _, _, os_, trace = S.oracle(c)
        assert S._decisive(os_, trace), name
        if name == "rejections":
            assert dbg[0]["rejected"] >= 2, dbg
        if name == "zero_info":              # lambda_0 = 0, every solve fails, the tenth rejection ends the LM
            assert (dbg[0]["it"], dbg[0]["trials"], dbg[0]["rejected"]) == (1, 10, 10) and os_[2] == 1 < c["iters"]
        if name == "divergence" or name.startswith("zero_depth"):   # every solve fails; each trial is accepted at DBL_MAX
            assert r["stats"][0] == np.inf and r["stats"][1] == S.DBL_MAX and dbg[0]["rejected"] == 0, (r["stats"], dbg)
