"""The RANSAC PnP in the complete library built for the host (tests/emu_build.py, as in test_full_library_emu.py) against the
fp64 oracle and the float rule, in a child process (MVO_LIB points the wrapper at the emulated build).  The CPU-tier subset of
test_pnp_cases_gpu.py: the grid-stride scoring loop, the consensus kernel's re-read path with a small H, the device count with
inlier copies past it in both modes, adversarial scoring inputs, ties and a sole winner at 65534 of 65535, no model, and
pnp_mode = 1 at n = 4097.  The emulation's __fdividef is an exact division, so only the H100 tests the fp32 bound of the
scoring kernel as compiled.  Cases and checks: tests/pnp_cases.py."""
import pytest

import pnp_cases as PC


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    import emu_build
    return emu_build.build(tmp_path_factory.mktemp("pnpemu"), emu_build.ALL_UNITS)


# four groups, run concurrently: mode 1 costs ~45 s per run on the emulation (the one-sided Jacobi of k_pnp_epnp synchronises its
# warp at every rotation), so its two larger device-count cases run without the two comparison runs here
GROUPS = [["b_h4225_n1025", "b_h512_n4097_off", "b_h8_n5_thr05", "adv_default", "none_valid", "none_4_inliers"],
          ["tie_1500_3000_65534", "sole_65534"],
          [n for n in PC.CASES if n.startswith("cnt_b300")],
          ["cnt_cv4500_c4097", "cnt_cv300_c299", "cnt_cv300_c5", "cnt_cv300_c0"]]
LIGHT = ["cnt_cv4500_c4097", "cnt_cv300_c299"]


def test_pnp_cases(emu_lib, tmp_path):
    out = PC.run_children(GROUPS, tmp_path, lib=emu_lib, light=LIGHT)
    report = {}
    for n in [n for g in GROUPS for n in g]:
        c = PC.CASES[n]()
        cfg = PC.check(c, out[n], report)
        if n in PC.EXPECT:
            assert cfg == PC.EXPECT[n], (n, cfg)
    assert PC.config(PC.CASES["b_h4225_n1025"]())[1] and PC.config(PC.CASES["cnt_cv4500_c4097"]())[3]
