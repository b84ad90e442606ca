"""The free-points Schur bundle adjustment (k_ba, csrc/ba.cu) in the complete library built for the host (tests/emu_build.py,
as in test_full_library_emu.py) against the C oracle, in a child process (MVO_LIB points the wrapper at the emulated build).
The CPU-tier subset of test_ba_schur_gpu.py: CTAs without points and two linearisation rounds, a one-point staging tail, the
structure-only problem, sixteen frames with the first one fixed, both solve failures (every Hll singular, and one singular
block on one CTA only), the input on which the gain denominator took a failed solve's NaN, and duplicated observations.
Cases and checks: tests/ba_schur_cases.py.  85 s on 8 CPU cores, the emulated build (about 20 s) included."""
import pytest

import ba_schur_cases as S

SUBSET = ["P1", "P7", "P2049", "stage_F5_pc+1", "structure_only_P7", "F16_fix_small", "zero_info", "zero_depth_rank0_fix",
          "zero_depth_rank5_fix", "divergence", "duplicates"]


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    import emu_build
    return emu_build.build(tmp_path_factory.mktemp("schuremu"), emu_build.ALL_UNITS)


def test_schur_subset_matches_the_oracle(emu_lib):
    got = set()
    for n, (r, dbg) in S.run_children(SUBSET, lib=emu_lib).items():
        got |= S.check(S.CASES[n](), r, dbg)
    assert {"cta_without_points", "rounds=2_and_1", "one_point_tail", "n=0", "n=90"} <= got, sorted(got)


def test_every_configuration_is_reached():
    """The cases, by the host's rules restated in ba_schur_cases (which every case checks against the library's debug line),
    reach every configuration of k_ba in REQUIRED: one, two, three and ten linearisation rounds per CTA, two rounds on ranks 0..6
    and one on rank 7, a CTA without points, a one-point staging tail, per = pc - 1, pc, pc + 1 and 2 pc + 1 for F = 1, 4, 5, 8
    and 16, and n = 0, 6, 90 and 96."""
    got = set()
    for make in S.CASES.values():
        got |= S.configs(make())
    assert S.REQUIRED <= got, sorted(S.REQUIRED - got)
    assert S.rounds(2049) == [2] * 7 + [1] and S.rounds(20000) == [10] * 8
    assert [S.pc_rule(F) for F in (1, 3, 4, 5, 6, 8, 12, 16)] == [64, 64, 55, 44, 37, 28, 18, 14]
