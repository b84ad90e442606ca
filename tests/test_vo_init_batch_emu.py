"""mvo_vo_init_candidates_batch_dev EXECUTED ON THE CPU: the whole library built for the host (tests/emu_build.py, every
translation unit plus vo_init_batch.cu), so the kernel runs through tests/cpp/cuda_emu.h and its device code is compiled by g++:
acos is glibc's there, and every pair's record, kept matches, kept points and kept angles must be BYTE-IDENTICAL to the host
reference (tests/vo_init_batch_cases.py: the state machine's own sequence over the library's host entry points).  Also: the
restatements of std::nth_element and std::sort (csrc/vo_init_math.cuh) against libstdc++ on NaN-laden and tie-heavy arrays.  The
emulation cannot show the device's acos or a contraction difference: tests/test_vo_init_batch_gpu.py is the check on the
hardware."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import vo_init_batch_cases as cases

CAP = 320


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    import emu_build
    import mvo_b200
    so = emu_build.build(tmp_path_factory.mktemp("voinitbatchemu"), emu_build.ALL_UNITS + ["vo_init_batch.cu"])
    lib = C.CDLL(str(so))
    for name in ("mvo_default_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_kernel_launches", "mvo_vo_default_params",
                 "mvo_retain_good_triangulation", "mvo_normalize_init_depth", "mvo_is_vo_good_to_init", "mvo_vo_init_candidates_batch_dev"):
        res, args = mvo_b200.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def ctx(lib):
    import mvo_b200
    p = mvo_b200.Params()
    lib.mvo_default_params(C.byref(p))
    h = C.c_void_p()
    assert lib.mvo_create(C.byref(h), 0, C.byref(p)) == 0
    yield h
    lib.mvo_destroy(h)


def _run(lib, ctx, b, T_ref, vp):
    l0 = lib.mvo_kernel_launches(ctx)
    rc, got = cases.call(lib, ctx, b, T_ref, vp)
    assert rc == 0, lib.mvo_last_error(ctx)
    assert lib.mvo_kernel_launches(ctx) - l0 == 1
    return got


@pytest.mark.parametrize("T_ref", ["general", "identity"])
def test_emulated_batch_equals_the_state_machine(lib, ctx, T_ref):
    T = cases.T_REF if T_ref == "general" else np.eye(4)
    specs = cases.mixed_specs(CAP, CAP)
    b = cases.Batch(specs, CAP, seed=3)
    vp = cases.vo_params(lib)
    got = _run(lib, ctx, b, T, vp)
    refs = [cases.reference(lib, b, p, T, vp) for p in range(b.n_pairs)]
    for p in range(b.n_pairs):
        cases.check_exact(refs[p], got, p)
    recs = [r[1] for r in refs]
    # the batch reaches what it was built for
    assert [recs[i]["best_sol"] for i in (0, 1, 2)] == [0, 1, 2]
    assert recs[0]["good"] == 1 and recs[0]["normalized"] == 1
    assert recs[3]["usable"] == 1 and recs[3]["n_inliers"] == 0 and recs[3]["n_kept"] == 0 and np.isnan(recs[3]["mean_pixel_dist"])
    assert recs[4]["n_inliers"] == 40 and recs[4]["n_kept"] == 0 and recs[4]["median_angle"] == 0
    assert (recs[5]["n_kept"], recs[5]["normalized"], recs[6]["n_kept"], recs[6]["normalized"]) == (19, 0, 20, 1)
    assert recs[7]["n_kept"] == 117
    for i in (8, 9, 10):
        assert np.isnan(refs[i][4]).any(), i                             # NaN angles are kept
    assert np.isnan(recs[9]["median_angle"])                            # ... and one is the median
    assert recs[11]["good"] == 0
    assert recs[12]["n_inliers"] == CAP
    assert recs[13]["usable"] == 0 and recs[13]["status"] == 0 and (recs[13]["T_w_c"] == np.ravel(T)).all()
    assert refs[14][0] == cases.INVALID_ARG
    assert [r[0] for r in refs[15:15 + len(cases.BAD_KINDS)]] == [cases.INVALID_ARG] * len(cases.BAD_KINDS)


def test_emulated_thresholds_exactly_on_an_angle(lib, ctx):
    for b, vp in cases.boundary_batches(lib, CAP):
        got = _run(lib, ctx, b, cases.T_REF, vp)
        ref = cases.reference(lib, b, 0, cases.T_REF, vp)
        cases.check_exact(ref, got, 0)
    base = cases.reference(lib, b, 0, cases.T_REF, cases.vo_params(lib))[1]
    kept = [cases.reference(lib, b, 0, cases.T_REF, vp)[1] for b, vp in cases.boundary_batches(lib, CAP)]
    assert kept[0]["n_kept"] == base["n_kept"] - 10                      # the angle at the minimum stays, the ten below go
    assert kept[1]["n_kept"] == base["n_kept"] - 1                       # the one above max_ratio x median goes
    assert base["good"] == 1 and kept[2]["good"] == 0


def test_emulated_call_level_checks(lib, ctx):
    b = cases.Batch([dict(n=30)], CAP)
    vp = cases.vo_params(lib)
    assert cases.call(lib, ctx, b, cases.T_REF, vp)[0] == 0
    for q in (np.nan, np.inf):
        T = cases.T_REF.copy()
        T[1, 3] = q
        assert cases.call(lib, ctx, b, T, vp)[0] == cases.INVALID_ARG
        for f in ("min_triang_angle", "max_ratio_angle_to_median", "min_pixel_dist", "min_median_triangulation_angle", "assumed_mean_depth_init"):
            assert cases.call(lib, ctx, b, cases.T_REF, cases.vo_params(lib, **{f: q}))[0] == cases.INVALID_ARG, f


HARNESS = r"""
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
#include "vo_init_math.cuh"
int main() {
  std::mt19937_64 rng(7);
  int bad = 0, runs = 0;
  const int sizes[] = {1, 2, 3, 4, 5, 16, 17, 18, 33, 64, 100, 257, 1000, 6400};
  for (int n : sizes)
    for (int kind = 0; kind < 6; ++kind)
      for (int rep = 0; rep < 20; ++rep) {
        std::vector<double> v(n);
        for (int i = 0; i < n; ++i) {
          const unsigned long long r = rng();
          double x = kind == 2 || kind == 5 ? (double)(r % 4) : (double)(r % 100000) / 7.0;          // ties
          if (kind == 1 && r % 5 == 0) x = NAN;                                                      // NaN-laden
          if (kind == 3 && r % 2 == 0) x = NAN;
          if (kind == 4 && r % 11 == 0) x = -NAN;
          if (kind == 5 && r % 3 == 0) x = NAN;
          v[i] = x;
        }
        if (kind == 0 && rep % 2) std::sort(v.begin(), v.end());                                    // presorted / reversed
        if (kind == 0 && rep % 4 == 3) std::reverse(v.begin(), v.end());
        std::vector<double> a = v, b = v, c = v, d = v;
        std::nth_element(a.begin(), a.begin() + n / 2, a.end());
        voi::nth_element_d(b.data(), n / 2, n);
        std::sort(c.begin(), c.end());
        int stack[3 * voi::SORT_STACK];
        voi::sort_d(d.data(), n, stack);
        bad += memcmp(a.data(), b.data(), n * 8) != 0;
        bad += memcmp(c.data(), d.data(), n * 8) != 0;
        runs += 2;
      }
  printf("%d %d\n", bad, runs);
  return 0;
}
"""


def test_selection_and_sort_restate_libstdcxx(tmp_path):
    """The whole array after the call, not only the value at n / 2, equals libstdc++'s: with and without NaN, with ties, presorted
    and reversed, across the 16-element and 3-element switches."""
    import emu_build
    src = tmp_path / "stl_restate.cpp"
    src.write_text(HARNESS)
    exe = tmp_path / "stl_restate"
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I", str(emu_build.CSRC), str(src), "-o", str(exe)], check=True)
    bad, runs = (int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    assert runs == 14 * 6 * 20 * 2 and bad == 0, bad
