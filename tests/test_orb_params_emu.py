"""The ORB extraction over its parameter space on the library built for the host (tests/emu_build.py: csrc/ctx.cu, orb.cu and
orb_host.cpp, every kernel executed on the CPU) against the numpy oracle, bit-exact: the small-image cases of tests/orb_cases.py
(`tier == "both"`) on one context per child process, four children at once, plus a batch that mixes the ovf0 and device retainBest
paths followed by a batch of one on the same context, and the grid selection's treatment of keypoints outside the grid.
Among them: a single-level pyramid (k_pyramid once wrote level 0 into shared memory it had not sized for it), grid cells past the
covered image (the device kernels once clamped such keypoints into the last cell, the host path skipped them) and rejected
configurations that must be rejected again on the same context.  About 75 s on 8 CPU cores, the emulated build included."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import pytest

import orb_cases as O

ROOT = Path(__file__).resolve().parent.parent
SUBSET = [c["name"] for c in O.CASES if c["tier"] == "both"]

CHILD = r'''
import sys, ctypes as C, numpy as np
sys.path.insert(0, r"{root}/tests"); sys.path.insert(0, r"{root}"); sys.path.insert(0, r"{root}/monocular-visual-odometry_b200/python")
import orb_cases as O
lib = O.bind(C.CDLL(r"{lib}"))
h = C.c_void_p()
assert lib.mvo_create(C.byref(h), 0, None) == 0
for name in {names!r}:
    if name == "batch":
        frames, paths = O.batch_frames(small=True)
        p = dict(orb_nfeatures=300, max_keypoints=200)
        O.set_params(lib, h, p)
        refs = [O.reference_oracle(f, p) for f in frames]
        B, cap = len(frames), 201
        imgs = np.ascontiguousarray(np.stack(frames))
        kp, desc, cnt = np.zeros(B * cap * 28, np.uint8), np.zeros(B * cap * 32, np.uint8), np.zeros(B, np.int32)
        read = lambda: (kp, desc, cnt)
        O.check_batch(frames, paths, O.batch_run(lib, h, frames, imgs.ctypes.data, kp.ctypes.data, desc.ctypes.data, cnt.ctypes.data, cap, read),
                      refs, p)
        one = np.ascontiguousarray(imgs[1:2])                 # a batch of one after a batch of three: workspace carved with the capacity
        kp[:], desc[:], cnt[:] = 0, 0, 0
        O.check_batch(frames[1:2], paths[1:2], O.batch_run(lib, h, frames[1:2], one.ctypes.data, kp.ctypes.data, desc.ctypes.data,
                                                           cnt.ctypes.data, cap, read), refs[1:2], p)
    elif name == "grid_rank_outside":
        O.check_grid_rank_outside(lib, h)
    else:
        c = O.CASE[name]
        O.check(c, O.run(lib, h, c), None if c["err"] is not None else O.reference_oracle(O.image(c), c["p"]))
    print("ok", name, flush=True)
lib.mvo_destroy(h)
'''


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    import emu_build
    return emu_build.build(tmp_path_factory.mktemp("orbparams"), ["ctx.cu", "orb.cu", "orb_host.cpp"])


def _child(lib, names):
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=str(ROOT), lib=str(lib), names=names)], capture_output=True, text=True,
                       timeout=900, env=dict(os.environ))
    done = {ln.split()[1] for ln in r.stdout.splitlines() if ln.startswith("ok ")}
    return names, done, r


def test_parameter_cases_match_the_oracle(emu_lib):
    names = SUBSET + ["batch", "grid_rank_outside"]
    chunks = [names[i::4] for i in range(4)]
    with ThreadPoolExecutor(4) as ex:
        results = list(ex.map(lambda ch: _child(emu_lib, ch), chunks))
    failed = []
    for chunk, done, r in results:
        if set(chunk) - done:
            failed.append((sorted(set(chunk) - done), r.returncode, r.stdout[-400:], r.stderr[-2000:]))
    assert not failed, failed


def test_every_configuration_is_reached():
    """The cases, by the host's rules restated in orb_cases, reach every configuration in REQUIRED: pyramid depths 1, 2, 3, 4 and 8,
    scale factors 1.05, 1.2, 1.5 and 2, thresholds on both sides of the packed / scalar quick reject, the fused pyramid and its
    fallback, TMA and vector staging, grid cell by shift and by division, the two-pass and the round selection in k_select and
    k_select_kept, the three retainBest paths (also with keypoints in the uncovered strip), widths of every residue mod 4, short last
    bands, 1 and 3 channels, padded and unaligned strides, the largest orb_nfeatures accepted and every rejection."""
    got = set()
    for c in O.CASES:
        got |= O.configs(c)
    assert O.REQUIRED <= got, sorted(O.REQUIRED - got)
    assert O.max_nfeatures(1200) == 21561 and O.plan(480, 640, {})["pyr_rows"] == [13, 10, 7, 5]
    assert O.plan(480, 640, dict(orb_nfeatures=21562)) == {"err": "select_smem"}
    small = O.CASE["nl1_200x152"]
    assert "pyramid:fused" in O.configs(small) and O.case_plan(small)["pyr_smem"] == 16
