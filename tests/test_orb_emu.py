"""The ORB extraction of the library EXECUTED ON THE CPU: csrc/ctx.cu, csrc/orb.cu and csrc/orb_host.cpp compiled for the host
(tests/emu_build.py: kernels through tests/cpp/cuda_emu.h, one OS thread per CUDA thread; the CUDA runtime calls of the host
code through tests/emu/cuda_runtime_emu.cpp) — the real host orchestration and every ORB kernel — against the numpy
restatement of cv::ORB + selectUniformKptsByGrid (oracle/, pinned against cv2): keypoints and descriptors bit-exact, like the
hardware test tests/test_orb_gpu.py, on small images.  Also run with the geometry fallbacks forced on (MVO_PYR_FUSED /
MVO_GRID_ROUNDS select the kernels that very wide images and high per-cell limits take; separate processes: the switches are read once)."""
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

CHILD = r'''
import sys, ctypes as C, numpy as np
sys.path.insert(0, r"{root}/tests"); sys.path.insert(0, r"{root}"); sys.path.insert(0, r"{root}/monocular-visual-odometry_b200/python")
import emu_build, mvo_synth, mvo_b200
from oracle import oracle_lib, orb_oracle
lib = C.CDLL(str(emu_build.build(r"{tmp}", ["ctx.cu", "orb.cu", "orb_host.cpp"])))
for name in ("mvo_default_params", "mvo_create", "mvo_destroy", "mvo_last_error", "mvo_orb_extract", "mvo_calc_keypoints", "mvo_calc_descriptors"):
    res, args = mvo_b200.SIGNATURES[name]
    getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
cases = [(mvo_synth.gray_to_bgr(mvo_synth.rect_scene(3, 320, 240, n_rect=300)), 500, 8000), (mvo_synth.rect_scene(4, 200, 152, n_rect=120), 1500, 8000),
         # levels above OpenCV's featuresPerLevel: cv::KeyPointsFilter::retainBest (libstdc++ nth_element + partition) restated on the
         # device (k_retain: warp-level and CTA-level partitions), then the grid selection over the retained order (k_select_kept)
         (mvo_synth.rect_scene(4, 200, 152, n_rect=120), 120, 300), (mvo_synth.noise_scene(2, 256, 200), 900, 2000)]
import os
if os.environ.get("MVO_PYR_FUSED", "1") == "0":
    cases = cases[1:3]                     # the fallback kernels: the smaller image only (run time)
lib.mvo_test_orb_host_fallbacks.restype = C.c_uint64
for img, cap, nfeat in cases:
    p = mvo_b200.Params()
    lib.mvo_default_params(C.byref(p))
    p.max_keypoints = cap
    p.orb_nfeatures = nfeat
    h = C.c_void_p()
    assert lib.mvo_create(C.byref(h), 0, C.byref(p)) == 0
    rows, cols = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    kp, desc, n = np.zeros(cap + 8, mvo_b200.KEYPOINT_DTYPE), np.zeros((cap + 8, 32), np.uint8), C.c_int(cap + 8)
    assert lib.mvo_orb_extract(h, img.ctypes.data, rows, cols, ch, cols * ch, kp.ctypes.data, C.byref(n), desc.ctypes.data) == 0, lib.mvo_last_error(h)
    sel = oracle_lib.select_uniform_kpts_by_grid(orb_oracle.detect(img, nfeatures=nfeat), rows, cols, cap, 16, 8)
    assert n.value == len(sel) > 50 and kp[: n.value].tobytes() == sel.tobytes(), "keypoints differ from the oracle"
    assert np.array_equal(desc[: n.value], orb_oracle.compute(img, sel)), "descriptors differ from the oracle"
    lib.mvo_destroy(h)
assert lib.mvo_test_orb_host_fallbacks() == 0, "retainBest fell back to the host"
print("orb emu child ok")
'''


@pytest.mark.parametrize("env", [{}, {"MVO_PYR_FUSED": "0", "MVO_GRID_ROUNDS": "1"}], ids=["shipped", "geometry_fallbacks"])
def test_emulated_orb_extraction_is_bit_exact(tmp_path, env):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=str(ROOT), tmp=str(tmp_path))], capture_output=True, text=True, timeout=900, env=e)
    assert r.returncode == 0 and "orb emu child ok" in r.stdout, (r.stdout[-800:], r.stderr[-2500:])
