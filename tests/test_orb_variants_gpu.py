"""The geometry fallbacks of the ORB path, forced on ordinary scenes (MVO_PYR_FUSED=0: k_gray + k_resize, taken for very wide images
with many levels; MVO_FAST_TMA=0: vector-load staging, taken above 1024 px; MVO_GRID_ROUNDS=1: round-based grid selection, taken above
254 points per cell; MVO_PDL=0: plain launches).  The switches are read once per process, so each configuration runs in its own child
process; keypoints and descriptors must be byte-identical with the default kernels' (which are themselves bit-exact with cv2,
tests/test_orb_gpu.py)."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import os as _os
_TIMEOUT_SCALE = float(_os.environ.get("MVO_TEST_TIMEOUT_SCALE", "1"))      # > 1 when the library under test is the CPU emulation (MVO_LIB)

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.gpu

CHILD = r'''
import sys
import numpy as np
sys.path.insert(0, r"{root}"); sys.path.insert(0, r"{root}/monocular-visual-odometry_b200/python")
import mvo_b200, mvo_synth
out = {{}}
for cap in (1500, 2000):
    ctx = mvo_b200.Context(0, max_keypoints=cap)
    scenes = [mvo_synth.gray_to_bgr(mvo_synth.rect_scene(s)) for s in range(3)] + [mvo_synth.color_scene(5), mvo_synth.noise_scene(2),
              mvo_synth.gray_to_bgr(mvo_synth.rect_scene(7, 517, 389, n_rect=900)), mvo_synth.rect_scene(9)]
    for i, img in enumerate(scenes):
        kp, desc = ctx.orb_extract(img)
        out["kp_%d_%d" % (cap, i)] = kp.view(np.uint8)
        out["desc_%d_%d" % (cap, i)] = desc
    ctx.close()
np.savez(r"{out}", **out)
print("orb variant child ok")
'''


def _extract(tmp_path, name, env):
    out = tmp_path / f"{name}.npz"
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=str(ROOT), out=str(out))], capture_output=True, text=True, timeout=240 * _TIMEOUT_SCALE, env=e)
    assert r.returncode == 0 and "orb variant child ok" in r.stdout, (r.stdout[-800:], r.stderr[-2500:])
    return np.load(out)


@pytest.mark.parametrize("env", [{"MVO_PYR_FUSED": "0", "MVO_FAST_TMA": "0", "MVO_GRID_ROUNDS": "1", "MVO_PDL": "0"}], ids=["geometry_fallbacks"])
def test_variant_is_byte_identical_with_the_shipped_kernels(built, tmp_path, env):
    ref = _extract(tmp_path, "shipped", {})
    got = _extract(tmp_path, "variant", env)
    assert sorted(ref.files) == sorted(got.files)
    for k in ref.files:
        assert np.array_equal(ref[k], got[k]), k
