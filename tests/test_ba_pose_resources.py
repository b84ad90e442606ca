"""Compiled resources of the pose-only LM kernel (k_ba_pose, csrc/ba.cu), read from libmvo.so with cuobjdump.

The per-thread accumulators of the pass (32 doubles) and the warp fold over them must stay in registers: when the front end
demotes them to local memory every instantiation gets a >= 512-byte stack frame and the fold runs through L1.  What may
remain is the local array of sincos' slow-path argument reduction (huge rotation angles only), a few dozen bytes."""
import re
import shutil
from pathlib import Path

import pytest

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def _pose_kernel_stacks(lib):
    import subprocess
    if not Path(CUOBJDUMP).exists():
        pytest.skip("cuobjdump not available")
    out = subprocess.run([CUOBJDUMP, "-res-usage", str(lib)], capture_output=True, text=True, check=True).stdout
    stacks = {}
    for m in re.finditer(r"Function (\S*k_ba_poseILi(\d)ELb(\d)ELb(\d)E\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", out):
        stacks[(int(m.group(2)), int(m.group(3)), int(m.group(4)))] = int(m.group(6))
    return stacks


def test_pose_lm_accumulators_in_registers(built):
    stacks = _pose_kernel_stacks(built)
    assert (1, 1, 1) in stacks and (1, 1, 0) in stacks, sorted(stacks)
    for key, stack in stacks.items():
        assert stack < 128, f"k_ba_pose<{key}>: {stack}-byte stack frame (accumulators demoted to local memory?)"
    # the instantiations of the PnP refit and of the tracker's window BA (one edge per thread): no spills either
    for key in ((1, 1, 1), (1, 1, 0)):
        assert stacks[key] <= 48, f"k_ba_pose<{key}>: {stacks[key]}-byte stack frame"
