"""Timing of the ORB geometry fallbacks (and of plain launches) against the default kernels: batched device-resident extraction (64 frames
per call, as bench.py's orb_batch entry) per kernel class.  The switches are read once per process, so this script
re-executes itself once per configuration.  Usage: python tools/dev_orb_variants.py  -> one JSON line per configuration."""
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CONFIGS = [{}, {"MVO_PYR_FUSED": "0"}, {"MVO_FAST_TMA": "0"}, {"MVO_GRID_ROUNDS": "1"}, {"MVO_PDL_ORB": "0"}]


def child():
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "monocular-visual-odometry_b200" / "python"))
    import mvo_b200
    import mvo_synth
    import torch
    B, H, W = 64, 480, 640
    cap = 2001
    stream = torch.cuda.Stream()
    ctx = mvo_b200.Context(0, max_keypoints=2000)
    ctx.set_stream(stream.cuda_stream)
    frames, _, _ = mvo_synth.planar_sequence(0, n_frames=16, plane_z=4.0)
    d_frames = torch.empty((2 * B, H, W, 3), dtype=torch.uint8, device="cuda")
    for s in range(2 * B):
        d_frames[s].copy_(torch.from_numpy(mvo_synth.gray_to_bgr(frames[s % 16])))
    d_k = torch.empty(B * cap * 28, dtype=torch.uint8, device="cuda")
    d_d = torch.empty(B * cap * 32, dtype=torch.uint8, device="cuda")
    d_c = torch.empty(B, dtype=torch.int32, device="cuda")

    def call(first):
        ctx.orb_extract_batch_dev(d_frames[first].data_ptr(), B, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), cap)
    for _ in range(3):
        call(0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for it in range(10):
        call((it % 2) * B)
    e1.record(stream)
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 10
    names = mvo_b200.kernel_names()
    mvo_b200.timing_enable(ctx, (1 << len(names)) - 1)
    mvo_b200.timing_read(ctx)
    for it in range(2):
        call((it % 2) * B)
    ms, cnt = mvo_b200.timing_read(ctx)
    print(json.dumps({"config": {k: v for k, v in os.environ.items() if k in ("MVO_PYR_FUSED", "MVO_FAST_TMA", "MVO_GRID_ROUNDS", "MVO_PDL_ORB")}, "us_per_frame": us / B,
                      "frames_per_s": B / (us * 1e-6), "kernel_us_per_frame": {names[k]: round(1e3 * ms[k] / (2 * B), 3) for k in range(len(names)) if cnt[k]},
                      "checksum": int(d_d.to(torch.int64).sum().item())}))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "child":
        child()
    else:
        for cfg in CONFIGS:
            env = dict(os.environ)
            env.update(cfg)
            r = subprocess.run([sys.executable, __file__, "child"], env=env, capture_output=True, text=True)
            print(r.stdout.strip() or json.dumps({"config": cfg, "error": r.stderr[-600:]}), flush=True)
