"""RANSAC PnP and the pose decision of the tracked frames: the batched device call against the per-frame host composition, on the
bench sequence.

  vo      mvo_vo over the bench's room sequence (max_keypoints 2000, host-array mode) records, for every tracked frame, the map
          before it, the reference keyframe's pose and the previous frame's pose (tests/vo_pnp_batch_cases.py: record_tracking).
  rows    one mvo_orb_extract_batch_dev over the tracked frames, one mvo_vo_map_matches_batch_dev per map version (not timed).
  batch   one mvo_vo_pnp_batch_dev per map version.
  host    per frame: the job's record and 3D-2D pairs downloaded, then mvo_solve_pnp_ransac on them.
Timed with CUDA events after warm-up, alternating in the same run; the replay's outcome is checked against the state machine first
(check_replay: the run fails otherwise).  Reported: us per frame of both paths, the card's name and power limit read in the same
run.  Needs a GPU.
Usage: python tools/vo_pnp_batch.py [--reps N] -> one JSON line."""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "monocular-visual-odometry_b200" / "python"))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))
import mvo_b200  # noqa: E402
import mvo_synth  # noqa: E402
import vo_pnp_batch_cases as cases  # noqa: E402
from two_view_stream import card  # noqa: E402


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vo_pnp_batch: no CUDA device (this measurement has no CPU path)")
    imgs = [mvo_synth.gray_to_bgr(f) for f in mvo_synth.cached_room_loop_sequence(seed=0)[0]]
    ev, vp = cases.record_tracking(imgs, mvo_synth.K_DEFAULT)
    ctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    rp = cases.Replay(ctx, ev, imgs, vp, mvo_synth.K_DEFAULT)
    worst = cases.check_replay(rp)
    NF = len(ev)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)

    def batch():
        for g in rp.groups:
            rp.pnp(g)

    def host():
        for g in rp.groups:
            for j in range(g["n_jobs"]):
                rp.host_pnp(g, j)

    l0 = ctx.kernel_launches
    batch()
    ctx.synchronize()
    launches = ctx.kernel_launches - l0
    host()
    t_b, t_h = [], []
    for _ in range(args.reps):
        for fn, acc in ((batch, t_b), (host, t_h)):
            ctx.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            with torch.cuda.stream(stream):
                fn()
            e1.record(stream)
            ctx.synchronize()
            e1.synchronize()
            acc.append(e0.elapsed_time(e1) * 1e3 / NF)
    res = {"tool": "vo_pnp_batch", "frames": NF, "calls": len(rp.groups), "launches_per_pass": launches,
           "batch_us_per_frame_median": float(np.median(t_b)), "host_us_per_frame_median": float(np.median(t_h)),
           "batch_us_per_frame": [round(x, 2) for x in t_b], "host_us_per_frame": [round(x, 2) for x in t_h],
           "max_T_w_c_pnp_diff": worst, "card": card(),
           "timing": "CUDA events on the context stream around all PnP calls of the replay (batch) / all per-frame downloads and "
                     "mvo_solve_pnp_ransac calls (host), divided by the tracked frames"}
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
