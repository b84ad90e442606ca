"""Finding the initialisation pair: the batched device chain against the state machine, on the first 32 frames of the bench sequence.

  batch   one mvo_orb_extract_batch_dev over the 32 frames (resident in HBM), one mvo_match_features_batch_dev of the pairs (0, k)
          for k = 1..31 with the initialisation's settings (match_method_init, max_match_dist_init), one
          mvo_estimate_relative_poses_batch_dev (motion_cam2_to_cam1 = 1, triangulation) and one mvo_vo_init_candidates_batch_dev:
          every candidate checked at once; the first pair with good = 1 is the pick.
  vo      mvo_vo_run_sequence from a BLANK state over the same frames (host images, as run_vo.cpp hands them over) up to the one it
          initialises on: one candidate after the other, each with its host round trips.
Both paths run on one context stream with the bench's parameters (max_keypoints 2000, the state machine's findEssentialMat threshold
for the batch), timed with CUDA events after warm-up, alternating in the same run.  The run fails unless both pick the same frame.
Reported: us per candidate pair of each path (batch: 31 candidates; vo: the candidates it examined), launches per call of every
batch stage, the card's name and power limit read in the same run.  Needs a GPU.
Usage: python tools/vo_init_search.py [--reps N] -> one JSON line."""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "monocular-visual-odometry_b200" / "python"))
sys.path.insert(0, str(ROOT / "tools"))
import mvo_b200  # noqa: E402
import mvo_synth  # noqa: E402
from two_view_stream import card  # noqa: E402

NF, H, W, CAP = 32, 480, 640, 2008
K = mvo_synth.K_DEFAULT


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vo_init_search: no CUDA device (this measurement has no CPU path)")
    stream = torch.cuda.Stream()
    frames = mvo_synth.cached_room_loop_sequence(seed=0)[0][:NF]
    imgs = [mvo_synth.gray_to_bgr(f) for f in frames]
    vctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    vctx.set_stream(stream.cuda_stream)
    vo = mvo_b200.VisualOdometry(vctx, K, H, W)
    vp = vo.params
    ctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10, essential_threshold=vp.essential_threshold)
    ctx.set_stream(stream.cuda_stream)
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack(imgs))).cuda()
    pairs = np.array([(0, k) for k in range(1, NF)], np.int32)
    n = len(pairs)
    z = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device="cuda")  # noqa: E731
    d_k, d_d, d_c = z(NF * CAP * 28), z(NF * CAP * 32), torch.zeros(NF, dtype=torch.int32, device="cuda")
    d_p = torch.from_numpy(pairs.reshape(-1)).cuda()
    d_m, d_n = z(n * CAP * 16), torch.zeros(n, dtype=torch.int32, device="cuda")
    d_rp, d_ri, d_rx = z(n * mvo_b200.RELATIVE_POSES_RESULT_DTYPE.itemsize), z(n * 5 * CAP * 4), z(n * 5 * CAP * 12)
    d_o, d_km, d_kp, d_ka = z(n * mvo_b200.INIT_CANDIDATE_RESULT_DTYPE.itemsize), z(n * CAP * 16), z(n * CAP * 12), z(n * CAP * 8)
    T_ref = np.eye(4)                                               # the first keyframe's pose (BLANK -> identity)
    torch.cuda.synchronize()
    stages = {
        "extract": lambda: ctx.orb_extract_batch_dev(d_img.data_ptr(), NF, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(),
                                                     d_c.data_ptr(), CAP),
        "match": lambda: ctx.match_features_batch_dev(d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), NF, CAP, d_p.data_ptr(), n,
                                                      vp.match_method_init, vp.max_match_dist_init, d_m.data_ptr(), d_n.data_ptr()),
        "relative_poses": lambda: ctx.estimate_relative_poses_batch_dev(d_k.data_ptr(), d_c.data_ptr(), NF, CAP, d_p.data_ptr(), n,
                                                                        d_m.data_ptr(), d_n.data_ptr(), K, d_rp.data_ptr(), d_ri.data_ptr(),
                                                                        d_rx.data_ptr(), motion_cam2_to_cam1=True),
        "init_candidates": lambda: ctx.vo_init_candidates_batch_dev(d_k.data_ptr(), d_c.data_ptr(), NF, CAP, d_p.data_ptr(), n,
                                                                    d_m.data_ptr(), d_n.data_ptr(), d_rp.data_ptr(), d_ri.data_ptr(),
                                                                    d_rx.data_ptr(), T_ref, vp, d_o.data_ptr(), d_km.data_ptr(),
                                                                    d_kp.data_ptr(), d_ka.data_ptr()),
    }

    def batch():
        for fn in stages.values():
            fn()

    vo.reset()                                                      # the frame it initialises on, frame by frame
    k_vo = None
    for k in range(NF):
        _, infos = vo.run_sequence(imgs[k:k + 1])
        if infos[0].state_in == 1 and infos[0].state_out == 2:
            k_vo = k
            break
    if k_vo is None:
        raise SystemExit(f"vo_init_search: the state machine did not initialise within {NF} frames")

    def run_vo():                                                   # run_vo.cpp's loop over the frames up to that one
        vo.reset()
        _, infos = vo.run_sequence(imgs[:k_vo + 1])
        assert infos[k_vo].state_out == 2 and all(i.state_out != 2 for i in infos[:k_vo])

    def ev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3                            # us

    for _ in range(2):                                              # warm-up: module loads, scratch growth
        batch()
        run_vo()
    ctx.synchronize()
    launches = {}
    for name, fn in stages.items():
        l0 = ctx.kernel_launches
        fn()
        launches[name] = int(ctx.kernel_launches - l0)
    t_batch, t_init, t_vo = [], [], []
    for _ in range(args.reps):                                      # alternating
        t_batch.append(ev_time(batch))
        t_init.append(ev_time(stages["init_candidates"]))
        t_vo.append(ev_time(run_vo))
    out = d_o.cpu().numpy().view(mvo_b200.INIT_CANDIDATE_RESULT_DTYPE)
    good = [int(pairs[p][1]) for p in range(n) if out[p]["status"] == 0 and out[p]["good"]]
    k_batch = good[0] if good else None
    if k_batch != k_vo:
        raise SystemExit(f"vo_init_search: the batch picks frame {k_batch}, the state machine initialised on frame {k_vo}")
    med = lambda v: float(np.median(v))  # noqa: E731
    line = {"tool": "vo_init_search", "frames": NF, "candidates": n, "cap": CAP, "max_keypoints": 2000, "card": card(),
            "init_frame": k_vo, "candidates_examined_by_vo": k_vo, "good_candidates": good,
            "batch_chain_us": med(t_batch), "batch_chain_us_per_candidate": med(t_batch) / n,
            "init_candidates_call_us": med(t_init), "init_candidates_us_per_candidate": med(t_init) / n, "launches_per_call": launches,
            "vo_us_until_initialised": med(t_vo), "vo_us_per_candidate": med(t_vo) / k_vo,
            "timing": f"CUDA events on the shared context stream, median of {args.reps} alternating repetitions after 2 warm-up rounds; "
                      "vo includes the first keyframe's frame"}
    print(json.dumps(line), flush=True)
    vo.close()
    ctx.close()
    vctx.close()


if __name__ == "__main__":
    main()
