"""The "ORB + match" stream of BASELINE config 2 at throughput: 64 frames of the bench sequence resident in HBM, extracted in one
mvo_orb_extract_batch_dev call (max_keypoints 2000), then the 63 consecutive pairs matched in one mvo_match_features_batch_dev
call, for each matchFeatures method.  CUDA events time the extraction batch, the match batch and both back to back after
warm-up; the kernel time of the two match kernels comes from the context's per-class events (class match_kernel).

Reported per method: us per frame, frames/s, algorithmic GB/s by SURVEY.md section 8d (ORB: 1,041,660 B per frame; match:
32 (N1 + N2) + 16 N1 B per pair, + 8 (N1 + N2) for method 3's keypoint coordinates) as a fraction of the 3.35 TB/s data-sheet
HBM figure, and for the Hamming methods the POPC rate (8 POPC.32 per descriptor pair, 3.2e7 per 2001 x 2001 pair) against
16 per clock per SM at the SM clock NVML reads after the timed loops.  The card's name and power limit are read in the same
run.  The timed outputs are then checked against per-pair mvo_match_features calls on host copies of the same frames; a
mismatch fails the run.  Needs a GPU.  Usage: python tools/orb_match_stream.py [--reps N] -> one JSON line."""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "monocular-visual-odometry_b200" / "python"))
import mvo_b200  # noqa: E402
import mvo_synth  # noqa: E402

B, H, W, CAP = 64, 480, 640, 2001
ORB_BYTES_PER_FRAME = 1_041_660          # SURVEY.md section 8d: BGR frame in, keypoints and descriptors out
HBM_PEAK_GBPS = 3350.0                   # H100 SXM data sheet, not measured
RADIUS = 100.0                           # method 3: max_matching_pixel_dist_in_initialization (config.yaml)


def card():
    out = {"name": None, "power_limit_w": None, "sm_mhz": None, "sm_max_mhz": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        name = pynvml.nvmlDeviceGetName(h)
        out["name"] = name.decode() if isinstance(name, bytes) else name
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        out["sm_mhz"] = pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
        out["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception as e:                                       # reported, not guessed
        out["nvml_error"] = repr(e)
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("orb_match_stream: no CUDA device (this measurement has no CPU path)")
    stream = torch.cuda.Stream()
    ctx = mvo_b200.Context(0, max_keypoints=2000)
    ctx.set_stream(stream.cuda_stream)
    names = mvo_b200.kernel_names()
    km = names.index("match_kernel")
    frames = mvo_synth.cached_room_loop_sequence(seed=0)[0][:B]
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack([mvo_synth.gray_to_bgr(f) for f in frames]))).cuda()
    d_k = torch.zeros(B * CAP * 28, dtype=torch.uint8, device="cuda")
    d_d = torch.zeros(B * CAP * 32, dtype=torch.uint8, device="cuda")
    d_c = torch.zeros(B, dtype=torch.int32, device="cuda")
    pairs = np.array([(i, i + 1) for i in range(B - 1)], np.int32)
    d_p = torch.from_numpy(pairs).cuda()
    d_out = torch.zeros(len(pairs) * CAP * 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(len(pairs), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def extract(_=0):
        ctx.orb_extract_batch_dev(d_img.data_ptr(), B, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), CAP)

    def match(method):
        ctx.match_features_batch_dev(d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), B, CAP, d_p.data_ptr(), len(pairs), method,
                                     RADIUS if method == 3 else 0.0, d_out.data_ptr(), d_n.data_ptr())

    def ev_time(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / reps                   # us per call

    for _ in range(3):
        extract()
    us_orb = ev_time(extract, args.reps)
    counts = d_c.cpu().numpy().astype(np.int64)
    n1, n2 = counts[pairs[:, 0]], counts[pairs[:, 1]]
    kp = d_k.cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE).reshape(B, CAP)
    desc = d_d.cpu().numpy().reshape(B, CAP, 32)
    orb = {"us_per_batch": us_orb, "us_per_frame": us_orb / B, "frames_per_s": B / (us_orb * 1e-6),
           "keypoints_per_frame": float(counts.mean()), "GBps": B * ORB_BYTES_PER_FRAME / (us_orb * 1e-6) / 1e9}
    orb["hbm_frac"] = orb["GBps"] / HBM_PEAK_GBPS

    res = {}
    for method in (1, 2, 3):
        for _ in range(3):
            match(method)
        us_m = ev_time(lambda: match(method), args.reps)
        us_both = ev_time(lambda: (extract(), match(method)), max(2, args.reps // 2))
        mvo_b200.timing_enable(ctx, 1 << km)
        mvo_b200.timing_read(ctx)
        for _ in range(args.reps):
            match(method)
        ms_k, cnt_k = mvo_b200.timing_read(ctx)
        mvo_b200.timing_enable(ctx, 0)
        us_k = 1e3 * ms_k[km] / args.reps                          # both match kernels of one call
        clk = card()
        mbytes = float(np.sum(32 * (n1 + n2) + 16 * n1 + (8 * (n1 + n2) if method == 3 else 0)))
        r = {"match_us_per_call": us_m, "match_kernel_us_per_call": us_k, "match_launches_per_call": int(cnt_k[km]) // args.reps,
             "match_us_per_pair": us_m / len(pairs), "match_pairs_per_s": len(pairs) / (us_m * 1e-6),
             "match_bytes_per_call": mbytes, "match_GBps": mbytes / (us_m * 1e-6) / 1e9,
             "both_us_per_batch": us_both, "both_us_per_frame": us_both / B, "both_frames_per_s": B / (us_both * 1e-6),
             "both_GBps": (B * ORB_BYTES_PER_FRAME + mbytes) / (us_both * 1e-6) / 1e9, "sm_mhz_after": clk["sm_mhz"]}
        r["match_hbm_frac"] = r["match_GBps"] / HBM_PEAK_GBPS
        r["both_hbm_frac"] = r["both_GBps"] / HBM_PEAK_GBPS
        if method in (1, 2) and clk["sm_mhz"]:
            popc = float(np.sum(8 * n1 * n2))
            peak = 16.0 * torch.cuda.get_device_properties(0).multi_processor_count * clk["sm_mhz"] * 1e6
            r["popc_per_call"] = popc
            r["popc_per_s_kernel"] = popc / (us_k * 1e-6)
            r["popc_frac_of_peak_kernel"] = popc / (us_k * 1e-6) / peak
        # the timed outputs against per-pair mvo_match_features on host copies of the same frames
        out = d_out.cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(len(pairs), CAP)
        n_out = d_n.cpu().numpy()
        bad = 0
        for p, (q, t) in enumerate(pairs):
            xy = lambda f: np.ascontiguousarray(np.stack([kp[f]["x"], kp[f]["y"]], 1)[: counts[f]], np.float32)  # noqa: E731
            ref = ctx.match_features(np.ascontiguousarray(desc[q, : counts[q]]), np.ascontiguousarray(desc[t, : counts[t]]), method,
                                     xy(q), xy(t), RADIUS if method == 3 else 0.0)
            bad += not (n_out[p] == len(ref) and out[p, : len(ref)].tobytes() == ref.tobytes())
        r["matches_per_pair"] = float(n_out.mean())
        r["pairs_differing_from_match_features"] = int(bad)
        res[f"method{method}"] = r

    line = {"tool": "orb_match_stream", "frames": B, "pairs": len(pairs), "cap": CAP, "max_keypoints": 2000, "card": card(),
            "hbm_peak_GBps": HBM_PEAK_GBPS, "hbm_peak_source": "H100 SXM data sheet, not measured", "radius_method3": RADIUS,
            "orb": orb, "match": res,
            "timing": "CUDA events on the context stream after 3 warm-up calls; match_kernel_us from per-class events in a separate loop"}
    print(json.dumps(line), flush=True)
    ctx.close()
    if any(r["pairs_differing_from_match_features"] for r in res.values()):
        raise SystemExit("orb_match_stream: batched matches differ from mvo_match_features")


if __name__ == "__main__":
    main()
