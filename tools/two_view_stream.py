"""Two-view motion for the matched frame pairs of a batch, on the device, against today's per-pair host path.

64 frames of the bench sequence resident in HBM are extracted in one mvo_orb_extract_batch_dev call (max_keypoints 2000), the
pairs (i, i+1) and (i, i+8) are matched in one mvo_match_features_batch_dev call with the initialisation's settings (method 1,
threshold 1.0), and the essential-matrix motion plus the triangulation of every pair's inliers runs as
  batch     one mvo_esti_motion_by_essential_batch_dev call on the device-resident keypoints and match lists;
  per pair  download of the counts, keypoints and match lists, then per pair pts1 / pts2 on the host, mvo_esti_motion_by_essential
            and mvo_do_triangulation (two synchronisations per pair).
and, with the homography branch and the E / H choice (what the reference's callers use), as
  rp batch     one mvo_estimate_relative_poses_batch_dev call (motion_cam2_to_cam1 = 1, triangulation of every solution);
  rp per pair  the same download, then mvo_estimate_relative_poses(calc_homo = 1) per pair.
Each pair of paths is timed with CUDA events on the context stream after warm-up, alternating in the same run.  Reported: us per
pair for every path, launches per batch call, the card's name and power limit read in the same run.  Every pair's result of a
batch call (status, E, R, t, inliers, triangulated points; for the relative poses the whole mvo_two_view_solutions record and
every solution's rows) is compared byte for byte with its per-pair path; a mismatch fails the run.
Needs a GPU.  Usage: python tools/two_view_stream.py [--reps N] -> one JSON line."""
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
K = mvo_synth.K_DEFAULT
THRESHOLD = 1.0                          # findEssentialMat_threshold (config.yaml)


def card():
    out = {"name": None, "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        name = pynvml.nvmlDeviceGetName(h)
        out["name"] = name.decode() if isinstance(name, bytes) else name
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception as e:                                       # reported, not guessed
        out["nvml_error"] = repr(e)
    return out


def per_pair(ctx, d_k, d_c, d_m, d_n, pairs):
    """Today's host path: one download of the batch's keypoints, counts and match lists, then two calls per pair.  Returns,
    per pair, (status, E, R, t, inliers, pts3d)."""
    counts = d_c.cpu().numpy()
    kp = d_k.cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE).reshape(B, CAP)
    matches = d_m.cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(len(pairs), CAP)
    n_m = d_n.cpu().numpy()
    out = []
    for p, (q, t) in enumerate(pairs):
        m = matches[p, :n_m[p]]
        p1 = np.ascontiguousarray(np.stack([kp[q]["x"][m["query_idx"]], kp[q]["y"][m["query_idx"]]], 1), np.float32)
        p2 = np.ascontiguousarray(np.stack([kp[t]["x"][m["train_idx"]], kp[t]["y"][m["train_idx"]]], 1), np.float32)
        try:
            E, R, tt, inl = ctx.esti_motion_by_essential(p1, p2, K, THRESHOLD)
        except mvo_b200.MvoError as e:
            out.append((e.code, None, None, None, None, None))
            continue
        norm = lambda a: np.stack([((a[:, 0].astype(np.float64) - K[0, 2]) / K[0, 0]).astype(np.float32),  # noqa: E731
                                   ((a[:, 1].astype(np.float64) - K[1, 2]) / K[1, 1]).astype(np.float32)], 1)
        pts = ctx.do_triangulation(norm(p1), norm(p2), R, tt, inl)
        out.append((0, E, R, tt, np.asarray(inl, np.int32), np.asarray(pts, np.float32)))
    assert counts.min() > 0
    return out


def per_pair_rp(ctx, d_k, d_c, d_m, d_n, pairs):
    """Today's host path for the relative poses: the same download, then mvo_estimate_relative_poses(calc_homo = 1) per pair.
    Returns, per pair, (status, the mvo_two_view_solutions bytes, inlier rows 5 x n, triangulated rows 5 x n x 3)."""
    import ctypes as C
    kp = d_k.cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE).reshape(B, CAP)
    matches = d_m.cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(len(pairs), CAP)
    n_m = d_n.cpu().numpy()
    Kc = np.ascontiguousarray(K, np.float64)
    out = []
    for p, (q, t) in enumerate(pairs):
        m = matches[p, :n_m[p]]
        n = len(m)
        p1 = np.ascontiguousarray(np.stack([kp[q]["x"][m["query_idx"]], kp[q]["y"][m["query_idx"]]], 1), np.float32)
        p2 = np.ascontiguousarray(np.stack([kp[t]["x"][m["train_idx"]], kp[t]["y"][m["train_idx"]]], 1), np.float32)
        sol = mvo_b200.TwoViewSolutions()
        inl = np.zeros((5, max(n, 1)), np.int32)
        pts = np.zeros((5, max(n, 1), 3), np.float32)
        rc = ctx.lib.mvo_estimate_relative_poses(ctx.h, p1.ctypes.data, p2.ctypes.data, n, Kc.ctypes.data, 1, 1, C.byref(sol),
                                                 inl.ctypes.data, pts.ctypes.data)
        out.append((rc, bytes(sol) if rc == 0 else None, inl, pts))
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("two_view_stream: no CUDA device (this measurement has no CPU path)")
    stream = torch.cuda.Stream()
    ctx = mvo_b200.Context(0, max_keypoints=2000)
    ctx.set_stream(stream.cuda_stream)
    frames = mvo_synth.cached_room_loop_sequence(seed=0)[0][:B]
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack([mvo_synth.gray_to_bgr(f) for f in frames]))).cuda()
    d_k = torch.zeros(B * CAP * 28, dtype=torch.uint8, device="cuda")
    d_d = torch.zeros(B * CAP * 32, dtype=torch.uint8, device="cuda")
    d_c = torch.zeros(B, dtype=torch.int32, device="cuda")
    pairs = np.array([(i, i + 1) for i in range(B - 1)] + [(i, i + 8) for i in range(B - 8)], np.int32)
    n = len(pairs)
    d_p = torch.from_numpy(pairs).cuda()
    d_m = torch.zeros(n * CAP * 16, dtype=torch.uint8, device="cuda")
    d_n = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_res = torch.zeros(n * mvo_b200.TWO_VIEW_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    d_inl = torch.zeros(n * CAP, dtype=torch.int32, device="cuda")
    d_pts = torch.zeros(n * CAP * 3, dtype=torch.float32, device="cuda")
    d_res2 = torch.zeros(n * mvo_b200.RELATIVE_POSES_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    d_inl2 = torch.zeros(n * 5 * CAP, dtype=torch.int32, device="cuda")
    d_pts2 = torch.zeros(n * 5 * CAP * 3, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.orb_extract_batch_dev(d_img.data_ptr(), B, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), CAP)
    ctx.match_features_batch_dev(d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), B, CAP, d_p.data_ptr(), n, 1, 0.0, d_m.data_ptr(),
                                 d_n.data_ptr())
    ctx.synchronize()

    def batch():
        ctx.esti_motion_by_essential_batch_dev(d_k.data_ptr(), d_c.data_ptr(), B, CAP, d_p.data_ptr(), n, d_m.data_ptr(), d_n.data_ptr(), K,
                                               THRESHOLD, d_res.data_ptr(), d_inl.data_ptr(), d_pts.data_ptr())

    def batch_rp():
        ctx.estimate_relative_poses_batch_dev(d_k.data_ptr(), d_c.data_ptr(), B, CAP, d_p.data_ptr(), n, d_m.data_ptr(), d_n.data_ptr(), K,
                                              d_res2.data_ptr(), d_inl2.data_ptr(), d_pts2.data_ptr(), motion_cam2_to_cam1=True)

    def ev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        r = fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3, r                        # us

    for _ in range(2):                                             # warm-up: module loads, scratch growth
        batch()
        ref = per_pair(ctx, d_k, d_c, d_m, d_n, pairs)
        batch_rp()
        ref_rp = per_pair_rp(ctx, d_k, d_c, d_m, d_n, pairs)
    ctx.synchronize()
    l0 = ctx.lib.mvo_kernel_launches(ctx.h)
    batch()
    launches = int(ctx.lib.mvo_kernel_launches(ctx.h) - l0)
    l0 = ctx.lib.mvo_kernel_launches(ctx.h)
    batch_rp()
    launches_rp = int(ctx.lib.mvo_kernel_launches(ctx.h) - l0)
    t_batch, t_host, t_batch_rp, t_host_rp = [], [], [], []
    for _ in range(args.reps):                                     # alternating
        us, _ = ev_time(batch)
        t_batch.append(us)
        us, ref = ev_time(lambda: per_pair(ctx, d_k, d_c, d_m, d_n, pairs))
        t_host.append(us)
        us, _ = ev_time(batch_rp)
        t_batch_rp.append(us)
        us, ref_rp = ev_time(lambda: per_pair_rp(ctx, d_k, d_c, d_m, d_n, pairs))
        t_host_rp.append(us)

    res = d_res.cpu().numpy().view(mvo_b200.TWO_VIEW_RESULT_DTYPE)
    inl = d_inl.cpu().numpy().reshape(n, CAP)
    pts = d_pts.cpu().numpy().reshape(n, CAP, 3)
    bad = []
    for p, (rc, E, R, t, il, pt) in enumerate(ref):
        r = res[p]
        if rc != 0:
            ok = r["status"] == rc
        else:
            ni = len(il)
            ok = (r["status"] == 0 and r["n_inliers"] == ni and r["E"].tobytes() == np.asarray(E, np.float64).tobytes()
                  and r["R"].tobytes() == np.asarray(R, np.float64).tobytes() and r["t"].tobytes() == np.asarray(t, np.float64).tobytes()
                  and inl[p, :ni].tobytes() == il.tobytes() and pts[p, :ni].tobytes() == pt.tobytes())
        if not ok:
            bad.append(p)
    res2 = d_res2.cpu().numpy().view(mvo_b200.RELATIVE_POSES_RESULT_DTYPE)
    inl2 = d_inl2.cpu().numpy().reshape(n, 5, CAP)
    pts2 = d_pts2.cpu().numpy().reshape(n, 5, CAP, 3)
    bad_rp = []
    for p, (rc, sol, il, pt) in enumerate(ref_rp):
        r = res2[p]
        ok = r["status"] == rc and r["n_matches"] == d_n[p].item()
        if ok and rc == 0:
            ok = r.tobytes()[8:] == sol
            for s_ in range(int(r["num_solutions"])):
                ni = int(r["n_inliers"][s_])
                ok = ok and inl2[p, s_, :ni].tobytes() == il[s_, :ni].tobytes() and pts2[p, s_, :ni].tobytes() == pt[s_, :ni].tobytes()
        if not ok:
            bad_rp.append(p)
    okp = res2["status"] == 0
    med = lambda v: float(np.median(v))  # noqa: E731
    line = {"tool": "two_view_stream", "frames": B, "pairs": n, "pair_kinds": "(i, i+1) and (i, i+8)", "cap": CAP, "max_keypoints": 2000,
            "match_method": 1, "threshold_px": THRESHOLD, "epi_hypotheses": int(ctx.params.epi_hypotheses), "card": card(),
            "matches_per_pair": float(d_n.cpu().numpy().mean()), "pairs_ok": int((res["status"] == 0).sum()),
            "inliers_per_ok_pair": float(res["n_inliers"][res["status"] == 0].mean()),
            "batch_us_per_call": med(t_batch), "batch_us_per_pair": med(t_batch) / n, "batch_launches_per_call": launches,
            "per_pair_host_us_per_call": med(t_host), "per_pair_host_us_per_pair": med(t_host) / n,
            "speedup": med(t_host) / med(t_batch), "pairs_differing_from_per_pair_path": len(bad),
            "rp_homography_threshold_px": float(ctx.params.homography_threshold), "rp_eh_ratio_threshold": float(ctx.params.eh_ratio_threshold),
            "rp_pairs_ok": int(okp.sum()), "rp_pairs_h_chosen": int((res2["best"][okp] > 0).sum()),
            "rp_homography_solutions_per_ok_pair": float((res2["num_solutions"][okp] - 1).mean()),
            "rp_batch_us_per_call": med(t_batch_rp), "rp_batch_us_per_pair": med(t_batch_rp) / n, "rp_batch_launches_per_call": launches_rp,
            "rp_per_pair_host_us_per_call": med(t_host_rp), "rp_per_pair_host_us_per_pair": med(t_host_rp) / n,
            "rp_speedup": med(t_host_rp) / med(t_batch_rp), "rp_pairs_differing_from_per_pair_path": len(bad_rp),
            "timing": f"CUDA events on the context stream, median of {args.reps} alternating repetitions after 2 warm-up rounds"}
    print(json.dumps(line), flush=True)
    ctx.close()
    if bad or bad_rp:
        raise SystemExit(f"two_view_stream: batch results differ from the per-pair path for pairs {bad[:10]} (essential), "
                         f"{bad_rp[:10]} (relative poses)")


if __name__ == "__main__":
    main()
