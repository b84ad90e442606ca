"""New map points of the keyframe insertions: the batched device chain against the per-pair host composition, on the bench sequence.

  vo      mvo_vo_run_sequence over the bench's room sequence (max_keypoints 2000) records every keyframe insertion: the reference
          keyframe, the new keyframe and the two poses insert_keyframe used.
  batch   one mvo_orb_extract_batch_dev over the frames involved, one mvo_match_features_batch_dev of the (reference keyframe,
          keyframe) pairs with track.match_method and max_match_dist_triangulation, one mvo_esti_motion_by_essential_batch_dev at
          vp.essential_threshold and one mvo_vo_keyframe_points_batch_dev: every insertion at once.
  host    per pair: the matches and keypoints downloaded, mvo_esti_motion_by_essential, mvo_do_triangulation with the known motion,
          transCoord and mvo_retain_good_triangulation, as insert_keyframe composes them.
Timed with CUDA events after warm-up, alternating in the same run; every pair's kept points are compared byte for byte between
the two paths in the same run (the run fails otherwise).  Reported: us per pair of both paths, launches per call of every batch
stage, the card's name and power limit read in the same run.  Needs a GPU.
Usage: python tools/vo_keyframe_points.py [--reps N] -> one JSON line."""
import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "monocular-visual-odometry_b200" / "python"))
sys.path.insert(0, str(ROOT / "tools"))
import mvo_b200  # noqa: E402
import mvo_synth  # noqa: E402
from two_view_stream import card  # noqa: E402

H, W, CAP = 480, 640, 2008
K = mvo_synth.K_DEFAULT


def trans_coord(p, R, t):
    return np.array([R[3 * r] * float(p[0]) + R[3 * r + 1] * float(p[1]) + R[3 * r + 2] * float(p[2]) + t[r] for r in range(3)]).astype(np.float32)


def known_motion(Tc, Tr):
    Ri = Tc[:3, :3].T
    ti = [-(Ri[i, 0] * Tc[0, 3] + Ri[i, 1] * Tc[1, 3] + Ri[i, 2] * Tc[2, 3]) for i in range(3)]
    Tci = [0.0] * 16
    for i in range(3):
        for j in range(3):
            Tci[i * 4 + j] = float(Ri[i, j])
        Tci[i * 4 + 3] = ti[i]
    Tci[15] = 1.0
    Trl = [float(x) for x in Tr.ravel()]
    T = [0.0] * 16
    for i in range(4):
        for j in range(4):
            a = 0.0
            for k in range(4):
                a += Tci[i * 4 + k] * Trl[k * 4 + j]
            T[i * 4 + j] = a
    return [T[i * 4 + j] for i in range(3) for j in range(3)], [T[i * 4 + 3] for i in range(3)]


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vo_keyframe_points: no CUDA device (this measurement has no CPU path)")
    stream = torch.cuda.Stream()
    frames = mvo_synth.cached_room_loop_sequence(seed=0)[0]
    imgs = [mvo_synth.gray_to_bgr(f) for f in frames]
    vctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    vo = mvo_b200.VisualOdometry(vctx, K, H, W)
    vp = vo.params
    ev, last_kf = [], None                                          # (ref id, frame id, T_ref, T_curr, kf_matches, kf_new_points)
    for im in imgs:
        T, info = vo.add_frame(im)
        if info.keyframe and info.state_in == 2:
            ev.append((last_kf, info.frame_id, vo.frame_pose(info.frame_id - last_kf), T.copy(), info.kf_matches, info.kf_new_points))
        if info.keyframe:
            last_kf = info.frame_id
    vo.close()
    n = len(ev)
    NF = 2 * n                                                      # every pair its own two slots: each with the pose of that insertion
    ctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10, essential_threshold=vp.essential_threshold)
    ctx.set_stream(stream.cuda_stream)
    z = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device="cuda")  # noqa: E731
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack([imgs[f] for e in ev for f in e[:2]]))).cuda()
    Ts = np.stack([T for e in ev for T in (e[2], e[3])])
    d_T = torch.from_numpy(Ts.reshape(-1).copy()).cuda()
    pairs = np.arange(NF, dtype=np.int32).reshape(-1, 2)
    d_p = torch.from_numpy(pairs.reshape(-1).copy()).cuda()
    d_k, d_d, d_c = z(NF * CAP * 28), z(NF * CAP * 32), torch.zeros(NF, dtype=torch.int32, device="cuda")
    d_m, d_n = z(n * CAP * 16), torch.zeros(n, dtype=torch.int32, device="cuda")
    d_e, d_i = z(n * mvo_b200.TWO_VIEW_RESULT_DTYPE.itemsize), z(n * CAP * 4)
    OUT = mvo_b200.KEYFRAME_POINTS_RESULT_DTYPE
    d_o, d_km, d_kp, d_ka = z(n * OUT.itemsize), z(n * CAP * 16), z(n * CAP * 12), z(n * CAP * 8)
    d_kw, d_kn = z(n * CAP * 12), z(n * CAP * 24)
    torch.cuda.synchronize()
    stages = {
        "extract": lambda: ctx.orb_extract_batch_dev(d_img.data_ptr(), NF, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(),
                                                     d_c.data_ptr(), CAP),
        "match": lambda: ctx.match_features_batch_dev(d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), NF, CAP, d_p.data_ptr(), n,
                                                      vp.track.match_method, vp.max_match_dist_triangulation, d_m.data_ptr(), d_n.data_ptr()),
        "essential": lambda: ctx.esti_motion_by_essential_batch_dev(d_k.data_ptr(), d_c.data_ptr(), NF, CAP, d_p.data_ptr(), n, d_m.data_ptr(),
                                                                    d_n.data_ptr(), K, vp.essential_threshold, d_e.data_ptr(), d_i.data_ptr()),
        "keyframe_points": lambda: ctx.vo_keyframe_points_batch_dev(d_k.data_ptr(), d_c.data_ptr(), NF, CAP, d_p.data_ptr(), n, d_m.data_ptr(),
                                                                    d_n.data_ptr(), d_e.data_ptr(), d_i.data_ptr(), d_T.data_ptr(), K, vp,
                                                                    d_o.data_ptr(), d_km.data_ptr(), d_kp.data_ptr(), d_ka.data_ptr(),
                                                                    d_kw.data_ptr(), d_kn.data_ptr()),
    }

    def batch():
        for fn in stages.values():
            fn()

    batch()
    ctx.synchronize()
    kpts = d_k.cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE).reshape(NF, CAP)
    matches = d_m.cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(n, CAP)
    nmatch = d_n.cpu().numpy()
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]

    def host():                                                     # insert_keyframe's composition, pair by pair
        res = []
        for p in range(n):
            q, tr = 2 * p, 2 * p + 1
            m = matches[p, :int(nmatch[p])]
            if len(m) < 8:
                res.append(None)
                continue
            p1 = np.ascontiguousarray(np.stack([kpts[q]["x"][m["query_idx"]], kpts[q]["y"][m["query_idx"]]], 1), np.float32)
            p2 = np.ascontiguousarray(np.stack([kpts[tr]["x"][m["train_idx"]], kpts[tr]["y"][m["train_idx"]]], 1), np.float32)
            try:
                _, _, _, inl = ctx.esti_motion_by_essential(p1, p2, K, vp.essential_threshold)
            except mvo_b200.MvoError:
                res.append(None)
                continue
            R, t = known_motion(Ts[tr], Ts[q])
            np1 = np.ascontiguousarray(((p1[inl].astype(np.float64) - [cx, cy]) / [fx, fy]).astype(np.float32))
            np2 = np.ascontiguousarray(((p2[inl].astype(np.float64) - [cx, cy]) / [fx, fy]).astype(np.float32))
            tri = ctx.do_triangulation(np1, np2, np.array(R).reshape(3, 3), np.array(t), np.arange(len(inl), dtype=np.int32))
            pts = np.ascontiguousarray(np.array([trans_coord(x, R, t) for x in tri], np.float32).reshape(-1, 3))
            Tc, Tr = np.ascontiguousarray(Ts[tr].ravel()), np.ascontiguousarray(Ts[q].ravel())
            keep, ang, nk = np.zeros(max(len(pts), 1), np.int32), np.zeros(max(len(pts), 1)), C.c_int(0)
            vctx.lib.mvo_retain_good_triangulation(pts.ctypes.data, len(pts), Tc.ctypes.data, Tr.ctypes.data, vp.min_triang_angle,
                                                   vp.max_ratio_angle_to_median, keep.ctypes.data, ang.ctypes.data, C.byref(nk))
            res.append(pts[keep[:nk.value]])
        return res

    def ev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3                            # us

    def host_time():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e6

    for _ in range(2):                                              # warm-up: module loads, scratch growth
        batch()
        host()
    ctx.synchronize()
    launches = {}
    for name, fn in stages.items():
        l0 = ctx.kernel_launches
        fn()
        launches[name] = int(ctx.kernel_launches - l0)
    t_batch, t_kf, t_host = [], [], []
    for _ in range(args.reps):                                      # alternating
        t_batch.append(ev_time(batch))
        t_kf.append(ev_time(stages["keyframe_points"]))
        t_host.append(host_time())
    ctx.synchronize()
    out = d_o.cpu().numpy().view(OUT)
    kp = d_kp.cpu().numpy().view(np.float32).reshape(n, CAP, 3)
    ref = host()
    identical = 0
    for p in range(n):
        if ref[p] is None:
            ok = out[p]["status"] == 0 and out[p]["usable"] == 0
        else:
            nk = int(out[p]["n_kept"])
            ok = out[p]["status"] == 0 and out[p]["usable"] == 1 and nk == len(ref[p]) and kp[p, :nk].tobytes() == ref[p].tobytes()
        identical += int(ok)
    sm_same = sum(int(out[p]["n_matches"] == ev[p][4] and out[p]["n_kept"] == ev[p][5]) for p in range(n))
    if identical != n:
        raise SystemExit(f"vo_keyframe_points: {n - identical} of {n} pairs differ between the batch and the host composition")
    med = lambda v: float(np.median(v))  # noqa: E731
    line = {"tool": "vo_keyframe_points", "frames": len(imgs), "pairs": n, "cap": CAP, "max_keypoints": 2000, "card": card(),
            "pairs_byte_identical": identical, "pairs_matching_state_machine_counts": sm_same,
            "batch_chain_us": med(t_batch), "batch_chain_us_per_pair": med(t_batch) / n,
            "keyframe_points_call_us": med(t_kf), "keyframe_points_us_per_pair": med(t_kf) / n,
            "host_composition_us": med(t_host), "host_composition_us_per_pair": med(t_host) / n, "launches_per_call": launches,
            "timing": f"batch: CUDA events on the context stream; host: wall clock around the per-pair composition (download, "
                      f"essential, triangulation, retain) with the device idle before and after; median of {args.reps} alternating "
                      "repetitions after 2 warm-up rounds"}
    print(json.dumps(line), flush=True)
    ctx.close()
    vctx.close()


if __name__ == "__main__":
    main()
