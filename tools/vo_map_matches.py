"""Map points in view and the 3D-2D matches of the tracked frames: the batched device call against the per-frame host composition,
on the bench sequence.

  vo      mvo_vo over the bench's room sequence (max_keypoints 2000, host-array mode) records, for every tracked frame, the map in
          container order before the frame and the reference keyframe's pose as it stood then.
  batch   one mvo_orb_extract_batch_dev over the tracked frames, then one mvo_vo_map_matches_batch_dev per map version.
  host    per frame: keypoints and descriptors downloaded, the map projected on the host (pose_estimation_pnp's arithmetic) and
          mvo_match_features on the candidates.
Timed with CUDA events after warm-up, alternating in the same run; every frame's match list is compared byte for byte between the
two paths in the same run (the run fails otherwise).  Reported: us per frame of both paths, launches per batch call, the card's
name and power limit read in the same run.  Needs a GPU.
Usage: python tools/vo_map_matches.py [--reps N] -> one JSON line."""
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
import map_matches_batch_cases as cases  # noqa: E402
from two_view_stream import card  # noqa: E402

H, W, CAP = 480, 640, 2008
K = mvo_synth.K_DEFAULT


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vo_map_matches: no CUDA device (this measurement has no CPU path)")
    imgs = [mvo_synth.gray_to_bgr(f) for f in mvo_synth.cached_room_loop_sequence(seed=0)[0]]
    vctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    vo = mvo_b200.VisualOdometry(vctx, K, H, W, track={"device_resident": 0})
    vp = vo.params
    ev, last_kf, added = [], None, 0
    for i, im in enumerate(imgs):
        before = None
        if vo.is_initialized() and last_kf is not None:
            ids, pts, desc, _ = vo.get_map()
            before = (pts.copy(), desc.copy(), vo.frame_pose(added - 1 - last_kf))
        _, info = vo.add_frame(im)
        added += 1
        if info.state_in == 2 and before is not None:
            ev.append((i, before))
        if info.keyframe:
            last_kf = info.frame_id
    vo.close()
    method, radius = vp.track.match_method, vp.track.match_radius
    NF = len(ev)
    ctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    z = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device="cuda")  # noqa: E731
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()  # noqa: E731
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack([imgs[e[0]] for e in ev]))).cuda()
    d_k, d_d, d_c = z(NF * CAP * 28), z(NF * CAP * 32), torch.zeros(NF, dtype=torch.int32, device="cuda")
    ctx.orb_extract_batch_dev(d_img.data_ptr(), NF, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), CAP)
    ctx.synchronize()
    groups = {}
    for f, (_, (pts, desc, _)) in enumerate(ev):
        groups.setdefault(pts.tobytes() + desc.tobytes(), []).append(f)
    calls = []
    for fs in groups.values():
        pts, desc, _ = ev[fs[0]][1]
        n_map, n_jobs = len(pts), len(fs)
        bufs = dict(p=dev(np.ascontiguousarray(pts, np.float32)), d=dev(desc), fr=dev(np.array(fs, np.int32)),
                    T=dev(np.stack([ev[f][1][2] for f in fs]).astype(np.float64)), o=z(n_jobs * 16), c=z(max(n_jobs * n_map, 1) * 4),
                    m=z(n_jobs * CAP * 16), p3=z(n_jobs * CAP * 12), p2=z(n_jobs * CAP * 8))
        calls.append((fs, n_map, bufs))

    def batch():
        for fs, n_map, b in calls:
            ctx.vo_map_matches_batch_dev(d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), NF, CAP, b["fr"].data_ptr(), b["T"].data_ptr(),
                                         len(fs), b["p"].data_ptr(), b["d"].data_ptr(), n_map, K, H, W, method, radius, b["o"].data_ptr(),
                                         b["c"].data_ptr(), b["m"].data_ptr(), d_pts3d=b["p3"].data_ptr(), d_pts2d=b["p2"].data_ptr())

    def host():                                                     # download, host projection, mvo_match_features, per frame
        res = {}
        for f, (_, (pts, desc, T)) in enumerate(ev):
            n = int(d_c[f].item())
            kp = d_k[f * CAP * 28:(f * CAP + n) * 28].cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE)
            dd = np.ascontiguousarray(d_d[f * CAP * 32:(f * CAP + n) * 32].cpu().numpy().reshape(n, 32))
            cand, cxy = cases.candidates(pts, T, K, H, W)
            if len(cand) == 0 or n == 0 or (method == 2 and n < 2):
                res[f] = np.zeros(0, mvo_b200.DMATCH_DTYPE)
                continue
            kxy = np.ascontiguousarray(np.stack([kp["x"], kp["y"]], 1), np.float32)
            res[f] = ctx.match_features(np.ascontiguousarray(desc[cand]), dd, method, cxy, kxy, radius)
        return res

    batch()
    ctx.synchronize()
    ref = host()
    for fs, n_map, b in calls:                                      # byte for byte in the same run
        out = b["o"].cpu().numpy().view(cases.OUT)
        m = b["m"].cpu().numpy().view(mvo_b200.DMATCH_DTYPE).reshape(len(fs), CAP)
        for j, f in enumerate(fs):
            assert out[j]["status"] == 0, (f, out[j])
            got, want = m[j, :out[j]["n_matches"]], np.ascontiguousarray(ref[f])
            if got.tobytes() != want.tobytes():
                bad = [k for k in range(min(len(got), len(want))) if got[k].tobytes() != want[k].tobytes()][:3]
                raise SystemExit(f"frame {f}: batch {out[j]} host {len(want)} matches; first differences "
                                 f"{[(got[k], want[k]) for k in bad]}")

    def ev_time(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        with torch.cuda.stream(stream):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3

    tb, th = [], []
    l0 = ctx.kernel_launches
    batch()
    ctx.synchronize()
    launches = (ctx.kernel_launches - l0) / len(calls)
    for _ in range(args.reps):
        tb.append(ev_time(batch))
        th.append(ev_time(host))
    print(json.dumps({"tool": "vo_map_matches", "frames": NF, "calls": len(calls), "method": method,
                      "batch_us_per_frame": float(np.median(tb)) / NF, "host_us_per_frame": float(np.median(th)) / NF,
                      "launches_per_call": launches, "identical": True, "card": card()}))


if __name__ == "__main__":
    main()
