"""mvo_vo_map_matches_batch_dev on the hardware.

- The fabricated scene of tests/map_matches_batch_cases.py at full size (cap 8192, and 2008 as the bench uses) for every method,
  byte for byte against the host reference (the state machine's projection restated, the library's mvo_match_features on the
  candidate arrays), with sentinels past every count.  The two sizes put the filter's dynamic shared memory on either side of the
  48 KB opt-in.
- A 65535-point map with few points in view; a map of more than 8192 visible matching points, which the job reports as
  MVO_ERR_UNSUPPORTED with its status alone written.
- Determinism and the launch count for 1, 63 and 500 jobs.
- The state machine end to end on the bench's room sequence: every tracked frame replayed through one extraction and one batch call
  per map version, with the reference keyframe's pose as the guess."""
import numpy as np
import pytest

import map_matches_batch_cases as cases

pytestmark = pytest.mark.gpu

H, W, KCAP = 480, 640, 2008


@pytest.fixture(scope="module")
def gctx(built):
    import mvo_b200
    c = mvo_b200.Context(0)
    yield c
    c.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _run(gctx, s, method, xy=True, pnp=True, **kw):
    """Device copies of the scene, one call, the outputs back on the host; also the launches the call made."""
    import torch
    host = cases.outputs(s.n_jobs, s.n_map, s.cap, xy=xy, pnp=pnp)
    keep = {id(a): _dev(a) for a in (s.kpts, s.desc, s.counts, s.frames, s.T, s.map_pts, s.map_desc) + tuple(h for h in host if h is not None)}
    torch.cuda.synchronize()
    l0 = gctx.kernel_launches
    rc, _ = cases.call(gctx.lib, gctx.h, s, method, ptr=lambda a: keep[id(a)].data_ptr(), outs=host, **kw)
    gctx._chk(rc)
    launches = gctx.kernel_launches - l0
    gctx.synchronize()
    got = tuple(None if h is None else keep[id(h)].cpu().numpy().view(h.dtype).reshape(h.shape) for h in host)
    return got, launches


@pytest.mark.parametrize("cap,n_map", [(8192, 3000), (2008, 2000)])
@pytest.mark.parametrize("method", [1, 2, 3])
def test_full_size_batch_equals_the_state_machine(gctx, cap, n_map, method):
    s = cases.Scene(cap, n_map=n_map, seed=cap + method)
    refs = [cases.reference(gctx.lib, gctx.h, s, j, method) for j in range(s.n_jobs)]
    cases.check_scene_coverage(gctx.lib, gctx.h, s, refs, method)
    got, launches = _run(gctx, s, method)
    assert launches == cases.launches(method)
    for j in range(s.n_jobs):
        cases.check_exact(refs[j], got, j, s.n_map, cap)
    got, _ = _run(gctx, s, method, xy=False, pnp=False)
    for j in range(s.n_jobs):
        cases.check_exact(refs[j], got, j, s.n_map, cap)


def test_large_map_few_in_view(gctx):
    s = cases.Scene(KCAP, n_map=400, seed=11)
    rng = np.random.default_rng(5)
    extra = 65535 - s.n_map                                          # far behind every guess
    X = np.stack([rng.uniform(-50, 50, extra), rng.uniform(-50, 50, extra), rng.uniform(-90, -20, extra)], 1).astype(np.float32)
    s.map_pts = np.ascontiguousarray(np.concatenate([s.map_pts, X]))
    s.map_desc = np.ascontiguousarray(np.concatenate([s.map_desc, rng.integers(0, 256, (extra, 32), dtype=np.uint8)]))
    s.n_map = 65535
    s = cases.with_jobs(s, [0, 1, 2, 3, 8, s.n_jobs - 1])
    for method in (1, 3):
        refs = [cases.reference(gctx.lib, gctx.h, s, j, method) for j in range(s.n_jobs)]
        assert 0 < refs[0][1]["n_candidates"] < 400 and refs[0][1]["n_matches"] > 20
        got, launches = _run(gctx, s, method)
        assert launches == cases.launches(method)
        for j in range(s.n_jobs):
            cases.check_exact(refs[j], got, j, s.n_map, s.cap)


def test_too_many_visible_matches_is_unsupported(gctx):
    """9000 map points in view, 8192 keypoints that are exact copies of 8192 of them: more matches pass the threshold than the
    filter holds.  The job reports MVO_ERR_UNSUPPORTED and writes nothing else; a job on an empty frame beside it is unaffected."""
    s = cases.Scene(8192, n_map=400, seed=2)
    rng = np.random.default_rng(9)
    n = 9000
    Xc = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 7, n)], 1).astype(np.float32)
    s.map_pts = Xc
    s.map_desc = np.ascontiguousarray(rng.integers(0, 256, (n, 32), dtype=np.uint8))
    s.n_map = n
    uv, _ = cases.project(np.eye(4), Xc.astype(np.float64))
    pick = rng.permutation(n)[:8192]
    rest = np.setdiff1d(np.arange(n), pick)
    s.map_desc[rest] = s.map_desc[pick[:len(rest)]]                 # every point in view has a keypoint at distance 0
    s.kpts = s.kpts.copy()
    s.desc = s.desc.copy()
    s.kpts[1]["x"], s.kpts[1]["y"] = uv[pick, 0], uv[pick, 1]
    s.desc[1] = s.map_desc[pick]
    s.counts = s.counts.copy()
    s.counts[1] = 8192
    s = cases.with_jobs(s, [1, 3])                                    # frame 1 under the identity guess; frame 2 (empty)
    ref = cases.reference(gctx.lib, gctx.h, s, 0, 1)
    assert ref[1]["n_candidates"] > 8192 and ref[1]["n_matches"] > 8000, ref[1]
    got, _ = _run(gctx, s, 1)
    cases.check_failed(got, 0, cases.UNSUPPORTED, s.n_map, s.cap)
    ref1 = cases.reference(gctx.lib, gctx.h, s, 1, 1)
    cases.check_exact(ref1, got, 1, s.n_map, s.cap)


@pytest.mark.parametrize("n_jobs", [1, 63, 500])
def test_determinism_and_launches(gctx, n_jobs):
    s = cases.Scene(KCAP, n_map=1500, seed=4)
    idx = np.arange(n_jobs) % 8                                       # the valid jobs, repeated
    t = cases.with_jobs(s, idx)
    for method in (1, 2, 3):
        a, la = _run(gctx, t, method)
        b, lb = _run(gctx, t, method)
        assert la == lb == cases.launches(method)
        for x, y in zip(a, b):
            assert x.tobytes() == y.tobytes()
        out = a[0]
        for j in range(n_jobs):                                      # a repeated job gives the same rows
            assert out[j].tobytes() == out[j % 8].tobytes()


def test_state_machine_tracking_end_to_end(built):
    """Every tracked frame of the state machine on the bench's room sequence (host-array mode: matches_with_map keeps the
    reference's DMatch), replayed through one extraction and one batch call per map version."""
    import torch
    import mvo_b200
    import mvo_synth
    frames, _ = mvo_synth.cached_room_loop_sequence(seed=0)
    imgs = [mvo_synth.gray_to_bgr(f) for f in frames]
    K = mvo_synth.K_DEFAULT

    def run(device_resident):
        ctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
        vo = mvo_b200.VisualOdometry(ctx, K, H, W, track={"device_resident": device_resident})
        ev, last_kf, added = [], None, 0
        for i, im in enumerate(imgs):
            before = None
            if vo.is_initialized() and last_kf is not None:
                ids, pts, desc, _ = vo.get_map()
                before = (ids, pts, desc, vo.frame_pose(added - 1 - last_kf))
            T, info = vo.add_frame(im)
            added += 1
            if info.state_in == 2 and before is not None:
                ev.append((i, info.n_candidates, info.n_matches, info.pnp_ok, vo.frame_data("matches_with_map", 0).copy(),
                           info.T_w_c_pnp[:], before))
            if info.keyframe:
                last_kf = info.frame_id
        vp = vo.params
        vo.close()
        ctx.close()
        return ev, vp

    ev, vp = run(0)
    assert len(ev) > 50, len(ev)
    method, radius = vp.track.match_method, vp.track.match_radius
    bctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    z = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device="cuda")  # noqa: E731
    NF = len(ev)
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack([imgs[e[0]] for e in ev]))).cuda()
    d_k, d_d, d_c = z(NF * KCAP * 28), z(NF * KCAP * 32), torch.zeros(NF, dtype=torch.int32, device="cuda")
    bctx.orb_extract_batch_dev(d_img.data_ptr(), NF, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), KCAP)
    groups = {}
    for f, e in enumerate(ev):                                       # one call per map version
        ids, pts, desc, _ = e[6]
        key = ids.tobytes() + pts.tobytes() + desc.tobytes()
        groups.setdefault(key, []).append(f)
    counts = {}
    for key, fs in groups.items():
        ids, pts, desc, _ = ev[fs[0]][6]
        n_map, n_jobs = len(ids), len(fs)
        d_map_p, d_map_d = _dev(np.ascontiguousarray(pts, np.float32)), _dev(np.ascontiguousarray(desc, np.uint8))
        d_fr = _dev(np.array(fs, np.int32))
        d_T = _dev(np.stack([ev[f][6][3] for f in fs]).astype(np.float64))
        d_o, d_cand = z(n_jobs * 16), z(max(n_jobs * n_map, 1) * 4)
        d_m, d_p3, d_p2 = z(n_jobs * KCAP * 16), z(n_jobs * KCAP * 12), z(n_jobs * KCAP * 8)
        bctx.vo_map_matches_batch_dev(d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), NF, KCAP, d_fr.data_ptr(), d_T.data_ptr(), n_jobs,
                                      d_map_p.data_ptr(), d_map_d.data_ptr(), n_map, K, H, W, method, radius, d_o.data_ptr(), d_cand.data_ptr(),
                                      d_m.data_ptr(), d_pts3d=d_p3.data_ptr(), d_pts2d=d_p2.data_ptr())
        bctx.synchronize()
        out = d_o.cpu().numpy().view(cases.OUT)
        cand = d_cand.cpu().numpy().view(np.int32)[: n_jobs * n_map].reshape(n_jobs, n_map)
        m = d_m.cpu().numpy().view(cases.DM).reshape(n_jobs, KCAP)
        p3 = d_p3.cpu().numpy().view(np.float32).reshape(n_jobs, KCAP, 3)
        for j, f in enumerate(fs):
            i, n_cand, n_match, pnp_ok, inl, T_pnp, _ = ev[f]
            o = out[j]
            assert o["status"] == 0 and o["n_candidates"] == n_cand and o["n_matches"] == n_match, (i, o, n_cand, n_match)
            counts[i] = (n_cand, n_match)
            if not pnp_ok:
                continue
            mine = m[j, :n_match]
            rows = {r.tobytes(): k for k, r in enumerate(mine)}
            Tcw = np.linalg.inv(np.asarray(T_pnp, np.float64).reshape(4, 4))
            for d in inl:
                assert d.tobytes() in rows, (i, d)
                mp = int(cand[j, d["query_idx"]])                     # the map point through d_cand
                assert p3[j, rows[d.tobytes()]].tobytes() == np.ascontiguousarray(pts[mp], np.float32).tobytes()
                Xc = Tcw[:3, :3] @ pts[mp].astype(np.float64) + Tcw[:3, 3]
                kp = d_k[(f * KCAP + d["train_idx"]) * 28:(f * KCAP + d["train_idx"] + 1) * 28].cpu().numpy().view(mvo_b200.KEYPOINT_DTYPE)[0]
                err = np.hypot(K[0, 0] * Xc[0] / Xc[2] + K[0, 2] - kp["x"], K[1, 1] * Xc[1] / Xc[2] + K[1, 2] - kp["y"])
                assert err < 4 * bctx.params.pnp_reproj_error, (i, err)          # the PnP inlier's own map point
    # the default device-resident run: its poses and map are its own and part ways with the host-array run's later in the
    # sequence, so its counts are held to the batch's on every frame before the first difference, which must be most of them
    ev_dev, _ = run(1)
    dev_counts = {e[0]: (e[1], e[2]) for e in ev_dev}
    agree = 0
    for i in sorted(counts):
        if dev_counts.get(i) != counts[i]:
            break
        agree += 1
    assert agree > 0.5 * len(counts), (agree, len(counts))
    print(f"{len(ev)} tracked frames replayed in {len(groups)} calls; the device-resident run agrees on the first {agree}")
    bctx.close()
