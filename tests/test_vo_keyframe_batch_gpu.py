"""mvo_vo_keyframe_points_batch_dev on the hardware.

- The fabricated batches of tests/vo_keyframe_batch_cases.py at full size (n = cap = 6400) and at the caps around the point where
  the last kernel's static and dynamic shared memory together cross 48 KB, against the host reference: every kept angle and
  median_angle within 4 ulp of the host's (the device's acos is not glibc's), float rows NaN where the host's are, every other byte
  identical.  A pair counts only if no angle lies within 4 ulp of a decision boundary (16 ulp for the angle / median quotient), and
  the test asserts that margin for every pair it counts; the largest angle difference is reported.
- Determinism and three launches for 1 / 63 / 500 pairs.
- The state machine end to end on the bench's room sequence: every keyframe insertion replayed through the batch chain."""
import ctypes as C

import numpy as np
import pytest

import vo_keyframe_batch_cases as cases

pytestmark = pytest.mark.gpu

CAP = 6400
MAX_ULP = [0]


@pytest.fixture(scope="module")
def gctx(built):
    import mvo_b200
    c = mvo_b200.Context(0)
    yield c
    c.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _run(gctx, b, vp, n_pairs=None):
    """Device copies of the batch, one call, the outputs back on the host; also the launches the call made."""
    import torch
    host = cases.outputs(b.n_pairs, b.cap)
    keep = {id(a): _dev(a) for a in (b.kpts, b.counts, b.pairs, b.matches, b.n_matches, b.ess, b.inl, b.T) + host}
    torch.cuda.synchronize()
    l0 = gctx.kernel_launches
    rc, _ = cases.call(gctx.lib, gctx.h, b, vp, ptr=lambda a: keep[id(a)].data_ptr(), outs=host, n_pairs=n_pairs)
    gctx._chk(rc)
    launches = gctx.kernel_launches - l0
    gctx.synchronize()
    got = tuple(keep[id(h)].cpu().numpy().view(h.dtype).reshape(h.shape) for h in host)
    return got, launches


def _same_floats(d, h, p, what):
    d, h = np.asarray(d).reshape(-1), np.asarray(h).reshape(-1)
    nan = np.isnan(h)
    assert (np.isnan(d) == nan).all() and d[~nan].tobytes() == h[~nan].tobytes(), (p, what)


def check_bounded(gctx, b, p, vp, ref, got):
    """The GPU tier's promise for one pair; returns the reasons the pair is not held to it (empty: it was checked)."""
    out, kept, kpts, kang, kw, kn = got
    st, rec, km, kp, ka, hw, hn = ref
    if rec is None:
        cases.check_failed(got, p, st)
        return []
    if rec["usable"] and rec["n_inliers"] > 0:
        ang, med = cases.all_angles(gctx.lib, gctx.h, b, p)
        reasons = cases.vi.margin_failures(ang, med, vp, np.nan)
        if reasons:
            return reasons
    g = out[p]
    for f in cases.OUT.names:
        if f == "median_angle":
            d = cases.vi.ulp_diff(g[f], rec[f])
            assert d <= 4, (p, g[f], rec[f])
            MAX_ULP[0] = max(MAX_ULP[0], int(d))
        else:
            assert np.asarray(g[f]).tobytes() == np.asarray(rec[f]).tobytes(), (p, f, g[f], rec[f])
    nk = int(rec["n_kept"])
    assert kept[p, :nk].tobytes() == km.tobytes(), p
    _same_floats(kpts[p, :nk], kp, p, "points")
    _same_floats(kw[p, :nk], hw, p, "world")
    _same_floats(kn[p, :nk], hn, p, "norm")
    if nk:
        d = cases.vi.ulp_diff(kang[p, :nk], ka)
        assert max(d) <= 4, (p, max(d))
        MAX_ULP[0] = max(MAX_ULP[0], int(max(d)))
    cases.check_untouched_past(got, p, nk, int(rec["n_inliers"]) if rec["usable"] else 0)
    return []


# cap 6400 is the limit; the last kernel's rows need 20 B per entry beside its 1472 B of static shared memory: 2384 still fits in
# 48 KB together, 2385 does not (the launch has to opt in), and 2457 is the last cap whose rows alone fit
@pytest.mark.parametrize("cap,seed", [(CAP, 11), (2384, 12), (2385, 12), (2457, 13)])
def test_batch_equals_the_state_machine_within_the_acos_bound(gctx, cap, seed):
    b = cases.Batch(cases.mixed_specs(cap), cap, seed=seed)
    vp = cases.vi.vo_params(gctx.lib)
    got, launches = _run(gctx, b, vp)
    assert launches == cases.LAUNCHES
    not_held = {}
    for p in range(b.n_pairs):
        reasons = check_bounded(gctx, b, p, vp, cases.reference(gctx.lib, gctx.h, b, p, vp), got)
        if reasons:
            not_held[p] = reasons
    assert not not_held, not_held
    print(f"cap {cap}: largest angle difference so far {MAX_ULP[0]} ulp, every pair checked")


def test_deterministic_and_three_launches(gctx):
    specs = [cases.mixed_specs(400)[i % 16] for i in range(500)]
    specs = [s if "of" not in s else dict(n=80) for s in specs]
    b = cases.Batch(specs, 400, seed=2)
    vp = cases.vi.vo_params(gctx.lib)
    first, l1 = _run(gctx, b, vp)
    again, l2 = _run(gctx, b, vp)
    for x, y in zip(first, again):
        assert x.tobytes() == y.tobytes()
    counts = {l1, l2}
    for n_pairs in (1, 63):
        sub, n = _run(gctx, b, vp, n_pairs=n_pairs)
        counts.add(n)
        assert sub[0][:n_pairs].tobytes() == first[0][:n_pairs].tobytes()
    assert counts == {cases.LAUNCHES}


def test_call_level_limits(gctx):
    import torch
    lib, h = gctx.lib, gctx.h
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    a = buf.data_ptr()
    K = np.ascontiguousarray(cases.K, np.float64)
    vp0 = cases.vi.vo_params(lib)

    def call(kpts=a, counts=a, batch=2, cap=100, pairs=a, n_pairs=1, matches=a, n_matches=a, ess=a, inl=a, T=a, Kp=K.ctypes.data, vp=vp0,
             out=a, kept=a, kpts3=a, kang=a, kw=None, kn=None):
        return lib.mvo_vo_keyframe_points_batch_dev(h, kpts, counts, batch, cap, pairs, n_pairs, matches, n_matches, ess, inl, T, Kp,
                                                    None if vp is None else C.byref(vp), out, kept, kpts3, kang, kw, kn)

    for kw in ("kpts", "counts", "pairs", "matches", "n_matches", "ess", "inl", "T", "Kp", "vp", "out", "kept", "kpts3", "kang"):
        assert call(**{kw: None}) == cases.INVALID_ARG, kw
    assert call(vp=cases.vi.vo_params(lib, min_triang_angle=np.inf)) == cases.INVALID_ARG
    assert call(n_pairs=-1) == cases.INVALID_ARG and call(batch=0) == cases.INVALID_ARG and call(cap=0) == cases.INVALID_ARG
    UNSUPPORTED = -5
    assert call(cap=6401) == UNSUPPORTED and call(n_pairs=65536) == UNSUPPORTED
    l0 = lib.mvo_kernel_launches(h)
    assert call(cap=6400, n_pairs=0) == 0 and lib.mvo_kernel_launches(h) == l0
    gctx.synchronize()


H, W, KCAP = 480, 640, 2008


def test_state_machine_keyframes_end_to_end(built):
    """Every keyframe insertion of the state machine on the bench's room sequence, replayed through extract -> match -> essential
    -> keyframe points with the poses the insertion used."""
    import torch
    import mvo_b200
    import mvo_synth
    frames, _ = mvo_synth.cached_room_loop_sequence(seed=0)
    imgs = [mvo_synth.gray_to_bgr(f) for f in frames]
    K = mvo_synth.K_DEFAULT
    ctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10)
    vo = mvo_b200.VisualOdometry(ctx, K, H, W)
    vp = vo.params
    ev = []                                   # (ref id, frame id, kf_matches, kf_new_points, points, T_ref, T_curr, new map points)
    last_kf, known = None, set()
    for i, im in enumerate(imgs):
        T, info = vo.add_frame(im)
        if info.keyframe and info.state_in == 2:
            k = info.frame_id - last_kf
            assert 0 < k < 20, (i, k)                                 # the reference keyframe is still in the frame buffer
            ids, pts, _, _ = vo.get_map()
            new = [(int(x), p) for x, p in zip(ids, pts) if int(x) not in known]
            ev.append((last_kf, info.frame_id, info.kf_matches, info.kf_new_points, vo.frame_data("inliers_pts3d", 0), vo.frame_pose(k),
                       T.copy(), new))
        if info.keyframe:
            last_kf = info.frame_id
        known |= {int(x) for x in vo.get_map()[0]}
    vo.close()
    assert len(ev) >= 3, len(ev)
    n = len(ev)
    NF = 2 * n                                # every pair its own two slots: a keyframe's pose moves between its insertions
    bctx = mvo_b200.Context(0, max_keypoints=2000, ba_iterations=10, essential_threshold=vp.essential_threshold)
    z = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device="cuda")  # noqa: E731
    d_img = torch.from_numpy(np.ascontiguousarray(np.stack([imgs[f] for e in ev for f in e[:2]]))).cuda()
    d_k, d_d, d_c = z(NF * KCAP * 28), z(NF * KCAP * 32), torch.zeros(NF, dtype=torch.int32, device="cuda")
    pairs = np.arange(NF, dtype=np.int32).reshape(-1, 2)
    Ts = np.stack([T for e in ev for T in (e[5], e[6])])
    d_T = torch.from_numpy(Ts.reshape(-1).copy()).cuda()
    d_p = torch.from_numpy(pairs.reshape(-1).copy()).cuda()
    d_m, d_n = z(n * KCAP * 16), torch.zeros(n, dtype=torch.int32, device="cuda")
    d_e, d_i = z(n * cases.ESS.itemsize), z(n * KCAP * 4)
    d_o, d_km, d_kp, d_ka = z(n * cases.OUT.itemsize), z(n * KCAP * 16), z(n * KCAP * 12), z(n * KCAP * 8)
    d_kw, d_kn = z(n * KCAP * 12), z(n * KCAP * 24)
    torch.cuda.synchronize()
    bctx.orb_extract_batch_dev(d_img.data_ptr(), NF, H, W, 3, W * 3, H * W * 3, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), KCAP)
    bctx.match_features_batch_dev(d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), NF, KCAP, d_p.data_ptr(), n, vp.track.match_method,
                                  vp.max_match_dist_triangulation, d_m.data_ptr(), d_n.data_ptr())
    bctx.esti_motion_by_essential_batch_dev(d_k.data_ptr(), d_c.data_ptr(), NF, KCAP, d_p.data_ptr(), n, d_m.data_ptr(), d_n.data_ptr(), K,
                                            vp.essential_threshold, d_e.data_ptr(), d_i.data_ptr())
    bctx.vo_keyframe_points_batch_dev(d_k.data_ptr(), d_c.data_ptr(), NF, KCAP, d_p.data_ptr(), n, d_m.data_ptr(), d_n.data_ptr(),
                                      d_e.data_ptr(), d_i.data_ptr(), d_T.data_ptr(), K, vp, d_o.data_ptr(), d_km.data_ptr(), d_kp.data_ptr(),
                                      d_ka.data_ptr(), d_kw.data_ptr(), d_kn.data_ptr())
    bctx.synchronize()
    out = d_o.cpu().numpy().view(cases.OUT)
    kp = d_kp.cpu().numpy().view(np.float32).reshape(n, KCAP, 3)
    kw = d_kw.cpu().numpy().view(np.float32).reshape(n, KCAP, 3)
    checked = 0
    for p, e in enumerate(ev):
        ref_id, cur_id, kf_matches, kf_new, pts_sm, T_ref, T_cur, new = e
        o = out[p]
        assert o["status"] == 0 and o["usable"] == 1, (p, o)
        assert o["n_matches"] == kf_matches and o["n_kept"] == kf_new, (p, o["n_matches"], kf_matches, o["n_kept"], kf_new)
        nk = int(o["n_kept"])
        assert kp[p, :nk].tobytes() == np.ascontiguousarray(pts_sm, np.float32).reshape(-1, 3).tobytes(), p
        world = {kw[p, i].tobytes() for i in range(nk)}
        rows = [kw[p, i].tobytes() for i in range(nk)]
        pos = [rows.index(np.ascontiguousarray(x, np.float32).tobytes()) for _, x in sorted(new)]
        assert all(np.ascontiguousarray(x, np.float32).tobytes() in world for _, x in new), p
        assert pos == sorted(pos), p                                  # in order
        checked += 1
    assert checked == n
    print(f"{n} keyframe insertions replayed")
    bctx.close()
