"""Cases of the ORB extraction over its parameter and image-geometry space, the host's launch rules restated and the checks, shared
by test_orb_params_gpu.py (the H100, against cv2 live or the committed goldens) and test_orb_params_emu.py (the library built for
the host, against the numpy oracle).

The reference passes scale_factor, level_pyramid, score_threshold and number_of_keypoints_to_extract to cv::ORB::create and reads
the grid size and the per-cell limit in selectUniformKptsByGrid (feature_match.cpp:11-84).  Which kernels and paths run depends on
them and on the image size (csrc/orb_host.cpp: build_plan, csrc/orb.cu: the launchers); `plan` restates those rules and `configs`
names what a case reaches.  Every case is checked field by field (x, y, size, angle, response, octave, class_id and the 32
descriptor bytes) through mvo_orb_extract, mvo_calc_keypoints + mvo_calc_descriptors and, for batches, mvo_orb_extract_batch_dev,
and checks that its frames took the retainBest path it was built for:
  ovf0    no level above OpenCV's featuresPerLevel: k_select selects at once;
  retain  a level above its cap: retainBest and the grid selection on the device (k_retain, k_select_kept);
  host    a level holds more candidates than k_retain does (RET_MAX), or k_retain declines the frame (where libstdc++'s nth_element
          would leave quickselect, or ties keep more than nfeatures): retainBest on the host (mvo_test_orb_host_fallbacks counts it).
Cases with `err` must be rejected with that error code, and again on a second call on the same context."""
import ctypes as C

import numpy as np

import mvo_synth
from oracle import oracle_lib, orb_oracle as oo

EDGE, BAND_H, MAX_BANDS, MAX_W, RET_MAX, SMEM_MAX = 31, 8, 1024, 4096, 12288, 220 * 1024
ERR_UNSUPPORTED = -5
DEFAULTS = dict(orb_nfeatures=8000, orb_scale_factor=1.2, orb_nlevels=4, orb_fast_threshold=20, max_keypoints=1500, grid_size=16,
                max_pts_per_grid=8)
FIELDS = ("x", "y", "size", "angle", "response", "octave", "class_id")


# ---- the host's launch rules, restated ----------------------------------------------------------------------------------------
def _axis_rows(src, dst):
    return oo._axis_coeffs(src, dst)[0]


def pyramid_rows(sizes, rows):
    """build_plan's band table of k_pyramid: the most rows of each level one band holds (its own rows plus the source rows of the
    rows it holds of the level above)."""
    nl, nb = len(sizes), max(1, rows // 8)
    yofs = [None] + [_axis_rows(sizes[l - 1][1], sizes[l][1]) for l in range(1, nl)]
    out = [0] * nl
    for b in range(nb):
        lo = hi = 0
        for l in range(nl - 1, -1, -1):
            H = sizes[l][1]
            olo, ohi = b * H // nb, (b + 1) * H // nb
            nlo, nhi = olo, ohi
            if l + 1 < nl and hi > lo:
                y = yofs[l + 1]
                slo, shi = int(y[lo]), min(int(y[hi - 1]) + 1, H - 1) + 1
                nlo, nhi = (min(nlo, slo), max(nhi, shi)) if nhi > nlo else (slo, shi)
            out[l] = max(out[l], nhi - nlo)
            lo, hi = nlo, nhi
    return out


def select_smem(ncell, nfeat):
    """Dynamic shared memory of k_select and of k_select_kept without the per-warp count tables."""
    return ((MAX_BANDS + 1) * 4 + (ncell + 1) * 4 + ncell * 4 + nfeat * 4 + nfeat + 64, (2 * ncell + 1) * 4 + nfeat * 10 + 64)


def max_nfeatures(ncell):
    """The largest orb_nfeatures both selection kernels fit in 220 KB of shared memory for."""
    return min((SMEM_MAX - (MAX_BANDS + 1) * 4 - 8 * ncell - 4 - 64) // 5, (SMEM_MAX - 8 * ncell - 4 - 64) // 10)


def plan(rows, cols, p):
    """What build_plan and the launchers choose for an image of rows x cols under params p (DEFAULTS overridden by p), or
    {"err": reason} where the call is rejected with MVO_ERR_UNSUPPORTED."""
    q = {**DEFAULTS, **p}
    nl, sf, nf, g, mpc = q["orb_nlevels"], q["orb_scale_factor"], q["orb_nfeatures"], q["grid_size"], q["max_pts_per_grid"]
    if rows < 2 * EDGE + 8 or cols < 2 * EDGE + 8:
        return {"err": "image_under_70"}
    if rows >= MAX_W or cols >= MAX_W:
        return {"err": "width_4096"}
    gr, gc = rows // g, cols // g
    if gr < 1 or gc < 1 or gr * gc > 65535:
        return {"err": "ncell"}
    sizes = oo.level_sizes(cols, rows, nl, sf)
    if any(w < 2 * EDGE + 2 or h < 2 * EDGE + 2 for w, h in sizes):
        return {"err": "level_under_border"}
    nbands = [-(-(h - 2 * EDGE) // BAND_H) for _, h in sizes]
    if sum(nbands) > MAX_BANDS:
        return {"err": "bands"}
    pitch = [(w + 127) & ~127 for w, _ in sizes]
    prow = pyramid_rows(sizes, rows)
    pyr_smem = sum(prow[l] * pitch[l] for l in range(nl - 1)) + 16
    ncell = gr * gc
    s1, s2 = select_smem(ncell, nf)
    if s1 > SMEM_MAX or s2 > SMEM_MAX:
        return {"err": "select_smem"}
    return dict(sizes=sizes, caps=oo.features_per_level(nf, nl, sf), nbands=nbands, pitch=pitch, pyr_rows=prow, pyr_smem=pyr_smem,
                pyramid="fused" if pyr_smem <= 200 * 1024 else "gray+resize",
                staging="tma" if pitch[0] // 4 <= 256 else "vector",
                reject="packed" if q["orb_fast_threshold"] <= 127 else "scalar",
                cell="shift" if g & (g - 1) == 0 else "division",
                select="two_pass" if mpc <= 254 and s1 + 32 * ncell + 32 <= SMEM_MAX else "rounds",
                select_kept="two_pass" if mpc <= 254 and s2 + 32 * ncell + 32 <= SMEM_MAX else "rounds",
                grid=(gr, gc), strip=(cols - gc * g > EDGE or rows - gr * g > EDGE))


def expected_path(counts, caps):
    """The retainBest path of a frame whose levels hold `counts` FAST candidates inside the border."""
    if all(n <= c for n, c in zip(counts, caps)):
        return "ovf0"
    return "host" if max(counts) > RET_MAX else "retain"


# ---- scenes -------------------------------------------------------------------------------------------------------------------
def threshold_scene(t, width=256, height=200):
    """Isolated dots and 4 x 4 squares whose contrast to a flat background is t - 1, t, t + 1 and t + 2: bright ones on a dark left
    half, dark ones on a bright right half.  A dot is a FAST corner iff its contrast exceeds t, so an off-by-one in the quick reject
    (packed K4 compare or scalar test) or in the exact re-test adds or drops keypoints."""
    lo = max(0, (253 - t) // 2)
    hi = 255 - lo
    img = np.full((height, width), lo, np.uint8)
    img[:, width // 2:] = hi
    k = 0
    for y in range(36, height - 36, 11):
        for x in range(36, width - 36, 11):
            if abs(x - width // 2) < 8:
                continue
            d = t - 1 + (k % 4)
            k += 1
            bg = lo if x < width // 2 else hi
            v = bg + d if bg == lo else bg - d
            if not 0 <= v <= 255:
                continue
            if (k // 4) % 3 == 2:
                img[y:y + 4, x:x + 4] = v
            else:
                img[y, x] = v
    return img


def _bgr(g):
    return mvo_synth.gray_to_bgr(g)


def _rect(seed, w, h, n=None, bgr=True):
    g = mvo_synth.rect_scene(seed, w, h, n_rect=n if n is not None else max(60, w * h // 205))
    return _bgr(g) if bgr else g


def _dots70():
    """The smallest image ORB accepts: FAST looks at the 8 x 8 pixels inside the border; four dots there, 5 px apart."""
    img = np.full((70, 70), 90, np.uint8)
    for y, x, v in ((32, 32, 200), (32, 37, 10), (37, 32, 150), (37, 37, 30)):
        img[y, x] = v
    return img


def case(name, img, path=None, err=None, stride_pad=0, base_offset=0, tier="gpu", **p):
    return dict(name=name, img=img, p=p, path=path, err=err, stride_pad=stride_pad, base_offset=base_offset, tier=tier)


# tier: "gpu" runs on the H100 only, "both" also on the emulated library (small images)
CASES = [
    # pyramid depth and scale factor
    case("nl1_70x70", _dots70, "ovf0", tier="both", orb_nlevels=1, grid_size=10),
    case("nl1_200x152", lambda: _rect(4, 200, 152, 120, False), "ovf0", tier="both", orb_nlevels=1),
    case("nl1_640x480", lambda: _rect(1, 640, 480), "ovf0", orb_nlevels=1),
    case("nl2_sf2_641x477", lambda: _rect(2, 641, 477), "ovf0", orb_nlevels=2, orb_scale_factor=2.0),
    case("nl3_sf1.5_517x389", lambda: _rect(5, 517, 389), "ovf0", orb_nlevels=3, orb_scale_factor=1.5),
    case("nl3_sf1.5_203x161", lambda: _rect(6, 203, 161, 150), "ovf0", tier="both", orb_nlevels=3, orb_scale_factor=1.5),
    case("nl8_sf1.2_642x480", lambda: _rect(7, 642, 480), "retain", orb_nlevels=8),
    case("nl8_sf1.05_643x470", lambda: _rect(8, 643, 470), "retain", orb_nlevels=8, orb_scale_factor=1.05),
    case("nl8_sf1.2_256x240", lambda: _rect(9, 256, 240, 250, False), "ovf0", tier="both", orb_nlevels=8),
    case("nl4_sf2_1100x900", lambda: _rect(10, 1100, 900), "retain", orb_nlevels=4, orb_scale_factor=2.0),
    case("nl8_sf1.2_3000x800", lambda: _rect(11, 3000, 800), "host", orb_nlevels=8),
    case("nl8_sf1.3_2000x1100", lambda: _rect(12, 2000, 1100), "host", orb_nlevels=8, orb_scale_factor=1.3),
    # FAST thresholds on both sides of the packed / scalar switch
    *[case(f"t{t}_dots", (lambda t=t: threshold_scene(t)), "ovf0", tier="both", orb_fast_threshold=t)
      for t in (1, 20, 126, 127, 128, 200, 254)],
    case("t1_rect", lambda: _rect(13, 640, 480), "retain", orb_fast_threshold=1),
    case("t127_rect", lambda: _rect(14, 640, 480), "ovf0", orb_fast_threshold=127),
    case("t128_rect", lambda: _rect(14, 640, 480), "ovf0", orb_fast_threshold=128),
    # orb_nfeatures: every level over its cap, nothing over, a level beyond RET_MAX, the largest accepted and the first rejected
    case("nf300_every_level_over", lambda: _rect(15, 640, 480), "host", orb_nfeatures=300),     # every level over: k_retain declines
    case("nf120_small", lambda: _rect(4, 200, 152, 120, False), "retain", tier="both", orb_nfeatures=120, max_keypoints=60),
    case("nf20000_nothing_over", lambda: _rect(16, 640, 480), "ovf0", orb_nfeatures=20000, max_keypoints=2000),
    case("nf2000_host", lambda: _bgr(mvo_synth.noise_scene(17)), "host", orb_nfeatures=2000),
    case("nf_max_accepted", lambda: _rect(18, 640, 480), "ovf0", orb_nfeatures=max_nfeatures(1200)),
    case("nf_first_rejected", lambda: _rect(18, 640, 480), err=ERR_UNSUPPORTED, orb_nfeatures=max_nfeatures(1200) + 1),
    case("nf_first_rejected_small", lambda: _rect(4, 200, 152, 120, False), err=ERR_UNSUPPORTED, tier="both",
         orb_nfeatures=max_nfeatures(108) + 1),
    # grid size: power of two (shift) or not (division), one pixel, cells past the covered image
    case("grid1_128x128", lambda: _rect(19, 128, 128, 60, False), "ovf0", tier="both", grid_size=1, orb_nlevels=1, orb_nfeatures=2000),
    case("grid1_640x480", lambda: _rect(19, 640, 480), err=ERR_UNSUPPORTED, tier="both", grid_size=1),
    case("grid12", lambda: _rect(20, 640, 480), "ovf0", grid_size=12),
    case("grid20_retain", lambda: _rect(21, 640, 480), "retain", grid_size=20, orb_nfeatures=1000),
    case("grid12_small", lambda: _rect(22, 200, 152, 150, False), "ovf0", tier="both", grid_size=12, max_pts_per_grid=3),
    case("grid64_strip_630x500", lambda: _rect(23, 630, 500), "ovf0", grid_size=64, max_pts_per_grid=20, orb_nfeatures=12000),
    case("grid64_strip_retain", lambda: _rect(24, 630, 500), "retain", grid_size=64, max_pts_per_grid=20, orb_nfeatures=3000),
    case("grid64_strip_host", lambda: _bgr(mvo_synth.noise_scene(25, 630, 500)), "host", grid_size=64, max_pts_per_grid=20),
    case("grid64_strip_250x200", lambda: _rect(26, 250, 200, 250, False), "ovf0", tier="both", grid_size=64, max_pts_per_grid=6),
    case("grid64_strip_250x200_retain", lambda: _rect(26, 250, 200, 250, False), "retain", tier="both", grid_size=64,
         max_pts_per_grid=6, orb_nfeatures=150),
    # per-cell limit (two-pass below 255, rounds from 255) and max_keypoints (the reference keeps max_keypoints + 1)
    case("mpc0", lambda: _rect(27, 640, 480), "retain", max_pts_per_grid=0),
    case("mpc1", lambda: _rect(27, 640, 480), "retain", max_pts_per_grid=1),
    case("mpc254", lambda: _rect(28, 640, 480), "retain", max_pts_per_grid=254, orb_nfeatures=2000, max_keypoints=2000),
    case("mpc255", lambda: _rect(28, 640, 480), "retain", max_pts_per_grid=255, orb_nfeatures=2000, max_keypoints=2000),
    case("mpc255_small", lambda: _rect(29, 200, 152, 150, False), "ovf0", tier="both", max_pts_per_grid=255, grid_size=32),
    case("mpc0_small", lambda: _rect(29, 200, 152, 150, False), "ovf0", tier="both", max_pts_per_grid=0),
    case("maxkp0", lambda: _rect(30, 640, 480), "ovf0", max_keypoints=0),
    case("maxkp1", lambda: _rect(30, 640, 480), "ovf0", max_keypoints=1),
    case("maxkp2000", lambda: _rect(30, 640, 480), "ovf0", max_keypoints=2000),
    # geometry: staging widths, short last FAST band, strides and channel counts
    case("w1024", lambda: _rect(31, 1024, 600), "retain"),
    case("w1025", lambda: _rect(32, 1025, 600), "retain"),
    case("w1100_gray_stride", lambda: _rect(33, 1100, 601, bgr=False), "retain", stride_pad=20),
    case("w641_bgr_unaligned_stride", lambda: _rect(34, 641, 481), "ovf0", stride_pad=5),
    case("w642_bgr_unaligned_base", lambda: _rect(35, 642, 482), "retain", base_offset=1),
    case("w201_bgr_unaligned", lambda: _rect(36, 201, 153, 150), "ovf0", tier="both", stride_pad=3),   # level 1: 128 rows, not 127
    case("w202_gray_stride", lambda: _rect(37, 202, 155, 150, False), "ovf0", tier="both", stride_pad=9),
    case("w203_bgr_aligned_stride", lambda: _rect(38, 203, 157, 150), "ovf0", tier="both", stride_pad=3),
    case("too_small_69x70", lambda: _rect(39, 69, 70, 40, False), err=ERR_UNSUPPORTED, tier="both", orb_nlevels=1, grid_size=10),
    case("level_under_border_200x152", lambda: _rect(4, 200, 152, 120, False), err=ERR_UNSUPPORTED, tier="both", orb_scale_factor=1.5),
    case("bands_over_1024", lambda: _rect(41, 300, 1300, 400, False), err=ERR_UNSUPPORTED, tier="both", orb_nlevels=8,
         orb_scale_factor=1.05),
    case("width_4096", lambda: np.zeros((100, 4096), np.uint8), err=ERR_UNSUPPORTED, orb_nlevels=1),
]
CASE = {c["name"]: c for c in CASES}
assert len(CASE) == len(CASES)


def image(c):
    if "_img" not in c:
        c["_img"] = c["img"]()
    return c["_img"]


def case_plan(c):
    img = image(c)
    return plan(img.shape[0], img.shape[1], c["p"])


def configs(c):
    """The configurations case c reaches by the rules above."""
    q = {**DEFAULTS, **c["p"]}
    pl = case_plan(c)
    if "err" in pl:
        return {"err:" + pl["err"]}
    img = image(c)
    out = {f"nlevels={q['orb_nlevels']}", f"sf={q['orb_scale_factor']}", f"t={q['orb_fast_threshold']}", f"mpc={q['max_pts_per_grid']}",
           f"maxkp={q['max_keypoints']}", f"grid={q['grid_size']}", "pyramid:" + pl["pyramid"], "staging:" + pl["staging"],
           "reject:" + pl["reject"], "cell:" + pl["cell"], "path:" + c["path"], f"w%4={img.shape[1] % 4}", f"ch={1 if img.ndim == 2 else 3}"}
    out.add("select:" + pl["select"] if c["path"] == "ovf0" else "select_kept:" + pl["select_kept"])
    if (img.shape[0] - 2 * EDGE) % BAND_H:
        out.add("short_last_band")
    if pl["strip"]:
        out.add("strip:" + c["path"])
    if c["stride_pad"] % 4 or c["base_offset"] % 4:
        out.add("unaligned")
    elif c["stride_pad"]:
        out.add("padded_stride")
    if q["orb_nfeatures"] == max_nfeatures(pl["grid"][0] * pl["grid"][1]):
        out.add("nf_max_accepted")
    if img.shape[0] == img.shape[1] == 2 * EDGE + 8:
        out.add("smallest_image")
    return out


REQUIRED = ({f"nlevels={n}" for n in (1, 2, 3, 4, 8)} | {f"sf={s}" for s in (1.2, 1.05, 1.5, 2.0)}
            | {f"t={t}" for t in (1, 20, 126, 127, 128, 200, 254)} | {f"mpc={m}" for m in (0, 1, 8, 254, 255)}
            | {f"maxkp={m}" for m in (0, 1, 1500, 2000)} | {f"grid={g}" for g in (1, 12, 16, 20, 64)}
            | {"pyramid:fused", "pyramid:gray+resize", "staging:tma", "staging:vector", "reject:packed", "reject:scalar",
               "cell:shift", "cell:division", "path:ovf0", "path:retain", "path:host", "select:two_pass", "select:rounds",
               "select_kept:two_pass", "select_kept:rounds", "w%4=0", "w%4=1", "w%4=2", "w%4=3", "ch=1", "ch=3", "short_last_band",
               "strip:ovf0", "strip:retain", "strip:host", "unaligned", "padded_stride", "nf_max_accepted", "smallest_image",
               "err:image_under_70", "err:width_4096", "err:ncell", "err:bands", "err:level_under_border", "err:select_smem"})


# ---- references ---------------------------------------------------------------------------------------------------------------
def _gray(img):
    return img if img.ndim == 2 else oo.bgr_to_gray(img)


def _fast_counts_cv2(img, q):
    """FAST candidates inside the border per level, by cv2 (resize INTER_LINEAR_EXACT chained as cv::ORB builds its pyramid)."""
    import cv2
    g = _gray(img)
    sizes = oo.level_sizes(g.shape[1], g.shape[0], q["orb_nlevels"], q["orb_scale_factor"])
    lv, out = g, []
    fd = cv2.FastFeatureDetector_create(q["orb_fast_threshold"], True)
    for l, (w, h) in enumerate(sizes):
        if l:
            lv = cv2.resize(lv, (w, h), interpolation=cv2.INTER_LINEAR_EXACT)
        out.append(sum(1 for k in fd.detect(lv) if EDGE <= k.pt[0] < w - EDGE and EDGE <= k.pt[1] < h - EDGE))
    return out


def reference_cv2(img, p):
    """cv::ORB::create(nfeat, sf, nl, 31, 0, 2, HARRIS, 31, t)->detect, selectUniformKptsByGrid, cv::ORB::create(nfeat, sf, nl)->compute
    (feature_match.cpp:22-23,34,45,48,51-84); returns (selected keypoints, descriptors, per-level candidate counts)."""
    import cv2
    q = {**DEFAULTS, **p}
    nf, sf, nl, t = q["orb_nfeatures"], q["orb_scale_factor"], q["orb_nlevels"], q["orb_fast_threshold"]
    kps = cv2.ORB_create(nf, sf, nl, 31, 0, 2, cv2.ORB_HARRIS_SCORE, 31, t).detect(img, None)
    det = np.array([(k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, k.class_id) for k in kps], oo.KEYPOINT_DTYPE)
    sel = oracle_lib.select_uniform_kpts_by_grid(det, img.shape[0], img.shape[1], q["max_keypoints"], q["grid_size"], q["max_pts_per_grid"])
    desc = np.zeros((0, 32), np.uint8)
    if len(sel):
        ck = [cv2.KeyPoint(float(k["x"]), float(k["y"]), float(k["size"]), float(k["angle"]), float(k["response"]), int(k["octave"]),
                           int(k["class_id"])) for k in sel]
        ck2, desc = cv2.ORB_create(nf, sf, nl).compute(img, ck)
        assert len(ck2) == len(sel)
    return sel, desc, _fast_counts_cv2(img, q)


def reference_oracle(img, p):
    """The same through the numpy oracle (oracle/orb_oracle.py, pinned against cv2 at these parameters by test_orb_oracle.py)."""
    q = {**DEFAULTS, **p}
    det, _, stages = oo.detect(img, nfeatures=q["orb_nfeatures"], scale_factor=q["orb_scale_factor"], nlevels=q["orb_nlevels"],
                               fast_threshold=q["orb_fast_threshold"], return_stages=True)
    sel = oracle_lib.select_uniform_kpts_by_grid(det, img.shape[0], img.shape[1], q["max_keypoints"], q["grid_size"], q["max_pts_per_grid"])
    desc = oo.compute(img, sel, scale_factor=q["orb_scale_factor"], nlevels=q["orb_nlevels"]) if len(sel) else np.zeros((0, 32), np.uint8)
    return sel, desc, [len(s[0]) for s in stages]


# ---- running a case through the C ABI -----------------------------------------------------------------------------------------
def bind(lib):
    """Signatures for a library handle (the installed library or an emulated build)."""
    import mvo_b200
    for name, (res, args) in mvo_b200.SIGNATURES.items():
        if hasattr(lib, name):
            getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    lib.mvo_test_orb_host_fallbacks.restype = C.c_uint64
    lib.mvo_test_orb_host_fallbacks.argtypes = []
    lib.mvo_test_grid_rank.restype = C.c_int
    lib.mvo_test_grid_rank.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return lib


def set_params(lib, h, p):
    import mvo_b200
    prm = mvo_b200.Params()
    lib.mvo_default_params(C.byref(prm))
    for k, v in {**DEFAULTS, **p}.items():
        setattr(prm, k, v)
    assert lib.mvo_set_params(h, C.byref(prm)) == 0, lib.mvo_last_error(h)


def host_image(img, stride_pad=0, base_offset=0):
    """The image in a buffer with rows `stride_pad` bytes longer than cols x channels, starting `base_offset` bytes into it.
    Returns (keep-alive array, address, stride)."""
    rows, cols = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    stride = cols * ch + stride_pad
    buf = np.zeros(rows * stride + base_offset + 64, np.uint8)
    view = buf[base_offset:base_offset + rows * stride].reshape(rows, stride)
    view[:, :cols * ch] = img.reshape(rows, cols * ch)
    return buf, buf.ctypes.data + base_offset, stride


def run(lib, h, c):
    """One case through mvo_orb_extract and mvo_calc_keypoints + mvo_calc_descriptors: {rc, kp, desc, kp2, desc2, host}."""
    import mvo_b200
    img = image(c)
    rows, cols = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    set_params(lib, h, c["p"])
    buf, addr, stride = host_image(img, c["stride_pad"], c["base_offset"])
    cap = {**DEFAULTS, **c["p"]}["max_keypoints"] + 8
    kp, desc, n = np.zeros(cap, mvo_b200.KEYPOINT_DTYPE), np.zeros((cap, 32), np.uint8), C.c_int(cap)
    h0 = lib.mvo_test_orb_host_fallbacks()
    rc = lib.mvo_orb_extract(h, addr, rows, cols, ch, stride, kp.ctypes.data, C.byref(n), desc.ctypes.data)
    out = dict(rc=rc, host=lib.mvo_test_orb_host_fallbacks() - h0)
    if rc != 0:
        out["rc2"] = lib.mvo_orb_extract(h, addr, rows, cols, ch, stride, kp.ctypes.data, C.byref(C.c_int(cap)), desc.ctypes.data)
        return out
    out.update(kp=kp[:n.value].copy(), desc=desc[:n.value].copy())
    kp2, n2 = np.zeros(cap, mvo_b200.KEYPOINT_DTYPE), C.c_int(cap)
    assert lib.mvo_calc_keypoints(h, addr, rows, cols, ch, stride, kp2.ctypes.data, C.byref(n2)) == 0, lib.mvo_last_error(h)
    out["kp2"] = kp2[:n2.value].copy()
    desc2 = np.zeros((n2.value, 32), np.uint8)
    assert lib.mvo_calc_descriptors(h, addr, rows, cols, ch, stride, out["kp2"].ctypes.data, n2.value, desc2.ctypes.data) == 0, \
        lib.mvo_last_error(h)
    out["desc2"] = desc2
    return out


def assert_kp_equal(got, ref, what=""):
    assert len(got) == len(ref), (what, len(got), len(ref))
    for f in FIELDS:
        bad = np.nonzero(got[f] != ref[f])[0]
        assert bad.size == 0, f"{what} {f}: {bad.size} mismatches, first at {bad[:5]}: {got[f][bad[:5]]} vs {ref[f][bad[:5]]}"


def check(c, r, ref):
    """r: what `run` returned; ref: (selected keypoints, descriptors, per-level candidate counts) of a reference, or None for an
    error case."""
    name = c["name"]
    if c["err"] is not None:
        assert r["rc"] == c["err"] and r["rc2"] == c["err"], (name, r["rc"], r["rc2"])
        assert r["host"] == 0, name
        return
    assert r["rc"] == 0, (name, r["rc"])
    sel, desc, counts = ref
    pl = case_plan(c)
    path = expected_path(counts, pl["caps"])
    taken = "host" if r["host"] else path                  # the device retainBest may also decline an overflowing frame (orb.cu: k_retain)
    assert r["host"] in (0, 1) and (path != "host" or taken == "host") and (path != "ovf0" or taken == "ovf0"), (name, path, r["host"])
    assert taken == c["path"], f"{name}: built for path {c['path']}, took {taken} (candidate counts {counts}, caps {pl['caps']})"
    assert_kp_equal(r["kp"], sel, name + " orb_extract")
    assert np.array_equal(r["desc"], desc), f"{name}: {int(np.any(r['desc'] != desc, axis=1).sum())} descriptor rows differ"
    assert_kp_equal(r["kp2"], sel, name + " calc_keypoints")
    assert np.array_equal(r["desc2"], desc), f"{name}: calc_descriptors differs"


# ---- batches ------------------------------------------------------------------------------------------------------------------
BATCH_PARAMS = dict(orb_nfeatures=2000, max_keypoints=1500)


def batch_frames(small=False):
    """Frames of one geometry that take every path under BATCH_PARAMS: ovf0 (few rectangles), retain (dense rectangles) and, at
    640 x 480, host (noise: a level beyond RET_MAX)."""
    if small:
        w, h = 200, 152
        return [_rect(50, w, h, 10), _rect(51, w, h, 300), _rect(52, w, h, 12)], ["ovf0", "retain", "ovf0"]
    return ([_rect(53, 640, 480, 12), _rect(54, 640, 480), _bgr(mvo_synth.noise_scene(55)), _rect(56, 640, 480, 15)],
            ["ovf0", "retain", "host", "ovf0"])


def batch_run(lib, h, frames, d_images, d_kp, d_desc, d_cnt, cap, read):
    """mvo_orb_extract_batch_dev over frames already at d_images; read(): (keypoints [B, cap], descriptors [B, cap, 32], counts)."""
    import mvo_b200
    B, (rows, cols, ch) = len(frames), frames[0].shape
    h0 = lib.mvo_test_orb_host_fallbacks()
    rc = lib.mvo_orb_extract_batch_dev(h, d_images, B, rows, cols, ch, cols * ch, rows * cols * ch, d_kp, d_desc, d_cnt, cap)
    assert rc == 0, lib.mvo_last_error(h)
    kp, desc, cnt = read()
    return (kp.view(mvo_b200.KEYPOINT_DTYPE)[:B * cap].reshape(B, cap), desc[:B * cap * 32].reshape(B, cap, 32), cnt[:B],
            lib.mvo_test_orb_host_fallbacks() - h0)


def check_batch(frames, paths, got, refs, p):
    kp, desc, cnt, host = got
    caps = plan(frames[0].shape[0], frames[0].shape[1], p)["caps"]
    for f, (sel, d, counts) in enumerate(refs):
        assert expected_path(counts, caps) == paths[f], (f, counts, caps, paths[f])
        assert cnt[f] == len(sel), (f, cnt[f], len(sel))
        assert_kp_equal(kp[f, :cnt[f]], sel, f"batch frame {f}")
        assert np.array_equal(desc[f, :cnt[f]], d), f"batch frame {f}: descriptors differ"
    assert host == paths.count("host"), host


# ---- grid selection with keypoints outside the grid ---------------------------------------------------------------------------
def check_grid_rank_outside(lib, h):
    """Both device formulations of the per-cell counter skip items marked outside the grid (0xFFFF): never kept, no quota used."""
    rng = np.random.default_rng(3)
    for n, ncell, mpc in ((5000, 300, 4), (2000, 7, 254), (700, 1, 1), (33, 2, 8)):
        cells = rng.integers(0, ncell, n).astype(np.uint16)
        cells[rng.random(n) < 0.3] = 0xFFFF
        cnt, ref = {}, np.zeros(n, np.uint8)
        for i, cl in enumerate(cells.tolist()):
            if cl != 0xFFFF:
                ref[i] = cnt.get(cl, 0) < mpc
                cnt[cl] = cnt.get(cl, 0) + 1
        for seg in (1, 0):
            keep = np.full(n, 7, np.uint8)
            assert lib.mvo_test_grid_rank(h, cells.ctypes.data, n, ncell, mpc, seg, keep.ctypes.data) == 0
            assert np.array_equal(keep, ref), (n, ncell, mpc, seg, int(np.count_nonzero(keep != ref)))
