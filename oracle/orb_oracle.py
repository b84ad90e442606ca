"""TEST ORACLE — numpy restatement of OpenCV's cv::ORB as the reference calls it.

Not product code: only tests/, smoke() and bench.py's cpu_baseline may import this.

Reference call sites (paths relative to the reference repo root):
  src/geometry/feature_match.cpp:22-23,34   cv::ORB::create(8000, 1.2, 4, 31, 0, 2, HARRIS_SCORE, 31, 20)->detect
  src/geometry/feature_match.cpp:45,48      cv::ORB::create(8000, 1.2, 4)->compute
  src/geometry/feature_match.cpp:51-84      selectUniformKptsByGrid  (in oracle/match_oracle.cpp)
OpenCV is a third-party dependency whose source is absent from the reference tree
(find_package(OpenCV 3.4) CMakeLists.txt:27); the algorithm below follows OpenCV's published
features2d/orb.cpp, fast.cpp, fast_score.cpp, keypoint.cpp and imgproc resize/filter code as
verified against the cv2 4.13 wheel (SURVEY.md Appendix A).  tests/test_orb_oracle.py pins every
stage here against cv2 live and against tests/golden/orb_*.npz.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np

from . import oracle_lib

KEYPOINT_DTYPE = oracle_lib.KEYPOINT_DTYPE
PATTERN = np.load(Path(__file__).resolve().parent / "orb_bit_pattern_31.npy")   # 256 x 4 int32 (x0,y0,x1,y1)

EDGE_THRESHOLD = 31
PATCH_SIZE = 31
HALF_PATCH = 15
HARRIS_BLOCK = 7
HARRIS_K = np.float32(0.04)
UMAX = np.array([15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3], np.int32)
# FAST-9/16 Bresenham ring, OpenCV order (dx, dy)
RING = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1),
        (-3, 0), (-3, 1), (-2, 2), (-1, 3)]


# ------------------------------------------------------------------------------ A.1 gray
def bgr_to_gray(bgr):
    """cv::cvtColor(BGR2GRAY) of OpenCV 4.x: 15-bit fixed point."""
    b = bgr[:, :, 0].astype(np.int32)
    g = bgr[:, :, 1].astype(np.int32)
    r = bgr[:, :, 2].astype(np.int32)
    return ((3735 * b + 19235 * g + 9798 * r + 16384) >> 15).astype(np.uint8)


# --------------------------------------------------------------------------- A.2 pyramid
def level_scales(nlevels, scale_factor):
    sf = float(np.float32(scale_factor))
    return [np.float32(sf ** l) for l in range(nlevels)]   # (float)pow((double)1.2f, level)


def _cv_round(x):
    return int(np.rint(x))   # round half to even, like cvRound


def level_sizes(cols, rows, nlevels, scale_factor):
    out = []
    for s in level_scales(nlevels, scale_factor):
        inv = np.float32(1.0) / s     # Size(cvRound(cols * invScale), cvRound(rows * invScale)), float invScale = 1.0f / scale
        out.append((_cv_round(np.float32(np.float32(cols) * inv)), _cv_round(np.float32(np.float32(rows) * inv))))
    return out


def _axis_coeffs(src, dst):
    scale = 1.0 / (dst / float(src))
    ofs = np.zeros(dst, np.int64)
    w1 = np.zeros(dst, np.int64)
    for d in range(dst):
        f = scale * (d + 0.5) - 0.5
        i = int(np.floor(f))
        if i < 0:
            ofs[d], w1[d] = 0, 0
        elif i >= src - 1:
            ofs[d], w1[d] = src - 1, 0
        else:
            ofs[d] = i
            w1[d] = int(np.rint((f - i) * 256))
    return ofs, w1


def resize_linear_exact(src, dw, dh):
    """cv::resize(..., INTER_LINEAR_EXACT) for 8-bit single channel: 8.8 x 8.8 fixed point."""
    sh, sw = src.shape
    ox, wx = _axis_coeffs(sw, dw)
    oy, wy = _axis_coeffs(sh, dh)
    s = src.astype(np.int64)
    ox1 = np.minimum(ox + 1, sw - 1)
    hrow = s[:, ox] * (256 - wx) + s[:, ox1] * wx            # (sh, dw)
    oy1 = np.minimum(oy + 1, sh - 1)
    v = hrow[oy, :] * (256 - wy)[:, None] + hrow[oy1, :] * wy[:, None]
    return ((v + 32768) >> 16).astype(np.uint8)


def build_pyramid(gray, nlevels=4, scale_factor=1.2):
    sizes = level_sizes(gray.shape[1], gray.shape[0], nlevels, scale_factor)
    levels = [gray]
    for l in range(1, nlevels):
        levels.append(resize_linear_exact(levels[-1], sizes[l][0], sizes[l][1]))   # chained from level l-1
    return levels


# ------------------------------------------------------------------------------ A.3 FAST
def fast_score_map(img, t):
    """cornerScore<16> for every FAST-9/16 corner of img (3-px margin), 0 elsewhere (int32)."""
    h, w = img.shape
    I = img.astype(np.int32)
    c = I[3:h - 3, 3:w - 3]
    d = [c - I[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for dx, dy in RING]
    d = d + d[:9]
    best_a = np.full(c.shape, -10000, np.int32)
    best_b = np.full(c.shape, -10000, np.int32)
    for k in range(16):
        arc = np.stack(d[k:k + 9])
        best_a = np.maximum(best_a, arc.min(0))          # centre brighter than the whole arc
        best_b = np.maximum(best_b, (-arc).min(0))       # centre darker than the whole arc
    m = np.maximum(best_a, best_b)
    score = np.zeros((h, w), np.int32)
    score[3:h - 3, 3:w - 3] = np.where(m > t, m - 1, 0)
    return score


def fast_detect(img, t=20):
    """cv::FAST(img, t, nonmax=true, TYPE_9_16): (x, y, score) in raster order."""
    s = fast_score_map(img, t)
    h, w = s.shape
    p = np.pad(s, 1)
    keep = s > 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx or dy:
                keep &= s > p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w]
    ys, xs = np.nonzero(keep)       # raster order
    return xs.astype(np.int32), ys.astype(np.int32), s[ys, xs].astype(np.int32)


# --------------------------------------------------------------------- A.4 per-level caps
def features_per_level(nfeatures, nlevels, scale_factor):
    factor = np.float32(1.0 / float(np.float32(scale_factor)))
    ndes = np.float32(nfeatures * (1 - factor) / (1 - np.float32(float(factor) ** nlevels)))
    out, s = [], 0
    for l in range(nlevels - 1):
        n = _cv_round(ndes)
        out.append(n)
        s += n
        ndes = np.float32(ndes * factor)
    out.append(max(nfeatures - s, 0))
    return out


# --------------------------------------------------------------------- A.5 Harris + angle
def harris_response(img, xs, ys):
    I = img.astype(np.int32)
    scale = np.float32(1.0) / np.float32((1 << 2) * HARRIS_BLOCK * np.float32(255.0))
    s4 = np.float32(np.float32(np.float32(scale * scale) * scale) * scale)
    out = np.zeros(len(xs), np.float32)
    r = HARRIS_BLOCK // 2
    for n, (x0, y0) in enumerate(zip(xs, ys)):
        blk = I[y0 - r - 1:y0 + r + 2, x0 - r - 1:x0 + r + 2]       # 9x9
        Ix = (blk[1:-1, 2:] - blk[1:-1, :-2]) * 2 + (blk[:-2, 2:] - blk[:-2, :-2]) + (blk[2:, 2:] - blk[2:, :-2])
        Iy = (blk[2:, 1:-1] - blk[:-2, 1:-1]) * 2 + (blk[2:, :-2] - blk[:-2, :-2]) + (blk[2:, 2:] - blk[:-2, 2:])
        a, b, c = int((Ix * Ix).sum()), int((Iy * Iy).sum()), int((Ix * Iy).sum())
        fa, fb, fc = np.float32(a), np.float32(b), np.float32(c)
        ab = np.float32(fa + fb)
        out[n] = np.float32(np.float32(np.float32(np.float32(fa * fb) - np.float32(fc * fc))
                                       - np.float32(np.float32(HARRIS_K * ab) * ab)) * s4)
    return out


_P1 = np.float32(np.float32(0.9997878412794807) * np.float32(57.29577951308232))
_P3 = np.float32(np.float32(-0.3258083974640975) * np.float32(57.29577951308232))
_P5 = np.float32(np.float32(0.1555786518463281) * np.float32(57.29577951308232))
_P7 = np.float32(np.float32(-0.04432655554792128) * np.float32(57.29577951308232))
_EPS = np.float32(2.220446049250313e-16)


def fast_atan2(y, x):
    """cv::fastAtan2 scalar path (degrees), float32 ops without contraction."""
    y, x = np.float32(y), np.float32(x)
    ax, ay = np.abs(x), np.abs(y)
    if ax >= ay:
        c = np.float32(ay / np.float32(ax + _EPS))
        c2 = np.float32(c * c)
        a = np.float32(np.float32(np.float32(np.float32(np.float32(np.float32(_P7 * c2) + _P5) * c2) + _P3) * c2) + _P1)
        a = np.float32(a * c)
    else:
        c = np.float32(ax / np.float32(ay + _EPS))
        c2 = np.float32(c * c)
        a = np.float32(np.float32(np.float32(np.float32(np.float32(np.float32(_P7 * c2) + _P5) * c2) + _P3) * c2) + _P1)
        a = np.float32(np.float32(90.0) - np.float32(a * c))
    if x < 0:
        a = np.float32(np.float32(180.0) - a)
    if y < 0:
        a = np.float32(np.float32(360.0) - a)
    return a


def ic_angle(img, xs, ys):
    I = img.astype(np.int64)
    out = np.zeros(len(xs), np.float32)
    for n, (x0, y0) in enumerate(zip(xs, ys)):
        m01 = m10 = 0
        for v in range(-HALF_PATCH, HALF_PATCH + 1):
            d = int(UMAX[abs(v)])
            row = I[y0 + v, x0 - d:x0 + d + 1]
            u = np.arange(-d, d + 1)
            m10 += int((u * row).sum())
            m01 += v * int(row.sum())
        out[n] = fast_atan2(np.float32(m01), np.float32(m10))
    return out


# ------------------------------------------------------------------------------- detect
def detect(image, nfeatures=8000, scale_factor=1.2, nlevels=4, fast_threshold=20, return_stages=False):
    """cv::ORB::detect: keypoints in OpenCV's output order (level-major)."""
    gray = bgr_to_gray(image) if image.ndim == 3 and image.shape[2] == 3 else image.reshape(image.shape[:2])
    levels = build_pyramid(gray, nlevels, scale_factor)
    scales = level_scales(nlevels, scale_factor)
    caps = features_per_level(nfeatures, nlevels, scale_factor)
    out = []
    stages = []
    for l, img in enumerate(levels):
        h, w = img.shape
        xs, ys, sc = fast_detect(img, fast_threshold)
        inb = (xs >= EDGE_THRESHOLD) & (xs < w - EDGE_THRESHOLD) & (ys >= EDGE_THRESHOLD) & (ys < h - EDGE_THRESHOLD)
        xs, ys, sc = xs[inb], ys[inb], sc[inb]
        stages.append((xs.copy(), ys.copy(), sc.copy()))
        keep = oracle_lib.retain_best(sc.astype(np.float32), 2 * caps[l])       # by FAST score
        xs, ys = xs[keep], ys[keep]
        resp = harris_response(img, xs, ys)
        keep = oracle_lib.retain_best(resp, caps[l])                           # by Harris
        xs, ys, resp = xs[keep], ys[keep], resp[keep]
        ang = ic_angle(img, xs, ys)
        kp = np.zeros(len(xs), KEYPOINT_DTYPE)
        s = scales[l]
        kp["x"] = xs.astype(np.float32) * s if l else xs.astype(np.float32)
        kp["y"] = ys.astype(np.float32) * s if l else ys.astype(np.float32)
        kp["size"] = np.float32(PATCH_SIZE) * s
        kp["angle"] = ang
        kp["response"] = resp
        kp["octave"] = l
        kp["class_id"] = -1
        out.append(kp)
    res = np.concatenate(out) if out else np.zeros(0, KEYPOINT_DTYPE)
    return (res, levels, stages) if return_stages else res


# --------------------------------------------------------------------------- A.6 compute
def gaussian_kernel7():
    """cv::getGaussianKernel(7, 2, CV_32F)."""
    x = np.arange(7, dtype=np.float64) - 3
    k = np.exp(-x * x / (2 * 2.0 * 2.0))
    return (k / k.sum()).astype(np.float32)


def blur7(img):
    """GaussianBlur(7x7, sigma 2, BORDER_REFLECT_101) as ORB gets it: the classic float separable
    filter (row pass u8->f32 ascending taps, symmetric column pass, round half to even)."""
    k = gaussian_kernel7()
    p = np.pad(img, 3, mode="reflect").astype(np.float32)
    h, w = img.shape
    row = np.zeros((h + 6, w), np.float32)
    for i in range(7):
        term = k[i] * p[:, i:i + w]
        row = term if i == 0 else (row + term).astype(np.float32)
    col = (k[3] * row[3:3 + h]).astype(np.float32)
    for i in range(1, 4):
        col = (col + k[3 + i] * (row[3 + i:3 + i + h] + row[3 - i:3 - i + h]).astype(np.float32)).astype(np.float32)
    return np.clip(np.rint(col), 0, 255).astype(np.uint8)


def compute(image, kpts, scale_factor=1.2, nlevels=4):
    """cv::ORB::compute for level-sorted keypoints that are all inside the 31-px border."""
    gray = bgr_to_gray(image) if image.ndim == 3 and image.shape[2] == 3 else image.reshape(image.shape[:2])
    levels = [blur7(l) for l in build_pyramid(gray, nlevels, scale_factor)]
    scales = level_scales(nlevels, scale_factor)
    px = PATTERN.reshape(512, 2)[:, 0].astype(np.float32)
    py = PATTERN.reshape(512, 2)[:, 1].astype(np.float32)
    desc = np.zeros((len(kpts), 32), np.uint8)
    deg2rad = np.float32(np.pi / 180.0)
    for n, kp in enumerate(kpts):
        img = levels[int(kp["octave"])]
        s = np.float32(1.0) / scales[int(kp["octave"])]
        cx = _cv_round(np.float32(kp["x"] * s))
        cy = _cv_round(np.float32(kp["y"] * s))
        th = np.float32(kp["angle"] * deg2rad)
        a, b = np.float32(np.cos(np.float64(th))), np.float32(np.sin(np.float64(th)))
        x = (px * a).astype(np.float32) - (py * b).astype(np.float32)
        y = (px * b).astype(np.float32) + (py * a).astype(np.float32)
        ix = np.rint(x).astype(np.int64) + cx
        iy = np.rint(y).astype(np.int64) + cy
        v = img[iy, ix].astype(np.int32)
        bits = (v[0::2] < v[1::2]).astype(np.uint8)
        desc[n] = np.packbits(bits.reshape(32, 8), axis=1, bitorder="little").ravel()
    return desc
