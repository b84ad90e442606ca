"""Pins the ORB oracle (oracle/orb_oracle.py, numpy) against OpenCV's cv::ORB — the third-party
code the reference calls at src/geometry/feature_match.cpp:22-23,34,45,48 — live via cv2 when it
is importable, and against the committed golden vectors (generated from cv2 4.13)."""
import numpy as np
import pytest
from conftest import GOLDEN, have_cv2

import mvo_synth
from oracle import oracle_lib, orb_oracle as oo


def _cvkp(kps):
    return np.array([(k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, k.class_id) for k in kps], oo.KEYPOINT_DTYPE)


SCENES = {
    "rect0": lambda: mvo_synth.gray_to_bgr(mvo_synth.rect_scene(0)),
    "color1": lambda: mvo_synth.color_scene(1),              # above the per-level caps on levels 0-1
    "odd": lambda: mvo_synth.gray_to_bgr(mvo_synth.rect_scene(5, 517, 389)),
}


@pytest.mark.skipif(not have_cv2(), reason="cv2 not importable")
@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_detect_compute_vs_cv2(name):
    import cv2
    img = SCENES[name]()
    ref = _cvkp(cv2.ORB_create(8000, 1.2, 4, 31, 0, 2, cv2.ORB_HARRIS_SCORE, 31, 20).detect(img, None))
    got = oo.detect(img)
    assert got.tobytes() == ref.tobytes()
    sel = oracle_lib.select_uniform_kpts_by_grid(ref, img.shape[0], img.shape[1], 2000, 16, 8)
    kps = [cv2.KeyPoint(float(k["x"]), float(k["y"]), float(k["size"]), float(k["angle"]), float(k["response"]),
                        int(k["octave"]), int(k["class_id"])) for k in sel]
    kps2, dref = cv2.ORB_create(8000, 1.2, 4).compute(img, kps)
    assert len(kps2) == len(sel)
    assert np.array_equal(oo.compute(img, sel), dref)


@pytest.mark.skipif(not have_cv2(), reason="cv2 not importable")
def test_oracle_stages_vs_cv2():
    import cv2
    g = mvo_synth.rect_scene(3)
    bgr = mvo_synth.color_scene(2)
    assert np.array_equal(oo.bgr_to_gray(bgr), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY))
    lv = oo.build_pyramid(g)
    prev = g
    for l in range(1, 4):
        prev = cv2.resize(prev, (lv[l].shape[1], lv[l].shape[0]), interpolation=cv2.INTER_LINEAR_EXACT)
        assert np.array_equal(prev, lv[l])
    fast = cv2.FastFeatureDetector_create(20, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16).detect(g, None)
    xs, ys, sc = oo.fast_detect(g, 20)
    assert [(int(k.pt[0]), int(k.pt[1]), int(k.response)) for k in fast] == list(zip(xs.tolist(), ys.tolist(), sc.tolist()))
    for y, x in [(3.0, 4.0), (-1.0, 2.0), (0.0, -5.0), (7.0, 0.0), (-3.0, -3.0), (1e-3, 250.0)]:
        assert oo.fast_atan2(y, x) == np.float32(cv2.fastAtan2(y, x))


def test_oracle_vs_golden():
    for name in ("rect0", "color1"):
        g = np.load(GOLDEN / f"orb_{name}.npz")
        img = SCENES[name]()
        assert np.array_equal(img, g["image"])
        kp = oo.detect(img)
        assert kp.tobytes() == g["detect"].tobytes()
        sel = oracle_lib.select_uniform_kpts_by_grid(kp, img.shape[0], img.shape[1], 2000, 16, 8)
        assert sel.tobytes() == g["selected"].tobytes()
        assert np.array_equal(oo.compute(img, sel), g["descriptors"])


def test_level_geometry():
    assert oo.level_sizes(640, 480, 4, 1.2) == [(640, 480), (533, 400), (444, 333), (370, 278)]
    assert oo.features_per_level(8000, 4, 1.2) == [2575, 2146, 1788, 1491]
    # cv::ORB sizes a level as cvRound(rows * (1.0f / scale)): 153 * 0.8333333f rounds to 127.5f, hence 128 (153 / 1.2f gives 127)
    assert oo.level_sizes(201, 153, 4, 1.2) == [(201, 153), (168, 128), (140, 106), (116, 89)]


@pytest.mark.skipif(not have_cv2(), reason="cv2 not importable")
def test_oracle_level_sizes_vs_cv2():
    """Image heights whose level sizes depend on multiplying by the inverse scale rather than dividing by it: detection equal to cv2."""
    import cv2
    for w, h in ((201, 153), (200, 153), (202, 153)):
        img = mvo_synth.gray_to_bgr(mvo_synth.rect_scene(36, w, h, n_rect=150))
        ref = _cvkp(cv2.ORB_create(8000, 1.2, 4, 31, 0, 2, cv2.ORB_HARRIS_SCORE, 31, 20).detect(img, None))
        assert oo.detect(img).tobytes() == ref.tobytes(), (w, h)


# ---- the parameter space of tests/orb_cases.py ----------------------------------------------------------------------------------
def _param_sets():
    """Every parameter set of the cases the library accepts, with an image small enough for the numpy oracle: the case's own image
    where it is small, else a rectangle scene of the smallest of a few sizes the parameters accept."""
    import orb_cases as O
    out = {}
    for c in O.CASES:
        if c["err"] is not None:
            continue
        key = tuple(sorted(c["p"].items()))
        if key in out:
            continue
        if c["tier"] == "both":
            out[key] = (c["name"], c["p"], c["img"])
            continue
        for w, h in ((256, 200), (320, 240), (420, 330)):
            if "err" not in O.plan(h, w, c["p"]):
                out[key] = (c["name"], c["p"], lambda w=w, h=h: mvo_synth.rect_scene(60, w, h, n_rect=w * h // 205))
                break
    return list(out.values())


PARAM_SETS = _param_sets()


@pytest.mark.skipif(not have_cv2(), reason="cv2 not importable")
@pytest.mark.parametrize("name,p,img", PARAM_SETS, ids=[s[0] for s in PARAM_SETS])
def test_oracle_vs_cv2_at_case_parameters(name, p, img):
    """The oracle the emulated tier compares against equals cv2 at every non-default parameter set the GPU cases use: detection
    (incl. the per-level FAST candidate counts that decide the retainBest path), the grid selection's input and the descriptors."""
    import orb_cases as O
    im = img()
    sel, desc, counts = O.reference_cv2(im, p)
    osel, odesc, ocounts = O.reference_oracle(im, p)
    assert ocounts == counts
    assert osel.tobytes() == sel.tobytes()
    assert np.array_equal(odesc, desc)


def test_oracle_vs_parameter_goldens():
    """The committed cv2 output at non-default parameters (tests/golden/orb_params.npz) against the oracle: the GPU tier's reference
    where cv2 cannot be imported."""
    import orb_cases as O
    g = np.load(GOLDEN / "orb_params.npz")
    names = sorted({k.split("/")[0] for k in g.files if "/" in k})
    assert len(names) >= 6
    for n in names:
        c = O.CASE[n]
        assert np.array_equal(O.image(c), g[f"{n}/image"]), n
        sel, desc, counts = O.reference_oracle(g[f"{n}/image"], c["p"])
        assert sel.tobytes() == g[f"{n}/selected"].tobytes(), n
        assert np.array_equal(desc, g[f"{n}/descriptors"]), n
        assert counts == list(g[f"{n}/counts"]), n
        assert O.expected_path(counts, O.case_plan(c)["caps"]) == c["path"], n


def test_grid_selection_skips_the_uncovered_strip():
    """selectUniformKptsByGrid (feature_match.cpp:51-84) with keypoints right of / below the last whole cell, which the reference
    indexes out of range: the oracle skips them (no keep, no quota), the project's reading that the library's device and host
    paths share."""
    rng = np.random.default_rng(11)
    rows, cols, grid, mpc, cap = 500, 630, 64, 3, 60
    kp = np.zeros(3000, oo.KEYPOINT_DTYPE)
    kp["x"] = rng.uniform(31, cols - 31, 3000).astype(np.float32)
    kp["y"] = rng.uniform(31, rows - 31, 3000).astype(np.float32)
    gr, gc = rows // grid, cols // grid
    cnt, keep = {}, []
    for i, (x, y) in enumerate(zip(kp["x"].tolist(), kp["y"].tolist())):
        r, c = int(y) // grid, int(x) // grid
        if r >= gr or c >= gc:
            continue
        if cnt.get((r, c), 0) < mpc:
            keep.append(i)
            cnt[(r, c)] = cnt.get((r, c), 0) + 1
            if len(keep) > cap:
                break
    got = oracle_lib.select_uniform_kpts_by_grid(kp, rows, cols, cap, grid, mpc)
    assert got.tobytes() == kp[keep].tobytes() and len(got) == cap + 1
    assert np.all((got["x"] < gc * grid) & (got["y"] < gr * grid))
    assert np.any((kp["x"] >= gc * grid) | (kp["y"] >= gr * grid))
