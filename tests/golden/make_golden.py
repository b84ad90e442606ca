"""Generates the committed golden vectors from the third-party code the reference calls
(OpenCV, via the cv2 4.13 wheel in this container).  Run from the repo root:
    python tests/golden/make_golden.py [match|orb|pnp|all]
The reference ships no fixtures of its own (SURVEY.md §4); these pin the oracle."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT / "monocular-visual-odometry_b200" / "python"))
sys.path.insert(0, str(ROOT))
OUT = Path(__file__).resolve().parent


def make_match():
    import cv2
    import mvo_synth
    d1 = mvo_synth.random_descriptors(101, 211, dup_every=9)
    d2 = mvo_synth.random_descriptors(102, 197, dup_every=6)
    d1[::4] = d2[(np.arange(0, 211, 4) * 5) % 197]
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    nn = bf.match(d1, d2)
    kn = bf.knnMatch(d1, d2, k=2)
    np.savez_compressed(OUT / "match_golden.npz", d1=d1, d2=d2,
                        nn_train=np.array([m.trainIdx for m in nn], np.int32),
                        nn_dist=np.array([m.distance for m in nn], np.float32),
                        knn_train=np.array([[m.trainIdx for m in mm] for mm in kn], np.int32),
                        knn_dist=np.array([[m.distance for m in mm] for mm in kn], np.float32),
                        cv_version=cv2.__version__)


def make_orb():
    """cv::ORB detect (feature_match.cpp:22-23,34) -> selectUniformKptsByGrid restatement -> compute (:45,48)."""
    import cv2
    import mvo_synth
    from oracle import oracle_lib
    scenes = {"rect0": mvo_synth.gray_to_bgr(mvo_synth.rect_scene(0)), "color1": mvo_synth.color_scene(1),
              "noise0": mvo_synth.gray_to_bgr(mvo_synth.noise_scene(0))}
    for name, img in scenes.items():
        kps = cv2.ORB_create(8000, 1.2, 4, 31, 0, 2, cv2.ORB_HARRIS_SCORE, 31, 20).detect(img, None)
        det = np.array([(k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, k.class_id) for k in kps],
                       oracle_lib.KEYPOINT_DTYPE)
        sel = oracle_lib.select_uniform_kpts_by_grid(det, img.shape[0], img.shape[1], 2000, 16, 8)
        ck = [cv2.KeyPoint(float(k["x"]), float(k["y"]), float(k["size"]), float(k["angle"]), float(k["response"]),
                           int(k["octave"]), int(k["class_id"])) for k in sel]
        ck2, desc = cv2.ORB_create(8000, 1.2, 4).compute(img, ck)
        assert len(ck2) == len(sel)
        extra = {} if name == "noise0" else {"image": img}      # the noise image is regenerated from its seed
        np.savez_compressed(OUT / f"orb_{name}.npz", detect=det, selected=sel, descriptors=desc,
                            cv_version=cv2.__version__, **extra)


# small cases of tests/orb_cases.py at non-default parameters: one level, three at 1.5, eight at 1.2, both sides of the packed /
# scalar FAST threshold switch, the highest threshold, and a 64-px grid with keypoints in the uncovered strip on the retainBest path
ORB_PARAM_GOLDENS = ["nl1_200x152", "nl3_sf1.5_203x161", "nl8_sf1.2_256x240", "t127_dots", "t128_dots", "t254_dots",
                     "grid64_strip_250x200_retain"]


def make_orb_params():
    """cv::ORB at the parameters of ORB_PARAM_GOLDENS -> selectUniformKptsByGrid restatement -> compute: orb_params.npz holds
    <case>/image, /selected, /descriptors and /counts (FAST candidates inside the border per level)."""
    import cv2
    sys.path.insert(0, str(ROOT / "tests"))
    import orb_cases as O
    out = {}
    for name in ORB_PARAM_GOLDENS:
        c = O.CASE[name]
        img = O.image(c)
        sel, desc, counts = O.reference_cv2(img, c["p"])
        out.update({f"{name}/image": img, f"{name}/selected": sel, f"{name}/descriptors": desc,
                    f"{name}/counts": np.array(counts, np.int32)})
    np.savez_compressed(OUT / "orb_params.npz", cv_version=cv2.__version__, **out)


def make_pnp():
    """cv::solvePnPRansac exactly as called at src/vo/vo.cpp:318-320 on the config-3 instance."""
    import cv2
    import mvo_synth
    P, uv, rvec_true, tvec_true, is_out = mvo_synth.pnp_problem(0)
    K = mvo_synth.K_DEFAULT
    ok, rvec, tvec, inl = cv2.solvePnPRansac(P, uv, K, None, None, None, False, 100, 2.0, 0.999)
    assert ok
    inl = inl.ravel().astype(np.int32)
    ok2, r2, t2 = cv2.solvePnP(P[inl], uv[inl], K, None, flags=cv2.SOLVEPNP_ITERATIVE)
    np.savez_compressed(OUT / "pnp_config3.npz", P=P, uv=uv, K=K, rvec=rvec.ravel(), tvec=tvec.ravel(), inliers=inl,
                        rvec_refit=r2.ravel(), tvec_refit=t2.ravel(), rvec_true=rvec_true, tvec_true=tvec_true,
                        cv_version=cv2.__version__)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what in ("match", "all"):
        make_match()
    if what in ("orb", "all") and "make_orb" in globals():
        make_orb()
    if what in ("orb", "all"):
        make_orb_params()
    if what in ("pnp", "all") and "make_pnp" in globals():
        make_pnp()
