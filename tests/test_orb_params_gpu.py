"""ORB extraction on the H100 over its parameter and image-geometry space (tests/orb_cases.py): every case bit-exact with cv2 live
(cv::ORB at the case's nfeatures, scale factor, levels and threshold + the reference's grid selection), or with the committed
goldens (tests/golden/orb_params.npz) where cv2 cannot be imported, through mvo_orb_extract and mvo_calc_keypoints +
mvo_calc_descriptors; rejected configurations return their error code twice on the same context; batches through
mvo_orb_extract_batch_dev mix the three retainBest paths, grow from 4 to 8 frames, shrink to 1, and change geometry and parameters
between calls.  All cases share one context, so every case also follows a plan built for another geometry or other parameters."""
import ctypes as C

import numpy as np
import pytest
from conftest import GOLDEN, have_cv2

import orb_cases as O

pytestmark = pytest.mark.gpu

GPU_CASES = [c["name"] for c in O.CASES]


def _goldens():
    path = GOLDEN / "orb_params.npz"
    if not path.exists():
        return {}
    g = np.load(path)
    return {n: (g[f"{n}/selected"], g[f"{n}/descriptors"], list(g[f"{n}/counts"])) for n in {k.split("/")[0] for k in g.files}}


@pytest.fixture(scope="module")
def lib_ctx(built):
    import mvo_b200
    ctx = mvo_b200.Context(0)
    yield O.bind(mvo_b200.load_library()), ctx.h
    ctx.close()


@pytest.fixture(scope="module")
def reference():
    if have_cv2():
        return lambda name, img, p: O.reference_cv2(img, p)
    gold = _goldens()
    return lambda name, img, p: gold[name] if name in gold else pytest.skip("cv2 not importable and no golden for this case")


@pytest.mark.parametrize("name", GPU_CASES)
def test_case_matches_cv2(lib_ctx, reference, name):
    lib, h = lib_ctx
    c = O.CASE[name]
    r = O.run(lib, h, c)
    O.check(c, r, None if c["err"] is not None else reference(name, O.image(c), c["p"]))


def test_grid_selection_skips_keypoints_outside_the_grid(lib_ctx):
    O.check_grid_rank_outside(*lib_ctx)


def test_batches_grow_shrink_and_replan(lib_ctx, reference):
    import torch
    lib, h = lib_ctx
    frames, paths = O.batch_frames()
    p = O.BATCH_PARAMS
    refs = [reference(None, f, p) for f in frames]
    other = O.CASE["nl3_sf1.5_517x389"]

    def batch(fr, cap, check_paths, check_refs, params):
        B = len(fr)
        d_img = torch.from_numpy(np.ascontiguousarray(np.stack(fr))).cuda()
        d_kp = torch.zeros(B * cap * 28, dtype=torch.uint8, device="cuda")
        d_desc = torch.zeros(B * cap * 32, dtype=torch.uint8, device="cuda")
        d_cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        read = lambda: (torch.cuda.synchronize(), d_kp.cpu().numpy(), d_desc.cpu().numpy(), d_cnt.cpu().numpy())[1:]
        got = O.batch_run(lib, h, fr, d_img.data_ptr(), d_kp.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), cap, read)
        O.check_batch(fr, check_paths, got, check_refs, params)

    cap = p["max_keypoints"] + 1
    O.set_params(lib, h, p)
    batch(frames, cap, paths, refs, p)                                   # ovf0, retain, host and ovf0 in one batch
    batch(frames + frames[::-1], cap, paths + paths[::-1], refs + refs[::-1], p)     # the workspace grows: the planes move
    batch(frames[1:2], cap, paths[1:2], refs[1:2], p)                    # one frame in the workspace carved for eight
    oimg, op = O.image(other), other["p"]
    O.set_params(lib, h, op)                                             # other geometry and parameters
    oref = reference(other["name"], oimg, op)
    batch([oimg, oimg], op.get("max_keypoints", 1500) + 1, [other["path"]] * 2, [oref] * 2, op)
    O.set_params(lib, h, p)                                              # and back
    batch(frames[2:], cap, paths[2:], refs[2:], p)
