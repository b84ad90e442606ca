"""ctypes binding of libmvo.so (include/mvo.h) — test/bench harness only.

The product is the C ABI; this file is the thinnest possible Python view of it so that
pytest and bench.py can drive the library with numpy (host) buffers or raw device pointers
(``tensor.data_ptr()``).  There is NO fallback: if libmvo.so is missing or no H100 is
visible, loading / ``Context()`` raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

_PKG_DIR = Path(__file__).resolve().parent.parent
LIB_PATH = Path(os.environ.get("MVO_LIB", _PKG_DIR / "libmvo.so"))

KEYPOINT_DTYPE = np.dtype(
    [("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
     ("octave", "<i4"), ("class_id", "<i4")], align=False)
DMATCH_DTYPE = np.dtype(
    [("query_idx", "<i4"), ("train_idx", "<i4"), ("img_idx", "<i4"), ("distance", "<f4")])
assert KEYPOINT_DTYPE.itemsize == 28 and DMATCH_DTYPE.itemsize == 16
# mvo_two_view_result (esti_motion_by_essential_batch_dev): one record per frame pair
TWO_VIEW_RESULT_DTYPE = np.dtype(
    [("status", "<i4"), ("n_matches", "<i4"), ("n_inliers", "<i4"), ("votes", "<i4"), ("E", "<f8", (9,)), ("R", "<f8", (9,)),
     ("t", "<f8", (3,))])
assert TWO_VIEW_RESULT_DTYPE.itemsize == 184
# mvo_relative_poses_result (estimate_relative_poses_batch_dev): status, n_matches, then mvo_two_view_solutions as it is laid out
# in memory (TwoViewSolutions below)
RELATIVE_POSES_RESULT_DTYPE = np.dtype(
    [("status", "<i4"), ("n_matches", "<i4"), ("num_solutions", "<i4"), ("best", "<i4"), ("n_inliers", "<i4", (5,)), ("pad_", "<i4"),
     ("R", "<f8", (5, 9)), ("t", "<f8", (5, 3)), ("normal", "<f8", (5, 3)), ("E", "<f8", (9,)), ("H", "<f8", (9,)), ("score_e", "<f8"),
     ("score_h", "<f8"), ("ratio", "<f8")])
assert RELATIVE_POSES_RESULT_DTYPE.itemsize == 808
# mvo_init_candidate_result (vo_init_candidates_batch_dev): one record per frame pair
INIT_CANDIDATE_RESULT_DTYPE = np.dtype(
    [("status", "<i4"), ("usable", "<i4"), ("good", "<i4"), ("best_sol", "<i4"), ("n_inliers", "<i4"), ("n_kept", "<i4"),
     ("normalized", "<i4"), ("pad", "<i4"), ("scale", "<f8"), ("mean_pixel_dist", "<f8"), ("median_angle", "<f8"),
     ("t_curr_to_prev", "<f8", (3,)), ("T_w_c", "<f8", (16,))])
assert INIT_CANDIDATE_RESULT_DTYPE.itemsize == 208
# mvo_keyframe_points_result (vo_keyframe_points_batch_dev): one record per frame pair
KEYFRAME_POINTS_RESULT_DTYPE = np.dtype(
    [("status", "<i4"), ("usable", "<i4"), ("n_matches", "<i4"), ("n_inliers", "<i4"), ("n_kept", "<i4"), ("pad", "<i4"),
     ("median_angle", "<f8"), ("R_curr_to_prev", "<f8", (9,)), ("t_curr_to_prev", "<f8", (3,))])
assert KEYFRAME_POINTS_RESULT_DTYPE.itemsize == 128
# mvo_map_matches_result (vo_map_matches_batch_dev): one record per (frame, guess pose) job
MAP_MATCHES_RESULT_DTYPE = np.dtype([("status", "<i4"), ("n_candidates", "<i4"), ("n_matches", "<i4"), ("pad", "<i4")])
assert MAP_MATCHES_RESULT_DTYPE.itemsize == 16
# mvo_vo_pnp_result (vo_pnp_batch_dev): one record per map-matches job
VO_PNP_RESULT_DTYPE = np.dtype(
    [("status", "<i4"), ("pnp_ok", "<i4"), ("n_matches", "<i4"), ("n_inliers", "<i4"), ("best", "<i4"), ("pad", "<i4", (3,)),
     ("Rt", "<f8", (12,)), ("T_w_c", "<f8", (16,))])
assert VO_PNP_RESULT_DTYPE.itemsize == 256

MVO_OK = 0
ERR_NAMES = {0: "MVO_OK", -1: "MVO_ERR_INVALID_ARG", -2: "MVO_ERR_NO_DEVICE", -3: "MVO_ERR_CUDA",
             -4: "MVO_ERR_CAPACITY", -5: "MVO_ERR_UNSUPPORTED", -6: "MVO_ERR_DEGENERATE"}


class Params(C.Structure):
    _fields_ = [
        ("orb_nfeatures", C.c_int32), ("orb_scale_factor", C.c_float), ("orb_nlevels", C.c_int32),
        ("orb_fast_threshold", C.c_int32), ("max_keypoints", C.c_int32), ("grid_size", C.c_int32),
        ("max_pts_per_grid", C.c_int32), ("xiang_gao_ratio", C.c_double), ("lowe_ratio", C.c_double),
        ("pnp_hypotheses", C.c_int32), ("pnp_reproj_error", C.c_float), ("pnp_seed", C.c_uint64),
        ("pnp_refine_iters", C.c_int32), ("ba_iterations", C.c_int32), ("ba_huber_delta", C.c_double),
        ("ba_fix_first_pose", C.c_int32), ("ba_step_tol", C.c_double), ("epi_hypotheses", C.c_int32), ("pnp_mode", C.c_int32), ("eh_ratio_threshold", C.c_double),
        ("essential_threshold", C.c_double), ("homography_threshold", C.c_double),
    ]


class TrackParams(C.Structure):
    _fields_ = [("match_method", C.c_int32), ("match_radius", C.c_float), ("min_pnp_points", C.c_int32),
                ("max_dist_to_prev", C.c_double), ("min_dist_keyframe", C.c_double), ("ba_enable", C.c_int32),
                ("ba_window", C.c_int32), ("ba_fix_points", C.c_int32), ("information", C.c_double * 4),
                ("buffer_size", C.c_int32), ("ba_step_tol", C.c_double), ("device_resident", C.c_int32),
                ("pad", C.c_int32)]


class TrackResult(C.Structure):
    _fields_ = [("n_keypoints", C.c_int32), ("n_candidates", C.c_int32), ("n_matches", C.c_int32),
                ("n_inliers", C.c_int32), ("pnp_ok", C.c_int32), ("ba_frames", C.c_int32), ("ba_edges", C.c_int32),
                ("pad", C.c_int32), ("T_w_c_pnp", C.c_double * 16)]


class TwoViewSolutions(C.Structure):
    _fields_ = [("num_solutions", C.c_int32), ("best", C.c_int32), ("n_inliers", C.c_int32 * 5), ("pad_", C.c_int32),
                ("R", (C.c_double * 9) * 5), ("t", (C.c_double * 3) * 5), ("normal", (C.c_double * 3) * 5),
                ("E", C.c_double * 9), ("H", C.c_double * 9), ("score_e", C.c_double), ("score_h", C.c_double), ("ratio", C.c_double)]


class VoParams(C.Structure):
    _fields_ = [("track", TrackParams), ("match_method_init", C.c_int32), ("max_match_dist_init", C.c_float),
                ("max_match_dist_triangulation", C.c_float), ("init_calc_homography", C.c_int32),
                ("min_inlier_matches", C.c_int32), ("pad", C.c_int32), ("essential_threshold", C.c_double),
                ("min_triang_angle", C.c_double), ("max_ratio_angle_to_median", C.c_double), ("min_pixel_dist", C.c_double),
                ("min_median_triangulation_angle", C.c_double), ("assumed_mean_depth_init", C.c_double)]


class VoFrameInfo(C.Structure):
    _fields_ = [("frame_id", C.c_int32), ("state_in", C.c_int32), ("state_out", C.c_int32), ("keyframe", C.c_int32),
                ("n_keypoints", C.c_int32), ("n_matches", C.c_int32), ("n_candidates", C.c_int32), ("n_inliers", C.c_int32),
                ("pnp_ok", C.c_int32), ("ba_frames", C.c_int32), ("ba_edges", C.c_int32), ("best_sol", C.c_int32),
                ("map_points", C.c_int32), ("kf_matches", C.c_int32), ("kf_new_points", C.c_int32), ("pad", C.c_int32),
                ("score_e", C.c_double), ("score_h", C.c_double), ("eh_ratio", C.c_double),
                ("init_mean_pixel_dist", C.c_double), ("init_median_angle", C.c_double), ("T_w_c_pnp", C.c_double * 16)]


class MvoError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"{ERR_NAMES.get(code, code)}: {msg}")
        self.code = code


# Every exported symbol of include/mvo.h with its signature (also used by the CPU-side
# "library loads and exports everything" test).
_vp, _i, _sz, _f = C.c_void_p, C.c_int, C.c_size_t, C.c_float
_pi = C.POINTER(C.c_int)
SIGNATURES = {
    "mvo_default_params": (None, [C.POINTER(Params)]),
    "mvo_create": (_i, [C.POINTER(_vp), _i, C.POINTER(Params)]),
    "mvo_destroy": (None, [_vp]),
    "mvo_last_error": (C.c_char_p, [_vp]),
    "mvo_get_params": (_i, [_vp, C.POINTER(Params)]),
    "mvo_set_params": (_i, [_vp, C.POINTER(Params)]),
    "mvo_set_stream": (_i, [_vp, _vp]),
    "mvo_synchronize": (_i, [_vp]),
    "mvo_kernel_launches": (C.c_uint64, [_vp]),
    "mvo_calc_keypoints": (_i, [_vp, _vp, _i, _i, _i, _sz, _vp, _pi]),
    "mvo_calc_descriptors": (_i, [_vp, _vp, _i, _i, _i, _sz, _vp, _i, _vp]),
    "mvo_orb_extract": (_i, [_vp, _vp, _i, _i, _i, _sz, _vp, _pi, _vp]),
    "mvo_select_uniform_kpts_by_grid": (_i, [_vp, _vp, _pi, _i, _i]),
    "mvo_orb_extract_batch_dev": (_i, [_vp, _vp, _i, _i, _i, _i, _sz, _sz, _vp, _vp, _vp, _i]),
    "mvo_match_features_batch_dev": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _i, _i, _f, _vp, _vp]),
    "mvo_esti_motion_by_essential_batch_dev": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, C.c_double, _vp, _vp, _vp]),
    "mvo_estimate_relative_poses_batch_dev": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "mvo_match_hamming_nn": (_i, [_vp, _vp, _i, _vp, _i, _vp]),
    "mvo_match_hamming_knn2": (_i, [_vp, _vp, _i, _vp, _i, _vp]),
    "mvo_match_radius_sad": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _f, _vp, _pi]),
    "mvo_match_features": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _vp, _f, _vp, _pi]),
    "mvo_remove_duplicated_matches": (_i, [_vp, _pi]),
    "mvo_match_dev": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _i, _f, _vp]),
    "mvo_solve_pnp_ransac": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _pi]),
    "mvo_pnp_last_hypotheses": (_i, [_vp, _vp, _vp, _i, _pi]),
    "mvo_pnp_refine": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "mvo_bundle_adjustment": (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _vp]),
    "mvo_optimize_single_frame": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _i]),
    "mvo_default_track_params": (None, [C.POINTER(TrackParams)]),
    "mvo_tracker_create": (_i, [_vp, _vp, _i, _i, C.POINTER(TrackParams), C.POINTER(_vp)]),
    "mvo_tracker_destroy": (None, [_vp]),
    "mvo_tracker_set_map": (_i, [_vp, _vp, _vp, _i]),
    "mvo_tracker_reset": (_i, [_vp, _vp]),
    "mvo_tracker_track": (_i, [_vp, _vp, _i, _sz, _i, _vp, C.POINTER(TrackResult)]),
    "mvo_tracker_frame_pose": (_i, [_vp, _i, _vp]),
    "mvo_tracker_prefetch": (_i, [_vp, _vp, _i, _sz, _i]),
    "mvo_tracker_timing_enable": (_i, [_vp, C.c_uint32]),
    "mvo_tracker_timing_read": (_i, [_vp, _vp, _vp]),
    "mvo_tracker_kernel_launches": (C.c_uint64, [_vp]),
    "mvo_kernel_classes": (_i, []),
    "mvo_kernel_name": (C.c_char_p, [_i]),
    "mvo_timing_enable": (_i, [_vp, C.c_uint32]),
    "mvo_timing_read": (_i, [_vp, _vp, _vp]),
    "mvo_esti_motion_by_essential": (_i, [_vp, _vp, _vp, _i, _vp, C.c_double, _vp, _vp, _vp, _vp, _pi]),
    "mvo_do_triangulation": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp]),
    "mvo_esti_motion_by_homography": (_i, [_vp, _vp, _vp, _i, _vp, C.c_double, _vp, _vp, _vp, _vp, _pi, _vp, _pi]),
    "mvo_remove_wrong_rt_of_homography": (_i, [_vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _pi]),
    "mvo_estimate_relative_poses": (_i, [_vp, _vp, _vp, _i, _vp, _i, _i, C.POINTER(TwoViewSolutions), _vp, _vp]),
    "mvo_check_essential_score": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _pi, C.c_double, C.POINTER(C.c_double)]),
    "mvo_check_homography_score": (_i, [_vp, _vp, _vp, _i, _vp, _pi, C.c_double, C.POINTER(C.c_double)]),
    "mvo_choose_e_or_h_thr": (_i, [C.c_double, C.c_double, _vp, _i, C.c_double, _pi, C.POINTER(C.c_double)]),
    "mvo_choose_e_or_h": (_i, [C.c_double, C.c_double, _vp, _i, _pi, C.POINTER(C.c_double)]),
    "mvo_retain_good_triangulation": (_i, [_vp, _i, _vp, _vp, C.c_double, C.c_double, _vp, _vp, _pi]),
    "mvo_normalize_init_depth": (_i, [_vp, _i, _vp, C.c_double, C.POINTER(C.c_double)]),
    "mvo_is_vo_good_to_init": (_i, [_vp, _vp, _i, _vp, _i, _i, C.c_double, C.c_double, _pi, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "mvo_check_large_move": (_i, [_vp, _vp, C.c_double, _pi, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "mvo_vo_default_params": (None, [C.POINTER(VoParams)]),
    "mvo_vo_create": (_i, [_vp, _vp, _i, _i, C.POINTER(VoParams), C.POINTER(_vp)]),
    "mvo_vo_destroy": (None, [_vp]),
    "mvo_vo_add_frame": (_i, [_vp, _vp, _i, _sz, _vp, C.POINTER(VoFrameInfo)]),
    "mvo_vo_is_initialized": (_i, [_vp]),
    "mvo_vo_map_size": (_i, [_vp]),
    "mvo_vo_num_keyframes": (_i, [_vp]),
    "mvo_vo_add_frame_ex": (_i, [_vp, _vp, _i, _sz, _i, _vp, C.POINTER(VoFrameInfo)]),
    "mvo_vo_prefetch": (_i, [_vp, _vp, _i, _sz, _i]),
    "mvo_vo_run_sequence": (_i, [_vp, _vp, _i, _i, _sz, _i, _vp, _vp, _vp]),
    "mvo_vo_device_resident": (_i, [_vp]),
    "mvo_vo_reset": (_i, [_vp]),
    "mvo_vo_kernel_launches": (C.c_uint64, [_vp]),
    "mvo_vo_timing_enable": (_i, [_vp, C.c_uint32]),
    "mvo_vo_timing_read": (_i, [_vp, _vp, _vp]),
    "mvo_vo_get_map": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _pi]),
    "mvo_vo_frame_pose": (_i, [_vp, _i, _vp]),
    "mvo_vo_frame_data": (_i, [_vp, _i, _i, _vp, _i, _pi]),
    "mvo_vo_init_candidates_batch_dev": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(VoParams), _vp, _vp, _vp,
                                              _vp]),
    "mvo_vo_keyframe_points_batch_dev": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(VoParams), _vp, _vp,
                                              _vp, _vp, _vp, _vp]),
    "mvo_vo_map_matches_batch_dev": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _vp, _vp, _i, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _vp,
                                          _vp, _vp]),
    "mvo_vo_pnp_batch_dev": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, C.POINTER(TrackParams), _vp, _vp, _vp]),
    "mvo_vo_has_keyframe": (_i, [_vp, _i]),
    "mvo_write_pose_file": (_i, [C.c_char_p, _vp, _i]),
    "mvo_read_pose_file": (_i, [C.c_char_p, _vp, _i, _pi]),
    "mvo_image_path": (_i, [C.c_char_p, C.c_char_p, _i, C.c_char_p, _sz]),
    "mvo_config_load": (_i, [C.c_char_p, C.POINTER(_vp)]),
    "mvo_config_free": (None, [_vp]),
    "mvo_config_get_string": (_i, [_vp, C.c_char_p, C.c_char_p, _sz]),
    "mvo_config_get_double": (_i, [_vp, C.c_char_p, C.POINTER(C.c_double)]),
    "mvo_config_get_int": (_i, [_vp, C.c_char_p, _pi]),
    "mvo_config_get_bool": (_i, [_vp, C.c_char_p, _pi]),
    "mvo_config_apply": (_i, [_vp, C.POINTER(Params), C.POINTER(TrackParams), _vp]),
    "mvo_config_apply_vo": (_i, [_vp, C.POINTER(VoParams)]),
}

_lib = None


def load_library():
    """dlopen libmvo.so and attach signatures.  Raises if the library is not built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise FileNotFoundError(
                f"{LIB_PATH} not built — run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(no CPU fallback exists)")
        lib = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def default_params() -> Params:
    p = Params()
    load_library().mvo_default_params(C.byref(p))
    return p


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return C.c_void_p(a.ctypes.data)


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


class Context:
    """One mvo_ctx (one GPU, one stream)."""

    def __init__(self, device: int = 0, params: Params | None = None, **overrides):
        self.lib = load_library()
        p = params or default_params()
        for k, v in overrides.items():
            if not hasattr(p, k):
                raise AttributeError(k)
            setattr(p, k, v)
        h = C.c_void_p()
        rc = self.lib.mvo_create(C.byref(h), device, C.byref(p))
        if rc != MVO_OK:
            raise MvoError(rc, "mvo_create failed (no usable sm_90 GPU? this library has no CPU path)")
        self.h = h
        self.params = p

    def close(self):
        if getattr(self, "h", None):
            self.lib.mvo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc != MVO_OK:
            raise MvoError(rc, self.lib.mvo_last_error(self.h).decode())

    def set_params(self, **kw):
        for k, v in kw.items():
            setattr(self.params, k, v)
        self._chk(self.lib.mvo_set_params(self.h, C.byref(self.params)))

    def set_stream(self, cuda_stream: int):
        self._chk(self.lib.mvo_set_stream(self.h, C.c_void_p(cuda_stream)))

    def synchronize(self):
        self._chk(self.lib.mvo_synchronize(self.h))

    @property
    def kernel_launches(self) -> int:
        return int(self.lib.mvo_kernel_launches(self.h))

    # ---- ORB ---------------------------------------------------------------------------
    @staticmethod
    def _img(image):
        img = np.ascontiguousarray(image, dtype=np.uint8)
        if img.ndim == 2:
            img = img[:, :, None]
        rows, cols, ch = img.shape
        return img, rows, cols, ch

    def calc_keypoints(self, image, cap: int = 16384):
        img, rows, cols, ch = self._img(image)
        kp = np.zeros(cap, KEYPOINT_DTYPE)
        n = C.c_int(cap)
        self._chk(self.lib.mvo_calc_keypoints(self.h, _ptr(img), rows, cols, ch, cols * ch, _ptr(kp), C.byref(n)))
        return kp[: n.value].copy()

    def calc_descriptors(self, image, kpts):
        img, rows, cols, ch = self._img(image)
        kp = _c(kpts, KEYPOINT_DTYPE)
        desc = np.zeros((len(kp), 32), np.uint8)
        self._chk(self.lib.mvo_calc_descriptors(self.h, _ptr(img), rows, cols, ch, cols * ch, _ptr(kp), len(kp), _ptr(desc)))
        return desc

    def orb_extract(self, image, cap: int = 16384):
        img, rows, cols, ch = self._img(image)
        kp = np.zeros(cap, KEYPOINT_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(cap)
        self._chk(self.lib.mvo_orb_extract(self.h, _ptr(img), rows, cols, ch, cols * ch, _ptr(kp), C.byref(n), _ptr(desc)))
        return kp[: n.value].copy(), desc[: n.value].copy()

    def select_uniform_kpts_by_grid(self, kpts, rows, cols):
        kp = _c(kpts, KEYPOINT_DTYPE).copy()
        n = C.c_int(len(kp))
        self._chk(self.lib.mvo_select_uniform_kpts_by_grid(self.h, _ptr(kp), C.byref(n), rows, cols))
        return kp[: n.value].copy()

    def orb_extract_batch_dev(self, d_images, batch, rows, cols, ch, stride, frame_stride, d_kpts, d_desc, d_counts, cap):
        self._chk(self.lib.mvo_orb_extract_batch_dev(self.h, _ptr(d_images), batch, rows, cols, ch, stride,
                                                     frame_stride, _ptr(d_kpts), _ptr(d_desc), _ptr(d_counts), cap))

    def match_features_batch_dev(self, d_kpts, d_desc, d_counts, batch, cap, d_pairs, n_pairs, method_index, radius, d_out, d_n_out):
        """matchFeatures for n_pairs (query frame, train frame) pairs of an orb_extract_batch_dev output, all device pointers;
        pair p's matches land at d_out + p * cap records, their count (or MVO_ERR_INVALID_ARG for a bad pair) in d_n_out[p]."""
        self._chk(self.lib.mvo_match_features_batch_dev(self.h, _ptr(d_kpts), _ptr(d_desc), _ptr(d_counts), batch, cap, _ptr(d_pairs),
                                                        n_pairs, method_index, C.c_float(radius), _ptr(d_out), _ptr(d_n_out)))

    def esti_motion_by_essential_batch_dev(self, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, K, threshold,
                                           d_res, d_inliers, d_pts3d=None):
        """estiMotionByEssential (+ doTriangulation when d_pts3d is given) for n_pairs matched frame pairs of a batched
        extraction, all device pointers except K (host 3x3): pair p's TWO_VIEW_RESULT_DTYPE record in d_res[p], its inlier
        indices at d_inliers + p * cap, its triangulated inliers at d_pts3d + p * cap * 3."""
        K = _c(K, np.float64)
        self._chk(self.lib.mvo_esti_motion_by_essential_batch_dev(self.h, _ptr(d_kpts), _ptr(d_counts), batch, cap, _ptr(d_pairs), n_pairs,
                                                                  _ptr(d_matches), _ptr(d_n_matches), _ptr(K), float(threshold), _ptr(d_res),
                                                                  _ptr(d_inliers), _ptr(d_pts3d)))

    def estimate_relative_poses_batch_dev(self, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, K,
                                          d_res, d_inliers, d_pts3d=None, motion_cam2_to_cam1=True):
        """estimate_relative_poses(calc_homo=True) for n_pairs matched frame pairs of a batched extraction, all device pointers
        except K (host 3x3): pair p's RELATIVE_POSES_RESULT_DTYPE record in d_res[p], solution s's inlier indices at
        d_inliers + (p * 5 + s) * cap and its triangulated inliers at d_pts3d + (p * 5 + s) * cap * 3.  Thresholds, hypothesis
        count and seed come from the context's parameters."""
        K = _c(K, np.float64)
        self._chk(self.lib.mvo_estimate_relative_poses_batch_dev(self.h, _ptr(d_kpts), _ptr(d_counts), batch, cap, _ptr(d_pairs), n_pairs,
                                                                 _ptr(d_matches), _ptr(d_n_matches), _ptr(K), int(bool(motion_cam2_to_cam1)),
                                                                 _ptr(d_res), _ptr(d_inliers), _ptr(d_pts3d)))

    def vo_init_candidates_batch_dev(self, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, d_rp, d_rp_inliers,
                                     d_rp_pts3d, T_w_c_ref, vo_params, d_out, d_kept, d_kept_pts3d, d_kept_angles):
        """The initialisation check of the state machine (estimateMotionAnd3DPoints_ + isVoGoodToInit_) for every pair of an
        estimate_relative_poses_batch_dev call (motion_cam2_to_cam1 = True, with d_pts3d), all device pointers except T_w_c_ref
        (host 4x4) and vo_params (VoParams): pair p's INIT_CANDIDATE_RESULT_DTYPE record in d_out[p], its kept matches at
        d_kept + p * cap, kept points at d_kept_pts3d + p * cap * 3 and kept angles at d_kept_angles + p * cap."""
        T = _c(T_w_c_ref, np.float64)
        assert T.size == 16
        self._chk(self.lib.mvo_vo_init_candidates_batch_dev(self.h, _ptr(d_kpts), _ptr(d_counts), batch, cap, _ptr(d_pairs), n_pairs,
                                                            _ptr(d_matches), _ptr(d_n_matches), _ptr(d_rp), _ptr(d_rp_inliers),
                                                            _ptr(d_rp_pts3d), _ptr(T), C.byref(vo_params), _ptr(d_out), _ptr(d_kept),
                                                            _ptr(d_kept_pts3d), _ptr(d_kept_angles)))

    def vo_keyframe_points_batch_dev(self, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, d_ess, d_ess_inliers,
                                     d_T_w_c, K, vo_params, d_out, d_kept, d_kept_pts3d, d_kept_angles, d_kept_world=None, d_kept_norm=None):
        """The new map points of the state machine's keyframe branch for every (reference keyframe, frame) pair of an
        esti_motion_by_essential_batch_dev call, triangulated with the known motion T_w_c_curr^-1 * T_w_c_ref of the frames' poses
        (d_T_w_c: batch x 16 doubles on the device).  All device pointers except K (host 3x3) and vo_params (VoParams): pair p's
        KEYFRAME_POINTS_RESULT_DTYPE record in d_out[p], its kept matches at d_kept + p * cap, kept points (current camera) at
        d_kept_pts3d + p * cap * 3, kept angles at d_kept_angles + p * cap and, when given, the map points' world positions at
        d_kept_world + p * cap * 3 and viewing directions at d_kept_norm + p * cap * 3."""
        K = _c(K, np.float64)
        self._chk(self.lib.mvo_vo_keyframe_points_batch_dev(self.h, _ptr(d_kpts), _ptr(d_counts), batch, cap, _ptr(d_pairs), n_pairs,
                                                            _ptr(d_matches), _ptr(d_n_matches), _ptr(d_ess), _ptr(d_ess_inliers),
                                                            _ptr(d_T_w_c), _ptr(K), C.byref(vo_params), _ptr(d_out), _ptr(d_kept),
                                                            _ptr(d_kept_pts3d), _ptr(d_kept_angles), _ptr(d_kept_world), _ptr(d_kept_norm)))

    def vo_map_matches_batch_dev(self, d_kpts, d_desc, d_counts, batch, cap, d_frames, d_T_w_c_guess, n_jobs, d_map_pts, d_map_desc, n_map,
                                 K, rows, cols, method_index, radius, d_out, d_cand, d_matches, d_cand_xy=None, d_pts3d=None, d_pts2d=None):
        """The state machine's tracking step before PnP (getMappointsInCurrentView_, the match against the map, the 3D-2D pairs)
        for n_jobs (frame, guess pose) jobs of an orb_extract_batch_dev output against one map of n_map points, all device
        pointers except K (host 3x3): job j's MAP_MATCHES_RESULT_DTYPE record in d_out[j], its candidates' map indices at
        d_cand + j * n_map (and pixels at d_cand_xy + j * n_map * 2), its matches at d_matches + j * cap (query_idx = candidate
        rank) and, when given, the PnP inputs at d_pts3d + j * cap * 3 and d_pts2d + j * cap * 2."""
        K = _c(K, np.float64)
        self._chk(self.lib.mvo_vo_map_matches_batch_dev(self.h, _ptr(d_kpts), _ptr(d_desc), _ptr(d_counts), batch, cap, _ptr(d_frames),
                                                        _ptr(d_T_w_c_guess), n_jobs, _ptr(d_map_pts), _ptr(d_map_desc), n_map, _ptr(K),
                                                        rows, cols, method_index, C.c_float(radius), _ptr(d_out), _ptr(d_cand),
                                                        _ptr(d_cand_xy), _ptr(d_matches), _ptr(d_pts3d), _ptr(d_pts2d)))

    def vo_pnp_batch_dev(self, d_mm, d_matches, d_pts3d, d_pts2d, n_jobs, cap, d_T_w_c_prev, K, track_params, d_out, d_inliers,
                         d_kept=None):
        """The rest of the state machine's poseEstimationPnP_ (solvePnPRansac with its refit, the inlier matches, T_w_c and the
        jump check) for the n_jobs jobs of a vo_map_matches_batch_dev output (same rows, same cap), all device pointers except K
        (host 3x3) and track_params (TrackParams: min_pnp_points, max_dist_to_prev): d_T_w_c_prev holds each job's previous-frame
        pose (16 doubles); job j's VO_PNP_RESULT_DTYPE record lands in d_out[j], its ascending inlier indices at
        d_inliers + j * cap and, when given, the inlier matches at d_kept + j * cap."""
        K = _c(K, np.float64)
        self._chk(self.lib.mvo_vo_pnp_batch_dev(self.h, _ptr(d_mm), _ptr(d_matches), _ptr(d_pts3d), _ptr(d_pts2d), n_jobs, cap,
                                                _ptr(d_T_w_c_prev), _ptr(K), C.byref(track_params), _ptr(d_out), _ptr(d_inliers),
                                                _ptr(d_kept)))

    # ---- matching ----------------------------------------------------------------------
    def match_hamming_nn(self, d1, d2):
        d1, d2 = _c(d1, np.uint8), _c(d2, np.uint8)
        out = np.zeros(len(d1), DMATCH_DTYPE)
        self._chk(self.lib.mvo_match_hamming_nn(self.h, _ptr(d1), len(d1), _ptr(d2), len(d2), _ptr(out)))
        return out

    def match_hamming_knn2(self, d1, d2):
        d1, d2 = _c(d1, np.uint8), _c(d2, np.uint8)
        out = np.zeros((len(d1), 2), DMATCH_DTYPE)
        self._chk(self.lib.mvo_match_hamming_knn2(self.h, _ptr(d1), len(d1), _ptr(d2), len(d2), _ptr(out)))
        return out

    def match_radius_sad(self, d1, xy1, d2, xy2, radius):
        d1, d2 = _c(d1, np.uint8), _c(d2, np.uint8)
        xy1, xy2 = _c(xy1, np.float32), _c(xy2, np.float32)
        out = np.zeros(len(d1), DMATCH_DTYPE)
        n = C.c_int(0)
        self._chk(self.lib.mvo_match_radius_sad(self.h, _ptr(d1), _ptr(xy1), len(d1), _ptr(d2), _ptr(xy2), len(d2),
                                                 C.c_float(radius), _ptr(out), C.byref(n)))
        return out[: n.value].copy()

    def match_features(self, d1, d2, method_index=1, xy1=None, xy2=None, radius=0.0):
        d1, d2 = _c(d1, np.uint8), _c(d2, np.uint8)
        if xy1 is not None:
            xy1, xy2 = _c(xy1, np.float32), _c(xy2, np.float32)
        out = np.zeros(max(len(d1), 1), DMATCH_DTYPE)
        n = C.c_int(0)
        self._chk(self.lib.mvo_match_features(self.h, _ptr(d1), len(d1), _ptr(d2), len(d2), method_index,
                                               _ptr(xy1), _ptr(xy2), C.c_float(radius), _ptr(out), C.byref(n)))
        return out[: n.value].copy()

    def match_dev(self, mode, d_d1, d_xy1, n1, d_d2, d_xy2, n2, radius, d_keys):
        self._chk(self.lib.mvo_match_dev(self.h, mode, _ptr(d_d1), _ptr(d_xy1), n1, _ptr(d_d2), _ptr(d_xy2), n2,
                                          C.c_float(radius), _ptr(d_keys)))

    # ---- PnP ---------------------------------------------------------------------------
    def solve_pnp_ransac(self, pts3d, pts2d, K):
        p3, p2, K = _c(pts3d, np.float32), _c(pts2d, np.float32), _c(K, np.float64)
        rvec, tvec = np.zeros(3), np.zeros(3)
        inl = np.zeros(len(p3), np.int32)
        n = C.c_int(len(p3))
        self._chk(self.lib.mvo_solve_pnp_ransac(self.h, _ptr(p3), _ptr(p2), len(p3), _ptr(K), _ptr(rvec), _ptr(tvec),
                                                 _ptr(inl), C.byref(n)))
        return rvec, tvec, inl[: n.value].copy()

    def pnp_last_hypotheses(self):
        cap = int(self.params.pnp_hypotheses)
        poses = np.zeros((cap, 12))
        counts = np.zeros(cap, np.int32)
        n = C.c_int(0)
        self._chk(self.lib.mvo_pnp_last_hypotheses(self.h, _ptr(poses), _ptr(counts), cap, C.byref(n)))
        return poses[: n.value].copy(), counts[: n.value].copy()

    def pnp_refine(self, pts3d, pts2d, K, rvec, tvec):
        p3, p2, K = _c(pts3d, np.float32), _c(pts2d, np.float32), _c(K, np.float64)
        rvec, tvec = _c(rvec, np.float64).copy().reshape(3), _c(tvec, np.float64).copy().reshape(3)
        self._chk(self.lib.mvo_pnp_refine(self.h, _ptr(p3), _ptr(p2), len(p3), _ptr(K), _ptr(rvec), _ptr(tvec)))
        return rvec, tvec

    # ---- two-view geometry ---------------------------------------------------------------
    def esti_motion_by_essential(self, pts1, pts2, K, threshold=1.0):
        p1, p2, K = _c(pts1, np.float32), _c(pts2, np.float32), _c(K, np.float64)
        E, R, t = np.zeros((3, 3)), np.zeros((3, 3)), np.zeros(3)
        inl = np.zeros(max(len(p1), 1), np.int32)
        n = C.c_int(len(p1))
        self._chk(self.lib.mvo_esti_motion_by_essential(self.h, _ptr(p1), _ptr(p2), len(p1), _ptr(K), float(threshold), _ptr(E), _ptr(R),
                                                        _ptr(t), _ptr(inl), C.byref(n)))
        return E, R, t, inl[: n.value].copy()

    def esti_motion_by_homography(self, pts1, pts2, K, threshold=3.0):
        p1, p2, K = _c(pts1, np.float32), _c(pts2, np.float32), _c(K, np.float64)
        H, Rs, ts, ns = np.zeros((3, 3)), np.zeros((4, 3, 3)), np.zeros((4, 3)), np.zeros((4, 3))
        inl = np.zeros(max(len(p1), 1), np.int32)
        n, nsol = C.c_int(len(p1)), C.c_int(0)
        self._chk(self.lib.mvo_esti_motion_by_homography(self.h, _ptr(p1), _ptr(p2), len(p1), _ptr(K), float(threshold), _ptr(H), _ptr(Rs),
                                                         _ptr(ts), _ptr(ns), C.byref(nsol), _ptr(inl), C.byref(n)))
        k = nsol.value
        return H, Rs[:k].copy(), ts[:k].copy(), ns[:k].copy(), inl[: n.value].copy()

    def remove_wrong_rt_of_homography(self, pts_np1, pts_np2, inliers, Rs, ts, normals):
        p1, p2, inl = _c(pts_np1, np.float32), _c(pts_np2, np.float32), _c(inliers, np.int32)
        k = len(Rs)
        R4, t4, n4 = np.zeros((4, 3, 3)), np.zeros((4, 3)), np.zeros((4, 3))
        R4[:k], t4[:k], n4[:k] = Rs, ts, normals
        nsol = C.c_int(k)
        self._chk(self.lib.mvo_remove_wrong_rt_of_homography(self.h, _ptr(p1), _ptr(p2), len(p1), _ptr(inl), len(inl), _ptr(R4), _ptr(t4),
                                                             _ptr(n4), C.byref(nsol)))
        k = nsol.value
        return R4[:k].copy(), t4[:k].copy(), n4[:k].copy()

    def estimate_relative_poses(self, pts1, pts2, K, calc_homo=True, motion_cam2_to_cam1=True):
        p1, p2, K = _c(pts1, np.float32), _c(pts2, np.float32), _c(K, np.float64)
        n = len(p1)
        sol = TwoViewSolutions()
        inl = np.zeros((5, max(n, 1)), np.int32)
        pts3d = np.zeros((5, max(n, 1), 3), np.float32)
        self._chk(self.lib.mvo_estimate_relative_poses(self.h, _ptr(p1), _ptr(p2), n, _ptr(K), int(calc_homo), int(motion_cam2_to_cam1),
                                                       C.byref(sol), _ptr(inl), _ptr(pts3d)))
        out = []
        for s in range(sol.num_solutions):
            k = sol.n_inliers[s]
            out.append(dict(R=np.array(sol.R[s]).reshape(3, 3), t=np.array(sol.t[s]), normal=np.array(sol.normal[s]),
                            inliers=inl[s, :k].copy(), pts3d=pts3d[s, :k].copy()))
        return out, sol.best, dict(score_e=sol.score_e, score_h=sol.score_h, ratio=sol.ratio, E=np.array(sol.E).reshape(3, 3),
                                   H=np.array(sol.H).reshape(3, 3))

    def do_triangulation(self, pts_np1, pts_np2, R, t, inliers):
        p1, p2 = _c(pts_np1, np.float32), _c(pts_np2, np.float32)
        R, t, inl = _c(R, np.float64), _c(t, np.float64).reshape(3), _c(inliers, np.int32)
        out = np.zeros((len(inl), 3), np.float32)
        self._chk(self.lib.mvo_do_triangulation(self.h, _ptr(p1), _ptr(p2), len(p1), _ptr(R), _ptr(t), _ptr(inl), len(inl), _ptr(out)))
        return out

    # ---- BA ----------------------------------------------------------------------------
    def bundle_adjustment(self, poses_T_w_c, points, edge_frame, edge_point, obs, K, information=None,
                          fix_points=False, update_points=True):
        poses = _c(poses_T_w_c, np.float64).copy().reshape(-1, 16)
        pts = _c(points, np.float32).copy().reshape(-1, 3)
        ef, ep = _c(edge_frame, np.int32), _c(edge_point, np.int32)
        ob = _c(obs, np.float32).reshape(-1, 2)
        K = _c(K, np.float64)
        info = _c(np.eye(2) if information is None else information, np.float64)
        stats = np.zeros(4)
        self._chk(self.lib.mvo_bundle_adjustment(self.h, _ptr(poses), len(poses), _ptr(pts), len(pts), _ptr(ef), _ptr(ep),
                                                  _ptr(ob), len(ef), _ptr(K), _ptr(info), int(fix_points),
                                                  int(update_points), _ptr(stats)))
        return poses.reshape(-1, 4, 4), pts, stats

    def optimize_single_frame(self, pose_T_w_c, points, obs, K, fix_points=False, update_points=True):
        pose = _c(pose_T_w_c, np.float64).copy().reshape(16)
        pts = _c(points, np.float32).copy().reshape(-1, 3)
        ob = _c(obs, np.float32).reshape(-1, 2)
        K = _c(K, np.float64)
        self._chk(self.lib.mvo_optimize_single_frame(self.h, _ptr(pose), _ptr(pts), _ptr(ob), len(pts), _ptr(K),
                                                      int(fix_points), int(update_points)))
        return pose.reshape(4, 4), pts


class VisualOdometry:
    """mvo_vo: the whole addFrame state machine (initialisation, tracking, keyframes, map maintenance)."""

    def __init__(self, ctx: "Context", K, rows, cols, track=None, **overrides):
        self.ctx, self.lib = ctx, ctx.lib
        p = VoParams()
        self.lib.mvo_vo_default_params(C.byref(p))
        for k, v in (track or {}).items():
            if k == "information":
                for i, x in enumerate(np.asarray(v, np.float64).ravel()):
                    p.track.information[i] = float(x)
            else:
                if not hasattr(p.track, k):
                    raise AttributeError(k)
                setattr(p.track, k, v)
        for k, v in overrides.items():
            if not hasattr(p, k) or k == "track":
                raise AttributeError(k)
            setattr(p, k, v)
        self.params = p
        K = _c(K, np.float64)
        h = C.c_void_p()
        ctx._chk(self.lib.mvo_vo_create(ctx.h, _ptr(K), rows, cols, C.byref(p), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.mvo_vo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _image_args(self, image, channels, stride, on_device):
        if on_device:
            return C.c_void_p(int(image)), int(channels), int(stride)
        img = image if (isinstance(image, np.ndarray) and image.dtype == np.uint8 and image.flags.c_contiguous) else np.ascontiguousarray(image, np.uint8)
        channels = 1 if img.ndim == 2 else img.shape[2]
        self._keep = (getattr(self, "_keep", []) + [img])[-4:]      # a prefetched image must stay alive until its add_frame returns
        return _ptr(img), channels, img.shape[1] * channels

    def add_frame(self, image, channels=None, stride=None, on_device=False):
        """image: HxW(x3) uint8 array, or a device pointer (int) with channels / stride when on_device."""
        p, ch, st = self._image_args(image, channels, stride, on_device)
        T, info = np.zeros(16), VoFrameInfo()
        self.ctx._chk(self.lib.mvo_vo_add_frame_ex(self.h, p, ch, st, 1 if on_device else 0, _ptr(T), C.byref(info)))
        return T.reshape(4, 4), info

    def run_sequence(self, images, channels=None, stride=None, on_device=False):
        """run_vo.cpp's main loop over frames in memory (mvo_vo_run_sequence): images = list of HxW(x3) uint8 arrays, or of device
        pointers (ints) with channels / stride when on_device.  Returns (poses n x 4 x 4, list of VoFrameInfo)."""
        n = len(images)
        if on_device:
            addrs, ch, st, keep = [int(im) for im in images], int(channels), int(stride), None
        else:
            keep = [im if (isinstance(im, np.ndarray) and im.dtype == np.uint8 and im.flags.c_contiguous) else np.ascontiguousarray(im, np.uint8)
                    for im in images]
            shapes = {(1 if k.ndim == 2 else k.shape[2], k.shape[1]) for k in keep}
            if len(shapes) > 1:
                raise ValueError("run_sequence: all frames must share width and channels")
            ch, w = next(iter(shapes)) if shapes else (3, 0)
            st = w * ch
            addrs = [k.ctypes.data for k in keep]
        ptrs = (C.c_void_p * max(n, 1))(*addrs)
        T = np.zeros((max(n, 1), 16))
        infos = (VoFrameInfo * max(n, 1))()
        done = C.c_int(0)
        self.ctx._chk(self.lib.mvo_vo_run_sequence(self.h, ptrs, n, ch, st, 1 if on_device else 0, _ptr(T), infos, C.byref(done)))
        del keep
        return T[:n].reshape(n, 4, 4), [infos[i] for i in range(n)]

    def prefetch(self, image, channels=None, stride=None, on_device=False):
        """Hand the NEXT frame over (same array object / pointer as the later add_frame call)."""
        p, ch, st = self._image_args(image, channels, stride, on_device)
        self.ctx._chk(self.lib.mvo_vo_prefetch(self.h, p, ch, st, 1 if on_device else 0))

    @property
    def device_resident(self):
        return bool(self.lib.mvo_vo_device_resident(self.h))

    def reset(self):
        self.ctx._chk(self.lib.mvo_vo_reset(self.h))

    @property
    def kernel_launches(self) -> int:
        return int(self.lib.mvo_vo_kernel_launches(self.h))

    def timing_enable(self, mask: int):
        self.ctx._chk(self.lib.mvo_vo_timing_enable(self.h, int(mask)))

    def timing_read(self):
        n = self.lib.mvo_kernel_classes()
        ms, cnt = np.zeros(n, np.float64), np.zeros(n, np.uint64)
        self.ctx._chk(self.lib.mvo_vo_timing_read(self.h, _ptr(ms), _ptr(cnt)))
        return ms, cnt

    def is_initialized(self):
        return bool(self.lib.mvo_vo_is_initialized(self.h))

    def num_keyframes(self):
        return self.lib.mvo_vo_num_keyframes(self.h)

    def get_map(self):
        n = C.c_int(self.lib.mvo_vo_map_size(self.h))
        cap = max(n.value, 1)
        ids, pts, desc, rgb = np.zeros(cap, np.int32), np.zeros((cap, 3), np.float32), np.zeros((cap, 32), np.uint8), np.zeros((cap, 3), np.uint8)
        self.ctx._chk(self.lib.mvo_vo_get_map(self.h, _ptr(ids), _ptr(pts), _ptr(desc), _ptr(rgb), cap, C.byref(n)))
        return ids[: n.value], pts[: n.value], desc[: n.value], rgb[: n.value]

    def frame_pose(self, k=0):
        T = np.zeros(16)
        self.ctx._chk(self.lib.mvo_vo_frame_pose(self.h, k, _ptr(T)))
        return T.reshape(4, 4)

    _FRAME_DATA = {"keypoints": (0, KEYPOINT_DTYPE, ()), "descriptors": (1, np.uint8, (32,)), "matches_with_ref": (2, DMATCH_DTYPE, ()),
                   "matches_with_map": (3, DMATCH_DTYPE, ()), "inliers_pts3d": (4, np.float32, (3,)), "id": (5, np.int32, ())}

    def frame_data(self, what, which=0):
        """Members of the `which`-th newest frame (or -1 = getPrevRef()) that run_vo.cpp's display code reads."""
        code, dtype, tail = self._FRAME_DATA[what]
        n = C.c_int(0)
        rc = self.lib.mvo_vo_frame_data(self.h, which, code, None, 0, C.byref(n))
        if rc not in (0, -4):
            self.ctx._chk(rc)
        out = np.zeros((max(n.value, 1),) + tail, dtype)
        self.ctx._chk(self.lib.mvo_vo_frame_data(self.h, which, code, _ptr(out), max(n.value, 1), C.byref(n)))
        return out[: n.value]

    def has_keyframe(self, frame_id):
        return bool(self.lib.mvo_vo_has_keyframe(self.h, int(frame_id)))


class Tracker:
    """mvo_tracker: the per-frame tracking step (extract -> match map -> PnP -> BA)."""

    def __init__(self, ctx: Context, K, rows, cols, **overrides):
        self.ctx = ctx
        self.lib = ctx.lib
        p = TrackParams()
        self.lib.mvo_default_track_params(C.byref(p))
        for k, v in overrides.items():
            if k == "information":
                for i, x in enumerate(np.asarray(v, np.float64).ravel()):
                    p.information[i] = float(x)
            else:
                if not hasattr(p, k):
                    raise AttributeError(k)
                setattr(p, k, v)
        self.params = p
        self.rows, self.cols = rows, cols
        K = _c(K, np.float64)
        h = C.c_void_p()
        ctx._chk(self.lib.mvo_tracker_create(ctx.h, _ptr(K), rows, cols, C.byref(p), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.mvo_tracker_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_map(self, pts3d, desc):
        p, d = _c(pts3d, np.float32), _c(desc, np.uint8)
        self.ctx._chk(self.lib.mvo_tracker_set_map(self.h, _ptr(p), _ptr(d), len(p)))

    def reset(self, T_w_c_ref):
        T = _c(T_w_c_ref, np.float64)
        self.ctx._chk(self.lib.mvo_tracker_reset(self.h, _ptr(T)))

    def track(self, image, channels=None, stride=None, on_device=False):
        """image: numpy array (host) or an integer device pointer (with channels/stride given)."""
        T = np.zeros(16)
        res = TrackResult()
        if on_device:
            ptr = C.c_void_p(int(image))
        else:
            img = image if (isinstance(image, np.ndarray) and image.flags["C_CONTIGUOUS"] and image.dtype == np.uint8) \
                else np.ascontiguousarray(image, np.uint8)
            channels = 1 if img.ndim == 2 else img.shape[2]
            stride = img.shape[1] * channels
            ptr = _ptr(img)
        self.ctx._chk(self.lib.mvo_tracker_track(self.h, ptr, channels, stride, int(on_device), _ptr(T), C.byref(res)))
        return T.reshape(4, 4), res

    def prefetch(self, image, channels=None, stride=None, on_device=False):
        """Enqueue the extraction of a future frame (device pointer, or a numpy array that must stay alive
        and be passed again, unchanged, to track())."""
        if on_device:
            ptr = C.c_void_p(int(image))
        else:
            assert image.flags["C_CONTIGUOUS"] and image.dtype == np.uint8
            channels = 1 if image.ndim == 2 else image.shape[2]
            stride = image.shape[1] * channels
            ptr = _ptr(image)
        self.ctx._chk(self.lib.mvo_tracker_prefetch(self.h, ptr, channels, stride, int(on_device)))

    def timing_enable(self, mask: int):
        self.ctx._chk(self.lib.mvo_tracker_timing_enable(self.h, mask))

    def timing_read(self):
        n = self.lib.mvo_kernel_classes()
        ms = np.zeros(n)
        cnt = np.zeros(n, np.uint64)
        self.ctx._chk(self.lib.mvo_tracker_timing_read(self.h, _ptr(ms), _ptr(cnt)))
        return ms, cnt

    @property
    def kernel_launches(self) -> int:
        return int(self.lib.mvo_tracker_kernel_launches(self.h))

    def frame_pose(self, k=0):
        T = np.zeros(16)
        self.ctx._chk(self.lib.mvo_tracker_frame_pose(self.h, k, _ptr(T)))
        return T.reshape(4, 4)


def kernel_names():
    lib = load_library()
    return [lib.mvo_kernel_name(i).decode() for i in range(lib.mvo_kernel_classes())]


def timing_enable(ctx: Context, mask: int):
    ctx._chk(ctx.lib.mvo_timing_enable(ctx.h, mask))


def timing_read(ctx: Context):
    n = ctx.lib.mvo_kernel_classes()
    ms = np.zeros(n)
    cnt = np.zeros(n, np.uint64)
    ctx._chk(ctx.lib.mvo_timing_read(ctx.h, _ptr(ms), _ptr(cnt)))
    return ms, cnt


def remove_duplicated_matches(matches):
    m = _c(matches, DMATCH_DTYPE).copy()
    n = C.c_int(len(m))
    rc = load_library().mvo_remove_duplicated_matches(_ptr(m), C.byref(n))
    if rc != MVO_OK:
        raise MvoError(rc, "mvo_remove_duplicated_matches")
    return m[: n.value].copy()
