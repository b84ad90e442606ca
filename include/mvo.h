/*
 * mvo.h — C ABI of libmvo.so: the H100 (sm_90a) implementation of the per-frame
 * hot path of felixchenfy/Monocular-Visual-Odometry.
 *
 * The reference has no FFI of its own: its "operator API" is a set of free C++
 * functions in my_slam::geometry / my_slam::optimization plus one inline OpenCV
 * call in the VO layer (SURVEY.md §8b).  Each entry point below names the
 * reference interface it replaces (paths relative to the reference repo root).
 * The C++ adapters with the reference's exact signatures live in
 * monocular-visual-odometry_b200/my_slam_adapter/ and forward to these functions.
 *
 * Conventions
 *  - All pointers in the mvo_* (non-_dev) functions are HOST pointers owned by
 *    the caller; outputs are caller-allocated with an explicit capacity.
 *  - *_dev functions take DEVICE pointers (resident in HBM) and are enqueued on
 *    the context's stream without synchronising; they exist so that a pipeline
 *    can keep a frame on the GPU between stages (and so bench.py can time the
 *    kernels with inputs already resident).
 *  - Return value: 0 = MVO_OK, negative = error (mvo_status).  mvo_last_error()
 *    returns a human-readable message for the last failure on that context.
 *  - A context is bound to one GPU and one stream; calls on one context must be
 *    serialised by the caller (the reference is single-threaded, non-reentrant).
 *  - No CPU fallback exists: if no CUDA device is usable mvo_create fails with
 *    MVO_ERR_NO_DEVICE.
 */
#ifndef MVO_H_
#define MVO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MVO_VERSION 100

typedef enum mvo_status {
  MVO_OK = 0,
  MVO_ERR_INVALID_ARG = -1,   /* null pointer, bad size, bad method index (reference throws
                                 std::runtime_error at src/geometry/feature_match.cpp:225) */
  MVO_ERR_NO_DEVICE = -2,     /* no usable CUDA device / wrong architecture */
  MVO_ERR_CUDA = -3,          /* a CUDA runtime call or kernel failed */
  MVO_ERR_CAPACITY = -4,      /* caller-provided output capacity too small */
  MVO_ERR_UNSUPPORTED = -5,   /* size beyond a documented limit */
  MVO_ERR_DEGENERATE = -6     /* numerically degenerate problem (e.g. < 4 PnP points) */
} mvo_status;

/* cv::KeyPoint, 28 bytes, same field order as OpenCV (features2d). */
typedef struct mvo_keypoint {
  float x, y;       /* pt, pixels in level-0 coordinates */
  float size;       /* 31 * level scale */
  float angle;      /* degrees [0,360) */
  float response;   /* Harris response */
  int32_t octave;   /* pyramid level */
  int32_t class_id; /* always -1 */
} mvo_keypoint;

/* cv::DMatch, 16 bytes. */
typedef struct mvo_dmatch {
  int32_t query_idx;
  int32_t train_idx;
  int32_t img_idx;  /* reference leaves OpenCV's default: 0 from the matchers, -1 from DMatch(i,j,d) */
  float distance;
} mvo_dmatch;

/* Parameters the hot path latches from config/config.yaml (SURVEY.md §5).
 * mvo_default_params() fills the shipped values (with max_number_of_keypoints
 * raised to the BASELINE's 2000 only if the caller does so explicitly). */
typedef struct mvo_params {
  /* ORB — src/geometry/feature_match.cpp:16-23 */
  int32_t orb_nfeatures;      /* number_of_keypoints_to_extract = 8000 */
  float orb_scale_factor;     /* scale_factor = 1.2 */
  int32_t orb_nlevels;        /* level_pyramid = 4 (<= 8 supported) */
  int32_t orb_fast_threshold; /* score_threshold = 20 */
  /* grid NMS — feature_match.cpp:56-59 */
  int32_t max_keypoints;      /* max_number_of_keypoints = 1500 */
  int32_t grid_size;          /* kpts_uniform_selection_grid_size = 16 */
  int32_t max_pts_per_grid;   /* kpts_uniform_selection_max_pts_per_grid = 8 */
  /* matching — feature_match.cpp:137-139 (values after the reference's get<int> rounding) */
  double xiang_gao_ratio;     /* xiang_gao_method_match_ratio = 2 */
  double lowe_ratio;          /* lowe_method_dist_ratio: 0.8 read as int -> 1 */
  /* PnP — src/vo/vo.cpp:314-317 (hard-coded in the reference) */
  int32_t pnp_hypotheses;     /* batched hypothesis count (reference: <=100 adaptive); default 4096 */
  float pnp_reproj_error;     /* 2.0 px */
  uint64_t pnp_seed;          /* counter-based RNG seed for minimal sets */
  int32_t pnp_refine_iters;   /* LM iterations of the final refit on inliers; default 20 */
  /* BA — src/optimization/g2o_ba.cpp:275, g2o defaults (SURVEY.md App. B) */
  int32_t ba_iterations;      /* reference: 50; BASELINE config 4: 10 */
  double ba_huber_delta;      /* 1.0 */
  int32_t ba_fix_first_pose;  /* 0 = reference behaviour (no pose fixed, g2o_ba.cpp:210-211) */
  double ba_step_tol;         /* 0 = g2o's control flow to the letter (default).  > 0: the pose-only LM (fixed map
                                 points) stops as soon as a trial step is below this bound — at convergence g2o
                                 spends up to 10 rejected trials on steps of ~1e-10 that it then restores; the
                                 poses agree with the full run to within the bound (tests/test_ba_gpu.py) */
  /* two-view geometry — src/geometry/epipolar_geometry.cpp:17-57 */
  int32_t epi_hypotheses;     /* batched essential-matrix hypotheses (reference: adaptive RANSAC, prob 0.999); default 4096 */
  int32_t pnp_mode;           /* 0 (default): pnp_hypotheses batched P3P hypotheses, all scored; 1: cv::solvePnPRansac's own flow as
                                 the reference calls it (vo.cpp:314-320) — cv::RNG sampler, 5-point EPnP minimal models, <= 100
                                 adaptive iterations at confidence 0.999, float scoring (csrc/pnp_cv_kernels.cuh; CPU restatement
                                 pinned inlier-index-exact to cv2: oracle/pnp_cv_oracle.py).  Its result agrees with OpenCV's up to
                                 correspondences within ~1e-3 px of the threshold (the minimal solver's SVD noise, see the oracle) */
  double eh_ratio_threshold;  /* mvo_estimate_relative_poses takes the homography branch when H/(E+H) exceeds this: 0.5
                                 (motion_estimation.cpp:140; the reference's README.md:57 documents 0.45).  The locally
                                 optimised essential matrix keeps more inliers than OpenCV's un-refined five-point model, so
                                 the ratio sits ~0.03 lower here: exactly planar scenes come out at 0.485-0.492 (OpenCV
                                 0.50-0.52) and fall on the E side of 0.5 (DESIGN.md section 10) */
  double essential_threshold; /* mvo_estimate_relative_poses: cv::findEssentialMat threshold in pixels (config findEssentialMat_threshold = 1.0,
                                 epipolar_geometry.cpp:29-36) */
  double homography_threshold;/* mvo_estimate_relative_poses: cv::findHomography ransacReprojThreshold = 3 (epipolar_geometry.cpp:101) */
} mvo_params;

typedef struct mvo_ctx mvo_ctx;

/* ---- context -------------------------------------------------------------------------- */
void mvo_default_params(mvo_params *p);
/* Replaces the reference's process-global state (function-local static ORB objects, matchers
 * and latched config values, feature_match.cpp:16-23,42-45,56-62,137-141). */
int mvo_create(mvo_ctx **out, int device, const mvo_params *params /* NULL = defaults */);
void mvo_destroy(mvo_ctx *ctx);
const char *mvo_last_error(const mvo_ctx *ctx);
int mvo_get_params(const mvo_ctx *ctx, mvo_params *out);
int mvo_set_params(mvo_ctx *ctx, const mvo_params *p);
/* Use an externally created cudaStream_t (e.g. torch's current stream) for all work. */
int mvo_set_stream(mvo_ctx *ctx, void *cuda_stream);
int mvo_synchronize(mvo_ctx *ctx);
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
uint64_t mvo_kernel_launches(const mvo_ctx *ctx);

/* ---- ORB extraction --------------------------------------------------------------------
 * mvo_calc_keypoints  == geometry::calcKeyPoints   (src/geometry/feature_match.cpp:11-36):
 *     cv::ORB(8000,1.2,4,31,0,2,HARRIS,31,20)->detect + selectUniformKptsByGrid (:51-84).
 * mvo_calc_descriptors == geometry::calcDescriptors (feature_match.cpp:38-49):
 *     cv::ORB(8000,1.2,4)->compute on caller keypoints (level-sorted, as produced above).
 * mvo_orb_extract      == both, fused (one upload, keypoints never leave the GPU in between);
 *     this is what vo::Frame::calcKeyPoints + calcDescriptors (include/my_slam/vo/frame.h:73-86)
 *     amount to per frame.
 * image: rows x cols, `channels` = 3 (BGR, as cv::imread gives run_vo.cpp:114) or 1 (gray),
 * `stride` bytes per row.  Keypoint order, coordinates, angle, response and descriptor bytes
 * are bit-exact with OpenCV 4.13's cv::ORB.
 * *n_kpts: in = capacity of kpts (and rows of desc), out = number written. */
int mvo_calc_keypoints(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels,
                       size_t stride, mvo_keypoint *kpts, int *n_kpts);
int mvo_calc_descriptors(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels,
                         size_t stride, const mvo_keypoint *kpts, int n_kpts,
                         uint8_t *desc /* n_kpts x 32 */);
int mvo_orb_extract(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels,
                    size_t stride, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc);
/* geometry::selectUniformKptsByGrid (feature_match.cpp:51-84) on host data (tiny, sequential).
 * Unlike the reference, the grid dimensions are taken from THIS call's image size rather than
 * latched from the first call. */
int mvo_select_uniform_kpts_by_grid(mvo_ctx *ctx, mvo_keypoint *kpts, int *n_kpts,
                                    int image_rows, int image_cols);

/* Batched, device-resident extraction for throughput (extraction does not depend on VO state,
 * SURVEY.md §8e): d_images = B frames, each rows x cols x channels with `stride` bytes per row
 * and `frame_stride` bytes per frame.  Outputs are device arrays with `cap` entries per frame:
 * d_kpts[B][cap], d_desc[B][cap][32], d_counts[B].  Asynchronous on the context stream. */
int mvo_orb_extract_batch_dev(mvo_ctx *ctx, const uint8_t *d_images, int batch, int rows,
                              int cols, int channels, size_t stride, size_t frame_stride,
                              mvo_keypoint *d_kpts, uint8_t *d_desc, int32_t *d_counts, int cap);
/* geometry::matchFeatures (feature_match.cpp:126-239) for n_pairs frame pairs of a batched extraction, entirely on the
 * device.  d_kpts / d_desc / d_counts / cap: the layout mvo_orb_extract_batch_dev writes (`batch` frames; counts are
 * clamped to [0, cap]).  d_pairs: n_pairs x 2 int32 frame indices (query frame, train frame), device memory; any pairs:
 * consecutive, windowed, reversed, repeated, or a frame with itself.  method_index 1 / 2 / 3 and radius as for
 * mvo_match_features; method 3 reads the keypoints' pt (d_kpts may be NULL otherwise).
 * d_out: n_pairs x cap mvo_dmatch, pair p's list at d_out + p * cap, byte-identical to mvo_match_features(query frame,
 * train frame).  d_n_out[p] = number of matches of pair p, or MVO_ERR_INVALID_ARG (and nothing written to its list) for a
 * frame index outside [0, batch) or a method-2 pair whose train frame has fewer than 2 keypoints.
 * cap <= 8192 and n_pairs <= 65535 (MVO_ERR_UNSUPPORTED beyond).  Asynchronous on the context stream: two kernel
 * launches whatever n_pairs is, no host synchronisation (except when a scratch buffer of the context has to grow). */
int mvo_match_features_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const uint8_t *d_desc, const int32_t *d_counts,
                                 int batch, int cap, const int32_t *d_pairs, int n_pairs, int method_index, float radius,
                                 mvo_dmatch *d_out, int32_t *d_n_out);
/* geometry::estiMotionByEssential (+ doTriangulation) for the matched frame pairs of a batch, entirely on the device: what
 * mvo_estimate_relative_poses(calc_homo = 0, motion_cam2_to_cam1 = 1) returns as its solution 0, pair by pair.
 * d_kpts / d_counts / batch / cap: the layout of mvo_orb_extract_batch_dev (counts clamped to [0, cap]).  d_pairs: n_pairs x 2
 * int32 (query frame, train frame); d_matches / d_n_matches: what mvo_match_features_batch_dev wrote for those pairs (pair p's
 * list at d_matches + p * cap).  Pair p's correspondences are pts1[i] = kpts[query frame][m_i.query_idx].pt and pts2[i] =
 * kpts[train frame][m_i.train_idx].pt in match-list order; K: host 3x3, threshold: pixels (mvo_params::essential_threshold of the
 * per-pair path).  Every pair uses mvo_params::epi_hypotheses and pnp_seed as a single call on its points does.
 * d_res[p]: status MVO_OK, or the mvo_status of that pair alone; then nothing else of the pair is written (not the rest of
 * its record, its inlier rows or its points):
 *   MVO_ERR_INVALID_ARG  a frame index outside [0, batch), a match count outside [0, cap], a query_idx / train_idx outside
 *                        [0, count) of its frame (checked before anything is read through it);
 *   MVO_ERR_DEGENERATE   fewer than 8 matches, or no model reaches 8 inliers.
 * On MVO_OK: E, R, t byte-identical to mvo_esti_motion_by_essential on those points; d_inliers + p * cap: the n_inliers
 * inlier indices into the pair's match list, ascending; d_pts3d (NULL: no triangulation) + p * cap * 3: the inliers
 * triangulated as mvo_do_triangulation does on pixel2CamNormPlane points.
 * MVO_ERR_INVALID_ARG: a null pointer, fx or fy <= 0, threshold <= 0.  MVO_ERR_UNSUPPORTED: cap > 6400 (the consensus
 * kernel's shared memory, as for a single call), n_pairs > 65535, n_pairs x epi_hypotheses > 2^22 (80 bytes of scratch per
 * hypothesis).  Asynchronous on the context stream: six kernel launches (seven with d_pts3d) whatever n_pairs is, no host
 * synchronisation except when the call's own scratch buffer of the context has to grow. */
typedef struct mvo_two_view_result {
  int32_t status;      /* MVO_OK, or the mvo_status the per-pair call would have returned */
  int32_t n_matches;   /* correspondences of the pair (its match count) */
  int32_t n_inliers;   /* findEssentialMat's mask count; rows of the pair's inlier list */
  int32_t votes;       /* recoverPose's good-point count of the chosen (R, t) */
  double E[9], R[9], t[3];   /* as mvo_esti_motion_by_essential returns them: E[8] = 1, x2 ~ R x1 + t, |t| = 1 */
} mvo_two_view_result;
int mvo_esti_motion_by_essential_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                           const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches,
                                           const int32_t *d_n_matches, const double *K, double threshold,
                                           mvo_two_view_result *d_res, int32_t *d_inliers, float *d_pts3d);

/* ---- descriptor matching ---------------------------------------------------------------
 * Raw all-pairs kernels.  d1: n1 x 32 bytes (query), d2: n2 x 32 bytes (train).
 * n1, n2 <= 65535.  Ties are broken towards the lowest train index (OpenCV BFMatcher rule).
 *  mvo_match_hamming_nn   == cv::BFMatcher(NORM_HAMMING).match    (the exact search that
 *      FLANN-LSH, feature_match.cpp:140,162, approximates): out[i] = best train for query i.
 *  mvo_match_hamming_knn2 == matcher_bf->knnMatch(d1,d2,knn,2)    (feature_match.cpp:208):
 *      out[2*i], out[2*i+1] = best and second best (n2 >= 2 required).
 *  mvo_match_radius_sad   == geometry::matchByRadiusAndBruteForce (feature_match.cpp:86-124):
 *      xy1/xy2 = keypoint pt (x,y) pairs; distance = sum|a-b| / 32 (double -> float);
 *      queries with no train inside the radius are omitted.  *n_out receives the count. */
int mvo_match_hamming_nn(mvo_ctx *ctx, const uint8_t *d1, int n1, const uint8_t *d2, int n2,
                         mvo_dmatch *out /* n1 */);
int mvo_match_hamming_knn2(mvo_ctx *ctx, const uint8_t *d1, int n1, const uint8_t *d2, int n2,
                           mvo_dmatch *out /* 2*n1 */);
int mvo_match_radius_sad(mvo_ctx *ctx, const uint8_t *d1, const float *xy1, int n1,
                         const uint8_t *d2, const float *xy2, int n2, float radius,
                         mvo_dmatch *out /* n1 */, int *n_out);
/* geometry::matchFeatures (feature_match.cpp:126-239) end to end: method 1 (exact Hamming NN
 * in place of FLANN-LSH), 2 (knn2 + Lowe ratio) or 3 (radius-gated SAD), the
 * max(min_dis*ratio, 30) threshold (:187-196) and removeDuplicatedMatches (:241-260).
 * xy1/xy2/radius are only read for method 3.  out capacity >= n1. */
int mvo_match_features(mvo_ctx *ctx, const uint8_t *d1, int n1, const uint8_t *d2, int n2,
                       int method_index, const float *xy1, const float *xy2, float radius,
                       mvo_dmatch *out, int *n_out);
/* geometry::removeDuplicatedMatches (feature_match.cpp:241-260): libstdc++ std::sort by
 * trainIdx (unstable, like the reference) then keep the first of each run.  Host only. */
int mvo_remove_duplicated_matches(mvo_dmatch *matches, int *n);

/* Device-resident raw matcher: packed result keys, one (mode 0,2) or two (mode 1) per query:
 * key = (distance << 16) | train_idx, 0xFFFFFFFF = no match.  mode: 0 = Hamming NN,
 * 1 = Hamming knn2, 2 = radius SAD (d_xy1/d_xy2 required).  Asynchronous. */
int mvo_match_dev(mvo_ctx *ctx, int mode, const uint8_t *d_d1, const float *d_xy1, int n1,
                  const uint8_t *d_d2, const float *d_xy2, int n2, float radius,
                  uint32_t *d_keys);

/* ---- PnP -------------------------------------------------------------------------------
 * Replaces the inline call cv::solvePnPRansac(pts_3d, pts_2d, K, noArray(), rvec, t, false,
 * 100, 2.0, 0.999, inliers) at src/vo/vo.cpp:318-320.
 * pts3d: n x 3 float (cv::Point3f), pts2d: n x 2 float (cv::Point2f), K: 3x3 row-major double.
 * Outputs: rvec[3] (Rodrigues), tvec[3], inliers (indices into the input, ascending; the
 * consensus set of the best minimal model, as OpenCV returns), *n_inliers in = capacity,
 * out = count.  Returns MVO_ERR_DEGENERATE if n < 4 or no hypothesis has >= 4 inliers. */
int mvo_solve_pnp_ransac(mvo_ctx *ctx, const float *pts3d, const float *pts2d, int n,
                         const double *K, double *rvec, double *tvec, int32_t *inliers,
                         int *n_inliers);
/* Debug/parity hook: the hypotheses of the last mvo_solve_pnp_ransac call.
 * poses: H x 12 doubles (R row-major 3x3, then t), counts: H inlier counts (-1 = invalid). */
int mvo_pnp_last_hypotheses(mvo_ctx *ctx, double *poses, int32_t *counts, int cap, int *n_hyp);
/* Final refit only: LM on the reprojection error over all n points from (rvec,tvec) in/out —
 * the deterministic part of solvePnPRansac (SURVEY.md App. C (1)). */
int mvo_pnp_refine(mvo_ctx *ctx, const float *pts3d, const float *pts2d, int n, const double *K,
                   double *rvec, double *tvec);

/* ---- bundle adjustment -----------------------------------------------------------------
 * Replaces optimization::bundleAdjustment (src/optimization/g2o_ba.cpp:172-317), flattened:
 *   poses_T_w_c : F x 16 doubles, row-major 4x4 camera->world (Frame::T_w_c_), in/out.
 *   points      : P x 3 floats (MapPoint::pos_), in/out (written only if update_points).
 *   edges       : E observations; edge e = (frame edge_frame[e], point edge_point[e],
 *                 pixel obs[2e], obs[2e+1]) — the flattening of v_pts_2d/v_pts_2d_to_3d_idx.
 *   K           : 3x3 row-major; only K[0] (fx), K[2], K[5] are used, like g2o's
 *                 CameraParameters at g2o_ba.cpp:219-220.
 *   information : 2x2 row-major (config information_matrix).
 * g2o semantics restated in SURVEY.md App. B: LM (tau 1e-5, <=10 trials), Huber(delta),
 * Schur complement over points when they are free, dense 6F x 6F solve.  F <= 16.
 * stats (optional, 4 doubles): initial robust chi2, final robust chi2, LM iterations run,
 * final lambda. */
int mvo_bundle_adjustment(mvo_ctx *ctx, double *poses_T_w_c, int n_frames, float *points,
                          int n_points, const int32_t *edge_frame, const int32_t *edge_point,
                          const float *obs, int n_edges, const double *K,
                          const double *information, int fix_points, int update_points,
                          double *stats);
/* optimization::optimizeSingleFrame (g2o_ba.cpp:34-145): one pose + its points, identity
 * information, NO robust kernel, 50 iterations in the reference (ctx ba_iterations here). */
int mvo_optimize_single_frame(mvo_ctx *ctx, double *pose_T_w_c, float *points, const float *obs,
                              int n_points, const double *K, int fix_points, int update_points);

/* ---- tracking step ---------------------------------------------------------------------
 * The DOING_TRACKING branch of vo::VisualOdometry::addFrame (src/vo/vo_addFrame.cpp:71-91) over
 * flat arrays, host logic in C++ like the reference:
 *   Frame::calcKeyPoints + calcDescriptors        include/my_slam/vo/frame.h:73-86
 *   getMappointsInCurrentView_                    src/vo/vo.cpp:16-49   (project every map point
 *                                                 with the guess pose, keep z >= 0 and inside image)
 *   matchFeatures(map descriptors, frame)         src/vo/vo.cpp:283-289
 *   poseEstimationPnP_                            src/vo/vo.cpp:293-381 (>= 5 pairs, PnP, T_w_c =
 *                                                 [R|t]^-1, reject if it jumps >= 0.3 from prev)
 *   callBundleAdjustment_                         src/vo/vo.cpp:384-478 (newest <= 5 frames of the
 *                                                 buffer that have >= 3 map links)
 * The map (3-D points + descriptors) is supplied by the caller: keyframe insertion, triangulation
 * and map culling (vo_addFrame.cpp:93-124) are outside the hot path (SURVEY.md §8f).  The pose
 * guess is the reference keyframe's pose, moved forward whenever the camera has travelled more
 * than min_dist_between_two_keyframes from it (checkLargeMoveForAddKeyFrame_, vo.cpp:247-265). */
typedef struct mvo_tracker mvo_tracker;

typedef struct mvo_track_params {
  int32_t match_method;        /* feature_match_method_index_pnp = 1 (config.yaml:75) */
  float match_radius;          /* max_matching_pixel_dist_in_pnp = 50 (:91) */
  int32_t min_pnp_points;      /* kMinPtsForPnP = 5 (vo.cpp:304) */
  double max_dist_to_prev;     /* max_possible_dist_to_prev_keyframe = 0.3 (config.yaml:107 region) */
  double min_dist_keyframe;    /* min_dist_between_two_keyframes = 0.03 */
  int32_t ba_enable;           /* is_enable_ba "true" (:120) */
  int32_t ba_window;           /* num_prev_frames_to_opti_by_ba = 5 (:121) */
  int32_t ba_fix_points;       /* is_ba_fix_map_points "true" (:123) */
  double information[4];       /* information_matrix "1 0 0 1" (:122) */
  int32_t buffer_size;         /* kBuffSize_ = 20 (include/my_slam/vo/vo.h:77) */
  double ba_step_tol;          /* mvo_params::ba_step_tol used for the tracker's BA calls; default 1e-9 */
  int32_t device_resident;     /* 1 (default): map, frame buffer and BA graph stay on the GPU between the stages
                                  (two host synchronisations per frame); 0: every stage through its host-array
                                  C-ABI entry point, as a caller of the reference functions would.  Same results
                                  (tests/test_tracker_gpu.py).  Free map points (ba_fix_points = 0) always take the
                                  host-array path. */
  int32_t pad;
} mvo_track_params;

typedef struct mvo_track_result {
  int32_t n_keypoints;         /* keypoints extracted from the frame */
  int32_t n_candidates;        /* map points projected into the view */
  int32_t n_matches;           /* 3d-2d pairs after matchFeatures */
  int32_t n_inliers;           /* PnP consensus set */
  int32_t pnp_ok;              /* poseEstimationPnP_ return value */
  int32_t ba_frames;           /* frames that entered bundle adjustment */
  int32_t ba_edges;
  int32_t pad;
  double T_w_c_pnp[16];        /* pose right after PnP (before BA) */
} mvo_track_result;

void mvo_default_track_params(mvo_track_params *p);
int mvo_tracker_create(mvo_ctx *ctx, const double *K /* 3x3 */, int rows, int cols,
                       const mvo_track_params *params /* NULL = defaults */, mvo_tracker **out);
void mvo_tracker_destroy(mvo_tracker *t);
/* Replace the map: n points (x,y,z float) with their 32-byte descriptors (MapPoint::pos_,
 * MapPoint::descriptor_).  Copied.  Point index = map point ID, and ids are stable: frames already in the
 * buffer keep their connections by id, so a new map must keep every surviving point at its index (append new points, never
 * reorder); connections to ids >= n leave the BA graph, as connections to erased map points do in the reference
 * (vo.cpp:438-440).  Call mvo_tracker_reset as well when the new map is unrelated to the old one. */
int mvo_tracker_set_map(mvo_tracker *t, const float *pts3d, const uint8_t *desc, int n);
/* Clear the frame buffer and set the reference keyframe pose (camera->world 4x4 row-major). */
int mvo_tracker_reset(mvo_tracker *t, const double *T_w_c_ref);
/* Track one frame.  image: rows x cols x channels, host memory, or device memory when
 * image_on_device != 0.  T_w_c_out receives the frame's pose after PnP (+ BA). */
int mvo_tracker_track(mvo_tracker *t, const uint8_t *image, int channels, size_t stride,
                      int image_on_device, double *T_w_c_out, mvo_track_result *res);
/* Optional look-ahead: hand a FUTURE frame to the tracker's extraction worker (own host thread, own stream) so that
 * its upload, ORB extraction and — for match methods 1/2, which do not depend on the pose — its descriptor matching
 * against the map overlap the tracking of the current frame.  At most two frames in flight next to the one being tracked.  Frames must then be
 * passed to mvo_tracker_track in the same order, with the same image pointer, and the image memory must stay valid
 * and unchanged until that mvo_tracker_track call returns (page-locked host images are copied from directly).  The
 * result is identical to tracking without prefetch. */
int mvo_tracker_prefetch(mvo_tracker *t, const uint8_t *image, int channels, size_t stride,
                         int image_on_device);
/* Pose of the k-th newest buffered frame (k = 0 is the last tracked one) after BA updates. */
int mvo_tracker_frame_pose(const mvo_tracker *t, int k, double *T_w_c);

/* ---- per-kernel timing (CUDA events on the context stream) ------------------------------
 * mask bit i enables event pairs around every launch of kernel class i (see mvo_kernel_name).
 * mvo_timing_read synchronises the stream and ADDS the elapsed milliseconds / launch counts
 * since the last read into ms[] / counts[] (arrays of mvo_kernel_classes() entries). */
int mvo_kernel_classes(void);
const char *mvo_kernel_name(int kernel_class);
int mvo_timing_enable(mvo_ctx *ctx, uint32_t mask);
int mvo_timing_read(mvo_ctx *ctx, double *ms, uint64_t *counts);
/* The same over every context a tracker owns (its extraction runs on two internal contexts). */
int mvo_tracker_timing_enable(mvo_tracker *t, uint32_t mask);
int mvo_tracker_timing_read(mvo_tracker *t, double *ms, uint64_t *counts);
uint64_t mvo_tracker_kernel_launches(const mvo_tracker *t);

/* ---- two-view geometry (SURVEY.md 8f-1, first part) -------------------------------------------
 * geometry::estiMotionByEssential (src/geometry/epipolar_geometry.cpp:17-57): cv::findEssentialMat(pts1, pts2,
 * focal = (K00+K11)/2, pp = (K02, K12), RANSAC, prob, threshold) + E /= E(2,2) + cv::recoverPose + t /= |t|.
 * pts1/pts2: n x 2 float pixels.  Outputs: E (3x3 row-major, E[8] = 1), R (3x3), t (unit 3-vector) with
 * x2 ~ R x1 + t as recoverPose returns them, inliers = indices with mask == 1 after findEssentialMat (ascending;
 * *n_inliers in = capacity, out = count).  `threshold` is config findEssentialMat_threshold (pixels); the
 * reference's `prob` has no counterpart: mvo_params::epi_hypotheses minimal samples are always scored.
 * MVO_ERR_DEGENERATE if n < 8 or no model reaches 8 inliers. */
int mvo_esti_motion_by_essential(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K,
                                 double threshold, double *E, double *R, double *t, int32_t *inliers,
                                 int *n_inliers);
/* geometry::estiMotionByHomography (epipolar_geometry.cpp:90-128): cv::findHomography(pts1, pts2, RANSAC, threshold = 3)
 * + H /= H(2,2) + inliers from its mask + cv::decomposeHomographyMat(H, K) + t /= |t|.  Outputs: H (3x3 pixel
 * homography, H[8] = 1), up to 4 solutions Rs (4 x 9), ts (4 x 3, unit; zero for a pure rotation), normals (4 x 3) with
 * K^-1 H K ~ R + t n^T — the solution SET of cv::decomposeHomographyMat, ordered (a, -a, b, -b) —, *n_solutions,
 * inliers ascending (*n_inliers in = capacity, out = count).  MVO_ERR_DEGENERATE if n < 4 or no model reaches 4 inliers.
 * NOT yet exercised on hardware by the round-1 GPU budget: tests/test_homography_gpu.py runs it in a child process. */
int mvo_esti_motion_by_homography(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K,
                                  double threshold, double *H, double *Rs, double *ts, double *normals,
                                  int *n_solutions, int32_t *inliers, int *n_inliers);
/* geometry::removeWrongRtOfHomography (epipolar_geometry.cpp:59-88) = cv::filterHomographyDecompByVisibleRefpoints on
 * the inlier points (normalised image planes): solutions that put a reference point behind the plane in either view
 * are removed in place; *n_solutions in = count (<= 4), out = survivors.  Host only. */
int mvo_remove_wrong_rt_of_homography(mvo_ctx *ctx, const float *pts_np1, const float *pts_np2, int n,
                                      const int32_t *inliers, int n_inliers, double *Rs, double *ts,
                                      double *normals, int *n_solutions);
/* geometry::doTriangulation (epipolar_geometry.cpp:130-175): cv::triangulatePoints([I|0], [R|t], inlier points on
 * the normalised plane) followed by the division by the fourth coordinate.  pts_np1/pts_np2: n x 2 float,
 * inliers: n_inliers indices into them, pts3d: n_inliers x 3 float (in camera 1). */
int mvo_do_triangulation(mvo_ctx *ctx, const float *pts_np1, const float *pts_np2, int n, const double *R,
                         const double *t, const int32_t *inliers, int n_inliers, float *pts3d);

/* checkEssentialScore / checkHomographyScore (src/geometry/motion_estimation.cpp:501-581, :583-664): ORB-SLAM's
 * symmetric chi-square scores (thresholds 3.841 / 5.991, sigma as in the reference's default 1.0) summed over the
 * inlier list, which is pruned IN PLACE to the points that pass both directions (*n_inliers in/out).  pts: n x 2
 * float pixels.  Host only, no context. */
int mvo_check_essential_score(const double *E21, const double *K, const float *pts_img1, const float *pts_img2,
                              int n, int32_t *inliers, int *n_inliers, double sigma, double *score);
int mvo_check_homography_score(const double *H21, const float *pts_img1, const float *pts_img2, int n,
                               int32_t *inliers, int *n_inliers, double sigma, double *score);
/* The E / H choice of helperEstimatePossibleRelativePosesByEpipolarGeometry (motion_estimation.cpp:134-154):
 * ratio = score_h / (score_e + score_h); > 0.5 picks, among the num_h homography solutions (indices 1..num_h,
 * h_normals = num_h x 3), the one with the largest |normal.z|; otherwise solution 0 (essential).  Host only. */
int mvo_choose_e_or_h(double score_e, double score_h, const double *h_normals, int num_h, int *best_sol,
                      double *ratio);
/* The same with the threshold as an argument (mvo_params::eh_ratio_threshold is what mvo_estimate_relative_poses passes). */
int mvo_choose_e_or_h_thr(double score_e, double score_h, const double *h_normals, int num_h, double threshold,
                          int *best_sol, double *ratio);

/* helperEstimatePossibleRelativePosesByEpipolarGeometry (motion_estimation.cpp:10-158) over flat arrays of MATCHED
 * points (pts_img1[i] <-> pts_img2[i], n x 2 float pixels): solution 0 is the essential-matrix motion, solutions
 * 1..num_solutions-1 the homography motions that survive removeWrongRtOfHomography (calc_homo != 0); every solution's
 * inliers are triangulated (camera 1 frame); motion_cam2_to_cam1 == 0 inverts every (R, t) afterwards (basics::invRt);
 * `best` is the E/H choice.  inliers: 5 x n int32 (row s holds n_inliers[s] indices), pts3d: 5 x n x 3 float. */
typedef struct mvo_two_view_solutions {
  int32_t num_solutions, best;
  int32_t n_inliers[5];
  int32_t pad_;
  double R[5][9], t[5][3], normal[5][3];   /* normal of solution 0 is zero (the reference pushes an empty cv::Mat) */
  double E[9], H[9];
  double score_e, score_h, ratio;
} mvo_two_view_solutions;
int mvo_estimate_relative_poses(mvo_ctx *ctx, const float *pts_img1, const float *pts_img2, int n, const double *K,
                                int calc_homo, int motion_cam2_to_cam1, mvo_two_view_solutions *sol,
                                int32_t *inliers, float *pts3d);
/* helperEstimatePossibleRelativePosesByEpipolarGeometry with the homography branch (what the reference's callers use:
 * vo.cpp:65-75, test_epipolor_geometry.cpp:105-113) for the matched frame pairs of a batch, entirely on the device: pair p gets
 * what mvo_estimate_relative_poses(calc_homo = 1, motion_cam2_to_cam1) returns for its points.
 * d_kpts / d_counts / batch / cap / d_pairs / d_matches / d_n_matches: as for mvo_esti_motion_by_essential_batch_dev (same
 * layouts, same per-pair input checks); pair p's correspondences are kpts[query frame][m.query_idx].pt <->
 * kpts[train frame][m.train_idx].pt in match-list order.  K: host 3x3.  The thresholds are those of a single call:
 * mvo_params::essential_threshold, homography_threshold, eh_ratio_threshold, epi_hypotheses and pnp_seed.
 * d_res[p]: status MVO_OK or the mvo_status of that pair alone, n_matches = d_n_matches[p] as given, and on MVO_OK `sol`
 * byte-identical to what mvo_estimate_relative_poses writes (every byte: unused solution slots, normal[0] and pad_ are 0; H and
 * score_h are 0 when the homography RANSAC found no model).  A failed pair writes its status and n_matches only (not the rest
 * of its record, its inlier rows or its points):
 *   MVO_ERR_INVALID_ARG  a frame index outside [0, batch), a match count outside [0, cap], a keypoint index outside its frame;
 *   MVO_ERR_DEGENERATE   fewer than 8 matches, or no essential matrix reaches 8 inliers.
 * A homography that reaches fewer than 4 inliers is not a failure: num_solutions = 1, as in the single call.
 * Solution s of pair p: its n_inliers[s] inlier indices at d_inliers + (p * 5 + s) * cap (row 0 the essential inliers, rows
 * 1..num_solutions-1 the homography inliers), its triangulated inliers at d_pts3d + (p * 5 + s) * cap * 3 (d_pts3d NULL: no
 * triangulation); rows past num_solutions are not written.
 * NaN: ratio = score_h / (score_e + score_h) is 0 / 0 when both scores are 0.  The single call computes it on x86-64, whose
 * default NaN is 0xFFF8000000000000; the device writes that bit pattern for a NaN score_e, score_h or ratio, so such a pair
 * is byte-identical too (points with NaN coordinates, whose payloads the host would propagate, are outside this promise).
 * MVO_ERR_INVALID_ARG: a null pointer, fx or fy <= 0, a singular K.  MVO_ERR_UNSUPPORTED: cap > 6400, n_pairs > 65535,
 * n_pairs x epi_hypotheses > 2^22 (80 bytes of scratch per hypothesis, shared by the essential and the homography half).
 * Asynchronous on the context stream: ten kernel launches (eleven with d_pts3d) whatever n_pairs is, no host synchronisation
 * except when the call's own scratch buffer of the context has to grow. */
typedef struct mvo_relative_poses_result {
  int32_t status;              /* MVO_OK, or the mvo_status the per-pair call would have returned */
  int32_t n_matches;           /* the pair's match count, d_n_matches[p] */
  mvo_two_view_solutions sol;  /* byte-identical to what mvo_estimate_relative_poses writes */
} mvo_relative_poses_result;
int mvo_estimate_relative_poses_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                          const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches,
                                          const int32_t *d_n_matches, const double *K, int motion_cam2_to_cam1,
                                          mvo_relative_poses_result *d_res, int32_t *d_inliers, float *d_pts3d);

/* ---- host-side decisions of the initialisation / keyframe logic (SURVEY.md 8f-2; no context, no GPU) ----------
 * retainGoodTriangulationResult_ (src/vo/vo.cpp:181-244): triangulation angle (degrees, with the reference's
 * pi = 3.1415926) of every point between the two camera centres; points below min_triang_angle or above
 * max_ratio x the median angle are dropped.  keep: surviving indices, angles: their angles (n capacity each). */
int mvo_retain_good_triangulation(const float *pts3d_in_curr, int n, const double *T_w_c_curr, const double *T_w_c_ref,
                                  double min_triang_angle, double max_ratio_to_median, int32_t *keep, double *angles,
                                  int *n_keep);
/* The depth normalisation of estimateMotionAnd3DPoints_ (vo.cpp:96-110): scale = assumed_mean_depth / mean z;
 * points (n x 3 float) and t_curr_to_prev (3) are scaled in place. */
int mvo_normalize_init_depth(float *pts3d, int n, double *t_curr_to_prev, double assumed_mean_depth, double *scale);
/* isVoGoodToInit_ (vo.cpp:113-172) over the matched keypoint positions (n_matches x 2 each, row i = one match) and
 * the triangulation angles that survived: enough matches, mean pixel displacement and median angle above their
 * thresholds (config min_inlier_matches, min_pixel_dist, min_median_triangulation_angle). */
int mvo_is_vo_good_to_init(const float *kpts_ref_xy, const float *kpts_curr_xy, int n_matches,
                           const double *triangulation_angles, int n_angles, int min_inlier_matches, double min_pixel_dist,
                           double min_median_triangulation_angle, int *good, double *mean_pixel_dist, double *median_angle);
/* checkLargeMoveForAddKeyFrame_ (vo.cpp:247-265): translation of ref^-1 * curr above min_dist_between_two_keyframes. */
int mvo_check_large_move(const double *T_w_c_curr, const double *T_w_c_ref, double min_dist_between_two_keyframes, int *large,
                         double *moved_dist, double *rotated_angle);

/* ---- the whole VisualOdometry state machine (SURVEY.md 8f-2) ---------------------------------------------------
 * vo::VisualOdometry::addFrame (src/vo/vo_addFrame.cpp:10-142) with the reference's containers (Frame, MapPoint, Map as
 * std::unordered_map, the 20-frame buffer) on the host and every numeric stage on the GPU through the entry points
 * above: BLANK -> first keyframe; DOING_INITIALIZATION -> match against the first keyframe, two-view motion (E / H),
 * triangulation, depth normalisation, isVoGoodToInit_ -> map + second keyframe; DOING_TRACKING -> map points in view,
 * match, RANSAC PnP, windowed BA, and on a large move a new keyframe (match, essential inliers, triangulation with the
 * known motion, pushCurrPointsToMap_, optimizeMap_).  This is the slower, complete counterpart of the mvo_tracker_* calls, which
 * keep a caller-supplied map resident on the GPU and do no map maintenance.
 * Where the reference would abort — fewer than 5 matched points handed to findEssentialMat, an empty rvec after a
 * failed solvePnPRansac — the frame is skipped / the PnP reported as failed. */
typedef struct mvo_vo mvo_vo;

typedef struct mvo_vo_params {
  mvo_track_params track;              /* tracking keys (match method / radius for PnP, BA window, keyframe distance ...);
                                          device_resident = 1 (default): tracked frames run through the device-resident
                                          tracker with the map kept in HBM (re-uploaded when a keyframe changes it) */
  int32_t match_method_init;           /* feature_match_method_index_initialization = 1 */
  float max_match_dist_init;           /* max_matching_pixel_dist_in_initialization = 100 */
  float max_match_dist_triangulation;  /* max_matching_pixel_dist_in_triangulation = 100 */
  int32_t init_calc_homography;        /* is_calc_homo = true (vo.cpp:68) */
  int32_t min_inlier_matches;          /* 15 */
  int32_t pad;
  double essential_threshold;          /* findEssentialMat_threshold = 1.0 (initialisation and keyframe branch) */
  double min_triang_angle;             /* 1.0 */
  double max_ratio_angle_to_median;    /* max_ratio_between_max_angle_and_median_angle = 20 */
  double min_pixel_dist;               /* 50 */
  double min_median_triangulation_angle; /* 2.0 */
  double assumed_mean_depth_init;      /* assumed_mean_pts_depth_during_vo_init = 0.8 */
} mvo_vo_params;

/* The initialisation check of the state machine (estimateMotionAnd3DPoints_ + isVoGoodToInit_, src/vo/vo.cpp:53-172) for the
 * matched frame pairs of a batch, entirely on the device: the step after mvo_estimate_relative_poses_batch_dev.  Pair p = (query
 * frame, train frame) is (reference keyframe, candidate frame); its record says what the state machine decides when that candidate
 * is the frame being added and T_w_c_ref is the reference keyframe's pose:
 *   the chosen solution's inlier matches (img_idx = -1), its triangulated points moved into the candidate's camera (transCoord),
 *   T_w_c = T_w_c_ref * [R|t]^-1, retainGoodTriangulationResult_ (angles, their median, the drop by angle), the depth
 *   normalisation when at least 20 points survive, and the three criteria of isVoGoodToInit_.
 * Inputs: d_kpts / d_counts / batch / cap / d_pairs / n_pairs / d_matches / d_n_matches exactly as given to
 * mvo_estimate_relative_poses_batch_dev, and what it wrote (d_rp, d_rp_inliers, d_rp_pts3d, same row layouts).  Precondition:
 * that call was made with motion_cam2_to_cam1 = 1 and a non-NULL d_pts3d (the state machine's call).  T_w_c_ref: host 4x4
 * row-major; vp: host, the fields min_triang_angle, max_ratio_angle_to_median, min_inlier_matches, min_pixel_dist,
 * min_median_triangulation_angle and assumed_mean_depth_init (init_calc_homography is not read: the inputs are those of the
 * homography branch, the reference's is_calc_homo = true).
 * Outputs of pair p: d_out[p]; inliers_matches_for_3d_ at d_kept + p * cap, inliers_pts3d_ (candidate camera, after the
 * normalisation) at d_kept_pts3d + p * cap * 3 and triangulation_angles_of_inliers_ at d_kept_angles + p * cap, n_kept of each, in
 * the reference's order; nothing past n_kept is written.
 * Per pair: a relative-poses status MVO_ERR_DEGENERATE gives usable = 0, good = 0, best_sol = -1, T_w_c = T_w_c_ref and status
 * MVO_OK (as the state machine treats it); any other non-MVO_OK status is propagated.  MVO_ERR_INVALID_ARG for that pair alone,
 * checked before anything is read through the value checked: a frame index outside [0, batch), d_n_matches[p] outside [0, cap],
 * best outside [0, num_solutions) or num_solutions outside [1, 5], n_inliers[best] outside [0, d_n_matches[p]], an inlier index
 * outside [0, d_n_matches[p]), a keypoint index of an inlier match outside its frame.  A failed pair writes its status only.
 * Numerics: the host's order of operations, without contraction; every sum over points is sequential in list order.  Each
 * angle uses the device's acos (2 ulp), the one step that is not the host's (glibc) bit for bit: the angles and median_angle
 * are within a few ulp of the state machine's, and everything else is byte-identical unless an angle lies that close to a
 * threshold.  A NaN angle, median_angle or mean_pixel_dist (0 / 0 when n_kept = 0) has x86-64's default NaN bits.
 * MVO_ERR_INVALID_ARG: a null pointer, a T_w_c_ref or vp value that is not finite, batch or cap < 1, n_pairs < 0.
 * MVO_ERR_UNSUPPORTED: cap > 6400 or n_pairs > 65535 (the limits of mvo_estimate_relative_poses_batch_dev), or a library built
 * without the kernel's translation unit.  Asynchronous on the context stream: one kernel launch whatever n_pairs is, no host
 * synchronisation. */
typedef struct mvo_init_candidate_result {
  int32_t status;      /* MVO_OK, or the pair's mvo_status */
  int32_t usable;      /* estimateMotionAnd3DPoints_ got past the two-view step (0: degenerate pair) */
  int32_t good;        /* isVoGoodToInit_ */
  int32_t best_sol;    /* the E/H choice of the relative-poses record; -1 when not usable */
  int32_t n_inliers;   /* inliers of the chosen solution (inliers_matches_with_ref_) */
  int32_t n_kept;      /* after retainGoodTriangulationResult_ (inliers_matches_for_3d_) */
  int32_t normalized;  /* n_kept >= 20: depth normalised (vo.cpp:97-108) */
  int32_t pad;
  double scale;                          /* assumed_mean_depth_init / mean depth; 0 when not normalised */
  double mean_pixel_dist, median_angle;  /* what isVoGoodToInit_ compares; median_angle = 0 when n_kept = 0 */
  double t_curr_to_prev[3];              /* the chosen t after the depth scaling */
  double T_w_c[16];                      /* the candidate's pose as estimateMotionAnd3DPoints_ leaves it (T_w_c_ref if not usable) */
} mvo_init_candidate_result;
int mvo_vo_init_candidates_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                     const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches, const int32_t *d_n_matches,
                                     const mvo_relative_poses_result *d_rp, const int32_t *d_rp_inliers, const float *d_rp_pts3d,
                                     const double *T_w_c_ref, const mvo_vo_params *vp, mvo_init_candidate_result *d_out,
                                     mvo_dmatch *d_kept, float *d_kept_pts3d, double *d_kept_angles);

/* The new map points of the state machine's keyframe branch (vo_addFrame.cpp:93-124: helperFindInlierMatchesByEpipolarCons,
 * helperTriangulatePoints with the known motion, retainGoodTriangulationResult_, pushCurrPointsToMap_) for the matched frame
 * pairs of a batch, entirely on the device: the step after mvo_esti_motion_by_essential_batch_dev.  Pair p = (query frame, train
 * frame) is (reference keyframe, current frame), as matchFeatures(ref_->descriptors_, curr_->descriptors_); its record says what
 * the state machine computes when that frame is inserted as a keyframe with those two poses:
 *   the essential RANSAC's inlier matches (img_idx = -1), the known motion T_curr_to_prev = T_w_c_curr^-1 * T_w_c_ref
 *   (getMotionFromFrame1to2), the inliers triangulated with it on pixel2CamNormPlane points as mvo_do_triangulation does and moved
 *   into the current camera (transCoord), retainGoodTriangulationResult_ (angles, their median, the drop by angle), and for every
 *   kept point the map point's world position (preTranslatePoint3f with T_w_c_curr) and unit viewing direction (pos - camera
 *   centre, normalised).
 * Inputs: d_kpts / d_counts / batch / cap / d_pairs / n_pairs / d_matches / d_n_matches exactly as given to
 * mvo_esti_motion_by_essential_batch_dev, and what it wrote (d_ess, d_ess_inliers; its d_pts3d is not needed and may have been
 * NULL).  d_T_w_c: batch x 16 doubles on the device, each frame's camera->world pose (row-major), indexed like d_kpts.  K: host
 * 3x3.  vp: host, the fields min_triang_angle and max_ratio_angle_to_median.
 * Outputs of pair p: d_out[p]; inliers_matches_for_3d_ at d_kept + p * cap, inliers_pts3d_ (current camera) at d_kept_pts3d +
 * p * cap * 3, triangulation_angles_of_inliers_ at d_kept_angles + p * cap, and optionally (NULL: not written) the world positions
 * at d_kept_world + p * cap * 3 and the viewing directions at d_kept_norm + p * cap * 3, n_kept of each in the reference's order;
 * nothing past n_kept is written, with one exception: the d_kept_pts3d row holds the pair's triangulated inliers between the
 * second and the third launch (the call has no scratch memory of its own), so its entries n_kept .. n_inliers - 1 are left
 * unspecified; nothing past n_inliers is written there.  A position and a direction are written for every kept point: whether the reference keypoint
 * already has a map point (which the reference then reuses) is a question for the caller's map.
 * Per pair: an essential status MVO_ERR_DEGENERATE gives usable = 0 and status MVO_OK (insert_keyframe returns before adding the
 * keyframe); any other non-MVO_OK status is propagated.  MVO_ERR_INVALID_ARG for that pair alone, checked before anything is read
 * through the value checked: a frame index outside [0, batch), d_n_matches[p] outside [0, cap] (both also for a degenerate
 * pair), and for a pair whose essential status is MVO_OK n_inliers outside [0, d_n_matches[p]], an inlier index outside
 * [0, d_n_matches[p]), a keypoint index of an inlier match outside its frame, a non-finite entry in either frame's pose.  A failed
 * pair writes its status only.
 * Numerics: the triangulation is the device's own (the arithmetic of mvo_do_triangulation); everything the state machine computes
 * on the host is restated in the host's order of operations, without contraction.  Each angle uses the device's acos (2 ulp),
 * the one step that is not the host's (glibc) bit for bit: the angles and median_angle are within a few ulp of the state
 * machine's, and everything else is byte-identical unless an angle lies that close to a threshold.  A NaN angle, median_angle or
 * direction has x86-64's default NaN bits.
 * MVO_ERR_INVALID_ARG: a null required pointer, fx or fy not finite and > 0, a vp threshold that is not finite, batch or cap < 1,
 * n_pairs < 0.  MVO_ERR_UNSUPPORTED: cap > 6400 or n_pairs > 65535 (the limits of mvo_esti_motion_by_essential_batch_dev), or a
 * library built without the kernels' translation unit.  Asynchronous on the context stream: three kernel launches whatever
 * n_pairs is (the checks and the known motion, the triangulation, the retain step and the map points), no host
 * synchronisation, no scratch memory of the context (see d_kept_pts3d). */
typedef struct mvo_keyframe_points_result {
  int32_t status;      /* MVO_OK, or the pair's mvo_status */
  int32_t usable;      /* 0: the essential RANSAC was degenerate, the state machine inserts no keyframe */
  int32_t n_matches;   /* matches_with_ref_ (mvo_vo_frame_info::kf_matches) */
  int32_t n_inliers;   /* inliers_matches_with_ref_ */
  int32_t n_kept;      /* inliers_matches_for_3d_ (mvo_vo_frame_info::kf_new_points) */
  int32_t pad;
  double median_angle;                        /* retainGoodTriangulationResult_'s median (element n / 2); 0 when n_inliers = 0 */
  double R_curr_to_prev[9], t_curr_to_prev[3];   /* the known motion the triangulation used */
} mvo_keyframe_points_result;
int mvo_vo_keyframe_points_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                     const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches, const int32_t *d_n_matches,
                                     const mvo_two_view_result *d_ess, const int32_t *d_ess_inliers, const double *d_T_w_c,
                                     const double *K, const mvo_vo_params *vp, mvo_keyframe_points_result *d_out,
                                     mvo_dmatch *d_kept, float *d_kept_pts3d, double *d_kept_angles, float *d_kept_world,
                                     double *d_kept_norm);
/* The first step of the state machine's tracking branch (poseEstimationPnP_) for many frames at once, entirely on the device:
 * for every job (frame, guess pose) what pose_estimation_pnp computes before solvePnPRansac — getMappointsInCurrentView_, the
 * match of the map points in view against the frame (matchFeatures with the tracking method and radius, xiang_gao_ratio /
 * lowe_ratio of the context) and the 3D-2D pairs.  The batched PnP that consumes them is mvo_vo_pnp_batch_dev.
 * Inputs: d_kpts / d_desc / d_counts / batch / cap in the layout of mvo_orb_extract_batch_dev; d_frames: n_jobs int32 frame
 * indices; d_T_w_c_guess: n_jobs x 16 doubles, the guess pose of each job (camera->world, row-major; the state machine uses the
 * reference keyframe's pose); d_map_pts / d_map_desc: one map, n_map points (float x, y, z) and descriptors, whose position is
 * the map index (the state machine's container order, as mvo_vo_get_map returns it).  K: host 3x3; rows / cols: the image size
 * of the inside test; method_index / radius: mvo_vo_params::track.match_method / match_radius.
 * Job j: T_c_w = inverse of the guess; every map point in index order is projected (preTranslatePoint3f, z < 0 rejected,
 * cam2pixel) and kept when 0 < u < cols and 0 < v < rows; the candidates, in map order, are matched as the query set of
 * mvo_match_features against the frame's keypoints (method 3: candidate pixels against keypoint pts within radius).
 * Outputs of job j (nothing past a count is written):
 *   d_out[j]; d_cand + j * n_map: the candidates' map indices (n_candidates); d_cand_xy + j * n_map * 2: their projected pixels
 *   (optional, NULL: not written); d_matches + j * cap: matches_with_map_, byte-identical to what the state machine's matcher
 *   returns (query_idx = rank in the candidate list, train_idx = keypoint); d_pts3d + j * cap * 3 / d_pts2d + j * cap * 2: the map
 *   point and keypoint pt of every match, the solvePnPRansac inputs (optional, NULL: not written; both or neither).
 * Per job: no candidates, no keypoints, or method 2 with fewer than 2 keypoints: status MVO_OK with 0 matches (the state machine
 * skips the matcher there).  Counts are clamped to [0, cap].  MVO_ERR_INVALID_ARG for that job alone: a frame index outside
 * [0, batch), a non-finite entry of its guess pose.  MVO_ERR_UNSUPPORTED for that job alone when the device filter cannot finish
 * it: more map points in view pass the distance threshold than the filter's capacity (2048 up to 8192, the power of two that
 * covers cap and n_map), or libstdc++'s introsort would heapsort at its depth limit; the state machine would still produce a
 * match list for such a frame.  A failed job writes its status only.
 * MVO_ERR_INVALID_ARG: a null required pointer (d_desc, d_counts, d_frames, d_T_w_c_guess, K, d_out, d_cand, d_matches, and
 * d_map_pts / d_map_desc when n_map > 0, d_kpts for method 3 or with d_pts2d), fx or fy not finite and > 0, rows or cols < 1, a method index outside
 * 1..3, batch or cap < 1, n_jobs or n_map < 0, only one of d_pts3d / d_pts2d.  MVO_ERR_UNSUPPORTED: cap > 8192, n_map > 65535,
 * n_jobs > 65535, n_jobs * n_map > 2^26 (the matcher keys of every job).  Asynchronous on the context stream: methods 1 and 2
 * make two kernel launches (the matcher of every map point against every job's frame, then the filter, which projects the
 * map), method 3 three (the projection first: the radius gate needs the pixels), whatever n_jobs is; n_map = 0 makes one (the
 * filter) and n_jobs = 0 none.  No host synchronisation once the context's scratch has reached its size. */
typedef struct mvo_map_matches_result {
  int32_t status;        /* MVO_OK, or the job's mvo_status */
  int32_t n_candidates;  /* map points in view (mvo_vo_frame_info::n_candidates) */
  int32_t n_matches;     /* matches_with_map_ before PnP (mvo_vo_frame_info::n_matches) */
  int32_t pad;
} mvo_map_matches_result;
int mvo_vo_map_matches_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const uint8_t *d_desc, const int32_t *d_counts, int batch,
                                 int cap, const int32_t *d_frames, const double *d_T_w_c_guess, int n_jobs, const float *d_map_pts,
                                 const uint8_t *d_map_desc, int n_map, const double *K, int rows, int cols, int method_index,
                                 float radius, mvo_map_matches_result *d_out, int32_t *d_cand, float *d_cand_xy, mvo_dmatch *d_matches,
                                 float *d_pts3d, float *d_pts2d);

/* The rest of poseEstimationPnP_ on the device for every job of a map-matches batch: solvePnPRansac with its least-squares refit,
 * the inlier matches (matches_with_map_ after the swap), T_w_c = [R|t]^-1 and the jump check against the previous frame.
 * Inputs: d_mm / d_matches / d_pts3d / d_pts2d / n_jobs / cap exactly as mvo_vo_map_matches_batch_dev wrote them (job j's pairs at
 * + j * cap); d_T_w_c_prev: n_jobs x 16 doubles, each job's previous-frame pose (prev_->T_w_c_ at PnP time); K: host 3x3; from tp
 * the call reads min_pnp_points and max_dist_to_prev; the context supplies pnp_hypotheses, pnp_reproj_error, pnp_seed and
 * pnp_refine_iters (pnp_mode 0 only).
 * Job j: n_matches < min_pnp_points gives status MVO_OK, pnp_ok 0, no model and T_w_c = T_w_c_prev.  Otherwise the job gets the
 * consensus set and refit that a single mvo_solve_pnp_ransac call on its pairs returns (the same hypotheses, counts and arg-max;
 * the refit's sums run in the order of a single device call on cap pairs); no model is not an error (pnp_ok 0).  T_w_c is taken
 * from Rt without a Rodrigues round trip, and trans_dist(T_w_c, T_w_c_prev) >= max_dist_to_prev (host operation order, no
 * contraction) rejects the pose: T_w_c = T_w_c_prev.  A rejected job still writes n_inliers and its rows.
 * Outputs of job j (nothing past a count is written): d_out[j]; d_inliers + j * cap: the consensus set as ascending indices into
 * the match list (n_inliers); d_kept + j * cap: those matches (optional, NULL: not written).
 * Per job, status only: the map-matches status when it is not MVO_OK; MVO_ERR_INVALID_ARG for n_matches outside [0, cap] or a
 * non-finite entry of its T_w_c_prev.
 * MVO_ERR_INVALID_ARG: a null required pointer (all but d_kept), fx or fy not finite and > 0, cap < 1, n_jobs < 0, a non-finite
 * max_dist_to_prev.  MVO_ERR_UNSUPPORTED: pnp_mode 1, cap > 8192, n_jobs > 65535, n_jobs * pnp_hypotheses > 2^22.
 * Asynchronous on the context stream: five kernel launches (hypotheses, scoring, consensus set, refit, record) whatever n_jobs
 * is, none for n_jobs = 0.  No host synchronisation once the context's scratch has reached its size. */
typedef struct mvo_vo_pnp_result {
  int32_t status;     /* MVO_OK, or the job's mvo_status */
  int32_t pnp_ok;     /* poseEstimationPnP_'s is_pnp_good (mvo_vo_frame_info::pnp_ok) */
  int32_t n_matches;  /* pairs handed to solvePnPRansac (the map-matches record's n_matches) */
  int32_t n_inliers;  /* consensus-set size (mvo_vo_frame_info::n_inliers); 0 without a model */
  int32_t best;       /* winning hypothesis, -1 without a model */
  int32_t pad[3];
  double Rt[12];      /* world->camera R (row-major), t after the refit; identity without a model */
  double T_w_c[16];   /* curr_->T_w_c_ when poseEstimationPnP_ returns (mvo_vo_frame_info::T_w_c_pnp) */
} mvo_vo_pnp_result;  /* 256 bytes */
int mvo_vo_pnp_batch_dev(mvo_ctx *ctx, const mvo_map_matches_result *d_mm, const mvo_dmatch *d_matches, const float *d_pts3d,
                         const float *d_pts2d, int n_jobs, int cap, const double *d_T_w_c_prev, const double *K,
                         const mvo_track_params *tp, mvo_vo_pnp_result *d_out, int32_t *d_inliers, mvo_dmatch *d_kept /* optional */);

typedef struct mvo_vo_frame_info {
  int32_t frame_id, state_in, state_out;   /* states: 0 BLANK, 1 DOING_INITIALIZATION, 2 DOING_TRACKING (vo.h:52-58) */
  int32_t keyframe;                        /* this frame became a keyframe */
  int32_t n_keypoints, n_matches, n_candidates, n_inliers;
  int32_t pnp_ok, ba_frames, ba_edges;
  int32_t best_sol;                        /* initialisation: chosen two-view solution (0 = essential), -1 = none */
  int32_t map_points;                      /* map size after the frame */
  int32_t kf_matches, kf_new_points, pad;  /* keyframe branch: matches with the previous keyframe, points kept by
                                              retainGoodTriangulationResult_ */
  double score_e, score_h, eh_ratio, init_mean_pixel_dist, init_median_angle;
  double T_w_c_pnp[16];                    /* tracking: pose right after PnP (before BA) */
} mvo_vo_frame_info;

void mvo_vo_default_params(mvo_vo_params *p);
int mvo_vo_create(mvo_ctx *ctx, const double *K /* 3x3 */, int rows, int cols, const mvo_vo_params *params /* NULL = defaults */,
                  mvo_vo **out);
void mvo_vo_destroy(mvo_vo *v);
/* addFrame: image rows x cols x channels (3 = BGR, 1 = gray) in host memory.  T_w_c_out = the frame's pose when the
 * call returns (run_vo.cpp:137 records exactly this), info optional.  When the call fails the frame is not kept: the
 * frame buffer (mvo_vo_frame_pose / mvo_vo_frame_data) only holds frames whose call returned MVO_OK. */
int mvo_vo_add_frame(mvo_vo *v, const uint8_t *image, int channels, size_t stride, double *T_w_c_out, mvo_vo_frame_info *info);
/* The same with the image optionally already in device memory (image_on_device != 0). */
int mvo_vo_add_frame_ex(mvo_vo *v, const uint8_t *image, int channels, size_t stride, int image_on_device, double *T_w_c_out,
                        mvo_vo_frame_info *info);
/* Optional look-ahead (device-resident mode; a no-op otherwise): hand the NEXT frame over so that its upload, ORB extraction
 * and descriptor matching against the map overlap the current frame (mvo_tracker_prefetch).  Frames must then be added in
 * the same order with the same image pointer; at most two frames in flight next to the one being added (three between calls); results
 * are identical. */
int mvo_vo_prefetch(mvo_vo *v, const uint8_t *image, int channels, size_t stride, int image_on_device);
/* The main loop of run_vo.cpp (:107-140: for every image: createFrame, vo->addFrame, cam_pose_history.push_back) over n_frames images
 * that are already in memory, with the look-ahead of mvo_vo_prefetch applied to frame i + 1 while frame i is added.  images[i]:
 * rows x cols x channels, host or device memory alike for all frames; T_w_c_out: n_frames x 16 doubles (the pose of every
 * frame when its addFrame returned); infos: n_frames records or NULL; *n_done = frames added when the call returns (it stops at
 * the first frame whose addFrame fails and returns that code; frames handed over ahead of it stay queued: add them in order or call
 * mvo_vo_reset).  Results equal n_frames calls of mvo_vo_add_frame_ex. */
int mvo_vo_run_sequence(mvo_vo *v, const uint8_t *const *images, int n_frames, int channels, size_t stride, int images_on_device,
                        double *T_w_c_out, mvo_vo_frame_info *infos, int *n_done);
/* 1 when the tracking branch runs through the device-resident tracker (mvo_vo_params::track.device_resident, fixed map
 * points), 0 when every stage goes through its host-array entry point. */
int mvo_vo_device_resident(const mvo_vo *v);
/* Back to the BLANK state (empty map, no frames, ids restart at 0) keeping the allocations: the next frame is the first
 * frame of a new sequence.  Frames handed to mvo_vo_prefetch but not added yet are dropped. */
int mvo_vo_reset(mvo_vo *v);
/* Kernel launch count / per-kernel-class timing over every context the state machine owns (see mvo_timing_*). */
uint64_t mvo_vo_kernel_launches(const mvo_vo *v);
int mvo_vo_timing_enable(mvo_vo *v, uint32_t mask);
int mvo_vo_timing_read(mvo_vo *v, double *ms, uint64_t *counts);
int mvo_vo_is_initialized(const mvo_vo *v);                  /* VisualOdometry::isInitialized */
int mvo_vo_map_size(const mvo_vo *v);
int mvo_vo_num_keyframes(const mvo_vo *v);
/* The map in container order (VisualOdometry::getMap): ids, positions (x 3 float), descriptors (x 32), colours (x 3,
 * r g b); any output may be NULL.  MVO_ERR_CAPACITY (with *n = map size) when cap is too small. */
int mvo_vo_get_map(const mvo_vo *v, int32_t *ids, float *pts3d, uint8_t *desc, uint8_t *rgb, int cap, int *n);
/* Pose of the k-th newest buffered frame (k = 0: the last one) including later BA updates. */
int mvo_vo_frame_pose(const mvo_vo *v, int k, double *T_w_c);
/* What run_vo.cpp's display code reads from a Frame (run_vo.cpp:184-232, 286-300): `which` = k-th newest buffered frame
 * (0 = the one just added) or -1 = VisualOdometry::getPrevRef(); `what` selects the member.  *n = element count;
 * MVO_ERR_CAPACITY when cap is too small. */
enum {
  MVO_VO_KEYPOINTS = 0,          /* keypoints_                 mvo_keypoint[] */
  MVO_VO_DESCRIPTORS = 1,        /* descriptors_               32 bytes each */
  MVO_VO_MATCHES_WITH_REF = 2,   /* matches_with_ref_          mvo_dmatch[] */
  MVO_VO_MATCHES_WITH_MAP = 3,   /* matches_with_map_ (PnP inliers after tracking)  mvo_dmatch[] */
  MVO_VO_INLIERS_PTS3D = 4,      /* inliers_pts3d_ (in the frame's camera coordinates)  3 floats each */
  MVO_VO_FRAME_ID = 5            /* id_                        one int32 */
};
int mvo_vo_frame_data(const mvo_vo *v, int which, int what, void *out, int cap, int *n);
int mvo_vo_has_keyframe(const mvo_vo *v, int frame_id);       /* Map::hasKeyFrame */

/* ---- on-disk formats either side of the path (host only; SURVEY.md 8f-3) -------------------
 * Trajectory file of my_slam::vo::writePoseToFile / readPoseFromFile (src/vo/vo_io.cpp:51-120): one pose
 * per line, "tx ty tz R00 R10 R20 R01 R11 R21 R02 R12 R22", C++ stream defaults (6 significant digits).
 * T_list: n x 16 doubles, row-major 4x4 camera->world.  mvo_read_pose_file returns MVO_ERR_CAPACITY (with
 * *n = poses in the file) when cap is too small. */
int mvo_write_pose_file(const char *filename, const double *T_list, int n);
int mvo_read_pose_file(const char *filename, double *T_list, int cap, int *n);
/* readImagePaths (vo_io.cpp:12-37): dataset_dir + image_formatting with one %0Nd directive ("/rgb_%05d.png",
 * run_vo.cpp:90) applied to `index`. */
int mvo_image_path(const char *dataset_dir, const char *image_formatting, int index, char *out, size_t cap);
/* config/config.yaml (OpenCV "%YAML:1.0" dialect as the shipped file uses it: flat scalars, one nesting level
 * for the dataset sections — addressed as "section/key" —, optional double quotes, # comments), the file
 * my_slam::basics::Config reads (src/basics/config.cpp:12-47).  get_int rounds like cv::FileNode -> int,
 * get_bool follows Config::getBool ("true"/"True").  A missing key returns MVO_ERR_INVALID_ARG (the
 * reference throws std::runtime_error, config.cpp:35). */
typedef struct mvo_config mvo_config;
int mvo_config_load(const char *filename, mvo_config **out);
void mvo_config_free(mvo_config *c);
int mvo_config_get_string(const mvo_config *c, const char *key, char *out, size_t cap);
int mvo_config_get_double(const mvo_config *c, const char *key, double *out);
int mvo_config_get_int(const mvo_config *c, const char *key, int *out);
int mvo_config_get_bool(const mvo_config *c, const char *key, int *out);
/* Fill the parameters the hot path latches from the config (any of p / tp / K9 may be NULL): ORB, grid
 * selection and match ratios (feature_match.cpp:16-23,56-58,137-139), the tracking keys of vo.cpp, and the
 * 3x3 intrinsics of the dataset selected by dataset_name (readCameraIntrinsics, vo_io.cpp:40-49).  Fields
 * without a config key (PnP hypotheses, BA iterations, ...) are left as they are. */
int mvo_config_apply(const mvo_config *c, mvo_params *p, mvo_track_params *tp, double *K9);
/* The same for the state machine: vp->track as above plus the initialisation / triangulation keys of vo.cpp and
 * vo_addFrame.cpp. */
int mvo_config_apply_vo(const mvo_config *c, mvo_vo_params *vp);

#ifdef __cplusplus
}
#endif
#endif /* MVO_H_ */
