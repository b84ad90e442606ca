// Host-side decisions of the VO initialisation and keyframe logic that are plain arithmetic on a few hundred values
// in the reference (SURVEY.md §8f-2), restated over flat arrays:
//   retainGoodTriangulationResult_   reference src/vo/vo.cpp:181-244
//   the depth normalisation of estimateMotionAnd3DPoints_   src/vo/vo.cpp:96-110
//   isVoGoodToInit_                  src/vo/vo.cpp:113-172
//   checkLargeMoveForAddKeyFrame_    src/vo/vo.cpp:247-265
// No GPU work and no context: double arithmetic in the reference's order of operations.  The per-point terms live in
// vo_init_math.cuh, shared with mvo_vo_init_candidates_batch_dev (vo_init_batch.cu).
#include <algorithm>
#include <math.h>
#include <numeric>
#include <stdint.h>
#include <vector>
#include "mvo.h"
#include "vo_init_math.cuh"

extern "C" {

int mvo_retain_good_triangulation(const float *pts3d_in_curr, int n, const double *T_w_c_curr, const double *T_w_c_ref,
                                  double min_triang_angle, double max_ratio_to_median, int32_t *keep, double *angles, int *n_keep) {
  if (n < 0 || !T_w_c_curr || !T_w_c_ref || !n_keep || (n > 0 && (!pts3d_in_curr || !keep || !angles))) return MVO_ERR_INVALID_ARG;
  *n_keep = 0;
  if (n == 0) return MVO_OK;                                    // vo.cpp:203-205
  std::vector<double> all((size_t)n);
  for (int i = 0; i < n; ++i) all[(size_t)i] = voi::triangulation_angle(pts3d_in_curr + 3 * i, T_w_c_curr, T_w_c_ref);    // :206-214
  std::vector<double> sorted = all;
  std::nth_element(sorted.begin(), sorted.begin() + n / 2, sorted.end());      // the reference sorts and reads element n / 2 (:216-220): same value
  const double median = sorted[(size_t)(n / 2)];
  int w = 0;
  for (int i = 0; i < n; ++i) {                                  // :236-244
    if (all[(size_t)i] < min_triang_angle || all[(size_t)i] / median > max_ratio_to_median) continue;
    keep[w] = i;
    angles[w] = all[(size_t)i];
    ++w;
  }
  *n_keep = w;
  return MVO_OK;
}

int mvo_normalize_init_depth(float *pts3d, int n, double *t_curr_to_prev, double assumed_mean_depth, double *scale_out) {
  if (n <= 0 || !pts3d || !t_curr_to_prev) return MVO_ERR_INVALID_ARG;
  double mean_depth = 0;                                         // basics::calcMeanDepth (opencv_funcs.cpp:138-145)
  for (int i = 0; i < n; ++i) mean_depth += pts3d[3 * i + 2];
  mean_depth /= n;
  const double scale = assumed_mean_depth / mean_depth;          // vo.cpp:105
  for (int q = 0; q < 3; ++q) t_curr_to_prev[q] *= scale;        // :106
  for (int i = 0; i < 3 * n; ++i) pts3d[i] = (float)(pts3d[i] * scale);      // basics::scalePointPos: float *= double (:107-108)
  if (scale_out) *scale_out = scale;
  return MVO_OK;
}

int mvo_is_vo_good_to_init(const float *kpts_ref_xy, const float *kpts_curr_xy, int n_matches, const double *triangulation_angles,
                           int n_angles, int min_inlier_matches, double min_pixel_dist, double min_median_triangulation_angle,
                           int *good, double *mean_pixel_dist, double *median_angle) {
  if (!good || n_matches < 0 || n_angles < 0 || (n_matches > 0 && (!kpts_ref_xy || !kpts_curr_xy)) || (n_angles > 0 && !triangulation_angles))
    return MVO_ERR_INVALID_ARG;
  const bool criteria_0 = n_matches >= min_inlier_matches;       // vo.cpp:127-133
  double mean_dist = 0;                                          // computeMeanDistBetweenKeypoints (feature_match.cpp:262-279)
  for (int i = 0; i < n_matches; ++i) mean_dist += voi::pixel_dist(kpts_ref_xy[2 * i], kpts_ref_xy[2 * i + 1], kpts_curr_xy[2 * i], kpts_curr_xy[2 * i + 1]);
  mean_dist /= n_matches;                                        // 0/0 = NaN for no matches, like the reference: the comparison below is false
  const bool criteria_1 = mean_dist > min_pixel_dist;            // :136-143
  bool criteria_2 = false;                                       // :146-168
  double med = 0;
  if (n_angles > 0) {
    std::vector<double> a(triangulation_angles, triangulation_angles + n_angles);
    std::sort(a.begin(), a.end());
    med = a[(size_t)(n_angles / 2)];
    criteria_2 = med > min_median_triangulation_angle;
  }
  *good = criteria_0 && criteria_1 && criteria_2;
  if (mean_pixel_dist) *mean_pixel_dist = mean_dist;
  if (median_angle) *median_angle = med;
  return MVO_OK;
}

int mvo_check_large_move(const double *T_w_c_curr, const double *T_w_c_ref, double min_dist_between_two_keyframes, int *large,
                         double *moved_dist, double *rotated_angle) {
  if (!T_w_c_curr || !T_w_c_ref || !large) return MVO_ERR_INVALID_ARG;
  // T_key_to_curr = ref^-1 * curr (vo.cpp:249); rigid inverse of ref
  double Rr[9], tr[3], R[9], t[3];
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) Rr[i * 3 + j] = T_w_c_ref[j * 4 + i]; }
  for (int i = 0; i < 3; ++i) tr[i] = -(Rr[i * 3] * T_w_c_ref[3] + Rr[i * 3 + 1] * T_w_c_ref[7] + Rr[i * 3 + 2] * T_w_c_ref[11]);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = Rr[i * 3] * T_w_c_curr[j] + Rr[i * 3 + 1] * T_w_c_curr[4 + j] + Rr[i * 3 + 2] * T_w_c_curr[8 + j];
    t[i] = Rr[i * 3] * T_w_c_curr[3] + Rr[i * 3 + 1] * T_w_c_curr[7] + Rr[i * 3 + 2] * T_w_c_curr[11] + tr[i];
  }
  const double dist = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);          // calcMatNorm(t) (:256)
  const double c = (R[0] + R[4] + R[8] - 1) / 2;                               // |Rodrigues(R)| = rotation angle (:252,257)
  const double ang = acos(c > 1 ? 1.0 : (c < -1 ? -1.0 : c));
  *large = dist > min_dist_between_two_keyframes;                              // :262 (the rotation is printed only)
  if (moved_dist) *moved_dist = dist;
  if (rotated_angle) *rotated_angle = ang;
  return MVO_OK;
}

}  // extern "C"
