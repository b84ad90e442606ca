// Host-side pieces of the two-view initialisation that are plain loops in the reference (SURVEY.md §8f-1):
//   checkEssentialScore   reference src/geometry/motion_estimation.cpp:501-581
//   checkHomographyScore  reference src/geometry/motion_estimation.cpp:583-664
//   the E / H chooser     reference src/geometry/motion_estimation.cpp:134-154
// ORB-SLAM's symmetric chi-square scores over an inlier list (pruned in place) and the rule that picks the essential
// solution or one of the homography solutions.  O(n) double arithmetic on a few hundred points: no GPU work.
#include <math.h>
#include <stdint.h>
#include <vector>
#include "eh_scores.cuh"
#include "mvo.h"

extern "C" {

int mvo_check_essential_score(const double *E21, const double *K, const float *pts_img1, const float *pts_img2, int n,
                              int32_t *inliers, int *n_inliers, double sigma, double *score_out) {
  if (!E21 || !K || !n_inliers || *n_inliers < 0 || !score_out || (*n_inliers > 0 && (!inliers || !pts_img1 || !pts_img2)) || !(sigma > 0))
    return MVO_ERR_INVALID_ARG;
  double Ki[9], F[9];
  if (!epi::inv3(K, Ki)) return MVO_ERR_INVALID_ARG;
  epi::essential_score_F(E21, Ki, F);                // F21 = K^-T E21 K^-1 (:507-509)
  const double th = epi::EH_ESSENTIAL_TH, thScore = epi::EH_ESSENTIAL_TH_SCORE, invSigmaSquare = 1.0 / (sigma * sigma);     // :524-527
  double score = 0;
  int w = 0;
  for (int k = 0; k < *n_inliers; ++k) {
    const int i = inliers[k];
    if (i < 0 || i >= n) return MVO_ERR_INVALID_ARG;
    bool good = true;
    double chi1, chi2;                               // x2 against l2 = F21 x1, x1 against l1 = x2^T F21 (:543-573)
    epi::essential_score_chi(F, pts_img1[2 * i], pts_img1[2 * i + 1], pts_img2[2 * i], pts_img2[2 * i + 1], invSigmaSquare, &chi1, &chi2);
    if (chi1 > th) good = false;
    else score += thScore - chi1;
    if (chi2 > th) good = false;
    else score += thScore - chi2;
    if (good) inliers[w++] = i;                      // :575-576 (w <= k: in place)
  }
  *n_inliers = w;
  *score_out = score;
  return MVO_OK;
}

int mvo_check_homography_score(const double *H21, const float *pts_img1, const float *pts_img2, int n, int32_t *inliers,
                               int *n_inliers, double sigma, double *score_out) {
  if (!H21 || !n_inliers || *n_inliers < 0 || !score_out || (*n_inliers > 0 && (!inliers || !pts_img1 || !pts_img2)) || !(sigma > 0))
    return MVO_ERR_INVALID_ARG;
  double H12[9];
  if (!epi::inv3(H21, H12)) return MVO_ERR_INVALID_ARG;
  const double th = epi::EH_HOMOGRAPHY_TH, invSigmaSquare = 1.0 / (sigma * sigma);       // :613-614
  double score = 0;          // the reference leaves `score` uninitialised (:586); zero is what the sum is meant to start from
  int w = 0;
  for (int k = 0; k < *n_inliers; ++k) {
    const int i = inliers[k];
    if (i < 0 || i >= n) return MVO_ERR_INVALID_ARG;
    bool good = true;
    double chi1, chi2;                               // x2 in image 1 through H12, x1 in image 2 through H21 (:628-656)
    epi::homography_score_chi(H21, H12, pts_img1[2 * i], pts_img1[2 * i + 1], pts_img2[2 * i], pts_img2[2 * i + 1], invSigmaSquare, &chi1, &chi2);
    if (chi1 > th) good = false;
    else score += th - chi1;
    if (chi2 > th) good = false;
    else score += th - chi2;
    if (good) inliers[w++] = i;
  }
  *n_inliers = w;
  *score_out = score;
  return MVO_OK;
}

int mvo_choose_e_or_h(double score_e, double score_h, const double *h_normals, int num_h, int *best_sol, double *ratio_out) {
  return mvo_choose_e_or_h_thr(score_e, score_h, h_normals, num_h, 0.5, best_sol, ratio_out);      // :140
}

int mvo_choose_e_or_h_thr(double score_e, double score_h, const double *h_normals, int num_h, double threshold, int *best_sol,
                          double *ratio_out) {
  if (!best_sol || num_h < 0 || (num_h > 0 && !h_normals) || !(threshold > 0 && threshold < 1)) return MVO_ERR_INVALID_ARG;
  int best = 0;
  const double ratio = epi::eh_choose(score_e, score_h, h_normals, num_h, threshold, &best);
  *best_sol = best;
  if (ratio_out) *ratio_out = ratio;
  return MVO_OK;
}

}  // extern "C"
