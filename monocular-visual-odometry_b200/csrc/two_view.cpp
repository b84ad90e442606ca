// helperEstimatePossibleRelativePosesByEpipolarGeometry (reference src/geometry/motion_estimation.cpp:10-158) over flat
// arrays of MATCHED points: the essential-matrix motion, the homography motions that survive the visibility filter, a
// triangulation of every solution's inliers, ORB-SLAM's E / H scores and the choice between them.  Host orchestration in
// C++ like the reference; every numeric stage is one of the C-ABI entry points of this library.
#include <math.h>
#include <string.h>
#include <vector>
#include "mvo_internal.h"

extern "C" int mvo_estimate_relative_poses(mvo_ctx *ctx, const float *pts_img1, const float *pts_img2, int n, const double *K,
                                           int calc_homo, int motion_cam2_to_cam1, mvo_two_view_solutions *sol, int32_t *inliers,
                                           float *pts3d) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!pts_img1 || !pts_img2 || !K || !sol || !inliers || !pts3d || n < 8)
    return mvo_fail(ctx, n < 8 && n >= 0 ? MVO_ERR_DEGENERATE : MVO_ERR_INVALID_ARG, "estimate_relative_poses: bad arguments (n = %d)", n);
  memset(sol, 0, sizeof *sol);
  // matched points on the normalised image planes: pixel2CamNormPlane (:35-41), double arithmetic narrowed to Point2f
  std::vector<float> np1((size_t)n * 2), np2((size_t)n * 2);
  for (int i = 0; i < n; ++i) {
    np1[2 * i] = (float)(((double)pts_img1[2 * i] - K[2]) / K[0]); np1[2 * i + 1] = (float)(((double)pts_img1[2 * i + 1] - K[5]) / K[4]);
    np2[2 * i] = (float)(((double)pts_img2[2 * i] - K[2]) / K[0]); np2[2 * i + 1] = (float)(((double)pts_img2[2 * i + 1] - K[5]) / K[4]);
  }
  // ---- essential (:43-48); threshold = config findEssentialMat_threshold (mvo_params::essential_threshold) ----
  std::vector<int32_t> inl_e((size_t)n), inl_h((size_t)n);
  int n_e = n, n_h = 0;
  // The two RANSACs are independent: the homography job is enqueued on the context's side stream while the essential-matrix job
  // runs on the main one (separate scratch buffers); with per-kernel event timing enabled they run one after the other.
  double Rh[36], th[12], nh[12];
  int num_h = 0;
  {
    MvoEpiJob je, jh;
    bool h_running = false;
    MVO_TRY(mvo_epi_essential_begin(ctx, pts_img1, pts_img2, n, K, ctx->prm.essential_threshold, 1, nullptr, nullptr, nullptr, nullptr, false, &je));
    int rc_h = MVO_OK;
    if (calc_homo) {
      cudaStream_t main_stream = ctx->stream, side = ctx->timing_mask ? nullptr : mvo_side_stream(ctx);
      if (side) ctx->stream = side;
      rc_h = mvo_epi_homography_begin(ctx, pts_img1, pts_img2, n, K, ctx->prm.homography_threshold, &jh);
      ctx->stream = main_stream;
      h_running = rc_h == MVO_OK;
    }
    const int rc_e = mvo_epi_essential_end(ctx, &je, sol->E, sol->R[0], sol->t[0], inl_e.data(), &n_e, nullptr);
    // ---- homography + removeWrongRtOfHomography (:56-67) ----
    if (h_running) {
      n_h = n;
      rc_h = mvo_epi_homography_end(ctx, &jh, K, sol->H, Rh, th, nh, &num_h, inl_h.data(), &n_h);
    }
    if (rc_e != MVO_OK) return rc_e;
    if (calc_homo) {
      if (rc_h == MVO_ERR_DEGENERATE) { num_h = 0; n_h = 0; }
      else if (rc_h != MVO_OK) return rc_h;
      if (num_h > 0) MVO_TRY(mvo_remove_wrong_rt_of_homography(ctx, np1.data(), np2.data(), n, inl_h.data(), n_h, Rh, th, nh, &num_h));
    }
  }
  // ---- combine (:75-89): solution 0 = essential, then the homography survivors, each with ITS inlier list ----
  sol->num_solutions = 1 + num_h;
  sol->n_inliers[0] = n_e;
  memcpy(inliers, inl_e.data(), (size_t)n_e * 4);
  for (int s = 0; s < num_h; ++s) {
    memcpy(sol->R[1 + s], Rh + 9 * s, 72);
    memcpy(sol->t[1 + s], th + 3 * s, 24);
    memcpy(sol->normal[1 + s], nh + 3 * s, 24);
    sol->n_inliers[1 + s] = n_h;
    memcpy(inliers + (size_t)(1 + s) * n, inl_h.data(), (size_t)n_h * 4);
  }
  // ---- triangulation of every solution (:105-112) ----
  {
    const double *Rs[8], *ts[8];
    const int32_t *is[8];
    float *ps[8];
    int ns[8];
    for (int s = 0; s < sol->num_solutions; ++s) { Rs[s] = sol->R[s]; ts[s] = sol->t[s]; is[s] = inliers + (size_t)s * n; ns[s] = sol->n_inliers[s]; ps[s] = pts3d + (size_t)s * n * 3; }
    MVO_TRY(mvo_do_triangulation_multi(ctx, np1.data(), np2.data(), n, sol->num_solutions, Rs, ts, is, ns, ps));
  }
  // ---- change of frame, after everything else (:114-118): basics::invRt ----
  if (!motion_cam2_to_cam1)
    for (int s = 0; s < sol->num_solutions; ++s) inv_rt(sol->R[s], sol->t[s]);
  // ---- choose a solution (:134-154); the score functions prune copies of the inlier lists, as in the reference ----
  int ne2 = n_e, nh2 = n_h;
  MVO_TRY(mvo_check_essential_score(sol->E, K, pts_img1, pts_img2, n, inl_e.data(), &ne2, 1.0, &sol->score_e));
  sol->score_h = 0;
  if (calc_homo && n_h > 0) {
    const int rc = mvo_check_homography_score(sol->H, pts_img1, pts_img2, n, inl_h.data(), &nh2, 1.0, &sol->score_h);
    if (rc != MVO_OK) sol->score_h = 0;          // a singular H cannot be inverted for the symmetric transfer error
  }
  int best = 0;
  MVO_TRY(mvo_choose_e_or_h_thr(sol->score_e, sol->score_h, &sol->normal[1][0], num_h, ctx->prm.eh_ratio_threshold, &best, &sol->ratio));
  sol->best = best;
  return MVO_OK;
}
