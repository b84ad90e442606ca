// Two-view geometry for sm_90a (SURVEY.md §8f-1, first part) — replaces
//   geometry::estiMotionByEssential  reference src/geometry/epipolar_geometry.cpp:17-57:
//       cv::findEssentialMat(pts1, pts2, focal, pp, RANSAC, prob 0.999, threshold 1.0, mask)  +  E /= E(2,2)
//       + inliers from the mask  +  cv::recoverPose(E, pts1, pts2, R, t, focal, pp, mask)  +  t /= |t|
//   geometry::doTriangulation        :130-175:  cv::triangulatePoints([I|0], [R|t], inlier points on the normalised
//       plane) and the division by the fourth coordinate
// Structure kept from OpenCV: hypotheses from minimal samples -> Sampson-distance consensus -> decomposeEssentialMat ->
// the cheirality vote of recoverPose over its four (R, t) candidates (triangulation of every inlier, depth in (0, 50)
// in both cameras, OpenCV's tie order).  What differs by design, as for PnP: all H hypotheses
// (mvo_params::epi_hypotheses, default 4096 — not the adaptive <= ~1000 of prob 0.999) are generated and scored in one
// batch; the minimal solver is the linear eight-point method projected onto the essential manifold instead of
// Nister's five-point solver; and the best minimal model is locally optimised on its consensus set (k_epi_finish).
//   k_epi_hypotheses  one thread per hypothesis: counter-based sampling, epi::essential_from_8
//   k_epi_score       one warp per hypothesis, points staged once per CTA in shared memory, count(Sampson <= thr^2)
//   k_epi_finish      one CTA: arg-max (ties -> lowest hypothesis), ordered inlier list, recoverPose vote
//   k_triangulate     one thread per point: epi::triangulate_dlt
// mvo_esti_motion_by_essential_batch_dev runs the same kernel bodies over a batch of matched frame pairs (a pair dimension on
// every kernel, one finish cluster per pair, recoverPose's pick on the device: epipolar_kernels.cuh, "batch of frame pairs").
// The numerics live in epipolar_math.cuh and are unit-tested on the host (tests/test_epipolar_math.py).
#include <cooperative_groups.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "epipolar_math.cuh"
#include "eh_scores.cuh"
#include "mvo_internal.h"

namespace {

#define EPI_DYN_SMEM(type, name) extern __shared__ type name[]
#ifdef __CUDACC__
#define EPI_NOINLINE __noinline__
#else
#define EPI_NOINLINE
#endif
#include "epipolar_kernels.cuh"

// device-side unit test of epipolar_math.cuh (test hook: tests compare with the host build of the same header)
__global__ void k_epi_math_test(const double *__restrict__ in, double *__restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  // in: [0..15] xy1 (8x2), [16..31] xy2, [32..40] a 3x3 matrix, [41..112] an 8x9 matrix
  double E[9];
  int reason = -1;
  const bool ok = epi::essential_from_8(in, in + 16, E, &reason);
  out[0] = ok ? 1 : 0; out[1] = reason;
  for (int q = 0; q < 9; ++q) out[2 + q] = E[q];
  double U[9], sv[3], V[9];
  epi::svd3(in + 32, U, sv, V);
  for (int q = 0; q < 9; ++q) { out[11 + q] = U[q]; out[23 + q] = V[q]; }
  for (int q = 0; q < 3; ++q) out[20 + q] = sv[q];
  double M[72], x[9];
  for (int q = 0; q < 72; ++q) M[q] = in[41 + q];
  out[32] = epi::null_vector_8x9(M, x) ? 1 : 0;
  for (int q = 0; q < 9; ++q) out[33 + q] = x[q];
  double A[9], w[3], Q[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) A[i * 3 + j] = in[32 + i * 3 + j] + in[32 + j * 3 + i];      // a symmetric matrix
  epi::sym_eigen_jacobi<3>(A, w, Q);
  for (int q = 0; q < 3; ++q) out[42 + q] = w[q];
  for (int q = 0; q < 9; ++q) out[45 + q] = Q[q];
  // the inside of essential_from_8, step by step
  double M8[72], f[9];
  for (int k = 0; k < 8; ++k) {
    const double x1 = in[2 * k], y1 = in[2 * k + 1], x2 = in[16 + 2 * k], y2 = in[16 + 2 * k + 1];
    double *r = M8 + 9 * k;
    r[0] = x2 * x1; r[1] = x2 * y1; r[2] = x2; r[3] = y2 * x1; r[4] = y2 * y1; r[5] = y2; r[6] = x1; r[7] = y1; r[8] = 1.0;
  }
  out[54] = epi::null_vector_8x9(M8, f) ? 1 : 0;
  epi::svd3(f, U, sv, V);
  for (int q = 0; q < 3; ++q) out[55 + q] = sv[q];
  double A2[9], w2[3], Q2[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A2[i * 3 + j] = f[0 * 3 + i] * f[0 * 3 + j] + f[1 * 3 + i] * f[1 * 3 + j] + f[2 * 3 + i] * f[2 * 3 + j];
  for (int q = 0; q < 3; ++q) out[58 + q] = A2[q * 4];          // diagonal of f^T f
  epi::sym_eigen_jacobi<3>(A2, w2, Q2);
  for (int q = 0; q < 3; ++q) out[61 + q] = w2[q];
}

// `clusters` thread-block clusters of EFIN_C CTAs each (distributed shared memory between them), one after the other along x;
// all block state in dynamic shared memory
template <class K, class... A>
cudaError_t launch_finish_cluster(mvo_ctx *ctx, unsigned clusters, size_t smem, K kernel, A... args) {
  static const int env_c = getenv("MVO_EFIN_CLUSTER") ? atoi(getenv("MVO_EFIN_CLUSTER")) : EFIN_C;     // A/B hook: CTAs per cluster
  const int csz = (env_c >= 1 && env_c <= 8) ? env_c : EFIN_C;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(csz * clusters);
  cfg.blockDim = dim3(EFIN_T);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = csz;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}
}  // namespace

extern "C" int mvo_test_epi_math(mvo_ctx *ctx, const double *in /* 113 */, double *out /* 64 */) {
  if (!ctx || !in || !out) return MVO_ERR_INVALID_ARG;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  MVO_TRY(mvo_reserve(ctx, ctx->d_c, 4096));
  double *d = (double *)ctx->d_c.p;
  MVO_CUDA(ctx, cudaMemcpyAsync(d, in, 113 * 8, cudaMemcpyHostToDevice, ctx->stream));
  k_epi_math_test<<<1, 32, 0, ctx->stream>>>(d, d + 128);
  MVO_CHECK_LAUNCH(ctx);
  MVO_CUDA(ctx, cudaMemcpyAsync(out, d + 128, 64 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MVO_OK;
}

extern "C" {

int mvo_esti_motion_by_essential(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold,
                                 double *E, double *R, double *t, int32_t *inliers, int *n_inliers) {
  return mvo_epi_essential_ex(ctx, pts1, pts2, n, K, threshold, E, R, t, inliers, n_inliers, 1, nullptr, nullptr, nullptr, nullptr, nullptr);
}

}  // extern "C"

// estiMotionByEssential with the options of the keyframe branch (internal, mvo_internal.h):
//   want_pose = 0   the caller only uses the RANSAC inliers (helperFindInlierMatchesByEpipolarCons, motion_estimation.cpp:180-196,
//                   passes dummy R / t): recoverPose's cheirality vote is not launched, R / t are left untouched
//   tri_*           doTriangulation (epipolar_geometry.cpp:130-175) of ALL n correspondences (normalised-plane points tri_np1 /
//                   tri_np2, known motion tri_R / tri_t) in the same submission: the motion between two tracked frames is known
//                   before the RANSAC runs, a point's triangulation does not depend on the inlier list, so the keyframe branch
//                   needs one synchronisation for both stages; tri_out: n x 3 floats, the caller picks the inliers' rows
int mvo_epi_essential_ex(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold,
                         double *E, double *R, double *t, int32_t *inliers, int *n_inliers, int want_pose,
                         const float *tri_np1, const float *tri_np2, const double *tri_R, const double *tri_t, float *tri_out) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!E || !R || !t || !n_inliers || (*n_inliers > 0 && !inliers)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByEssential: null pointer");
  MvoEpiJob job;
  MVO_TRY(mvo_epi_essential_begin(ctx, pts1, pts2, n, K, threshold, want_pose, tri_np1, tri_np2, tri_R, tri_t, tri_out != nullptr, &job));
  return mvo_epi_essential_end(ctx, &job, E, R, t, inliers, n_inliers, tri_out);
}

namespace {

// the call-level checks of both batch calls (mvo.h)
int epi_batch_check(mvo_ctx *ctx, const char *what, int batch, int cap, int n_pairs, const double *K) {
  if (n_pairs < 0 || batch < 1 || cap < 1) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "%s: n_pairs=%d batch=%d cap=%d", what, n_pairs, batch, cap);
  if (!(K[0] > 0 && K[4] > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "K: focal lengths must be positive");
  if ((size_t)cap * 4 * sizeof(double) > 200 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "%s: cap %d above %d correspondences", what, cap, 200 * 1024 / 32);
  if (n_pairs > 65535) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "%s: %d pairs, at most 65535 per call", what, n_pairs);
  const int H = ctx->prm.epi_hypotheses;
  if ((size_t)n_pairs * H > ((size_t)1 << 22)) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "%s: %d pairs x %d hypotheses above 2^22 per call", what, n_pairs, H);
  return MVO_OK;
}

// Scratch of the essential half: gathered points (np1 / np2 optional), pn, hypothesis rows (Es 72 B + valid 4 B + cnt 4 B per
// hypothesis), finish outputs
struct EpiBatchScratch {
  float *p1, *p2, *np1, *np2;
  int32_t *pn, *valid, *cnt, *oi;
  double *Es, *od;
};

// gather, hypotheses, scoring, finish, vote, pick: six launches; pair p's inliers at inl + p * cap, its record in res[p]
int epi_essential_batch_enqueue(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap, const int32_t *d_pairs,
                                int n_pairs, const mvo_dmatch *d_matches, const int32_t *d_n_matches, const double *K, double threshold,
                                const EpiBatchScratch &b, mvo_two_view_result *res, int32_t *inl) {
  EpiCam cam;
  cam.f = (K[0] + K[4]) / 2; cam.cx = K[2]; cam.cy = K[5];
  const int H = ctx->prm.epi_hypotheses;
  const size_t smem = (size_t)cap * 4 * sizeof(double);
  const double thr2 = (threshold / cam.f) * (threshold / cam.f);          // as mvo_epi_essential_begin
  { KTimer kt(ctx, KC_EPI);
  k_epi_gather<<<n_pairs, 256, 0, ctx->stream>>>(d_kpts, d_counts, batch, cap, (const int2 *)d_pairs, d_matches, d_n_matches, K[0], K[4], K[2], K[5],
                                                 b.p1, b.p2, b.np1, b.np2, b.pn); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI);
  k_epi_hypotheses_batch<<<dim3((H + 127) / 128, n_pairs), 128, 0, ctx->stream>>>(b.p1, b.p2, b.pn, cap, cam, ctx->prm.pnp_seed, H, b.Es, b.valid); }
  MVO_CHECK_LAUNCH(ctx);
  if (smem > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_epi_score_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // about as many CTAs in all as the single call uses for its one pair, at least one per pair
  int per_pair = (4 * ctx->sm_count + n_pairs - 1) / n_pairs;
  if (per_pair > (H + 7) / 8) per_pair = (H + 7) / 8;
  { KTimer kt(ctx, KC_EPI_SCORE);
  k_epi_score_batch<<<dim3(per_pair, n_pairs), 256, smem, ctx->stream>>>(b.p1, b.p2, b.pn, cap, cam, thr2, H, b.Es, b.valid, b.cnt); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_FINISH);
    MVO_CUDA(ctx, launch_finish_cluster(ctx, (unsigned)n_pairs, sizeof(EpiFinSmem), k_epi_finish_batch, (const float *)b.p1, (const float *)b.p2,
                                        (const int32_t *)b.pn, cap, cam, thr2, H, (const double *)b.Es, (const int32_t *)b.cnt, b.od, b.oi, inl)); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI);
  k_epi_vote_batch<<<dim3((cap + 63) / 64, n_pairs), 256, 0, ctx->stream>>>(b.p1, b.p2, b.pn, cap, cam, b.od, b.oi, inl); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI);
  k_epi_pick<<<(n_pairs + 127) / 128, 128, 0, ctx->stream>>>(b.pn, n_pairs, b.od, b.oi, res); }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

}  // namespace

// mvo_esti_motion_by_essential_batch_dev (mvo.h): gather, hypotheses, scoring, finish, vote, pick (+ triangulation) for every
// pair at once; the scratch lives in ctx->epib_buf
extern "C" int mvo_esti_motion_by_essential_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                                      const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches,
                                                      const int32_t *d_n_matches, const double *K, double threshold,
                                                      mvo_two_view_result *d_res, int32_t *d_inliers, float *d_pts3d) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!d_kpts || !d_counts || !d_pairs || !d_matches || !d_n_matches || !K || !d_res || !d_inliers)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByEssential batch: null pointer");
  if (!(threshold > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByEssential batch: threshold must be positive");
  MVO_TRY(epi_batch_check(ctx, "estiMotionByEssential batch", batch, cap, n_pairs, K));
  if (n_pairs == 0) return MVO_OK;
  const int H = ctx->prm.epi_hypotheses;
  const bool tri = d_pts3d != nullptr;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t np = (size_t)n_pairs, pts = al(np * cap * 8);
  const size_t o_p1 = 0, o_p2 = o_p1 + pts, o_n1 = o_p2 + pts, o_n2 = o_n1 + (tri ? pts : 0), o_pn = o_n2 + (tri ? pts : 0);
  const size_t o_E = al(o_pn + np * 4), o_valid = al(o_E + np * H * 72), o_cnt = al(o_valid + np * H * 4), o_od = al(o_cnt + np * H * 4);
  const size_t o_oi = al(o_od + np * EPIB_OUT_D * 8), o_end = o_oi + np * EPIB_OUT_I * 4;
  MVO_TRY(mvo_reserve(ctx, ctx->epib_buf, o_end));
  uint8_t *d = (uint8_t *)ctx->epib_buf.p;
  EpiBatchScratch b;
  b.p1 = (float *)(d + o_p1); b.p2 = (float *)(d + o_p2); b.np1 = tri ? (float *)(d + o_n1) : nullptr; b.np2 = tri ? (float *)(d + o_n2) : nullptr;
  b.pn = (int32_t *)(d + o_pn); b.valid = (int32_t *)(d + o_valid); b.cnt = (int32_t *)(d + o_cnt); b.oi = (int32_t *)(d + o_oi);
  b.Es = (double *)(d + o_E); b.od = (double *)(d + o_od);
  MVO_TRY(epi_essential_batch_enqueue(ctx, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, K, threshold, b, d_res, d_inliers));
  if (tri) {
    KTimer kt(ctx, KC_EPI);
    k_triangulate_batch<<<dim3((cap + 127) / 128, n_pairs), 128, 0, ctx->stream>>>(b.np1, b.np2, d_res, cap, d_inliers, d_pts3d);
    MVO_CHECK_LAUNCH(ctx);
  }
  return MVO_OK;
}

// The combine step lives in two_view_batch.cu, a translation unit of its own that is compiled without contraction (Makefile).
// libmvo.so always links it; a library assembled from a subset of the units without it reports MVO_ERR_UNSUPPORTED for the call.
int mvo_relative_poses_combine(mvo_ctx *ctx, const MvoRelPosesCombine &a) __attribute__((weak));

// mvo_estimate_relative_poses_batch_dev (mvo.h): the essential half (six launches, into an internal mvo_two_view_result array),
// the homography half (three launches), the combine step (two_view_batch.cu: decomposition, visibility filter, inlier rows,
// invRt, scores, E/H choice) and, with d_pts3d, one triangulation launch over (pair, solution).  Scratch in ctx->epib_buf: the
// homography half reuses the essential half's hypothesis rows (80 B per hypothesis), which k_epi_finish_batch has consumed by the
// time k_homo_hypotheses_batch runs on the same stream.
extern "C" int mvo_estimate_relative_poses_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                                     const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches,
                                                     const int32_t *d_n_matches, const double *K, int motion_cam2_to_cam1,
                                                     mvo_relative_poses_result *d_res, int32_t *d_inliers, float *d_pts3d) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!d_kpts || !d_counts || !d_pairs || !d_matches || !d_n_matches || !K || !d_res || !d_inliers)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estimate_relative_poses batch: null pointer");
  if (!mvo_relative_poses_combine)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "estimate_relative_poses batch: the library was built without two_view_batch.cu");
  MVO_TRY(epi_batch_check(ctx, "estimate_relative_poses batch", batch, cap, n_pairs, K));
  double Ki[9];
  if (!epi::inv3(K, Ki)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "K: singular (checkEssentialScore inverts it)");
  if (n_pairs == 0) return MVO_OK;
  const int H = ctx->prm.epi_hypotheses;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t np = (size_t)n_pairs, pts = al(np * cap * 8), idx = al(np * cap * 4);
  const size_t o_p1 = 0, o_p2 = o_p1 + pts, o_n1 = o_p2 + pts, o_n2 = o_n1 + pts, o_pn = o_n2 + pts;
  const size_t o_E = al(o_pn + np * 4), o_valid = al(o_E + np * H * 72), o_cnt = al(o_valid + np * H * 4), o_od = al(o_cnt + np * H * 4);
  const size_t o_oi = al(o_od + np * EPIB_OUT_D * 8), o_hd = al(o_oi + np * EPIB_OUT_I * 4), o_hi = al(o_hd + np * EPIB_OUT_D * 8);
  const size_t o_ess = al(o_hi + np * EPIB_OUT_I * 4), o_ie = al(o_ess + np * sizeof(mvo_two_view_result)), o_ih = o_ie + idx;
  const size_t o_rt = o_ih + idx, o_end = o_rt + np * 5 * 12 * 8;
  MVO_TRY(mvo_reserve(ctx, ctx->epib_buf, o_end));
  uint8_t *d = (uint8_t *)ctx->epib_buf.p;
  EpiBatchScratch b;
  b.p1 = (float *)(d + o_p1); b.p2 = (float *)(d + o_p2); b.np1 = (float *)(d + o_n1); b.np2 = (float *)(d + o_n2);
  b.pn = (int32_t *)(d + o_pn); b.valid = (int32_t *)(d + o_valid); b.cnt = (int32_t *)(d + o_cnt); b.oi = (int32_t *)(d + o_oi);
  b.Es = (double *)(d + o_E); b.od = (double *)(d + o_od);
  mvo_two_view_result *ess = (mvo_two_view_result *)(d + o_ess);
  int32_t *inl_e = (int32_t *)(d + o_ie), *inl_h = (int32_t *)(d + o_ih), *hoi = (int32_t *)(d + o_hi);
  double *hod = (double *)(d + o_hd), *rt = (double *)(d + o_rt);
  // ---- essential half (:43-48) ----
  MVO_TRY(epi_essential_batch_enqueue(ctx, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, K, ctx->prm.essential_threshold,
                                      b, ess, inl_e));
  // ---- homography half (:56-67), as mvo_epi_homography_begin on the same points ----
  HomoCam hc;
  hc.f = (K[0] + K[4]) / 2; hc.cx = K[2]; hc.cy = K[5];
  const double hthr2 = (ctx->prm.homography_threshold / hc.f) * (ctx->prm.homography_threshold / hc.f);
  const size_t smem = (size_t)cap * 4 * sizeof(double);
  { KTimer kt(ctx, KC_EPI);
  k_homo_hypotheses_batch<<<dim3((H + 127) / 128, n_pairs), 128, 0, ctx->stream>>>(b.p1, b.p2, b.pn, cap, hc, ctx->prm.pnp_seed, H, b.Es, b.valid, hod, hoi); }
  MVO_CHECK_LAUNCH(ctx);
  if (smem > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_homo_score_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_pair = (4 * ctx->sm_count + n_pairs - 1) / n_pairs;
  if (per_pair > (H + 7) / 8) per_pair = (H + 7) / 8;
  { KTimer kt(ctx, KC_EPI_SCORE);
  k_homo_score_batch<<<dim3(per_pair, n_pairs), 256, smem, ctx->stream>>>(b.p1, b.p2, b.pn, cap, hc, hthr2, H, b.Es, b.valid, b.cnt); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_FINISH);
    MVO_CUDA(ctx, launch_finish_cluster(ctx, (unsigned)n_pairs, sizeof(HomoFinSmem), k_homo_finish_batch, (const float *)b.p1, (const float *)b.p2,
                                        (const int32_t *)b.pn, cap, hc, hthr2, H, (const double *)b.Es, (const int32_t *)b.cnt, hod, hoi, inl_h)); }
  MVO_CHECK_LAUNCH(ctx);
  // ---- combine (:56-154 after the RANSACs) ----
  MvoRelPosesCombine a;
  a.n_matches = d_n_matches; a.ess = ess; a.inl_e = inl_e; a.hom_i = hoi; a.inl_h = inl_h; a.hom_d = hod;
  a.p1 = b.p1; a.p2 = b.p2; a.np1 = b.np1; a.np2 = b.np2;
  a.n_pairs = n_pairs; a.cap = cap; a.hom_d_stride = EPIB_OUT_D; a.hom_i_stride = EPIB_OUT_I; a.motion_cam2_to_cam1 = motion_cam2_to_cam1;
  for (int q = 0; q < 9; ++q) a.K[q] = K[q];
  a.eh_ratio_threshold = ctx->prm.eh_ratio_threshold;
  a.res = d_res; a.inliers = d_inliers; a.rt = rt;
  MVO_TRY(mvo_relative_poses_combine(ctx, a));
  // ---- triangulation of every solution (:105-112), with the (R, t) from before invRt ----
  if (d_pts3d) {
    KTimer kt(ctx, KC_EPI);
    k_triangulate_solutions_batch<<<dim3((cap + 127) / 128, 5, n_pairs), 128, 0, ctx->stream>>>(b.np1, b.np2, d_res, rt, cap, d_inliers, d_pts3d);
    MVO_CHECK_LAUNCH(ctx);
  }
  return MVO_OK;
}

// first half: everything up to the device-to-host copies, enqueued on ctx->stream (the caller may have pointed that at a side
// stream); no synchronisation
int mvo_epi_essential_begin(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold, int want_pose,
                            const float *tri_np1, const float *tri_np2, const double *tri_R, const double *tri_t, bool tri, MvoEpiJob *job) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (tri && (!tri_np1 || !tri_np2 || !tri_R || !tri_t)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByEssential: null triangulation input");
  if (!pts1 || !pts2 || !K || !job) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByEssential: null pointer");
  if (n < 8) return mvo_fail(ctx, MVO_ERR_DEGENERATE, "estiMotionByEssential: %d correspondences (< 8)", n);
  if (!(threshold > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByEssential: threshold must be positive");
  EpiCam cam;
  cam.f = (K[0] + K[4]) / 2; cam.cx = K[2]; cam.cy = K[5];               // epipolar_geometry.cpp:26-27
  if (!(cam.f > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "K: focal length must be positive");
  const size_t smem = (size_t)n * 4 * sizeof(double);
  if (smem > 200 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "estiMotionByEssential: more than %d correspondences", 200 * 1024 / 32);
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int H = ctx->prm.epi_hypotheses;
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t o_p1 = 0, o_p2 = al(o_p1 + (size_t)n * 8), o_inl = al(o_p2 + (size_t)n * 8), o_E = al(o_inl + (size_t)n * 4);
  const size_t o_valid = al(o_E + (size_t)H * 72), o_cnt = al(o_valid + (size_t)H * 4), o_out = al(o_cnt + (size_t)H * 4);
  // optional triangulation block: np1, np2 (n x 2 floats each), R | t (12 doubles), out (n x 3 floats)
  const size_t o_t1 = al(o_out + 512), o_t2 = al(o_t1 + (size_t)n * 8), o_trt = al(o_t2 + (size_t)n * 8), o_tout = al(o_trt + 96);
  const size_t o_end = tri ? o_tout + (size_t)n * 12 : o_out + 512;
  // pinned staging: [p1 p2 | np1 np2 Rt] in, [out block 512 B + inliers | triangulated points] out
  const size_t h_in = al((size_t)n * 16) + (tri ? al((size_t)n * 16) + 256 : 0), h_res = 512 + al((size_t)n * 4) + 256;
  MVO_TRY(mvo_reserve(ctx, ctx->d_a, o_end));
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_a, h_in + h_res + (tri ? (size_t)n * 12 : 0) + 1024));
  uint8_t *d = (uint8_t *)ctx->d_a.p, *h = (uint8_t *)ctx->h_a.p;
  memcpy(h, pts1, (size_t)n * 8);
  memcpy(h + (size_t)n * 8, pts2, (size_t)n * 8);
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_p1, h, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_p2, h + (size_t)n * 8, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  // the triangulation does not depend on the RANSAC: it runs on the context's side stream next to it (on the same stream when
  // per-kernel event timing is on, or when this job itself was pointed at the side stream)
  cudaStream_t tri_stream = ctx->stream;
  float *h_tri = (float *)(h + h_in + h_res);
  if (tri) {
    cudaStream_t side = ctx->timing_mask ? nullptr : mvo_side_stream(ctx);
    if (side && side != ctx->stream) tri_stream = side;
    uint8_t *ht = h + al((size_t)n * 16);
    memcpy(ht, tri_np1, (size_t)n * 8);
    memcpy(ht + (size_t)n * 8, tri_np2, (size_t)n * 8);
    memcpy(ht + al((size_t)n * 16), tri_R, 72);
    memcpy(ht + al((size_t)n * 16) + 72, tri_t, 24);
    MVO_CUDA(ctx, cudaMemcpyAsync(d + o_t1, ht, (size_t)n * 8, cudaMemcpyHostToDevice, tri_stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(d + o_t2, ht + (size_t)n * 8, (size_t)n * 8, cudaMemcpyHostToDevice, tri_stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(d + o_trt, ht + al((size_t)n * 16), 96, cudaMemcpyHostToDevice, tri_stream));
    {
      cudaStream_t keep = ctx->stream;
      ctx->stream = tri_stream;              // KTimer records on ctx->stream
      { KTimer kt(ctx, KC_EPI);
      k_triangulate<<<(n + 127) / 128, 128, 0, tri_stream>>>((const float *)(d + o_t1), (const float *)(d + o_t2), nullptr, n, (const double *)(d + o_trt),
                                                              (float *)(d + o_tout)); }
      ctx->stream = keep;
    }
    MVO_CHECK_LAUNCH(ctx);
    MVO_CUDA(ctx, cudaMemcpyAsync(h_tri, d + o_tout, (size_t)n * 12, cudaMemcpyDeviceToHost, tri_stream));
  }
  const float *d1 = (const float *)(d + o_p1), *d2 = (const float *)(d + o_p2);
  double *dE = (double *)(d + o_E), *dout = (double *)(d + o_out);
  int32_t *dvalid = (int32_t *)(d + o_valid), *dcnt = (int32_t *)(d + o_cnt), *dinl = (int32_t *)(d + o_inl), *dout_i = (int32_t *)(d + o_out + 256);
  const double thr2 = (threshold / cam.f) * (threshold / cam.f);          // findEssentialMat: threshold /= focal
  { KTimer kt(ctx, KC_EPI);
  k_epi_hypotheses<<<(H + 127) / 128, 128, 0, ctx->stream>>>(d1, d2, n, cam, ctx->prm.pnp_seed, H, dE, dvalid); }
  MVO_CHECK_LAUNCH(ctx);
  if (smem > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_epi_score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (H + 7) / 8;
  if (grid > 4 * ctx->sm_count) grid = 4 * ctx->sm_count;
  { KTimer kt(ctx, KC_EPI_SCORE);
  k_epi_score<<<grid, 256, smem, ctx->stream>>>(d1, d2, n, cam, thr2, H, dE, dvalid, dcnt); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_FINISH);
    MVO_CUDA(ctx, launch_finish_cluster(ctx, 1, sizeof(EpiFinSmem), k_epi_finish, d1, d2, n, cam, thr2, H, (const double *)dE, (const int32_t *)dcnt, dout, dout_i, dinl)); }
  MVO_CHECK_LAUNCH(ctx);
  if (want_pose) {
    KTimer kt(ctx, KC_EPI);
    k_epi_vote<<<(n + 63) / 64, 256, 0, ctx->stream>>>(d1, d2, cam, dout, dout_i, dinl);
    MVO_CHECK_LAUNCH(ctx);
  }
  double *h_out = (double *)(h + h_in);
  int32_t *h_inl = (int32_t *)((uint8_t *)h_out + 512);
  MVO_CUDA(ctx, cudaMemcpyAsync(h_out, dout, 512, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(h_inl, dinl, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  job->tri_stream = tri_stream;
  job->stream = ctx->stream; job->n = n; job->H = H; job->want_pose = want_pose != 0; job->tri = tri; job->thr2 = thr2; job->f = cam.f;
  job->h_out = h_out; job->h_inl = h_inl; job->h_tri = h_tri; job->d_valid = dvalid; job->d_cnt = dcnt; job->d_model = dE;
  return MVO_OK;
}

// second half: wait for the job's stream, recoverPose's pick, outputs
int mvo_epi_essential_end(mvo_ctx *ctx, MvoEpiJob *job, double *E, double *R, double *t, int32_t *inliers, int *n_inliers, float *tri_out) {
  MVO_CUDA(ctx, cudaStreamSynchronize(job->stream));
  if (job->tri && job->tri_stream != job->stream) MVO_CUDA(ctx, cudaStreamSynchronize(job->tri_stream));
  const int n = job->n, H = job->H;
  double *h_out = job->h_out;
  int32_t *h_i = (int32_t *)((uint8_t *)h_out + 256), *h_inl = job->h_inl;
  if (job->tri && tri_out) memcpy(tri_out, job->h_tri, (size_t)n * 12);
  const int ni = h_i[0];
  if (getenv("MVO_EPI_DEBUG")) {
    std::vector<int32_t> hv(H), hc(H);
    std::vector<double> hE(9);
    cudaMemcpy(hv.data(), job->d_valid, (size_t)H * 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(hc.data(), job->d_cnt, (size_t)H * 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(hE.data(), job->d_model, 72, cudaMemcpyDeviceToHost);
    int nv = 0, mx = -2, why[4] = {0, 0, 0, 0};
    for (int h2 = 0; h2 < H; ++h2) { nv += hv[h2] > 0; if (hv[h2] <= 0 && hv[h2] > -4) why[-hv[h2]]++; if (hc[h2] > mx) mx = hc[h2]; }
    fprintf(stderr, "epi debug: rejected samples by reason 0..3: %d %d %d %d\n", why[0], why[1], why[2], why[3]);
    fprintf(stderr, "epi debug: H=%d valid=%d max count=%d | finish: inliers %d best %d votes %d minimal %d after LO %d | thr2 %.3e f %.1f | E[0]= %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f\n",
            H, nv, mx, h_i[0], h_i[1], h_i[2], h_i[3], h_i[4], job->thr2, job->f, hE[0], hE[1], hE[2], hE[3], hE[4], hE[5], hE[6], hE[7], hE[8]);
  }
  if (ni < 8) {
    *n_inliers = 0;
    return mvo_fail(ctx, MVO_ERR_DEGENERATE, "estiMotionByEssential: no model reached 8 inliers (best minimal model %d, after local optimisation %d, final %d)",
                    h_i[3], h_i[4], ni);
  }
  if (ni > *n_inliers) return mvo_fail(ctx, MVO_ERR_CAPACITY, "inlier capacity %d < %d", *n_inliers, ni);
  if (!job->want_pose) {
    memcpy(E, h_out, 72);
    memcpy(inliers, h_inl, (size_t)ni * 4);
    *n_inliers = ni;
    return MVO_OK;
  }
  // recoverPose's choice among (R1,t) (R2,t) (R1,-t) (R2,-t), OpenCV's order: the first candidate whose vote count is a maximum
  const int32_t *g = h_i + 8;
  int pick = 3;
  if (g[0] >= g[1] && g[0] >= g[2] && g[0] >= g[3]) pick = 0;
  else if (g[1] >= g[0] && g[1] >= g[2] && g[1] >= g[3]) pick = 1;
  else if (g[2] >= g[0] && g[2] >= g[1] && g[2] >= g[3]) pick = 2;
  h_i[2] = g[pick];
  const double *tt = h_out + 27, sg = pick < 2 ? 1.0 : -1.0;
  const double nt = sqrt(tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2]);                 // t /= |t| (epipolar_geometry.cpp:54-55)
  memcpy(E, h_out, 72);
  memcpy(R, h_out + ((pick & 1) ? 18 : 9), 72);
  for (int q = 0; q < 3; ++q) t[q] = sg * tt[q] / nt;
  memcpy(inliers, h_inl, (size_t)ni * 4);
  *n_inliers = ni;
  return MVO_OK;
}

extern "C" {

int mvo_esti_motion_by_homography(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold,
                                  double *Hout, double *Rs, double *ts, double *normals, int *n_solutions, int32_t *inliers,
                                  int *n_inliers) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!Hout || !Rs || !ts || !normals || !n_solutions || !n_inliers || (*n_inliers > 0 && !inliers))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByHomography: null pointer");
  *n_solutions = 0;
  MvoEpiJob job;
  MVO_TRY(mvo_epi_homography_begin(ctx, pts1, pts2, n, K, threshold, &job));
  return mvo_epi_homography_end(ctx, &job, K, Hout, Rs, ts, normals, n_solutions, inliers, n_inliers);
}

}  // extern "C"

// first half (own device / pinned scratch, so that it can run next to an essential-matrix job on another stream)
int mvo_epi_homography_begin(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold, MvoEpiJob *job) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!pts1 || !pts2 || !K || !job) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByHomography: null pointer");
  if (n < 4) return mvo_fail(ctx, MVO_ERR_DEGENERATE, "estiMotionByHomography: %d correspondences (< 4)", n);
  if (!(threshold > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByHomography: threshold must be positive");
  HomoCam cam;
  cam.f = (K[0] + K[4]) / 2; cam.cx = K[2]; cam.cy = K[5];
  if (!(K[0] > 0 && K[4] > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "K: focal lengths must be positive");
  const size_t smem = (size_t)n * 4 * sizeof(double);
  if (smem > 200 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "estiMotionByHomography: more than %d correspondences", 200 * 1024 / 32);
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int H = ctx->prm.epi_hypotheses;
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t o_p1 = 0, o_p2 = al(o_p1 + (size_t)n * 8), o_inl = al(o_p2 + (size_t)n * 8), o_H = al(o_inl + (size_t)n * 4);
  const size_t o_valid = al(o_H + (size_t)H * 72), o_cnt = al(o_valid + (size_t)H * 4), o_out = al(o_cnt + (size_t)H * 4), o_end = o_out + 512;
  MVO_TRY(mvo_reserve(ctx, ctx->d_e, o_end));
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_c, al((size_t)n * 16) + (size_t)n * 4 + 1024));
  uint8_t *d = (uint8_t *)ctx->d_e.p, *h = (uint8_t *)ctx->h_c.p;
  memcpy(h, pts1, (size_t)n * 8);
  memcpy(h + (size_t)n * 8, pts2, (size_t)n * 8);
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_p1, h, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_p2, h + (size_t)n * 8, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  const float *d1 = (const float *)(d + o_p1), *d2 = (const float *)(d + o_p2);
  double *dH = (double *)(d + o_H), *dout = (double *)(d + o_out);
  int32_t *dvalid = (int32_t *)(d + o_valid), *dcnt = (int32_t *)(d + o_cnt), *dinl = (int32_t *)(d + o_inl), *dout_i = (int32_t *)(d + o_out + 256);
  const double thr2 = (threshold / cam.f) * (threshold / cam.f);          // pixels -> scaled coordinates
  MVO_CUDA(ctx, cudaMemsetAsync(dout, 0, 512, ctx->stream));
  { KTimer kt(ctx, KC_EPI);
  k_homo_hypotheses<<<(H + 127) / 128, 128, 0, ctx->stream>>>(d1, d2, n, cam, ctx->prm.pnp_seed, H, dH, dvalid); }
  MVO_CHECK_LAUNCH(ctx);
  if (smem > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_homo_score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (H + 7) / 8;
  if (grid > 4 * ctx->sm_count) grid = 4 * ctx->sm_count;
  { KTimer kt(ctx, KC_EPI_SCORE);
  k_homo_score<<<grid, 256, smem, ctx->stream>>>(d1, d2, n, cam, thr2, H, dH, dvalid, dcnt); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_FINISH);
    MVO_CUDA(ctx, launch_finish_cluster(ctx, 1, sizeof(HomoFinSmem), k_homo_finish, d1, d2, n, cam, thr2, H, (const double *)dH, (const int32_t *)dcnt, dout, dout_i, dinl)); }
  MVO_CHECK_LAUNCH(ctx);
  double *h_out = (double *)(h + al((size_t)n * 16));
  int32_t *h_inl = (int32_t *)((uint8_t *)h_out + 512);
  MVO_CUDA(ctx, cudaMemcpyAsync(h_out, dout, 512, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(h_inl, dinl, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  memset(job, 0, sizeof *job);
  job->stream = ctx->stream; job->n = n; job->H = H; job->thr2 = thr2; job->f = cam.f; job->h_out = h_out; job->h_inl = h_inl;
  return MVO_OK;
}

int mvo_epi_homography_end(mvo_ctx *ctx, MvoEpiJob *job, const double *K, double *Hout, double *Rs, double *ts, double *normals, int *n_solutions,
                           int32_t *inliers, int *n_inliers) {
  MVO_CUDA(ctx, cudaStreamSynchronize(job->stream));
  double *h_out = job->h_out;
  int32_t *h_i = (int32_t *)((uint8_t *)h_out + 256), *h_inl = job->h_inl;
  *n_solutions = 0;
  const int ni = h_i[0];
  if (ni < 4) {
    *n_inliers = 0;
    return mvo_fail(ctx, MVO_ERR_DEGENERATE, "estiMotionByHomography: no model reached 4 inliers (best minimal model %d, after local optimisation %d)",
                    h_i[3], h_i[4]);
  }
  if (ni > *n_inliers) return mvo_fail(ctx, MVO_ERR_CAPACITY, "inlier capacity %d < %d", *n_inliers, ni);
  memcpy(Hout, h_out, 72);
  memcpy(inliers, h_inl, (size_t)ni * 4);
  *n_inliers = ni;
  // cv::decomposeHomographyMat(H, K) (:119-120) on the host: Hn = K^-1 H K, then t /= |t| (:122-126)
  const double fx = K[0], fy = K[4], cx = K[2], cy = K[5];
  const double Km[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1}, Ki[9] = {1 / fx, 0, -cx / fx, 0, 1 / fy, -cy / fy, 0, 0, 1};
  double T[9], Hn[9];
  epi::mat3_mul(Hout, Km, T);
  epi::mat3_mul(Ki, T, Hn);
  const int ns = epi::decompose_homography(Hn, Rs, ts, normals);
  for (int s = 0; s < ns; ++s) {
    const double nt = sqrt(ts[3 * s] * ts[3 * s] + ts[3 * s + 1] * ts[3 * s + 1] + ts[3 * s + 2] * ts[3 * s + 2]);
    if (nt > 0) for (int q = 0; q < 3; ++q) ts[3 * s + q] /= nt;      // a pure rotation keeps t = 0 (the reference divides by zero here)
  }
  *n_solutions = ns;
  return MVO_OK;
}

extern "C" {

int mvo_remove_wrong_rt_of_homography(mvo_ctx *ctx, const float *pts_np1, const float *pts_np2, int n, const int32_t *inliers, int n_inliers,
                                      double *Rs, double *ts, double *normals, int *n_solutions) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!n_solutions || *n_solutions < 0 || *n_solutions > 4 || !Rs || !ts || !normals || (n_inliers > 0 && (!inliers || !pts_np1 || !pts_np2)) || n_inliers < 0)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "removeWrongRtOfHomography: bad arguments");
  for (int j = 0; j < n_inliers; ++j)
    if (inliers[j] < 0 || inliers[j] >= n) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "removeWrongRtOfHomography: inlier index %d outside [0,%d)", inliers[j], n);
  int keep[4] = {0, 0, 0, 0};
  static_assert(sizeof(int) == sizeof(int32_t), "int32 indices");
  epi::filter_homography_solutions(Rs, normals, *n_solutions, pts_np1, pts_np2, (const int *)inliers, n_inliers, keep);
  int w = 0;
  for (int s = 0; s < *n_solutions; ++s)
    if (keep[s]) {
      if (w != s) { memmove(Rs + 9 * w, Rs + 9 * s, 72); memmove(ts + 3 * w, ts + 3 * s, 24); memmove(normals + 3 * w, normals + 3 * s, 24); }
      ++w;
    }
  *n_solutions = w;
  return MVO_OK;
}

}  // extern "C"

// doTriangulation of several (R, t, inlier list) candidates over the same matched points (the initialisation triangulates the
// essential-matrix solution and every surviving homography solution, motion_estimation.cpp:105-112): one upload of the points, one
// launch per candidate, one download, ONE synchronisation
int mvo_do_triangulation_multi(mvo_ctx *ctx, const float *pts_np1, const float *pts_np2, int n, int nsol, const double *const *R,
                               const double *const *t, const int32_t *const *inliers, const int *n_inliers, float *const *pts3d) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (n < 0 || nsol < 0 || nsol > 8 || (nsol > 0 && (!R || !t || !inliers || !n_inliers || !pts3d)) || (n > 0 && (!pts_np1 || !pts_np2)))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "doTriangulation: bad arguments");
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  size_t o = al(al((size_t)n * 8) + (size_t)n * 8), o_in_end = 0, total_out = 0;
  size_t o_inl[8], o_rt[8], o_out[8];
  for (int s = 0; s < nsol; ++s) {
    if (n_inliers[s] < 0 || !R[s] || !t[s] || (n_inliers[s] > 0 && (!inliers[s] || !pts3d[s]))) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "doTriangulation: null pointer");
    for (int j = 0; j < n_inliers[s]; ++j)
      if (inliers[s][j] < 0 || inliers[s][j] >= n) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "doTriangulation: inlier index %d outside [0,%d)", inliers[s][j], n);
    o_inl[s] = o; o = al(o + (size_t)n_inliers[s] * 4);
    o_rt[s] = o;  o = al(o + 96);
  }
  o_in_end = o;
  for (int s = 0; s < nsol; ++s) { o_out[s] = o; o = al(o + (size_t)n_inliers[s] * 12); total_out += (size_t)n_inliers[s]; }
  if (total_out == 0) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  MVO_TRY(mvo_reserve(ctx, ctx->d_b, o + 256));
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_a, o + 256));
  uint8_t *d = (uint8_t *)ctx->d_b.p, *h = (uint8_t *)ctx->h_a.p;
  memcpy(h, pts_np1, (size_t)n * 8);
  memcpy(h + al((size_t)n * 8), pts_np2, (size_t)n * 8);
  for (int s = 0; s < nsol; ++s) {
    memcpy(h + o_inl[s], inliers[s], (size_t)n_inliers[s] * 4);
    memcpy(h + o_rt[s], R[s], 72);
    memcpy(h + o_rt[s] + 72, t[s], 24);
  }
  MVO_CUDA(ctx, cudaMemcpyAsync(d, h, o_in_end, cudaMemcpyHostToDevice, ctx->stream));
  for (int s = 0; s < nsol; ++s) {
    if (n_inliers[s] == 0) continue;
    { KTimer kt(ctx, KC_EPI);
    k_triangulate<<<(n_inliers[s] + 127) / 128, 128, 0, ctx->stream>>>((const float *)d, (const float *)(d + al((size_t)n * 8)), (const int32_t *)(d + o_inl[s]),
                                                                        n_inliers[s], (const double *)(d + o_rt[s]), (float *)(d + o_out[s])); }
    MVO_CHECK_LAUNCH(ctx);
  }
  MVO_CUDA(ctx, cudaMemcpyAsync(h + o_in_end, d + o_in_end, o - o_in_end, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < nsol; ++s)
    if (n_inliers[s] > 0) memcpy(pts3d[s], h + o_out[s], (size_t)n_inliers[s] * 12);
  return MVO_OK;
}

extern "C" {

int mvo_do_triangulation(mvo_ctx *ctx, const float *pts_np1, const float *pts_np2, int n, const double *R, const double *t,
                         const int32_t *inliers, int n_inliers, float *pts3d) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (n < 0 || n_inliers < 0 || !R || !t || (n > 0 && (!pts_np1 || !pts_np2)) || (n_inliers > 0 && (!inliers || !pts3d)))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "doTriangulation: null pointer");
  for (int j = 0; j < n_inliers; ++j)
    if (inliers[j] < 0 || inliers[j] >= n) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "doTriangulation: inlier index %d outside [0,%d)", inliers[j], n);
  if (n_inliers == 0) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t o_p1 = 0, o_p2 = al((size_t)n * 8), o_inl = al(o_p2 + (size_t)n * 8), o_rt = al(o_inl + (size_t)n_inliers * 4);
  const size_t o_out = al(o_rt + 96), o_end = o_out + (size_t)n_inliers * 12;
  MVO_TRY(mvo_reserve(ctx, ctx->d_b, o_end + 256));
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_a, o_end + 256));
  uint8_t *d = (uint8_t *)ctx->d_b.p, *h = (uint8_t *)ctx->h_a.p;
  memcpy(h + o_p1, pts_np1, (size_t)n * 8);
  memcpy(h + o_p2, pts_np2, (size_t)n * 8);
  memcpy(h + o_inl, inliers, (size_t)n_inliers * 4);
  memcpy(h + o_rt, R, 72);
  memcpy(h + o_rt + 72, t, 24);
  MVO_CUDA(ctx, cudaMemcpyAsync(d, h, o_out, cudaMemcpyHostToDevice, ctx->stream));
  { KTimer kt(ctx, KC_EPI);
  k_triangulate<<<(n_inliers + 127) / 128, 128, 0, ctx->stream>>>((const float *)(d + o_p1), (const float *)(d + o_p2), (const int32_t *)(d + o_inl),
                                                                  n_inliers, (const double *)(d + o_rt), (float *)(d + o_out)); }
  MVO_CHECK_LAUNCH(ctx);
  MVO_CUDA(ctx, cudaMemcpyAsync(h + o_out, d + o_out, (size_t)n_inliers * 12, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(pts3d, h + o_out, (size_t)n_inliers * 12);
  return MVO_OK;
}

}  // extern "C"
