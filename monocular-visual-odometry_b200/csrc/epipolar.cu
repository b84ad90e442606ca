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
// Nister's five-point solver; and the best minimal model is locally optimised on its consensus set (k_epi_finish_batch).
//   k_epi_hypotheses_batch  one thread per hypothesis: counter-based sampling, epi::essential_from_8
//   k_epi_score_batch       one warp per hypothesis, points staged once per CTA in shared memory, count(Sampson <= thr^2)
//   k_epi_finish_batch      one 8-CTA cluster: arg-max (ties -> lowest hypothesis), local optimisation, ordered inlier list
//   k_epi_vote_batch        recoverPose's cheirality vote, one thread per (inlier, candidate)
//   k_triangulate           one thread per point: epi::triangulate_dlt
// Every RANSAC kernel, essential and homography (k_homo_*_batch), has a pair dimension (one pair per blockIdx.y, one finish
// cluster per pair).  The batch calls run them over the matched frame pairs of a batch; the single-pair calls run them as a batch
// of one (cap = n, pn[0] = n uploaded with the points), with the same row layout (ransac_rows).  What follows the RANSACs is
// written once for host and device: recoverPose's pick (epi::recover_pose_pick, in k_epi_pick and mvo_epi_essential_end) and the
// homography motions (epi::homography_motions, in mvo_epi_homography_end and two_view_batch.cu).
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
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(EFIN_C * clusters);
  cfg.blockDim = dim3(EFIN_T);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = EFIN_C;
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

// Blocks one after the other at 256-byte boundaries from base.  A layout runs twice: with base == nullptr it only measures (`end`),
// then it runs again over the buffer reserved for that many bytes.
struct Blocks {
  uint8_t *base;
  size_t end = 0;
  template <class T> T *take(size_t count) {
    T *p = base ? (T *)(base + end) : nullptr;
    end = (end + count * sizeof(T) + 255) & ~(size_t)255;
    return p;
  }
};

// One RANSAC's device rows for n_pairs pairs (epipolar_kernels.cuh, "batch of frame pairs"), inputs first and outputs last: points
// and pn, hypothesis rows (72 B model, valid, count), finish outputs and inlier lists.  The batch calls and the single-pair jobs
// (one pair, cap = n) both lay them out here.
struct RansacRows {
  float *p1, *p2;
  int32_t *pn;
  double *models, *od;
  int32_t *valid, *cnt, *oi, *inl;
};

RansacRows ransac_rows(Blocks &L, int n_pairs, int cap, int H) {
  const size_t np = (size_t)n_pairs, nh = np * H;
  RansacRows r;
  r.p1 = L.take<float>(np * cap * 2); r.p2 = L.take<float>(np * cap * 2); r.pn = L.take<int32_t>(np);
  r.models = L.take<double>(nh * 9); r.valid = L.take<int32_t>(nh); r.cnt = L.take<int32_t>(nh);
  r.od = L.take<double>(np * EPIB_OUT_D); r.oi = L.take<int32_t>(np * EPIB_OUT_I); r.inl = L.take<int32_t>(np * cap);
  return r;
}

// The launch geometry of both RANSACs for n_pairs pairs of at most cap correspondences.  One focal length f = (fx + fy) / 2
// (epipolar_geometry.cpp:26-27) and thr2 = (threshold / f)^2: findEssentialMat divides the threshold by the focal length, the
// homography works in pixels scaled by 1 / f.  Scoring: about as many CTAs in all as 4 per SM (what one pair gets on its own), at
// least one per pair and at most one per 8 hypotheses, each staging its pair's points (cap x 32 B of shared memory).
struct RansacGeom {
  double f, cx, cy, thr2;
  int H;
  dim3 hyp, score;
  size_t smem;
};

template <class Score>
int ransac_geom(mvo_ctx *ctx, Score score, const double *K, double threshold, int cap, int n_pairs, RansacGeom *g) {
  g->f = (K[0] + K[4]) / 2; g->cx = K[2]; g->cy = K[5];
  g->thr2 = (threshold / g->f) * (threshold / g->f);
  g->H = ctx->prm.epi_hypotheses;
  int per_pair = (4 * ctx->sm_count + n_pairs - 1) / n_pairs;
  if (per_pair > (g->H + 7) / 8) per_pair = (g->H + 7) / 8;
  g->hyp = dim3((g->H + 127) / 128, n_pairs);
  g->score = dim3(per_pair, n_pairs);
  g->smem = (size_t)cap * 4 * sizeof(double);
  if (g->smem > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(score, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->smem));
  return MVO_OK;
}

// hypotheses, scoring, finish and, with vote, recoverPose's cheirality vote of the essential-matrix RANSAC
int epi_essential_enqueue(mvo_ctx *ctx, const RansacRows &r, int cap, int n_pairs, const double *K, double threshold, bool vote, RansacGeom *g) {
  MVO_TRY(ransac_geom(ctx, k_epi_score_batch, K, threshold, cap, n_pairs, g));
  const EpiCam cam = {g->f, g->cx, g->cy};
  { KTimer kt(ctx, KC_EPI);
  k_epi_hypotheses_batch<<<g->hyp, 128, 0, ctx->stream>>>(r.p1, r.p2, r.pn, cap, cam, ctx->prm.pnp_seed, g->H, r.models, r.valid); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_SCORE);
  k_epi_score_batch<<<g->score, 256, g->smem, ctx->stream>>>(r.p1, r.p2, r.pn, cap, cam, g->thr2, g->H, r.models, r.valid, r.cnt); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_FINISH);
    MVO_CUDA(ctx, launch_finish_cluster(ctx, (unsigned)n_pairs, sizeof(EpiFinSmem), k_epi_finish_batch, (const float *)r.p1, (const float *)r.p2,
                                        (const int32_t *)r.pn, cap, cam, g->thr2, g->H, (const double *)r.models, (const int32_t *)r.cnt, r.od, r.oi, r.inl)); }
  MVO_CHECK_LAUNCH(ctx);
  if (vote) {
    KTimer kt(ctx, KC_EPI);
    k_epi_vote_batch<<<dim3((cap + 63) / 64, n_pairs), 256, 0, ctx->stream>>>(r.p1, r.p2, r.pn, cap, cam, r.od, r.oi, r.inl);
    MVO_CHECK_LAUNCH(ctx);
  }
  return MVO_OK;
}

// hypotheses (which also zero each pair's finish outputs), scoring and finish of the homography RANSAC
int epi_homography_enqueue(mvo_ctx *ctx, const RansacRows &r, int cap, int n_pairs, const double *K, double threshold, RansacGeom *g) {
  MVO_TRY(ransac_geom(ctx, k_homo_score_batch, K, threshold, cap, n_pairs, g));
  const HomoCam cam = {g->f, g->cx, g->cy};
  { KTimer kt(ctx, KC_EPI);
  k_homo_hypotheses_batch<<<g->hyp, 128, 0, ctx->stream>>>(r.p1, r.p2, r.pn, cap, cam, ctx->prm.pnp_seed, g->H, r.models, r.valid, r.od, r.oi); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_SCORE);
  k_homo_score_batch<<<g->score, 256, g->smem, ctx->stream>>>(r.p1, r.p2, r.pn, cap, cam, g->thr2, g->H, r.models, r.valid, r.cnt); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_EPI_FINISH);
    MVO_CUDA(ctx, launch_finish_cluster(ctx, (unsigned)n_pairs, sizeof(HomoFinSmem), k_homo_finish_batch, (const float *)r.p1, (const float *)r.p2,
                                        (const int32_t *)r.pn, cap, cam, g->thr2, g->H, (const double *)r.models, (const int32_t *)r.cnt, r.od, r.oi, r.inl)); }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

// The scratch of both batch calls in ctx->epib_buf, for n_pairs pairs of at most cap correspondences: the essential RANSAC's rows
// (with tri also the normalised-plane points).  With rel (mvo_estimate_relative_poses_batch_dev; tri must be set too) also the
// homography finish outputs and inlier rows, the internal essential records and the (R | t) of every solution.  The homography rows
// reuse the points and the hypothesis rows, which k_epi_finish_batch has consumed by the time k_homo_hypotheses_batch runs on the
// same stream.  Without rel the caller points e.inl at its own inlier rows.
struct EpiBatchScratch {
  RansacRows e, h;
  float *np1, *np2;
  mvo_two_view_result *ess;
  double *rt;
};

int epi_batch_scratch(mvo_ctx *ctx, int n_pairs, int cap, bool tri, bool rel, EpiBatchScratch *b) {
  const size_t np = (size_t)n_pairs, pts = np * cap * 2;
  auto lay = [&](uint8_t *base) {
    Blocks L{base};
    *b = EpiBatchScratch();
    b->e = ransac_rows(L, n_pairs, cap, ctx->prm.epi_hypotheses);
    if (tri) { b->np1 = L.take<float>(pts); b->np2 = L.take<float>(pts); }
    if (rel) {
      b->h = b->e;
      b->h.od = L.take<double>(np * EPIB_OUT_D); b->h.oi = L.take<int32_t>(np * EPIB_OUT_I); b->h.inl = L.take<int32_t>(np * cap);
      b->ess = L.take<mvo_two_view_result>(np); b->rt = L.take<double>(np * 5 * 12);
    }
    return L.end;
  };
  MVO_TRY(mvo_reserve(ctx, ctx->epib_buf, lay(nullptr)));
  lay((uint8_t *)ctx->epib_buf.p);
  return MVO_OK;
}

// The single-pair job of either RANSAC, a batch of one (cap = n) in the job's own buffers: pts1 / pts2 / pn staged and uploaded in
// one copy, the model's RANSAC (essential with recoverPose's vote when vote, else homography), the finish outputs and the inlier
// list queued back in one copy; nothing waits.  `extra` more bytes of both buffers are the caller's (*d_extra, *h_extra).
int epi_job_begin(mvo_ctx *ctx, DevBuf &dbuf, PinBuf &hbuf, bool essential, const float *pts1, const float *pts2, int n, const double *K,
                  double threshold, bool vote, size_t extra, uint8_t **d_extra, uint8_t **h_extra, MvoEpiJob *job) {
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int H = ctx->prm.epi_hypotheses;
  Blocks L{nullptr};
  ransac_rows(L, 1, n, H);
  MVO_TRY(mvo_reserve(ctx, dbuf, L.end + extra));
  uint8_t *d = (uint8_t *)dbuf.p;
  L = Blocks{d};
  const RansacRows r = ransac_rows(L, 1, n, H);
  // pinned staging: the inputs at their device offsets, then the outputs from od to the end of the inlier list, then the extra
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  uint8_t *od = (uint8_t *)r.od;
  const size_t in = (uint8_t *)(r.pn + 1) - d, o_res = al(in), res = (uint8_t *)(r.inl + n) - od, o_extra = al(o_res + res);
  MVO_TRY(mvo_reserve_pinned(ctx, hbuf, o_extra + extra));
  uint8_t *h = (uint8_t *)hbuf.p, *hr = h + o_res;
  memcpy(h + ((uint8_t *)r.p1 - d), pts1, (size_t)n * 8);
  memcpy(h + ((uint8_t *)r.p2 - d), pts2, (size_t)n * 8);
  memcpy(h + ((uint8_t *)r.pn - d), &n, 4);
  MVO_CUDA(ctx, cudaMemcpyAsync(d, h, in, cudaMemcpyHostToDevice, ctx->stream));
  RansacGeom g;
  if (essential) MVO_TRY(epi_essential_enqueue(ctx, r, n, 1, K, threshold, vote, &g));
  else MVO_TRY(epi_homography_enqueue(ctx, r, n, 1, K, threshold, &g));
  MVO_CUDA(ctx, cudaMemcpyAsync(hr, od, res, cudaMemcpyDeviceToHost, ctx->stream));
  memset(job, 0, sizeof *job);
  job->stream = ctx->stream; job->n = n; job->H = H; job->thr2 = g.thr2; job->f = g.f;
  job->h_out = (double *)hr; job->h_oi = (int32_t *)(hr + ((uint8_t *)r.oi - od)); job->h_inl = (int32_t *)(hr + ((uint8_t *)r.inl - od));
  job->d_valid = r.valid; job->d_cnt = r.cnt; job->d_model = r.models;
  if (d_extra) { *d_extra = d + L.end; *h_extra = h + o_extra; }
  return MVO_OK;
}

// gather, the essential RANSAC with its vote, pick: six launches; pair p's inliers at b.e.inl + p * cap, its record in res[p]
int epi_essential_batch_enqueue(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap, const int32_t *d_pairs,
                                int n_pairs, const mvo_dmatch *d_matches, const int32_t *d_n_matches, const double *K, double threshold,
                                const EpiBatchScratch &b, mvo_two_view_result *res) {
  { KTimer kt(ctx, KC_EPI);
  k_epi_gather<<<n_pairs, 256, 0, ctx->stream>>>(d_kpts, d_counts, batch, cap, (const int2 *)d_pairs, d_matches, d_n_matches, K[0], K[4], K[2], K[5],
                                                 b.e.p1, b.e.p2, b.np1, b.np2, b.e.pn); }
  MVO_CHECK_LAUNCH(ctx);
  RansacGeom g;
  MVO_TRY(epi_essential_enqueue(ctx, b.e, cap, n_pairs, K, threshold, true, &g));
  { KTimer kt(ctx, KC_EPI);
  k_epi_pick<<<(n_pairs + 127) / 128, 128, 0, ctx->stream>>>(b.e.pn, n_pairs, b.e.od, b.e.oi, res); }
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
  const bool tri = d_pts3d != nullptr;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  EpiBatchScratch b;
  MVO_TRY(epi_batch_scratch(ctx, n_pairs, cap, tri, false, &b));
  b.e.inl = d_inliers;
  MVO_TRY(epi_essential_batch_enqueue(ctx, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, K, threshold, b, d_res));
  if (tri) {
    KTimer kt(ctx, KC_EPI);
    k_triangulate_batch<<<dim3((cap + 127) / 128, n_pairs), 128, 0, ctx->stream>>>(b.np1, b.np2, d_res, cap, d_inliers, d_pts3d);
    MVO_CHECK_LAUNCH(ctx);
  }
  return MVO_OK;
}

// declared in mvo_internal.h: the triangulation of mvo_vo_keyframe_points_batch_dev (its other two launches are in vo_init_batch.cu)
int mvo_kf_triangulate_launch(mvo_ctx *ctx, const MvoKeyframePoints &a) {
  { KTimer kt(ctx, KC_EPI);
  k_kf_triangulate<<<dim3((a.cap + 127) / 128, a.n_pairs), 128, 0, ctx->stream>>>(a.kpts, (const int2 *)a.pairs, a.matches, a.ess_inliers, a.out,
                                                                                 a.cap, a.fx, a.fy, a.cx, a.cy, a.kept_pts3d); }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

// The combine step lives in two_view_batch.cu, a translation unit of its own that is compiled without contraction (Makefile).
// libmvo.so always links it; a library assembled from a subset of the units without it reports MVO_ERR_UNSUPPORTED for the call.
int mvo_relative_poses_combine(mvo_ctx *ctx, const MvoRelPosesCombine &a) __attribute__((weak));

// mvo_estimate_relative_poses_batch_dev (mvo.h): the essential half (six launches, into an internal mvo_two_view_result array),
// the homography half (three launches), the combine step (two_view_batch.cu: decomposition, visibility filter, inlier rows,
// invRt, scores, E/H choice) and, with d_pts3d, one triangulation launch over (pair, solution).  Scratch in ctx->epib_buf.
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
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  EpiBatchScratch b;
  MVO_TRY(epi_batch_scratch(ctx, n_pairs, cap, true, true, &b));
  // ---- essential half (:43-48) ----
  MVO_TRY(epi_essential_batch_enqueue(ctx, d_kpts, d_counts, batch, cap, d_pairs, n_pairs, d_matches, d_n_matches, K, ctx->prm.essential_threshold,
                                      b, b.ess));
  // ---- homography half (:56-67), on the same points ----
  RansacGeom g;
  MVO_TRY(epi_homography_enqueue(ctx, b.h, cap, n_pairs, K, ctx->prm.homography_threshold, &g));
  // ---- combine (:56-154 after the RANSACs) ----
  MvoRelPosesCombine a;
  a.n_matches = d_n_matches; a.ess = b.ess; a.inl_e = b.e.inl; a.hom_i = b.h.oi; a.inl_h = b.h.inl; a.hom_d = b.h.od;
  a.p1 = b.e.p1; a.p2 = b.e.p2; a.np1 = b.np1; a.np2 = b.np2;
  a.n_pairs = n_pairs; a.cap = cap; a.hom_d_stride = EPIB_OUT_D; a.hom_i_stride = EPIB_OUT_I; a.motion_cam2_to_cam1 = motion_cam2_to_cam1;
  for (int q = 0; q < 9; ++q) a.K[q] = K[q];
  a.eh_ratio_threshold = ctx->prm.eh_ratio_threshold;
  a.res = d_res; a.inliers = d_inliers; a.rt = b.rt;
  MVO_TRY(mvo_relative_poses_combine(ctx, a));
  // ---- triangulation of every solution (:105-112), with the (R, t) from before invRt ----
  if (d_pts3d) {
    KTimer kt(ctx, KC_EPI);
    k_triangulate_solutions_batch<<<dim3((cap + 127) / 128, 5, n_pairs), 128, 0, ctx->stream>>>(b.np1, b.np2, d_res, b.rt, cap, d_inliers, d_pts3d);
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
  if (!((K[0] + K[4]) / 2 > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "K: focal length must be positive");
  if ((size_t)n * 4 * sizeof(double) > 200 * 1024)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "estiMotionByEssential: more than %d correspondences", 200 * 1024 / 32);
  // the triangulation block after the RANSAC's, laid out alike in both buffers: np1, np2 (n x 2 floats each), R | t (12 doubles) in,
  // n x 3 floats out
  const size_t tri_in = (size_t)n * 16 + 96, o_tout = (tri_in + 255) & ~(size_t)255;
  uint8_t *d, *h;
  MVO_TRY(epi_job_begin(ctx, ctx->epi_ess_buf, ctx->epi_ess_h, true, pts1, pts2, n, K, threshold, want_pose != 0, tri ? o_tout + (size_t)n * 12 : 0,
                        &d, &h, job));
  job->want_pose = want_pose != 0; job->tri = tri; job->tri_stream = ctx->stream;
  if (!tri) return MVO_OK;
  // the triangulation does not depend on the RANSAC: it runs on the context's side stream next to it (on the same stream when
  // per-kernel event timing is on, or when this job itself was pointed at the side stream)
  cudaStream_t tri_stream = ctx->stream, side = ctx->timing_mask ? nullptr : mvo_side_stream(ctx);
  if (side && side != ctx->stream) tri_stream = side;
  memcpy(h, tri_np1, (size_t)n * 8);
  memcpy(h + (size_t)n * 8, tri_np2, (size_t)n * 8);
  memcpy(h + (size_t)n * 16, tri_R, 72);
  memcpy(h + (size_t)n * 16 + 72, tri_t, 24);
  MVO_CUDA(ctx, cudaMemcpyAsync(d, h, tri_in, cudaMemcpyHostToDevice, tri_stream));
  {
    cudaStream_t keep = ctx->stream;
    ctx->stream = tri_stream;              // KTimer records on ctx->stream
    { KTimer kt(ctx, KC_EPI);
    k_triangulate<<<(n + 127) / 128, 128, 0, tri_stream>>>((const float *)d, (const float *)(d + (size_t)n * 8), nullptr, n,
                                                            (const double *)(d + (size_t)n * 16), (float *)(d + o_tout)); }
    ctx->stream = keep;
  }
  MVO_CHECK_LAUNCH(ctx);
  MVO_CUDA(ctx, cudaMemcpyAsync(h + o_tout, d + o_tout, (size_t)n * 12, cudaMemcpyDeviceToHost, tri_stream));
  job->tri_stream = tri_stream; job->h_tri = (float *)(h + o_tout);
  return MVO_OK;
}

// second half: wait for the job's stream, recoverPose's pick, outputs
int mvo_epi_essential_end(mvo_ctx *ctx, MvoEpiJob *job, double *E, double *R, double *t, int32_t *inliers, int *n_inliers, float *tri_out) {
  MVO_CUDA(ctx, cudaStreamSynchronize(job->stream));
  if (job->tri && job->tri_stream != job->stream) MVO_CUDA(ctx, cudaStreamSynchronize(job->tri_stream));
  const int n = job->n, H = job->H;
  const double *h_out = job->h_out;
  const int32_t *h_i = job->h_oi, *h_inl = job->h_inl;
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
  epi::recover_pose_pick(h_out, h_i + 8, E, R, t);
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

// first half (own device / pinned buffers, so that it can run next to an essential-matrix job on another stream)
int mvo_epi_homography_begin(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold, MvoEpiJob *job) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!pts1 || !pts2 || !K || !job) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByHomography: null pointer");
  if (n < 4) return mvo_fail(ctx, MVO_ERR_DEGENERATE, "estiMotionByHomography: %d correspondences (< 4)", n);
  if (!(threshold > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "estiMotionByHomography: threshold must be positive");
  if (!(K[0] > 0 && K[4] > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "K: focal lengths must be positive");
  if ((size_t)n * 4 * sizeof(double) > 200 * 1024)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "estiMotionByHomography: more than %d correspondences", 200 * 1024 / 32);
  return epi_job_begin(ctx, ctx->epi_homo_buf, ctx->epi_homo_h, false, pts1, pts2, n, K, threshold, false, 0, nullptr, nullptr, job);
}

int mvo_epi_homography_end(mvo_ctx *ctx, MvoEpiJob *job, const double *K, double *Hout, double *Rs, double *ts, double *normals, int *n_solutions,
                           int32_t *inliers, int *n_inliers) {
  MVO_CUDA(ctx, cudaStreamSynchronize(job->stream));
  const double *h_out = job->h_out;
  const int32_t *h_i = job->h_oi, *h_inl = job->h_inl;
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
  *n_solutions = epi::homography_motions(Hout, K, Rs, ts, normals);
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
  return mvo_do_triangulation_multi(ctx, pts_np1, pts_np2, n, 1, &R, &t, &inliers, &n_inliers, &pts3d);
}

}  // extern "C"
