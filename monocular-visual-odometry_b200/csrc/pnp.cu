// Batched RANSAC PnP for sm_90a — replaces the inline cv::solvePnPRansac call at reference
// src/vo/vo.cpp:318-320 (iterationsCount 100, reprojectionError 2.0, confidence 0.999,
// useExtrinsicGuess false, default SOLVEPNP_ITERATIVE).  Structure kept from OpenCV (SURVEY.md
// App. C): hypotheses from minimal sets -> consensus set of the best hypothesis (returned as
// ascending indices) -> iterative least-squares refit on exactly those inliers.  What differs by
// design: all H hypotheses (default 4096, not <=100 adaptive) are generated and scored in one
// batch; the minimal solver is a P3P (3 points + 1 to disambiguate) instead of 5-point EPnP.
//
//   k_pnp_hypotheses  one thread per hypothesis: counter-based sampling (splitmix64), P3P by
//                     intersecting the two distance-ratio conics through their degenerate
//                     pencil member, pose from the three depths, 4th point picks the root.
//   k_pnp_score       persistent grid, one warp per hypothesis at a time, the N correspondences
//                     staged once per CTA in shared memory; fp64 reprojection, count(err^2<=thr^2).
//   k_pnp_finish      one CTA: arg-max (ties -> lowest hypothesis), ordered inlier compaction,
//                     damped Gauss-Newton on SE(3) over the inliers (fp64).
// All arithmetic fp64: the stage is latency-bound (N*H = 8.2e6 reprojections), not FLOP-bound.
#include <string.h>
#include <algorithm>
#include <cmath>
#include "mvo_internal.h"

namespace {

#define PNP_DYN_SMEM(type, name) extern __shared__ type name[]
#include "launch_pdl.cuh"
#include "pnp_kernels.cuh"

// The rest of poseEstimationPnP_ (vo.cpp:333-380) for every job of mvo_vo_pnp_batch_dev, one CTA per job: the record, the inlier
// matches (matches_with_map_ after the swap), T_w_c = [R|t]^-1 and the jump check against the previous frame.  The inverse and
// the distance use __dmul_rn / __dadd_rn in the host's operation order (inv_rigid, trans_dist): no contraction, the host's bits.
__global__ void __launch_bounds__(128)
k_pnp_batch_tail(const mvo_map_matches_result *__restrict__ mm, const mvo_dmatch *__restrict__ matches, int cap,
                 const double *__restrict__ T_prev, double max_dist, const int32_t *__restrict__ job_st,
                 const double *__restrict__ pose_io, const int32_t *__restrict__ out_i, const int32_t *__restrict__ inl,
                 mvo_vo_pnp_result *__restrict__ out, mvo_dmatch *__restrict__ kept) {
  const int j = blockIdx.x, tid = threadIdx.x;
  pdl_wait();
  pdl_launch_dependents();
  mvo_vo_pnp_result *o = out + j;
  const int st = job_st[j];
  if (st != MVO_OK) { if (tid == 0) o->status = st; return; }
  const int ni = out_i[4 * j], best = out_i[4 * j + 1];          // 0 and -1 without a model (also below min_pnp_points)
  if (kept)
    for (int k = tid; k < ni; k += blockDim.x) kept[(size_t)j * cap + k] = matches[(size_t)j * cap + inl[(size_t)j * cap + k]];
  if (tid != 0) return;
  const double *P = pose_io + (size_t)j * 12, *Tp = T_prev + (size_t)j * 16;
  double T[16];
  int ok = best >= 0;
  if (ok) {
    for (int i = 0; i < 3; ++i) {
      for (int c = 0; c < 3; ++c) T[i * 4 + c] = P[c * 3 + i];
      T[i * 4 + 3] = -__dadd_rn(__dadd_rn(__dmul_rn(P[i], P[9]), __dmul_rn(P[3 + i], P[10])), __dmul_rn(P[6 + i], P[11]));
    }
    T[12] = T[13] = T[14] = 0; T[15] = 1;
    const double dx = __dadd_rn(T[3], -Tp[3]), dy = __dadd_rn(T[7], -Tp[7]), dz = __dadd_rn(T[11], -Tp[11]);
    if (sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))) >= max_dist) ok = 0;
  }
  if (!ok)
    for (int q = 0; q < 16; ++q) T[q] = Tp[q];
  o->status = MVO_OK;
  o->pnp_ok = ok;
  o->n_matches = mm[j].n_matches;
  o->n_inliers = ni;
  o->best = best;
  o->pad[0] = o->pad[1] = o->pad[2] = 0;
  for (int q = 0; q < 12; ++q) o->Rt[q] = P[q];
  for (int q = 0; q < 16; ++q) o->T_w_c[q] = T[q];
}

}  // namespace

// ---------------------------------------------------------------------------- host entry
static void rotation_to_rvec(const double *R, double *rvec) {
  // via the unit quaternion: robust for every angle in [0, pi]
  double q[4];
  const double tr = R[0] + R[4] + R[8];
  if (tr > 0) { double s = sqrt(tr + 1.0) * 2; q[0] = 0.25 * s; q[1] = (R[7] - R[5]) / s; q[2] = (R[2] - R[6]) / s; q[3] = (R[3] - R[1]) / s; }
  else if (R[0] > R[4] && R[0] > R[8]) { double s = sqrt(1.0 + R[0] - R[4] - R[8]) * 2; q[0] = (R[7] - R[5]) / s; q[1] = 0.25 * s; q[2] = (R[1] + R[3]) / s; q[3] = (R[2] + R[6]) / s; }
  else if (R[4] > R[8]) { double s = sqrt(1.0 + R[4] - R[0] - R[8]) * 2; q[0] = (R[2] - R[6]) / s; q[1] = (R[1] + R[3]) / s; q[2] = 0.25 * s; q[3] = (R[5] + R[7]) / s; }
  else { double s = sqrt(1.0 + R[8] - R[0] - R[4]) * 2; q[0] = (R[3] - R[1]) / s; q[1] = (R[2] + R[6]) / s; q[2] = (R[5] + R[7]) / s; q[3] = 0.25 * s; }
  if (q[0] < 0) for (int i = 0; i < 4; ++i) q[i] = -q[i];
  const double vn = sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (vn < 1e-15) { rvec[0] = rvec[1] = rvec[2] = 0; return; }
  const double th = 2 * atan2(vn, q[0]);
  for (int i = 0; i < 3; ++i) rvec[i] = th * q[1 + i] / vn;
}

static void rvec_to_rotation(const double *w, double *R) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double A, B;
  if (th < 1e-8) { A = 1 - th2 / 6; B = 0.5 - th2 / 24; }
  else { A = sin(th) / th; B = (1 - cos(th)) / th2; }
  const double wx = w[0], wy = w[1], wz = w[2];
  R[0] = 1 - B * (wy * wy + wz * wz); R[1] = -A * wz + B * wx * wy;       R[2] = A * wy + B * wx * wz;
  R[3] = A * wz + B * wx * wy;        R[4] = 1 - B * (wx * wx + wz * wz); R[5] = -A * wx + B * wy * wz;
  R[6] = -A * wy + B * wx * wz;       R[7] = A * wx + B * wy * wz;        R[8] = 1 - B * (wx * wx + wy * wy);
}

static int pnp_hyp_count(const mvo_ctx *ctx);
struct PnpWs { float *p3, *p2; double *poses, *pose_io, *ex, *eo, *stats; int32_t *valid, *counts, *out_i, *inl, *ef; };

// ba.cu
int mvo_ba_pose_launch(mvo_ctx *ctx, int F, int E, int chunk, const int32_t *d_eframe, const double *d_X, const double *d_obs, double fx, double fy,
                       double cx, double cy, const double *info, int iters, int use_huber, double huber, int fix_first,
                       double step_tol, double *d_poses, double *d_stats, int n_jobs = 0);

static int pnp_ws(mvo_ctx *ctx, int n, int H, PnpWs *w) {
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t o_p3 = 0, o_p2 = al(o_p3 + (size_t)n * 12), o_inl = al(o_p2 + (size_t)n * 8), o_ex = al(o_inl + (size_t)n * 4);
  const size_t o_eo = al(o_ex + (size_t)n * 24), o_ef = al(o_eo + (size_t)n * 16), o_end = al(o_ef + (size_t)n * 4);
  MVO_TRY(mvo_reserve(ctx, ctx->pnp_pts, o_end));
  MVO_TRY(mvo_reserve(ctx, ctx->pnp_hyp, (size_t)H * 12 * 8 + 256));
  MVO_TRY(mvo_reserve(ctx, ctx->pnp_cnt, (size_t)H * 8 + 512));
  MVO_TRY(mvo_reserve(ctx, ctx->pnp_out, 1024));
  uint8_t *b = (uint8_t *)ctx->pnp_pts.p;
  w->p3 = (float *)(b + o_p3); w->p2 = (float *)(b + o_p2); w->inl = (int32_t *)(b + o_inl);
  w->ex = (double *)(b + o_ex); w->eo = (double *)(b + o_eo); w->ef = (int32_t *)(b + o_ef);
  w->poses = (double *)ctx->pnp_hyp.p;
  w->valid = (int32_t *)ctx->pnp_cnt.p;
  w->counts = w->valid + ((H + 63) & ~63);
  w->pose_io = (double *)ctx->pnp_out.p;
  w->out_i = (int32_t *)((uint8_t *)ctx->pnp_out.p + 256);
  w->stats = (double *)((uint8_t *)ctx->pnp_out.p + 512);
  return MVO_OK;
}

static int pnp_cam(mvo_ctx *ctx, const double *K, PnpCam *cam) {
  if (!K) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "null K");
  cam->fx = K[0]; cam->fy = K[4]; cam->cx = K[2]; cam->cy = K[5];
  if (!(cam->fx > 0 && cam->fy > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "K: focal lengths must be positive");
  return MVO_OK;
}

// Least-squares refit of the pose on the one-frame edge list written by k_pnp_finish: the same
// pose-only LM as the fixed-points BA (no robust kernel, identity information, fx/fy), stopping
// once an accepted step is below 1e-8 (quadratic convergence: the next step would be ~1e-16).  E = n is an upper bound: unused edge slots carry frame -1.
static int pnp_refit(mvo_ctx *ctx, const PnpWs &w, int n, const PnpCam &cam) {
  static const double I2[4] = {1, 0, 0, 1};
  return mvo_ba_pose_launch(ctx, 1, n, 1, w.ef, w.ex, w.eo, cam.fx, cam.fy, cam.cx, cam.cy, I2, ctx->prm.pnp_refine_iters, 0, 1.0, 0,
                            1e-8, w.pose_io, w.stats);
}

// hypotheses -> scores -> consensus set of the best hypothesis -> least-squares refit, all on ctx->stream;
// w.p3 / w.p2 hold the n correspondences on the device
static int pnp_hyp_count(const mvo_ctx *ctx) { return ctx->prm.pnp_mode == 1 ? 100 : ctx->prm.pnp_hypotheses; }   // vo.cpp:315: iterationsCount = 100

// The hypotheses of either mode into w.poses / w.valid: P3P on counter-based samples (pnp_mode = 0), or the EPnP poses of
// cv::solvePnPRansac's 100 iterations (pnp_mode = 1, pnp_cv_kernels.cuh).
static int pnp_enqueue_hypotheses(mvo_ctx *ctx, const PnpWs &w, int n, const PnpCam &cam, const int32_t *n_dev) {
  const int H = pnp_hyp_count(ctx);
  if (ctx->prm.pnp_mode == 1) {
    { KTimer kt(ctx, KC_PNP_HYP);
    k_pnp_epnp<<<(H + CVP_WARPS - 1) / CVP_WARPS, CVP_WARPS * 32, 0, ctx->stream>>>(w.p3, w.p2, n, n_dev, cam, H, w.poses, w.valid); }
    MVO_CHECK_LAUNCH(ctx);
    return MVO_OK;
  }
  { KTimer kt(ctx, KC_PNP_HYP);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, (unsigned)((H + 127) / 128), 128, 0, 0, k_pnp_hypotheses<false>, (const float *)w.p3, (const float *)w.p2, n, n_dev, cam,
                           (uint64_t)ctx->prm.pnp_seed, H, w.poses, w.valid, PnpJobs())); }
  ctx->launches++;
  return MVO_OK;
}

// The scoring kernel of pnp_mode = 0 stages the n correspondences in shared memory (20 bytes each)
static int pnp_check_size(mvo_ctx *ctx, int n) {
  if (ctx->prm.pnp_mode != 1 && (size_t)n * 5 * sizeof(float) > 200 * 1024)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "solvePnPRansac: more than %d correspondences", 200 * 1024 / 20);
  return MVO_OK;
}

// pnp_mode = 1: cv::solvePnPRansac's own flow (pnp_cv_kernels.cuh) — 100 EPnP iterations evaluated in parallel, the adaptive loop replayed
static int pnp_score_finish_cv(mvo_ctx *ctx, const PnpWs &w, int n, const PnpCam &cam, const int32_t *n_dev) {
  const int H = pnp_hyp_count(ctx);
  const double thr2 = (double)ctx->prm.pnp_reproj_error * (double)ctx->prm.pnp_reproj_error;
  { KTimer kt(ctx, KC_PNP_SCORE);
  k_pnp_score_cv<<<(H + 7) / 8, 256, 0, ctx->stream>>>(w.p3, w.p2, n, n_dev, cam, (float)thr2, H, w.poses, w.valid, w.counts); }
  MVO_CHECK_LAUNCH(ctx);
  { KTimer kt(ctx, KC_PNP_FINISH);
  k_pnp_finish<false><<<1, FIN_T, 0, ctx->stream>>>(w.p3, w.p2, n, n_dev, cam, thr2, H, w.poses, w.counts, 2, ctx->prm.pnp_refine_iters,
                                             w.pose_io, w.out_i, w.inl, w.ex, w.eo, w.ef); }
  MVO_CHECK_LAUNCH(ctx);
  ctx->pnp_last_h = H;
  return pnp_refit(ctx, w, n, cam);
}

// scores -> consensus set of the best hypothesis -> least-squares refit, on the hypotheses in w.poses / w.valid
static int pnp_score_finish(mvo_ctx *ctx, const PnpWs &w, int n, const PnpCam &cam, const int32_t *n_dev) {
  if (ctx->prm.pnp_mode == 1) return pnp_score_finish_cv(ctx, w, n, cam, n_dev);
  MVO_TRY(pnp_check_size(ctx, n));
  const int H = ctx->prm.pnp_hypotheses;
  const size_t smem = (size_t)n * 5 * sizeof(float);
  const double thr2 = (double)ctx->prm.pnp_reproj_error * (double)ctx->prm.pnp_reproj_error;
  // the 48 KB default covers static and dynamic shared memory together: k_pnp_score's own s_wmax[8] counts as well
  if (smem + 8 * sizeof(float) > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_pnp_score<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (H + 7) / 8;                                   // one hypothesis per warp while the CTAs of one wave allow it
  if (grid > 4 * ctx->sm_count) grid = 4 * ctx->sm_count;
  { KTimer kt(ctx, KC_PNP_SCORE);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, (unsigned)grid, 256, smem, 0, k_pnp_score<false>, (const float *)w.p3, (const float *)w.p2, n, n_dev, cam, thr2, H,
                           (const double *)w.poses, (const int32_t *)w.valid, w.counts)); }
  ctx->launches++;
  { KTimer kt(ctx, KC_PNP_FINISH);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, 1, FIN_T, 0, 0, k_pnp_finish<false>, (const float *)w.p3, (const float *)w.p2, n, n_dev, cam, thr2, H,
                           (const double *)w.poses, (const int32_t *)w.counts, 0, (int)ctx->prm.pnp_refine_iters, w.pose_io, w.out_i, w.inl, w.ex, w.eo, w.ef)); }
  ctx->launches++;
  ctx->pnp_last_h = H;
  // the refit runs on the consensus set whose size only the device knows: launch it for the
  // worst case E = n with the real count read on the device (edges beyond n_in are masked out)
  return pnp_refit(ctx, w, n, cam);
}

static int pnp_enqueue(mvo_ctx *ctx, const PnpWs &w, int n, const PnpCam &cam, const int32_t *n_dev = nullptr) {
  MVO_TRY(pnp_check_size(ctx, n));
  MVO_TRY(pnp_enqueue_hypotheses(ctx, w, n, cam, n_dev));
  return pnp_score_finish(ctx, w, n, cam, n_dev);
}

// Device-resident entry points for the tracker (tracker.cpp): reserve the workspace for n correspondences
// (the caller gathers them into *p3 / *p2 on ctx->stream), then enqueue the whole solvePnPRansac replacement.
// Results stay on the device: pose_io = [R|t] world->camera after the refit, out_i[0] = consensus-set size
// (< 4: no model), inl = its ascending indices.
int mvo_pnp_dev_buffers(mvo_ctx *ctx, int n, float **p3, float **p2, double **pose_io, int32_t **out_i, int32_t **inl) {
  PnpWs w;
  MVO_TRY(pnp_ws(ctx, n, pnp_hyp_count(ctx), &w));
  *p3 = w.p3; *p2 = w.p2; *pose_io = w.pose_io; *out_i = w.out_i; *inl = w.inl;
  return MVO_OK;
}

// n = number of correspondences, or their upper bound when d_n (device counter) is given.  own_hypotheses = false scores
// the hypotheses already in the workspace (mvo_test_pnp_dev).
static int pnp_dev_run(mvo_ctx *ctx, int n, const double *K, const int32_t *d_n, bool own_hypotheses) {
  if (n < 4) return mvo_fail(ctx, MVO_ERR_DEGENERATE, "solvePnPRansac: %d correspondences (< 4)", n);
  PnpCam cam;
  MVO_TRY(pnp_cam(ctx, K, &cam));
  PnpWs w;
  MVO_TRY(pnp_ws(ctx, n, pnp_hyp_count(ctx), &w));
  return own_hypotheses ? pnp_enqueue(ctx, w, n, cam, d_n) : pnp_score_finish(ctx, w, n, cam, d_n);
}

int mvo_pnp_dev_run(mvo_ctx *ctx, int n, const double *K, const int32_t *d_n) { return pnp_dev_run(ctx, n, K, d_n, true); }

// Test entry (not part of the C ABI): the device-resident PnP as the tracker runs it.  Uploads n_upper correspondences and
// the device count (any value: the kernels clamp it to n_upper), optionally H = pnp_hypotheses caller-supplied hypotheses
// (poses H x 12, valid H; pnp_mode = 0 only) in place of k_pnp_hypotheses, runs mvo_pnp_dev_run's sequence with that count,
// waits, and returns pose_io[12], out_i[4], the inlier list inl[n_upper] and the H scores (counts, -1 = invalid).
extern "C" int mvo_test_pnp_dev(mvo_ctx *ctx, const float *pts3d, const float *pts2d, int n_upper, int count, const double *K,
                                const double *poses, const int32_t *valid, double *pose_io, int32_t *out_i, int32_t *inl,
                                int32_t *counts) {
  if (!ctx || !pts3d || !pts2d || !K || !pose_io || !out_i || !inl || !counts || (!poses) != (!valid)) return MVO_ERR_INVALID_ARG;
  if (poses && ctx->prm.pnp_mode == 1) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp test: supplied hypotheses need pnp_mode 0");
  if (n_upper < 4) return mvo_fail(ctx, MVO_ERR_DEGENERATE, "solvePnPRansac: %d correspondences (< 4)", n_upper);
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int H = pnp_hyp_count(ctx);
  float *d_p3, *d_p2;
  double *d_pose;
  int32_t *d_out, *d_inl;
  MVO_TRY(mvo_pnp_dev_buffers(ctx, n_upper, &d_p3, &d_p2, &d_pose, &d_out, &d_inl));
  PnpWs w;
  MVO_TRY(pnp_ws(ctx, n_upper, H, &w));
  MVO_TRY(mvo_reserve(ctx, ctx->ba_buf, 256));
  int32_t *d_n = (int32_t *)ctx->ba_buf.p;
  MVO_CUDA(ctx, cudaMemcpyAsync(d_p3, pts3d, (size_t)n_upper * 12, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d_p2, pts2d, (size_t)n_upper * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d_n, &count, 4, cudaMemcpyHostToDevice, ctx->stream));
  if (poses) {
    MVO_CUDA(ctx, cudaMemcpyAsync(w.poses, poses, (size_t)H * 96, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(w.valid, valid, (size_t)H * 4, cudaMemcpyHostToDevice, ctx->stream));
  }
  const int rc = pnp_dev_run(ctx, n_upper, K, d_n, !poses);
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));      // the uploads above are done with the host arrays on every path
  if (rc != MVO_OK) return rc;
  MVO_CUDA(ctx, cudaMemcpyAsync(pose_io, d_pose, 96, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(out_i, d_out, 16, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(inl, d_inl, (size_t)n_upper * 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(counts, w.counts, (size_t)H * 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MVO_OK;
}

// Scoring grid of the batch: the CTAs of all jobs together fill about one wave of 4 per SM, and no job gets more CTAs than it has
// warps of hypotheses.  Every hypothesis is scored by one warp over all of its job's points, so the counts do not depend on it.
static int pnp_batch_score_grid(const mvo_ctx *ctx, int n_jobs, int H) {
  const int per_job = (4 * ctx->sm_count + n_jobs - 1) / n_jobs;
  return std::max(1, std::min((H + 7) / 8, per_job));
}

// n_jobs x H hypothesis rows at most (96 + 8 bytes each): the bound of the essential-matrix batch
static const long long PNP_BATCH_MAX_HYP = 1ll << 22;

extern "C" {

int mvo_vo_pnp_batch_dev(mvo_ctx *ctx, const mvo_map_matches_result *d_mm, const mvo_dmatch *d_matches, const float *d_pts3d,
                         const float *d_pts2d, int n_jobs, int cap, const double *d_T_w_c_prev, const double *K,
                         const mvo_track_params *tp, mvo_vo_pnp_result *d_out, int32_t *d_inliers, mvo_dmatch *d_kept) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!d_mm || !d_matches || !d_pts3d || !d_pts2d || !d_T_w_c_prev || !K || !tp || !d_out || !d_inliers)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp batch: null pointer");
  if (!(std::isfinite(K[0]) && K[0] > 0 && std::isfinite(K[4]) && K[4] > 0))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp batch: focal lengths must be finite and positive");
  if (cap < 1 || n_jobs < 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp batch: cap %d, n_jobs %d", cap, n_jobs);
  if (!std::isfinite(tp->max_dist_to_prev)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp batch: max_dist_to_prev not finite");
  if (ctx->prm.pnp_mode == 1) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "pnp batch: pnp_mode 1 has no batch form");
  const int H = ctx->prm.pnp_hypotheses;
  if (cap > 8192 || n_jobs > 65535 || (long long)n_jobs * H > PNP_BATCH_MAX_HYP)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "pnp batch: cap %d (<= 8192), n_jobs %d (<= 65535), n_jobs x pnp_hypotheses %lld (<= %lld)",
                    cap, n_jobs, (long long)n_jobs * H, PNP_BATCH_MAX_HYP);
  if (n_jobs == 0) return MVO_OK;
  PnpCam cam;
  MVO_TRY(pnp_cam(ctx, K, &cam));
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  // scratch: hypotheses, validity and counts of every job, the finish outputs, the refit's edge rows and stats, job counts/statuses
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t nj = (size_t)n_jobs, nh = nj * H, ne = nj * cap;
  const size_t o_poses = 0, o_valid = al(o_poses + nh * 96), o_counts = al(o_valid + nh * 4), o_pose = al(o_counts + nh * 4);
  const size_t o_outi = al(o_pose + nj * 96), o_ex = al(o_outi + nj * 16), o_eo = al(o_ex + ne * 24), o_ef = al(o_eo + ne * 16);
  const size_t o_stats = al(o_ef + ne * 4), o_n = al(o_stats + nj * 128), o_st = al(o_n + nj * 4), o_end = al(o_st + nj * 4);
  MVO_TRY(mvo_reserve(ctx, ctx->pnpb_buf, o_end));
  uint8_t *b = (uint8_t *)ctx->pnpb_buf.p;
  double *poses = (double *)(b + o_poses), *pose_io = (double *)(b + o_pose), *ex = (double *)(b + o_ex), *eo = (double *)(b + o_eo);
  double *stats = (double *)(b + o_stats);
  int32_t *valid = (int32_t *)(b + o_valid), *counts = (int32_t *)(b + o_counts), *out_i = (int32_t *)(b + o_outi);
  int32_t *ef = (int32_t *)(b + o_ef), *job_n = (int32_t *)(b + o_n), *job_st = (int32_t *)(b + o_st);
  const double thr2 = (double)ctx->prm.pnp_reproj_error * (double)ctx->prm.pnp_reproj_error;
  PnpJobs jb;
  jb.mm = d_mm; jb.T_prev = d_T_w_c_prev; jb.min_pts = tp->min_pnp_points; jb.n = job_n; jb.status = job_st;
  { KTimer kt(ctx, KC_PNP_HYP);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, dim3((unsigned)((H + 127) / 128), (unsigned)n_jobs), dim3(128), 0, k_pnp_hypotheses<true>, d_pts3d,
                            d_pts2d, cap, (const int32_t *)nullptr, cam, (uint64_t)ctx->prm.pnp_seed, H, poses, valid, jb)); }
  ctx->launches++;
  // the job's points in shared memory (20 bytes each); with the kernel's 32 B of static shared memory above the 48 KB default
  // from cap = 2457 on
  const size_t smem = (size_t)cap * 5 * sizeof(float);
  if (smem + 8 * sizeof(float) > 48 * 1024)
    MVO_CUDA(ctx, cudaFuncSetAttribute(k_pnp_score<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  { KTimer kt(ctx, KC_PNP_SCORE);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, dim3((unsigned)pnp_batch_score_grid(ctx, n_jobs, H), (unsigned)n_jobs), dim3(256), smem,
                            k_pnp_score<true>, d_pts3d, d_pts2d, cap, (const int32_t *)job_n, cam, thr2, H, (const double *)poses,
                            (const int32_t *)valid, counts)); }
  ctx->launches++;
  { KTimer kt(ctx, KC_PNP_FINISH);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, (unsigned)n_jobs, FIN_T, 0, 0, k_pnp_finish<true>, d_pts3d, d_pts2d, cap, (const int32_t *)job_n, cam,
                           thr2, H, (const double *)poses, (const int32_t *)counts, 0, (int)ctx->prm.pnp_refine_iters, pose_io, out_i,
                           d_inliers, ex, eo, ef)); }
  ctx->launches++;
  // one cluster per job with E = cap: each refit sums in the order of a single device call on n_upper = cap pairs
  static const double I2[4] = {1, 0, 0, 1};
  MVO_TRY(mvo_ba_pose_launch(ctx, 1, cap, 1, ef, ex, eo, cam.fx, cam.fy, cam.cx, cam.cy, I2, ctx->prm.pnp_refine_iters, 0, 1.0, 0, 1e-8,
                             pose_io, stats, n_jobs));
  MVO_CUDA(ctx, launch_pdl(ctx->stream, (unsigned)n_jobs, 128, 0, 0, k_pnp_batch_tail, d_mm, d_matches, cap, d_T_w_c_prev,
                           tp->max_dist_to_prev, (const int32_t *)job_st, (const double *)pose_io, (const int32_t *)out_i,
                           (const int32_t *)d_inliers, d_out, d_kept));
  ctx->launches++;
  return MVO_OK;
}

int mvo_solve_pnp_ransac(mvo_ctx *ctx, const float *pts3d, const float *pts2d, int n, const double *K,
                         double *rvec, double *tvec, int32_t *inliers, int *n_inliers) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!pts3d || !pts2d || !rvec || !tvec || !n_inliers || (*n_inliers > 0 && !inliers))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "solvePnPRansac: null pointer");
  if (n < 4) return mvo_fail(ctx, MVO_ERR_DEGENERATE, "solvePnPRansac: %d correspondences (< 4)", n);
  PnpCam cam;
  MVO_TRY(pnp_cam(ctx, K, &cam));
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int H = pnp_hyp_count(ctx);
  PnpWs w;
  MVO_TRY(pnp_ws(ctx, n, H, &w));
  if ((size_t)n * 20 > 200 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "solvePnPRansac: more than %d correspondences", 200 * 1024 / 20);
  const size_t hb = (size_t)n * 20 + (size_t)n * 4 + 1024;
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_b, hb));
  float *h3 = (float *)ctx->h_b.p, *h2 = h3 + (size_t)n * 3;
  memcpy(h3, pts3d, (size_t)n * 12);
  memcpy(h2, pts2d, (size_t)n * 8);
  MVO_CUDA(ctx, cudaMemcpyAsync(w.p3, h3, (size_t)n * 12, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(w.p2, h2, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_TRY(pnp_enqueue(ctx, w, n, cam));
  uint8_t *hout = (uint8_t *)ctx->h_b.p + (size_t)n * 20;
  double *h_pose = (double *)hout;
  int32_t *h_i = (int32_t *)(hout + 128), *h_inl = (int32_t *)(hout + 256);
  MVO_CUDA(ctx, cudaMemcpyAsync(h_pose, w.pose_io, 96, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(h_i, w.out_i, 16, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(h_inl, w.inl, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const int ni = h_i[0];
  if (ni < 4) { *n_inliers = 0; return mvo_fail(ctx, MVO_ERR_DEGENERATE, "solvePnPRansac: no hypothesis reached 4 inliers"); }
  if (ni > *n_inliers) return mvo_fail(ctx, MVO_ERR_CAPACITY, "inlier capacity %d < %d", *n_inliers, ni);
  rotation_to_rvec(h_pose, rvec);
  tvec[0] = h_pose[9]; tvec[1] = h_pose[10]; tvec[2] = h_pose[11];
  memcpy(inliers, h_inl, (size_t)ni * 4);
  *n_inliers = ni;
  return MVO_OK;
}

int mvo_pnp_last_hypotheses(mvo_ctx *ctx, double *poses, int32_t *counts, int cap, int *n_hyp) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!poses || !counts || !n_hyp) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "null pointer");
  const int H = ctx->pnp_last_h;
  if (H <= 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "no PnP call yet");
  if (cap < H) return mvo_fail(ctx, MVO_ERR_CAPACITY, "capacity %d < %d", cap, H);
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int32_t *d_counts = (int32_t *)ctx->pnp_cnt.p + ((H + 63) & ~63);
  MVO_CUDA(ctx, cudaMemcpyAsync(poses, ctx->pnp_hyp.p, (size_t)H * 96, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(counts, d_counts, (size_t)H * 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *n_hyp = H;
  return MVO_OK;
}

int mvo_pnp_refine(mvo_ctx *ctx, const float *pts3d, const float *pts2d, int n, const double *K, double *rvec,
                   double *tvec) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!pts3d || !pts2d || !rvec || !tvec) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp_refine: null pointer");
  if (n < 3) return mvo_fail(ctx, MVO_ERR_DEGENERATE, "pnp_refine: %d correspondences (< 3)", n);
  PnpCam cam;
  MVO_TRY(pnp_cam(ctx, K, &cam));
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  PnpWs w;
  MVO_TRY(pnp_ws(ctx, n, pnp_hyp_count(ctx), &w));
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_b, (size_t)n * 20 + 1024));
  float *h3 = (float *)ctx->h_b.p, *h2 = h3 + (size_t)n * 3;
  double *h_pose = (double *)((uint8_t *)ctx->h_b.p + (size_t)n * 20);
  memcpy(h3, pts3d, (size_t)n * 12);
  memcpy(h2, pts2d, (size_t)n * 8);
  rvec_to_rotation(rvec, h_pose);
  h_pose[9] = tvec[0]; h_pose[10] = tvec[1]; h_pose[11] = tvec[2];
  MVO_CUDA(ctx, cudaMemcpyAsync(w.p3, h3, (size_t)n * 12, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(w.p2, h2, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(w.pose_io, h_pose, 96, cudaMemcpyHostToDevice, ctx->stream));
  { KTimer kt(ctx, KC_PNP_FINISH);
  k_pnp_finish<false><<<1, FIN_T, 0, ctx->stream>>>(w.p3, w.p2, n, nullptr, cam, 0.0, 0, nullptr, nullptr, 1, ctx->prm.pnp_refine_iters,
                                             w.pose_io, w.out_i, w.inl, w.ex, w.eo, w.ef); }
  MVO_CHECK_LAUNCH(ctx);
  MVO_TRY(pnp_refit(ctx, w, n, cam));
  MVO_CUDA(ctx, cudaMemcpyAsync(h_pose, w.pose_io, 96, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  rotation_to_rvec(h_pose, rvec);
  tvec[0] = h_pose[9]; tvec[1] = h_pose[10]; tvec[2] = h_pose[11];
  return MVO_OK;
}

}  // extern "C"
