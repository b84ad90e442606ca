// The combine step of mvo_estimate_relative_poses_batch_dev (mvo.h): what mvo_estimate_relative_poses (two_view.cpp) does on the
// host once its two RANSACs have returned, for every pair of a batch in one launch, one CTA per pair:
//   cv::decomposeHomographyMat(H, K) + t /= |t|      epipolar.cu mvo_epi_homography_end (reference epipolar_geometry.cpp:119-126)
//   removeWrongRtOfHomography                        epi::filter_homography_solutions (epipolar_geometry.cpp:59-88)
//   the solutions, their inlier rows, basics::invRt  two_view.cpp (motion_estimation.cpp:75-118)
//   checkEssentialScore / checkHomographyScore       eh_scores.cuh, sigma = 1 (motion_estimation.cpp:501-664)
//   the E / H choice                                 epi::eh_choose with mvo_params::eh_ratio_threshold (:134-154)
// The host path runs all of this in g++ code for x86-64, which has no fused multiply-add.  This translation unit is compiled
// with --fmad=false (Makefile), so every product and sum here rounds as on the host and the batch returns the host's bits; the
// RANSAC kernels (epipolar.cu) keep their contraction, the host path runs those same kernels.
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "eh_scores.cuh"
#include "mvo_internal.h"

namespace {

constexpr int RPC_T = 256;

struct RpcSmem {
  mvo_two_view_solutions sol;            // the pair's record, zeroed first as the host memsets its struct
  double Rh[36], th[12], nh[12], F[9], H12[9];
  int ns, num_h, h_inv, keep[4];
};
constexpr size_t RPC_TERMS_OFFSET = (sizeof(RpcSmem) + 15) & ~(size_t)15;

// the two score terms of point k of a list; the sum stays sequential (one thread, list order) because the host's is.  A term that
// fails its test is +0.0: added to a sum of non-negative terms that started at +0.0, it leaves the sum's bits unchanged.
__device__ __forceinline__ double sum_terms(const double *terms, int n_terms) {
  double score = 0;
  for (int k = 0; k < n_terms; ++k) score += terms[k];
  return score;
}

__global__ void __launch_bounds__(RPC_T) k_relative_poses_combine(const MvoRelPosesCombine a) {
  extern __shared__ double smraw[];
  RpcSmem &S = *reinterpret_cast<RpcSmem *>(smraw);
  double *terms = reinterpret_cast<double *>(reinterpret_cast<uint8_t *>(smraw) + RPC_TERMS_OFFSET);      // [cap][2]
  const int pair = blockIdx.x, tid = threadIdx.x;
  const mvo_two_view_result &er = a.ess[pair];
  mvo_relative_poses_result &out = a.res[pair];
  const int status = er.status;                    // k_epi_pick wrote every pair's status: input faults, n < 8, no essential model
  if (tid == 0) { out.status = status; out.n_matches = a.n_matches[pair]; }
  if (status != MVO_OK) return;                    // the whole CTA
  const size_t op = (size_t)pair * a.cap;
  const float *p1 = a.p1 + op * 2, *p2 = a.p2 + op * 2, *np1 = a.np1 + op * 2, *np2 = a.np2 + op * 2;
  const int32_t *inl_e = a.inl_e + op, *inl_h = a.inl_h + op;
  const double *hd = a.hom_d + (size_t)pair * a.hom_d_stride;
  const int n_e = er.n_inliers, hi0 = a.hom_i[(size_t)pair * a.hom_i_stride];
  const int n_h = hi0 >= 4 ? hi0 : 0;              // fewer than 4 homography inliers: MVO_ERR_DEGENERATE there, num_h = 0 (two_view.cpp:50)
  {
    unsigned long long *w = reinterpret_cast<unsigned long long *>(&S.sol);
    for (int q = tid; q < (int)(sizeof S.sol / 8); q += RPC_T) w[q] = 0;
  }
  __syncthreads();
  if (tid == 0) {
    mvo_two_view_solutions &sol = S.sol;
    for (int q = 0; q < 9; ++q) { sol.E[q] = er.E[q]; sol.R[0][q] = er.R[q]; }
    for (int q = 0; q < 3; ++q) sol.t[0][q] = er.t[q];
    S.ns = 0;
    if (n_h > 0) {
      // mvo_epi_homography_end: Hn = K^-1 H K, decomposition, t /= |t| (a pure rotation keeps t = 0)
      for (int q = 0; q < 9; ++q) sol.H[q] = hd[q];
      const double fx = a.K[0], fy = a.K[4], cx = a.K[2], cy = a.K[5];
      const double Km[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1}, Ki[9] = {1 / fx, 0, -cx / fx, 0, 1 / fy, -cy / fy, 0, 0, 1};
      double T[9], Hn[9];
      epi::mat3_mul(sol.H, Km, T);
      epi::mat3_mul(Ki, T, Hn);
      const int ns = epi::decompose_homography(Hn, S.Rh, S.th, S.nh);
      for (int s = 0; s < ns; ++s) {
        double *ts = S.th + 3 * s;
        const double nt = sqrt(ts[0] * ts[0] + ts[1] * ts[1] + ts[2] * ts[2]);
        if (nt > 0) for (int q = 0; q < 3; ++q) ts[q] /= nt;
      }
      S.ns = ns;
    }
    for (int s = 0; s < 4; ++s) S.keep[s] = 1;
  }
  __syncthreads();
  // ---- removeWrongRtOfHomography: a solution survives when every inlier passes; each thread tests a contiguous chunk of the list
  // with the host's function, the chunks' verdicts are ANDed ----
  const int ns = S.ns;
  if (ns > 0) {
    const int per = (n_h + RPC_T - 1) / RPC_T, b0 = min(tid * per, n_h), e0 = min(b0 + per, n_h);
    int keep[4] = {1, 1, 1, 1};
    static_assert(sizeof(int) == sizeof(int32_t), "int32 indices");
    if (e0 > b0) epi::filter_homography_solutions(S.Rh, S.nh, ns, np1, np2, (const int *)inl_h + b0, e0 - b0, keep);
    for (int s = 0; s < ns; ++s) if (!keep[s]) atomicAnd(&S.keep[s], 0);
  }
  __syncthreads();
  if (tid == 0) {
    mvo_two_view_solutions &sol = S.sol;
    int num_h = 0;                                 // survivors, in order
    for (int s = 0; s < ns; ++s)
      if (S.keep[s]) {
        for (int q = 0; q < 9; ++q) sol.R[1 + num_h][q] = S.Rh[9 * s + q];
        for (int q = 0; q < 3; ++q) { sol.t[1 + num_h][q] = S.th[3 * s + q]; sol.normal[1 + num_h][q] = S.nh[3 * s + q]; }
        sol.n_inliers[1 + num_h] = n_h;
        ++num_h;
      }
    sol.num_solutions = 1 + num_h;
    sol.n_inliers[0] = n_e;
    S.num_h = num_h;
    // the triangulation (k_triangulate_solutions_batch) uses (R, t) as they are before the change of frame
    double *rt = a.rt + (size_t)pair * 5 * 12;
    for (int s = 0; s < sol.num_solutions; ++s) {
      for (int q = 0; q < 9; ++q) rt[12 * s + q] = sol.R[s][q];
      for (int q = 0; q < 3; ++q) rt[12 * s + 9 + q] = sol.t[s][q];
    }
    if (!a.motion_cam2_to_cam1)                    // basics::invRt, after everything else (:114-118)
      for (int s = 0; s < sol.num_solutions; ++s) {
        double Rt[9], tt[3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = sol.R[s][j * 3 + i];
        for (int i = 0; i < 3; ++i) tt[i] = -(Rt[i * 3] * sol.t[s][0] + Rt[i * 3 + 1] * sol.t[s][1] + Rt[i * 3 + 2] * sol.t[s][2]);
        for (int q = 0; q < 9; ++q) sol.R[s][q] = Rt[q];
        for (int q = 0; q < 3; ++q) sol.t[s][q] = tt[q];
      }
    double Ki[9];
    epi::inv3(a.K, Ki);                            // the call checked that K inverts
    epi::essential_score_F(sol.E, Ki, S.F);
    S.h_inv = n_h > 0 && epi::inv3(sol.H, S.H12);  // a singular H cannot be inverted for the symmetric transfer error: score_h = 0
  }
  __syncthreads();
  // ---- inlier rows: 0 the essential list, 1..num_h the homography list ----
  const int num_h = S.num_h;
  int32_t *rows = a.inliers + (size_t)pair * 5 * a.cap;
  for (int k = tid; k < n_e; k += RPC_T) rows[k] = inl_e[k];
  for (int s = 1; s <= num_h; ++s)
    for (int k = tid; k < n_h; k += RPC_T) rows[(size_t)s * a.cap + k] = inl_h[k];
  // ---- checkEssentialScore over the essential inliers ----
  for (int k = tid; k < n_e; k += RPC_T) {
    const int i = inl_e[k];
    double chi1, chi2;
    epi::essential_score_chi(S.F, p1[2 * i], p1[2 * i + 1], p2[2 * i], p2[2 * i + 1], 1.0, &chi1, &chi2);
    terms[2 * k] = chi1 > epi::EH_ESSENTIAL_TH ? 0.0 : epi::EH_ESSENTIAL_TH_SCORE - chi1;
    terms[2 * k + 1] = chi2 > epi::EH_ESSENTIAL_TH ? 0.0 : epi::EH_ESSENTIAL_TH_SCORE - chi2;
  }
  __syncthreads();
  if (tid == 0) S.sol.score_e = sum_terms(terms, 2 * n_e);
  __syncthreads();
  // ---- checkHomographyScore over the homography inliers ----
  if (S.h_inv) {
    for (int k = tid; k < n_h; k += RPC_T) {
      const int i = inl_h[k];
      double chi1, chi2;
      epi::homography_score_chi(S.sol.H, S.H12, p1[2 * i], p1[2 * i + 1], p2[2 * i], p2[2 * i + 1], 1.0, &chi1, &chi2);
      terms[2 * k] = chi1 > epi::EH_HOMOGRAPHY_TH ? 0.0 : epi::EH_HOMOGRAPHY_TH - chi1;
      terms[2 * k + 1] = chi2 > epi::EH_HOMOGRAPHY_TH ? 0.0 : epi::EH_HOMOGRAPHY_TH - chi2;
    }
    __syncthreads();
    if (tid == 0) S.sol.score_h = sum_terms(terms, 2 * n_h);
  }
  if (tid == 0) {
    mvo_two_view_solutions &sol = S.sol;
    int best = 0;
    const double ratio = epi::eh_choose(sol.score_e, sol.score_h, &sol.normal[1][0], num_h, a.eh_ratio_threshold, &best);
    sol.best = best;
    sol.ratio = as_host_nan(ratio);
    sol.score_e = as_host_nan(sol.score_e);
    sol.score_h = as_host_nan(sol.score_h);
  }
  __syncthreads();
  {
    const unsigned long long *src = reinterpret_cast<const unsigned long long *>(&S.sol);
    unsigned long long *dst = reinterpret_cast<unsigned long long *>(&out.sol);
    for (int q = tid; q < (int)(sizeof S.sol / 8); q += RPC_T) dst[q] = src[q];
  }
}

}  // namespace

// declared in epipolar.cu, which launches the batch call
int mvo_relative_poses_combine(mvo_ctx *ctx, const MvoRelPosesCombine &a) {
  static_assert(sizeof(mvo_two_view_solutions) % 8 == 0 && offsetof(mvo_relative_poses_result, sol) == 8, "8-byte words");
  const size_t smem = RPC_TERMS_OFFSET + (size_t)a.cap * 2 * sizeof(double);
  if (smem > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_relative_poses_combine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  { KTimer kt(ctx, KC_EPI);
  k_relative_poses_combine<<<a.n_pairs, RPC_T, smem, ctx->stream>>>(a); }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}
