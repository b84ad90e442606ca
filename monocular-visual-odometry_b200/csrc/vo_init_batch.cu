// mvo_vo_init_candidates_batch_dev (mvo.h): what the state machine (vo_pipeline.cpp) does with one candidate frame of the
// initialisation once its two-view step has returned, for every pair of a batch in one launch, one CTA per pair:
//   estimateMotionAnd3DPoints_   estimate_motion_and_3d_points (reference vo.cpp:53-111)
//   retainGoodTriangulationResult_   mvo_retain_good_triangulation (vo_host.cpp; vo.cpp:181-244)
//   the depth normalisation      mvo_normalize_init_depth (vo.cpp:96-110)
//   isVoGoodToInit_              mvo_is_vo_good_to_init (vo.cpp:113-172)
// The host path is g++ code for x86-64, which has no fused multiply-add.  This translation unit is compiled with --fmad=false
// (Makefile), and the per-point numerics are the host's own functions (vo_init_math.cuh, inv_rigid / rt_to_T of mvo_internal.h),
// so every product and sum rounds as on the host.  The per-point terms run in parallel; every sum over points runs on one
// thread in list order, as on the host.  The medians: without a NaN angle any exact selection gives the host's value, here a
// radix select over the order-preserving bit patterns; with one, the value depends on the algorithm, and one thread runs the
// restatement of std::nth_element (retainGoodTriangulationResult_) or std::sort (isVoGoodToInit_).
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "mvo_internal.h"
#include "vo_init_math.cuh"

namespace {

constexpr int VIB_T = 256;

struct VibSmem {
  mvo_init_candidate_result rec;
  double Tref[16], Tc[16], R[9], t[3], med;     // Tref: a copy, so that no pointer into the kernel parameters is taken
  unsigned hist[256];
  int sort_stack[3 * voi::SORT_STACK];
  unsigned long long prefix;
  int rank, bad, nan, n_kept, warp_sum[VIB_T / 32];
};

// doubles -> unsigned keys in the same order (NaN excluded)
__device__ __forceinline__ unsigned long long order_key(double v) {
  unsigned long long b;
  memcpy(&b, &v, sizeof b);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double from_order_key(unsigned long long k) {
  const unsigned long long b = (k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
  double v;
  memcpy(&v, &b, sizeof v);
  return v;
}

// the element of rank k of v[0, n) (no NaN): eight passes of an 8-bit histogram over the keys that share the prefix so far
__device__ double radix_select(const double *v, int n, int k, VibSmem &S) {
  const int tid = threadIdx.x;
  unsigned long long prefix = 0, mask = 0;
  if (tid == 0) S.rank = k;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int b = tid; b < 256; b += VIB_T) S.hist[b] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += VIB_T) {
      const unsigned long long key = order_key(v[i]);
      if ((key & mask) == prefix) atomicAdd(&S.hist[(key >> shift) & 255], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      int acc = 0, b = 0;
      for (; b < 255; ++b) {
        if (acc + (int)S.hist[b] > S.rank) break;
        acc += (int)S.hist[b];
      }
      S.rank -= acc;
      S.prefix = prefix | ((unsigned long long)b << shift);
    }
    __syncthreads();
    prefix = S.prefix;
    mask |= 0xFFull << shift;
    __syncthreads();                               // S.prefix is rewritten in the next pass
  }
  return from_order_key(prefix);
}

// T_w_c = T_w_c_ref * [R|t]^-1 (vo.cpp:91, :110); one thread, a call of its own so that its 4x4 temporaries stay out of the
// kernel's registers
__device__ __attribute__((noinline)) void candidate_pose(const double *R, const double *t, const double *T_ref, double *T_w_c) {
  double Trt[16], Tinv[16];
  rt_to_T(R, t, Trt);
  inv_rigid(Trt, Tinv);
  voi::mul44(T_ref, Tinv, T_w_c);
}

__global__ void __launch_bounds__(VIB_T, 2) k_vo_init_candidates(const MvoInitCandidates a) {
  extern __shared__ double vib_dyn[];
  __shared__ VibSmem S;
  double *ang = vib_dyn;                                              // [cap] angles, then the kept angles, then the pixel terms
  float *pts = reinterpret_cast<float *>(vib_dyn + a.cap);            // [cap][3] points in the candidate's camera
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const mvo_relative_poses_result &rp = a.rp[pair];
  mvo_init_candidate_result &out = a.out[pair];
  const int status = rp.status;
  if (status != MVO_OK && status != MVO_ERR_DEGENERATE) { if (tid == 0) out.status = status; return; }
  if (tid == 0) {
    memset(&S.rec, 0, sizeof S.rec);
    S.rec.best_sol = -1;
    for (int q = 0; q < 16; ++q) S.rec.T_w_c[q] = S.Tref[q] = a.T_ref[q];
    S.bad = 0; S.nan = 0; S.n_kept = 0;
  }
  // ---- per-pair checks, each before anything is read through the value it checks ----
  const int2 fr = reinterpret_cast<const int2 *>(a.pairs)[pair];
  const int nm = a.n_matches[pair];
  const int ns = rp.sol.num_solutions, best = rp.sol.best;
  bool bad = status == MVO_OK && (fr.x < 0 || fr.x >= a.batch || fr.y < 0 || fr.y >= a.batch || nm < 0 || nm > a.cap || ns < 1 || ns > 5 ||
                                  best < 0 || best >= ns);
  const int ni = status == MVO_OK && !bad ? rp.sol.n_inliers[best] : 0;
  bad = bad || ni < 0 || ni > nm;
  if (bad) { if (tid == 0) out.status = MVO_ERR_INVALID_ARG; return; }
  const size_t row = (size_t)pair * a.cap;
  const int32_t *inl = a.rp_inliers + ((size_t)pair * 5 + (status == MVO_OK ? best : 0)) * a.cap;
  const mvo_dmatch *matches = a.matches + row;
  const mvo_keypoint *kq = a.kpts + (size_t)(status == MVO_OK ? fr.x : 0) * a.cap, *kt = a.kpts + (size_t)(status == MVO_OK ? fr.y : 0) * a.cap;
  __syncthreads();
  if (status == MVO_OK) {
    const int cq = min(max(a.counts[fr.x], 0), a.cap), ct = min(max(a.counts[fr.y], 0), a.cap);
    for (int k = tid; k < ni; k += VIB_T) {
      const int i = inl[k];
      if (i < 0 || i >= nm) { atomicOr(&S.bad, 1); continue; }
      const mvo_dmatch m = matches[i];
      if (m.query_idx < 0 || m.query_idx >= cq || m.train_idx < 0 || m.train_idx >= ct) atomicOr(&S.bad, 1);
    }
  }
  __syncthreads();
  if (S.bad) { if (tid == 0) out.status = MVO_ERR_INVALID_ARG; return; }
  if (status != MVO_OK) {                                             // MVO_ERR_DEGENERATE: the frame keeps the reference's pose
    const unsigned long long *src = reinterpret_cast<const unsigned long long *>(&S.rec);
    unsigned long long *dst = reinterpret_cast<unsigned long long *>(&out);
    for (int q = tid; q < (int)(sizeof S.rec / 8); q += VIB_T) dst[q] = src[q];
    return;
  }
  // ---- the chosen solution, T_w_c = T_w_c_ref * [R|t]^-1 (vo.cpp:76-91) ----
  if (tid == 0) {
    for (int q = 0; q < 9; ++q) S.R[q] = rp.sol.R[best][q];
    for (int q = 0; q < 3; ++q) S.t[q] = rp.sol.t[best][q];
    candidate_pose(S.R, S.t, S.Tref, S.Tc);
  }
  __syncthreads();
  // ---- points in the candidate's camera (transCoord) and their triangulation angles ----
  const float *p3 = a.rp_pts3d + ((size_t)pair * 5 + best) * a.cap * 3;
  for (int k = tid; k < ni; k += VIB_T) {
    float p[3] = {p3[3 * k], p3[3 * k + 1], p3[3 * k + 2]};
    voi::trans_coord(p, S.R, S.t, pts + 3 * k);
    const double an = voi::triangulation_angle(pts + 3 * k, S.Tc, S.Tref);
    ang[k] = an;
    if (an != an) atomicOr(&S.nan, 1);
  }
  __syncthreads();
  const bool has_nan = S.nan != 0;
  double *kept_ang = a.kept_angles + row;
  if (ni > 0) {                                                       // n = 0 returns before the median (vo.cpp:203-205)
    // ---- the median at n / 2: std::nth_element on the host ----
    double med;
    if (has_nan) {
      // the restatement on a copy of the angles in the point rows (12 B per row hold the 8 B of an angle); the points are
      // computed again afterwards, from the same inputs, so they are the same bits
      double *work = reinterpret_cast<double *>(pts);
      if (tid == 0) {
        for (int k = 0; k < ni; ++k) work[k] = ang[k];
        voi::nth_element_d(work, ni / 2, ni);
        S.med = work[ni / 2];
      }
      __syncthreads();
      med = S.med;
      for (int k = tid; k < ni; k += VIB_T) {
        float p[3] = {p3[3 * k], p3[3 * k + 1], p3[3 * k + 2]};
        voi::trans_coord(p, S.R, S.t, pts + 3 * k);
      }
      __syncthreads();
    } else {
      med = radix_select(ang, ni, ni / 2, S);
    }
    // ---- keep decision (:236-244) and compaction in list order, 256 points at a time ----
    for (int c = 0; c < ni; c += VIB_T) {
      const int k = c + tid;
      bool keep = false;
      double an = 0;
      float q0 = 0, q1 = 0, q2 = 0;
      if (k < ni) {
        an = ang[k];
        keep = !(an < a.min_triang_angle || an / med > a.max_ratio_angle_to_median);
        q0 = pts[3 * k]; q1 = pts[3 * k + 1]; q2 = pts[3 * k + 2];
      }
      const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
      if (lane == 0) S.warp_sum[warp] = __popc(bal);
      __syncthreads();                                                // every read of this chunk is done before any write
      int pos = S.n_kept + __popc(bal & ((1u << lane) - 1u));
      for (int w = 0; w < warp; ++w) pos += S.warp_sum[w];
      if (keep) {
        ang[pos] = an;
        pts[3 * pos] = q0; pts[3 * pos + 1] = q1; pts[3 * pos + 2] = q2;
        mvo_dmatch m = matches[inl[k]];
        m.img_idx = -1;                                               // cv::DMatch(queryIdx, trainIdx, distance)
        a.kept[row + pos] = m;
        kept_ang[pos] = as_host_nan(an);
      }
      __syncthreads();
      if (tid == 0) for (int w = 0; w < VIB_T / 32; ++w) S.n_kept += S.warp_sum[w];
      __syncthreads();
    }
  }
  const int nk = S.n_kept;
  // ---- depth normalisation (vo.cpp:96-110): mean depth summed in list order, then the points, t and the pose ----
  if (tid == 0) {
    S.rec.usable = 1;
    S.rec.best_sol = best;
    S.rec.n_inliers = ni;
    S.rec.n_kept = nk;
    if (nk >= 20) {
      double mean_depth = 0;
      for (int i = 0; i < nk; ++i) mean_depth += pts[3 * i + 2];
      mean_depth /= nk;
      const double scale = a.assumed_mean_depth_init / mean_depth;
      for (int q = 0; q < 3; ++q) S.t[q] *= scale;
      candidate_pose(S.R, S.t, S.Tref, S.Tc);
      S.rec.normalized = 1;
      S.rec.scale = as_host_nan(scale);
    }
    for (int q = 0; q < 3; ++q) S.rec.t_curr_to_prev[q] = S.t[q];
    for (int q = 0; q < 16; ++q) S.rec.T_w_c[q] = S.Tc[q];
  }
  __syncthreads();
  float *kept_pts = a.kept_pts3d + row * 3;
  if (nk >= 20) {
    const double scale = S.rec.scale;
    for (int i = tid; i < 3 * nk; i += VIB_T) kept_pts[i] = (float)(pts[i] * scale);      // float *= double (basics::scalePointPos)
  } else {
    for (int i = tid; i < 3 * nk; i += VIB_T) kept_pts[i] = pts[i];
  }
  // ---- isVoGoodToInit_: the median of the kept angles (std::sort, element n / 2) ----
  double med2 = 0;
  if (nk > 0) {
    if (has_nan) {
      if (tid == 0) { voi::sort_d(ang, nk, S.sort_stack); S.med = ang[nk / 2]; }
      __syncthreads();
      med2 = S.med;
    } else {
      med2 = radix_select(ang, nk, nk / 2, S);
    }
  }
  __syncthreads();                                                    // ang is reused for the pixel distances
  // ---- mean pixel displacement over the kept matches (computeMeanDistBetweenKeypoints), summed in list order ----
  for (int i = tid; i < nk; i += VIB_T) {
    const mvo_dmatch m = a.kept[row + i];
    ang[i] = voi::pixel_dist(kq[m.query_idx].x, kq[m.query_idx].y, kt[m.train_idx].x, kt[m.train_idx].y);
  }
  __syncthreads();
  if (tid == 0) {
    double mean_dist = 0;
    for (int i = 0; i < nk; ++i) mean_dist += ang[i];
    mean_dist /= nk;                                                  // 0 / 0 for no match, as on the host
    const bool criteria_0 = nk >= a.min_inlier_matches, criteria_1 = mean_dist > a.min_pixel_dist;
    const bool criteria_2 = nk > 0 && med2 > a.min_median_triangulation_angle;
    S.rec.good = criteria_0 && criteria_1 && criteria_2;
    S.rec.mean_pixel_dist = as_host_nan(mean_dist);
    S.rec.median_angle = as_host_nan(med2);
  }
  __syncthreads();
  const unsigned long long *src = reinterpret_cast<const unsigned long long *>(&S.rec);
  unsigned long long *dst = reinterpret_cast<unsigned long long *>(&out);
  for (int q = tid; q < (int)(sizeof S.rec / 8); q += VIB_T) dst[q] = src[q];
}

}  // namespace

// declared in mvo_internal.h; mvo_vo_init_candidates_batch_dev (vo_pipeline.cpp) checks the arguments and calls it
int mvo_vo_init_candidates_launch(mvo_ctx *ctx, const MvoInitCandidates &a) {
  static_assert(sizeof(mvo_init_candidate_result) == 208 && sizeof(mvo_init_candidate_result) % 8 == 0, "8-byte words");
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t smem = (size_t)a.cap * (sizeof(double) + 3 * sizeof(float));
  // the 48 KB a launch gets without opting in cover the static shared memory (VibSmem) and the dynamic part together
  if (smem + sizeof(VibSmem) > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_vo_init_candidates, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  { KTimer kt(ctx, KC_EPI);
  k_vo_init_candidates<<<a.n_pairs, VIB_T, smem, ctx->stream>>>(a); }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}
