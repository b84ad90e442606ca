// Two batch calls of the state machine's (vo_pipeline.cpp) host logic after a two-view step, for every pair of a batch, one CTA
// per pair:
//   mvo_vo_init_candidates_batch_dev (mvo.h): what the state machine does with one candidate frame of the initialisation once its
//   two-view step has returned, in one launch:
//     estimateMotionAnd3DPoints_   estimate_motion_and_3d_points (reference vo.cpp:53-111)
//     retainGoodTriangulationResult_   mvo_retain_good_triangulation (vo_host.cpp; vo.cpp:181-244)
//     the depth normalisation      mvo_normalize_init_depth (vo.cpp:96-110)
//     isVoGoodToInit_              mvo_is_vo_good_to_init (vo.cpp:113-172)
//   mvo_vo_keyframe_points_batch_dev (mvo.h): the new map points of the keyframe branch (insert_keyframe), in three launches:
//     k_kf_motion                  the per-pair checks and the known motion T_w_c_curr^-1 * T_w_c_ref (vo_commons.cpp:9-15)
//     mvo_kf_triangulate_launch    doTriangulation with that motion (epipolar.cu: the device's own triangulation arithmetic)
//     k_kf_points                  transCoord, retainGoodTriangulationResult_, and the position / direction of each new map point
//                                  (pushCurrPointsToMap_, vo.cpp:528-576)
// The host path is g++ code for x86-64, which has no fused multiply-add.  This translation unit is compiled with --fmad=false
// (Makefile), and the per-point numerics are the host's own functions (vo_init_math.cuh, inv_rigid / rt_to_T / pre_translate of
// mvo_internal.h), so every product and sum rounds as on the host.  The per-point terms run in parallel; every sum over points
// runs on one thread in list order, as on the host.  The medians: without a NaN angle any exact selection gives the host's value,
// here a radix select over the order-preserving bit patterns; with one, the value depends on the algorithm, and one thread runs
// the restatement of std::nth_element (retainGoodTriangulationResult_) or std::sort (isVoGoodToInit_).
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "mvo_internal.h"
#include "vo_init_math.cuh"

namespace {

constexpr int VIB_T = 256;

// what the retain step (retain_good_triangulation below) keeps in static shared memory
struct RetainSmem {
  double R[9], t[3], Tc[16], Tref[16], med;     // the motion and both poses the points and angles are computed with
  unsigned hist[256];
  unsigned long long prefix;
  int rank, nan, n_kept, warp_sum[VIB_T / 32];
};

struct VibSmem {
  mvo_init_candidate_result rec;
  RetainSmem r;
  int sort_stack[3 * voi::SORT_STACK];
  int bad;
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
__device__ double radix_select(const double *v, int n, int k, RetainSmem &S) {
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

// retainGoodTriangulationResult_ (vo.cpp:181-244) over the n inliers of one pair, by the whole CTA.  Point k is p3[k] (the
// triangulation, camera 1) moved into the current camera with S.R, S.t (transCoord); its angle is taken between the camera
// centres of S.Tc (current) and S.Tref.  Every point is staged in pts / ang (shared, cap rows) before anything is written, so p3
// may be the row that the caller overwrites afterwards.  The kept matches (img_idx = -1) and angles go to kept / kept_ang in list
// order; the kept points and angles end up compacted at the front of pts / ang.  Returns the median (element n / 2 of
// std::nth_element; 0 when n = 0); S.n_kept holds the count and S.nan whether an angle was NaN.
__device__ double retain_good_triangulation(const float *p3, int n, const int32_t *inl, const mvo_dmatch *matches, double min_angle,
                                            double max_ratio, double *ang, float *pts, mvo_dmatch *kept, double *kept_ang,
                                            RetainSmem &S) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { S.nan = 0; S.n_kept = 0; }
  __syncthreads();
  // ---- points in the current camera (transCoord) and their triangulation angles ----
  for (int k = tid; k < n; k += VIB_T) {
    float p[3] = {p3[3 * k], p3[3 * k + 1], p3[3 * k + 2]};
    voi::trans_coord(p, S.R, S.t, pts + 3 * k);
    const double an = voi::triangulation_angle(pts + 3 * k, S.Tc, S.Tref);
    ang[k] = an;
    if (an != an) atomicOr(&S.nan, 1);
  }
  __syncthreads();
  if (n == 0) return 0;                                               // no median (vo.cpp:203-205)
  // ---- the median at n / 2: std::nth_element on the host ----
  double med;
  if (S.nan) {
    // the restatement on a copy of the angles in the point rows (12 B per row hold the 8 B of an angle); the points are
    // computed again afterwards, from the same inputs, so they are the same bits
    double *work = reinterpret_cast<double *>(pts);
    if (tid == 0) {
      for (int k = 0; k < n; ++k) work[k] = ang[k];
      voi::nth_element_d(work, n / 2, n);
      S.med = work[n / 2];
    }
    __syncthreads();
    med = S.med;
    for (int k = tid; k < n; k += VIB_T) {
      float p[3] = {p3[3 * k], p3[3 * k + 1], p3[3 * k + 2]};
      voi::trans_coord(p, S.R, S.t, pts + 3 * k);
    }
    __syncthreads();
  } else {
    med = radix_select(ang, n, n / 2, S);
  }
  // ---- keep decision (:236-244) and compaction in list order, 256 points at a time ----
  for (int c = 0; c < n; c += VIB_T) {
    const int k = c + tid;
    bool keep = false;
    double an = 0;
    float q0 = 0, q1 = 0, q2 = 0;
    if (k < n) {
      an = ang[k];
      keep = !(an < min_angle || an / med > max_ratio);
      q0 = pts[3 * k]; q1 = pts[3 * k + 1]; q2 = pts[3 * k + 2];
    }
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
    if (lane == 0) S.warp_sum[warp] = __popc(bal);
    __syncthreads();                                                  // every read of this chunk is done before any write
    int pos = S.n_kept + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) pos += S.warp_sum[w];
    if (keep) {
      ang[pos] = an;
      pts[3 * pos] = q0; pts[3 * pos + 1] = q1; pts[3 * pos + 2] = q2;
      mvo_dmatch m = matches[inl[k]];
      m.img_idx = -1;                                                 // cv::DMatch(queryIdx, trainIdx, distance)
      kept[pos] = m;
      kept_ang[pos] = as_host_nan(an);
    }
    __syncthreads();
    if (tid == 0) for (int w = 0; w < VIB_T / 32; ++w) S.n_kept += S.warp_sum[w];
    __syncthreads();
  }
  return med;
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
  const int pair = blockIdx.x, tid = threadIdx.x;
  const mvo_relative_poses_result &rp = a.rp[pair];
  mvo_init_candidate_result &out = a.out[pair];
  const int status = rp.status;
  if (status != MVO_OK && status != MVO_ERR_DEGENERATE) { if (tid == 0) out.status = status; return; }
  if (tid == 0) {
    memset(&S.rec, 0, sizeof S.rec);
    S.rec.best_sol = -1;
    for (int q = 0; q < 16; ++q) S.rec.T_w_c[q] = S.r.Tref[q] = a.T_ref[q];
    S.bad = 0;
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
    for (int q = 0; q < 9; ++q) S.r.R[q] = rp.sol.R[best][q];
    for (int q = 0; q < 3; ++q) S.r.t[q] = rp.sol.t[best][q];
    candidate_pose(S.r.R, S.r.t, S.r.Tref, S.r.Tc);
  }
  __syncthreads();
  // ---- retainGoodTriangulationResult_ on the chosen solution's points ----
  const float *p3 = a.rp_pts3d + ((size_t)pair * 5 + best) * a.cap * 3;
  retain_good_triangulation(p3, ni, inl, matches, a.min_triang_angle, a.max_ratio_angle_to_median, ang, pts, a.kept + row,
                            a.kept_angles + row, S.r);
  const bool has_nan = S.r.nan != 0;
  const int nk = S.r.n_kept;
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
      for (int q = 0; q < 3; ++q) S.r.t[q] *= scale;
      candidate_pose(S.r.R, S.r.t, S.r.Tref, S.r.Tc);
      S.rec.normalized = 1;
      S.rec.scale = as_host_nan(scale);
    }
    for (int q = 0; q < 3; ++q) S.rec.t_curr_to_prev[q] = S.r.t[q];
    for (int q = 0; q < 16; ++q) S.rec.T_w_c[q] = S.r.Tc[q];
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
      if (tid == 0) { voi::sort_d(ang, nk, S.sort_stack); S.r.med = ang[nk / 2]; }
      __syncthreads();
      med2 = S.r.med;
    } else {
      med2 = radix_select(ang, nk, nk / 2, S.r);
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

// ---------------------------------------------------------------------------------------------- mvo_vo_keyframe_points_batch_dev
// getMotionFromFrame1to2(curr_, ref_) = T_w_c_curr^-1 * T_w_c_ref (insert_keyframe's order of operations); one thread
__device__ __attribute__((noinline)) void known_motion(const double *T_curr, const double *T_ref, double *R, double *t) {
  double Tci[16], T[16];
  inv_rigid(T_curr, Tci);
  voi::mul44(Tci, T_ref, T);
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[i * 3 + j] = T[i * 4 + j]; t[i] = T[i * 4 + 3]; }
}

// Launch 1 of 3: the per-pair checks, each before anything is read through the value it checks, and the record of every pair.  A
// usable pair's record carries the known motion to the triangulation and to k_kf_points; n_kept and median_angle follow there.
__global__ void __launch_bounds__(VIB_T) k_kf_motion(const MvoKeyframePoints a) {
  __shared__ mvo_keyframe_points_result rec;
  __shared__ double Tq[16], Tt[16];
  __shared__ int bad;
  const int pair = blockIdx.x, tid = threadIdx.x;
  const mvo_two_view_result &e = a.ess[pair];
  mvo_keyframe_points_result &out = a.out[pair];
  const int status = e.status;
  if (status != MVO_OK && status != MVO_ERR_DEGENERATE) { if (tid == 0) out.status = status; return; }
  const int2 fr = reinterpret_cast<const int2 *>(a.pairs)[pair];
  const int nm = a.n_matches[pair];
  if (fr.x < 0 || fr.x >= a.batch || fr.y < 0 || fr.y >= a.batch || nm < 0 || nm > a.cap) {
    if (tid == 0) out.status = MVO_ERR_INVALID_ARG;
    return;
  }
  const int ni = status == MVO_OK ? e.n_inliers : 0;
  if (ni < 0 || ni > nm) { if (tid == 0) out.status = MVO_ERR_INVALID_ARG; return; }
  if (tid == 0) {
    memset(&rec, 0, sizeof rec);
    rec.n_matches = nm;
    bad = 0;
  }
  __syncthreads();
  if (status == MVO_OK) {
    const size_t row = (size_t)pair * a.cap;
    const int32_t *inl = a.ess_inliers + row;
    const mvo_dmatch *matches = a.matches + row;
    const int cq = min(max(a.counts[fr.x], 0), a.cap), ct = min(max(a.counts[fr.y], 0), a.cap);
    for (int k = tid; k < ni; k += VIB_T) {
      const int i = inl[k];
      if (i < 0 || i >= nm) { atomicOr(&bad, 1); continue; }
      const mvo_dmatch m = matches[i];
      if (m.query_idx < 0 || m.query_idx >= cq || m.train_idx < 0 || m.train_idx >= ct) atomicOr(&bad, 1);
    }
    if (tid < 32) {
      const double x = a.T_w_c[(size_t)(tid < 16 ? fr.x : fr.y) * 16 + (tid & 15)];
      if (!isfinite(x)) atomicOr(&bad, 1);
      (tid < 16 ? Tq : Tt)[tid & 15] = x;
    }
  }
  __syncthreads();
  if (bad) { if (tid == 0) out.status = MVO_ERR_INVALID_ARG; return; }
  if (tid == 0 && status == MVO_OK) {
    rec.usable = 1;
    rec.n_inliers = ni;
    known_motion(Tt, Tq, rec.R_curr_to_prev, rec.t_curr_to_prev);
  }
  __syncthreads();
  const unsigned long long *src = reinterpret_cast<const unsigned long long *>(&rec);
  unsigned long long *dst = reinterpret_cast<unsigned long long *>(&out);
  for (int q = tid; q < (int)(sizeof rec / 8); q += VIB_T) dst[q] = src[q];
}

struct KfSmem {
  RetainSmem r;
  double cam[3];
  int ok, ni;
};

// Launch 3 of 3: the triangulated inliers (in the pair's kept_pts3d row, camera of the reference keyframe) through transCoord and
// the retain step, then the kept rows and, per kept point, the map point's world position and viewing direction
// (pushCurrPointsToMap_: preTranslatePoint3f(p, T_w_c_curr) and getNormalizedMat(pos - camera centre)).
__global__ void __launch_bounds__(VIB_T, 2) k_kf_points(const MvoKeyframePoints a) {
  extern __shared__ double kfp_dyn[];
  __shared__ KfSmem S;
  double *ang = kfp_dyn;                                              // [cap] angles, then the kept angles
  float *pts = reinterpret_cast<float *>(kfp_dyn + a.cap);            // [cap][3] points in the current camera, then the kept ones
  const int pair = blockIdx.x, tid = threadIdx.x;
  mvo_keyframe_points_result &out = a.out[pair];
  if (tid == 0) {
    S.ok = out.status == MVO_OK && out.usable == 1;
    if (S.ok) {
      const int2 fr = reinterpret_cast<const int2 *>(a.pairs)[pair];
      for (int q = 0; q < 9; ++q) S.r.R[q] = out.R_curr_to_prev[q];
      for (int q = 0; q < 3; ++q) S.r.t[q] = out.t_curr_to_prev[q];
      for (int q = 0; q < 16; ++q) { S.r.Tc[q] = a.T_w_c[(size_t)fr.y * 16 + q]; S.r.Tref[q] = a.T_w_c[(size_t)fr.x * 16 + q]; }
      for (int q = 0; q < 3; ++q) S.cam[q] = S.r.Tc[q * 4 + 3];       // Frame::getCamCenter
      S.ni = out.n_inliers;
    }
  }
  __syncthreads();
  if (!S.ok) return;
  const int ni = S.ni;
  const size_t row = (size_t)pair * a.cap;
  float *rows = a.kept_pts3d + row * 3;
  const double med = retain_good_triangulation(rows, ni, a.ess_inliers + row, a.matches + row, a.min_triang_angle,
                                               a.max_ratio_angle_to_median, ang, pts, a.kept + row, a.kept_angles + row, S.r);
  const int nk = S.r.n_kept;                                          // every point is staged: the rows may be overwritten now
  for (int i = tid; i < 3 * nk; i += VIB_T) rows[i] = pts[i];
  if (a.kept_world || a.kept_norm) {
    for (int i = tid; i < nk; i += VIB_T) {
      float pos[3];
      pre_translate(pts + 3 * i, S.r.Tc, pos);
      if (a.kept_world) for (int q = 0; q < 3; ++q) a.kept_world[(row + i) * 3 + q] = pos[q];
      if (a.kept_norm) {
        const double d[3] = {(double)pos[0] - S.cam[0], (double)pos[1] - S.cam[1], (double)pos[2] - S.cam[2]};
        const double len = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        for (int q = 0; q < 3; ++q) a.kept_norm[(row + i) * 3 + q] = as_host_nan(d[q] / len);
      }
    }
  }
  if (tid == 0) {
    out.n_kept = nk;
    out.median_angle = as_host_nan(med);
  }
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

// declared in mvo_internal.h; mvo_vo_keyframe_points_batch_dev (vo_pipeline.cpp) checks the arguments and calls it: three launches
int mvo_vo_keyframe_points_launch(mvo_ctx *ctx, const MvoKeyframePoints &a) {
  static_assert(sizeof(mvo_keyframe_points_result) == 128, "mvo_keyframe_points_result: 128 bytes, 8-byte words");
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  { KTimer kt(ctx, KC_EPI);
  k_kf_motion<<<a.n_pairs, VIB_T, 0, ctx->stream>>>(a); }
  MVO_CHECK_LAUNCH(ctx);
  MVO_TRY(mvo_kf_triangulate_launch(ctx, a));
  const size_t smem = (size_t)a.cap * (sizeof(double) + 3 * sizeof(float));
  // as above: KfSmem and the dynamic rows together against the 48 KB
  if (smem + sizeof(KfSmem) > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_kf_points, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  { KTimer kt(ctx, KC_EPI);
  k_kf_points<<<a.n_pairs, VIB_T, smem, ctx->stream>>>(a); }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}
