// All-pairs descriptor matching for sm_90a.
//
// Replaces, bit-exactly (integer distances, lowest-train-index tie rule):
//   mode 0  cv::BFMatcher(NORM_HAMMING).match   — the exact search behind
//           matcher_flann.match at reference src/geometry/feature_match.cpp:162
//   mode 1  matcher_bf->knnMatch(d1, d2, knn, 2) at feature_match.cpp:208
//   mode 2  geometry::matchByRadiusAndBruteForce, feature_match.cpp:86-124
//
// Layout: descriptors are N x 32 bytes, row-major, 16-byte aligned rows (two uint4 per row).
// One thread owns one QUERY descriptor in 8 registers and streams a chunk of TRAIN
// descriptors out of shared memory (every lane reads the same address -> LDS broadcast).
// The train set is split over blockIdx.y so that ~2000 x 2000 problems still fill the 132 SMs of an H100;
// each CTA writes its partial winners and the last CTA of a query tile (atomic ticket)
// merges them, so the whole match is ONE launch and no atomics touch the result itself
// (deterministic).  The result of a (query, train) comparison is folded into one u32 key
// (distance << 16 | train index) so "smaller distance, then lower index" is a single IMNMX.
//
// Arithmetic per pair, Hamming: 8 LOP3 (xor) + 8 LOP3 (carry-save adders) + 4 POPC + 3 adds
// + 1 pack + 1 min.  No tensor cores: integer/POPC-issue bound (SURVEY.md §8d).
#include <algorithm>
#include "mvo_internal.h"
#include "launch_pdl.cuh"

namespace {

constexpr int kQ = 128;          // queries (threads) per CTA
constexpr int kMaxChunk = 128;   // train descriptors per CTA (upper bound)

__device__ __forceinline__ void csa(uint32_t a, uint32_t b, uint32_t c, uint32_t &s, uint32_t &k) {
  s = a ^ b ^ c;
  k = (a & b) | (c & (a ^ b));
}

// 256-bit Hamming distance between q[0..7] and t (two uint4).
__device__ __forceinline__ uint32_t hamming256(const uint32_t (&q)[8], const uint4 &t0, const uint4 &t1) {
  uint32_t w0 = q[0] ^ t0.x, w1 = q[1] ^ t0.y, w2 = q[2] ^ t0.z, w3 = q[3] ^ t0.w;
  uint32_t w4 = q[4] ^ t1.x, w5 = q[5] ^ t1.y, w6 = q[6] ^ t1.z, w7 = q[7] ^ t1.w;
#ifdef MVO_MATCH_NAIVE_POPC
  return __popc(w0) + __popc(w1) + __popc(w2) + __popc(w3) + __popc(w4) + __popc(w5) + __popc(w6) + __popc(w7);
#else
  uint32_t s1, c1, s2, c2, s3, c3, t1_, f1;
  csa(w0, w1, w2, s1, c1);
  csa(s1, w3, w4, s2, c2);
  csa(s2, w5, w6, s3, c3);
  csa(c1, c2, c3, t1_, f1);
  return (__popc(s3) + __popc(w7)) + 2u * (__popc(t1_) + 2u * __popc(f1));
#endif
}

// sum_i |a_i - b_i| over 32 bytes (feature_match.cpp:110-111: absdiff + sum).
__device__ __forceinline__ uint32_t sad256(const uint32_t (&q)[8], const uint4 &t0, const uint4 &t1) {
  uint32_t s = __vsadu4(q[0], t0.x);
  s += __vsadu4(q[1], t0.y);
  s += __vsadu4(q[2], t0.z);
  s += __vsadu4(q[3], t0.w);
  s += __vsadu4(q[4], t1.x);
  s += __vsadu4(q[5], t1.y);
  s += __vsadu4(q[6], t1.z);
  s += __vsadu4(q[7], t1.w);
  return s;
}

__device__ __forceinline__ void top2_insert(uint32_t &b1, uint32_t &b2, uint32_t k) {
  b2 = min(b2, max(b1, k));
  b1 = min(b1, k);
}

// MODE 0: Hamming NN, 1: Hamming top-2, 2: radius-gated SAD NN.
template <int MODE>
__global__ void __launch_bounds__(kQ)
match_kernel(const uint4 *__restrict__ d1, const float2 *__restrict__ xy1, int n1,
             const uint4 *__restrict__ d2, const float2 *__restrict__ xy2, int n2, int chunk,
             float r2, uint32_t *__restrict__ part, unsigned int *__restrict__ tickets,
             uint32_t *__restrict__ keys, const uint8_t *__restrict__ qmask, const int32_t *__restrict__ n2_dev) {
  pdl_wait();                              // the describe kernel wrote the train descriptors (and their count, n2_dev)
  pdl_launch_dependents();
  // n2_dev (optional): the number of train descriptors lives on the device (the extraction's keypoint count never visited the
  // host); n2 is then its upper bound and the grid was sized for it — splits beyond the real count report "no match"
  if (n2_dev) n2 = min(n2, *n2_dev);
  __shared__ uint4 s_t[kMaxChunk * 2];
  __shared__ float2 s_xy[MODE == 2 ? kMaxChunk : 1];
  __shared__ bool s_last;

  const int q = blockIdx.x * kQ + threadIdx.x;
  const int split = blockIdx.y, nsplit = gridDim.y;
  const int j0 = split * chunk;
  const int cnt = max(0, min(chunk, n2 - j0));

  for (int i = threadIdx.x; i < cnt * 2; i += kQ) s_t[i] = d2[(size_t)j0 * 2 + i];
  if (MODE == 2)
    for (int i = threadIdx.x; i < cnt; i += kQ) s_xy[i] = xy2[j0 + i];

  uint32_t qw[8];
  float qx = 0.f, qy = 0.f;
  const int qc = min(q, n1 - 1);   // clamp: out-of-range threads compute on a valid row, never store
  {
    uint4 a = d1[(size_t)qc * 2], b = d1[(size_t)qc * 2 + 1];
    qw[0] = a.x; qw[1] = a.y; qw[2] = a.z; qw[3] = a.w;
    qw[4] = b.x; qw[5] = b.y; qw[6] = b.z; qw[7] = b.w;
    if (MODE == 2) { float2 p = xy1[qc]; qx = p.x; qy = p.y; }
  }
  __syncthreads();

  uint32_t b1 = 0xFFFFFFFFu, b2 = 0xFFFFFFFFu;
#pragma unroll 4
  for (int j = 0; j < cnt; ++j) {
    const uint4 t0 = s_t[2 * j], t1 = s_t[2 * j + 1];
    uint32_t key;
    if (MODE == 2) {
      // feature_match.cpp:105: (x-x2)*(x-x2) + (y-y2)*(y-y2) <= r2 in float, no contraction.
      const float2 p = s_xy[j];
      const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y);
      const float dd = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
      const uint32_t d = sad256(qw, t0, t1);
      key = (dd <= r2) ? ((d << 16) | (uint32_t)(j0 + j)) : 0xFFFFFFFFu;
    } else {
      key = (hamming256(qw, t0, t1) << 16) | (uint32_t)(j0 + j);
    }
    if (MODE == 1) top2_insert(b1, b2, key);
    else b1 = min(b1, key);
  }

  constexpr int W = (MODE == 1) ? 2 : 1;
  // qmask (optional): queries whose mask byte is 0 report "no match" (the tracker matches the whole resident
  // map and masks the points outside the current view instead of compacting them first)
  const bool masked = qmask != nullptr && q < n1 && qmask[q] == 0;
  if (nsplit == 1) {
    if (masked) b1 = b2 = 0xFFFFFFFFu;
    if (q < n1) {
      keys[(size_t)q * W] = b1;
      if (MODE == 1) keys[(size_t)q * W + 1] = b2;
    }
    return;
  }
  if (q < n1) {
    part[((size_t)split * n1 + q) * W] = b1;
    if (MODE == 1) part[((size_t)split * n1 + q) * W + 1] = b2;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = atomicAdd(&tickets[blockIdx.x], 1u);
    s_last = (t == (unsigned)nsplit - 1);
    if (s_last) tickets[blockIdx.x] = 0;   // leave the counter ready for the next launch
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (q < n1) {
    uint32_t m1 = 0xFFFFFFFFu, m2 = 0xFFFFFFFFu;
    for (int s = 0; s < nsplit; ++s) {
      const uint32_t *p = part + ((size_t)s * n1 + q) * W;
      const uint32_t k1 = __ldcg(p);
      if (MODE == 1) {
        const uint32_t k2 = __ldcg(p + 1);
        top2_insert(m1, m2, k1);
        top2_insert(m1, m2, k2);
      } else {
        m1 = min(m1, k1);
      }
    }
    if (masked) m1 = m2 = 0xFFFFFFFFu;
    keys[(size_t)q * W] = m1;
    if (MODE == 1) keys[(size_t)q * W + 1] = m2;
  }
}

// The same search over a batch of frame pairs of a batched extraction (mvo_match_features_batch_dev): grid = query tiles x
// train splits x pairs, sized from the per-frame capacity; both counts are read on the device.  A split covers `span` trains
// and streams them through shared memory kMaxChunk at a time, so that a batch with many pairs can use one split per tile and
// skip the merge.  Tiles beyond a pair's query count and splits beyond its train count exit; pairs with a frame index outside
// [0, batch) (and method-2 pairs with fewer than two trains) are left to the tail kernel, which reports them.
// kMapQuery (mvo_vo_map_matches_batch_dev): the queries are one map's descriptors, shared by every job, and the trains are frame
// frames[z] of job z; MODE 2 takes job z's query pixels from qxy.  Keys and partial winners are then laid out per job with n_map
// query rows instead of cap.
struct MatchBatchArgs {
  const uint4 *desc;             // [batch][cap][2]
  const mvo_keypoint *kpts;      // [batch][cap] (MODE 2: pt)
  const int32_t *counts;         // [batch]
  const int2 *pairs;             // [n_pairs] (query frame, train frame)
  int batch, cap, span;
  float r2;
  uint32_t *part;                // [n_pairs][gridDim.y][cap][W] partial winners
  unsigned int *tickets;         // [n_pairs][gridDim.x], zero between launches
  uint32_t *keys;                // [n_pairs][cap][W]
  // kMapQuery only
  const uint4 *qdesc;            // [n_map][2]
  const float2 *qxy;             // [n_jobs][n_map] (MODE 2)
  const int32_t *frames;         // [n_jobs]
  int nq;                        // n_map
};

template <int MODE, bool kMapQuery = false>
__global__ void __launch_bounds__(kQ) match_batch_kernel(MatchBatchArgs a) {
  pdl_wait();                              // the extraction wrote descriptors, keypoints and counts
  pdl_launch_dependents();
  __shared__ uint4 s_t[kMaxChunk * 2];
  __shared__ float2 s_xy[MODE == 2 ? kMaxChunk : 1];
  __shared__ bool s_last;
  const int p = blockIdx.z;
  int2 pr;
  if (kMapQuery) {
    pr = make_int2(0, a.frames[p]);
    if (pr.y < 0 || pr.y >= a.batch) return;
  } else {
    pr = a.pairs[p];
    if (pr.x < 0 || pr.x >= a.batch || pr.y < 0 || pr.y >= a.batch) return;
  }
  const int n1 = kMapQuery ? a.nq : min(max(a.counts[pr.x], 0), a.cap), n2 = min(max(a.counts[pr.y], 0), a.cap);
  const int rows = kMapQuery ? a.nq : a.cap;           // query rows per pair in keys and part
  const int nsplit = (n2 + a.span - 1) / a.span;       // splits that hold trains of this pair
  const int split = blockIdx.y;
  if ((int)blockIdx.x * kQ >= n1 || split >= nsplit || (MODE == 1 && n2 < 2)) return;
  const uint4 *d1 = kMapQuery ? a.qdesc : a.desc + (size_t)pr.x * a.cap * 2, *d2 = a.desc + (size_t)pr.y * a.cap * 2;
  const mvo_keypoint *k1 = a.kpts + (size_t)pr.x * a.cap, *k2 = a.kpts + (size_t)pr.y * a.cap;

  const int q = blockIdx.x * kQ + threadIdx.x;
  const int j0 = split * a.span, j1 = min(j0 + a.span, n2);
  uint32_t qw[8];
  float qx = 0.f, qy = 0.f;
  const int qc = min(q, n1 - 1);   // clamp: out-of-range threads compute on a valid row, never store
  {
    uint4 u = d1[(size_t)qc * 2], v = d1[(size_t)qc * 2 + 1];
    qw[0] = u.x; qw[1] = u.y; qw[2] = u.z; qw[3] = u.w;
    qw[4] = v.x; qw[5] = v.y; qw[6] = v.z; qw[7] = v.w;
    if (MODE == 2 && kMapQuery) { const float2 pt = a.qxy[(size_t)p * a.nq + qc]; qx = pt.x; qy = pt.y; }
    else if (MODE == 2) { qx = k1[qc].x; qy = k1[qc].y; }
  }

  uint32_t b1 = 0xFFFFFFFFu, b2 = 0xFFFFFFFFu;
  for (int c0 = j0; c0 < j1; c0 += kMaxChunk) {
    const int cnt = min(kMaxChunk, j1 - c0);
    __syncthreads();                       // the previous chunk has been consumed
    for (int i = threadIdx.x; i < cnt * 2; i += kQ) s_t[i] = d2[(size_t)c0 * 2 + i];
    if (MODE == 2)
      for (int i = threadIdx.x; i < cnt; i += kQ) s_xy[i] = make_float2(k2[c0 + i].x, k2[c0 + i].y);
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < cnt; ++j) {
      const uint4 t0 = s_t[2 * j], t1 = s_t[2 * j + 1];
      uint32_t key;
      if (MODE == 2) {
        const float2 pt = s_xy[j];
        const float dx = __fsub_rn(qx, pt.x), dy = __fsub_rn(qy, pt.y);
        const float dd = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
        const uint32_t d = sad256(qw, t0, t1);
        key = (dd <= a.r2) ? ((d << 16) | (uint32_t)(c0 + j)) : 0xFFFFFFFFu;
      } else {
        key = (hamming256(qw, t0, t1) << 16) | (uint32_t)(c0 + j);
      }
      if (MODE == 1) top2_insert(b1, b2, key);
      else b1 = min(b1, key);
    }
  }

  constexpr int W = (MODE == 1) ? 2 : 1;
  uint32_t *keys = a.keys + (size_t)p * rows * W;
  if (nsplit == 1) {
    if (q < n1) {
      keys[(size_t)q * W] = b1;
      if (MODE == 1) keys[(size_t)q * W + 1] = b2;
    }
    return;
  }
  uint32_t *part = a.part + (size_t)p * gridDim.y * rows * W;
  if (q < n1) {
    part[((size_t)split * rows + q) * W] = b1;
    if (MODE == 1) part[((size_t)split * rows + q) * W + 1] = b2;
  }
  __threadfence();
  __syncthreads();
  unsigned int *ticket = a.tickets + (size_t)p * gridDim.x + blockIdx.x;
  if (threadIdx.x == 0) {
    unsigned int t = atomicAdd(ticket, 1u);
    s_last = (t == (unsigned)nsplit - 1);
    if (s_last) *ticket = 0;               // leave the counter ready for the next launch
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (q < n1) {
    uint32_t m1 = 0xFFFFFFFFu, m2 = 0xFFFFFFFFu;
    for (int s = 0; s < nsplit; ++s) {
      const uint32_t *pp = part + ((size_t)s * rows + q) * W;
      const uint32_t x1 = __ldcg(pp);
      if (MODE == 1) {
        const uint32_t x2 = __ldcg(pp + 1);
        top2_insert(m1, m2, x1);
        top2_insert(m1, m2, x2);
      } else {
        m1 = min(m1, x1);
      }
    }
    keys[(size_t)q * W] = m1;
    if (MODE == 1) keys[(size_t)q * W + 1] = m2;
  }
}

// The grid, scratch and launch of match_batch_kernel for n_pairs pairs of `rows` query rows each (a.cap trains at most): everything
// but the pair / job fields of a, which the caller has set.
int match_batch_enqueue(mvo_ctx *ctx, int mode, bool map_query, MatchBatchArgs a, int rows, int n_pairs, float radius) {
  const int W = mode == 1 ? 2 : 1;
  const int cap = a.cap;
  const int qtiles = (rows + kQ - 1) / kQ;
  // The whole batch, not one pair, has to fill the SMs: about `waves` CTAs per SM over all pairs (the rule of the single-pair
  // launch above), so a pair gets waves * sm_count / (qtiles * n_pairs) splits, at least one and no shorter than 32 trains.
  // With a chunk loop in the CTA there is no upper bound on a split's length: 63 pairs of 2001 keypoints run unsplit
  // (16 tiles x 63 pairs = 1008 CTAs, about 8 per SM on an H100), one pair is split 33 ways as before.
  const int waves = 4;
  const long long tiles = (long long)qtiles * n_pairs;
  int nsplit = (int)std::min<long long>(((long long)waves * ctx->sm_count + tiles - 1) / tiles, 65535);
  const int max_split = (cap + 31) / 32;
  if (nsplit > max_split) nsplit = max_split;
  if (nsplit < 1) nsplit = 1;
  const int span = (cap + nsplit - 1) / nsplit;
  nsplit = (cap + span - 1) / span;

  a.span = span;
  a.r2 = radius * radius;   // feature_match.cpp:96
  a.part = nullptr; a.tickets = nullptr;
  if (nsplit > 1) {
    MVO_TRY(mvo_reserve(ctx, ctx->matchb_part, (size_t)n_pairs * nsplit * rows * W * 4));
    const size_t had = ctx->matchb_tickets.cap;
    MVO_TRY(mvo_reserve(ctx, ctx->matchb_tickets, (size_t)n_pairs * qtiles * 4));
    if (ctx->matchb_tickets.cap != had)    // a new block: zero once, the kernel leaves it zeroed
      MVO_CUDA(ctx, cudaMemsetAsync(ctx->matchb_tickets.p, 0, ctx->matchb_tickets.cap, ctx->stream));
    a.part = (uint32_t *)ctx->matchb_part.p;
    a.tickets = (unsigned int *)ctx->matchb_tickets.p;
  }
  dim3 grid(qtiles, nsplit, n_pairs), block(kQ);
  KTimer kt(ctx, KC_MATCH);
  if (map_query) {
    if (mode == 0) MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_batch_kernel<0, true>, a));
    else if (mode == 1) MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_batch_kernel<1, true>, a));
    else MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_batch_kernel<2, true>, a));
  } else {
    if (mode == 0) MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_batch_kernel<0>, a));
    else if (mode == 1) MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_batch_kernel<1>, a));
    else MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_batch_kernel<2>, a));
  }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

}  // namespace

// match_batch_kernel over n_pairs pairs (mvo_internal.h); d_keys: [n_pairs][cap][W] (W = 2 for mode 1)
int mvo_match_batch_launch(mvo_ctx *ctx, int mode, const mvo_keypoint *d_kpts, const uint8_t *d_desc, const int32_t *d_counts,
                           int batch, int cap, const int32_t *d_pairs, int n_pairs, float radius, uint32_t *d_keys) {
  if (mode < 0 || mode > 2) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "match batch: bad mode %d", mode);
  if (cap < 1 || cap > 65535 || n_pairs > 65535)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "match batch: cap=%d n_pairs=%d outside [1,65535]", cap, n_pairs);
  if (n_pairs <= 0) return MVO_OK;
  MatchBatchArgs a = {};
  a.desc = (const uint4 *)d_desc; a.kpts = d_kpts; a.counts = d_counts; a.pairs = (const int2 *)d_pairs;
  a.batch = batch; a.cap = cap; a.keys = d_keys;
  return match_batch_enqueue(ctx, mode, false, a, cap, n_pairs, radius);
}

// the map-query form (mvo_internal.h); d_keys: [n_jobs][n_map][W]
int mvo_match_map_batch_launch(mvo_ctx *ctx, int mode, const mvo_keypoint *d_kpts, const uint8_t *d_desc, const int32_t *d_counts,
                               int batch, int cap, const int32_t *d_frames, int n_jobs, const uint8_t *d_map_desc, int n_map,
                               const float *d_qxy, float radius, uint32_t *d_keys) {
  if (mode < 0 || mode > 2) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "match map batch: bad mode %d", mode);
  if (cap < 1 || cap > 65535 || n_jobs > 65535 || n_map > 65535)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "match map batch: cap=%d n_jobs=%d n_map=%d outside [1,65535]", cap, n_jobs, n_map);
  if (n_jobs <= 0 || n_map <= 0) return MVO_OK;
  MatchBatchArgs a = {};
  a.desc = (const uint4 *)d_desc; a.kpts = d_kpts; a.counts = d_counts;
  a.batch = batch; a.cap = cap; a.keys = d_keys;
  a.qdesc = (const uint4 *)d_map_desc; a.qxy = (const float2 *)d_qxy; a.frames = d_frames; a.nq = n_map;
  return match_batch_enqueue(ctx, mode, true, a, n_map, n_jobs, radius);
}

int mvo_match_launch(mvo_ctx *ctx, int mode, const uint8_t *d_d1, const float *d_xy1, int n1,
                     const uint8_t *d_d2, const float *d_xy2, int n2, float radius,
                     uint32_t *d_keys) {
  return mvo_match_launch_masked(ctx, mode, d_d1, d_xy1, n1, d_d2, d_xy2, n2, radius, d_keys, nullptr);
}

int mvo_match_launch_masked(mvo_ctx *ctx, int mode, const uint8_t *d_d1, const float *d_xy1, int n1,
                            const uint8_t *d_d2, const float *d_xy2, int n2, float radius,
                            uint32_t *d_keys, const uint8_t *d_qmask) {
  return mvo_match_launch_ndev(ctx, mode, d_d1, d_xy1, n1, d_d2, d_xy2, n2, nullptr, radius, d_keys, d_qmask);
}

// d_n2 != nullptr: the train count is read on the device, n2 is its upper bound (mvo_internal.h)
int mvo_match_launch_ndev(mvo_ctx *ctx, int mode, const uint8_t *d_d1, const float *d_xy1, int n1,
                          const uint8_t *d_d2, const float *d_xy2, int n2, const int32_t *d_n2, float radius,
                          uint32_t *d_keys, const uint8_t *d_qmask) {
  if (mode < 0 || mode > 2) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "match: bad mode %d", mode);
  if (n1 < 0 || n2 < 0 || n1 > 65535 || n2 > 65535)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "match: n1=%d n2=%d outside [0,65535]", n1, n2);
  if (mode == 1 && n2 < 2) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "knn2 needs >= 2 train descriptors");
  if (mode == 2 && (!d_xy1 || !d_xy2)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "radius match needs keypoint coordinates");
  if (n1 == 0) return MVO_OK;
  const int W = mode == 1 ? 2 : 1;
  if (n2 == 0) {
    MVO_CUDA(ctx, cudaMemsetAsync(d_keys, 0xFF, (size_t)n1 * W * 4, ctx->stream));
    return MVO_OK;
  }
  const int qtiles = (n1 + kQ - 1) / kQ;
  // about 4 CTAs per SM (on the H100, 2 and 4 are within run-to-run noise of the VO pass, 8 is slower), chunks of at least 32
  // and at most kMaxChunk trains
  const int waves = 4;
  int nsplit = (waves * ctx->sm_count + qtiles - 1) / qtiles;
  const int min_split = (n2 + kMaxChunk - 1) / kMaxChunk;
  const int max_split = (n2 + 31) / 32;
  if (nsplit > max_split) nsplit = max_split;
  if (nsplit < min_split) nsplit = min_split;
  int chunk = (n2 + nsplit - 1) / nsplit;
  nsplit = (n2 + chunk - 1) / chunk;

  // scratch: partial keys [nsplit][n1][W]; tickets[qtiles] are zeroed at context creation
  // and reset by the kernel itself
  MVO_TRY(mvo_reserve(ctx, ctx->match_part, (size_t)nsplit * n1 * W * 4));
  uint32_t *part = (uint32_t *)ctx->match_part.p;
  unsigned int *tickets = (unsigned int *)ctx->match_tickets.p;
  const float r2 = radius * radius;   // feature_match.cpp:96
  dim3 grid(qtiles, nsplit), block(kQ);
  const uint4 *a = (const uint4 *)d_d1, *b = (const uint4 *)d_d2;
  const float2 *xa = (const float2 *)d_xy1, *xb = (const float2 *)d_xy2;
  KTimer kt(ctx, KC_MATCH);
  if (mode == 0)
    MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_kernel<0>, a, xa, n1, b, xb, n2, chunk, r2, part, tickets, d_keys, d_qmask, d_n2));
  else if (mode == 1)
    MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_kernel<1>, a, xa, n1, b, xb, n2, chunk, r2, part, tickets, d_keys, d_qmask, d_n2));
  else
    MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, block, 0, match_kernel<2>, a, xa, n1, b, xb, n2, chunk, r2, part, tickets, d_keys, d_qmask, d_n2));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}
