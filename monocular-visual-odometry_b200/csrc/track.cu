// Glue kernels of the device-resident tracking step (tracker.cpp): the pieces of
// vo::VisualOdometry::addFrame's tracking branch (reference src/vo/vo_addFrame.cpp:71-91) that the
// reference does with host loops over cv::Mat / std::vector, kept on the GPU so that the map, the frame
// buffer and the BA graph never cross PCIe:
//   k_project_map   getMappointsInCurrentView_ (src/vo/vo.cpp:16-49): project every map point with the
//                   guess pose, flag the ones in front of the camera and inside the image
//   k_kpt_xy        keypoint pt pairs for the radius-gated matcher (method 3)
//   k_gather_pairs  the 3d-2d pairs of poseEstimationPnP_ (vo.cpp:293-301) from the match list
//   k_track_glue    vo.cpp:333-379: inlier connections of the new frame (-> its slot of the frame buffer),
//                   T_w_c = [R|t]^-1 jump test against the previous frame, pose fallback, BA gate
// All tiny (<= 2001 elements): one or a few CTAs each; they exist to remove host round trips, not for FLOPs.
#include <algorithm>
#include <string.h>
#include "mvo_internal.h"

namespace {

#define MVO_DYN_SMEM(type, name) extern __shared__ __align__(16) type name[]
#include "launch_pdl.cuh"
#include "track_filter.cuh"

__global__ void __launch_bounds__(256)
k_project_map(const float *__restrict__ map_pts, int nmap, Rt12 Tcw, double fx, double fy, double cx, double cy,
              float fcols, float frows, uint8_t *__restrict__ vis, float2 *__restrict__ cxy) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nmap) return;
  float2 uv;
  const bool ok = project_point(map_pts, i, Tcw, fx, fy, cx, cy, fcols, frows, uv);
  vis[i] = ok ? 1 : 0;
  cxy[i] = uv;
}

__global__ void __launch_bounds__(256)
k_kpt_xy(const mvo_keypoint *__restrict__ kpts, int n, float2 *__restrict__ xy) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) xy[i] = make_float2(kpts[i].x, kpts[i].y);
}

// Frame::calcDescriptors' colour sampling (frame.h:80-84, basics::getPixelAt): {r, g, b} of pixel (floor x, floor y)
__global__ void __launch_bounds__(256)
k_kpt_colors(const mvo_keypoint *__restrict__ kpts, int n, const uint8_t *__restrict__ image, int channels, size_t stride, uint8_t *__restrict__ rgb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = (int)floorf(kpts[i].x), y = (int)floorf(kpts[i].y);
  const uint8_t *px = image + (size_t)y * stride + (size_t)x * channels;
  if (channels == 3) { rgb[3 * i] = px[2]; rgb[3 * i + 1] = px[1]; rgb[3 * i + 2] = px[0]; }
  else { rgb[3 * i] = rgb[3 * i + 1] = rgb[3 * i + 2] = px[0]; }
}

__global__ void __launch_bounds__(256)
k_gather_pairs(const int2 *__restrict__ pairs, int n, const int32_t *__restrict__ n_dev, const float *__restrict__ map_pts,
               const mvo_keypoint *__restrict__ kpts, float *__restrict__ p3, float *__restrict__ p2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) n = min(n, *n_dev);
  if (i >= n) return;
  const int2 pr = pairs[i];
  p3[3 * i] = map_pts[3 * pr.x]; p3[3 * i + 1] = map_pts[3 * pr.x + 1]; p3[3 * i + 2] = map_pts[3 * pr.x + 2];
  p2[2 * i] = kpts[pr.y].x; p2[2 * i + 1] = kpts[pr.y].y;
}

__global__ void __launch_bounds__(1024) k_track_glue(MvoTrackGlue a) {
  const int tid = threadIdx.x;
  pdl_wait();
  pdl_launch_dependents();
  // every thread derives the (uniform) control values itself, so the edge copy below does not wait for thread 0
  int mode = a.mode;
  if (mode == 2) mode = (*a.n_pairs_dev >= a.min_pnp && *a.n_pairs_dev >= 4) ? 1 : 0;     // vo.cpp:304,311
  int n_in = 0;
  bool model = false;
  if (mode == 1) { n_in = a.out_i[0]; model = n_in >= 4; if (!model) n_in = 0; }
  if (tid == 0) {
    int ok = 0;
    double P[12];
    for (int q = 0; q < 12; ++q) P[q] = a.fallback[q];
    if (model) {
      ok = 1;
      for (int q = 0; q < 12; ++q) P[q] = a.pose_io[q];
      // T_w_c = [R|t]^-1 (vo.cpp:357): translation -R^T t; reject jumps relative to the previous frame (:360-369)
      const double tx = -(P[0] * P[9] + P[3] * P[10] + P[6] * P[11]);
      const double ty = -(P[1] * P[9] + P[4] * P[10] + P[7] * P[11]);
      const double tz = -(P[2] * P[9] + P[5] * P[10] + P[8] * P[11]);
      const double dx = tx - a.prev_twc[0], dy = ty - a.prev_twc[1], dz = tz - a.prev_twc[2];
      if (a.has_prev && sqrt(dx * dx + dy * dy + dz * dz) >= a.max_dist) ok = 0;
      if (!ok) for (int q = 0; q < 12; ++q) P[q] = a.fallback[q];
    }
    for (int q = 0; q < 12; ++q) { a.pose[(size_t)a.slot * 12 + q] = P[q]; a.res_d[q] = P[q]; }
    a.cnt[a.slot] = n_in;                       // the connections are recorded before the jump test (vo.cpp:333-354)
    a.skip_flag[0] = (ok && a.ba_enable) ? 0 : 1;
    a.res_i[0] = model; a.res_i[1] = ok; a.res_i[2] = n_in;
  }
  n_in = min(n_in, a.cap);
  for (int j = tid; j < n_in; j += blockDim.x) {
    const int2 pr = a.pairs[a.inl[j]];
    a.edge_map[(size_t)a.slot * a.cap + j] = a.map_ids[pr.x];
    a.edge_kp[(size_t)a.slot * a.cap + j] = pr.y;
    a.edge_obs[(size_t)a.slot * a.cap + j] = make_float2(a.kpts[pr.y].x, a.kpts[pr.y].y);
    if (a.match_cnt) a.match_cnt[pr.x] += 1;        // matched_times_++ (vo.cpp:347); the pairs have distinct map points
  }
  if (a.vis_cnt)
    for (int q = tid; q < a.nmap; q += blockDim.x) a.vis_cnt[q] += a.vis[q] != 0;
}

// Up to MVO_PACK_SEGS device arrays gathered into one staging buffer (32-bit words; a segment may be zeroed behind the copy: the
// visible / matched counters are read and reset in one go), so that a keyframe fetch costs ONE device-to-host copy instead of seven
// small ones queued behind each other.
__global__ void __launch_bounds__(256) k_pack_segments(MvoPackSegs a, uint32_t *__restrict__ dst) {
  const uint32_t total = a.first[a.n];
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int s = 0;
    while (s + 1 < a.n && i >= a.first[s + 1]) ++s;
    const uint32_t k = i - a.first[s];
    dst[a.dst_word[s] + k] = a.src[s][k];
    if (a.zero_after[s]) const_cast<uint32_t *>(a.src[s])[k] = 0;
  }
}

}  // namespace

int mvo_track_pack_segments(mvo_ctx *ctx, const MvoPackSegs &segs, uint32_t *d_dst) {
  if (segs.n <= 0 || segs.first[segs.n] == 0) return MVO_OK;
  const uint32_t total = segs.first[segs.n];
  int grid = (int)((total + 255) / 256);
  if (grid > 2 * ctx->sm_count) grid = 2 * ctx->sm_count;
  KTimer kt(ctx, KC_TRACK);
  k_pack_segments<<<grid, 256, 0, ctx->stream>>>(segs, d_dst);
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

// ---- launchers (asynchronous on ctx->stream) ------------------------------------------------------------
int mvo_track_project_map(mvo_ctx *ctx, const float *d_map_pts, int nmap, const double *Tcw12, const double *K,
                          int rows, int cols, uint8_t *d_vis, float *d_cxy) {
  if (nmap <= 0) return MVO_OK;
  Rt12 T;
  for (int q = 0; q < 12; ++q) T.v[q] = Tcw12[q];
  KTimer kt(ctx, KC_TRACK);
  k_project_map<<<(nmap + 255) / 256, 256, 0, ctx->stream>>>(d_map_pts, nmap, T, K[0], K[4], K[2], K[5], (float)cols, (float)rows,
                                                               d_vis, (float2 *)d_cxy);
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int mvo_track_kpt_colors(mvo_ctx *ctx, const mvo_keypoint *d_kpts, int n, const uint8_t *d_image, int channels, size_t stride, uint8_t *d_rgb) {
  if (n <= 0) return MVO_OK;
  KTimer kt(ctx, KC_TRACK);
  k_kpt_colors<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_kpts, n, d_image, channels, stride, d_rgb);
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int mvo_track_kpt_xy(mvo_ctx *ctx, const mvo_keypoint *d_kpts, int n, float *d_xy) {
  if (n <= 0) return MVO_OK;
  KTimer kt(ctx, KC_TRACK);
  k_kpt_xy<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_kpts, n, (float2 *)d_xy);
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int mvo_track_gather_pairs(mvo_ctx *ctx, const int32_t *d_pairs, int n, const int32_t *d_n, const float *d_map_pts,
                           const mvo_keypoint *d_kpts, float *d_p3, float *d_p2) {
  if (n <= 0) return MVO_OK;
  KTimer kt(ctx, KC_TRACK);
  k_gather_pairs<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const int2 *)d_pairs, n, d_n, d_map_pts, d_kpts, d_p3, d_p2);
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int mvo_track_glue(mvo_ctx *ctx, const MvoTrackGlue &g) {
  KTimer kt(ctx, KC_TRACK);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, 1, 1024, 0, 0, k_track_glue, g));
  ctx->launches++;
  return MVO_OK;
}

// =========================================================================================================
// k_match_filter: the tail of geometry::matchFeatures on the device — the distance thresholds
// (feature_match.cpp:179-217) and removeDuplicatedMatches (:241-260) — so that the match list never visits the
// host between the matcher and PnP.
//
// removeDuplicatedMatches is `std::sort(matches, by trainIdx)` (unstable) + "keep the first of every run", so which
// of several map points matched to one keypoint survives is decided by libstdc++'s introsort.  That algorithm is
// restated here step by step rather than replaced:
//   std::sort = __introsort_loop (median-of-3 quicksort until every segment has <= 16 elements, depth limit
//               2*floor(log2 n), heapsort beyond it) + __final_insertion_sort.
//   * The final insertion sort is stable, so the first element of a run of equal keys is the one that stands
//     leftmost after the quicksort phase: the survivors need that phase only (one atomicMin per element afterwards).
//   * __unguarded_partition(first+1, last, pivot=*first) swaps the k-th element >= pivot from the left (Lo[k])
//     with the k-th element <= pivot from the right (Ro[k]) while Lo[k] < Ro[k]; both scans only ever look at
//     untouched elements, so Lo / Ro are properties of the segment BEFORE the partition: a warp lists them with
//     ballots, counts K = #{k : Lo[k] < Ro[k]}, performs the K swaps in parallel and returns the cut
//     min(Lo[K], Ro[K-1]) (Lo[0] when K = 0) — exactly where the sequential scan stops.
//   * Recursion order is irrelevant (segments are disjoint): segments are processed level by level, one warp
//     per segment.  (Measured alternatives that were slower on real match lists: whole-CTA partitions of the large
//     segments — ~4.5K cycles each, and unbalanced median-of-3 splits keep a few large segments alive for many
//     levels — and warp-local depth-first subtrees.)
//   * If a segment is still > 16 at the depth limit (libstdc++ would switch to heapsort: adversarial inputs
//     only) the kernel reports status 1 and the host finishes the frame through the host path.
// Parity: tests/test_tracker_gpu.py (same match lists as the host std::sort on every frame, all three methods).
// (kernel text: track_filter.cuh)

int mvo_track_match_filter(mvo_ctx *ctx, const MvoTrackFilter &f) {
  int cap = 2048;
  while (cap < std::max(std::min(f.nmap, 65535), f.nk) && cap < MF_MAXN) cap *= 2;
  FilterArgs a;
  memset(&a, 0, sizeof a);
  a.keys = f.d_keys; a.vis = f.d_vis; a.nmap = f.nmap; a.nk = f.nk; a.method = f.method; a.n_cap = cap;
  a.xg_ratio = ctx->prm.xiang_gao_ratio; a.lowe_ratio = ctx->prm.lowe_ratio;
  a.pairs = (int2 *)f.d_pairs; a.info = f.d_info;
  a.project = f.Tcw12 != nullptr || f.d_Tcw12 != nullptr;
  a.map_pts = f.d_map_pts;
  a.d_Tcw = f.d_Tcw12;
  if (a.project) {
    if (f.Tcw12) for (int q = 0; q < 12; ++q) a.Tcw.v[q] = f.Tcw12[q];
    a.fx = f.K[0]; a.fy = f.K[4]; a.cx = f.K[2]; a.cy = f.K[5];
    a.fcols = (float)f.cols; a.frows = (float)f.rows;
  }
  a.kpts = f.d_kpts; a.p3 = f.d_p3; a.p2 = f.d_p2;
  const size_t smem = (size_t)cap * (4 + 4 + 2 + 2 + 2) + 3 * ((size_t)cap / 16 + 2) * 4 + ((size_t)cap / 16 + 2) + 64;
  MVO_CUDA(ctx, cudaFuncSetAttribute(k_match_filter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KTimer kt(ctx, KC_TRACK);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, 1, MF_T, smem, 0, k_match_filter, a));
  ctx->launches++;
  return MVO_OK;
}

// geometry::matchFeatures over a batch of frame pairs, on the device: match_batch_kernel (match.cu) for all pairs in one launch,
// then k_match_filter_batch, one CTA per pair.  Two launches whatever n_pairs is; no host synchronisation once the scratch
// buffers have reached their size.
extern "C" int mvo_match_features_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const uint8_t *d_desc, const int32_t *d_counts,
                                            int batch, int cap, const int32_t *d_pairs, int n_pairs, int method_index, float radius,
                                            mvo_dmatch *d_out, int32_t *d_n_out) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (method_index < 1 || method_index > 3)   // feature_match.cpp:225 throws
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "matchFeatures batch: wrong method index %d", method_index);
  if (n_pairs < 0 || batch < 1 || cap < 1)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "matchFeatures batch: n_pairs=%d batch=%d cap=%d", n_pairs, batch, cap);
  if (!d_desc || !d_counts || !d_pairs || !d_out || !d_n_out || (method_index == 3 && !d_kpts))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "matchFeatures batch: null pointer");
  if (cap > MF_MAXN) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "matchFeatures batch: cap %d above the device filter's %d", cap, MF_MAXN);
  if (n_pairs > 65535) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "matchFeatures batch: %d pairs, at most 65535 per call", n_pairs);
  if (n_pairs == 0) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int mode = method_index == 1 ? 0 : (method_index == 2 ? 1 : 2);
  const int W = mode == 1 ? 2 : 1;
  MVO_TRY(mvo_reserve(ctx, ctx->matchb_keys, (size_t)n_pairs * cap * W * 4));
  uint32_t *keys = (uint32_t *)ctx->matchb_keys.p;
  MVO_TRY(mvo_match_batch_launch(ctx, mode, d_kpts, d_desc, d_counts, batch, cap, d_pairs, n_pairs, radius, keys));

  int n_cap = 2048;
  while (n_cap < cap) n_cap *= 2;
  FilterBatchArgs b;
  b.keys = keys; b.counts = d_counts; b.pairs = (const int2 *)d_pairs;
  b.batch = batch; b.cap = cap; b.method = method_index; b.n_cap = n_cap;
  b.xg_ratio = ctx->prm.xiang_gao_ratio; b.lowe_ratio = ctx->prm.lowe_ratio;
  b.out = d_out; b.n_out = d_n_out;
  const size_t smem = (size_t)n_cap * (4 + 4 + 2 + 2 + 2) + 3 * ((size_t)n_cap / 16 + 2) * 4 + ((size_t)n_cap / 16 + 2) + 64;
  MVO_CUDA(ctx, cudaFuncSetAttribute(k_match_filter_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KTimer kt(ctx, KC_MATCH);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, (unsigned)n_pairs, MF_T, smem, 0, k_match_filter_batch, b));
  ctx->launches++;
  return MVO_OK;
}

// poseEstimationPnP_ up to solvePnPRansac for a batch of (frame, guess pose) jobs against one map (mvo.h): methods 1 / 2 launch the
// map-query matcher (match.cu) and k_map_match_filter, which projects the map itself; method 3 projects first
// (k_project_map_batch), because the matcher's radius gate needs the pixels.  A fixed number of launches whatever n_jobs is; no host
// synchronisation once the scratch buffers have reached their size.
extern "C" int mvo_vo_map_matches_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const uint8_t *d_desc, const int32_t *d_counts,
                                            int batch, int cap, const int32_t *d_frames, const double *d_T_w_c_guess, int n_jobs,
                                            const float *d_map_pts, const uint8_t *d_map_desc, int n_map, const double *K, int rows,
                                            int cols, int method_index, float radius, mvo_map_matches_result *d_out, int32_t *d_cand,
                                            float *d_cand_xy, mvo_dmatch *d_matches, float *d_pts3d, float *d_pts2d) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (method_index < 1 || method_index > 3)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "map matches batch: wrong method index %d", method_index);
  if (batch < 1 || cap < 1 || n_jobs < 0 || n_map < 0 || rows < 1 || cols < 1)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "map matches batch: batch=%d cap=%d n_jobs=%d n_map=%d rows=%d cols=%d", batch, cap, n_jobs,
                    n_map, rows, cols);
  if (!d_desc || !d_counts || !d_frames || !d_T_w_c_guess || !K || !d_out || !d_cand || !d_matches ||
      (n_map > 0 && (!d_map_pts || !d_map_desc)) || ((method_index == 3 || d_pts2d) && !d_kpts) || (!d_pts3d != !d_pts2d))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "map matches batch: null pointer");
  if (!(isfinite(K[0]) && K[0] > 0 && isfinite(K[4]) && K[4] > 0))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "map matches batch: fx=%g fy=%g", K[0], K[4]);
  if (cap > MF_MAXN) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "map matches batch: cap %d above the device filter's %d", cap, MF_MAXN);
  if (n_map > 65535 || n_jobs > 65535 || (long long)n_jobs * n_map > (1ll << 26))
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "map matches batch: n_jobs=%d n_map=%d (at most 65535 each, 2^26 together)", n_jobs, n_map);
  if (n_jobs == 0) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int mode = method_index == 1 ? 0 : (method_index == 2 ? 1 : 2);
  const int W = mode == 1 ? 2 : 1;
  const size_t cells = (size_t)n_jobs * n_map;
  const size_t vis_bytes = (cells + 15) / 16 * 16;
  MVO_TRY(mvo_reserve(ctx, ctx->mapm_buf, vis_bytes + (mode == 2 ? cells * 8 : 0) + 16));
  uint8_t *vis = (uint8_t *)ctx->mapm_buf.p;
  float2 *xy = (float2 *)(vis + vis_bytes);
  uint32_t *keys = nullptr;
  if (n_map > 0) {
    MVO_TRY(mvo_reserve(ctx, ctx->matchb_keys, cells * W * 4));
    keys = (uint32_t *)ctx->matchb_keys.p;
    if (mode == 2) {
      KTimer kt(ctx, KC_TRACK);
      MVO_CUDA(ctx, launch_pdl3(ctx->stream, dim3((n_map + 255) / 256, n_jobs), dim3(256), 0, k_project_map_batch, d_map_pts, n_map,
                                d_T_w_c_guess, K[0], K[4], K[2], K[5], (float)cols, (float)rows, xy));
      ctx->launches++;
    }
    MVO_TRY(mvo_match_map_batch_launch(ctx, mode, d_kpts, d_desc, d_counts, batch, cap, d_frames, n_jobs, d_map_desc, n_map,
                                       (const float *)xy, radius, keys));
  }
  // the filter's capacity covers the frame capacity and, up to MF_MAXN, every map point in view
  int n_cap = 2048;
  while (n_cap < std::max(std::min(n_map, MF_MAXN), cap) && n_cap < MF_MAXN) n_cap *= 2;
  MapFilterArgs b;
  memset(&b, 0, sizeof b);
  b.keys = keys; b.vis = vis; b.kpts = d_kpts; b.counts = d_counts; b.frames = d_frames; b.T_w_c = d_T_w_c_guess; b.map_pts = d_map_pts;
  b.batch = batch; b.cap = cap; b.n_map = n_map; b.method = method_index; b.n_cap = n_cap;
  b.xg_ratio = ctx->prm.xiang_gao_ratio; b.lowe_ratio = ctx->prm.lowe_ratio;
  b.fx = K[0]; b.fy = K[4]; b.cx = K[2]; b.cy = K[5];
  b.fcols = (float)cols; b.frows = (float)rows;
  b.out = d_out; b.cand = d_cand; b.cand_xy = d_cand_xy; b.matches = d_matches; b.p3 = d_pts3d; b.p2 = d_pts2d;
  const size_t smem = (size_t)n_cap * (4 + 4 + 2 + 2 + 2) + 3 * ((size_t)n_cap / 16 + 2) * 4 + ((size_t)n_cap / 16 + 2) + 64;
  MVO_CUDA(ctx, cudaFuncSetAttribute(k_map_match_filter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KTimer kt(ctx, KC_TRACK);
  MVO_CUDA(ctx, launch_pdl(ctx->stream, (unsigned)n_jobs, MF_T, smem, 0, k_map_match_filter, b));
  ctx->launches++;
  return MVO_OK;
}
