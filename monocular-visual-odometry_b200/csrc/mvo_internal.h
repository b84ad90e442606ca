// Internal declarations shared by the CUDA translation units of libmvo.so.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>
#include "mvo.h"

#define MVO_MAX_LEVELS 8
#define MVO_DESC_BYTES 32

struct mvo_ctx;

// kernel classes for the optional CUDA-event timing (mvo_timing_*)
enum MvoKernelClass { KC_GRAY = 0, KC_RESIZE, KC_FAST, KC_SELECT, KC_BLUR, KC_DESCRIBE, KC_HARRIS, KC_MATCH,
                      KC_PNP_HYP, KC_PNP_SCORE, KC_PNP_FINISH, KC_BA, KC_TRACK, KC_EPI, KC_EPI_SCORE, KC_EPI_FINISH, KC_COUNT };
struct MvoEvPair { int id; cudaEvent_t a, b; };

// ---- error plumbing -------------------------------------------------------------------
int mvo_fail(mvo_ctx *ctx, int code, const char *fmt, ...);
#define MVO_CUDA(ctx, call)                                                              \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess)                                                              \
      return mvo_fail((ctx), MVO_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call,  \
                      cudaGetErrorString(e__));                                          \
  } while (0)
#define MVO_CHECK_LAUNCH(ctx)                                                            \
  do {                                                                                   \
    (ctx)->launches++;                                                                   \
    cudaError_t e__ = cudaGetLastError();                                                \
    if (e__ != cudaSuccess)                                                              \
      return mvo_fail((ctx), MVO_ERR_CUDA, "%s:%d kernel launch -> %s", __FILE__,        \
                      __LINE__, cudaGetErrorString(e__));                                \
  } while (0)
#define MVO_TRY(expr)            \
  do {                           \
    int rc__ = (expr);           \
    if (rc__ != MVO_OK) return rc__; \
  } while (0)

// Growable device / pinned-host scratch buffers owned by the context.
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
};
struct PinBuf {
  void *p = nullptr;
  size_t cap = 0;
};

// ---- ORB per-level geometry -------------------------------------------------------------
struct OrbLevel {
  int w, h;          // level size (unbordered)
  int pitch;         // bytes per row of the level planes (multiple of 128)
  size_t img_off;    // offset of the gray plane inside a frame slot
  size_t blur_off;   // offset of the blurred plane
  float scale;       // (float)pow((double)scaleFactor_f32, level)
  int cap;           // featuresPerLevel (OpenCV distribution)
  int band_first;    // index of this level's first FAST band
  int nbands;
};

struct OrbLayout {
  int rows = 0, cols = 0, nlevels = 0;
  OrbLevel lv[MVO_MAX_LEVELS];
  size_t slot_bytes = 0;   // bytes of image planes per frame
  int total_bands = 0;
  int band_cap = 0;        // staging capacity (candidates) per band
};

struct mvo_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  mvo_params prm;
  std::string err;
  uint64_t launches = 0;
  int sm_count = 0;

  // generic scratch
  DevBuf d_b, d_c, d_d, d_f;
  PinBuf h_a, h_b;
  cudaStream_t side_stream = nullptr;   // mvo_side_stream()

  // ORB workspace (sized for `orb_batch` frames of the current layout)
  OrbLayout orb;
  int orb_batch = 0;
  DevBuf orb_planes, orb_cand, orb_bandcnt, orb_sel, orb_misc, orb_in;
  DevBuf orb_kpts, orb_desc, orb_counts;
  PinBuf orb_h;
  void *orb_state = nullptr, *orb_pending = nullptr;   // orb_host.cpp: OrbState / OrbPending of this context
  void *orb_tma = nullptr;                             // orb.cu: tensor maps of the gray planes (OrbTmaState)

  // match
  DevBuf match_part, match_tickets, match_in, match_keys;
  PinBuf match_h;
  // batched matchFeatures (mvo_match_features_batch_dev): partial winners, merge tickets, packed keys of every pair
  DevBuf matchb_part, matchb_tickets, matchb_keys;
  // batched two-view calls (mvo_esti_motion_by_essential_batch_dev, mvo_estimate_relative_poses_batch_dev): points, hypotheses,
  // counts and finish outputs of every pair; its own block, so that it never aliases the single-pair jobs' buffers
  DevBuf epib_buf;
  // the single-pair essential-matrix and homography jobs (MvoEpiJob): device rows and pinned staging of each, so that the two can
  // run side by side on two streams
  DevBuf epi_ess_buf, epi_homo_buf;
  PinBuf epi_ess_h, epi_homo_h;

  // timing
  uint32_t timing_mask = 0;
  std::vector<MvoEvPair> ev_pending;
  std::vector<cudaEvent_t> ev_pool;
  double t_ms[KC_COUNT] = {0};
  uint64_t t_cnt[KC_COUNT] = {0};

  // PnP
  DevBuf pnp_pts, pnp_hyp, pnp_cnt, pnp_out;
  int pnp_last_h = 0;
  // BA
  DevBuf ba_buf;
};

// RAII event pair around the launches of one kernel class (no-op unless enabled in timing_mask)
struct KTimer {
  mvo_ctx *c;
  int id;
  cudaEvent_t a = nullptr, b = nullptr;
  KTimer(mvo_ctx *ctx, int kernel_class);
  ~KTimer();
};

int mvo_reserve(mvo_ctx *ctx, DevBuf &b, size_t bytes);
int mvo_reserve_pinned(mvo_ctx *ctx, PinBuf &b, size_t bytes);

// Host arithmetic on rigid transforms (4x4 row-major doubles) shared by the tracker and the VO state machine, in the reference's
// operation order: tracker.cpp and vo_pipeline.cpp get the same bits.  inv_rigid and rt_to_T also serve vo_init_batch.cu, which
// is compiled without contraction and so gets the host's bits as well.
#if defined(__CUDACC__)
#define MVO_HD __host__ __device__
#else
#define MVO_HD
#endif
// What 0 / 0 (and every NaN made from finite inputs) is on x86-64: the default NaN, sign bit set.  The device makes NaNs with other
// bits; the kernels that restate host arithmetic (two_view_batch.cu, vo_init_batch.cu) write the host's into their double outputs.
static inline MVO_HD double as_host_nan(double v) {
  if (v == v) return v;
  const unsigned long long bits = 0xFFF8000000000000ull;
  double d;
  memcpy(&d, &bits, sizeof d);
  return d;
}
static inline void set_identity(double *T) { memset(T, 0, 16 * sizeof(double)); T[0] = T[5] = T[10] = T[15] = 1; }
static inline MVO_HD void inv_rigid(const double *T, double *Ti) {        // [R t; 0 1]^-1 = [R^T, -R^T t]; Ti may be T
  double r[16];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r[i * 4 + j] = T[j * 4 + i];
  for (int i = 0; i < 3; ++i) r[i * 4 + 3] = -(r[i * 4] * T[3] + r[i * 4 + 1] * T[7] + r[i * 4 + 2] * T[11]);
  r[12] = r[13] = r[14] = 0; r[15] = 1;
  memcpy(Ti, r, sizeof r);
}
static inline MVO_HD void inv_rt(double *R, double *t) {                 // basics::invRt on a row-major R and t: R^T, -R^T t in place
  double Rt[9], tt[3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = R[j * 3 + i];
  for (int i = 0; i < 3; ++i) tt[i] = -(Rt[i * 3] * t[0] + Rt[i * 3 + 1] * t[1] + Rt[i * 3 + 2] * t[2]);
  for (int q = 0; q < 9; ++q) R[q] = Rt[q];
  for (int q = 0; q < 3; ++q) t[q] = tt[q];
}
static inline MVO_HD void rt_to_T(const double *R, const double *t, double *T) {      // basics::convertRt2T
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) T[i * 4 + j] = R[i * 3 + j]; T[i * 4 + 3] = t[i]; }
  T[12] = T[13] = T[14] = 0; T[15] = 1;
}
// basics::preTranslatePoint3f: T(row, j) * p[j] accumulated in double over j = 0..3, narrowed to Point3f
static inline void pre_translate(const float *p, const double *T, float *out) {
  const double p0 = p[0], p1 = p[1], p2 = p[2];
  for (int r = 0; r < 3; ++r) {
    double a = 0;
    a += T[r * 4] * p0; a += T[r * 4 + 1] * p1; a += T[r * 4 + 2] * p2; a += T[r * 4 + 3] * 1.0;
    out[r] = (float)a;
  }
}
static inline double trans_dist(const double *Ta, const double *Tb) {
  const double dx = Ta[3] - Tb[3], dy = Ta[7] - Tb[7], dz = Ta[11] - Tb[11];
  return sqrt(dx * dx + dy * dy + dz * dz);
}

// The tracker's device-resident frame buffer as the pose-only LM sees it (ba.cu: k_ba_pose<.., STORE>).
// A buffered frame lives in one ring slot: its world->camera pose, its observation list (map point index +
// pixel, in PnP-inlier order = Frame::inliers_to_mappt_connections_) and the length of that list.
struct MvoPoseStore {
  const float *map_pts;        // [n_ids][3] MapPoint::pos_, indexed by map point ID
  const uint8_t *alive;        // [n_ids] 0 = the point has left the map: its observations are dropped (vo.cpp:438-440)
  int n_ids;                   // ids >= n_ids are dropped as well
  const int32_t *edge_map;     // [ring][cap] map point id
  const float2 *edge_obs;      // [ring][cap]
  const int32_t *cnt;          // [ring]
  double *pose;                // [ring][12] R row-major, t (world->camera)
  int cap, nslots, min_links;
  int slot[16];                // the window, newest first
  const int32_t *skip_flag;    // device flag: != 0 -> the kernel does nothing (PnP failed)
  int32_t *out_info;           // MvoTrackResultBlock::ba_graph
};

// The match filter's record (MvoTrackFilter::d_info, MvoTrackResultBlock::filter): pairs in the filtered list, map points in view, status
// (0 ok, 1 the host filter has to redo the frame), then MVO_TRACK_DEBUG counters: segments heapsorted at the depth limit, cycles of the
// prologue / quicksort levels / epilogue, the longest heapsorted segment, the levels, and cycles / segments of level l < 7 at FI_LEVEL + 2 l
enum MvoFilterInfo { FI_PAIRS, FI_CANDIDATES, FI_STATUS, FI_HEAP_SEGS, FI_CYC_PROLOGUE, FI_CYC_SORT, FI_CYC_EPILOGUE, FI_HEAP_MAX,
                     FI_LEVELS, FI_LEVEL, FI_COUNT = 24 };

// The device-resident tracker's per-frame result block: written by the kernels of a tracked frame, read back in one copy.
// The offsets are fixed: bench.py counts these 768 bytes in a tracked frame's device-to-host traffic.
struct MvoTrackResultBlock {
  int32_t ba_skip;               // != 0: the window BA does nothing (PnP failed, or BA is off)
  int32_t pad0[7];
  int32_t pnp[3];                // model found, pnp_ok, consensus-set size
  int32_t pad1[5];
  int32_t ba_graph[18];          // frames in the graph (0 = skipped, < 0 = too large), edges, [2 + f] slot of frame f
  int32_t pad2[6];
  int32_t filter[FI_COUNT];      // MvoFilterInfo
  double pose_before_ba[12];     // world->camera [R | t] of the frame before BA
  double pad3[20];
  double ba_stats[16];           // d_stats of mvo_ba_pose_store_launch
  double pad4[16];
};
static_assert(offsetof(MvoTrackResultBlock, ba_skip) == 0, "result block layout");
static_assert(offsetof(MvoTrackResultBlock, pnp) == 32, "result block layout");
static_assert(offsetof(MvoTrackResultBlock, ba_graph) == 64, "result block layout");
static_assert(offsetof(MvoTrackResultBlock, filter) == 160, "result block layout");
static_assert(offsetof(MvoTrackResultBlock, pose_before_ba) == 256, "result block layout");
static_assert(offsetof(MvoTrackResultBlock, ba_stats) == 512, "result block layout");
static_assert(sizeof(MvoTrackResultBlock) == 768, "result block layout");

// track.cu: k_track_glue's argument, passed by value (the field order and types are the kernel's parameter layout)
struct MvoTrackGlue {
  int mode;                 // 1: a PnP ran (pose_io / out_i / inl valid); 0: too few pairs, only the fallback applies;
                            // 2: a PnP was enqueued for *n_pairs_dev pairs — it counts only if that is >= min_pnp
  int min_pnp;
  const int32_t *n_pairs_dev;
  int slot, cap, ba_enable, has_prev;
  double max_dist;          // max_possible_dist_to_prev_keyframe
  double prev_twc[3];       // translation of the previous frame's T_w_c
  double fallback[12];      // world->camera [R | t] the frame keeps when PnP fails (vo.cpp:376-379)
  const double *pose_io;
  const int32_t *out_i, *inl;
  const int2 *pairs;
  const mvo_keypoint *kpts;
  int32_t *edge_map;        // [ring][cap] map point ids
  float2 *edge_obs;
  int32_t *edge_kp;         // [ring][cap] keypoint index of every connection (the key of inliers_to_mappt_connections_)
  const int32_t *map_ids;   // position in the map arrays -> map point id (what the frame buffer stores)
  // MapPoint::visible_times_ / matched_times_ increments (vo.cpp:44, :347), per position in the map arrays; nullptr = not counted
  const uint8_t *vis;       // in-view flags of this frame
  int nmap;
  int32_t *vis_cnt, *match_cnt;
  int32_t *cnt;             // [ring]
  double *pose;             // [ring][12]
  int32_t *skip_flag, *res_i;  // MvoTrackResultBlock::ba_skip, ::pnp
  double *res_d;               // MvoTrackResultBlock::pose_before_ba
};
int mvo_track_project_map(mvo_ctx *ctx, const float *d_map_pts, int nmap, const double *Tcw12, const double *K,
                          int rows, int cols, uint8_t *d_vis, float *d_cxy);
int mvo_track_kpt_xy(mvo_ctx *ctx, const mvo_keypoint *d_kpts, int n, float *d_xy);
// gather of several device arrays into one staging buffer (track.cu: k_pack_segments); lengths and offsets in 32-bit words
#define MVO_PACK_SEGS 8
struct MvoPackSegs {
  int n;
  const uint32_t *src[MVO_PACK_SEGS];
  uint32_t first[MVO_PACK_SEGS + 1];       // running start of segment s in the concatenated index space; first[n] = total words
  uint32_t dst_word[MVO_PACK_SEGS];        // where segment s starts in the destination
  uint8_t zero_after[MVO_PACK_SEGS];       // clear the source behind the copy
};
int mvo_track_pack_segments(mvo_ctx *ctx, const MvoPackSegs &segs, uint32_t *d_dst);
int mvo_track_kpt_colors(mvo_ctx *ctx, const mvo_keypoint *d_kpts, int n, const uint8_t *d_image, int channels, size_t stride, uint8_t *d_rgb);
int mvo_track_gather_pairs(mvo_ctx *ctx, const int32_t *d_pairs, int n, const int32_t *d_n, const float *d_map_pts,
                           const mvo_keypoint *d_kpts, float *d_p3, float *d_p2);
int mvo_track_glue(mvo_ctx *ctx, const MvoTrackGlue &g);
// thresholds of matchFeatures + removeDuplicatedMatches on the device; d_info: the FI_COUNT ints of MvoFilterInfo
struct MvoTrackFilter {
  const uint32_t *d_keys;        // matcher keys of ALL map points
  uint8_t *d_vis;                // in-view flags: read, or written when Tcw12 != nullptr (projection done by the filter)
  int nmap, nk, method;
  int32_t *d_pairs, *d_info;
  const double *Tcw12, *K;       // optional projection (methods 1/2)
  const double *d_Tcw12;         // ... with the pose in device memory instead (K, rows, cols as above)
  int rows, cols;
  const float *d_map_pts;
  const mvo_keypoint *d_kpts;    // optional: write the PnP input arrays (d_p3, d_p2) as well
  float *d_p3, *d_p2;
};
int mvo_track_match_filter(mvo_ctx *ctx, const MvoTrackFilter &f);

// tracker.cpp: what the state machine (vo_pipeline.cpp) needs from the device-resident tracker beyond mvo.h
int mvo_trk_device_mode(const mvo_tracker *t);
void mvo_trk_configure(mvo_tracker *t, int external_ref, int count_stats);
int mvo_trk_acquire(mvo_tracker *t, const uint8_t *image, int channels, size_t stride, int image_on_device, int *slot, int *nk);
void mvo_trk_release(mvo_tracker *t, int slot);
int mvo_trk_fetch(mvo_tracker *t, int slot, mvo_keypoint *kpts, uint8_t *desc, uint8_t *rgb);
const uint8_t *mvo_trk_desc_dev(mvo_tracker *t, int slot);
unsigned mvo_trk_slot_serial(const mvo_tracker *t, int slot);
int mvo_trk_set_map_ids(mvo_tracker *t, const float *pts3d, const uint8_t *desc, const int32_t *ids, int n, int reset_ids);
int mvo_trk_push_frame(mvo_tracker *t, const double *T_w_c, const int32_t *ids, const int32_t *kp_idx, const float *obs_xy, int n);
int mvo_trk_append_links(mvo_tracker *t, int k, const int32_t *ids, const int32_t *kp_idx, const float *obs_xy, int n);
int mvo_trk_links(mvo_tracker *t, int k, int32_t *ids, int32_t *kp_idx, int cap, int *n);
// keyframe insertion in one submission / one synchronisation (tracker.cpp); the pointers address the context's pinned staging
// buffer and stay valid until the next fetch
struct MvoKfFetch {
  int n_kpts;
  const mvo_keypoint *kpts; const uint8_t *desc, *rgb;          // rgb: null unless asked for
  const int32_t *link_ids, *link_kp; int n_links;              // inliers_to_mappt_connections_ of the frame, insertion order
  const int32_t *vis, *matched; int n_counters;                // visible / matched increments per map position
  const uint32_t *keys; int n_ref;                             // matcher keys reference keyframe x this frame; n_ref = 0: not available
};
int mvo_trk_keyframe_fetch(mvo_tracker *t, int slot, int want_rgb, int with_links, int n_counters, int ref_tag, int match_mode, MvoKfFetch *out);
int mvo_trk_set_ref_desc(mvo_tracker *t, int slot, int tag);
// ref_k: the reference keyframe whose pose T_guess is = the ref_k-th newest buffered frame counting the frame being tracked as 0
// (-1: not in the buffer); allow_spec: the head of the NEXT prefetched frame's chain (match filter + PnP) may be enqueued ahead of time
int mvo_trk_track(mvo_tracker *t, int slot, const double *T_guess, const double *T_prev, double *T_w_c_out, mvo_track_result *res, int ref_k,
                  int allow_spec);

void orb_state_free(mvo_ctx *ctx);   // orb_host.cpp
void orb_tma_free(mvo_ctx *ctx);     // orb.cu
// mvo_orb_extract with the image optionally already resident on the device (orb_host.cpp)
int mvo_orb_extract_ex(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride,
                       int on_device, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc);

// asynchronous extraction (orb_host.cpp): begin enqueues on ctx->stream and returns; end waits, finishes the
// rare host retainBest path and copies out; *d_desc = descriptors on the device (valid until the next begin)
int mvo_orb_extract_begin(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride, int on_device);
int mvo_orb_extract_end(mvo_ctx *ctx, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc, const uint8_t **d_desc);
// the same with keypoints and descriptors left on the device (valid until the next begin on this context)
int mvo_orb_extract_begin_dev(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride, int on_device);
int mvo_orb_extract_end_dev(mvo_ctx *ctx, int *n_kpts, const mvo_keypoint **d_kpts, const uint8_t **d_desc);
// between the two: the buffers being filled and the device address of the keypoint count (orb_host.cpp)
int mvo_orb_extract_peek_dev(mvo_ctx *ctx, const mvo_keypoint **d_kpts, const uint8_t **d_desc, const int32_t **d_count, int *n_max);
int mvo_orb_extract_used_host_path(mvo_ctx *ctx);
// mvo_match_features with the train descriptors optionally already on the device (match_host.cpp)
int mvo_match_features_ex(mvo_ctx *ctx, const uint8_t *d1, int n1, const uint8_t *d2, int n2, int d2_on_device,
                          int method_index, const float *xy1, const float *xy2, float radius, mvo_dmatch *out, int *n_out);
// the thresholds + removeDuplicatedMatches tail of matchFeatures over packed matcher keys (match_host.cpp)
int mvo_match_filter_keys(mvo_ctx *ctx, int method_index, const uint32_t *keys, int n1, mvo_dmatch *out, int *n_out);
// estiMotionByEssential with the keyframe branch's options: no recoverPose vote, triangulation of all correspondences in the same
// submission (epipolar.cu)
// the same, and estiMotionByHomography, split at the synchronisation: _begin enqueues everything on ctx->stream (which the caller may
// point at ctx's side stream for the duration of the call), _end waits for that stream and post-processes.  Both jobs are a batch of
// one laid out like the batch calls' rows (epipolar.cu), each in its own buffers (epi_ess_* and epi_homo_*), so the initialisation
// runs them side by side (two_view.cpp).  h_out / h_oi: the finish outputs (EPIB_OUT_D doubles, EPIB_OUT_I ints) copied back.
struct MvoEpiJob {
  cudaStream_t stream; int n, H; bool want_pose, tri; double thr2, f;
  double *h_out; int32_t *h_oi, *h_inl; float *h_tri;
  cudaStream_t tri_stream;                    // where the fused triangulation runs (the context's side stream when there is one)
  const void *d_valid, *d_cnt, *d_model;      // MVO_EPI_DEBUG
};
int mvo_epi_essential_begin(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold, int want_pose,
                            const float *tri_np1, const float *tri_np2, const double *tri_R, const double *tri_t, bool tri, MvoEpiJob *job);
int mvo_epi_essential_end(mvo_ctx *ctx, MvoEpiJob *job, double *E, double *R, double *t, int32_t *inliers, int *n_inliers, float *tri_out);
int mvo_epi_homography_begin(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold, MvoEpiJob *job);
int mvo_epi_homography_end(mvo_ctx *ctx, MvoEpiJob *job, const double *K, double *Hout, double *Rs, double *ts, double *normals, int *n_solutions,
                           int32_t *inliers, int *n_inliers);
int mvo_do_triangulation_multi(mvo_ctx *ctx, const float *pts_np1, const float *pts_np2, int n, int nsol, const double *const *R,
                               const double *const *t, const int32_t *const *inliers, const int *n_inliers, float *const *pts3d);
// mvo_estimate_relative_poses_batch_dev (epipolar.cu) in three steps: the RANSAC halves (epipolar.cu), the combine step
// (two_view_batch.cu: one launch, one CTA per pair), the triangulation of every solution (epipolar.cu).  MvoRelPosesCombine holds
// what the first step leaves on the device for the others: the outputs of the essential half (ess, inl_e: pair p's list at
// p * cap) and of the homography half (hom_d / hom_i: the finish outputs at p * hom_d_stride / p * hom_i_stride, inl_h), the
// gathered pixel (p1, p2) and normalised-plane (np1, np2) points.  The combine step writes res, the inlier rows and rt: (R | t) of
// every solution before basics::invRt, 12 doubles at (p * 5 + s) * 12, which the triangulation reads.
struct MvoRelPosesCombine {
  const int32_t *n_matches;
  const mvo_two_view_result *ess;
  const int32_t *inl_e, *hom_i, *inl_h;
  const double *hom_d;
  const float *p1, *p2, *np1, *np2;
  int n_pairs, cap, hom_d_stride, hom_i_stride, motion_cam2_to_cam1;
  double K[9], eh_ratio_threshold;
  mvo_relative_poses_result *res;
  int32_t *inliers;
  double *rt;
};
// mvo_vo_init_candidates_batch_dev (vo_pipeline.cpp checks the arguments, vo_init_batch.cu launches one CTA per pair): the inputs
// as the call received them, T_w_c_ref and the thresholds by value
struct MvoInitCandidates {
  const mvo_keypoint *kpts;
  const int32_t *counts, *pairs, *n_matches, *rp_inliers;
  const mvo_dmatch *matches;
  const mvo_relative_poses_result *rp;
  const float *rp_pts3d;
  int batch, cap, n_pairs, min_inlier_matches;
  double T_ref[16];
  double min_triang_angle, max_ratio_angle_to_median, min_pixel_dist, min_median_triangulation_angle, assumed_mean_depth_init;
  mvo_init_candidate_result *out;
  mvo_dmatch *kept;
  float *kept_pts3d;
  double *kept_angles;
};
int mvo_vo_init_candidates_launch(mvo_ctx *ctx, const MvoInitCandidates &a);
cudaStream_t mvo_side_stream(mvo_ctx *ctx);      // a second non-blocking stream of the context, created on first use (ctx.cu)
int mvo_epi_essential_ex(mvo_ctx *ctx, const float *pts1, const float *pts2, int n, const double *K, double threshold,
                         double *E, double *R, double *t, int32_t *inliers, int *n_inliers, int want_pose,
                         const float *tri_np1, const float *tri_np2, const double *tri_R, const double *tri_t, float *tri_out);

// ---- stage entry points (host-side launchers, all asynchronous on ctx->stream) -----------
// match.cu
int mvo_match_launch(mvo_ctx *ctx, int mode, const uint8_t *d_d1, const float *d_xy1, int n1,
                     const uint8_t *d_d2, const float *d_xy2, int n2, float radius,
                     uint32_t *d_keys);
int mvo_match_launch_masked(mvo_ctx *ctx, int mode, const uint8_t *d_d1, const float *d_xy1, int n1,
                            const uint8_t *d_d2, const float *d_xy2, int n2, float radius,
                            uint32_t *d_keys, const uint8_t *d_qmask);
// the train count on the device (d_n2; n2 = its upper bound, for which the grid is sized)
int mvo_match_launch_ndev(mvo_ctx *ctx, int mode, const uint8_t *d_d1, const float *d_xy1, int n1,
                          const uint8_t *d_d2, const float *d_xy2, int n2, const int32_t *d_n2, float radius,
                          uint32_t *d_keys, const uint8_t *d_qmask);
// the same over n_pairs frame pairs of a batched extraction (layout of mvo_orb_extract_batch_dev, counts read on the device);
// d_keys: [n_pairs][cap][W] packed keys, W = 2 for mode 1.  Pairs with an out-of-range frame are skipped
int mvo_match_batch_launch(mvo_ctx *ctx, int mode, const mvo_keypoint *d_kpts, const uint8_t *d_desc, const int32_t *d_counts,
                           int batch, int cap, const int32_t *d_pairs, int n_pairs, float radius, uint32_t *d_keys);
// pnp.cu: device-resident solvePnPRansac replacement (see there)
int mvo_pnp_dev_buffers(mvo_ctx *ctx, int n, float **p3, float **p2, double **pose_io, int32_t **out_i, int32_t **inl);
int mvo_pnp_dev_run(mvo_ctx *ctx, int n, const double *K, const int32_t *d_n);
// ba.cu: pose-only LM over the tracker's device-resident frame buffer
int mvo_ba_pose_store_launch(mvo_ctx *ctx, const MvoPoseStore &st, int e_upper, double fx, double fy, double cx, double cy,
                             const double *info, int iters, int use_huber, double huber, double step_tol, double *d_stats);
