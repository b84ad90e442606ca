// Per-frame tracking step over flat arrays: the DOING_TRACKING branch of
// vo::VisualOdometry::addFrame (reference src/vo/vo_addFrame.cpp:71-91) with its callees
// getMappointsInCurrentView_ (src/vo/vo.cpp:16-49), poseEstimationPnP_ (:267-381) and
// callBundleAdjustment_ (:384-478).  Host logic in C++ like the reference; every numeric stage
// runs on the GPU (no CPU fallback anywhere).
//
// Two implementations of the same step, selected by mvo_track_params::device_resident:
//   * device-resident (default, shipped configuration = fixed map points): the map (points + descriptors),
//     the frame buffer (pose + inlier connections of the newest kBuffSize_ frames) and the BA graph live in
//     HBM.  Per frame the host synchronises ONCE, at the end of the frame (result block and pose ring, ~3 KB): the
//     reference's duplicate removal — an unstable libstdc++ std::sort — is restated on the device (track_filter.cuh;
//     the host variant remains for the inputs on which libstdc++ would leave quicksort).  Everything is launched back
//     to back on one stream with programmatic dependent launch, and the head of the NEXT frame's chain (match filter +
//     PnP) is enqueued behind the current frame's bundle adjustment when that frame has been prefetched.
//   * host-array: every stage through its public C-ABI entry point (mvo_match_features, mvo_solve_pnp_ransac,
//     mvo_bundle_adjustment), as a maintainer who only swaps the bodies of the reference functions gets it.
// ORB extraction does not depend on the VO state (SURVEY.md §8e): three extraction slots, each with its own context
// (stream + workspace) and worker thread, run the prefetched frames i+1 and i+2 — upload, kernels, the pre-match against
// the map, the rare host retainBest path — while frame i (which holds the third slot) is tracked.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <stdlib.h>
#include <math.h>
#include <string.h>
#include <thread>
#include <vector>
#include "mvo_internal.h"

namespace {

struct TrackedFrame {
  double T_w_c[16];
  // inliers_to_mappt_connections_: keypoint pixel + map point index, in insertion order (host-array path)
  std::vector<float> obs_xy;
  std::vector<int32_t> map_idx;
  // device-resident path: the same list lives in ring slot `slot` of the device frame buffer
  int slot = -1;
  int n_links = 0;
};

// One extraction in flight per slot, each slot with its own worker thread, context and stream.
// Extraction slots (contexts, streams, worker threads): the frame being added holds one while two prefetched frames are extracted.
constexpr int MVO_XSLOTS = 3;

struct ExtractJob {
  std::atomic<int> state{0};           // 0 free, 1 queued, 2 done
  const uint8_t *image = nullptr;
  int channels = 0, on_device = 0;
  size_t stride = 0;
  bool want_host = false;
  // methods 1/2: the matcher does not depend on the pose, so the worker runs it right after the extraction
  bool prematch = false, matched = false;
  int match_mode = 0, map_version = 0;
  unsigned serial = 0;                 // submission number: tells whether the slot still holds a given frame
  // snapshot taken at submission (the API thread may replace the map while the job runs; a stale match is redone)
  const uint8_t *d_map_desc = nullptr;
  uint32_t *d_keys = nullptr;
  int nmap = 0;
  int rc = MVO_OK, nk = 0;
  const mvo_keypoint *d_k = nullptr;
  const uint8_t *d_d = nullptr;
  std::vector<mvo_keypoint> kpts;      // want_host only
  std::vector<uint8_t> desc;
};

void inv_rigid(const double *T, double *Ti) {     // [R t; 0 1]^-1 = [R^T, -R^T t]
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Ti[i * 4 + j] = T[j * 4 + i];
    Ti[i * 4 + 3] = -(T[0 * 4 + i] * T[3] + T[1 * 4 + i] * T[7] + T[2 * 4 + i] * T[11]);
  }
  Ti[12] = Ti[13] = Ti[14] = 0;
  Ti[15] = 1;
}

// camera->world 4x4  ->  world->camera [R (9) | t (3)], and back (g2o_ba.cpp:183-190, :298-305)
void Twc_to_Rt12(const double *T, double *q) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) q[i * 3 + j] = T[j * 4 + i];
    q[9 + i] = -(T[0 * 4 + i] * T[3] + T[1 * 4 + i] * T[7] + T[2 * 4 + i] * T[11]);
  }
}
void Rt12_to_Twc(const double *p, double *T) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[i * 4 + j] = p[j * 3 + i];
    T[i * 4 + 3] = -(p[i] * p[9] + p[3 + i] * p[10] + p[6 + i] * p[11]);
  }
  T[12] = T[13] = T[14] = 0;
  T[15] = 1;
}

void rvec_to_R(const double *w, double *R) {      // cv::Rodrigues
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double A, B;
  if (th < 1e-12) { A = 1; B = 0.5; }
  else { A = sin(th) / th; B = (1 - cos(th)) / th2; }
  const double x = w[0], y = w[1], z = w[2];
  R[0] = 1 - B * (y * y + z * z); R[1] = -A * z + B * x * y;      R[2] = A * y + B * x * z;
  R[3] = A * z + B * x * y;       R[4] = 1 - B * (x * x + z * z); R[5] = -A * x + B * y * z;
  R[6] = -A * y + B * x * z;      R[7] = A * x + B * y * z;       R[8] = 1 - B * (x * x + y * y);
}

double trans_dist(const double *Ta, const double *Tb) {
  const double dx = Ta[3] - Tb[3], dy = Ta[7] - Tb[7], dz = Ta[11] - Tb[11];
  return sqrt(dx * dx + dy * dy + dz * dz);
}

double now_us() { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct MatchPair { int32_t train, map; };   // proxy record for removeDuplicatedMatches (see dedup_pairs)

}  // namespace

struct mvo_tracker {
  mvo_ctx *ctx = nullptr;
  double K[9];
  int rows = 0, cols = 0;
  mvo_track_params prm;
  // The map as the caller handed it over: n points in HIS order (the reference walks std::unordered_map<int, MapPoint::Ptr>
  // in container order, vo.cpp:25) with their stable ids.  Buffered frames refer to map points by ID.
  std::vector<float> map_pts;        // n x 3
  std::vector<uint8_t> map_desc;     // n x 32
  std::vector<int32_t> map_ids;      // n
  std::vector<float> pos_by_id;      // n_ids x 3
  std::vector<uint8_t> alive;        // n_ids: 1 = the id is in the current map
  bool external_ref = false;         // the caller (mvo_vo) supplies the guess / previous pose of every frame
  std::deque<TrackedFrame> frames;   // frames_buff_ (oldest first)
  double T_ref[16];                  // reference keyframe pose (initial guess for the next frame)
  bool has_prev = false;
  double T_prev[16];
  unsigned frame_counter = 0;
  int fused_holdoff = 0;             // frames left before the device-side match filter is tried again
  // scratch (host-array path)
  std::vector<uint8_t> cand_desc;
  std::vector<float> cand_xy, kp_xy, p3, p2;
  std::vector<int32_t> cand_idx, inliers;
  std::vector<mvo_dmatch> matches;
  std::vector<double> ba_poses;
  std::vector<int> ba_which;
  std::vector<int32_t> ba_ef, ba_ep, ba_used, ba_remap, ba_stamp;
  std::vector<float> ba_ob, ba_pts;
  int32_t ba_gen = 0;
  std::vector<MatchPair> pairs;      // device-resident path
  // extraction worker
  mvo_ctx *xctx[MVO_XSLOTS] = {nullptr, nullptr, nullptr};
  ExtractJob job[MVO_XSLOTS];
  bool held = false;                 // an acquired slot has not been released yet
  unsigned n_submit = 0, n_consume = 0, n_submit_total = 0;
  std::thread worker[MVO_XSLOTS];    // one per extraction slot / context: prefetched frames are extracted side by side
  std::mutex mu;
  std::condition_variable cv_job, cv_done;
  bool stop = false;
  unsigned n_run = 0;                // worker-side cursor
  // device-resident state: three allocations (map arrays by position, by-id arrays, frame ring), each grown by doubling
  uint8_t *dev = nullptr, *dev_map = nullptr, *dev_ids = nullptr;
  int dev_nmap = -1;                   // points in the device copy of the map; -1 = stale (refreshed by the next frame)
  int dev_mcap = 0, dev_idcap = 0, dev_cap = 0, dev_ring = 0;
  float *d_map_pts = nullptr;  uint8_t *d_map_desc = nullptr;
  int32_t *d_map_ids = nullptr, *d_vis_cnt = nullptr, *d_match_cnt = nullptr, *d_edge_kp = nullptr;
  float *d_pos_by_id = nullptr;  uint8_t *d_alive = nullptr;
  bool count_stats = false;            // accumulate visible / matched counts per map point on the device
  uint8_t *d_keysvis[MVO_XSLOTS] = {nullptr, nullptr, nullptr};   // per extraction slot: [keys nmap*2 u32][vis nmap u8] — one D2H after the match
  int map_version = 0;                 // bumped by set_map: keys matched ahead of time against an older map are redone
  float *d_cxy = nullptr, *d_kxy = nullptr;
  int32_t *d_pairs = nullptr, *d_edge_map = nullptr, *d_cnt = nullptr, *d_flags = nullptr;
  float *d_edge_obs = nullptr;
  double *d_pose = nullptr, *d_res = nullptr, *d_stats = nullptr;
  uint8_t *h_pin = nullptr;            // pinned staging: [keys+vis][pairs][results]
  size_t h_pin_bytes = 0;
  // descriptors of the reference keyframe (mvo_vo: ref_), kept on the device so that a keyframe insertion matches against them
  // without an upload (mvo_trk_set_ref_desc / mvo_trk_keyframe_fetch)
  uint8_t *d_ref_desc = nullptr;
  int n_ref = 0, ref_tag = -1;
  bool ref_copy_pending = false;       // a device-to-device copy out of an extraction slot is in flight: synchronise before the slot is released
  // Speculative head of the next frame's chain.  The match filter and the PnP kernels of frame i + 1 only read the map, the keys the
  // extraction worker left and the reference keyframe's pose, and only write scratch buffers: when frame i + 1 has been prefetched,
  // they are enqueued right behind frame i's bundle adjustment (guess pose read from the device-side pose ring), so the GPU works
  // on them while the host waits for frame i's results, decides about a keyframe and comes back with frame i + 1.  If anything they
  // depended on changed in between (a keyframe replaced the map, another reference keyframe, a declined filter) they are redone.
  struct Spec { bool valid = false; unsigned serial = 0; int map_version = 0, ref_slot = -1, nmap = 0, nk = 0, method = 0, n_upper = 0; } spec;
  std::vector<double> ring_host;       // host mirror of the pose ring (world->camera [R|t] per slot), refreshed with every frame's read-back
  cudaEvent_t ev_result = nullptr;     // recorded behind the device-to-host copy of a frame's result block
  uint64_t spec_hits = 0, spec_issued = 0;
};

namespace {

void worker_main(mvo_tracker *t, int slot) {
  for (;;) {
    ExtractJob *j = nullptr;
    {
      std::unique_lock<std::mutex> lk(t->mu);
      t->cv_job.wait(lk, [&] { return t->stop || t->job[slot].state.load(std::memory_order_acquire) == 1; });
      if (t->stop) return;
      j = &t->job[slot];
    }
    mvo_ctx *x = t->xctx[slot];
    int rc, nk = 0;
    static const bool dbg_worker = getenv("MVO_TRACK_DEBUG") != nullptr;
    const double tw0 = dbg_worker ? now_us() : 0;
    double tw1 = 0;
    if (j->want_host) {
      const int cap = x->prm.max_keypoints + 1;
      j->kpts.resize(cap);
      j->desc.resize((size_t)cap * 32);
      nk = cap;
      rc = mvo_orb_extract_begin(x, j->image, t->rows, t->cols, j->channels, j->stride, j->on_device);
      if (rc == MVO_OK) rc = mvo_orb_extract_end(x, j->kpts.data(), &nk, j->desc.data(), &j->d_d);
    } else {
      rc = mvo_orb_extract_begin_dev(x, j->image, t->rows, t->cols, j->channels, j->stride, j->on_device);
      j->matched = false;
      // All map descriptors x this frame's descriptors on the extraction stream, off the tracking chain — queued right behind
      // the describe kernel: the keypoint count is read on the device (its upper bound sizes the grid), so the extraction
      // chain of a frame is one submission and one synchronisation.
      bool queued = false;
      const bool want_match = j->prematch && j->nmap > 0;
      if (rc == MVO_OK && want_match) {
        const uint8_t *dd = nullptr;
        const int32_t *dn = nullptr;
        int n_max = 0;
        rc = mvo_orb_extract_peek_dev(x, nullptr, &dd, &dn, &n_max);
        if (rc == MVO_OK && n_max >= 2) {
          rc = mvo_match_launch_ndev(x, j->match_mode, j->d_map_desc, nullptr, j->nmap, dd, nullptr, n_max, dn, 0.f, j->d_keys, nullptr);
          queued = rc == MVO_OK;
        }
      }
      if (dbg_worker) tw1 = now_us();
      if (rc == MVO_OK) rc = mvo_orb_extract_end_dev(x, &nk, &j->d_k, &j->d_d);
      if (rc == MVO_OK && want_match && nk > 0 && !(j->match_mode == 1 && nk < 2)) {
        if (!queued || mvo_orb_extract_used_host_path(x))        // the host retainBest path replaced the keypoints: match again
          rc = mvo_match_launch_masked(x, j->match_mode, j->d_map_desc, nullptr, j->nmap, j->d_d, nullptr, nk, 0.f, j->d_keys, nullptr);
        if (rc == MVO_OK && cudaStreamSynchronize(x->stream) != cudaSuccess) rc = MVO_ERR_CUDA;
        j->matched = rc == MVO_OK;
      } else if (rc == MVO_OK && queued) {
        if (cudaStreamSynchronize(x->stream) != cudaSuccess) rc = MVO_ERR_CUDA;      // the queued kernel must not outlive the job
      }
    }
    j->rc = rc;
    j->nk = nk;
    if (dbg_worker && slot == 0) {       // how long the extraction chain of one frame takes on a worker (enqueue / until everything has run)
      static double acc_enq = 0, acc_all = 0;
      static int n_w = 0;
      const double t_end = now_us();
      acc_enq += tw1 - tw0; acc_all += t_end - tw0;
      if (++n_w % 50 == 0) { fprintf(stderr, "extraction worker: %.1f us/frame from job start to done (kernels enqueued after %.1f us)\n", acc_all / 50, acc_enq / 50); acc_enq = acc_all = 0; }
    }
    {
      std::lock_guard<std::mutex> lk(t->mu);
      ++t->n_run;
      j->state.store(2, std::memory_order_release);
    }
    t->cv_done.notify_all();
  }
}

// wait for the extraction in `slot`; spins briefly (the usual case: already done) before sleeping
void wait_job(mvo_tracker *t, int slot) {
  ExtractJob &j = t->job[slot];
  for (int spin = 0; spin < 2000; ++spin)
    if (j.state.load(std::memory_order_acquire) == 2) return;
  std::unique_lock<std::mutex> lk(t->mu);
  t->cv_done.wait(lk, [&] { return j.state.load(std::memory_order_acquire) == 2; });
}

void drain_jobs(mvo_tracker *t) {
  while (t->n_consume != t->n_submit) {
    const int slot = (int)(t->n_consume % MVO_XSLOTS);
    wait_job(t, slot);
    t->job[slot].state.store(0, std::memory_order_release);
    ++t->n_consume;
  }
}

// The device-resident path covers the shipped configuration (fixed map points) as long as the BA graph fits the
// shared-memory-cached pose kernel: window x (max_keypoints + 1) observations <= 4 per thread of the 8 x 512 cluster.
bool use_device_path(const mvo_tracker *t) {
  const long worst_edges = (long)std::min(t->prm.ba_window, t->prm.buffer_size) * (t->ctx->prm.max_keypoints + 1);
  return t->prm.device_resident && t->prm.ba_fix_points && worst_edges + 64 <= 4L * 8 * 512;
}

size_t al256(size_t v) { return (v + 255) & ~(size_t)255; }

// (Re)allocate / refresh the device-resident state.  Three blocks, each reallocated only when it has to grow (the map
// changes at every keyframe once mvo_vo drives the tracker): the frame ring (keypoint capacity x ring size; holds the
// buffered frames, so it is only rebuilt when those parameters change), the map arrays by position (capacity doubled on
// demand) and the by-id arrays (positions + alive flags the BA graph builder reads).  A stale device copy of the map
// (dev_nmap == -1) is re-uploaded here.
int dev_alloc(mvo_tracker *t) {
  mvo_ctx *ctx = t->ctx;
  const int nmap = (int)t->map_ids.size(), n_ids = (int)t->alive.size();
  const int cap = ctx->prm.max_keypoints + 1, ring = t->prm.buffer_size;
  const bool ring_ok = t->dev && cap == t->dev_cap && ring == t->dev_ring;
  const bool map_ok = t->dev_map && nmap <= t->dev_mcap, ids_ok = t->dev_ids && n_ids <= t->dev_idcap;
  if (ring_ok && map_ok && ids_ok && t->dev_nmap == nmap) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  // frames extracted (and matched) ahead of time hold pointers into the map arrays: let them finish first
  for (unsigned k = t->n_consume; k != t->n_submit; ++k) wait_job(t, (int)(k % MVO_XSLOTS));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (!ring_ok) {
    size_t o = 0;
    const size_t o_kxy = o;   o = al256(o + (size_t)cap * 8);
    const size_t o_emap = o;  o = al256(o + (size_t)ring * cap * 4);
    const size_t o_eobs = o;  o = al256(o + (size_t)ring * cap * 8);
    const size_t o_ekp = o;   o = al256(o + (size_t)ring * cap * 4);
    const size_t o_cnt = o;   o = al256(o + (size_t)ring * 4);
    const size_t o_pose = o;  o = al256(o + (size_t)ring * 96);
    const size_t o_flags = o; o = al256(o + 256);       // [0] BA skip flag, [8..] res_i (3), [16..] out_info (2 + 16)
    const size_t o_res = o;   o = al256(o + 256);       // res_d (12 doubles)
    const size_t o_stats = o; o = al256(o + 256);       // BA stats (16 doubles)
    const size_t o_ref = o;   o = al256(o + (size_t)cap * 32);
    uint8_t *nd = nullptr;
    MVO_CUDA(ctx, cudaMalloc(&nd, o));
    MVO_CUDA(ctx, cudaMemsetAsync(nd, 0, o, ctx->stream));
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (t->dev) cudaFree(t->dev);
    for (TrackedFrame &f : t->frames) f.slot = -1;      // frames buffered under the old layout leave the device-side BA window
    t->dev = nd; t->dev_cap = cap; t->dev_ring = ring;
    t->d_kxy = (float *)(nd + o_kxy); t->d_edge_map = (int32_t *)(nd + o_emap); t->d_edge_obs = (float *)(nd + o_eobs);
    t->d_edge_kp = (int32_t *)(nd + o_ekp); t->d_cnt = (int32_t *)(nd + o_cnt); t->d_pose = (double *)(nd + o_pose);
    t->d_flags = (int32_t *)(nd + o_flags); t->d_res = (double *)(nd + o_res); t->d_stats = (double *)(nd + o_stats);
    t->d_ref_desc = nd + o_ref; t->n_ref = 0; t->ref_tag = -1;
    t->ring_host.assign((size_t)ring * 12, 0.0);
    t->spec.valid = false;
  }
  if (!map_ok) {
    int mcap = std::max(t->dev_mcap, 1024);
    while (mcap < nmap) mcap *= 2;
    size_t o = 0;
    const size_t o_pts = o;   o = al256(o + (size_t)mcap * 12);
    const size_t o_desc = o;  o = al256(o + (size_t)mcap * 32);
    size_t o_kv[MVO_XSLOTS];
    for (int k = 0; k < MVO_XSLOTS; ++k) { o_kv[k] = o; o = al256(o + (size_t)mcap * 9); }
    const size_t o_cxy = o;   o = al256(o + (size_t)mcap * 8);
    const size_t o_pairs = o; o = al256(o + (size_t)mcap * 8);
    const size_t o_ids = o;   o = al256(o + (size_t)mcap * 4);
    const size_t o_vc = o;    o = al256(o + (size_t)mcap * 4);
    const size_t o_mc = o;    o = al256(o + (size_t)mcap * 4);
    uint8_t *nd = nullptr;
    MVO_CUDA(ctx, cudaMalloc(&nd, o));
    MVO_CUDA(ctx, cudaMemsetAsync(nd, 0, o, ctx->stream));
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (t->dev_map) cudaFree(t->dev_map);
    t->dev_map = nd; t->dev_mcap = mcap;
    t->d_map_pts = (float *)(nd + o_pts); t->d_map_desc = nd + o_desc;
    for (int k = 0; k < MVO_XSLOTS; ++k) t->d_keysvis[k] = nd + o_kv[k];
    t->d_cxy = (float *)(nd + o_cxy); t->d_pairs = (int32_t *)(nd + o_pairs); t->d_map_ids = (int32_t *)(nd + o_ids);
    t->d_vis_cnt = (int32_t *)(nd + o_vc); t->d_match_cnt = (int32_t *)(nd + o_mc);
    const size_t hb = al256((size_t)mcap * 9) + al256((size_t)mcap * 8 + 64) + al256((size_t)4096 * 96) + 1024;
    if (hb > t->h_pin_bytes) {
      if (t->h_pin) cudaFreeHost(t->h_pin);
      t->h_pin = nullptr;
      MVO_CUDA(ctx, cudaMallocHost(&t->h_pin, hb));
      t->h_pin_bytes = hb;
    }
  }
  if (!ids_ok) {
    int idcap = std::max(t->dev_idcap, 4096);
    while (idcap < n_ids) idcap *= 2;
    const size_t o_alive = al256((size_t)idcap * 12), tot = o_alive + al256((size_t)idcap);
    uint8_t *nd = nullptr;
    MVO_CUDA(ctx, cudaMalloc(&nd, tot));
    if (t->dev_ids) cudaFree(t->dev_ids);
    t->dev_ids = nd; t->dev_idcap = idcap;
    t->d_pos_by_id = (float *)nd; t->d_alive = nd + o_alive;
  }
  ++t->map_version;                 // keys matched ahead of time were computed against the previous device copy
  t->dev_nmap = nmap;
  if (nmap > 0) {
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_map_pts, t->map_pts.data(), (size_t)nmap * 12, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_map_desc, t->map_desc.data(), (size_t)nmap * 32, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_map_ids, t->map_ids.data(), (size_t)nmap * 4, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemsetAsync(t->d_vis_cnt, 0, (size_t)nmap * 4, ctx->stream));
    MVO_CUDA(ctx, cudaMemsetAsync(t->d_match_cnt, 0, (size_t)nmap * 4, ctx->stream));
  }
  if (n_ids > 0) {
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_pos_by_id, t->pos_by_id.data(), (size_t)n_ids * 12, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_alive, t->alive.data(), (size_t)n_ids, cudaMemcpyHostToDevice, ctx->stream));
  }
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));      // the extraction stream reads the map right away
  return MVO_OK;
}

// geometry::removeDuplicatedMatches (feature_match.cpp:241-260) on (train, map) records.  libstdc++'s std::sort
// decides from comparison results and element COUNTS only, so sorting these 8-byte records with the same
// comparator applies exactly the permutation it applies to the reference's cv::DMatch array
// (tests/test_capi_symbols.py::test_dedup_proxy_matches_dmatch_sort).
void dedup_pairs(std::vector<MatchPair> &v) {
  std::sort(v.begin(), v.end(), [](const MatchPair &a, const MatchPair &b) { return a.train < b.train; });
  size_t w = 0;
  for (size_t i = 0; i < v.size(); ++i)
    if (i == 0 || v[i].train != v[i - 1].train) v[w++] = v[i];
  v.resize(w);
}

// Thresholds of matchFeatures (feature_match.cpp:179-196 for methods 1/3, :210-217 for method 2) and
// removeDuplicatedMatches (:241-260) over the packed matcher keys of ALL map points (vis = in-view flags).
void host_match_filter(const mvo_params &prm, int method, bool can_match, const uint32_t *h_keys, const uint8_t *h_vis, int nmap,
                       std::vector<MatchPair> &pairs, int *ncand_out) {
  pairs.clear();
  int ncand = 0;
  for (int q = 0; q < nmap; ++q) ncand += h_vis[q] != 0;
  *ncand_out = ncand;
  if (!can_match || ncand == 0) return;
  if (method == 1 || method == 3) {
    const bool sad = method == 3;
    double min_dis = 9999999, max_dis = 0;
    for (int q = 0; q < nmap; ++q) {
      if (!h_vis[q] || h_keys[q] == 0xFFFFFFFFu) continue;
      const uint32_t d = h_keys[q] >> 16;
      const double dist = sad ? (double)(float)((double)d / 32.0) : (double)(float)d;
      if (dist < min_dis) min_dis = dist;
      if (dist > max_dis) max_dis = dist;
    }
    const double thr = std::max<float>(min_dis * prm.xiang_gao_ratio, 30.0);
    for (int q = 0; q < nmap; ++q) {
      if (!h_vis[q] || h_keys[q] == 0xFFFFFFFFu) continue;
      const uint32_t d = h_keys[q] >> 16;
      const float dist = sad ? (float)((double)d / 32.0) : (float)d;
      if (dist < thr) pairs.push_back(MatchPair{(int32_t)(h_keys[q] & 0xFFFFu), q});
    }
  } else {
    for (int q = 0; q < nmap; ++q) {
      if (!h_vis[q] || h_keys[2 * q] == 0xFFFFFFFFu) continue;
      const uint32_t k0 = h_keys[2 * q], k1 = h_keys[2 * q + 1];
      const double dist = (float)(k0 >> 16);
      if (dist < prm.lowe_ratio * (float)(k1 >> 16)) pairs.push_back(MatchPair{(int32_t)(k0 & 0xFFFFu), q});
    }
  }
  dedup_pairs(pairs);
}

}  // namespace

// exported for the CPU-side test of the proxy sort (not part of mvo.h: test hook)
extern "C" int mvo_test_dedup_pairs(int32_t *train, int32_t *map, int *n) {
  if (!train || !map || !n) return MVO_ERR_INVALID_ARG;
  std::vector<MatchPair> v(*n);
  for (int i = 0; i < *n; ++i) v[i] = MatchPair{train[i], map[i]};
  dedup_pairs(v);
  for (size_t i = 0; i < v.size(); ++i) { train[i] = v[i].train; map[i] = v[i].map; }
  *n = (int)v.size();
  return MVO_OK;
}


// Test hooks (not part of mvo.h): the match-list tail on the host and on the device, from the same packed keys.
// pairs: n x 2 int32 (map index, keypoint index); info: [0] pairs, [1] candidates, [2] status.
extern "C" int mvo_test_match_filter_host(mvo_ctx *ctx, const uint32_t *keys, const uint8_t *vis, int nmap, int nk, int method,
                                          int32_t *pairs, int32_t *info) {
  if (!ctx || !keys || !vis || !pairs || !info) return MVO_ERR_INVALID_ARG;
  std::vector<MatchPair> v;
  int ncand = 0;
  host_match_filter(ctx->prm, method, nk > 0, keys, vis, nmap, v, &ncand);
  for (size_t i = 0; i < v.size(); ++i) { pairs[2 * i] = v[i].map; pairs[2 * i + 1] = v[i].train; }
  info[0] = (int32_t)v.size(); info[1] = ncand; info[2] = 0;
  return MVO_OK;
}

extern "C" int mvo_test_match_filter_dev(mvo_ctx *ctx, const uint32_t *keys, const uint8_t *vis, int nmap, int nk, int method,
                                         int32_t *pairs, int32_t *info) {
  if (!ctx || !keys || !vis || !pairs || !info || nmap < 1) return MVO_ERR_INVALID_ARG;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int W = method == 2 ? 2 : 1;
  uint8_t *d = nullptr;
  const size_t o_vis = (size_t)nmap * 8, o_pairs = al256(o_vis + nmap), o_info = al256(o_pairs + (size_t)nmap * 8), tot = o_info + 256;   // info: 3 results + phase counters
  MVO_CUDA(ctx, cudaMalloc(&d, tot));
  cudaMemcpyAsync(d, keys, (size_t)nmap * W * 4, cudaMemcpyHostToDevice, ctx->stream);
  cudaMemcpyAsync(d + o_vis, vis, nmap, cudaMemcpyHostToDevice, ctx->stream);
  MvoTrackFilter f;
  memset(&f, 0, sizeof f);
  f.d_keys = (const uint32_t *)d; f.d_vis = d + o_vis; f.nmap = nmap; f.nk = nk; f.method = method;
  f.d_pairs = (int32_t *)(d + o_pairs); f.d_info = (int32_t *)(d + o_info);
  int rc = mvo_track_match_filter(ctx, f);
  if (rc == MVO_OK) {
    cudaMemcpyAsync(info, d + o_info, 48, cudaMemcpyDeviceToHost, ctx->stream);
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = mvo_fail(ctx, MVO_ERR_CUDA, "match filter kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
    else if (info[2] == 0 && info[0] > 0) cudaMemcpy(pairs, d + o_pairs, (size_t)info[0] * 8, cudaMemcpyDeviceToHost);
  }
  cudaFree(d);
  return rc;
}

static int submit_extraction(mvo_tracker *t, const uint8_t *image, int channels, size_t stride, int image_on_device) {
  mvo_ctx *ctx = t->ctx;
  if (!image) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: null image");
  if ((int)(t->n_submit - t->n_consume) + (t->held ? 1 : 0) >= MVO_XSLOTS)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: %d frames are already in flight", (int)(t->n_submit - t->n_consume));
  const int slot = (int)(t->n_submit % MVO_XSLOTS);
  ExtractJob &j = t->job[slot];
  mvo_ctx *x = t->xctx[slot];
  MVO_TRY(mvo_set_params(x, &ctx->prm));          // follow parameter changes made on the main context
  j.image = image; j.channels = channels; j.stride = stride; j.on_device = image_on_device;
  j.serial = t->n_submit_total + 1;
  j.want_host = !use_device_path(t);
  j.rc = MVO_OK; j.nk = 0; j.d_k = nullptr; j.d_d = nullptr;
  j.prematch = false; j.matched = false;
  if (!j.want_host && t->prm.match_method != 3) {
    MVO_TRY(dev_alloc(t));                          // the worker needs the device copy of the map
    j.prematch = true;
    j.match_mode = t->prm.match_method == 1 ? 0 : 1;
    j.map_version = t->map_version;
    j.d_map_desc = t->d_map_desc; j.nmap = t->dev_nmap; j.d_keys = (uint32_t *)t->d_keysvis[slot];
  }
  {
    std::lock_guard<std::mutex> lk(t->mu);
    j.state.store(1, std::memory_order_release);
  }
  t->cv_job.notify_all();
  ++t->n_submit;
  ++t->n_submit_total;
  return MVO_OK;
}

// checkLargeMoveForAddKeyFrame_ (vo.cpp:247-265), translation part + bookkeeping shared by both paths
static void finish_frame(mvo_tracker *t, bool pnp_ok, double *T_w_c_out) {
  if (!t->external_ref && pnp_ok && trans_dist(t->frames.back().T_w_c, t->T_ref) > t->prm.min_dist_keyframe)
    memcpy(t->T_ref, t->frames.back().T_w_c, sizeof t->T_ref);
  memcpy(t->T_prev, t->frames.back().T_w_c, sizeof t->T_prev);
  t->has_prev = true;
  memcpy(T_w_c_out, t->frames.back().T_w_c, 16 * sizeof(double));
}

static int track_device(mvo_tracker *t, ExtractJob &job, int slot, double *T_w_c_out, mvo_track_result *res, int ref_k = -1, int allow_spec = 0);
static int track_host_arrays(mvo_tracker *t, ExtractJob &job, double *T_w_c_out, mvo_track_result *res);

extern "C" {

void mvo_default_track_params(mvo_track_params *p) {
  if (!p) return;
  memset(p, 0, sizeof *p);
  p->match_method = 1;            // config/config.yaml:75
  p->match_radius = 50.f;         // :91
  p->min_pnp_points = 5;          // src/vo/vo.cpp:304
  p->max_dist_to_prev = 0.3;      // config.yaml:117
  p->min_dist_keyframe = 0.03;    // :116
  p->ba_enable = 1;               // :120
  p->ba_window = 5;               // :121
  p->ba_fix_points = 1;           // :123
  p->information[0] = 1; p->information[1] = 0; p->information[2] = 0; p->information[3] = 1;   // :122
  p->buffer_size = 20;            // include/my_slam/vo/vo.h:77
  p->ba_step_tol = 1e-9;
  p->device_resident = 1;
}

int mvo_tracker_create(mvo_ctx *ctx, const double *K, int rows, int cols, const mvo_track_params *params,
                       mvo_tracker **out) {
  if (!ctx || !out) return MVO_ERR_INVALID_ARG;
  *out = nullptr;
  if (!K || rows <= 0 || cols <= 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: bad K / image size");
  mvo_tracker *t = new mvo_tracker();
  t->ctx = ctx;
  memcpy(t->K, K, sizeof t->K);
  t->rows = rows;
  t->cols = cols;
  if (params) t->prm = *params;
  else mvo_default_track_params(&t->prm);
  if (t->prm.match_method < 1 || t->prm.match_method > 3 || t->prm.ba_window < 1 || t->prm.ba_window > 16 ||
      t->prm.buffer_size < 2 || t->prm.buffer_size > 4096 || !(t->prm.ba_step_tol >= 0)) {
    delete t;
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: bad parameters");
  }
  memset(t->T_ref, 0, sizeof t->T_ref);
  t->T_ref[0] = t->T_ref[5] = t->T_ref[10] = t->T_ref[15] = 1;
  for (int k = 0; k < MVO_XSLOTS; ++k) {
    const int rc = mvo_create(&t->xctx[k], ctx->device, &ctx->prm);
    if (rc != MVO_OK) {
      mvo_tracker_destroy(t);
      return mvo_fail(ctx, rc, "tracker: cannot create the extraction context");
    }
  }
  for (int k = 0; k < MVO_XSLOTS; ++k) t->worker[k] = std::thread(worker_main, t, k);
  *out = t;
  return MVO_OK;
}

void mvo_tracker_destroy(mvo_tracker *t) {
  if (!t) return;
  if (t->worker[0].joinable()) {
    drain_jobs(t);
    {
      std::lock_guard<std::mutex> lk(t->mu);
      t->stop = true;
    }
    t->cv_job.notify_all();
    for (int k = 0; k < MVO_XSLOTS; ++k)
      if (t->worker[k].joinable()) t->worker[k].join();
  }
  for (int k = 0; k < MVO_XSLOTS; ++k)
    if (t->xctx[k]) mvo_destroy(t->xctx[k]);
  if (t->ev_result) { cudaSetDevice(t->ctx->device); cudaEventDestroy(t->ev_result); t->ev_result = nullptr; }
  if (t->dev || t->dev_map || t->dev_ids) {
    cudaSetDevice(t->ctx->device);
    cudaStreamSynchronize(t->ctx->stream);
    if (t->dev) cudaFree(t->dev);
    if (t->dev_map) cudaFree(t->dev_map);
    if (t->dev_ids) cudaFree(t->dev_ids);
  }
  if (t->h_pin) cudaFreeHost(t->h_pin);
  delete t;
}

int mvo_tracker_prefetch(mvo_tracker *t, const uint8_t *image, int channels, size_t stride, int image_on_device) {
  if (!t) return MVO_ERR_INVALID_ARG;
  return submit_extraction(t, image, channels, stride, image_on_device);
}

int mvo_tracker_set_map(mvo_tracker *t, const float *pts3d, const uint8_t *desc, int n) {
  if (!t) return MVO_ERR_INVALID_ARG;
  if (n < 0 || (n > 0 && (!pts3d || !desc))) return mvo_fail(t->ctx, MVO_ERR_INVALID_ARG, "tracker: null map");
  if (n > 65535) return mvo_fail(t->ctx, MVO_ERR_UNSUPPORTED, "tracker: more than 65535 map points");
  // point index = map point id: frames already buffered keep their links by id, links to ids >= n leave the BA graph
  std::vector<int32_t> ids((size_t)n);
  for (int i = 0; i < n; ++i) ids[(size_t)i] = i;
  return mvo_trk_set_map_ids(t, pts3d, desc, ids.data(), n, 1);
}

int mvo_tracker_reset(mvo_tracker *t, const double *T_w_c_ref) {
  if (!t || !T_w_c_ref) return MVO_ERR_INVALID_ARG;
  memcpy(t->T_ref, T_w_c_ref, sizeof t->T_ref);
  t->frames.clear();
  t->has_prev = false;
  t->frame_counter = 0;
  t->fused_holdoff = 0;
  t->spec.valid = false;
  drain_jobs(t);                    // drop frames that were prefetched but never tracked
  t->n_submit = t->n_consume = 0;
  {
    std::lock_guard<std::mutex> lk(t->mu);
    t->n_run = 0;
  }
  return MVO_OK;
}

int mvo_tracker_timing_enable(mvo_tracker *t, uint32_t mask) {
  if (!t) return MVO_ERR_INVALID_ARG;
  if (t->n_submit != t->n_consume) return mvo_fail(t->ctx, MVO_ERR_INVALID_ARG, "tracker: timing calls need an idle tracker (frames are in flight)");
  MVO_TRY(mvo_timing_enable(t->ctx, mask));
  for (int k = 0; k < MVO_XSLOTS; ++k) MVO_TRY(mvo_timing_enable(t->xctx[k], mask));
  return MVO_OK;
}

int mvo_tracker_timing_read(mvo_tracker *t, double *ms, uint64_t *counts) {
  if (!t) return MVO_ERR_INVALID_ARG;
  if (t->n_submit != t->n_consume) return mvo_fail(t->ctx, MVO_ERR_INVALID_ARG, "tracker: timing calls need an idle tracker (frames are in flight)");
  MVO_TRY(mvo_timing_read(t->ctx, ms, counts));
  for (int k = 0; k < MVO_XSLOTS; ++k) MVO_TRY(mvo_timing_read(t->xctx[k], ms, counts));
  return MVO_OK;
}

uint64_t mvo_tracker_kernel_launches(const mvo_tracker *t) {
  if (!t) return 0;
  uint64_t n = mvo_kernel_launches(t->ctx);
  for (int k = 0; k < MVO_XSLOTS; ++k) n += mvo_kernel_launches(t->xctx[k]);
  return n;
}

int mvo_tracker_frame_pose(const mvo_tracker *t, int k, double *T_w_c) {
  if (!t || !T_w_c || k < 0 || k >= (int)t->frames.size()) return MVO_ERR_INVALID_ARG;
  memcpy(T_w_c, t->frames[t->frames.size() - 1 - k].T_w_c, 16 * sizeof(double));
  return MVO_OK;
}

int mvo_tracker_track(mvo_tracker *t, const uint8_t *image, int channels, size_t stride, int image_on_device,
                      double *T_w_c_out, mvo_track_result *res) {
  if (!t) return MVO_ERR_INVALID_ARG;
  if (!T_w_c_out) return mvo_fail(t->ctx, MVO_ERR_INVALID_ARG, "tracker: null pointer");
  int slot = 0, nk = 0;
  MVO_TRY(mvo_trk_acquire(t, image, channels, stride, image_on_device, &slot, &nk));
  ExtractJob &job = t->job[slot];
  const int rc = job.want_host ? track_host_arrays(t, job, T_w_c_out, res) : track_device(t, job, slot, T_w_c_out, res);
  mvo_trk_release(t, slot);
  return rc;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// Internal interface for the state machine (vo_pipeline.cpp, device-resident mode): mvo_vo keeps the reference's
// containers on the host and drives this tracker as the owner of everything that lives on the GPU — the map arrays, the
// frame ring mirroring frames_buff_, the per-point visibility / match counters.
// ------------------------------------------------------------------------------------------------------------
int mvo_trk_acquire(mvo_tracker *t, const uint8_t *image, int channels, size_t stride, int image_on_device, int *slot_out, int *nk_out) {
  mvo_ctx *ctx = t->ctx;
  if (!image) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: null pointer");
  // take the frame from the prefetch queue, or extract it now
  if (t->n_submit != t->n_consume && t->job[t->n_consume % MVO_XSLOTS].image != image)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: frames must be tracked in the order they were prefetched");
  if (t->n_submit == t->n_consume) MVO_TRY(submit_extraction(t, image, channels, stride, image_on_device));
  const int slot = (int)(t->n_consume % MVO_XSLOTS);
  ExtractJob &job = t->job[slot];
  if (!job.want_host) {
    // the device copy of the map is refreshed while the extraction runs
    const int rc = dev_alloc(t);
    if (rc != MVO_OK) { wait_job(t, slot); job.state.store(0, std::memory_order_release); ++t->n_consume; return rc; }
  }
  static const bool dbg_wait = getenv("MVO_TRACK_DEBUG") != nullptr;
  const double tw0 = dbg_wait ? now_us() : 0;
  wait_job(t, slot);
  if (dbg_wait) {                        // how long the tracking thread stood waiting for the extraction worker
    static double acc_wait = 0;
    static int n_wait = 0;
    acc_wait += now_us() - tw0;
    if (++n_wait % 50 == 0) { fprintf(stderr, "tracker: waited %.1f us/frame for the extraction of the frame\n", acc_wait / 50); acc_wait = 0; }
  }
  ++t->n_consume;
  if (job.rc != MVO_OK) {
    const int rc = mvo_fail(ctx, job.rc, "tracker: %s", mvo_last_error(t->xctx[slot]));
    job.state.store(0, std::memory_order_release);
    return rc;
  }
  *slot_out = slot;
  if (nk_out) *nk_out = job.nk;
  t->held = true;
  return MVO_OK;
}

void mvo_trk_release(mvo_tracker *t, int slot) {
  if (t->ref_copy_pending) {             // the worker may overwrite the slot's buffers as soon as it is released
    cudaSetDevice(t->ctx->device);
    cudaStreamSynchronize(t->ctx->stream);
    t->ref_copy_pending = false;
  }
  t->job[slot].state.store(0, std::memory_order_release);
  t->held = false;
}

// The acquired frame becomes the reference keyframe: its descriptors are kept on the device (asynchronous device-to-device
// copy; completed by the next synchronisation of the tracking stream, at the latest when the slot is released).
int mvo_trk_set_ref_desc(mvo_tracker *t, int slot, int tag) {
  mvo_ctx *ctx = t->ctx;
  ExtractJob &job = t->job[slot];
  t->n_ref = 0; t->ref_tag = -1;
  if (job.want_host || job.nk <= 0 || !job.d_d) return MVO_OK;
  MVO_TRY(dev_alloc(t));
  if (job.nk > t->dev_cap) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  MVO_CUDA(ctx, cudaMemcpyAsync(t->d_ref_desc, job.d_d, (size_t)job.nk * 32, cudaMemcpyDeviceToDevice, ctx->stream));
  t->n_ref = job.nk; t->ref_tag = tag;
  t->ref_copy_pending = true;
  return MVO_OK;
}

// Keyframe insertion, device-resident mode: everything the host needs of the frame that was just tracked, in ONE submission
// and ONE synchronisation — keypoints, descriptors, colours (gathered on the device for an image in device memory), the
// connections PnP gave it (inliers_to_mappt_connections_), the visible / matched increments since the last call (read and
// reset; with_links = 0 for a frame that has not been tracked: initialisation), and the matcher keys of the reference keyframe's descriptors against this frame's (match_mode 0 =
// nearest neighbour, 1 = two nearest; only when the descriptors kept by mvo_trk_set_ref_desc carry `ref_tag`).
int mvo_trk_keyframe_fetch(mvo_tracker *t, int slot, int want_rgb, int with_links, int n_counters, int ref_tag, int match_mode, MvoKfFetch *out) {
  mvo_ctx *ctx = t->ctx;
  ExtractJob &job = t->job[slot];
  memset(out, 0, sizeof *out);
  if (job.want_host) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "tracker: the frame was extracted for the host-array path");
  if (with_links && t->frames.empty()) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: no frame in the buffer");
  const int n = job.nk;
  static const TrackedFrame none = TrackedFrame();
  const TrackedFrame &f = with_links ? t->frames.back() : none;       // with_links: the acquired frame is the newest buffered one
  const int nl = (!with_links || f.slot < 0) ? 0 : f.n_links;
  const bool cnt_dev = n_counters > 0 && t->dev_nmap >= 0;
  if (cnt_dev && n_counters != t->dev_nmap)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: counters asked for %d points, the device map holds %d", n_counters, t->dev_nmap);
  if (want_rgb && !job.on_device) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: the image of this frame is in host memory");
  const bool do_match = match_mode >= 0 && match_mode <= 1 && t->n_ref > 0 && t->ref_tag == ref_tag && n > 0 && !(match_mode == 1 && n < 2);
  const int W = match_mode == 1 ? 2 : 1;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  size_t o = 0;
  const size_t o_k = o;   o = al256(o + (size_t)n * sizeof(mvo_keypoint));
  const size_t o_d = o;   o = al256(o + (size_t)n * 32);
  const size_t o_c = o;   o = al256(o + (size_t)n * 3);
  const size_t o_li = o;  o = al256(o + (size_t)nl * 4);
  const size_t o_lk = o;  o = al256(o + (size_t)nl * 4);
  const size_t o_v = o;   o = al256(o + (size_t)std::max(n_counters, 0) * 4);
  const size_t o_m = o;   o = al256(o + (size_t)std::max(n_counters, 0) * 4);
  const size_t o_key = o; o = al256(o + (do_match ? (size_t)t->n_ref * W * 4 : 0));
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_b, o + 256));
  MVO_TRY(mvo_reserve(ctx, ctx->d_d, o + 256));
  uint8_t *h = (uint8_t *)ctx->h_b.p;
  // every piece is gathered into one device staging buffer by one kernel and comes back in one copy
  MvoPackSegs segs;
  memset(&segs, 0, sizeof segs);
  uint32_t words = 0;
  auto add = [&](const void *src, size_t bytes, size_t dst_off, bool zero) {
    if (!bytes) return;
    segs.src[segs.n] = (const uint32_t *)src; segs.first[segs.n] = words; segs.dst_word[segs.n] = (uint32_t)(dst_off / 4);
    segs.zero_after[segs.n] = zero ? 1 : 0;
    words += (uint32_t)((bytes + 3) / 4);
    ++segs.n;
  };
  if (n > 0) {
    add(job.d_k, (size_t)n * sizeof(mvo_keypoint), o_k, false);
    add(job.d_d, (size_t)n * 32, o_d, false);
    if (want_rgb) {
      MVO_TRY(mvo_reserve(ctx, ctx->d_f, (size_t)n * 3 + 256));
      MVO_TRY(mvo_track_kpt_colors(ctx, job.d_k, n, job.image, job.channels, job.stride, (uint8_t *)ctx->d_f.p));
      add(ctx->d_f.p, (size_t)n * 3, o_c, false);
    }
  }
  if (do_match) {
    MVO_TRY(mvo_reserve(ctx, ctx->match_keys, (size_t)t->n_ref * W * 4 + 256));
    MVO_TRY(mvo_match_launch(ctx, match_mode, t->d_ref_desc, nullptr, t->n_ref, job.d_d, nullptr, n, 0.f, (uint32_t *)ctx->match_keys.p));
    add(ctx->match_keys.p, (size_t)t->n_ref * W * 4, o_key, false);
  }
  if (nl > 0) {
    const size_t oe = (size_t)f.slot * t->dev_cap;
    add(t->d_edge_map + oe, (size_t)nl * 4, o_li, false);
    add(t->d_edge_kp + oe, (size_t)nl * 4, o_lk, false);
  }
  if (cnt_dev) {
    add(t->d_vis_cnt, (size_t)n_counters * 4, o_v, true);
    add(t->d_match_cnt, (size_t)n_counters * 4, o_m, true);
  }
  segs.first[segs.n] = words;
  if (words) {
    MVO_TRY(mvo_track_pack_segments(ctx, segs, (uint32_t *)ctx->d_d.p));
    MVO_CUDA(ctx, cudaMemcpyAsync(h, ctx->d_d.p, o, cudaMemcpyDeviceToHost, ctx->stream));
  }
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  t->ref_copy_pending = false;
  if (!cnt_dev && n_counters > 0) {          // no frame has been tracked against this map yet: no increments
    memset(h + o_v, 0, (size_t)n_counters * 4);
    memset(h + o_m, 0, (size_t)n_counters * 4);
  }
  out->n_kpts = n;
  out->kpts = (const mvo_keypoint *)(h + o_k); out->desc = h + o_d; out->rgb = want_rgb ? h + o_c : nullptr;
  out->link_ids = (const int32_t *)(h + o_li); out->link_kp = (const int32_t *)(h + o_lk); out->n_links = nl;
  out->vis = (const int32_t *)(h + o_v); out->matched = (const int32_t *)(h + o_m); out->n_counters = std::max(n_counters, 0);
  out->keys = do_match ? (const uint32_t *)(h + o_key) : nullptr; out->n_ref = do_match ? t->n_ref : 0;
  return MVO_OK;
}

int mvo_trk_device_mode(const mvo_tracker *t) { return use_device_path(t) ? 1 : 0; }

void mvo_trk_configure(mvo_tracker *t, int external_ref, int count_stats) {
  t->external_ref = external_ref != 0;
  t->count_stats = count_stats != 0;
}

// keypoints / descriptors (/ colours, for an image in device memory: rgb != nullptr) of an acquired frame -> host, through a
// page-locked staging buffer (the device buffers stay valid until the slot is released)
int mvo_trk_fetch(mvo_tracker *t, int slot, mvo_keypoint *kpts, uint8_t *desc, uint8_t *rgb) {
  mvo_ctx *ctx = t->ctx;
  ExtractJob &job = t->job[slot];
  if (job.want_host) {
    if (kpts && job.nk) memcpy(kpts, job.kpts.data(), (size_t)job.nk * sizeof(mvo_keypoint));
    if (desc && job.nk) memcpy(desc, job.desc.data(), (size_t)job.nk * 32);
    if (rgb) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "tracker: colours of a host-path frame are sampled by the caller");
    return MVO_OK;
  }
  const int n = job.nk;
  if (n <= 0) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t o_d = al256((size_t)n * sizeof(mvo_keypoint)), o_c = o_d + al256((size_t)n * 32), tot = o_c + al256((size_t)n * 3);
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_b, tot));
  uint8_t *h = (uint8_t *)ctx->h_b.p;
  if (kpts) MVO_CUDA(ctx, cudaMemcpyAsync(h, job.d_k, (size_t)n * sizeof(mvo_keypoint), cudaMemcpyDeviceToHost, ctx->stream));
  if (desc) MVO_CUDA(ctx, cudaMemcpyAsync(h + o_d, job.d_d, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
  if (rgb) {
    if (!job.on_device) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "tracker: the image of this frame is in host memory");
    MVO_TRY(mvo_reserve(ctx, ctx->d_f, (size_t)n * 3 + 256));
    MVO_TRY(mvo_track_kpt_colors(ctx, job.d_k, n, job.image, job.channels, job.stride, (uint8_t *)ctx->d_f.p));
    MVO_CUDA(ctx, cudaMemcpyAsync(h + o_c, ctx->d_f.p, (size_t)n * 3, cudaMemcpyDeviceToHost, ctx->stream));
  }
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (kpts) memcpy(kpts, h, (size_t)n * sizeof(mvo_keypoint));
  if (desc) memcpy(desc, h + o_d, (size_t)n * 32);
  if (rgb) memcpy(rgb, h + o_c, (size_t)n * 3);
  return MVO_OK;
}

const uint8_t *mvo_trk_desc_dev(mvo_tracker *t, int slot) { return t->job[slot].d_d; }
unsigned mvo_trk_slot_serial(const mvo_tracker *t, int slot) { return t->job[slot].serial; }

int mvo_trk_set_map_ids(mvo_tracker *t, const float *pts3d, const uint8_t *desc, const int32_t *ids, int n, int reset_ids) {
  if (n < 0 || (n > 0 && (!pts3d || !desc || !ids))) return mvo_fail(t->ctx, MVO_ERR_INVALID_ARG, "tracker: null map");
  if (n > 65535) return mvo_fail(t->ctx, MVO_ERR_UNSUPPORTED, "tracker: more than 65535 map points");
  int max_id = -1;
  for (int i = 0; i < n; ++i) {
    if (ids[i] < 0) return mvo_fail(t->ctx, MVO_ERR_INVALID_ARG, "tracker: negative map point id");
    max_id = std::max(max_id, ids[i]);
  }
  t->map_pts.assign(pts3d, pts3d + (size_t)n * 3);
  t->map_desc.assign(desc, desc + (size_t)n * 32);
  t->map_ids.assign(ids, ids + (size_t)n);
  // ids are never reused (MapPoint::factory_id_): the by-id arrays only grow, except for the index-is-id maps of
  // mvo_tracker_set_map, which restart at every call
  const size_t n_ids = reset_ids ? (size_t)(max_id + 1) : std::max(t->alive.size(), (size_t)(max_id + 1));
  t->alive.assign(n_ids, 0);
  t->pos_by_id.resize(n_ids * 3, 0.f);
  for (int i = 0; i < n; ++i) {
    t->alive[(size_t)ids[i]] = 1;
    memcpy(&t->pos_by_id[3 * (size_t)ids[i]], pts3d + 3 * (size_t)i, 12);
  }
  t->dev_nmap = -1;                 // the device copy is refreshed by the next frame
  ++t->map_version;
  t->spec.valid = false;
  return MVO_OK;
}

// pushFrameToBuff_ for a frame that does not go through the tracking step (BLANK / DOING_INITIALIZATION): pose + its
// connections (map point id, keypoint index, pixel), so that the BA window sees the same frames_buff_ as the reference
int mvo_trk_push_frame(mvo_tracker *t, const double *T_w_c, const int32_t *ids, const int32_t *kp_idx, const float *obs_xy, int n) {
  mvo_ctx *ctx = t->ctx;
  MVO_TRY(dev_alloc(t));
  if (n > t->dev_cap) return mvo_fail(ctx, MVO_ERR_CAPACITY, "tracker: %d connections exceed the keypoint capacity %d", n, t->dev_cap);
  t->frames.emplace_back();
  if ((int)t->frames.size() > t->prm.buffer_size) t->frames.pop_front();
  TrackedFrame &cur = t->frames.back();
  cur.slot = (int)(t->frame_counter++ % (unsigned)t->dev_ring);
  cur.n_links = n;
  memcpy(cur.T_w_c, T_w_c, sizeof cur.T_w_c);
  double P[12];
  Twc_to_Rt12(T_w_c, P);
  const size_t o = (size_t)cur.slot * t->dev_cap;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  MVO_CUDA(ctx, cudaMemcpyAsync(t->d_pose + (size_t)cur.slot * 12, P, sizeof P, cudaMemcpyHostToDevice, ctx->stream));
  if (t->ring_host.size() >= ((size_t)cur.slot + 1) * 12) memcpy(&t->ring_host[(size_t)cur.slot * 12], P, sizeof P);
  t->spec.valid = false;
  MVO_CUDA(ctx, cudaMemcpyAsync(t->d_cnt + cur.slot, &n, 4, cudaMemcpyHostToDevice, ctx->stream));
  if (n > 0) {
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_edge_map + o, ids, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_edge_kp + o, kp_idx, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_edge_obs + 2 * o, obs_xy, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  }
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(t->T_prev, T_w_c, sizeof t->T_prev);
  t->has_prev = true;
  return MVO_OK;
}

// connections a keyframe gains from triangulation (pushCurrPointsToMap_, vo.cpp:528-576) appended to the k-th newest frame
int mvo_trk_append_links(mvo_tracker *t, int k, const int32_t *ids, const int32_t *kp_idx, const float *obs_xy, int n) {
  mvo_ctx *ctx = t->ctx;
  if (k < 0 || k >= (int)t->frames.size()) return MVO_ERR_INVALID_ARG;
  TrackedFrame &f = t->frames[t->frames.size() - 1 - (size_t)k];
  if (n <= 0 || f.slot < 0) return MVO_OK;
  if (f.n_links + n > t->dev_cap) return mvo_fail(ctx, MVO_ERR_CAPACITY, "tracker: %d connections exceed the keypoint capacity %d", f.n_links + n, t->dev_cap);
  const size_t o = (size_t)f.slot * t->dev_cap + f.n_links;
  const int total = f.n_links + n;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  MVO_CUDA(ctx, cudaMemcpyAsync(t->d_edge_map + o, ids, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(t->d_edge_kp + o, kp_idx, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(t->d_edge_obs + 2 * o, obs_xy, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(t->d_cnt + f.slot, &total, 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  t->ref_copy_pending = false;
  f.n_links = total;
  return MVO_OK;
}

// inliers_to_mappt_connections_ of the k-th newest frame: (map point id, keypoint index) in insertion order
int mvo_trk_links(mvo_tracker *t, int k, int32_t *ids, int32_t *kp_idx, int cap, int *n) {
  mvo_ctx *ctx = t->ctx;
  if (k < 0 || k >= (int)t->frames.size() || !n) return MVO_ERR_INVALID_ARG;
  const TrackedFrame &f = t->frames[t->frames.size() - 1 - (size_t)k];
  *n = f.slot < 0 ? 0 : f.n_links;
  if (*n > cap) return MVO_ERR_CAPACITY;
  if (*n == 0) return MVO_OK;
  const size_t o = (size_t)f.slot * t->dev_cap;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  MVO_CUDA(ctx, cudaMemcpyAsync(ids, t->d_edge_map + o, (size_t)*n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(kp_idx, t->d_edge_kp + o, (size_t)*n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MVO_OK;
}

// the tracking step of an acquired frame with the caller's guess (reference keyframe) and previous-frame poses
int mvo_trk_track(mvo_tracker *t, int slot, const double *T_guess, const double *T_prev, double *T_w_c_out, mvo_track_result *res, int ref_k,
                  int allow_spec) {
  ExtractJob &job = t->job[slot];
  if (job.want_host) return mvo_fail(t->ctx, MVO_ERR_UNSUPPORTED, "tracker: the frame was extracted for the host-array path");
  memcpy(t->T_ref, T_guess, sizeof t->T_ref);
  t->has_prev = T_prev != nullptr;
  if (T_prev) memcpy(t->T_prev, T_prev, sizeof t->T_prev);
  return track_device(t, job, slot, T_w_c_out, res, ref_k, allow_spec);
}

// ------------------------------------------------------------------------------------------------------------
// device-resident path
// ------------------------------------------------------------------------------------------------------------
// Layout of the 768-byte result block (d_flags, d_res, d_stats are contiguous):
//   int32 [0] BA skip flag   [8..10] model found, pnp_ok, inliers   [16..33] BA graph: frames, edges, slot of frame f
//         [40..48] match filter: pairs, candidates, status, -, phase cycle counters
//   +256: world->camera pose of the frame before BA (12 doubles)      +512: BA statistics (16 doubles)
static int track_device(mvo_tracker *t, ExtractJob &job, int slot, double *T_w_c_out, mvo_track_result *res, int ref_k, int allow_spec) {
  mvo_ctx *ctx = t->ctx;
  // ring slot of the reference keyframe (the frame whose pose is the initial guess), looked up before this frame enters the buffer
  int ref_slot = -1;
  if (ref_k >= 1 && ref_k <= (int)t->frames.size()) ref_slot = t->frames[t->frames.size() - (size_t)ref_k].slot;
  mvo_track_result r;
  memset(&r, 0, sizeof r);
  static const bool dbg = getenv("MVO_TRACK_DEBUG") != nullptr;
  static const bool force_host_filter = getenv("MVO_TRACK_HOST_FILTER") != nullptr;     // test hook: the two-sync variant
  static double acc[8] = {0};
  static int nacc = 0;
  double t0 = dbg ? now_us() : 0;
#define TMARK(i) do { if (dbg) { const double t_ = now_us(); acc[i] += t_ - t0; t0 = t_; } } while (0)
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int nmap = t->dev_nmap, cap = t->dev_cap, nk = job.nk;
  const int method = t->prm.match_method;
  r.n_keypoints = nk;

  // pushFrameToBuff_ (vo.h:81-86)
  t->frames.emplace_back();
  if ((int)t->frames.size() > t->prm.buffer_size) t->frames.pop_front();
  TrackedFrame &cur = t->frames.back();
  cur.slot = (int)(t->frame_counter++ % (unsigned)t->dev_ring);
  // curr_->T_w_c_ = ref_->T_w_c_.clone()  (vo_addFrame.cpp:74): initial guess = reference keyframe
  memcpy(cur.T_w_c, t->T_ref, sizeof cur.T_w_c);
  const int total = (int)t->frames.size();

  uint8_t *d_keysvis = t->d_keysvis[slot];
  uint32_t *d_keys = (uint32_t *)d_keysvis;
  uint8_t *d_vis = d_keysvis + (size_t)std::max(nmap, 1) * 8;
  const bool prematched = job.matched && job.map_version == t->map_version && job.match_mode == (method == 1 ? 0 : 1) && method != 3;
  int32_t *d_finfo = t->d_flags + 40, *d_res_i = t->d_flags + 8, *d_out_info = t->d_flags + 16;
  uint8_t *h_out = t->h_pin + al256((size_t)std::max(nmap, 1) * 9) + al256((size_t)std::max(nmap, 1) * 8 + 64);
  const int32_t *h_flags = (const int32_t *)h_out;
  const bool can_match = nmap > 0 && nk > 0 && !(method == 2 && nk < 2);

  // ---- getMappointsInCurrentView_ + matchFeatures(map descriptors, frame descriptors) (vo.cpp:16-49, 283-289) ----
  auto fail = [&](int rc) { cudaStreamSynchronize(ctx->stream); t->frames.pop_back(); return rc; };
  int rc = MVO_OK;
  double Tcw[12];
  Twc_to_Rt12(cur.T_w_c, Tcw);
  // When the guess is the pose of a buffered frame, its world->camera form is taken from the pose ring as it is (host mirror here,
  // device memory for a chain head enqueued ahead of time: the same twelve doubles) instead of inverting the inverse again.
  if (ref_slot >= 0 && t->ring_host.size() >= ((size_t)ref_slot + 1) * 12) {
    const double *rp = &t->ring_host[(size_t)ref_slot * 12];
    double dmax = 0;
    for (int q = 0; q < 12; ++q) dmax = std::max(dmax, fabs(rp[q] - Tcw[q]));
    if (dmax < 1e-9) memcpy(Tcw, rp, sizeof Tcw);
    else ref_slot = -1;                      // the caller's guess is not that frame's pose: no ring pose, no speculation
  } else ref_slot = -1;
  // methods 1/2: the matcher does not need the projections, so the in-view test is folded into the filter kernel
  // (the keys of points outside the view are simply ignored there); method 3 gates on the projected pixel
  const bool project_in_filter = method != 3 && !force_host_filter && t->fused_holdoff == 0;
  if (nmap > 0) {
    if (!project_in_filter) rc = mvo_track_project_map(ctx, t->d_map_pts, nmap, Tcw, t->K, t->rows, t->cols, d_vis, t->d_cxy);
    if (rc == MVO_OK && can_match && prematched) {
      // keys of every map point are already there (unmasked: the filter / host filter ignores points outside the view)
    } else if (rc == MVO_OK && can_match) {
      if (method == 3) rc = mvo_track_kpt_xy(ctx, job.d_k, nk, t->d_kxy);
      if (rc == MVO_OK)
        rc = mvo_match_launch_masked(ctx, method == 1 ? 0 : (method == 2 ? 1 : 2), t->d_map_desc, t->d_cxy, nmap, job.d_d, t->d_kxy, nk,
                                     t->prm.match_radius, d_keys, project_in_filter ? nullptr : d_vis);
    } else if (rc == MVO_OK) {
      if (cudaMemsetAsync(d_keys, 0xFF, (size_t)nmap * 8, ctx->stream) != cudaSuccess) rc = mvo_fail(ctx, MVO_ERR_CUDA, "tracker: memset");
    }
    if (rc != MVO_OK) return fail(rc);
  }

  // ---- everything after the matcher: thresholds + duplicate removal, PnP, frame-buffer update, BA ----
  // d_n != nullptr: the pair count lives on the device (n = its upper bound); otherwise n pairs are in d_pairs
  MvoPoseStore st;
  bool counted = false;            // visible_times_ / matched_times_ are accumulated by the first tail only
  bool pnp_enqueued = false;       // the PnP kernels of this frame were enqueued ahead of time (speculative chain head)
  std::function<int()> speculate;  // set by the fused path: enqueues the next frame's chain head behind this frame's result copy
  auto enqueue_tail = [&](int n, const int32_t *d_n, bool gathered) -> int {
    MvoTrackGlue g;
    memset(&g, 0, sizeof g);
    const bool run_pnp = n >= 4 && (d_n != nullptr || n >= t->prm.min_pnp_points);
    g.mode = run_pnp ? (d_n ? 2 : 1) : 0;
    g.min_pnp = t->prm.min_pnp_points; g.n_pairs_dev = d_n;
    g.slot = cur.slot; g.cap = cap; g.ba_enable = t->prm.ba_enable; g.has_prev = t->has_prev;
    g.max_dist = t->prm.max_dist_to_prev;
    if (t->has_prev) { g.prev_twc[0] = t->T_prev[3]; g.prev_twc[1] = t->T_prev[7]; g.prev_twc[2] = t->T_prev[11]; }
    Twc_to_Rt12(t->has_prev ? t->T_prev : cur.T_w_c, g.fallback);      // vo.cpp:376-379
    g.pairs = t->d_pairs; g.kpts = job.d_k;
    g.edge_map = t->d_edge_map; g.edge_obs = t->d_edge_obs; g.edge_kp = t->d_edge_kp; g.cnt = t->d_cnt; g.pose = t->d_pose;
    g.skip_flag = t->d_flags; g.res_i = d_res_i; g.res_d = t->d_res;
    g.map_ids = t->d_map_ids; g.vis = d_vis; g.nmap = nmap;
    // visible_times_ once per frame; matched_times_ by the tail whose PnP saw the pairs (a declined device filter hands
    // its tail zero pairs, so the redo through the host filter is the one that counts the inliers)
    if (t->count_stats && nmap > 0) { g.match_cnt = t->d_match_cnt; if (!counted) g.vis_cnt = t->d_vis_cnt; }
    int rc2 = MVO_OK;
    if (run_pnp) {
      float *d_p3, *d_p2;
      double *d_pose_io;
      int32_t *d_out_i, *d_inl;
      rc2 = mvo_pnp_dev_buffers(ctx, n, &d_p3, &d_p2, &d_pose_io, &d_out_i, &d_inl);
      if (rc2 == MVO_OK && !gathered) rc2 = mvo_track_gather_pairs(ctx, t->d_pairs, n, d_n, t->d_map_pts, job.d_k, d_p3, d_p2);
      if (rc2 == MVO_OK && !pnp_enqueued) rc2 = mvo_pnp_dev_run(ctx, n, t->K, d_n);
      pnp_enqueued = false;
      g.pose_io = d_pose_io; g.out_i = d_out_i; g.inl = d_inl;
    }
    if (rc2 == MVO_OK) rc2 = mvo_track_glue(ctx, g);
    // the BA window: newest min(ba_window, total-1) frames (vo.cpp:417-419); frames with < 3 links drop out on the
    // device (:423-426), where the newest frame's link count is known
    memset(&st, 0, sizeof st);
    if (rc2 == MVO_OK && run_pnp && t->prm.ba_enable) {
      int e_upper = 0;
      const int nba = std::min(t->prm.ba_window, total - 1);
      for (int b = total - 1; b >= total - nba; --b) {
        if (t->frames[b].slot < 0) continue;         // tracked through the host-array path (parameters changed mid-sequence)
        st.slot[st.nslots++] = t->frames[b].slot;
        e_upper += (b == total - 1) ? n : t->frames[b].n_links;
      }
      if (st.nslots > 0) {
        st.map_pts = t->d_pos_by_id; st.alive = t->d_alive; st.n_ids = (int)t->alive.size(); st.edge_map = t->d_edge_map; st.edge_obs = (const float2 *)t->d_edge_obs; st.cnt = t->d_cnt;
        st.pose = t->d_pose; st.cap = cap; st.min_links = 3; st.skip_flag = t->d_flags; st.out_info = d_out_info;
        rc2 = mvo_ba_pose_store_launch(ctx, st, e_upper, t->K[0], t->K[0], t->K[2], t->K[5], t->prm.information, ctx->prm.ba_iterations,
                                       ctx->prm.ba_huber_delta > 0, ctx->prm.ba_huber_delta, t->prm.ba_step_tol, t->d_stats);
      }
    }
    if (rc2 != MVO_OK) return rc2;
    // one D2H: the result block + the pose ring
    MVO_CUDA(ctx, cudaMemcpyAsync(h_out, t->d_flags, 768, cudaMemcpyDeviceToHost, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(h_out + 768, t->d_pose, (size_t)t->dev_ring * 96, cudaMemcpyDeviceToHost, ctx->stream));
    if (!t->ev_result) MVO_CUDA(ctx, cudaEventCreateWithFlags(&t->ev_result, cudaEventDisableTiming));
    MVO_CUDA(ctx, cudaEventRecord(t->ev_result, ctx->stream));
    if (speculate) { const int rcs = speculate(); if (rcs != MVO_OK) return rcs; }       // the next frame's chain head, behind this frame's results
    MVO_CUDA(ctx, cudaEventSynchronize(t->ev_result));
    return MVO_OK;
  };

  // thresholds of matchFeatures (feature_match.cpp:179-217) and removeDuplicatedMatches (:241-260) on the host,
  // from the keys the matcher left on the device: the variant with a second synchronisation, used when the
  // device-side duplicate removal declines (list beyond its capacity, or libstdc++ would have left quicksort)
  auto host_filter_tail = [&]() -> int {
    const uint32_t *h_keys = (const uint32_t *)t->h_pin;
    const uint8_t *h_vis = t->h_pin + (size_t)std::max(nmap, 1) * 8;
    if (nmap > 0) {
      MVO_CUDA(ctx, cudaMemcpyAsync(t->h_pin, d_keysvis, (size_t)nmap * 9, cudaMemcpyDeviceToHost, ctx->stream));
      MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    std::vector<MatchPair> &pairs = t->pairs;
    int ncand = 0;
    host_match_filter(ctx->prm, method, can_match, h_keys, h_vis, nmap, pairs, &ncand);
    const int nm = (int)pairs.size();
    int32_t *h_pairs = (int32_t *)(t->h_pin + al256((size_t)std::max(nmap, 1) * 9));
    for (int i = 0; i < nm; ++i) { h_pairs[2 * i] = pairs[i].map; h_pairs[2 * i + 1] = pairs[i].train; }
    int32_t *h_fi = h_pairs + 2 * (size_t)nm;          // filter record, same layout as the kernel writes
    h_fi[0] = nm; h_fi[1] = ncand; h_fi[2] = 0;
    MVO_CUDA(ctx, cudaMemcpyAsync(t->d_pairs, h_pairs, (size_t)nm * 8, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(d_finfo, h_fi, 12, cudaMemcpyHostToDevice, ctx->stream));
    return enqueue_tail(nm, nullptr, false);
  };

  // The device filter restates the quicksort phase of libstdc++'s std::sort and declines when that phase would hit
  // its depth limit (libstdc++ then heapsorts: inherently sequential).  Match lists in a presorted-by-level map order
  // do that on every frame, so after a decline the next frames go straight to the host filter.
  bool fused = nmap > 0 && !force_host_filter && t->fused_holdoff == 0;
  if (t->fused_holdoff > 0) --t->fused_holdoff;
  // the head of a frame's chain: match filter (in-view test, thresholds, duplicate removal, PnP input arrays) + the PnP kernels;
  // side-effect free apart from scratch buffers.  Tcw_host / d_Tcw: the guess pose as a kernel argument or in device memory.
  auto enqueue_head = [&](const ExtractJob &jb, int jslot, const double *Tcw_host, const double *d_Tcw, int *n_upper_out) -> int {
    uint8_t *kv = t->d_keysvis[jslot];
    const int n_up = std::min(nmap, std::max(jb.nk, 0));
    MvoTrackFilter f;
    memset(&f, 0, sizeof f);
    f.d_keys = (uint32_t *)kv; f.d_vis = kv + (size_t)std::max(nmap, 1) * 8; f.nmap = nmap; f.nk = jb.nk; f.method = method;
    f.d_pairs = t->d_pairs; f.d_info = d_finfo;
    if (Tcw_host || d_Tcw) { f.Tcw12 = Tcw_host; f.d_Tcw12 = d_Tcw; f.K = t->K; f.rows = t->rows; f.cols = t->cols; }
    f.d_map_pts = t->d_map_pts;
    int rch = MVO_OK;
    if (n_up >= 4) {             // the filter writes the PnP input arrays itself
      double *d_pose_io;
      int32_t *d_out_i, *d_inl;
      rch = mvo_pnp_dev_buffers(ctx, n_up, &f.d_p3, &f.d_p2, &d_pose_io, &d_out_i, &d_inl);
      f.d_kpts = jb.d_k;
    }
    if (rch == MVO_OK) rch = mvo_track_match_filter(ctx, f);
    *n_upper_out = n_up;
    return rch;
  };
  if (fused) {
    int n_upper = 0;
    const bool spec_ok = t->spec.valid && t->spec.serial == job.serial && t->spec.map_version == t->map_version && ref_slot >= 0 &&
                         t->spec.ref_slot == ref_slot && t->spec.nmap == nmap && t->spec.nk == nk && t->spec.method == method && prematched &&
                         project_in_filter && can_match;
    t->spec.valid = false;
    if (spec_ok) {               // the filter and the PnP kernels of this frame are already in the stream (or done)
      n_upper = t->spec.n_upper;
      pnp_enqueued = n_upper >= 4;
      ++t->spec_hits;
    } else {
      rc = enqueue_head(job, slot, project_in_filter ? Tcw : nullptr, nullptr, &n_upper);
    }
    // next frame: its extraction and pre-match run on the worker while this frame is tracked; once they are done its chain head
    // goes into the stream behind this frame's results, with the reference pose read from the ring slot this frame's BA may move
    if (allow_spec && ref_slot >= 0 && project_in_filter && can_match && prematched && t->n_submit != t->n_consume && rc == MVO_OK) {
      speculate = [&, ref_slot]() -> int {
        const int ns = (int)(t->n_consume % MVO_XSLOTS);
        ExtractJob &nj = t->job[ns];
        if (nj.want_host) return MVO_OK;
        wait_job(t, ns);
        const int mode = method == 1 ? 0 : 1;
        if (nj.rc != MVO_OK || !nj.matched || nj.map_version != t->map_version || nj.match_mode != mode || nj.nk <= 0 || (method == 2 && nj.nk < 2))
          return MVO_OK;
        int n_up = 0;
        int rcs = enqueue_head(nj, ns, nullptr, t->d_pose + (size_t)ref_slot * 12, &n_up);
        if (rcs == MVO_OK && n_up >= 4) rcs = mvo_pnp_dev_run(ctx, n_up, t->K, d_finfo);
        if (rcs != MVO_OK) return rcs;
        t->spec.valid = true; t->spec.serial = nj.serial; t->spec.map_version = t->map_version; t->spec.ref_slot = ref_slot;
        t->spec.nmap = nmap; t->spec.nk = nj.nk; t->spec.method = method; t->spec.n_upper = n_up;
        ++t->spec_issued;
        return MVO_OK;
      };
    }
    if (rc == MVO_OK) rc = enqueue_tail(n_upper, d_finfo, true);
    speculate = nullptr;
    if (rc != MVO_OK) { t->spec.valid = false; return fail(rc); }
    TMARK(0);
    // the device filter declined: redo the tail through the host (its first pass saw zero pairs: only the in-view counts were taken)
    if (h_flags[42] != 0) { fused = false; counted = true; t->fused_holdoff = 64; t->spec.valid = false; }
  }
  if (!fused) {
    rc = host_filter_tail();
    if (rc != MVO_OK) return fail(rc);
    TMARK(1);
  }

  const int32_t *h_res_i = h_flags + 8, *h_info = h_flags + 16;
  const double *h_res_d = (const double *)(h_out + 256), *h_stats = (const double *)(h_out + 512);
  const double *h_ring = (const double *)(h_out + 768);
  if (t->ring_host.size() >= (size_t)t->dev_ring * 12) memcpy(t->ring_host.data(), h_ring, (size_t)t->dev_ring * 96);
  r.n_matches = h_flags[40];
  r.n_candidates = h_flags[41];
  const bool pnp_ok = h_res_i[1] != 0;
  r.n_inliers = h_res_i[2];
  r.pnp_ok = pnp_ok;
  cur.n_links = h_res_i[2];
  if (pnp_ok) Rt12_to_Twc(h_res_d, cur.T_w_c);
  else if (t->has_prev) memcpy(cur.T_w_c, t->T_prev, sizeof cur.T_w_c);
  memcpy(r.T_w_c_pnp, cur.T_w_c, sizeof r.T_w_c_pnp);
  if (st.nslots > 0 && pnp_ok) {
    const int F = h_info[0];
    if (F < 0) { t->frames.pop_back(); return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "tracker: BA graph exceeds the device-resident kernel"); }
    for (int f = 0; f < F; ++f) {
      const int s = h_info[2 + f];
      for (int b = total - 1; b >= 0; --b)
        if (t->frames[b].slot == s) { Rt12_to_Twc(h_ring + (size_t)s * 12, t->frames[b].T_w_c); break; }
    }
    r.ba_frames = F;
    r.ba_edges = h_info[1];
    static const bool ba_dbg = getenv("MVO_BA_DEBUG") != nullptr;
    if (ba_dbg)
      fprintf(stderr, "k_ba_pose(store): F=%d E=%d it=%.0f trials=%.0f rejected=%.0f cycles solve=%.0f pass=%.0f gather=%.0f decide=%.0f | "
              "pdl_wait=%.0f setup=%.0f init=%.0f exit=%.0f kernel=%.0f\n", F, h_info[1], h_stats[2], h_stats[15], h_stats[7], h_stats[8],
              h_stats[9], h_stats[10], h_stats[11], h_stats[12], h_stats[4], h_stats[5], h_stats[6], h_stats[13]);
  }
  TMARK(2);
  if (dbg && ++nacc % 50 == 0) {
    fprintf(stderr, "tracker(device) us/frame: fused frame (launch .. sync) %.1f host-filter redo %.1f finish %.1f | filter kernel cycles: prologue %d sort %d (%d levels, %d segments heapsorted, longest %d) epilogue %d\n",
            acc[0] / 50, acc[1] / 50, acc[2] / 50, h_flags[44], h_flags[45], h_flags[48], h_flags[43], h_flags[47], h_flags[46]);
    fprintf(stderr, "  chain heads enqueued ahead of time: %llu issued, %llu used\n", (unsigned long long)t->spec_issued, (unsigned long long)t->spec_hits);
    fprintf(stderr, "  per level (cycles, nbig*1000+nsmall):");
    for (int l = 0; l < 7; ++l) fprintf(stderr, " %d/%d", h_flags[49 + 2 * l], h_flags[50 + 2 * l]);
    fprintf(stderr, "\n");
    for (double &a : acc) a = 0;
  }
#undef TMARK
  finish_frame(t, pnp_ok, T_w_c_out);
  if (res) *res = r;
  return MVO_OK;
}

// ------------------------------------------------------------------------------------------------------------
// host-array path: every stage through its public C-ABI entry point
// ------------------------------------------------------------------------------------------------------------
static int track_host_arrays(mvo_tracker *t, ExtractJob &job, double *T_w_c_out, mvo_track_result *res) {
  mvo_ctx *ctx = t->ctx;
  mvo_track_result r;
  memset(&r, 0, sizeof r);
  static const bool dbg = getenv("MVO_TRACK_DEBUG") != nullptr;
  static double acc[8] = {0};
  static int nacc = 0;
  double t0 = dbg ? now_us() : 0;
#define TMARK(i) do { if (dbg) { const double t_ = now_us(); acc[i] += t_ - t0; t0 = t_; } } while (0)

  // pushFrameToBuff_ (vo.h:81-86) + Frame::calcKeyPoints / calcDescriptors (done by the extraction worker)
  t->frames.emplace_back();
  if ((int)t->frames.size() > t->prm.buffer_size) t->frames.pop_front();
  TrackedFrame &cur = t->frames.back();
  const int nk = job.nk;
  const mvo_keypoint *kpts = job.kpts.data();
  const uint8_t *d_desc = job.d_d;
  int rc = MVO_OK;
  r.n_keypoints = nk;
  TMARK(0);

  // curr_->T_w_c_ = ref_->T_w_c_.clone()  (vo_addFrame.cpp:74): initial guess = reference keyframe
  memcpy(cur.T_w_c, t->T_ref, sizeof cur.T_w_c);

  // ---- getMappointsInCurrentView_ (vo.cpp:16-49) ----
  double Tcw[16];
  inv_rigid(cur.T_w_c, Tcw);
  const int nmap = (int)(t->map_pts.size() / 3);
  t->cand_idx.resize(nmap); t->cand_xy.resize((size_t)nmap * 2); t->cand_desc.resize((size_t)nmap * 32);
  int ncand = 0;
  {
    const float *mp = t->map_pts.data();
    const uint8_t *md = t->map_desc.data();
    uint8_t *cd = t->cand_desc.data();
    const float fcols = (float)t->cols, frows = (float)t->rows;
    for (int i = 0; i < nmap; ++i) {
      // basics::preTranslatePoint3f: double accumulation of T(row, j) * p[j] (j = 0..3), narrowed to float
      const double p0 = mp[3 * i], p1 = mp[3 * i + 1], p2 = mp[3 * i + 2];
      double q[3];
      for (int row = 0; row < 3; ++row) {
        double acc = 0;
        acc += Tcw[row * 4] * p0; acc += Tcw[row * 4 + 1] * p1; acc += Tcw[row * 4 + 2] * p2; acc += Tcw[row * 4 + 3] * 1.0;
        q[row] = acc;
      }
      const float cx = (float)q[0], cy = (float)q[1], cz = (float)q[2];
      if (cz < 0) continue;
      // geometry::cam2pixel (camera.cpp): K(0,0) * p.x / p.z + K(0,2) in double, narrowed to Point2f
      const float u = (float)(t->K[0] * cx / cz + t->K[2]), v = (float)(t->K[4] * cy / cz + t->K[5]);
      if (!(u > 0 && v > 0 && u < fcols && v < frows)) continue;
      t->cand_idx[ncand] = i;
      t->cand_xy[2 * ncand] = u;
      t->cand_xy[2 * ncand + 1] = v;
      memcpy(cd + (size_t)ncand * 32, md + (size_t)i * 32, 32);
      ++ncand;
    }
  }
  t->cand_idx.resize(ncand);
  const int nc = (int)t->cand_idx.size();
  r.n_candidates = nc;
  TMARK(1);

  // ---- matchFeatures(map descriptors, frame descriptors) (vo.cpp:283-289) ----
  t->kp_xy.resize((size_t)nk * 2);
  for (int i = 0; i < nk; ++i) { t->kp_xy[2 * i] = kpts[i].x; t->kp_xy[2 * i + 1] = kpts[i].y; }
  t->matches.resize(nc > 0 ? nc : 1);
  int nm = 0;
  if (nc > 0 && nk > 0 && !(t->prm.match_method == 2 && nk < 2)) {
    rc = mvo_match_features_ex(ctx, t->cand_desc.data(), nc, d_desc, nk, 1, t->prm.match_method, t->cand_xy.data(),
                               t->kp_xy.data(), t->prm.match_radius, t->matches.data(), &nm);
    if (rc != MVO_OK) { t->frames.pop_back(); return rc; }
  }
  r.n_matches = nm;
  TMARK(2);
  t->p3.resize((size_t)nm * 3);
  t->p2.resize((size_t)nm * 2);
  for (int i = 0; i < nm; ++i) {            // vo.cpp:293-301
    const int mi = t->cand_idx[t->matches[i].query_idx], ki = t->matches[i].train_idx;
    memcpy(&t->p3[3 * i], &t->map_pts[3 * mi], 12);
    t->p2[2 * i] = kpts[ki].x;
    t->p2[2 * i + 1] = kpts[ki].y;
  }

  // ---- poseEstimationPnP_ (vo.cpp:304-381) ----
  bool pnp_ok = nm >= t->prm.min_pnp_points;
  if (pnp_ok) {
    double rvec[3], tvec[3];
    t->inliers.resize(nm);
    int ni = nm;
    rc = mvo_solve_pnp_ransac(ctx, t->p3.data(), t->p2.data(), nm, t->K, rvec, tvec, t->inliers.data(), &ni);
    if (rc == MVO_ERR_DEGENERATE) { pnp_ok = false; ni = 0; }
    else if (rc != MVO_OK) { t->frames.pop_back(); return rc; }
    if (pnp_ok) {
      r.n_inliers = ni;
      for (int i = 0; i < ni; ++i) {        // vo.cpp:333-354
        const mvo_dmatch &m = t->matches[t->inliers[i]];
        cur.obs_xy.push_back(kpts[m.train_idx].x);
        cur.obs_xy.push_back(kpts[m.train_idx].y);
        cur.map_idx.push_back(t->cand_idx[m.query_idx]);
      }
      double Tc[16], R[9];
      rvec_to_R(rvec, R);
      for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) Tc[i * 4 + j] = R[i * 3 + j]; Tc[i * 4 + 3] = tvec[i]; }
      Tc[12] = Tc[13] = Tc[14] = 0; Tc[15] = 1;
      inv_rigid(Tc, cur.T_w_c);             // vo.cpp:357: T_w_c = [R|t]^-1
      // vo.cpp:360-369: reject jumps relative to the previous frame
      if (t->has_prev && trans_dist(cur.T_w_c, t->T_prev) >= t->prm.max_dist_to_prev) pnp_ok = false;
    }
  }
  if (!pnp_ok && t->has_prev) memcpy(cur.T_w_c, t->T_prev, sizeof cur.T_w_c);   // vo.cpp:376-379
  r.pnp_ok = pnp_ok;
  TMARK(3);
  memcpy(r.T_w_c_pnp, cur.T_w_c, sizeof r.T_w_c_pnp);

  // ---- callBundleAdjustment_ (vo.cpp:384-478) ----
  if (pnp_ok && t->prm.ba_enable) {
    const int total = (int)t->frames.size();
    const int nba = std::min(t->prm.ba_window, total - 1);
    std::vector<double> &poses = t->ba_poses;
    std::vector<int> &which = t->ba_which;
    std::vector<int32_t> &ef = t->ba_ef, &ep = t->ba_ep, &used = t->ba_used;
    std::vector<float> &ob = t->ba_ob, &pts = t->ba_pts;
    poses.clear(); which.clear(); ef.clear(); ep.clear(); ob.clear(); used.clear();
    for (int b = total - 1; b >= total - nba; --b) {          // newest first (vo.cpp:417-419)
      TrackedFrame &f = t->frames[b];
      if ((int)f.map_idx.size() < 3) continue;                // vo.cpp:423-426
      const int fi = (int)which.size();
      which.push_back(b);
      poses.insert(poses.end(), f.T_w_c, f.T_w_c + 16);
      for (size_t e = 0; e < f.map_idx.size(); ++e) {
        if (f.map_idx[e] >= nmap) continue;                   // the point left the map with a later mvo_tracker_set_map (vo.cpp:438-440)
        ef.push_back(fi);
        ep.push_back(f.map_idx[e]);
        ob.push_back(f.obs_xy[2 * e]); ob.push_back(f.obs_xy[2 * e + 1]);
      }
    }
    if (!which.empty() && !ef.empty()) {
      // only the map points that appear in the graph become vertices (um_pts_3d_in_prev_frames)
      if ((int)t->ba_remap.size() != nmap) { t->ba_remap.assign(nmap, 0); t->ba_stamp.assign(nmap, 0); t->ba_gen = 0; }
      const int32_t gen = ++t->ba_gen;
      for (int32_t &e : ep) {
        if (t->ba_stamp[e] != gen) { t->ba_stamp[e] = gen; t->ba_remap[e] = (int32_t)used.size(); used.push_back(e); }
        e = t->ba_remap[e];
      }
      pts.resize((size_t)used.size() * 3);
      for (size_t k = 0; k < used.size(); ++k) memcpy(&pts[3 * k], &t->map_pts[3 * (size_t)used[k]], 12);
      const int fix = t->prm.ba_fix_points ? 1 : 0;
      const double saved_tol = ctx->prm.ba_step_tol;
      ctx->prm.ba_step_tol = t->prm.ba_step_tol;
      rc = mvo_bundle_adjustment(ctx, poses.data(), (int)which.size(), pts.data(), (int)used.size(), ef.data(),
                                 ep.data(), ob.data(), (int)ef.size(), t->K, t->prm.information, fix, !fix, nullptr);
      ctx->prm.ba_step_tol = saved_tol;
      if (rc != MVO_OK) return rc;
      for (size_t k = 0; k < which.size(); ++k) memcpy(t->frames[which[k]].T_w_c, &poses[16 * k], 16 * sizeof(double));
      if (!fix) {
        for (size_t k = 0; k < used.size(); ++k) memcpy(&t->map_pts[3 * (size_t)used[k]], &pts[3 * k], 12);
        t->dev_nmap = -1;
      }
      r.ba_frames = (int)which.size();
      r.ba_edges = (int)ef.size();
    }
  }
  TMARK(4);
  if (dbg && ++nacc % 50 == 0) {
    fprintf(stderr, "tracker(host arrays) us/frame: extract %.1f candidates %.1f match %.1f pnp %.1f ba %.1f\n", acc[0] / 50, acc[1] / 50, acc[2] / 50, acc[3] / 50, acc[4] / 50);
    for (double &a : acc) a = 0;
  }
#undef TMARK
  finish_frame(t, pnp_ok, T_w_c_out);
  if (res) *res = r;
  return MVO_OK;
}
