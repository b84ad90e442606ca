// Host orchestration of ORB extraction: pyramid plan, workspace, the C-ABI entry points and the
// host-side steps that are deliberately NOT on the GPU because their result depends on libstdc++
// (cv::KeyPointsFilter::retainBest = std::nth_element + std::partition, SURVEY.md App. A.4).
#include <algorithm>
#include <atomic>
#include <math.h>
#include <string.h>
#include <vector>
#include "orb.cuh"

namespace {

struct OrbState {           // lives in mvo_ctx via the opaque DevBufs; plan kept here per context
  OrbPlanDev plan;
  std::vector<int32_t> tables;
  bool valid = false;
};

// one plan per context, owned by the context (contexts may be driven from different host threads)
OrbState *state_of(mvo_ctx *ctx) {
  if (!ctx->orb_state) ctx->orb_state = new OrbState();
  return (OrbState *)ctx->orb_state;
}

inline int cv_round(double v) { return (int)nearbyint(v); }   // cvRound: round half to even

// cv::resize INTER_LINEAR_EXACT coefficient tables for one axis (SURVEY.md App. A.2)
void axis_table(int src, int dst, int32_t *ofs, int32_t *w1) {
  const double scale = 1.0 / ((double)dst / (double)src);
  for (int d = 0; d < dst; ++d) {
    double f = scale * (d + 0.5) - 0.5;
    int i = (int)floor(f);
    if (i < 0) { ofs[d] = 0; w1[d] = 0; }
    else if (i >= src - 1) { ofs[d] = src - 1; w1[d] = 0; }
    else { ofs[d] = i; w1[d] = (int)nearbyint((f - i) * 256.0); }
  }
}

int build_plan(mvo_ctx *ctx, OrbState *st, int rows, int cols) {
  const mvo_params &P = ctx->prm;
  st->valid = false;           // a plan rejected below must not be taken for the previous one by the next call (ensure_ws)
  if (rows < 2 * ORB_EDGE + 8 || cols < 2 * ORB_EDGE + 8)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "image %dx%d too small for ORB (edge threshold 31)", cols, rows);
  if (cols >= ORB_MAX_W || rows >= ORB_MAX_W)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "image %dx%d too large (max %d)", cols, rows, ORB_MAX_W - 1);
  if (P.orb_nfeatures > 65535) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "orb_nfeatures > 65535");
  OrbPlanDev &pl = st->plan;
  memset(&pl, 0, sizeof pl);
  pl.nlevels = P.orb_nlevels;
  pl.rows = rows;
  pl.cols = cols;
  pl.fast_threshold = P.orb_fast_threshold;
  pl.grid_size = P.grid_size;
  pl.grid_rows = rows / P.grid_size;          // feature_match.cpp:59
  pl.grid_cols = cols / P.grid_size;
  pl.max_per_cell = P.max_pts_per_grid;
  pl.max_kpts = P.max_keypoints;
  pl.sel_cap = P.orb_nfeatures;
  if (pl.grid_rows < 1 || pl.grid_cols < 1 || pl.grid_rows * pl.grid_cols > 65535)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "selection grid %dx%d unsupported", pl.grid_rows, pl.grid_cols);

  // featuresPerLevel, OpenCV orb.cpp (float arithmetic exactly as there)
  const double scale_factor = (double)P.orb_scale_factor;      // ORB_Impl stores the float argument in a double
  {
    float factor = (float)(1.0 / scale_factor);
    float ndesired = P.orb_nfeatures * (1 - factor) / (1 - (float)pow((double)factor, (double)pl.nlevels));
    int sum = 0;
    for (int l = 0; l < pl.nlevels - 1; ++l) {
      pl.lv[l].cap = cv_round(ndesired);
      sum += pl.lv[l].cap;
      ndesired *= factor;
    }
    pl.lv[pl.nlevels - 1].cap = std::max(P.orb_nfeatures - sum, 0);
  }
  size_t off = 0, tab = 0;
  int bands = 0;
  long cand_cap = 0;
  int band_cap = 0;
  int nl = 0;
  for (int l = 0; l < pl.nlevels; ++l) {
    OrbLevelDev &L = pl.lv[l];
    L.scale = (float)pow(scale_factor, (double)l);
    const float inv = 1.0f / L.scale;                            // OpenCV orb.cpp: Size(cvRound(cols * invScale), cvRound(rows * invScale))
    L.w = cv_round((double)((float)cols * inv));                 // (cols / scale rounds the other way for e.g. 153 rows: 128 vs 127)
    L.h = cv_round((double)((float)rows * inv));
    if (L.w < 2 * ORB_EDGE + 2 || L.h < 2 * ORB_EDGE + 2) break;    // level has no pixel inside the border
    L.pitch = (L.w + 127) & ~127;
    L.img_off = (uint32_t)off;
    off += (size_t)L.pitch * L.h;
    off = (off + 255) & ~(size_t)255;
    L.blur_off = (uint32_t)off;
    off += (size_t)L.pitch * L.h;
    off = (off + 255) & ~(size_t)255;
    L.tab_off = (uint32_t)tab;
    if (l > 0) tab += 2 * (size_t)L.w + 2 * (size_t)L.h;
    const int nms_h = L.h - 2 * ORB_EDGE, nms_w = L.w - 2 * ORB_EDGE;
    L.band_first = bands;
    L.nbands = (nms_h + ORB_BAND_H - 1) / ORB_BAND_H;
    bands += L.nbands;
    band_cap = std::max(band_cap, (ORB_BAND_H / 2) * ((nms_w + 1) / 2));
    cand_cap += (long)((nms_w + 1) / 2) * ((nms_h + 1) / 2);
    nl = l + 1;
  }
  if (nl != pl.nlevels)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "pyramid level %d of a %dx%d image is smaller than the ORB border", nl, cols, rows);
  if (bands > ORB_MAX_BANDS) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "too many FAST bands (%d)", bands);
  pl.total_bands = bands;
  pl.band_cap = band_cap;
  pl.cand_cap = (int)cand_cap;
  pl.slot_bytes = (uint32_t)off;
  st->tables.assign(tab ? tab : 1, 0);
  for (int l = 1; l < pl.nlevels; ++l) {
    OrbLevelDev &L = pl.lv[l];
    int32_t *t = st->tables.data() + L.tab_off;
    axis_table(pl.lv[l - 1].w, L.w, t, t + L.w);
    axis_table(pl.lv[l - 1].h, L.h, t + 2 * L.w, t + 2 * L.w + L.h);
  }
  // band table of the fused gray + pyramid kernel: band b owns rows [b H_l / nb, (b + 1) H_l / nb) of every level; the rows of
  // level l it must HOLD are those plus the source rows (INTER_LINEAR_EXACT reads rows yofs[y] and yofs[y] + 1) of the rows it
  // holds of level l + 1
  {
    const int nb = std::max(1, rows / 8), nl = pl.nlevels;
    pl.pyr_nb = nb;
    pl.pyr_tab_off = (uint32_t)st->tables.size();
    st->tables.resize(st->tables.size() + (size_t)nb * nl * 4, 0);
    int32_t *bt = st->tables.data() + pl.pyr_tab_off;
    for (int l = 0; l < nl; ++l) pl.pyr_rows[l] = 0;
    for (int b = 0; b < nb; ++b) {
      int lo = 0, hi = 0;                                        // rows held of the level above (none above the top level)
      for (int l = nl - 1; l >= 0; --l) {
        const int H = pl.lv[l].h, olo = (int)((long)b * H / nb), ohi = (int)((long)(b + 1) * H / nb);
        int nlo = olo, nhi = ohi;
        if (l + 1 < nl && hi > lo) {
          const OrbLevelDev &U = pl.lv[l + 1];
          const int32_t *yofs = st->tables.data() + U.tab_off + 2 * U.w;
          const int slo = yofs[lo], shi = std::min(yofs[hi - 1] + 1, H - 1) + 1;
          if (nhi > nlo) { nlo = std::min(nlo, slo); nhi = std::max(nhi, shi); }
          else { nlo = slo; nhi = shi; }
        }
        int32_t *e = bt + ((size_t)b * nl + l) * 4;
        e[0] = nlo; e[1] = nhi; e[2] = olo; e[3] = ohi;
        pl.pyr_rows[l] = std::max(pl.pyr_rows[l], nhi - nlo);
        lo = nlo; hi = nhi;
      }
    }
  }
  st->valid = true;
  ctx->orb.rows = rows;
  ctx->orb.cols = cols;
  ctx->orb.nlevels = pl.nlevels;
  ctx->orb_batch = 0;
  return MVO_OK;
}

// workspace carve-up inside ctx buffers
struct OrbWs {
  uint8_t *planes;
  uint32_t *staging;
  int32_t *bandcnt;
  uint32_t *cand;
  float *harris;
  uint2 *sel;
  OrbFrameMeta *meta;
  int32_t *tables;
  int32_t *n_override;
  int32_t *bad_flag;
  uint16_t *kept;          // [batch][nlevels][orb_retain_max()] retained candidates of an overflowing level, in retainBest's order
  int32_t *kept_cnt;       // [batch][nlevels]
};

int ensure_ws(mvo_ctx *ctx, OrbState *st, int rows, int cols, int batch, OrbWs *ws) {
  if (!st->valid || ctx->orb.rows != rows || ctx->orb.cols != cols || st->plan.nlevels != ctx->prm.orb_nlevels ||
      st->plan.max_kpts != ctx->prm.max_keypoints || st->plan.grid_size != ctx->prm.grid_size ||
      st->plan.max_per_cell != ctx->prm.max_pts_per_grid || st->plan.fast_threshold != ctx->prm.orb_fast_threshold ||
      st->plan.sel_cap != ctx->prm.orb_nfeatures) {
    MVO_TRY(build_plan(ctx, st, rows, cols));
  }
  const OrbPlanDev &pl = st->plan;
  const bool grow = batch > ctx->orb_batch;
  if (grow) {
    MVO_TRY(mvo_reserve(ctx, ctx->orb_planes, (size_t)batch * pl.slot_bytes));
    MVO_TRY(mvo_reserve(ctx, ctx->orb_cand, (size_t)batch * pl.total_bands * pl.band_cap * 4));       // staging
    MVO_TRY(mvo_reserve(ctx, ctx->orb_bandcnt, (size_t)batch * pl.total_bands * 4));
    MVO_TRY(mvo_reserve(ctx, ctx->orb_sel, (size_t)batch * (pl.max_kpts + 1) * 8));
    // misc: cand + harris + meta + n_override + bad flag + tables
    const size_t misc = (size_t)batch * pl.cand_cap * 8 + (size_t)batch * 64 + (size_t)batch * 4 + 256 +
                        st->tables.size() * 4 + 4096 + (size_t)batch * pl.nlevels * orb_retain_max() * 2 + (size_t)batch * pl.nlevels * 4 + 1024;
    MVO_TRY(mvo_reserve(ctx, ctx->orb_misc, misc));
  }
  const bool fresh = grow || ctx->orb_batch == 0;
  if (grow) ctx->orb_batch = batch;
  batch = ctx->orb_batch;        // carve with the CAPACITY so offsets stay put for smaller calls
  uint8_t *m = (uint8_t *)ctx->orb_misc.p;
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  size_t o = 0;
  ws->cand = (uint32_t *)(m + o); o = al(o + (size_t)batch * pl.cand_cap * 4);
  ws->harris = (float *)(m + o);  o = al(o + (size_t)batch * pl.cand_cap * 4);
  ws->meta = (OrbFrameMeta *)(m + o); o = al(o + (size_t)batch * 64);
  ws->n_override = (int32_t *)(m + o); o = al(o + (size_t)batch * 4);
  ws->bad_flag = (int32_t *)(m + o); o = al(o + 64);
  ws->kept = (uint16_t *)(m + o); o = al(o + (size_t)batch * pl.nlevels * orb_retain_max() * 2);
  ws->kept_cnt = (int32_t *)(m + o); o = al(o + (size_t)batch * pl.nlevels * 4);
  ws->tables = (int32_t *)(m + o);
  ws->planes = (uint8_t *)ctx->orb_planes.p;
  ws->staging = (uint32_t *)ctx->orb_cand.p;
  ws->bandcnt = (int32_t *)ctx->orb_bandcnt.p;
  ws->sel = (uint2 *)ctx->orb_sel.p;
  if (fresh) {
    MVO_CUDA(ctx, cudaMemcpyAsync(ws->tables, st->tables.data(), st->tables.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));     // tables live in a std::vector
  }
  return MVO_OK;
}

struct HostCand { float response; int32_t idx; };

// cv::KeyPointsFilter::retainBest (OpenCV keypoint.cpp) on (response, payload) records.
void retain_best(std::vector<HostCand> &v, int n_points) {
  if (n_points >= 0 && v.size() > (size_t)n_points) {
    if (n_points == 0) { v.clear(); return; }
    std::nth_element(v.begin(), v.begin() + n_points - 1, v.end(),
                     [](const HostCand &a, const HostCand &b) { return a.response > b.response; });
    const float ambiguous = v[n_points - 1].response;
    auto new_end = std::partition(v.begin() + n_points, v.end(),
                                  [ambiguous](const HostCand &c) { return c.response >= ambiguous; });
    v.resize(new_end - v.begin());
  }
}

// geometry::selectUniformKptsByGrid (feature_match.cpp:51-84) over (x, y) in level-0 pixels.
template <class GetXY>
std::vector<int> grid_select(int n, GetXY xy, int rows, int cols, int grid, int max_per_cell, int max_kpts) {
  const int gr = rows / grid, gc = cols / grid;
  std::vector<int> cnt((size_t)std::max(gr, 1) * std::max(gc, 1), 0), keep;
  int kept = 0;
  for (int i = 0; i < n; ++i) {
    float x, y;
    xy(i, x, y);
    int row = ((int)y) / grid, col = ((int)x) / grid;
    if (row < 0 || col < 0 || row >= gr || col >= gc) continue;   // reference indexes out of bounds here (UB): skipped, as k_select does
    if (cnt[(size_t)row * gc + col] < max_per_cell) {
      keep.push_back(i);
      cnt[(size_t)row * gc + col]++;
      if (++kept > max_kpts) break;
    }
  }
  return keep;
}

std::atomic<uint64_t> g_host_fallbacks{0};

// Host retainBest + grid selection for one overflowing frame; uploads the selection list.
int slow_path_frame(mvo_ctx *ctx, const OrbPlanDev &pl, const OrbWs &ws, int f, const OrbFrameMeta &meta,
                    std::vector<uint32_t> &cand, std::vector<float> &harris, int *n_sel_out) {
  const int n = std::min(meta.n_cand, pl.cand_cap);
  g_host_fallbacks.fetch_add(1);
  cand.resize(n);
  harris.resize(n);
  if (n) {
    MVO_CUDA(ctx, cudaMemcpyAsync(cand.data(), ws.cand + (size_t)f * pl.cand_cap, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(harris.data(), ws.harris + (size_t)f * pl.cand_cap, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  }
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  std::vector<uint2> kept;     // (packed, level) in OpenCV's output order
  int base = 0;
  for (int l = 0; l < pl.nlevels; ++l) {
    const int cnt = meta.lvl_count[l];
    std::vector<HostCand> v(cnt);
    for (int i = 0; i < cnt; ++i) v[i] = HostCand{(float)orb_ps(cand[base + i]), base + i};
    retain_best(v, 2 * pl.lv[l].cap);                          // by FAST score
    for (auto &c : v) c.response = harris[c.idx];              // HarrisResponses in that order
    retain_best(v, pl.lv[l].cap);                              // by Harris response
    for (auto &c : v) kept.push_back(make_uint2(cand[c.idx], (uint32_t)l));
    base += cnt;
  }
  auto xy = [&](int i, float &x, float &y) {
    const int l = (int)kept[i].y;
    const float s = pl.lv[l].scale;
    x = l ? (float)orb_px(kept[i].x) * s : (float)orb_px(kept[i].x);
    y = l ? (float)orb_py(kept[i].x) * s : (float)orb_py(kept[i].x);
  };
  std::vector<int> keep = grid_select((int)kept.size(), xy, pl.rows, pl.cols, pl.grid_size, pl.max_per_cell, pl.max_kpts);
  std::vector<uint2> sel(keep.size());
  for (size_t i = 0; i < keep.size(); ++i) sel[i] = kept[keep[i]];
  const int32_t ns = (int32_t)sel.size();
  if (ns)
    MVO_CUDA(ctx, cudaMemcpyAsync(ws.sel + (size_t)f * (pl.max_kpts + 1), sel.data(), (size_t)ns * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(ws.n_override + f, &ns, 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));          // sel/ns are stack/heap temporaries
  *n_sel_out = ns;
  return MVO_OK;
}

// Shared front end: image already on the device -> pyramid, FAST, selection.
int run_detect(mvo_ctx *ctx, OrbState *st, const OrbWs &ws, const uint8_t *d_in, int channels, size_t stride,
               size_t frame_stride, int batch) {
  const OrbPlanDev &pl = st->plan;
  MVO_TRY(orb_launch_gray_pyramid(ctx, pl, d_in, channels, stride, frame_stride, ws.tables, ws.planes, batch));
  MVO_TRY(orb_launch_fast(ctx, pl, ws.planes, ws.staging, ws.bandcnt, batch));
  MVO_TRY(orb_launch_select(ctx, pl, ws.staging, ws.bandcnt, ws.cand, ws.sel, ws.meta, batch));
  // frames with a level above OpenCV's featuresPerLevel: Harris response of every candidate, retainBest (twice per level) and
  // the grid selection on the device; both kernels return at once for the other frames
  MVO_TRY(orb_launch_harris_all(ctx, pl, ws.planes, ws.cand, ws.meta, ws.harris, batch));
  MVO_TRY(orb_launch_retain(ctx, pl, ws.cand, ws.harris, ws.meta, ws.kept, ws.kept_cnt, ws.sel, batch));
  return MVO_OK;
}

int check_image(mvo_ctx *ctx, const void *image, int rows, int cols, int channels, size_t stride) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!image) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "null image");
  if (channels != 1 && channels != 3) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "channels must be 1 (gray) or 3 (BGR)");
  if (rows <= 0 || cols <= 0 || stride < (size_t)cols * channels) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "bad image geometry");
  return MVO_OK;
}

// upload a host image into ctx->orb_in; returns the device pointer
int upload_image(mvo_ctx *ctx, const uint8_t *image, int rows, size_t stride, uint8_t **d_out) {
  const size_t bytes = (size_t)rows * stride;
  MVO_TRY(mvo_reserve(ctx, ctx->orb_in, bytes + 256));
  // page-locked caller memory (cudaHostAlloc / cudaHostRegister, e.g. a pinned torch tensor) is copied from directly;
  // pageable memory is staged through the context's pinned buffer first.  Either way the image has to stay valid
  // until the extraction has been consumed (synchronous entry points: until they return).
  cudaPointerAttributes attr;
  const bool pinned = cudaPointerGetAttributes(&attr, image) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  if (!pinned) {
    cudaGetLastError();
    MVO_TRY(mvo_reserve_pinned(ctx, ctx->orb_h, bytes + 256));
    memcpy(ctx->orb_h.p, image, bytes);
  }
  MVO_CUDA(ctx, cudaMemcpyAsync(ctx->orb_in.p, pinned ? (const void *)image : ctx->orb_h.p, bytes, cudaMemcpyHostToDevice, ctx->stream));
  *d_out = (uint8_t *)ctx->orb_in.p;
  return MVO_OK;
}

// ---- asynchronous extraction: begin() enqueues everything and returns, end() waits and finishes ----
struct OrbPending {
  bool active = false, with_desc = false, want_host = true;
  int rows = 0, cols = 0, out_cap = 0;
  cudaEvent_t done = nullptr;
  OrbWs ws;
  mvo_keypoint *d_k = nullptr;
  uint8_t *d_d = nullptr;
  OrbFrameMeta *h_meta = nullptr;
  mvo_keypoint *h_k = nullptr;
  uint8_t *h_d = nullptr;
};
OrbPending *pending_of(mvo_ctx *ctx) {
  if (!ctx->orb_pending) ctx->orb_pending = new OrbPending();
  return (OrbPending *)ctx->orb_pending;
}

// want_host = false: keypoints and descriptors stay on the device (only the 64-byte frame record comes back)
int extract_begin(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride, bool with_desc,
                  bool on_device, bool want_host = true) {
  MVO_TRY(check_image(ctx, image, rows, cols, channels, stride));
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  OrbState *st = state_of(ctx);
  OrbPending *pd = pending_of(ctx);
  if (pd->active) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "extract_begin: an extraction is already pending on this context");
  MVO_TRY(ensure_ws(ctx, st, rows, cols, 1, &pd->ws));
  const OrbPlanDev &pl = st->plan;
  const int out_cap = pl.max_kpts + 1;
  // pinned layout: [image (host input only)] [meta 256][kpts][desc]
  const size_t img_bytes = on_device ? 0 : (((size_t)rows * stride + 255) & ~(size_t)255);
  const size_t kb = ((size_t)out_cap * sizeof(mvo_keypoint) + 255) & ~(size_t)255;
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->orb_h, img_bytes + 256 + kb + (size_t)out_cap * 32 + 512));
  uint8_t *d_in = nullptr;
  if (on_device) d_in = const_cast<uint8_t *>(image);
  else MVO_TRY(upload_image(ctx, image, rows, stride, &d_in));
  MVO_TRY(mvo_reserve(ctx, ctx->orb_kpts, kb + (size_t)out_cap * 32 + 512));
  pd->d_k = (mvo_keypoint *)ctx->orb_kpts.p;
  pd->d_d = (uint8_t *)ctx->orb_kpts.p + kb;
  uint8_t *h = (uint8_t *)ctx->orb_h.p + img_bytes;
  pd->h_meta = (OrbFrameMeta *)h;
  pd->h_k = (mvo_keypoint *)(h + 256);
  pd->h_d = h + 256 + kb;
  pd->rows = rows; pd->cols = cols; pd->out_cap = out_cap; pd->with_desc = with_desc; pd->want_host = want_host;
  MVO_TRY(run_detect(ctx, st, pd->ws, d_in, channels, stride, 0, 1));
  if (with_desc) MVO_TRY(orb_launch_blur(ctx, pl, pd->ws.planes, 1));
  // optimistic fast path: describe right away; end() looks at the overflow flag
  MVO_TRY(orb_launch_describe_sel(ctx, pl, pd->ws.planes, pd->ws.sel, pd->ws.meta, nullptr, pd->d_k, pd->d_d, nullptr, out_cap, with_desc, 1));
  MVO_CUDA(ctx, cudaMemcpyAsync(pd->h_meta, pd->ws.meta, sizeof(OrbFrameMeta), cudaMemcpyDeviceToHost, ctx->stream));
  if (want_host) {
    MVO_CUDA(ctx, cudaMemcpyAsync(pd->h_k, pd->d_k, (size_t)out_cap * sizeof(mvo_keypoint), cudaMemcpyDeviceToHost, ctx->stream));
    if (with_desc) MVO_CUDA(ctx, cudaMemcpyAsync(pd->h_d, pd->d_d, (size_t)out_cap * 32, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (!pd->done) MVO_CUDA(ctx, cudaEventCreateWithFlags(&pd->done, cudaEventDisableTiming));
  MVO_CUDA(ctx, cudaEventRecord(pd->done, ctx->stream));
  pd->active = true;
  return MVO_OK;
}

// Waits for the pending extraction; on return kpts/desc (host) are filled and *d_desc (optional) points at
// the descriptors on the device (valid until the next extract_begin on this context).
int extract_end(mvo_ctx *ctx, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc, const uint8_t **d_desc,
                const mvo_keypoint **d_kpts = nullptr) {
  OrbPending *pd = pending_of(ctx);
  if (!pd->active) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "extract_end: nothing pending");
  pd->active = false;
  if (!n_kpts || (pd->want_host && ((*n_kpts > 0 && !kpts) || (pd->with_desc && *n_kpts > 0 && !desc))))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "null output");
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  MVO_CUDA(ctx, cudaEventSynchronize(pd->done));
  OrbState *st = state_of(ctx);
  const OrbPlanDev &pl = st->plan;
  int n = pd->h_meta->n_sel;
  if (pd->h_meta->overflow == 2) {
    // a level exceeds featuresPerLevel AND the device retainBest declined (more candidates than it holds, or an input on
    // which libstdc++'s nth_element leaves quickselect for heap-select): the host runs the real std::nth_element
    OrbFrameMeta meta = *pd->h_meta;
    std::vector<uint32_t> cand;
    std::vector<float> harris;
    MVO_TRY(slow_path_frame(ctx, pl, pd->ws, 0, meta, cand, harris, &n));
    MVO_TRY(orb_launch_describe_sel(ctx, pl, pd->ws.planes, pd->ws.sel, pd->ws.meta, pd->ws.n_override, pd->d_k, pd->d_d, nullptr,
                                    pd->out_cap, pd->with_desc, 1));
    if (pd->want_host) {
      MVO_CUDA(ctx, cudaMemcpyAsync(pd->h_k, pd->d_k, (size_t)pd->out_cap * sizeof(mvo_keypoint), cudaMemcpyDeviceToHost, ctx->stream));
      if (pd->with_desc) MVO_CUDA(ctx, cudaMemcpyAsync(pd->h_d, pd->d_d, (size_t)pd->out_cap * 32, cudaMemcpyDeviceToHost, ctx->stream));
    }
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  if (pd->want_host) {
    if (n > *n_kpts) return mvo_fail(ctx, MVO_ERR_CAPACITY, "keypoint capacity %d < %d", *n_kpts, n);
    memcpy(kpts, pd->h_k, (size_t)n * sizeof(mvo_keypoint));
    if (pd->with_desc) memcpy(desc, pd->h_d, (size_t)n * 32);
  }
  if (d_desc) *d_desc = pd->d_d;
  if (d_kpts) *d_kpts = pd->d_k;
  *n_kpts = n;
  return MVO_OK;
}

// detect (+ optionally describe) one image synchronously
int extract_host(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride,
                 mvo_keypoint *kpts, int *n_kpts, uint8_t *desc, bool with_desc, bool on_device = false) {
  if (!n_kpts || (*n_kpts > 0 && !kpts) || (with_desc && *n_kpts > 0 && !desc))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "null output");
  MVO_TRY(extract_begin(ctx, image, rows, cols, channels, stride, with_desc, on_device));
  return extract_end(ctx, kpts, n_kpts, desc, nullptr);
}

}  // namespace

int mvo_orb_extract_begin(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride, int on_device) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  return extract_begin(ctx, image, rows, cols, channels, stride, true, on_device != 0);
}

int mvo_orb_extract_end(mvo_ctx *ctx, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc, const uint8_t **d_desc) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  return extract_end(ctx, kpts, n_kpts, desc, d_desc);
}

int mvo_orb_extract_ex(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride,
                       int on_device, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc) {
  return extract_host(ctx, image, rows, cols, channels, stride, kpts, n_kpts, desc, true, on_device != 0);
}

// Device-only variant for the tracker: nothing but the frame record crosses PCIe.
int mvo_orb_extract_begin_dev(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride, int on_device) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  return extract_begin(ctx, image, rows, cols, channels, stride, true, on_device != 0, false);
}

// Between begin_dev and end_dev: the device buffers the pending extraction is filling and the address of its keypoint count on the
// device, so that a consumer kernel (the tracker's pre-match) can be queued behind the extraction without waiting for the count.
// *host_path_possible: the count may still be replaced by the host retainBest path (overflow == 2, see extract_end) — the caller
// checks mvo_orb_extract_used_host_path() after end_dev and redoes its kernel in that (adversarial-input) case.
int mvo_orb_extract_peek_dev(mvo_ctx *ctx, const mvo_keypoint **d_kpts, const uint8_t **d_desc, const int32_t **d_count, int *n_max) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  OrbPending *pd = pending_of(ctx);
  if (!pd->active) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "extract_peek: nothing pending");
  if (d_kpts) *d_kpts = pd->d_k;
  if (d_desc) *d_desc = pd->d_d;
  if (d_count) *d_count = &pd->ws.meta[0].n_sel;
  if (n_max) *n_max = pd->out_cap;
  return MVO_OK;
}
int mvo_orb_extract_used_host_path(mvo_ctx *ctx) {
  OrbPending *pd = pending_of(ctx);
  return pd->h_meta && pd->h_meta->overflow == 2 ? 1 : 0;
}
int mvo_orb_extract_end_dev(mvo_ctx *ctx, int *n_kpts, const mvo_keypoint **d_kpts, const uint8_t **d_desc) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  return extract_end(ctx, nullptr, n_kpts, nullptr, d_desc, d_kpts);
}

void orb_state_free(mvo_ctx *ctx) {
  if (ctx->orb_pending) {
    OrbPending *pd = (OrbPending *)ctx->orb_pending;
    if (pd->done) cudaEventDestroy(pd->done);
    delete pd;
    ctx->orb_pending = nullptr;
  }
  if (ctx->orb_state) {
    delete (OrbState *)ctx->orb_state;
    ctx->orb_state = nullptr;
  }
}

extern "C" {

// test hook (not part of mvo.h): frames whose retainBest ran on the host because the device path declined
uint64_t mvo_test_orb_host_fallbacks(void) { return g_host_fallbacks.load(); }

int mvo_calc_keypoints(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride,
                       mvo_keypoint *kpts, int *n_kpts) {
  return extract_host(ctx, image, rows, cols, channels, stride, kpts, n_kpts, nullptr, false);
}

int mvo_orb_extract(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride,
                    mvo_keypoint *kpts, int *n_kpts, uint8_t *desc) {
  return extract_host(ctx, image, rows, cols, channels, stride, kpts, n_kpts, desc, true);
}

int mvo_calc_descriptors(mvo_ctx *ctx, const uint8_t *image, int rows, int cols, int channels, size_t stride,
                         const mvo_keypoint *kpts, int n_kpts, uint8_t *desc) {
  MVO_TRY(check_image(ctx, image, rows, cols, channels, stride));
  if (n_kpts < 0 || (n_kpts > 0 && (!kpts || !desc))) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "null keypoints/descriptors");
  if (n_kpts == 0) return MVO_OK;
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  OrbState *st = state_of(ctx);
  OrbWs ws;
  MVO_TRY(ensure_ws(ctx, st, rows, cols, 1, &ws));
  const OrbPlanDev &pl = st->plan;
  // cv::ORB::compute regroups unsorted keypoints by level; the reference never does that
  // (calcKeyPoints output is level-major), so anything else is rejected rather than reordered.
  for (int i = 1; i < n_kpts; ++i)
    if (kpts[i].octave < kpts[i - 1].octave)
      return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "calcDescriptors: keypoints must be sorted by octave");
  const size_t img_bytes = ((size_t)rows * stride + 255) & ~(size_t)255;
  const size_t kb = ((size_t)n_kpts * sizeof(mvo_keypoint) + 255) & ~(size_t)255;
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->orb_h, img_bytes + kb + (size_t)n_kpts * 32 + 1024));
  uint8_t *d_in = nullptr;
  MVO_TRY(upload_image(ctx, image, rows, stride, &d_in));
  MVO_TRY(mvo_reserve(ctx, ctx->orb_kpts, kb + (size_t)n_kpts * 32 + 512));
  uint8_t *h = (uint8_t *)ctx->orb_h.p + img_bytes;
  memcpy(h, kpts, (size_t)n_kpts * sizeof(mvo_keypoint));
  mvo_keypoint *d_k = (mvo_keypoint *)ctx->orb_kpts.p;
  uint8_t *d_d = (uint8_t *)ctx->orb_kpts.p + kb;
  MVO_CUDA(ctx, cudaMemcpyAsync(d_k, h, (size_t)n_kpts * sizeof(mvo_keypoint), cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemsetAsync(ws.bad_flag, 0, 4, ctx->stream));
  MVO_TRY(orb_launch_gray_pyramid(ctx, pl, d_in, channels, stride, 0, ws.tables, ws.planes, 1));
  MVO_TRY(orb_launch_blur(ctx, pl, ws.planes, 1));
  MVO_TRY(orb_launch_describe_kpts(ctx, pl, ws.planes, d_k, n_kpts, d_d, ws.bad_flag));
  int32_t *h_bad = (int32_t *)(h + kb);
  uint8_t *h_d = h + kb + 256;
  MVO_CUDA(ctx, cudaMemcpyAsync(h_bad, ws.bad_flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(h_d, d_d, (size_t)n_kpts * 32, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (*h_bad == 1) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "calcDescriptors: keypoint octave outside the pyramid");
  if (*h_bad == 2) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "calcDescriptors: keypoint closer than 20 px to its level border");
  memcpy(desc, h_d, (size_t)n_kpts * 32);
  return MVO_OK;
}

int mvo_select_uniform_kpts_by_grid(mvo_ctx *ctx, mvo_keypoint *kpts, int *n_kpts, int image_rows, int image_cols) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!n_kpts || (*n_kpts > 0 && !kpts) || *n_kpts < 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "null keypoints");
  const mvo_params &P = ctx->prm;
  auto xy = [&](int i, float &x, float &y) { x = kpts[i].x; y = kpts[i].y; };
  std::vector<int> keep = grid_select(*n_kpts, xy, image_rows, image_cols, P.grid_size, P.max_pts_per_grid, P.max_keypoints);
  for (size_t i = 0; i < keep.size(); ++i) kpts[i] = kpts[keep[i]];    // keep[i] >= i: in-place is safe
  *n_kpts = (int)keep.size();
  return MVO_OK;
}

int mvo_orb_extract_batch_dev(mvo_ctx *ctx, const uint8_t *d_images, int batch, int rows, int cols, int channels,
                              size_t stride, size_t frame_stride, mvo_keypoint *d_kpts, uint8_t *d_desc,
                              int32_t *d_counts, int cap) {
  MVO_TRY(check_image(ctx, d_images, rows, cols, channels, stride));
  if (batch < 1 || !d_kpts || !d_desc || !d_counts || cap < 1) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "bad batch arguments");
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  OrbState *st = state_of(ctx);
  OrbWs ws;
  MVO_TRY(ensure_ws(ctx, st, rows, cols, batch, &ws));
  const OrbPlanDev &pl = st->plan;
  if (cap < pl.max_kpts + 1) return mvo_fail(ctx, MVO_ERR_CAPACITY, "cap %d < max_keypoints+1 = %d", cap, pl.max_kpts + 1);
  MVO_TRY(run_detect(ctx, st, ws, d_images, channels, stride, frame_stride, batch));
  MVO_TRY(orb_launch_blur(ctx, pl, ws.planes, batch));
  MVO_TRY(orb_launch_describe_sel(ctx, pl, ws.planes, ws.sel, ws.meta, nullptr, d_kpts, d_desc, d_counts, cap, 1, batch));
  // overflow check: one small D2H per batch; frames above OpenCV's per-level caps take the host path
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_a, (size_t)batch * sizeof(OrbFrameMeta)));
  OrbFrameMeta *hm = (OrbFrameMeta *)ctx->h_a.p;
  MVO_CUDA(ctx, cudaMemcpyAsync(hm, ws.meta, (size_t)batch * sizeof(OrbFrameMeta), cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  bool any = false;
  for (int f = 0; f < batch; ++f) any |= hm[f].overflow == 2;      // the device retainBest declined (see extract_end)
  if (!any) return MVO_OK;
  std::vector<int32_t> ns(batch);
  std::vector<uint32_t> cand;
  std::vector<float> harris;
  std::vector<OrbFrameMeta> metas(hm, hm + batch);
  for (int f = 0; f < batch; ++f) {
    ns[f] = metas[f].n_sel;
    if (metas[f].overflow == 2) MVO_TRY(slow_path_frame(ctx, pl, ws, f, metas[f], cand, harris, &ns[f]));
  }
  MVO_CUDA(ctx, cudaMemcpyAsync(ws.n_override, ns.data(), (size_t)batch * 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  MVO_TRY(orb_launch_describe_sel(ctx, pl, ws.planes, ws.sel, ws.meta, ws.n_override, d_kpts, d_desc, d_counts, cap, 1, batch));
  return MVO_OK;
}

}  // extern "C"
