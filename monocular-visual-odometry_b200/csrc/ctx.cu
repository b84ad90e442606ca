// Context lifetime, scratch management and error reporting for libmvo.so.
#include <stdarg.h>
#include <string.h>
#include "mvo_internal.h"

int mvo_fail(mvo_ctx *ctx, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  return code;
}

int mvo_reserve(mvo_ctx *ctx, DevBuf &b, size_t bytes) {
  if (bytes <= b.cap) return MVO_OK;
  size_t want = bytes + bytes / 4 + 256;
  if (b.p) {
    // the old block may still be in use by queued work
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    MVO_CUDA(ctx, cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
  }
  MVO_CUDA(ctx, cudaMalloc(&b.p, want));
  b.cap = want;
  return MVO_OK;
}

int mvo_reserve_pinned(mvo_ctx *ctx, PinBuf &b, size_t bytes) {
  if (bytes <= b.cap) return MVO_OK;
  size_t want = bytes + bytes / 4 + 256;
  if (b.p) {
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    MVO_CUDA(ctx, cudaFreeHost(b.p));
    b.p = nullptr;
    b.cap = 0;
  }
  MVO_CUDA(ctx, cudaMallocHost(&b.p, want));
  b.cap = want;
  return MVO_OK;
}

KTimer::KTimer(mvo_ctx *ctx, int kernel_class) : c(ctx), id(kernel_class) {
  if (!c || !(c->timing_mask & (1u << id))) { c = nullptr; return; }
  for (cudaEvent_t *e : {&a, &b}) {
    if (!c->ev_pool.empty()) { *e = c->ev_pool.back(); c->ev_pool.pop_back(); }
    else if (cudaEventCreate(e) != cudaSuccess) { c = nullptr; return; }
  }
  cudaEventRecord(a, c->stream);
}

KTimer::~KTimer() {
  if (!c) return;
  cudaEventRecord(b, c->stream);
  c->ev_pending.push_back(MvoEvPair{id, a, b});
}

static const char *kKernelNames[KC_COUNT] = {"k_gray", "k_resize", "k_fast", "k_select", "k_blur", "k_describe",
                                              "k_harris_all", "match_kernel", "k_pnp_hypotheses", "k_pnp_score",
                                              "k_pnp_finish", "k_ba", "k_track_glue", "k_epi", "k_epi_score", "k_epi_finish"};

extern "C" {

int mvo_kernel_classes(void) { return KC_COUNT; }
const char *mvo_kernel_name(int k) { return (k >= 0 && k < KC_COUNT) ? kKernelNames[k] : "?"; }

int mvo_timing_enable(mvo_ctx *ctx, uint32_t mask) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  ctx->timing_mask = mask;
  return MVO_OK;
}

int mvo_timing_read(mvo_ctx *ctx, double *ms, uint64_t *counts) {
  if (!ctx || !ms || !counts) return MVO_ERR_INVALID_ARG;
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (const MvoEvPair &p : ctx->ev_pending) {
    float t = 0;
    if (cudaEventElapsedTime(&t, p.a, p.b) == cudaSuccess) { ctx->t_ms[p.id] += t; ctx->t_cnt[p.id]++; }
    ctx->ev_pool.push_back(p.a);
    ctx->ev_pool.push_back(p.b);
  }
  ctx->ev_pending.clear();
  for (int i = 0; i < KC_COUNT; ++i) { ms[i] += ctx->t_ms[i]; counts[i] += ctx->t_cnt[i]; ctx->t_ms[i] = 0; ctx->t_cnt[i] = 0; }
  return MVO_OK;
}

void mvo_default_params(mvo_params *p) {
  if (!p) return;
  memset(p, 0, sizeof *p);
  p->orb_nfeatures = 8000;       // config/config.yaml:65
  p->orb_scale_factor = 1.2f;    // :67
  p->orb_nlevels = 4;            // :68
  p->orb_fast_threshold = 20;    // :69
  p->max_keypoints = 1500;       // :66
  p->grid_size = 16;             // :94
  p->max_pts_per_grid = 8;       // :95
  p->xiang_gao_ratio = 2.0;      // :84
  p->lowe_ratio = 1.0;           // :85 (0.8 read through Config::get<int>, feature_match.cpp:138)
  p->pnp_hypotheses = 4096;
  p->pnp_mode = 0;
  p->essential_threshold = 1.0;
  p->homography_threshold = 3.0;
  p->pnp_reproj_error = 2.0f;    // src/vo/vo.cpp:316
  p->pnp_seed = 0x9E3779B97F4A7C15ull;
  p->pnp_refine_iters = 20;
  p->ba_iterations = 50;         // src/optimization/g2o_ba.cpp:275
  p->ba_huber_delta = 1.0;
  p->ba_fix_first_pose = 0;
  p->ba_step_tol = 0.0;
  p->epi_hypotheses = 4096;
  p->eh_ratio_threshold = 0.5;  // reference src/geometry/motion_estimation.cpp:140
}

static int validate_params(mvo_ctx *ctx, const mvo_params *p) {
  if (p->orb_nlevels < 1 || p->orb_nlevels > MVO_MAX_LEVELS)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "orb_nlevels %d outside [1,%d]", p->orb_nlevels, MVO_MAX_LEVELS);
  if (p->orb_scale_factor <= 1.0f) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "orb_scale_factor must be > 1");
  if (p->orb_nfeatures < 1 || p->max_keypoints < 0 || p->grid_size < 1 || p->max_pts_per_grid < 0)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "bad keypoint selection parameters");
  if (p->orb_fast_threshold < 1 || p->orb_fast_threshold > 254)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "orb_fast_threshold outside [1,254]");
  if (!(p->essential_threshold > 0) || !(p->homography_threshold > 0)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "two-view thresholds must be positive");
  if (p->pnp_mode != 0 && p->pnp_mode != 1) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp_mode must be 0 or 1");
  if (p->pnp_hypotheses < 1 || p->pnp_hypotheses > 65535)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pnp_hypotheses outside [1,65535]");
  if (p->epi_hypotheses < 1 || p->epi_hypotheses > 65535)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "epi_hypotheses outside [1,65535]");
  if (!(p->eh_ratio_threshold > 0 && p->eh_ratio_threshold < 1))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "eh_ratio_threshold outside (0,1)");
  if (p->ba_iterations < 0 || p->pnp_refine_iters < 0)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "negative iteration count");
  return MVO_OK;
}

int mvo_create(mvo_ctx **out, int device, const mvo_params *params) {
  if (!out) return MVO_ERR_INVALID_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    cudaGetLastError();
    return MVO_ERR_NO_DEVICE;   // no CPU fallback by design
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return MVO_ERR_NO_DEVICE;
  if (prop.major != 9 || prop.minor != 0) {
    fprintf(stderr, "libmvo: device %d is sm_%d%d; this library contains sm_90a code only\n", device,
            prop.major, prop.minor);
    return MVO_ERR_NO_DEVICE;
  }
  if (cudaSetDevice(device) != cudaSuccess) return MVO_ERR_NO_DEVICE;
  mvo_ctx *ctx = new mvo_ctx();
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  mvo_default_params(&ctx->prm);
  if (params) {
    int rc = validate_params(nullptr, params);
    if (rc != MVO_OK) { delete ctx; return rc; }
    ctx->prm = *params;
  }
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return MVO_ERR_CUDA;
  }
  ctx->own_stream = true;
  const size_t ticket_bytes = 4096 * sizeof(unsigned int);
  if (mvo_reserve(ctx, ctx->match_tickets, ticket_bytes) != MVO_OK ||
      cudaMemsetAsync(ctx->match_tickets.p, 0, ctx->match_tickets.cap, ctx->stream) != cudaSuccess) {
    mvo_destroy(ctx);
    return MVO_ERR_CUDA;
  }
  *out = ctx;
  return MVO_OK;
}

void mvo_destroy(mvo_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  orb_state_free(ctx);
  orb_tma_free(ctx);
  DevBuf *dbs[] = {&ctx->d_b, &ctx->d_c, &ctx->d_d, &ctx->d_f, &ctx->orb_planes,
                   &ctx->orb_cand, &ctx->orb_bandcnt, &ctx->orb_sel, &ctx->orb_misc, &ctx->orb_in,
                   &ctx->orb_kpts, &ctx->orb_desc, &ctx->orb_counts, &ctx->match_part,
                   &ctx->match_tickets, &ctx->match_in, &ctx->match_keys, &ctx->matchb_part, &ctx->matchb_tickets,
                   &ctx->matchb_keys, &ctx->epib_buf, &ctx->epi_ess_buf, &ctx->epi_homo_buf, &ctx->pnp_pts, &ctx->pnp_hyp,
                   &ctx->pnp_cnt, &ctx->pnp_out, &ctx->ba_buf};
  for (DevBuf *b : dbs)
    if (b->p) cudaFree(b->p);
  PinBuf *pbs[] = {&ctx->h_a, &ctx->h_b, &ctx->epi_ess_h, &ctx->epi_homo_h, &ctx->orb_h, &ctx->match_h};
  for (PinBuf *b : pbs)
    if (b->p) cudaFreeHost(b->p);
  for (const MvoEvPair &p : ctx->ev_pending) { cudaEventDestroy(p.a); cudaEventDestroy(p.b); }
  for (cudaEvent_t e : ctx->ev_pool) cudaEventDestroy(e);
  if (ctx->side_stream) cudaStreamDestroy(ctx->side_stream);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char *mvo_last_error(const mvo_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int mvo_get_params(const mvo_ctx *ctx, mvo_params *out) {
  if (!ctx || !out) return MVO_ERR_INVALID_ARG;
  *out = ctx->prm;
  return MVO_OK;
}

int mvo_set_params(mvo_ctx *ctx, const mvo_params *p) {
  if (!ctx || !p) return MVO_ERR_INVALID_ARG;
  MVO_TRY(validate_params(ctx, p));
  const bool orb_changed = p->orb_nlevels != ctx->prm.orb_nlevels ||
                           p->orb_scale_factor != ctx->prm.orb_scale_factor ||
                           p->orb_nfeatures != ctx->prm.orb_nfeatures;
  ctx->prm = *p;
  if (orb_changed) ctx->orb.rows = ctx->orb.cols = 0;   // force a re-plan of the pyramid layout
  return MVO_OK;
}

int mvo_set_stream(mvo_ctx *ctx, void *cuda_stream) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  ctx->stream = (cudaStream_t)cuda_stream;
  ctx->own_stream = false;
  return MVO_OK;
}

int mvo_synchronize(mvo_ctx *ctx) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MVO_OK;
}

uint64_t mvo_kernel_launches(const mvo_ctx *ctx) { return ctx ? ctx->launches : 0; }

}  // extern "C"

cudaStream_t mvo_side_stream(mvo_ctx *ctx) {
  if (!ctx->side_stream) {
    cudaSetDevice(ctx->device);
    if (cudaStreamCreateWithFlags(&ctx->side_stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); ctx->side_stream = nullptr; }
  }
  return ctx->side_stream;
}

