// ORB extraction kernels for sm_90a — bit-exact with OpenCV 4.13's cv::ORB as the reference
// calls it (src/geometry/feature_match.cpp:22-23,34,45,48) followed by the reference's own
// first-come grid selection (feature_match.cpp:51-84).  Algorithm: SURVEY.md Appendix A.
//
// HBM layout per frame slot: for every pyramid level one gray plane and one blurred plane,
// rows padded to a multiple of 128 B (16-byte vector / TMA-legal strides).  No 32-px border is
// materialised: with edgeThreshold 31 no bit-exact result ever depends on it (FAST needs 3+1 px,
// Harris 4, the orientation disc 15, rotated BRIEF samples <= 19 px from the keypoint).
//
// Kernels (all batched over frames in grid.y / grid.z):
//   k_gray        BGR -> gray, fixed point (3735 B + 19235 G + 9798 R + 16384) >> 15
//   k_resize      level l from level l-1, INTER_LINEAR_EXACT (8.8 x 8.8 fixed point, host tables)
//   k_fast        one CTA per 8-row band: image rows staged in shared memory, quick 4-point
//                 reject, cornerScore<16> only for survivors, 3x3 NMS, raster-ordered emit
//   k_select      one CTA per frame: candidate compaction + first-come grid selection, restated
//                 as rank-in-cell < max_per_cell and an ordered prefix count (deterministic)
//   k_blur2       7x7 sigma-2 Gaussian, float separable, round-half-even (ORB's descriptor blur; orb_variants.cuh)
//   k_describe    one warp per keypoint: Harris response, intensity-centroid angle, 256 steered
//                 BRIEF tests (lane i produces descriptor byte i)
// Float formulas that OpenCV evaluates without FMA use __fmul_rn/__fadd_rn explicitly.
#include <cooperative_groups.h>
#include <cuda.h>               // CUtensorMap: the FAST band tiles are staged by TMA (cp.async.bulk.tensor)
#include <stdlib.h>
#include "orb.cuh"
#include "launch_pdl.cuh"   // the extraction chain is launched with programmatic dependent launch: every kernel starts with pdl_wait()

namespace cg = cooperative_groups;

namespace {

#include "orb_pattern.inc"   // __constant__-free table: static const signed char kOrbPattern[512][2]

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// ------------------------------------------------------------------------------------ gray
__global__ void __launch_bounds__(128)
k_gray(OrbPlanDev plan, const uint8_t *__restrict__ in, int channels, size_t stride, size_t frame_stride,
       uint8_t *__restrict__ planes) {
  pdl_wait();
  pdl_launch_dependents();
  const int y = blockIdx.y, f = blockIdx.z;
  const int x4 = (blockIdx.x * 128 + threadIdx.x) * 4;
  const int w = plan.lv[0].w, pitch = plan.lv[0].pitch;
  if (x4 >= pitch) return;
  const uint8_t *row = in + (size_t)f * frame_stride + (size_t)y * stride;
  uint32_t out = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int x = x4 + i;
    uint32_t g = 0;
    if (x < w) {
      if (channels == 3) {
        const uint32_t b = row[3 * x], gg = row[3 * x + 1], r = row[3 * x + 2];
        g = (3735u * b + 19235u * gg + 9798u * r + 16384u) >> 15;
      } else {
        g = row[x];
      }
    }
    out |= g << (8 * i);
  }
  uint8_t *dst = planes + (size_t)f * plan.slot_bytes + plan.lv[0].img_off + (size_t)y * pitch;
  *reinterpret_cast<uint32_t *>(dst + x4) = out;
}

// ---------------------------------------------------------------------------------- resize
__global__ void __launch_bounds__(128)
k_resize(OrbPlanDev plan, int level, const int32_t *__restrict__ tables, uint8_t *__restrict__ planes) {
  pdl_wait();
  pdl_launch_dependents();
  const OrbLevelDev &L = plan.lv[level];
  const OrbLevelDev &S = plan.lv[level - 1];
  const int y = blockIdx.y, f = blockIdx.z;
  const int x4 = (blockIdx.x * 128 + threadIdx.x) * 4;
  if (x4 >= L.pitch) return;
  const int32_t *xofs = tables + L.tab_off, *xw1 = xofs + L.w, *yofs = xw1 + L.w, *yw1 = yofs + L.h;
  uint8_t *slot = planes + (size_t)f * plan.slot_bytes;
  const int oy = yofs[y], wy1 = yw1[y], wy0 = 256 - wy1;
  const int oy1 = min(oy + 1, S.h - 1);
  const uint8_t *r0 = slot + S.img_off + (size_t)oy * S.pitch;
  const uint8_t *r1 = slot + S.img_off + (size_t)oy1 * S.pitch;
  uint32_t out = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int x = x4 + i;
    uint32_t v = 0;
    if (x < L.w) {
      const int ox = xofs[x], wx1 = xw1[x], wx0 = 256 - wx1;
      const int ox1 = min(ox + 1, S.w - 1);
      const int h0 = r0[ox] * wx0 + r0[ox1] * wx1;
      const int h1 = r1[ox] * wx0 + r1[ox1] * wx1;
      v = (uint32_t)(h0 * wy0 + h1 * wy1 + 32768) >> 16;
    }
    out |= v << (8 * i);
  }
  *reinterpret_cast<uint32_t *>(slot + L.img_off + (size_t)y * L.pitch + x4) = out;
}

// ------------------------------------------------------------------- gray + pyramid, fused
// k_gray and the k_resize chain in ONE launch: a CTA takes a horizontal band of the image, converts the rows of level 0 it has to
// hold into shared memory, derives its rows of level 1 from those, level 2 from level 1, ... (each level is resized from the
// ROUNDED level below, as OpenCV's pyramid is) and writes the rows it OWNS of every level (orb_host.cpp: band table; neighbouring
// bands recompute the few rows they share).  Same arithmetic as k_gray / k_resize, so the planes are bit-identical; three
// launches, their gaps and two round trips of the lower levels through L2 go away.
constexpr int PYR_T = 256;

__device__ __forceinline__ uint32_t gray4(const uint8_t *__restrict__ row, int x4, int w, int channels, bool aligned) {
  if (x4 >= w) return 0;
  if (channels == 3) {
    if (aligned && x4 + 4 <= w) {
      const uint32_t *p = reinterpret_cast<const uint32_t *>(row + 3 * (size_t)x4);
      const uint32_t a = p[0], b = p[1], c = p[2];                 // B0 G0 R0 B1 | G1 R1 B2 G2 | R2 B3 G3 R3
      const uint32_t g0 = (3735u * (a & 0xFF) + 19235u * ((a >> 8) & 0xFF) + 9798u * ((a >> 16) & 0xFF) + 16384u) >> 15;
      const uint32_t g1 = (3735u * (a >> 24) + 19235u * (b & 0xFF) + 9798u * ((b >> 8) & 0xFF) + 16384u) >> 15;
      const uint32_t g2 = (3735u * ((b >> 16) & 0xFF) + 19235u * (b >> 24) + 9798u * (c & 0xFF) + 16384u) >> 15;
      const uint32_t g3 = (3735u * ((c >> 8) & 0xFF) + 19235u * ((c >> 16) & 0xFF) + 9798u * (c >> 24) + 16384u) >> 15;
      return g0 | (g1 << 8) | (g2 << 16) | (g3 << 24);
    }
    uint32_t out = 0;
    for (int i = 0; i < 4; ++i) {
      const int x = x4 + i;
      if (x < w) {
        const uint32_t b = row[3 * x], gg = row[3 * x + 1], r = row[3 * x + 2];
        out |= ((3735u * b + 19235u * gg + 9798u * r + 16384u) >> 15) << (8 * i);
      }
    }
    return out;
  }
  uint32_t out = 0;
  for (int i = 0; i < 4; ++i)
    if (x4 + i < w) out |= (uint32_t)row[x4 + i] << (8 * i);
  return out;
}

__global__ void __launch_bounds__(PYR_T)
k_pyramid(OrbPlanDev plan, const uint8_t *__restrict__ in, int channels, size_t stride, size_t frame_stride,
          const int32_t *__restrict__ tables, uint8_t *__restrict__ planes) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(128) uint8_t smem[];
  const int b = blockIdx.x, f = blockIdx.y, tid = threadIdx.x;
  const int nl = plan.nlevels;
  const int32_t *bt = tables + plan.pyr_tab_off + (size_t)b * nl * 4;
  uint8_t *slot = planes + (size_t)f * plan.slot_bytes;
  // level 0
  uint8_t *s_prev = smem;
  int plo = bt[0];
  {
    const OrbLevelDev &L = plan.lv[0];
    const int lo = bt[0], hi = bt[1], olo = bt[2], ohi = bt[3], wpr = L.pitch >> 2;
    const uint8_t *base = in + (size_t)f * frame_stride;
    const bool aligned = ((reinterpret_cast<uintptr_t>(base) | stride) & 3) == 0;
    const bool keep = nl > 1;                                      // a single level is not a source: no shared memory is sized for it
    for (int i = tid; i < (hi - lo) * wpr; i += PYR_T) {
      const int r = i / wpr, x4 = (i - r * wpr) << 2, y = lo + r;
      const uint32_t v = gray4(base + (size_t)y * stride, x4, L.w, channels, aligned);
      if (keep) *reinterpret_cast<uint32_t *>(s_prev + (size_t)r * L.pitch + x4) = v;
      if (y >= olo && y < ohi) *reinterpret_cast<uint32_t *>(slot + L.img_off + (size_t)y * L.pitch + x4) = v;
    }
  }
  __syncthreads();
  for (int l = 1; l < nl; ++l) {
    const OrbLevelDev &L = plan.lv[l];
    const OrbLevelDev &S = plan.lv[l - 1];
    const int32_t *e = bt + 4 * l;
    const int lo = e[0], hi = e[1], olo = e[2], ohi = e[3], wpr = L.pitch >> 2;
    const int32_t *xofs = tables + L.tab_off, *xw1 = xofs + L.w, *yofs = xw1 + L.w, *yw1 = yofs + L.h;
    uint8_t *s_cur = s_prev + (size_t)plan.pyr_rows[l - 1] * S.pitch;
    const bool keep = l + 1 < nl;                                  // the top level is not a source
    for (int i = tid; i < (hi - lo) * wpr; i += PYR_T) {
      const int r = i / wpr, x4 = (i - r * wpr) << 2, y = lo + r;
      const int oy = yofs[y], wy1 = yw1[y], wy0 = 256 - wy1;
      const int oy1 = min(oy + 1, S.h - 1);
      const uint8_t *r0 = s_prev + (size_t)(oy - plo) * S.pitch, *r1 = s_prev + (size_t)(oy1 - plo) * S.pitch;
      uint32_t out = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int x = x4 + k;
        uint32_t v = 0;
        if (x < L.w) {
          const int ox = __ldg(xofs + x), wx1 = __ldg(xw1 + x), wx0 = 256 - wx1;
          const int ox1 = min(ox + 1, S.w - 1);
          const int h0 = r0[ox] * wx0 + r0[ox1] * wx1;
          const int h1 = r1[ox] * wx0 + r1[ox1] * wx1;
          v = (uint32_t)(h0 * wy0 + h1 * wy1 + 32768) >> 16;
        }
        out |= v << (8 * k);
      }
      if (keep) *reinterpret_cast<uint32_t *>(s_cur + (size_t)r * L.pitch + x4) = out;
      if (y >= olo && y < ohi) *reinterpret_cast<uint32_t *>(slot + L.img_off + (size_t)y * L.pitch + x4) = out;
    }
    __syncthreads();
    s_prev = s_cur;
    plo = lo;
  }
}

// ------------------------------------------------------------------------------------ FAST
// cornerScore<16> (OpenCV fast_score.cpp) == max(t, A, B) - 1 with
//   A = max over the 16 arcs of 9 contiguous ring pixels of min(d), B the same for -d,
//   d[k] = centre - ring[k]; the pixel is a FAST-9 corner iff max(A, B) > t.
__device__ __forceinline__ int fast_score(const uint8_t *__restrict__ p, int stride, int t) {
  const int c = p[0];
  int d[16];
  d[0] = c - p[3 * stride];      d[1] = c - p[3 * stride + 1];   d[2] = c - p[2 * stride + 2];
  d[3] = c - p[stride + 3];      d[4] = c - p[3];                d[5] = c - p[-stride + 3];
  d[6] = c - p[-2 * stride + 2]; d[7] = c - p[-3 * stride + 1];  d[8] = c - p[-3 * stride];
  d[9] = c - p[-3 * stride - 1]; d[10] = c - p[-2 * stride - 2]; d[11] = c - p[-stride - 3];
  d[12] = c - p[-3];             d[13] = c - p[stride - 3];      d[14] = c - p[2 * stride - 2];
  d[15] = c - p[3 * stride - 1];
  int mn3[16], mx3[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    mn3[k] = min(min(d[k], d[(k + 1) & 15]), d[(k + 2) & 15]);
    mx3[k] = max(max(d[k], d[(k + 1) & 15]), d[(k + 2) & 15]);
  }
  int A = -1000, B = 1000;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    A = max(A, min(min(mn3[k], mn3[(k + 3) & 15]), mn3[(k + 6) & 15]));
    B = min(B, max(max(mx3[k], mx3[(k + 3) & 15]), mx3[(k + 6) & 15]));
  }
  const int m = max(A, -B);
  return m > t ? m - 1 : 0;
}

// One tensor map per pyramid level over the gray planes of all frame slots: (x in 4-byte words, y, frame slot), box =
// one whole band: pitch / 4 words x 16 rows x 1 frame.  TMA = true: one elected thread issues a single
// cp.async.bulk.tensor.3d for the band's 16 image rows (rows past the image are zero-filled by the unit) and the CTA waits on
// the mbarrier it completes; no thread moves image bytes through registers.  TMA = false: 16-byte vector loads (images wider
// than 1024 pixels, whose rows do not fit a 256-element box, and the CPU test tier).
struct FastMaps { CUtensorMap m[MVO_MAX_LEVELS]; };

#ifndef __CUDA_ARCH__
#ifndef __grid_constant__
#define __grid_constant__
#endif
#endif

template <bool TMA>
__global__ void __launch_bounds__(256)
k_fast(OrbPlanDev plan, const uint8_t *__restrict__ planes, uint32_t *__restrict__ staging,
       int32_t *__restrict__ bandcnt, const __grid_constant__ FastMaps maps) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(128) uint8_t smem[];
  const int band = blockIdx.x, f = blockIdx.y;
  int l = 0;
#pragma unroll 1
  while (l + 1 < plan.nlevels && band >= plan.lv[l + 1].band_first) ++l;
  const OrbLevelDev &L = plan.lv[l];
  const int w = L.w, h = L.h, pitch = L.pitch;
  const int t = plan.fast_threshold;
  const int y0 = ORB_EDGE + (band - L.band_first) * ORB_BAND_H;     // first NMS row
  const int nms_rows = min(ORB_BAND_H, h - ORB_EDGE - y0);
  const int sstride = TMA ? pitch : pitch + 16;                      // TMA lands dense rows; the vector path de-aliases rows across banks
  const int img_rows = nms_rows + 8;                                 // rows y0-4 .. y0+nms_rows+3
  const int sc_rows = nms_rows + 2;                                  // rows y0-1 .. y0+nms_rows
  const int w32 = (w + 31) >> 5;

  uint8_t *s_img = smem;                                             // [ORB_BAND_H+8][sstride]
  uint8_t *s_sc = s_img + (ORB_BAND_H + 8) * sstride;                // [ORB_BAND_H+2][sstride]
  uint32_t *s_bits = reinterpret_cast<uint32_t *>(s_sc + (ORB_BAND_H + 2) * sstride);   // [ORB_BAND_H][w32]
  uint16_t *s_list = reinterpret_cast<uint16_t *>(s_bits + ORB_BAND_H * w32);           // [(ORB_BAND_H+2)*w]
  __shared__ int s_cnt;
  __shared__ int s_wsum[8];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint8_t *img = planes + (size_t)f * plan.slot_bytes + L.img_off;

  // stage image rows (TMA: one bulk tensor copy of the whole band; otherwise whole padded rows as 16-byte vectors), clear
  // score rows and the keep bitmap
  __shared__ __align__(8) unsigned long long s_bar;
  {
    bool staged = false;
#if defined(__CUDA_ARCH__)
    if (TMA) {
      const unsigned bar = (unsigned)__cvta_generic_to_shared(&s_bar), dst = (unsigned)__cvta_generic_to_shared(s_img);
      if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        const unsigned bytes = (unsigned)((ORB_BAND_H + 8) * pitch);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        const unsigned long long mp = reinterpret_cast<unsigned long long>(&maps.m[l]);
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                     ::"r"(dst), "l"(mp), "r"(0), "r"(y0 - 4), "r"(f), "r"(bar) : "memory");
      }
      staged = true;
    }
#endif
    if (!staged) {
      const int vec_per_row = pitch >> 4;
      for (int i = tid; i < img_rows * vec_per_row; i += 256) {
        const int r = i / vec_per_row, v = i - r * vec_per_row;
        const uint4 val = *reinterpret_cast<const uint4 *>(img + (size_t)(y0 - 4 + r) * pitch + v * 16);
        *reinterpret_cast<uint4 *>(s_img + r * sstride + v * 16) = val;
      }
    }
    const int svec = (sc_rows * sstride) >> 4;
    for (int i = tid; i < svec; i += 256) reinterpret_cast<uint4 *>(s_sc)[i] = make_uint4(0, 0, 0, 0);
    for (int i = tid; i < ORB_BAND_H * w32; i += 256) s_bits[i] = 0;
    if (tid == 0) s_cnt = 0;
  }
  __syncthreads();
#if defined(__CUDA_ARCH__)
  if (TMA) {                                                        // the band has landed when the mbarrier's phase 0 completes
    const unsigned bar = (unsigned)__cvta_generic_to_shared(&s_bar);
    unsigned done = 0;
    for (int spin = 0; !done; ++spin) {
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(bar), "r"(0) : "memory");
      if (spin > (1 << 24)) __trap();                               // a faulty descriptor must not hang the GPU
    }
  }
#endif

  // phase 1: quick reject on the 4 compass points; survivors go to a shared list.
  // An arc of 9 contiguous ring pixels always contains one of {0,8} and one of {4,12}.
  // Four pixels per thread, as packed bytes: the centre word, the words 3 rows above / below and the two words beside it give the
  // four compass neighbours of the 4 pixels; |neighbour - centre| comes from one VABSDIFF4 each and "> t" for all four bytes from an
  // add-and-mask, so the common case (no candidate among the 4 pixels) costs ~30 instructions per WORD.  That packed test ignores the
  // sign of the difference (a superset of the reference's bright / dark test); the few bytes that pass it are re-tested exactly.
  if (t <= 127) {
    const int x_lo = ORB_EDGE - 1, x_hi = w - (ORB_EDGE - 1);         // columns 30 .. w-31
    const int w0 = x_lo >> 2, wpr = ((x_hi + 3) >> 2) - w0;           // words of a row that hold such columns
    const unsigned inv = (unsigned)(((1u << 24) + (unsigned)wpr - 1u) / (unsigned)wpr);      // i / wpr = (i * inv) >> 24 for i < 4096 * ...
    const uint32_t K4 = (uint32_t)(0x7F - t) * 0x01010101u;
    const int items = sc_rows * wpr;
    for (int i0 = 0; i0 < items; i0 += 256) {
      const int i = i0 + tid;
      uint32_t sup = 0, c = 0, wa = 0, wb = 0, we = 0, wg = 0;
      int r = 0, xw = 0;
      if (i < items) {
        r = (int)(((unsigned long long)(unsigned)i * inv) >> 24);     // score row (image row y0-1+r)
        xw = (w0 + (i - r * wpr)) << 2;
        const uint32_t *row = reinterpret_cast<const uint32_t *>(s_img + (r + 3) * sstride + xw);
        const int sw = sstride >> 2;
        c = row[0];
        wa = row[3 * sw]; wb = row[-3 * sw];
        const uint32_t prev = row[-1], next = row[1];
        we = (c >> 24) | (next << 8);                                   // pixels x + 3
        wg = (prev >> 8) | (c << 24);                                   // pixels x - 3
        const uint32_t da = __vabsdiffu4(wa, c), db = __vabsdiffu4(wb, c), de = __vabsdiffu4(we, c), dg = __vabsdiffu4(wg, c);
        const uint32_t ga = ((da & 0x7F7F7F7Fu) + K4) | da, gb = ((db & 0x7F7F7F7Fu) + K4) | db;
        const uint32_t ge = ((de & 0x7F7F7F7Fu) + K4) | de, gg = ((dg & 0x7F7F7F7Fu) + K4) | dg;
        sup = (ga | gb) & (ge | gg) & 0x80808080u;
        if (sup) {                                                      // exact test of the bytes that passed, columns outside [30, w-30) dropped
          uint32_t ex = 0;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (!(sup & (0x80u << (8 * k)))) continue;
            const int x = xw + k;
            if (x < x_lo || x >= x_hi) continue;
            const int cc = (c >> (8 * k)) & 0xFF, hi = cc + t, lo = cc - t;
            const int a = (wa >> (8 * k)) & 0xFF, bb = (wb >> (8 * k)) & 0xFF, e = (we >> (8 * k)) & 0xFF, g = (wg >> (8 * k)) & 0xFF;
            const bool bright = (a > hi || bb > hi) && (e > hi || g > hi);
            const bool dark = (a < lo || bb < lo) && (e < lo || g < lo);
            if (bright || dark) ex |= 1u << k;
          }
          sup = ex;
        }
      }
      if (__any_sync(0xffffffffu, sup != 0)) {
        // ordered by (byte position, lane) inside the warp; the list order does not matter downstream
        const unsigned m0 = __ballot_sync(0xffffffffu, sup & 1u), m1 = __ballot_sync(0xffffffffu, sup & 2u);
        const unsigned m2 = __ballot_sync(0xffffffffu, sup & 4u), m3 = __ballot_sync(0xffffffffu, sup & 8u);
        const int n0 = __popc(m0), n1 = __popc(m1), n2 = __popc(m2), n3 = __popc(m3);
        int base = 0;
        if (lane == 0) base = atomicAdd(&s_cnt, n0 + n1 + n2 + n3);
        base = __shfl_sync(0xffffffffu, base, 0);
        const unsigned lt = lanemask_lt();
        const uint16_t ent = (uint16_t)((r << 12) | xw);
        if (sup & 1u) s_list[base + __popc(m0 & lt)] = ent;
        if (sup & 2u) s_list[base + n0 + __popc(m1 & lt)] = (uint16_t)(ent + 1);
        if (sup & 4u) s_list[base + n0 + n1 + __popc(m2 & lt)] = (uint16_t)(ent + 2);
        if (sup & 8u) s_list[base + n0 + n1 + n2 + __popc(m3 & lt)] = (uint16_t)(ent + 3);
      }
    }
  } else {                                                             // thresholds beyond the packed compare: one pixel per lane
    const int xspan = w - 2 * (ORB_EDGE - 1);                        // columns 30 .. w-31
    const int nseg = (xspan + 31) >> 5;
    for (int s = warp; s < sc_rows * nseg; s += 8) {
      const int r = s / nseg, seg = s - r * nseg;                    // r: score row (image row y0-1+r)
      const int x = (ORB_EDGE - 1) + seg * 32 + lane;
      bool pass = false;
      if (x < w - (ORB_EDGE - 1)) {
        const uint8_t *p = s_img + (r + 3) * sstride + x;            // s_img row of image row y0-1+r
        const int c = p[0], hi = c + t, lo = c - t;
        const int a = p[3 * sstride], b = p[-3 * sstride], e = p[3], g = p[-3];
        const bool bright = (a > hi || b > hi) && (e > hi || g > hi);
        const bool dark = (a < lo || b < lo) && (e < lo || g < lo);
        pass = bright || dark;
      }
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (m) {
        int base = 0;
        if (lane == 0) base = atomicAdd(&s_cnt, __popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (pass) s_list[base + __popc(m & lanemask_lt())] = (uint16_t)((r << 12) | x);
      }
    }
  }
  __syncthreads();
  const int ncand = s_cnt;

  // phase 2: exact corner score for the survivors
  for (int i = tid; i < ncand; i += 256) {
    const int e = s_list[i], r = e >> 12, x = e & 0xFFF;
    const int sc = fast_score(s_img + (r + 3) * sstride + x, sstride, t);
    if (sc) s_sc[r * sstride + x] = (uint8_t)sc;
  }
  __syncthreads();

  // phase 3: 3x3 non-maximum suppression (strictly greater than all 8 neighbours), border filter
  for (int i = tid; i < ncand; i += 256) {
    const int e = s_list[i], r = e >> 12, x = e & 0xFFF;
    if (r < 1 || r > nms_rows || x < ORB_EDGE || x >= w - ORB_EDGE) continue;
    const uint8_t *q = s_sc + r * sstride + x;
    const int sc = q[0];
    if (sc == 0) continue;
    const bool keep = sc > q[-1] && sc > q[1] && sc > q[-sstride - 1] && sc > q[-sstride] && sc > q[-sstride + 1] &&
                      sc > q[sstride - 1] && sc > q[sstride] && sc > q[sstride + 1];
    if (keep) atomicOr(&s_bits[(r - 1) * w32 + (x >> 5)], 1u << (x & 31));
  }
  __syncthreads();

  // phase 4: raster-ordered emit.  Thread i owns a contiguous run of bitmap words.
  {
    const int nwords = nms_rows * w32;
    const int wpt = (nwords + 255) >> 8;
    const int wb = tid * wpt, we = min(wb + wpt, nwords);
    int mine = 0;
    for (int i = wb; i < we; ++i) mine += __popc(s_bits[i]);
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) s_wsum[warp] = incl;
    __syncthreads();
    int off = incl - mine, total = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (k < warp) off += s_wsum[k];
      total += s_wsum[k];
    }
    uint32_t *out = staging + ((size_t)f * plan.total_bands + band) * plan.band_cap;
    for (int i = wb; i < we; ++i) {
      uint32_t bits = s_bits[i];
      const int r = i / w32, xb = (i - r * w32) << 5;
      while (bits) {
        const int b = __ffs(bits) - 1;
        bits &= bits - 1;
        const int x = xb + b;
        out[off++] = orb_pack(x, y0 + r, s_sc[(r + 1) * sstride + x]);
      }
    }
    if (tid == 0) bandcnt[(size_t)f * plan.total_bands + band] = total;
  }
}

// Cell of a keypoint in the uncovered strip right of column grid_cols * grid_size or below row grid_rows * grid_size (images whose
// size is not a multiple of the grid size).  The reference indexes its grid out of range there (feature_match.cpp:70-72, undefined
// behaviour); the project's reading is that such a keypoint is skipped: it is not kept and uses up no cell's quota.  The host
// selection (orb_host.cpp: grid_select) and the oracle do the same, so a frame selects the same keypoints on every path.
constexpr int ORB_NO_CELL = 0xFFFF;      // grid_rows * grid_cols <= 65535: never a real cell

// cell index = (int)coordinate / grid_size (feature_match.cpp:70): a shift when the grid size is a power of two (the coordinates are >= 0)
__device__ __forceinline__ int orb_grid_shift(int g) {
  if (g <= 0 || (g & (g - 1)) != 0) return -1;
  int sh = 0;
  while ((1 << sh) < g) ++sh;
  return sh;
}

// keep[i] = 1 iff fewer than max_per_cell items j < i lie in item i's cell: the per-cell counter of selectUniformKptsByGrid
// (feature_match.cpp:68-81) in closed form.  max_per_cell rounds: in round r every pending item bids its index for its cell with an
// atomicMin, the smallest pending index of a cell wins the round and is kept.  Bids carry the round in their high half
// ((0xFFFF - r) << 16 | index: later rounds bid lower values), so the two bid arrays (rounds alternate between them) never need a reset,
// and one block barrier per round suffices: winners of round r - 1 are read from the array round r does not write.
// (Round 1 ranked every item against its whole cell bucket: quadratic in the population of the crowded cells.)
// Called by all 1024 threads; s_min: 2 * ncell words; item indices < 65536.
__device__ __forceinline__ void grid_rank_keep(int n, const uint16_t *__restrict__ s_cell, uint8_t *__restrict__ s_keep, uint32_t *__restrict__ s_min,
                                               int ncell, int max_per_cell) {
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * ncell; i += 1024) s_min[i] = 0xFFFFFFFFu;
  for (int i = tid; i < n; i += 1024) s_keep[i] = 0;
  __syncthreads();
  max_per_cell = min(max_per_cell, n);                     // a cell never holds more than n items (keeps the round tag inside 16 bits)
  for (int r = 0; r <= max_per_cell; ++r) {
    uint32_t *cur = s_min + (r & 1) * ncell;
    const uint32_t *prev = s_min + ((r & 1) ^ 1) * ncell;
    const uint32_t tag = (uint32_t)(0xFFFF - r) << 16, tag_prev = (uint32_t)(0xFFFF - (r - 1)) << 16;
    for (int i = tid; i < n; i += 1024) {
      if (s_keep[i]) continue;
      const int c = s_cell[i];
      if (c == ORB_NO_CELL) continue;
      if (r > 0 && prev[c] == (tag_prev | (uint32_t)i)) { s_keep[i] = 1; continue; }
      if (r < max_per_cell) atomicMin(&cur[c], tag | (uint32_t)i);
    }
    __syncthreads();
  }
}

// The same keep flags in two passes instead of max_per_cell rounds over all items (which cost 9 x 8000 item visits for an
// above-cap frame): the 32 warps of the CTA take 32 contiguous segments of the item list.  Pass 1: a warp walks its segment 32 items
// at a time; __match_any_sync groups the lanes by cell, rank inside the segment = the cell's count so far in this warp's private
// table + the number of lower lanes of the group; the group's highest lane adds the group size to the table.  Pass 2: exclusive
// prefix of the 32 tables per cell (one thread per cell).  Pass 3: keep = segment rank + prefix < max_per_cell.  Counts saturate
// at 255, which is exact while max_per_cell <= 254 (the caller falls back to the round version otherwise).
// s_tab: 32 x ncell bytes.  s_keep holds the segment ranks between the passes.
__device__ __forceinline__ void grid_rank_keep_seg(int n, const uint16_t *__restrict__ s_cell, uint8_t *__restrict__ s_keep, uint8_t *__restrict__ s_tab,
                                                   int ncell, int max_per_cell) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 8 * ncell; i += 1024) reinterpret_cast<uint32_t *>(s_tab)[i] = 0;       // 32 * ncell bytes, ncell-major per warp
  __syncthreads();
  const int seg = (((n + 31) >> 5) + 31) & ~31;               // items per warp: a multiple of 32
  const int b = min(warp * seg, n), e = min(b + seg, n);
  uint8_t *tab = s_tab + (size_t)warp * ncell;
  const unsigned lt = lanemask_lt();
  for (int i0 = b; i0 < e; i0 += 32) {
    const int i = i0 + lane;
    const bool in = i < e && s_cell[i] != ORB_NO_CELL;
    const unsigned c = in ? (unsigned)s_cell[i] : 0xFFFF0000u + (unsigned)lane;      // lanes past the end or outside the grid: a group of their own
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    const int leader = 31 - __clz((int)peers);               // only the group's highest lane touches the count: one warp barrier per step
    int base = 0;
    if (in && lane == leader) base = (int)tab[c];
    base = __shfl_sync(0xffffffffu, base, leader);
    if (in) {
      s_keep[i] = (uint8_t)min(base + __popc(peers & lt), 255);
      if (lane == leader) tab[c] = (uint8_t)min(base + __popc(peers), 255);
    }
    __syncwarp();
  }
  __syncthreads();
  for (int c = tid; c < ncell; c += 1024) {
    int run = 0;
#pragma unroll 8
    for (int w = 0; w < 32; ++w) {
      const int v = s_tab[(size_t)w * ncell + c];
      s_tab[(size_t)w * ncell + c] = (uint8_t)min(run, 255);
      run += v;
    }
  }
  __syncthreads();
  for (int i0 = b; i0 < e; i0 += 32) {
    const int i = i0 + lane;
    if (i < e) {
      const int c = s_cell[i];
      s_keep[i] = (uint8_t)(c != ORB_NO_CELL && ((int)s_keep[i] + (int)tab[c]) < max_per_cell);
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------- select
// Restates feature_match.cpp:68-81: walking keypoints in order, a keypoint is kept iff fewer than
// max_per_cell earlier keypoints fell into its 16x16 cell, and the walk stops right after the
// (max_kpts+1)-th kept keypoint.  Equivalent closed form: kept0 = (rank in cell < max_per_cell),
// kept = kept0 && (#kept0 before it) <= max_kpts.
__global__ void __launch_bounds__(1024)
k_select(OrbPlanDev plan, const uint32_t *__restrict__ staging, const int32_t *__restrict__ bandcnt,
         uint32_t *__restrict__ cand, uint2 *__restrict__ sel, OrbFrameMeta *__restrict__ meta, int seg_tab) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(128) uint8_t smem[];
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ncell = plan.grid_rows * plan.grid_cols;
  const int cap = plan.cand_cap, scap = plan.sel_cap;
  int32_t *s_boff = reinterpret_cast<int32_t *>(smem);            // [total_bands + 1]
  int32_t *s_cellcnt = s_boff + ORB_MAX_BANDS + 1;                // [ncell + 1]  start offsets after scan
  int32_t *s_cursor = s_cellcnt + ncell + 1;                      // [ncell]
  uint16_t *s_cell = reinterpret_cast<uint16_t *>(s_cursor + ncell);   // [cap] cell of candidate i
  uint16_t *s_bucket = s_cell + scap;                             // [cap] candidate ids grouped by cell
  uint8_t *s_keep = reinterpret_cast<uint8_t *>(s_bucket + scap);  // [cap]
  uint8_t *s_tab = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(s_keep + scap) + 15) & ~(uintptr_t)15);   // [32 * ncell] per-warp cell counts (seg_tab != 0)
  __shared__ int s_lvl_off[MVO_MAX_LEVELS + 1];
  __shared__ int s_warp[32];
  __shared__ int s_overflow;

  const int nb = plan.total_bands;
  const int32_t *bc = bandcnt + (size_t)f * nb;
  // exclusive scan of band counts (nb <= 1024): one element per thread
  {
    const int v = tid < nb ? bc[tid] : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int off = incl - v;
    for (int k = 0; k < warp; ++k) off += s_warp[k];
    if (tid < nb) s_boff[tid] = off;
    if (tid == nb - 1) s_boff[nb] = off + v;
  }
  __syncthreads();
  const int n = s_boff[nb];
  if (tid == 0) {
    int ovf = 0;
    for (int l = 0; l < plan.nlevels; ++l) {
      const int b0 = plan.lv[l].band_first;
      s_lvl_off[l] = s_boff[b0];
      const int cnt = s_boff[b0 + plan.lv[l].nbands] - s_boff[b0];
      meta[f].lvl_count[l] = cnt;
      if (cnt > plan.lv[l].cap) ovf = 1;          // OpenCV would call retainBest -> host path
    }
    s_lvl_off[plan.nlevels] = n;
    if (n > cap || n > scap) ovf = 1;
    s_overflow = ovf;
    meta[f].overflow = ovf;
    meta[f].n_cand = n;
    if (ovf) meta[f].n_sel = 0;
  }
  __syncthreads();
  const bool ovf = s_overflow != 0;

  // gather the band staging into the compact, level-major raster-ordered candidate array
  const int gshift = orb_grid_shift(plan.grid_size);
  uint32_t *cf = cand + (size_t)f * cap;
  for (int b = warp; b < nb; b += 32) {
    const int o = s_boff[b], c = s_boff[b + 1] - o;
    const uint32_t *src = staging + ((size_t)f * nb + b) * plan.band_cap;
    int l = 0;
    while (l + 1 < plan.nlevels && b >= plan.lv[l + 1].band_first) ++l;
    const float scale = plan.lv[l].scale;
    for (int i = lane; i < c; i += 32) {
      const uint32_t p = src[i];
      if (o + i < cap) {
        cf[o + i] = p;
        if (!ovf) {
          // feature_match.cpp:70: row = ((int)kpt.pt.y) / grid, col = ((int)kpt.pt.x) / grid
          const float fx = l ? __fmul_rn((float)orb_px(p), scale) : (float)orb_px(p);
          const float fy = l ? __fmul_rn((float)orb_py(p), scale) : (float)orb_py(p);
          int row = gshift >= 0 ? ((int)fy) >> gshift : ((int)fy) / plan.grid_size, col = gshift >= 0 ? ((int)fx) >> gshift : ((int)fx) / plan.grid_size;
          s_cell[o + i] = (uint16_t)(row < plan.grid_rows && col < plan.grid_cols ? row * plan.grid_cols + col : ORB_NO_CELL);
        }
      }
    }
  }
  __syncthreads();
  if (ovf) return;

  if (seg_tab) grid_rank_keep_seg(n, s_cell, s_keep, s_tab, ncell, plan.max_per_cell);
  else grid_rank_keep(n, s_cell, s_keep, reinterpret_cast<uint32_t *>(s_cellcnt), ncell, plan.max_per_cell);     // s_cellcnt + s_cursor: 2 * ncell + 1 words
  // ordered prefix count of kept0 (contiguous chunk per thread), cut after max_kpts + 1
  {
    const int per = (n + 1023) >> 10;
    const int b = tid * per, e = min(b + per, n);
    int mine = 0;
    for (int i = b; i < e; ++i) mine += s_keep[i];
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    __syncthreads();
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int pos = incl - mine, total = 0;
    for (int k = 0; k < 32; ++k) {
      if (k < warp) pos += s_warp[k];
      total += s_warp[k];
    }
    uint2 *sf = sel + (size_t)f * (plan.max_kpts + 1);
    for (int i = b; i < e; ++i) {
      if (s_keep[i]) {
        if (pos <= plan.max_kpts) {
          int l = 0;
          while (l + 1 < plan.nlevels && i >= s_lvl_off[l + 1]) ++l;
          sf[pos] = make_uint2(cf[i], (uint32_t)l);
        }
        ++pos;
      }
    }
    if (tid == 0) meta[f].n_sel = min(total, plan.max_kpts + 1);
  }
}


// ------------------------------------------------------------------------------ retainBest
// cv::KeyPointsFilter::retainBest as cv::ORB applies it per pyramid level (orb.cpp computeKeyPoints): first by FAST score to
// 2 x featuresPerLevel, then — with the Harris responses of the survivors — to featuresPerLevel.  retainBest is
//   std::nth_element(begin, begin + n - 1, end, response greater) ; ambiguous = v[n - 1].response ;
//   std::partition(begin + n, end, response >= ambiguous) ; resize
// and both the surviving SET and its ORDER (which the reference's first-come grid selection depends on) are decided by
// libstdc++'s algorithms, restated here step by step:
//   nth_element = __introselect: while the range holds more than 3 elements, __unguarded_partition_pivot (median of
//     first+1 / middle / last-1 moved to the front, then the unguarded Hoare partition) and continue in the part that
//     holds the nth position; __insertion_sort on the last <= 3 elements.  The partition is evaluated by one warp with the
//     technique of k_match_filter (track_filter.cuh): the stop positions of the left scan (Lo) and of the right scan (Ro)
//     are properties of the range before any swap, the k-th swap pairs Lo[k] with Ro[k] while Lo[k] < Ro[k], and the cut
//     is min(Lo[K], Ro[K-1]).  Beyond the depth limit 2 lg(n) libstdc++ switches to heap-select: the kernel then reports
//     the frame for the host path (adversarial inputs only).
//   partition (bidirectional): the k-th swap pairs the k-th element from the left that fails the predicate with the k-th
//     element from the right that passes it, while the former lies left of the latter; new end = begin + #passing.
// One CTA of RET_T threads per (level, frame); the level's records live in shared memory (response 4 B + index 2 B + the two
// stop lists).  Ranges of RET_WARP_LEN elements or more are scanned by the whole CTA (every warp lists the stops of its chunk,
// a prefix over the warps places them), shorter ones by warp 0 alone.
constexpr int RET_MAX = 12288;       // candidates of one level the device path holds; more -> host path
constexpr int RET_T = 256, RET_W = RET_T / 32;
constexpr int RET_WARP_LEN = 256;      // ranges from this length on are scanned by the whole CTA (round 2: 768; one warp needed ~100 cycles per 32 elements)

struct RetBuf { float *key; uint16_t *idx, *Ls, *Rs; int *s_i; };   // s_i: 2 * RET_W + 8 ints of block scratch

__device__ __forceinline__ void ret_swap(const RetBuf &b, int x, int y) {
  const float k = b.key[x]; b.key[x] = b.key[y]; b.key[y] = k;
  const uint16_t i = b.idx[x]; b.idx[x] = b.idx[y]; b.idx[y] = i;
}

// The two stop lists of a scan pair over positions lo .. lo + len - 1 (left list, ascending) and top .. top - len + 1 (right
// list, descending): Ls[lo + k] = k-th position from the left with left(key), Rs[lo + k] = k-th from the right with right(key).
// WHOLE: all RET_W warps take part (block barriers inside); otherwise the calling warp works alone.
template <bool WHOLE, class FL, class FR>
__device__ __forceinline__ void ret_stop_lists(const RetBuf &b, int lo, int len, int top, FL left, FR right, int &nL, int &nR) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned below = (1u << lane) - 1u;
  if (!WHOLE) {
    nL = nR = 0;
    for (int base = 0; base < len; base += 64) {          // two 32-element groups per trip: four independent loads in flight
      const int i0 = base + lane, i1 = i0 + 32;
      const bool in0 = i0 < len, in1 = i1 < len;
      const float kl0 = in0 ? b.key[lo + i0] : 0.f, kr0 = in0 ? b.key[top - i0] : 0.f;
      const float kl1 = in1 ? b.key[lo + i1] : 0.f, kr1 = in1 ? b.key[top - i1] : 0.f;
      const bool ls0 = in0 && left(kl0), rs0 = in0 && right(kr0), ls1 = in1 && left(kl1), rs1 = in1 && right(kr1);
      const unsigned bl0 = __ballot_sync(0xffffffffu, ls0), br0 = __ballot_sync(0xffffffffu, rs0);
      const unsigned bl1 = __ballot_sync(0xffffffffu, ls1), br1 = __ballot_sync(0xffffffffu, rs1);
      const int cl0 = __popc(bl0), cr0 = __popc(br0);
      if (ls0) b.Ls[lo + nL + __popc(bl0 & below)] = (uint16_t)(lo + i0);
      if (rs0) b.Rs[lo + nR + __popc(br0 & below)] = (uint16_t)(top - i0);
      if (ls1) b.Ls[lo + nL + cl0 + __popc(bl1 & below)] = (uint16_t)(lo + i1);
      if (rs1) b.Rs[lo + nR + cr0 + __popc(br1 & below)] = (uint16_t)(top - i1);
      nL += cl0 + __popc(bl1);
      nR += cr0 + __popc(br1);
    }
    __syncwarp();
    return;
  }
  const int chunk = ((len + RET_T - 1) / RET_T) * 32;               // per warp, a multiple of 32
  const int c0 = min(warp * chunk, len), c1 = min(c0 + chunk, len);
  int cl = 0, cr = 0;
  for (int base = c0; base < c1; base += 32) {
    const int i = base + lane;
    const bool inr = i < c1;
    cl += __popc(__ballot_sync(0xffffffffu, inr && left(b.key[lo + i])));
    cr += __popc(__ballot_sync(0xffffffffu, inr && right(b.key[top - i])));
  }
  if (lane == 0) { b.s_i[warp] = cl; b.s_i[RET_W + warp] = cr; }
  __syncthreads();
  int oL = 0, oR = 0;
  nL = nR = 0;
  for (int w = 0; w < RET_W; ++w) { if (w < warp) { oL += b.s_i[w]; oR += b.s_i[RET_W + w]; } nL += b.s_i[w]; nR += b.s_i[RET_W + w]; }
  for (int base = c0; base < c1; base += 32) {
    const int i = base + lane;
    const bool inr = i < c1;
    const bool ls = inr && left(b.key[lo + i]), rs = inr && right(b.key[top - i]);
    const unsigned bl = __ballot_sync(0xffffffffu, ls), br = __ballot_sync(0xffffffffu, rs);
    if (ls) b.Ls[lo + oL + __popc(bl & below)] = (uint16_t)(lo + i);
    if (rs) b.Rs[lo + oR + __popc(br & below)] = (uint16_t)(top - i);
    oL += __popc(bl);
    oR += __popc(br);
  }
  __syncthreads();
}

// the swaps of a Hoare-style scan pair: pairs (Ls[k], Rs[k]) while Ls[k] < Rs[k]; returns their number K
template <bool WHOLE>
__device__ __forceinline__ int ret_swap_pairs(const RetBuf &b, int lo, int nmin) {
  const int lane = threadIdx.x & 31;
  int K = 0;
  if (!WHOLE) {
    for (int base = 0; base < nmin; base += 32) {
      const int j = base + lane;
      const bool sw = j < nmin && b.Ls[lo + j] < b.Rs[lo + j];
      const unsigned m = __ballot_sync(0xffffffffu, sw);
      if (sw) ret_swap(b, b.Ls[lo + j], b.Rs[lo + j]);
      const int c = __popc(m);
      K += c;
      if (c < 32) break;
    }
    __syncwarp();
    return K;
  }
  if (threadIdx.x == 0) b.s_i[2 * RET_W] = 0;
  __syncthreads();
  int mine = 0;
  for (int j = threadIdx.x; j < nmin; j += RET_T)                   // Ls ascends, Rs descends: the condition holds on a prefix
    if (b.Ls[lo + j] < b.Rs[lo + j]) { ret_swap(b, b.Ls[lo + j], b.Rs[lo + j]); ++mine; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if (lane == 0 && mine) atomicAdd(&b.s_i[2 * RET_W], mine);
  __syncthreads();
  K = b.s_i[2 * RET_W];
  __syncthreads();
  return K;
}

// std::__unguarded_partition_pivot(first, last, greater); returns the cut.  Uniform over the calling group.
template <bool WHOLE>
__device__ int ret_partition_pivot(const RetBuf &b, int first, int last) {
  if (threadIdx.x == 0) {                // __move_median_to_first(first, first + 1, mid, last - 1), comp(a, b) = a > b
    const int ia = first + 1, ib = first + (last - first) / 2, ic = last - 1;
    const float ka = b.key[ia], kb = b.key[ib], kc = b.key[ic];
    int pick;
    if (ka > kb) pick = (kb > kc) ? ib : ((ka > kc) ? ic : ia);
    else pick = (ka > kc) ? ia : ((kb > kc) ? ic : ib);
    ret_swap(b, first, pick);
  }
  if (WHOLE) __syncthreads(); else __syncwarp();
  const float pivot = b.key[first];
  const int lo = first + 1, len = last - lo;
  int nL, nR;
  // the left scan `while (*first > pivot) ++first` stops at !(key > pivot); the right scan `while (pivot > *last) --last` at !(pivot > key)
  ret_stop_lists<WHOLE>(b, lo, len, last - 1, [pivot](float k) { return !(k > pivot); }, [pivot](float k) { return !(pivot > k); }, nL, nR);
  const int K = ret_swap_pairs<WHOLE>(b, lo, min(nL, nR));
  int cut;
  if (K == 0) cut = nL > 0 ? (int)b.Ls[lo] : last;
  else { cut = (int)b.Rs[lo + K - 1]; if (K < nL) cut = min(cut, (int)b.Ls[lo + K]); }
  return cut;
}

// cv::KeyPointsFilter::retainBest on b.key / b.idx [0, n): returns the new size, or -1 where libstdc++ would heap-select.
// Called by the whole CTA; n, npts uniform.
__device__ int ret_retain_best(const RetBuf &b, int n, int npts) {
  if (npts < 0 || n <= npts) return n;
  if (npts == 0) return 0;
  const int warp = threadIdx.x >> 5;
  // std::nth_element(begin, begin + npts - 1, end)
  {
    int first = 0, last = n;
    const int nth = npts - 1;
    int depth = 0;
    for (int m = n; m > 1; m >>= 1) ++depth;
    depth *= 2;
    while (last - first > 3) {
      if (depth == 0) return -1;
      --depth;
      int cut;
      if (last - first >= RET_WARP_LEN) cut = ret_partition_pivot<true>(b, first, last);
      else {
        if (warp == 0) { cut = ret_partition_pivot<false>(b, first, last); if (threadIdx.x == 0) b.s_i[2 * RET_W + 1] = cut; }
        __syncthreads();
        cut = b.s_i[2 * RET_W + 1];
        __syncthreads();
      }
      if (cut <= nth) first = cut; else last = cut;
    }
    if (threadIdx.x == 0) {              // __insertion_sort(first, last, greater)
      for (int i = first + 1; i < last; ++i) {
        const float v = b.key[i];
        const uint16_t vi = b.idx[i];
        int j = i - 1;
        if (v > b.key[first]) {          // move_backward(first, i, i + 1); *first = val
          for (; j >= first; --j) { b.key[j + 1] = b.key[j]; b.idx[j + 1] = b.idx[j]; }
          b.key[first] = v; b.idx[first] = vi;
        } else {                         // __unguarded_linear_insert
          for (; v > b.key[j]; --j) { b.key[j + 1] = b.key[j]; b.idx[j + 1] = b.idx[j]; }
          b.key[j + 1] = v; b.idx[j + 1] = vi;
        }
      }
    }
    __syncthreads();
  }
  // std::partition(begin + npts, end, response >= ambiguous): the k-th element from the left that fails is swapped with the
  // k-th from the right that passes while it lies left of it; new end = begin + npts + #passing
  const float amb = b.key[npts - 1];
  int nF, nT;
  ret_stop_lists<true>(b, npts, n - npts, n - 1, [amb](float k) { return !(k >= amb); }, [amb](float k) { return k >= amb; }, nF, nT);
  (void)ret_swap_pairs<true>(b, npts, min(nF, nT));
  return npts + nT;
}

__global__ void __launch_bounds__(RET_T)
k_retain(OrbPlanDev plan, const uint32_t *__restrict__ cand, const float *__restrict__ harris, OrbFrameMeta *__restrict__ meta,
         uint16_t *__restrict__ kept, int32_t *__restrict__ kept_cnt) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ int s_scratch[2 * RET_W + 8];
  const int l = blockIdx.x, f = blockIdx.y, tid = threadIdx.x;
  if (meta[f].overflow == 0) return;
  RetBuf b;
  b.key = reinterpret_cast<float *>(smem);
  b.idx = reinterpret_cast<uint16_t *>(b.key + RET_MAX);
  b.Ls = b.idx + RET_MAX;
  b.Rs = b.Ls + RET_MAX;
  b.s_i = s_scratch;
  const int n = meta[f].lvl_count[l];
  int base = 0;
  for (int q = 0; q < l; ++q) base += meta[f].lvl_count[q];
  uint16_t *out = kept + ((size_t)f * plan.nlevels + l) * RET_MAX;
  const int cap = plan.lv[l].cap;
  if (n > RET_MAX || base + n > plan.cand_cap) {           // beyond the device path: the host finishes this frame
    if (tid == 0) { atomicExch(&meta[f].overflow, 2); kept_cnt[f * plan.nlevels + l] = 0; }
    return;
  }
  if (n <= cap) {                                           // both retainBest calls are no-ops
    for (int i = tid; i < n; i += RET_T) out[i] = (uint16_t)i;
    if (tid == 0) kept_cnt[f * plan.nlevels + l] = n;
    return;
  }
  const uint32_t *cf = cand + (size_t)f * plan.cand_cap + base;
  const float *hf = harris + (size_t)f * plan.cand_cap + base;
  for (int i = tid; i < n; i += RET_T) { b.key[i] = (float)orb_ps(cf[i]); b.idx[i] = (uint16_t)i; }
  __syncthreads();
  int m = ret_retain_best(b, n, 2 * cap);                  // by FAST score
  if (m >= 0) {
    __syncthreads();
    for (int i = tid; i < m; i += RET_T) b.key[i] = hf[b.idx[i]];   // HarrisResponses of the survivors, in their order
    __syncthreads();
    m = ret_retain_best(b, m, cap);                         // by Harris response
  }
  if (m < 0) {
    if (tid == 0) { atomicExch(&meta[f].overflow, 2); kept_cnt[f * plan.nlevels + l] = 0; }
    return;
  }
  __syncthreads();
  for (int i = tid; i < m; i += RET_T) out[i] = b.idx[i];
  if (tid == 0) kept_cnt[f * plan.nlevels + l] = m;
}

// selectUniformKptsByGrid (feature_match.cpp:51-84) over the retained lists of a frame whose levels overflowed: the closed
// form of k_select (rank inside the 16 x 16 cell < max_per_cell, cut after max_kpts + 1 kept) in the retained ORDER.
__global__ void __launch_bounds__(1024)
k_select_kept(OrbPlanDev plan, const uint32_t *__restrict__ cand, const uint16_t *__restrict__ kept, const int32_t *__restrict__ kept_cnt,
              uint2 *__restrict__ sel, OrbFrameMeta *__restrict__ meta, int seg_tab) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(128) uint8_t smem[];
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (meta[f].overflow != 1) return;
  const int ncell = plan.grid_rows * plan.grid_cols, scap = plan.sel_cap;
  int32_t *s_cellcnt = reinterpret_cast<int32_t *>(smem);          // [ncell + 1]
  int32_t *s_cursor = s_cellcnt + ncell + 1;                        // [ncell]
  uint32_t *s_pk = reinterpret_cast<uint32_t *>(s_cursor + ncell);  // [scap] packed candidate of list item i
  uint16_t *s_cell = reinterpret_cast<uint16_t *>(s_pk + scap);     // [scap]
  uint16_t *s_bucket = s_cell + scap;                               // [scap]
  uint8_t *s_keep = reinterpret_cast<uint8_t *>(s_bucket + scap);   // [scap]
  uint8_t *s_lvl = s_keep + scap;                                   // [scap]
  uint8_t *s_tab = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(s_lvl + scap) + 15) & ~(uintptr_t)15);     // [32 * ncell] per-warp cell counts (seg_tab != 0)
  __shared__ int s_warp[32];
  __shared__ int s_off[MVO_MAX_LEVELS + 1], s_base[MVO_MAX_LEVELS + 1];
  if (tid == 0) {
    int o = 0, bb = 0;
    for (int l = 0; l < plan.nlevels; ++l) { s_off[l] = o; s_base[l] = bb; o += kept_cnt[f * plan.nlevels + l]; bb += meta[f].lvl_count[l]; }
    s_off[plan.nlevels] = o;
  }
  __syncthreads();
  const int n = s_off[plan.nlevels];
  if (n > scap) {                                                   // ties at the Harris cut beyond nfeatures: host path
    if (tid == 0) meta[f].overflow = 2;
    return;
  }
  const uint32_t *cf = cand + (size_t)f * plan.cand_cap;
  const int gshift = orb_grid_shift(plan.grid_size);
  // two dependent gathers per item (retained index -> packed candidate): eight items per thread with all loads of one kind in flight
  // together (one item at a time cost two L2 round trips each, a third of the kernel)
  for (int i0 = tid; i0 < n; i0 += 8 * 1024) {
    int lv[8];
    uint32_t kk[8], pp[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + u * 1024;
      lv[u] = 0; kk[u] = 0;
      if (i < n) {
        int l = 0;
        while (l + 1 < plan.nlevels && i >= s_off[l + 1]) ++l;
        lv[u] = l;
        kk[u] = kept[((size_t)f * plan.nlevels + l) * RET_MAX + (i - s_off[l])];
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) pp[u] = (i0 + u * 1024 < n) ? cf[s_base[lv[u]] + kk[u]] : 0u;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + u * 1024;
      if (i >= n) continue;
      const int l = lv[u];
      const uint32_t p = pp[u];
      const float scale = plan.lv[l].scale;
      const float fx = l ? __fmul_rn((float)orb_px(p), scale) : (float)orb_px(p);
      const float fy = l ? __fmul_rn((float)orb_py(p), scale) : (float)orb_py(p);
      int row = gshift >= 0 ? ((int)fy) >> gshift : ((int)fy) / plan.grid_size, col = gshift >= 0 ? ((int)fx) >> gshift : ((int)fx) / plan.grid_size;
      s_pk[i] = p; s_lvl[i] = (uint8_t)l;
      s_cell[i] = (uint16_t)(row < plan.grid_rows && col < plan.grid_cols ? row * plan.grid_cols + col : ORB_NO_CELL);
    }
  }
  __syncthreads();
  if (seg_tab) grid_rank_keep_seg(n, s_cell, s_keep, s_tab, ncell, plan.max_per_cell);
  else grid_rank_keep(n, s_cell, s_keep, reinterpret_cast<uint32_t *>(s_cellcnt), ncell, plan.max_per_cell);
  {
    const int per = (n + 1023) >> 10;
    const int b = tid * per, e = min(b + per, n);
    int mine = 0;
    for (int i = b; i < e; ++i) mine += s_keep[i];
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
    __syncthreads();
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int pos = incl - mine, total = 0;
    for (int k = 0; k < 32; ++k) { if (k < warp) pos += s_warp[k]; total += s_warp[k]; }
    uint2 *sf = sel + (size_t)f * (plan.max_kpts + 1);
    for (int i = b; i < e; ++i)
      if (s_keep[i]) {
        if (pos <= plan.max_kpts) sf[pos] = make_uint2(s_pk[i], (uint32_t)s_lvl[i]);
        ++pos;
      }
    if (tid == 0) { meta[f].n_sel = min(total, plan.max_kpts + 1); meta[f].overflow = 3; }      // 3 = resolved on the device
  }
}

// ------------------------------------------------------------------------------------ blur
// cv::GaussianBlur(7x7, 2, 2, BORDER_REFLECT_101) as ORB applies it to a pyramid level: float
// separable filter, row pass taps in ascending order, symmetric column pass, saturate_cast<uchar>
// (round half to even).  kernel = getGaussianKernel(7, 2, CV_32F).
__constant__ float c_gauss7[7];

constexpr int BLUR_TW = 128, BLUR_TH = 16;

// all pyramid levels of a frame in ONE launch: blockIdx.x walks the tiles of level 0, then level 1, ...
struct BlurTiles { int first[MVO_MAX_LEVELS + 1]; int nx[MVO_MAX_LEVELS]; };

#include "orb_variants.cuh"   // k_blur2, the descriptor blur; host-emulated in tests

// -------------------------------------------------------------------------------- describe
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// cv::fastAtan2 scalar path (degrees); every product/sum rounded separately, like the C++ build.
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
  // OpenCV: static const float atan2_p1 = 0.9997878412794807f*(float)(180/CV_PI); ... (float x float)
  constexpr float r2d = (float)(180.0 / 3.1415926535897932384626433832795);
  constexpr float p1 = 0.9997878412794807f * r2d, p3 = -0.3258083974640975f * r2d;
  constexpr float p5 = 0.1555786518463281f * r2d, p7 = -0.04432655554792128f * r2d;
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  const float eps = 2.2204460492503131e-16f;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, eps));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, eps));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0.f) a = __fsub_rn(180.f, a);
  if (y < 0.f) a = __fsub_rn(360.f, a);
  return a;
}

__device__ __forceinline__ float harris_warp(const uint8_t *__restrict__ img, int pitch, int x0, int y0, int lane) {
  // OpenCV HarrisResponses: 7x7 block, Sobel-like 3x3 gradients, integer sums.
  int a = 0, b = 0, c = 0;
#pragma unroll
  for (int rep = 0; rep < 2; ++rep) {
    const int k = lane + 32 * rep;
    if (k < 49) {
      const int i = k / 7, j = k - 7 * i;
      const uint8_t *p = img + (size_t)(y0 - 3 + i) * pitch + (x0 - 3 + j);
      const int Ix = (p[1] - p[-1]) * 2 + (p[-pitch + 1] - p[-pitch - 1]) + (p[pitch + 1] - p[pitch - 1]);
      const int Iy = (p[pitch] - p[-pitch]) * 2 + (p[pitch - 1] - p[-pitch - 1]) + (p[pitch + 1] - p[-pitch + 1]);
      a += Ix * Ix;
      b += Iy * Iy;
      c += Ix * Iy;
    }
  }
  a = warp_sum(a);
  b = warp_sum(b);
  c = warp_sum(c);
  const float scale = __fdiv_rn(1.f, __fmul_rn(28.f, 255.f));            // 1.f/((1<<2)*7*255.f)
  const float s4 = __fmul_rn(__fmul_rn(__fmul_rn(scale, scale), scale), scale);
  const float fa = (float)a, fb = (float)b, fc = (float)c;
  const float ab = __fadd_rn(fa, fb);
  return __fmul_rn(__fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, ab), ab)), s4);
}

__device__ __forceinline__ float ic_angle_warp(const uint8_t *__restrict__ img, int pitch, int x0, int y0, int lane) {
  // intensity centroid over the radius-15 disc (umax table of OpenCV's ORB)
  const int u = lane - ORB_HALF_PATCH;      // lanes 0..30 -> u = -15..15
  const unsigned long long umax_lo = 0x0D0E0E0E0F0F0F0FULL;   // umax[0..7]  = 15,15,15,15,14,14,14,13
  const unsigned long long umax_hi = 0x030608090A0B0C0DULL;   // umax[8..15] = 13,12,11,10,9,8,6,3
  int m10 = 0, m01 = 0;
  for (int v = -ORB_HALF_PATCH; v <= ORB_HALF_PATCH; ++v) {
    const int av = v < 0 ? -v : v;
    const int um = (int)(((av < 8 ? umax_lo >> (8 * av) : umax_hi >> (8 * (av - 8)))) & 0xFF);
    if (lane < 31 && u >= -um && u <= um) {
      const int val = img[(size_t)(y0 + v) * pitch + x0 + u];
      m10 += u * val;
      m01 += v * val;
    }
  }
  m10 = warp_sum(m10);
  m01 = warp_sum(m01);
  return fast_atan2_deg((float)m01, (float)m10);
}

__device__ __forceinline__ uint32_t brief_byte(const uint8_t *__restrict__ blur, int pitch, int cx, int cy,
                                               float angle_deg, int lane, const char2 *__restrict__ s_pat) {
  // orb.cpp computeOrbDescriptors: angle *= (float)(CV_PI/180.f); a = (float)cos(angle), b = (float)sin(angle)
  const float th = __fmul_rn(angle_deg, 0.017453292519943295f);
  const float a = (float)cos((double)th), b = (float)sin((double)th);
  const uint8_t *center = blur + (size_t)cy * pitch + cx;
  uint32_t byte = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const char2 p0 = s_pat[(lane * 8 + j) * 2], p1 = s_pat[(lane * 8 + j) * 2 + 1];
    const float x0 = __fsub_rn(__fmul_rn((float)p0.x, a), __fmul_rn((float)p0.y, b));
    const float y0 = __fadd_rn(__fmul_rn((float)p0.x, b), __fmul_rn((float)p0.y, a));
    const float x1 = __fsub_rn(__fmul_rn((float)p1.x, a), __fmul_rn((float)p1.y, b));
    const float y1 = __fadd_rn(__fmul_rn((float)p1.x, b), __fmul_rn((float)p1.y, a));
    const int t0 = center[__float2int_rn(y0) * pitch + __float2int_rn(x0)];
    const int t1 = center[__float2int_rn(y1) * pitch + __float2int_rn(x1)];
    byte |= (uint32_t)(t0 < t1) << j;
  }
  return byte;
}

constexpr int DESC_WARPS = 8;

// MODE 0: keypoints from the selection list (level coordinates) -> mvo_keypoint (+ descriptor)
// MODE 1: descriptors for caller-supplied keypoints
template <int MODE>
__global__ void __launch_bounds__(DESC_WARPS * 32)
k_describe(OrbPlanDev plan, const uint8_t *__restrict__ planes, const uint2 *__restrict__ sel,
           const OrbFrameMeta *__restrict__ meta, const int32_t *__restrict__ n_override,
           const mvo_keypoint *__restrict__ kin, int n_in, mvo_keypoint *__restrict__ kout,
           uint8_t *__restrict__ desc, int32_t *__restrict__ counts, int out_cap, int with_desc,
           int32_t *__restrict__ bad_flag) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ char2 s_pat[512];
  const int f = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 512; i += DESC_WARPS * 32) s_pat[i] = make_char2(kOrbPattern[i][0], kOrbPattern[i][1]);
  __syncthreads();
  int n;
  if (MODE == 0) {
    n = n_override ? n_override[f] : meta[f].n_sel;
    n = min(n, out_cap);
    if (blockIdx.x == 0 && threadIdx.x == 0 && counts) counts[f] = n;
  } else {
    n = n_in;
  }
  const uint8_t *slot = planes + (size_t)f * plan.slot_bytes;
  for (int k = blockIdx.x * DESC_WARPS + warp; k < n; k += gridDim.x * DESC_WARPS) {
    int l, x, y;
    float angle;
    if (MODE == 0) {
      const uint2 s = sel[(size_t)f * (plan.max_kpts + 1) + k];
      l = (int)s.y;
      x = orb_px(s.x);
      y = orb_py(s.x);
      const OrbLevelDev &L = plan.lv[l];
      const uint8_t *img = slot + L.img_off;
      const float resp = harris_warp(img, L.pitch, x, y, lane);
      angle = ic_angle_warp(img, L.pitch, x, y, lane);
      if (lane == 0) {
        mvo_keypoint kp;
        kp.x = l ? __fmul_rn((float)x, L.scale) : (float)x;
        kp.y = l ? __fmul_rn((float)y, L.scale) : (float)y;
        kp.size = __fmul_rn(31.f, L.scale);
        kp.angle = angle;
        kp.response = resp;
        kp.octave = l;
        kp.class_id = -1;
        kout[(size_t)f * out_cap + k] = kp;
      }
    } else {
      const mvo_keypoint kp = kin[k];
      l = kp.octave;
      if (l < 0 || l >= plan.nlevels) {
        if (lane == 0) atomicExch(bad_flag, 1);
        continue;
      }
      const OrbLevelDev &L = plan.lv[l];
      const float s = __fdiv_rn(1.f, L.scale);
      x = __float2int_rn(__fmul_rn(kp.x, s));
      y = __float2int_rn(__fmul_rn(kp.y, s));
      angle = kp.angle;
      // rotated samples reach at most round(13*sqrt(2)) = 19 px from the centre
      if (x < 20 || y < 20 || x >= L.w - 20 || y >= L.h - 20) {
        if (lane == 0) atomicExch(bad_flag, 2);
        continue;
      }
    }
    if (MODE == 1 || with_desc) {
      const OrbLevelDev &L = plan.lv[l];
      const uint32_t byte = brief_byte(slot + L.blur_off, L.pitch, x, y, angle, lane, s_pat);
      desc[((size_t)f * (MODE == 0 ? out_cap : n_in) + k) * 32 + lane] = (uint8_t)byte;
    }
  }
}

// Harris response of every compact candidate of the frames whose levels overflow (retainBest needs them all).  One THREAD
// per candidate: the 9 x 9 neighbourhood is read once into registers, the 49 Sobel-like gradients and the three integer sums
// follow from it (a warp per candidate spent ~100 instructions on three shuffle reductions for 49 pixels).  Same integer
// sums and the same float expression as harris_warp, so the responses are bit-identical with k_describe's.
__global__ void __launch_bounds__(128)
k_harris_all(OrbPlanDev plan, const uint8_t *__restrict__ planes, const uint32_t *__restrict__ cand,
             const OrbFrameMeta *__restrict__ meta, float *__restrict__ harris) {
  pdl_wait();
  pdl_launch_dependents();
  const int f = blockIdx.y;
  if (meta[f].overflow == 0) return;              // only retainBest needs the response of every candidate
  const int n = min(meta[f].n_cand, plan.cand_cap);
  const uint8_t *slot = planes + (size_t)f * plan.slot_bytes;
  const float scale = __fdiv_rn(1.f, __fmul_rn(28.f, 255.f));            // 1.f/((1<<2)*7*255.f)
  const float s4 = __fmul_rn(__fmul_rn(__fmul_rn(scale, scale), scale), scale);
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    int l = 0, acc = meta[f].lvl_count[0];
    while (l + 1 < plan.nlevels && k >= acc) acc += meta[f].lvl_count[++l];
    const uint32_t p = cand[(size_t)f * plan.cand_cap + k];
    const int pitch = plan.lv[l].pitch, x0 = orb_px(p), y0 = orb_py(p);
    const uint8_t *c0 = slot + plan.lv[l].img_off + (size_t)(y0 - 4) * pitch + (x0 - 4);
    int a = 0, b = 0, c = 0;
    // three rows at a time slide down the 9 rows: gradients of block row i need image rows i-1, i, i+1
    int r0[9], r1[9], r2[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) { r0[j] = c0[j]; r1[j] = c0[pitch + j]; }
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      const uint8_t *row = c0 + (size_t)(i + 2) * pitch;
#pragma unroll
      for (int j = 0; j < 9; ++j) r2[j] = row[j];
#pragma unroll
      for (int j = 1; j <= 7; ++j) {
        const int Ix = (r1[j + 1] - r1[j - 1]) * 2 + (r0[j + 1] - r0[j - 1]) + (r2[j + 1] - r2[j - 1]);
        const int Iy = (r2[j] - r0[j]) * 2 + (r2[j - 1] - r0[j - 1]) + (r2[j + 1] - r0[j + 1]);
        a += Ix * Ix;
        b += Iy * Iy;
        c += Ix * Iy;
      }
#pragma unroll
      for (int j = 0; j < 9; ++j) { r0[j] = r1[j]; r1[j] = r2[j]; }
    }
    const float fa = (float)a, fb = (float)b, fc = (float)c;
    const float ab = __fadd_rn(fa, fb);
    harris[(size_t)f * plan.cand_cap + k] =
        __fmul_rn(__fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, ab), ab)), s4);
  }
}

// test hook: the keep flags of the first-come grid selection for a given cell list, by either formulation
__global__ void __launch_bounds__(1024)
k_test_grid_rank(const uint16_t *__restrict__ cells, int n, int ncell, int max_per_cell, int seg, uint8_t *__restrict__ keep_out) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int npad = (n + 63) & ~63;
  uint16_t *s_cell = reinterpret_cast<uint16_t *>(smem);
  uint8_t *s_keep = reinterpret_cast<uint8_t *>(s_cell + npad);
  uint32_t *s_min = reinterpret_cast<uint32_t *>(s_keep + npad);
  uint8_t *s_tab = reinterpret_cast<uint8_t *>(s_min + 2 * ncell + 4);
  for (int i = threadIdx.x; i < n; i += 1024) s_cell[i] = cells[i];
  __syncthreads();
  if (seg) grid_rank_keep_seg(n, s_cell, s_keep, s_tab, ncell, max_per_cell);
  else grid_rank_keep(n, s_cell, s_keep, s_min, ncell, max_per_cell);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += 1024) keep_out[i] = s_keep[i];
}

}  // namespace

// test hook (not part of mvo.h): cells[i] < ncell or 0xFFFF (outside the grid: never kept), n <= 16384; seg = 1: grid_rank_keep_seg, 0: grid_rank_keep (rounds)
extern "C" int mvo_test_grid_rank(mvo_ctx *ctx, const uint16_t *cells, int n, int ncell, int max_per_cell, int seg, uint8_t *keep) {
  if (!ctx || !cells || !keep || n < 1 || n > 16384 || ncell < 1 || ncell > 4096 || max_per_cell < 0) return MVO_ERR_INVALID_ARG;
  if (seg && max_per_cell > 254) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "grid_rank_keep_seg: per-cell limit above the byte counters");
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  const int npad = (n + 63) & ~63;
  const size_t smem = (size_t)npad * 3 + (size_t)(2 * ncell + 4) * 4 + (size_t)32 * ncell + 256;
  MVO_TRY(mvo_reserve(ctx, ctx->d_c, (size_t)npad * 3 + 256));
  uint16_t *dc = (uint16_t *)ctx->d_c.p;
  uint8_t *dk = (uint8_t *)ctx->d_c.p + (size_t)npad * 2;
  MVO_CUDA(ctx, cudaMemcpyAsync(dc, cells, (size_t)n * 2, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaFuncSetAttribute(k_test_grid_rank, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_test_grid_rank<<<1, 1024, smem, ctx->stream>>>(dc, n, ncell, max_per_cell, seg, dk);
  MVO_CHECK_LAUNCH(ctx);
  MVO_CUDA(ctx, cudaMemcpyAsync(keep, dk, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MVO_OK;
}

// ------------------------------------------------------------------------------ launchers
static bool g_gauss_uploaded[64] = {false};

static int upload_gauss(mvo_ctx *ctx) {
  if (ctx->device < 64 && g_gauss_uploaded[ctx->device]) return MVO_OK;
  // cv::getGaussianKernel(7, 2, CV_32F): exp(-x^2/(2 sigma^2)) normalised in double, stored as float
  double k[7], s = 0;
  for (int i = 0; i < 7; ++i) { const double x = i - 3; k[i] = exp(-x * x / 8.0); s += k[i]; }
  float kf[7];
  for (int i = 0; i < 7; ++i) kf[i] = (float)(k[i] / s);
  MVO_CUDA(ctx, cudaMemcpyToSymbolAsync(c_gauss7, kf, sizeof kf, 0, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->device < 64) g_gauss_uploaded[ctx->device] = true;
  return MVO_OK;
}

int orb_launch_gray(mvo_ctx *ctx, const OrbPlanDev &plan, const uint8_t *d_in, int channels, size_t stride,
                    size_t frame_stride, uint8_t *planes, int batch) {
  dim3 grid((plan.lv[0].pitch / 4 + 127) / 128, plan.rows, batch);
  KTimer kt(ctx, KC_GRAY);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(128), 0, k_gray, plan, d_in, channels, stride, frame_stride, planes));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int orb_launch_pyramid(mvo_ctx *ctx, const OrbPlanDev &plan, const int32_t *tables, uint8_t *planes, int batch) {
  for (int l = 1; l < plan.nlevels; ++l) {
    dim3 grid((plan.lv[l].pitch / 4 + 127) / 128, plan.lv[l].h, batch);
    KTimer kt(ctx, KC_RESIZE);
    MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(128), 0, k_resize, plan, l, tables, planes));
    MVO_CHECK_LAUNCH(ctx);
  }
  return MVO_OK;
}

int orb_launch_gray_pyramid(mvo_ctx *ctx, const OrbPlanDev &plan, const uint8_t *d_in, int channels, size_t stride, size_t frame_stride,
                            const int32_t *tables, uint8_t *planes, int batch) {
  static const bool off = getenv("MVO_PYR_FUSED") != nullptr && atoi(getenv("MVO_PYR_FUSED")) == 0;      // test hook: forces the fallback below
  size_t smem = 0;
  for (int l = 0; l + 1 < plan.nlevels; ++l) smem += (size_t)plan.pyr_rows[l] * plan.lv[l].pitch;
  smem += 16;
  if (off || plan.pyr_nb < 1 || smem > 200 * 1024) {
    MVO_TRY(orb_launch_gray(ctx, plan, d_in, channels, stride, frame_stride, planes, batch));
    return orb_launch_pyramid(ctx, plan, tables, planes, batch);
  }
  if (smem > 48 * 1024) MVO_CUDA(ctx, cudaFuncSetAttribute(k_pyramid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KTimer kt(ctx, KC_GRAY);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, dim3(plan.pyr_nb, batch), dim3(PYR_T), smem, k_pyramid, plan, d_in, channels, stride, frame_stride, tables, planes));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

static size_t fast_smem_bytes(const OrbPlanDev &plan) {
  size_t m = 0;
  for (int l = 0; l < plan.nlevels; ++l) {
    const size_t sstride = plan.lv[l].pitch + 16, w32 = (plan.lv[l].w + 31) / 32;
    const size_t b = (ORB_BAND_H + 8) * sstride + (ORB_BAND_H + 2) * sstride + ORB_BAND_H * w32 * 4 +
                     (size_t)(ORB_BAND_H + 2) * plan.lv[l].w * 2 + 64;
    if (b > m) m = b;
  }
  return m;
}

// Tensor maps of the gray planes (one per level) for the current workspace; rebuilt when the planes move or the geometry changes.
struct OrbTmaState {
  const uint8_t *planes = nullptr;
  int slots = 0, nlevels = 0, w[MVO_MAX_LEVELS] = {0}, h[MVO_MAX_LEVELS] = {0};
  uint32_t slot_bytes = 0;
  bool ok = false;
  FastMaps maps;
};

static bool orb_tma_maps(mvo_ctx *ctx, const OrbPlanDev &plan, const uint8_t *planes, int slots, const FastMaps **out) {
  static const bool off = getenv("MVO_FAST_TMA") != nullptr && atoi(getenv("MVO_FAST_TMA")) == 0;      // test hook: forces the vector-load fallback
  if (off) return false;
  if (!ctx->orb_tma) ctx->orb_tma = new OrbTmaState();
  OrbTmaState *t = (OrbTmaState *)ctx->orb_tma;
  bool same = t->planes == planes && t->slots == slots && t->nlevels == plan.nlevels && t->slot_bytes == plan.slot_bytes;
  for (int l = 0; same && l < plan.nlevels; ++l) same = t->w[l] == plan.lv[l].w && t->h[l] == plan.lv[l].h;
  if (!same) {
    t->planes = planes; t->slots = slots; t->nlevels = plan.nlevels; t->slot_bytes = plan.slot_bytes; t->ok = false;
    typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                 const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn || qres != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      return false;
    }
    bool ok = true;
    for (int l = 0; l < plan.nlevels && ok; ++l) {
      const OrbLevelDev &L = plan.lv[l];
      t->w[l] = L.w; t->h[l] = L.h;
      if (L.pitch / 4 > 256) { ok = false; break; }                 // a row must fit one box (256 elements): images up to 1024 wide
      const cuuint64_t dims[3] = {(cuuint64_t)(L.pitch / 4), (cuuint64_t)L.h, (cuuint64_t)slots};
      const cuuint64_t strides[2] = {(cuuint64_t)L.pitch, (cuuint64_t)plan.slot_bytes};
      const cuuint32_t box[3] = {(cuuint32_t)(L.pitch / 4), (cuuint32_t)(ORB_BAND_H + 8), 1}, es[3] = {1, 1, 1};
      const CUresult r = ((EncodeFn)fn)(&t->maps.m[l], CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, (void *)(planes + L.img_off), dims, strides, box, es,
                                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      ok = r == CUDA_SUCCESS;
    }
    t->ok = ok;
  }
  *out = &t->maps;
  return t->ok;
}

void orb_tma_free(mvo_ctx *ctx) {
  delete (OrbTmaState *)ctx->orb_tma;
  ctx->orb_tma = nullptr;
}

int orb_launch_fast(mvo_ctx *ctx, const OrbPlanDev &plan, const uint8_t *planes, uint32_t *staging,
                    int32_t *bandcnt, int batch) {
  const size_t smem = fast_smem_bytes(plan);
  if (smem > 220 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "image too wide for the FAST band kernel");
  const FastMaps *maps = nullptr;
  const bool tma = orb_tma_maps(ctx, plan, planes, ctx->orb_batch > batch ? ctx->orb_batch : batch, &maps);
  dim3 grid(plan.total_bands, batch);
  KTimer kt(ctx, KC_FAST);
  if (tma) {
    MVO_CUDA(ctx, cudaFuncSetAttribute(k_fast<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(256), smem, k_fast<true>, plan, planes, staging, bandcnt, *maps));
  } else {
    static const FastMaps none = {};
    MVO_CUDA(ctx, cudaFuncSetAttribute(k_fast<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(256), smem, k_fast<false>, plan, planes, staging, bandcnt, none));
  }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

// 1 when the two-pass grid selection (grid_rank_keep_seg) can run: its 32 count tables fit next to `smem` bytes and the per-cell
// limit stays below the saturation value of a byte counter; MVO_GRID_ROUNDS=1 forces the round version (test hook)
static int orb_seg_tab(size_t smem, int ncell, int max_per_cell) {
  static const bool rounds = getenv("MVO_GRID_ROUNDS") != nullptr && atoi(getenv("MVO_GRID_ROUNDS")) != 0;
  return (!rounds && max_per_cell <= 254 && smem + (size_t)32 * ncell + 32 <= 220 * 1024) ? 1 : 0;
}

int orb_launch_select(mvo_ctx *ctx, const OrbPlanDev &plan, const uint32_t *staging, const int32_t *bandcnt,
                      uint32_t *cand, uint2 *sel, OrbFrameMeta *meta, int batch) {
  const int ncell = plan.grid_rows * plan.grid_cols;
  size_t smem = (size_t)(ORB_MAX_BANDS + 1) * 4 + (size_t)(ncell + 1) * 4 + (size_t)ncell * 4 +
                (size_t)plan.sel_cap * 2 * 2 + plan.sel_cap + 64;
  if (smem > 220 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "selection grid too large");
  const int seg_tab = orb_seg_tab(smem, ncell, plan.max_per_cell);      // the two-pass grid selection when its count tables fit
  if (seg_tab) smem += (size_t)32 * ncell + 32;
  if (smem > 48 * 1024)
    MVO_CUDA(ctx, cudaFuncSetAttribute(k_select, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  KTimer kt(ctx, KC_SELECT);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, dim3(batch), dim3(1024), smem, k_select, plan, staging, bandcnt, cand, sel, meta, seg_tab));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int orb_launch_blur(mvo_ctx *ctx, const OrbPlanDev &plan, uint8_t *planes, int batch) {
  MVO_TRY(upload_gauss(ctx));
  BlurTiles tiles;
  int total = 0;
  for (int l = 0; l < plan.nlevels; ++l) {
    tiles.first[l] = total;
    tiles.nx[l] = (plan.lv[l].w + BLUR_TW - 1) / BLUR_TW;
    total += tiles.nx[l] * ((plan.lv[l].h + BLUR_TH - 1) / BLUR_TH);
  }
  tiles.first[plan.nlevels] = total;
  dim3 grid(total, 1, batch);
  KTimer kt(ctx, KC_BLUR);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(256), 0, k_blur2, plan, tiles, planes));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int orb_launch_harris_all(mvo_ctx *ctx, const OrbPlanDev &plan, const uint8_t *planes, const uint32_t *cand,
                          const OrbFrameMeta *meta, float *harris, int batch) {
  dim3 grid(ctx->sm_count, batch);
  KTimer kt(ctx, KC_HARRIS);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(128), 0, k_harris_all, plan, planes, cand, meta, harris));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int orb_retain_max(void) { return RET_MAX; }

// retainBest + grid selection on the device for the frames whose levels overflowed (meta.overflow == 1 -> 3; 2 = host path needed)
int orb_launch_retain(mvo_ctx *ctx, const OrbPlanDev &plan, const uint32_t *cand, const float *harris, OrbFrameMeta *meta,
                      uint16_t *kept, int32_t *kept_cnt, uint2 *sel, int batch) {
  const size_t smem = (size_t)RET_MAX * 10;
  MVO_CUDA(ctx, cudaFuncSetAttribute(k_retain, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  { KTimer kt(ctx, KC_SELECT);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, dim3(plan.nlevels, batch), dim3(RET_T), smem, k_retain, plan, cand, harris, meta, kept, kept_cnt)); }
  MVO_CHECK_LAUNCH(ctx);
  const int ncell = plan.grid_rows * plan.grid_cols;
  size_t smem2 = (size_t)(2 * ncell + 1) * 4 + (size_t)plan.sel_cap * (4 + 2 + 2 + 1 + 1) + 64;
  if (smem2 > 220 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "selection grid too large");
  const int seg_tab = orb_seg_tab(smem2, ncell, plan.max_per_cell);
  if (seg_tab) smem2 += (size_t)32 * ncell + 32;
  MVO_CUDA(ctx, cudaFuncSetAttribute(k_select_kept, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
  { KTimer kt(ctx, KC_SELECT);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, dim3(batch), dim3(1024), smem2, k_select_kept, plan, cand, kept, kept_cnt, sel, meta, seg_tab)); }
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int orb_launch_describe_sel(mvo_ctx *ctx, const OrbPlanDev &plan, const uint8_t *planes, const uint2 *sel,
                            const OrbFrameMeta *meta, const int32_t *n_override, mvo_keypoint *kpts, uint8_t *desc,
                            int32_t *counts, int out_cap, int with_desc, int batch) {
  const int blocks = (plan.max_kpts + 1 + DESC_WARPS - 1) / DESC_WARPS;
  dim3 grid(blocks < 1 ? 1 : blocks, batch);
  KTimer kt(ctx, KC_DESCRIBE);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(DESC_WARPS * 32), 0, k_describe<0>, plan, planes, sel, meta, n_override, (const mvo_keypoint *)nullptr, 0, kpts,
                            desc, counts, out_cap, with_desc, (int32_t *)nullptr));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}

int orb_launch_describe_kpts(mvo_ctx *ctx, const OrbPlanDev &plan, const uint8_t *planes, const mvo_keypoint *kpts,
                             int n, uint8_t *desc, int32_t *bad_flag) {
  if (n <= 0) return MVO_OK;
  dim3 grid((n + DESC_WARPS - 1) / DESC_WARPS, 1);
  KTimer kt(ctx, KC_DESCRIBE);
  MVO_CUDA(ctx, launch_pdl3(ctx->stream, grid, dim3(DESC_WARPS * 32), 0, k_describe<1>, plan, planes, (const uint2 *)nullptr, (const OrbFrameMeta *)nullptr, (const int32_t *)nullptr, kpts, n,
                            (mvo_keypoint *)nullptr, desc, (int32_t *)nullptr, 0, 1, bad_flag));
  MVO_CHECK_LAUNCH(ctx);
  return MVO_OK;
}
