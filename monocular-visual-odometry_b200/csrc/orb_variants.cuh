// k_blur2: the descriptor blur.  Kept in a header of its own so that the CPU test tier can compile the very same kernel text
// for the host and run it thread by thread (tests/cpp/orb_variants_emu.cpp) against the oracle.
//
// Included by orb.cu INSIDE its anonymous namespace, after these have been defined there: c_gauss7[7] (the Gaussian taps),
// BLUR_TW / BLUR_TH, struct BlurTiles and the declarations of orb.cuh.
#pragma once

// No FMA, the operand order of OpenCV's float filter: the tile is moved as 32-bit words, the row pass produces four outputs
// per thread from three shared-memory words, the column pass two rows of four outputs per thread from eight float4 rows.
constexpr int BLUR2_INW = BLUR_TW / 4 + 2;      // input words per tile row: 4-px halo word left and right
constexpr int BLUR2_ROWF = BLUR_TW + 4;         // floats per row of the row-pass result (16-byte aligned rows, skewed banks)

__global__ void __launch_bounds__(256)
k_blur2(OrbPlanDev plan, BlurTiles tiles, uint8_t *__restrict__ planes) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ uint32_t s_in[BLUR_TH + 6][BLUR2_INW];
  __shared__ __align__(16) float s_row[BLUR_TH + 6][BLUR2_ROWF];
  int level = 0;
  while (level + 1 < plan.nlevels && (int)blockIdx.x >= tiles.first[level + 1]) ++level;
  const int tile = (int)blockIdx.x - tiles.first[level];
  const OrbLevelDev &L = plan.lv[level];
  const int f = blockIdx.z, tx0 = (tile % tiles.nx[level]) * BLUR_TW, ty0 = (tile / tiles.nx[level]) * BLUR_TH;
  const int w = L.w, h = L.h;
  const uint8_t *img = planes + (size_t)f * plan.slot_bytes + L.img_off;
  uint8_t *out = planes + (size_t)f * plan.slot_bytes + L.blur_off;
  const int tid = threadIdx.x;
  // ---- tile rows ty0-3 .. ty0+TH+2, columns tx0-4 .. tx0+TW+3, BORDER_REFLECT_101 on both axes ----
  for (int i = tid; i < (BLUR_TH + 6) * BLUR2_INW; i += 256) {
    const int r = i / BLUR2_INW, wc = i - r * BLUR2_INW;
    int y = ty0 + r - 3;
    y = y < 0 ? -y : (y >= h ? 2 * h - 2 - y : y);
    y = max(0, min(y, h - 1));
    const uint8_t *row = img + (size_t)y * L.pitch;
    const int x = tx0 + 4 * wc - 4;
    uint32_t v;
    if (x >= 0 && x + 3 < w) {
      v = *reinterpret_cast<const uint32_t *>(row + x);          // planes and pitches are 128-byte aligned, x is a multiple of 4
    } else {
      v = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int xx = x + j;
        xx = xx < 0 ? -xx : (xx >= w ? 2 * w - 2 - xx : xx);
        xx = max(0, min(xx, w - 1));
        v |= (uint32_t)row[xx] << (8 * j);
      }
    }
    s_in[r][wc] = v;
  }
  __syncthreads();
  // ---- row pass: outputs x = tx0 + 4q + j (j = 0..3) need inputs x-3 .. x+3 = bytes 4q+1+j .. 4q+7+j of the tile row ----
  for (int i = tid; i < (BLUR_TH + 6) * (BLUR_TW / 4); i += 256) {
    const int r = i / (BLUR_TW / 4), q = i - r * (BLUR_TW / 4);
    const uint32_t w0 = s_in[r][q], w1 = s_in[r][q + 1], w2 = s_in[r][q + 2];
    float v[10];
    v[0] = (float)((w0 >> 8) & 0xFF); v[1] = (float)((w0 >> 16) & 0xFF); v[2] = (float)(w0 >> 24);
    v[3] = (float)(w1 & 0xFF); v[4] = (float)((w1 >> 8) & 0xFF); v[5] = (float)((w1 >> 16) & 0xFF); v[6] = (float)(w1 >> 24);
    v[7] = (float)(w2 & 0xFF); v[8] = (float)((w2 >> 8) & 0xFF); v[9] = (float)((w2 >> 16) & 0xFF);
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float s = __fmul_rn(c_gauss7[0], v[j]);
#pragma unroll
      for (int k = 1; k < 7; ++k) s = __fadd_rn(s, __fmul_rn(c_gauss7[k], v[j + k]));
      o[j] = s;
    }
    *reinterpret_cast<float4 *>(&s_row[r][4 * q]) = make_float4(o[0], o[1], o[2], o[3]);
  }
  __syncthreads();
  // ---- column pass: thread = 4 columns x 2 output rows (r0, r0 + 1) from row-pass rows r0 .. r0 + 7 ----
  {
    const int q = tid & 31, r0 = (tid >> 5) * 2;
    float4 win[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) win[k] = *reinterpret_cast<const float4 *>(&s_row[r0 + k][4 * q]);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int y = ty0 + r0 + rr;
      if (y >= h || tx0 + 4 * q >= L.pitch) continue;
      uint32_t pk = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float c3 = j == 0 ? win[rr + 3].x : j == 1 ? win[rr + 3].y : j == 2 ? win[rr + 3].z : win[rr + 3].w;
        float s = __fmul_rn(c_gauss7[3], c3);
#pragma unroll
        for (int k = 1; k <= 3; ++k) {
          const float4 &hi = win[rr + 3 + k], &lo = win[rr + 3 - k];
          const float a = j == 0 ? hi.x : j == 1 ? hi.y : j == 2 ? hi.z : hi.w;
          const float b = j == 0 ? lo.x : j == 1 ? lo.y : j == 2 ? lo.z : lo.w;
          s = __fadd_rn(s, __fmul_rn(c_gauss7[3 + k], __fadd_rn(a, b)));
        }
        int vq = __float2int_rn(s);
        vq = max(0, min(255, vq));
        pk |= (uint32_t)vq << (8 * j);
      }
      *reinterpret_cast<uint32_t *>(out + (size_t)y * L.pitch + tx0 + 4 * q) = pk;
    }
  }
}
