// Local bundle adjustment for sm_90a — replaces optimization::bundleAdjustment
// (reference src/optimization/g2o_ba.cpp:172-317) and optimizeSingleFrame (:34-145), i.e. g2o's
// OptimizationAlgorithmLevenberg + BlockSolver<6,3> (Schur on the points) + LinearSolverDense
// + RobustKernelHuber over VertexSE3Expmap / VertexSBAPointXYZ / EdgeProjectXYZ2UV
// (semantics: SURVEY.md Appendix B).
//
// The problem is tiny (F <= 16 poses, ~2000 points, ~10^4 edges) and every LM step is a chain
// of dependent phases, so the whole optimisation is ONE kernel launched as ONE thread-block
// cluster (8 CTAs on 8 SMs of a GPC): phases are separated by cluster barriers (~0.3 us instead
// of a ~3 us grid sync or a kernel boundary), and cross-CTA reductions go through distributed
// shared memory: every CTA leaves its partial sums in its own shared memory and, after the
// barrier, every CTA reads all 8 partials in rank order.  All CTAs therefore hold bit-identical
// copies of Hpp, b, the Schur system, its solution and the LM control state, take the same
// accept/reject decisions without any broadcast, and the result is deterministic.
//
// Work split: points (with their edges, CSR by point, edges of a point sorted by frame) are
// partitioned over the CTAs.  Per LM iteration:
//   A  linearise: thread per point walks its edges; Hll, bl, W(point,frame) to global; Hpp/bp of
//      each frame by a warp-shuffle reduction (the "segmented" reduce: segments = frames)
//   B  reduce partials over the cluster, lambda init (first iteration)
//   C  Schur partials  S_part = sum_l Y_l W_l^T,  Y_l = W_l (Hll+lambda I)^-1   (staged in smem)
//   D  S = Hpp + lambda I - sum S_part; block-parallel LDL^T; pose step
//   E  point steps, trial state, new robust chi2 and the gain denominator
//   F  gain ratio, accept/reject, lambda update  (g2o's rule, <= 10 trials)
// fp64 throughout (g2o is double); no tensor cores: ~15 MFLOP per iteration, latency-bound.
#include <cooperative_groups.h>
#include <algorithm>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "mvo_internal.h"
#include "launch_pdl.cuh"
#if !defined(__CUDACC__)
#include "cuda_emu_mbarrier.h"     // CPU test tier (host compiler, tests/cpp on the include path): the emulated mbarrier
#endif

namespace cg = cooperative_groups;

namespace {

constexpr int BA_T = 256;
constexpr int BA_CLUSTER = 8;          // k_ba (Schur variant)
constexpr int PF_MAXC = 8;             // k_ba_pose: up to 8 CTAs (each receives the partials of all of them)
constexpr int BA_MAXF = 16;
constexpr int BA_NW = BA_T / 32;

struct BaArgs {
  int F, P, E, iters, fix_first, use_huber, pc;
  double f, cx, cy, i00, i01, i10, i11, huber;
  const int32_t *pt_start;
  const int32_t *e_frame;
  const double *obs;
  double *pts_a, *pts_b, *Hll, *bl, *Hinv, *Wd;
  double *poses;     // F x 12 (R row-major, t), world->camera, in/out
  double *stats;     // 4
  int32_t *pts_sel;  // [1]: which of pts_a / pts_b holds the final points
};

struct Lin {
  double e0, e1, chi, w;
  double A[6], B[12];
};

__device__ __forceinline__ void edge_residual(const double *Rt, const double *X, double ou, double ov, const BaArgs &a,
                                              double &x, double &y, double &z, double &e0, double &e1) {
  x = Rt[0] * X[0] + Rt[1] * X[1] + Rt[2] * X[2] + Rt[9];
  y = Rt[3] * X[0] + Rt[4] * X[1] + Rt[5] * X[2] + Rt[10];
  z = Rt[6] * X[0] + Rt[7] * X[1] + Rt[8] * X[2] + Rt[11];
  e0 = ou - (a.f * x / z + a.cx);
  e1 = ov - (a.f * y / z + a.cy);
}

__device__ __forceinline__ double robust_rho(double chi, const BaArgs &a) {
  const double d2 = a.huber * a.huber;
  return (a.use_huber && chi > d2) ? 2 * sqrt(chi) * a.huber - d2 : chi;
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// exp of a g2o SE3 update (omega, upsilon) applied on the left of (R, t): out = exp(d) * in.  Inlined: as a call its d[]
// argument went through the stack.
__device__ __forceinline__ void se3_update(const double *d, const double *in, double *out) {
  const double wx = d[0], wy = d[1], wz = d[2];
  const double th2 = wx * wx + wy * wy + wz * wz;
  double a, b, c;
  // g2o tests theta = sqrt(th2) < 0.00001; the square root is only taken where th2 is within rounding of that boundary (and on the
  // large-angle path), not on the chain of every trial
  const bool tiny = th2 < 0.99999e-10 ? true : (th2 > 1.00001e-10 ? false : sqrt(th2) < 0.00001);
  if (tiny) { a = 1; b = 1; c = 1; }                // g2o's small-angle branch: R = V = I + O + O^2
  else if (th2 < 0.0625) {
    // sin(th)/th, (1-cos th)/th^2, (th-sin th)/th^3 as Taylor polynomials in th^2 (next term < 1e-24 relative for
    // th < 0.25): LM steps are small rotations, and this keeps sincos, a square root and three divisions off the
    // dependent chain of every trial.  Larger angles take the closed form below.
    const double x = th2;
    a = 1.0 + x * (-1.0 / 6 + x * (1.0 / 120 + x * (-1.0 / 5040 + x * (1.0 / 362880 + x * (-1.0 / 39916800 + x * (1.0 / 6227020800.0 + x * (-1.0 / 1307674368000.0 + x * (1.0 / 355687428096000.0))))))));
    b = 0.5 + x * (-1.0 / 24 + x * (1.0 / 720 + x * (-1.0 / 40320 + x * (1.0 / 3628800 + x * (-1.0 / 479001600 + x * (1.0 / 87178291200.0 + x * (-1.0 / 20922789888000.0 + x * (1.0 / 6402373705728000.0))))))));
    c = 1.0 / 6 + x * (-1.0 / 120 + x * (1.0 / 5040 + x * (-1.0 / 362880 + x * (1.0 / 39916800 + x * (-1.0 / 6227020800.0 + x * (1.0 / 1307674368000.0 + x * (-1.0 / 355687428096000.0 + x * (1.0 / 121645100408832000.0))))))));
  }
  else { const double th = sqrt(th2); double sn, cs; sincos(th, &sn, &cs); const double ith = 1.0 / th; a = sn * ith; b = (1 - cs) * ith * ith; c = (th - sn) * ith * ith * ith; }
  const double O[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
  double O2[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) O2[i * 3 + j] = O[i * 3] * O[j] + O[i * 3 + 1] * O[3 + j] + O[i * 3 + 2] * O[6 + j];
  double Rd[9], V[9];
  for (int i = 0; i < 9; ++i) {
    const double I = (i % 4 == 0) ? 1.0 : 0.0;
    Rd[i] = I + a * O[i] + b * O2[i];
    V[i] = tiny ? Rd[i] : I + b * O[i] + c * O2[i];
  }
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) out[i * 3 + j] = Rd[i * 3] * in[j] + Rd[i * 3 + 1] * in[3 + j] + Rd[i * 3 + 2] * in[6 + j];
    out[9 + i] = Rd[i * 3] * in[9] + Rd[i * 3 + 1] * in[10] + Rd[i * 3 + 2] * in[11] +
                 V[i * 3] * d[3] + V[i * 3 + 1] * d[4] + V[i * 3 + 2] * d[5];
  }
}

__device__ __forceinline__ bool inv3_sym(const double *h, double lam, double *o) {   // h: 00 01 02 11 12 22
  const double a = h[0] + lam, b = h[1], c = h[2], d = h[3] + lam, e = h[4], f = h[5] + lam;
  const double c0 = d * f - e * e, c1 = c * e - b * f, c2 = b * e - c * d;
  const double det = a * c0 + b * c1 + c * c2;
  if (!(fabs(det) > 0)) return false;
  const double id = 1.0 / det;
  o[0] = c0 * id; o[1] = c1 * id; o[2] = c2 * id;
  o[3] = (a * f - c * c) * id; o[4] = (b * c - a * e) * id; o[5] = (a * d - b * b) * id;
  return true;
}

__global__ void __launch_bounds__(BA_T, 1) k_ba(BaArgs a) {
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), csize = cluster.num_blocks();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int F = a.F;
  extern __shared__ __align__(16) double sm[];

  // active pose blocks
  __shared__ int s_pidx[BA_MAXF], s_act[BA_MAXF];
  __shared__ int s_nact;
  __shared__ double s_ctl[8];     // 0 lambda, 1 ni, 2 chi_cur, 3 rho, 4 ok, 5 temp chi, 6 swap flag
  if (tid == 0) {
    int na = 0;
    for (int f = 0; f < F; ++f) {
      if (a.fix_first && f == 0) s_pidx[f] = -1;
      else { s_pidx[f] = na; s_act[na] = f; ++na; }
    }
    s_nact = na;
    s_ctl[6] = 0;
  }
  __syncthreads();
  const int n = 6 * s_nact;
  const int NA = F * 27 + 2;                 // per-frame (21 Hpp + 6 bp), chi2, max diag(Hll)
  const int NC = n * n + n;
  // shared carve-up (doubles)
  double *s_pose = sm;                        // F*12
  double *s_try = s_pose + F * 12;            // F*12
  double *s_full = s_try + F * 12;            // NA   reduced Hpp/bp/chi/maxdiag
  double *s_partA = s_full + NA;              // NA   this CTA's partial (read remotely)
  double *s_partE = s_partA + NA;             // 4
  double *s_dp = s_partE + 4;                 // n (+pad)
  double *s_partC = s_dp + ((n + 3) & ~3) + 4;   // NC  (read remotely)
  double *s_u = s_partC + ((NC + 3) & ~3);    // union: warp partials (A) | staging (C) | S + rhs (D)
  double *s_wred = s_u;                       // BA_NW * NA
  double *s_S = s_u;                          // n*n
  double *s_rhs = s_u + n * n;                // n

  for (int i = tid; i < F * 12; i += BA_T) s_pose[i] = a.poses[i];
  // this CTA's points
  const int per = (a.P + (int)csize - 1) / (int)csize;
  const int p0 = min((int)rank * per, a.P), p1 = min(p0 + per, a.P);
  double chi_init = 0;
  int it = 0, rejected = 0;
  bool terminate = false;
  long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0};     // cycles per phase (thread 0), debug only
  long long tmark = clock64();
#define BA_MARK(i) do { const long long t_ = clock64(); ph[i] += t_ - tmark; tmark = t_; } while (0)

  for (; it < a.iters && !terminate; ++it) {
    __syncthreads();
    const double *pts = (s_ctl[6] != 0) ? a.pts_b : a.pts_a;
    double *pts_try = (s_ctl[6] != 0) ? a.pts_a : a.pts_b;
    // ---------------- phase A: linearise ----------------
    for (int i = tid; i < BA_NW * NA; i += BA_T) s_wred[i] = 0;
    __syncthreads();
    double chi_t = 0, md_t = 0;
    for (int base = p0; base < p1; base += BA_T) {
      const int l = base + tid;
      const bool act = l < p1;
      double X[3] = {0, 0, 0};
      int k = 0, kend = 0;
      if (act) { X[0] = pts[3 * l]; X[1] = pts[3 * l + 1]; X[2] = pts[3 * l + 2]; k = a.pt_start[l]; kend = a.pt_start[l + 1]; }
      double hl[6] = {0, 0, 0, 0, 0, 0}, blv[3] = {0, 0, 0};
      for (int f = 0; f < F; ++f) {
        double hp[27];
#pragma unroll
        for (int q = 0; q < 27; ++q) hp[q] = 0;
        double wlf[18];
#pragma unroll
        for (int q = 0; q < 18; ++q) wlf[q] = 0;
        const double *Rt = s_pose + 12 * f;
        const bool pose_act = s_pidx[f] >= 0;
        while (k < kend && a.e_frame[k] == f) {
          double x, y, z, e0, e1;
          edge_residual(Rt, X, a.obs[2 * k], a.obs[2 * k + 1], a, x, y, z, e0, e1);
          const double iz = 1.0 / z, z2 = z * z, fl = a.f;
          // EdgeProjectXYZ2UV::linearizeOplus
          const double t0 = -x * iz * fl, t1 = -y * iz * fl;
          double A[6];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            A[c] = -iz * (fl * Rt[c] + t0 * Rt[6 + c]);
            A[3 + c] = -iz * (fl * Rt[3 + c] + t1 * Rt[6 + c]);
          }
          const double B[12] = {x * y / z2 * fl, -(1 + (x * x / z2)) * fl, y * iz * fl, -iz * fl, 0, x / z2 * fl,
                                (1 + y * y / z2) * fl, -x * y / z2 * fl, -x * iz * fl, 0, -iz * fl, y / z2 * fl};
          const double Oe0 = a.i00 * e0 + a.i01 * e1, Oe1 = a.i10 * e0 + a.i11 * e1;
          const double chi = e0 * Oe0 + e1 * Oe1;
          chi_t += robust_rho(chi, a);
          double w = 1.0;
          if (a.use_huber && chi > a.huber * a.huber) w = a.huber / sqrt(chi);
          const double o00 = w * a.i00, o01 = w * a.i01, o10 = w * a.i10, o11 = w * a.i11;
          const double r0 = -w * Oe0, r1 = -w * Oe1;
          double OA[6];
#pragma unroll
          for (int c = 0; c < 3; ++c) { OA[c] = o00 * A[c] + o01 * A[3 + c]; OA[3 + c] = o10 * A[c] + o11 * A[3 + c]; }
          blv[0] += A[0] * r0 + A[3] * r1; blv[1] += A[1] * r0 + A[4] * r1; blv[2] += A[2] * r0 + A[5] * r1;
          hl[0] += A[0] * OA[0] + A[3] * OA[3]; hl[1] += A[0] * OA[1] + A[3] * OA[4]; hl[2] += A[0] * OA[2] + A[3] * OA[5];
          hl[3] += A[1] * OA[1] + A[4] * OA[4]; hl[4] += A[1] * OA[2] + A[4] * OA[5]; hl[5] += A[2] * OA[2] + A[5] * OA[5];
          if (pose_act) {
            double OB[12];
#pragma unroll
            for (int c = 0; c < 6; ++c) { OB[c] = o00 * B[c] + o01 * B[6 + c]; OB[6 + c] = o10 * B[c] + o11 * B[6 + c]; }
            int q = 0;
#pragma unroll
            for (int r = 0; r < 6; ++r)
#pragma unroll
              for (int c = r; c < 6; ++c) hp[q++] += B[r] * OB[c] + B[6 + r] * OB[6 + c];
#pragma unroll
            for (int r = 0; r < 6; ++r) hp[21 + r] += B[r] * r0 + B[6 + r] * r1;
          }
          // W = B^T Omega A in a block of its own, after the Hpp terms: merged into the block above, or ahead of it, the
          // linearisation spills at the 255-register limit
          if (pose_act) {
#pragma unroll
            for (int r = 0; r < 6; ++r)
#pragma unroll
              for (int c = 0; c < 3; ++c) wlf[r * 3 + c] += B[r] * OA[c] + B[6 + r] * OA[3 + c];
          }
          ++k;
        }
        if (act && pose_act) {
          double *wd = a.Wd + ((size_t)l * F + f) * 18;
#pragma unroll
          for (int q = 0; q < 18; ++q) wd[q] = wlf[q];
        }
        if (pose_act) {
#pragma unroll
          for (int q = 0; q < 27; ++q) {
            const double s = warp_sum_d(hp[q]);
            if (lane == 0) s_wred[warp * NA + f * 27 + q] += s;
          }
        }
      }
      if (act) {
#pragma unroll
        for (int q = 0; q < 6; ++q) a.Hll[(size_t)l * 6 + q] = hl[q];
        a.bl[3 * l] = blv[0]; a.bl[3 * l + 1] = blv[1]; a.bl[3 * l + 2] = blv[2];
        if (kend > a.pt_start[l]) md_t = fmax(md_t, fmax(fabs(hl[0]), fmax(fabs(hl[3]), fabs(hl[5]))));
      }
    }
    {
      const double cs = warp_sum_d(chi_t);
      double m = md_t;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (lane == 0) { s_wred[warp * NA + F * 27] = cs; s_wred[warp * NA + F * 27 + 1] = m; }
    }
    __syncthreads();
    for (int i = tid; i < NA; i += BA_T) {
      double s = 0;
      if (i == NA - 1) { for (int w = 0; w < BA_NW; ++w) s = fmax(s, s_wred[w * NA + i]); }
      else { for (int w = 0; w < BA_NW; ++w) s += s_wred[w * NA + i]; }
      s_partA[i] = s;
    }
    BA_MARK(0);
    cluster.sync();                                                         // ---- barrier 1
    BA_MARK(6);
    // ---------------- phase B: cluster reduction ----------------
    for (int i = tid; i < NA; i += BA_T) {
      double s = 0;
      for (unsigned r = 0; r < csize; ++r) {
        const double v = *cluster.map_shared_rank(s_partA + i, r);
        s = (i == NA - 1) ? fmax(s, v) : s + v;
      }
      s_full[i] = s;
    }
    __syncthreads();
    if (tid == 0) {
      s_ctl[2] = s_full[F * 27];
      if (it == 0) {
        // computeLambdaInit: tau * max |diag| over all non-fixed vertices, tau = 1e-5
        double md = s_full[F * 27 + 1];
        for (int f = 0; f < F; ++f)
          if (s_pidx[f] >= 0) {
            const double *h = s_full + f * 27;
            md = fmax(md, fmax(fmax(fabs(h[0]), fabs(h[6])), fmax(fmax(fabs(h[11]), fabs(h[15])), fmax(fabs(h[18]), fabs(h[20])))));
          }
        s_ctl[0] = 1e-5 * md;
        s_ctl[1] = 2;
      }
    }
    __syncthreads();
    if (it == 0) chi_init = s_ctl[2];
    BA_MARK(1);

    // ---------------- LM trials ----------------
    int qmax = 0;
    double rho = 0;
    do {
      const double lambda = s_ctl[0];
      // ---- phase C: Schur partials ----
      for (int i = tid; i < NC; i += BA_T) s_partC[i] = 0;
      bool inv_ok = true;
      double *s_Y = s_u;                                   // [pc][F][18]
      double *s_W = s_Y + (size_t)a.pc * F * 18;           // [pc][F][18]
      double *s_b = s_W + (size_t)a.pc * F * 18;           // [pc][3]
      for (int c0 = p0; c0 < p1; c0 += a.pc) {
        const int cn = min(a.pc, p1 - c0);
        __syncthreads();
        for (int i = tid; i < cn * F; i += BA_T) {
          const int li = i / F, f = i - li * F, l = c0 + li;
          double *Ys = s_Y + (size_t)i * 18, *Ws = s_W + (size_t)i * 18;
          const bool has = a.pt_start[l + 1] > a.pt_start[l];
          double hi[6] = {0, 0, 0, 0, 0, 0};
          if (has) { if (!inv3_sym(a.Hll + (size_t)l * 6, lambda, hi)) { inv_ok = false; } }
          if (f == 0) {
#pragma unroll
            for (int q = 0; q < 6; ++q) a.Hinv[(size_t)l * 6 + q] = hi[q];
            s_b[li * 3] = a.bl[3 * l]; s_b[li * 3 + 1] = a.bl[3 * l + 1]; s_b[li * 3 + 2] = a.bl[3 * l + 2];
          }
          if (has && s_pidx[f] >= 0) {
            const double *wd = a.Wd + ((size_t)l * F + f) * 18;
#pragma unroll
            for (int r = 0; r < 6; ++r) {
              const double w0 = wd[r * 3], w1 = wd[r * 3 + 1], w2 = wd[r * 3 + 2];
              Ws[r * 3] = w0; Ws[r * 3 + 1] = w1; Ws[r * 3 + 2] = w2;
              Ys[r * 3] = w0 * hi[0] + w1 * hi[1] + w2 * hi[2];
              Ys[r * 3 + 1] = w0 * hi[1] + w1 * hi[3] + w2 * hi[4];
              Ys[r * 3 + 2] = w0 * hi[2] + w1 * hi[4] + w2 * hi[5];
            }
          } else {
#pragma unroll
            for (int q = 0; q < 18; ++q) { Ws[q] = 0; Ys[q] = 0; }
          }
        }
        __syncthreads();
        for (int o = tid; o < NC; o += BA_T) {
          double acc = 0;
          if (o < n * n) {
            const int i = o / n, j = o - i * n;
            const int fa = s_act[i / 6], ra = i % 6, fb = s_act[j / 6], rb = j % 6;
            const double *yp = s_Y + ((size_t)fa * 18 + ra * 3), *wp = s_W + ((size_t)fb * 18 + rb * 3);
            for (int li = 0; li < cn; ++li) {
              const double *y = yp + (size_t)li * F * 18, *w = wp + (size_t)li * F * 18;
              acc += y[0] * w[0] + y[1] * w[1] + y[2] * w[2];
            }
          } else {
            const int i = o - n * n, fa = s_act[i / 6], ra = i % 6;
            const double *yp = s_Y + ((size_t)fa * 18 + ra * 3);
            for (int li = 0; li < cn; ++li) {
              const double *y = yp + (size_t)li * F * 18, *b = s_b + li * 3;
              acc += y[0] * b[0] + y[1] * b[1] + y[2] * b[2];
            }
          }
          s_partC[o] += acc;
        }
      }
      if (tid == 0) s_partE[2] = 1.0;
      __syncthreads();
      if (!inv_ok) s_partE[2] = 0.0;                      // any thread that saw a singular Hll block
      BA_MARK(2);
      cluster.sync();                                                       // ---- barrier 2
      BA_MARK(6);
      // ---- phase D: assemble and solve the pose system (every CTA, identically) ----
      for (int o = tid; o < NC; o += BA_T) {
        double s = 0;
        for (unsigned r = 0; r < csize; ++r) s += *cluster.map_shared_rank(s_partC + o, r);
        if (o < n * n) {
          const int i = o / n, j = o - i * n;
          double h = 0;
          if (i / 6 == j / 6) {
            const int f = s_act[i / 6], r = min(i % 6, j % 6), c = max(i % 6, j % 6);
            h = s_full[f * 27 + (r * (13 - r)) / 2 + (c - r)];        // upper-triangular packing
            if (i == j) h += lambda;
          }
          s_S[o] = h - s;
        } else {
          const int i = o - n * n, f = s_act[i / 6];
          s_rhs[i] = s_full[f * 27 + 21 + i % 6] - s;
        }
      }
      double okf = 1.0;
      for (unsigned r = 0; r < csize; ++r) okf *= *cluster.map_shared_rank(s_partE + 2, r);
      __syncthreads();
      bool ok = okf != 0.0;
      // LDL^T, right-looking, in place (lower triangle holds L, diagonal holds D)
      for (int j = 0; j < n && ok; ++j) {
        const double d = s_S[j * n + j];
        if (!(fabs(d) > 0) || !isfinite(d)) { ok = false; break; }      // uniform: every thread reads the same d
        for (int i = j + 1 + tid; i < n; i += BA_T) s_S[i * n + j] /= d;
        __syncthreads();
        const int m = n - j - 1;
        for (int o = tid; o < m * m; o += BA_T) {
          const int i = j + 1 + o / m, k = j + 1 + o % m;
          if (k <= i) s_S[i * n + k] -= s_S[i * n + j] * s_S[k * n + j] * d;
        }
        __syncthreads();
      }
      if (ok) {
        for (int j = 0; j < n; ++j) {           // forward: L y = b
          const double bj = s_rhs[j];
          __syncthreads();
          for (int i = j + 1 + tid; i < n; i += BA_T) s_rhs[i] -= s_S[i * n + j] * bj;
          __syncthreads();
        }
        for (int i = tid; i < n; i += BA_T) s_rhs[i] /= s_S[i * n + i];
        __syncthreads();
        for (int j = n - 1; j >= 0; --j) {      // backward: L^T x = y
          const double bj = s_rhs[j];
          __syncthreads();
          for (int i = tid; i < j; i += BA_T) s_rhs[i] -= s_S[j * n + i] * bj;
          __syncthreads();
        }
        for (int i = tid; i < n; i += BA_T) s_dp[i] = s_rhs[i];
      } else {
        for (int i = tid; i < n; i += BA_T) s_dp[i] = 0;
      }
      __syncthreads();
      BA_MARK(3);
      // ---- phase E: trial state, new chi2, gain denominator ----
      for (int f = tid; f < F; f += BA_T) {
        if (s_pidx[f] >= 0 && ok) se3_update(s_dp + 6 * s_pidx[f], s_pose + 12 * f, s_try + 12 * f);
        else for (int q = 0; q < 12; ++q) s_try[12 * f + q] = s_pose[12 * f + q];
      }
      __syncthreads();
      double chi_n = 0, scale_t = 0;
      for (int l = p0 + tid; l < p1; l += BA_T) {
        double X[3] = {pts[3 * l], pts[3 * l + 1], pts[3 * l + 2]};
        const int kb = a.pt_start[l], ke = a.pt_start[l + 1];
        if (ok && ke > kb) {
          double c[3] = {a.bl[3 * l], a.bl[3 * l + 1], a.bl[3 * l + 2]};
          const double b0 = c[0], b1 = c[1], b2 = c[2];
          for (int f = 0; f < F; ++f) {
            const int pa = s_pidx[f];
            if (pa < 0) continue;
            const double *wd = a.Wd + ((size_t)l * F + f) * 18, *dp = s_dp + 6 * pa;
#pragma unroll
            for (int q = 0; q < 6; ++q) { c[0] -= wd[q * 3] * dp[q]; c[1] -= wd[q * 3 + 1] * dp[q]; c[2] -= wd[q * 3 + 2] * dp[q]; }
          }
          const double *hi = a.Hinv + (size_t)l * 6;
          const double d0 = hi[0] * c[0] + hi[1] * c[1] + hi[2] * c[2];
          const double d1 = hi[1] * c[0] + hi[3] * c[1] + hi[4] * c[2];
          const double d2 = hi[2] * c[0] + hi[4] * c[1] + hi[5] * c[2];
          X[0] += d0; X[1] += d1; X[2] += d2;
          scale_t += d0 * (lambda * d0 + b0) + d1 * (lambda * d1 + b1) + d2 * (lambda * d2 + b2);
        }
        pts_try[3 * l] = X[0]; pts_try[3 * l + 1] = X[1]; pts_try[3 * l + 2] = X[2];
        for (int k = kb; k < ke; ++k) {
          double x, y, z, e0, e1;
          edge_residual(s_try + 12 * a.e_frame[k], X, a.obs[2 * k], a.obs[2 * k + 1], a, x, y, z, e0, e1);
          chi_n += robust_rho(e0 * (a.i00 * e0 + a.i01 * e1) + e1 * (a.i10 * e0 + a.i11 * e1), a);
        }
      }
      {
        const double c = warp_sum_d(chi_n), s = warp_sum_d(scale_t);
        __syncthreads();                     // s_u (S, rhs) is dead from here on: reuse as scratch
        if (lane == 0) { s_u[warp * 2] = c; s_u[warp * 2 + 1] = s; }
        __syncthreads();
        if (tid == 0) {
          double cc = 0, ss = 0;
          for (int w = 0; w < BA_NW; ++w) { cc += s_u[w * 2]; ss += s_u[w * 2 + 1]; }
          s_partE[0] = cc; s_partE[1] = ss;
        }
      }
      BA_MARK(4);
      cluster.sync();                                                       // ---- barrier 3
      BA_MARK(6);
      // ---- phase F: gain ratio and LM control (g2o OptimizationAlgorithmLevenberg::solve) ----
      if (tid == 0) {
        double temp = 0, scale = 0;
        for (unsigned r = 0; r < csize; ++r) {
          temp += *cluster.map_shared_rank(s_partE + 0, r);
          scale += *cluster.map_shared_rank(s_partE + 1, r);
        }
        // a failed solve adds nothing (as g2o): its step is zero, but a pose row's b can be NaN (a point at zero depth), and
        // 0 * NaN would turn the gain ratio into a rejection
        if (ok)
          for (int i = 0; i < n; ++i) {
            const int f = s_act[i / 6];
            scale += s_dp[i] * (lambda * s_dp[i] + s_full[f * 27 + 21 + i % 6]);
          }
        if (!ok) temp = 1.7976931348623157e308;
        const double cur = s_ctl[2];
        double r_ = (cur - temp) / (scale + 1e-3);
        if (r_ > 0 && isfinite(temp)) {
          double alpha = 1. - pow(2 * r_ - 1, 3);
          alpha = fmin(alpha, 2. / 3.);
          s_ctl[0] = lambda * fmax(1. / 3., alpha);
          s_ctl[1] = 2;
          s_ctl[2] = temp;
          s_ctl[4] = 1;
        } else {
          s_ctl[0] = lambda * s_ctl[1];
          s_ctl[1] *= 2;
          s_ctl[4] = 0;
        }
        s_ctl[3] = r_;
      }
      __syncthreads();
      rho = s_ctl[3];
      if (s_ctl[4] != 0) {              // accepted: trial state becomes current
        for (int i = tid; i < F * 12; i += BA_T) s_pose[i] = s_try[i];
        __syncthreads();
        if (tid == 0) s_ctl[6] = (s_ctl[6] != 0) ? 0.0 : 1.0;
      } else {
        ++rejected;
      }
      __syncthreads();
      ++qmax;
      ph[7]++;
      BA_MARK(5);
      // the trial loop re-reads s_ctl / pts pointers only on acceptance, which ends the loop
    } while (rho < 0 && qmax < 10);
    if (qmax == 10 || rho == 0) terminate = true;
    // Each CTA reads remote s_partE / s_partC only between the barriers above; a trailing barrier
    // keeps a fast CTA from overwriting its partials while a slow one is still in phase F.
    cluster.sync();
  }
  if (rank == 0) {
    for (int i = tid; i < F * 12; i += BA_T) a.poses[i] = s_pose[i];
    if (tid == 0) {
      a.stats[0] = chi_init; a.stats[1] = s_ctl[2]; a.stats[2] = it; a.stats[3] = s_ctl[0];
      a.pts_sel[0] = s_ctl[6] != 0 ? 1 : 0;
      a.stats[7] = rejected;
      for (int q = 0; q < 8; ++q) a.stats[8 + q] = (double)ph[q];
    }
  }
}

size_t ba_smem_doubles(int F, int nact, int pc) {
  const size_t n = 6 * (size_t)nact, NA = (size_t)F * 27 + 2, NC = n * n + n;
  size_t u = (size_t)BA_NW * NA;
  u = std::max(u, n * n + n + 8);
  u = std::max(u, (size_t)pc * F * 36 + (size_t)pc * 3 + 8);
  return (size_t)F * 24 + 2 * NA + 4 + ((n + 3) & ~(size_t)3) + 4 + ((NC + 3) & ~(size_t)3) + u + 16;
}

// =========================================================================================
// Pose-only variant (all map points fixed: the shipped is_ba_fix_map_points "true", and the final
// refit of solvePnPRansac).  With the points fixed g2o's system is block diagonal: F independent
// 6x6 pose blocks that share only the LM damping and the accept/reject decision.  Edge-parallel:
// edges are stored frame-major with their (fixed) 3-D point, every thread of the cluster takes
// edges e = gtid, gtid + 4096, ...; the 27 sums per frame (21 Hessian + 6 gradient) and the robust
// chi2 are reduced by a warp shuffle tree per frame segment, then across warps in shared memory,
// then across the 8 CTAs through distributed shared memory (every CTA pushes its partials into the
// shared memory of all CTAs and sums what it received in rank order, so all CTAs hold identical state
// and decide identically).  The pass that evaluates a trial step also linearises at the trial point, so
// an accepted step needs no second pass: one pass and one exchange per LM trial, and no cluster barrier
// between the first exchange and the exit.  Per trial: solve (lane 0 of warp f for frame f) -> CTA
// barrier -> pass -> CTA barrier -> cross-warp sum and push -> wait for the CTA's mbarrier -> rank-order
// sum + decision (warp-local, no CTA barrier).
#ifndef MVO_PF_T
#define MVO_PF_T 512
#endif
constexpr int PF_T = MVO_PF_T;
constexpr int PF_NW = PF_T / 32;
constexpr int PF_V = 28;                      // 21 H + 6 b + chi2 per frame

struct PoseArgs {
  int F, E, iters, fix_first, use_huber, chunk;    // E = padded edge count (multiple of chunk)
  double fx, fy, cx, cy, i00, i01, i10, i11, huber, step_tol;
  const int32_t *e_frame;   // [E] frame-major
  const double *X;          // [E][3]
  const double *obs;        // [E][2]
  double *poses;            // F x 12 in/out
  double *stats;            // 16
  MvoPoseStore st;          // STORE variant only: the tracker's device-resident frame buffer (F = listed slots)
};

// fast double reciprocal / reciprocal square root: float seed + Newton steps (<= 1 ulp), no fp64
// division or sqrt on the dependent chain
__device__ __forceinline__ double fast_rcp(double z) {
  double r = (double)__frcp_rn((float)z);
  r = r * (2.0 - z * r);
  r = r * (2.0 - z * r);
  return r;
}
__device__ __forceinline__ double fast_rsqrt(double c) {
  double y = (double)rsqrtf((float)c);
  y = y * (1.5 - 0.5 * c * y * y);
  y = y * (1.5 - 0.5 * c * y * y);
  return y;
}
// The float seed is 0 or inf outside the float range (rsqrtf(inf) = 0, __frcp_rn(inf) = 0, the seed of a subnormal depth is
// inf and the Newton steps turn it into -inf or NaN), so a value the LM does not bound takes the exact fp64 operation outside
// [1e-30, 1e30], as chol6_solve does for its pivots.  A point next to a camera's principal plane (depth below ~1e-17 f |x|)
// has chi2 above FLT_MAX; g2o weights it by delta / sqrt(chi2) like any other edge.
__device__ __forceinline__ double ranged_rcp(double z) {
  const double m = fabs(z);
  return (m > 1e-30 && m < 1e30) ? fast_rcp(z) : 1.0 / z;
}
__device__ __forceinline__ double ranged_rsqrt(double c) {
  return (c > 1e-30 && c < 1e30) ? fast_rsqrt(c) : 1.0 / sqrt(c);
}

__device__ __forceinline__ bool chol6_solve(const double *h /*21 packed upper*/, const double *g, double lambda, double *x) {
  // Cholesky with reciprocal diagonal (one rsqrt per column, no divisions on the dependent chain)
  double L[21], inv[6];     // lower triangle, row-major packed: L[i*(i+1)/2 + j]
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      double v = h[(j * (13 - j)) / 2 + (i - j)];
      if (i == j) v += lambda;
      L[i * (i + 1) / 2 + j] = v;
    }
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double d = L[j * (j + 1) / 2 + j];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j * (j + 1) / 2 + k] * L[j * (j + 1) / 2 + k];
    if (!(d > 0) || !isfinite(d)) { ok = false; d = 1; }
    // float seed + two Newton steps (<= 1 ulp) while the pivot is inside the float range: the library rsqrt(double) is a ~20-instruction
    // dependent sequence, six of them sat on the chain of every LM trial
    double id;
    if (d > 1e-30 && d < 1e30) id = fast_rsqrt(d);
    else { id = rsqrt(d); id = id * (1.5 - 0.5 * d * id * id); }
    inv[j] = id;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double s2 = L[i * (i + 1) / 2 + j];
#pragma unroll
      for (int k = 0; k < j; ++k) s2 -= L[i * (i + 1) / 2 + k] * L[j * (j + 1) / 2 + k];
      L[i * (i + 1) / 2 + j] = s2 * id;
    }
  }
  double y[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double s2 = g[i];
#pragma unroll
    for (int k = 0; k < i; ++k) s2 -= L[i * (i + 1) / 2 + k] * y[k];
    y[i] = s2 * inv[i];
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double s2 = y[i];
#pragma unroll
    for (int k = i + 1; k < 6; ++k) s2 -= L[k * (k + 1) / 2 + i] * x[k];
    x[i] = s2 * inv[i];
  }
  return ok;
}

// 28 contributions of one edge at pose Rt (chi2 in v[27]); v is ACCUMULATED
__device__ __forceinline__ void edge_terms(const PoseArgs &a, const double *Rt, double X0, double X1, double X2, double ou,
                                           double ov, double (&v)[32]) {
  const double x = Rt[0] * X0 + Rt[1] * X1 + Rt[2] * X2 + Rt[9];
  const double y = Rt[3] * X0 + Rt[4] * X1 + Rt[5] * X2 + Rt[10];
  const double z = Rt[6] * X0 + Rt[7] * X1 + Rt[8] * X2 + Rt[11];
  const double iz = ranged_rcp(z);
  const double xz = x * iz, yz = y * iz;
  const double e0r = ou - (a.fx * xz + a.cx), e1r = ov - (a.fy * yz + a.cy);
  const double Oe0 = a.i00 * e0r + a.i01 * e1r, Oe1 = a.i10 * e0r + a.i11 * e1r;
  const double chi = e0r * Oe0 + e1r * Oe1;
  double w = 1.0, rho = chi;
  if (a.use_huber && chi > a.huber * a.huber) {     // RobustKernelHuber: rho = 2 sqrt(chi) d - d^2, rho' = d / sqrt(chi)
    const double ys = ranged_rsqrt(chi);
    w = a.huber * ys;
    rho = 2 * (chi * ys) * a.huber - a.huber * a.huber;
  }
  v[27] += rho;
  // EdgeProjectXYZ2UV::linearizeOplus, pose block (rows scaled by fx / fy).  B[4] and B[9] are structural zeros; the
  // products with them stay (DESIGN.md §8, tried and rejected: leaving them out changes the rounding of the sums).
  const double fxz = a.fx * iz, fyz = a.fy * iz;
  const double B[12] = {xz * yz * a.fx, -(1 + xz * xz) * a.fx, yz * a.fx, -fxz, 0, xz * fxz,
                        (1 + yz * yz) * a.fy, -xz * yz * a.fy, -xz * a.fy, 0, -fyz, yz * fyz};
  const double o00 = w * a.i00, o01 = w * a.i01, o10 = w * a.i10, o11 = w * a.i11;
  const double r0 = -w * Oe0, r1 = -w * Oe1;
  double OB[12];
#pragma unroll
  for (int q2 = 0; q2 < 6; ++q2) { OB[q2] = o00 * B[q2] + o01 * B[6 + q2]; OB[6 + q2] = o10 * B[q2] + o11 * B[6 + q2]; }
  int q = 0;
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int cc = r; cc < 6; ++cc) v[q++] += B[r] * OB[cc] + B[6 + r] * OB[6 + cc];
#pragma unroll
  for (int r = 0; r < 6; ++r) v[21 + r] += B[r] * r0 + B[6 + r] * r1;
}

// One halving step of warp_fold32: lanes with bit STEP set keep the upper half, the others the lower half.  STEP is a template
// argument so that the loop has a constant trip count before any unrolling: with a bound taken from an enclosing loop's variable
// the front end left the loop rolled and demoted v[] to local memory (every access of the fold an LDL / STL).
template <int STEP>
__device__ __forceinline__ void warp_fold_step(double (&v)[32], int lane) {
  const bool up = (lane & STEP) != 0;
#pragma unroll
  for (int i = 0; i < STEP; ++i) {
    const double send = up ? v[i] : v[i + STEP];
    const double keep = up ? v[i + STEP] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, STEP);
  }
}

// warp reduce-scatter of 32 values: afterwards lane L holds the warp-wide sum of v[L]
// (31 exchanges instead of 32 x 5 for a butterfly per value)
__device__ __forceinline__ double warp_fold32(double (&v)[32], int lane) {
  warp_fold_step<16>(v, lane);
  warp_fold_step<8>(v, lane);
  warp_fold_step<4>(v, lane);
  warp_fold_step<2>(v, lane);
  warp_fold_step<1>(v, lane);
  return v[0];
}

// The push exchange of the pose LM: every CTA stores its partials straight into the receive area of each CTA of the cluster with
// st.async, which counts the bytes on the receiver's mbarrier; a CTA has every partial of a round once that barrier's phase
// completes.  The CPU test tier runs the same protocol on an emulated barrier (tests/cpp/cuda_emu_mbarrier.h).
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
#if defined(__CUDA_ARCH__)
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
#elif !defined(__CUDACC__)
  emu_mbar_init(bar, count);
#endif
}

// makes initialised barriers visible to the st.async of the other CTAs (published by the next cluster barrier)
__device__ __forceinline__ void mbar_init_fence() {
#if defined(__CUDA_ARCH__)
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
}

// the barrier's one arrival per phase, with the bytes the phase has to receive
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long *bar, unsigned bytes) {
#if defined(__CUDA_ARCH__)
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
#elif !defined(__CUDACC__)
  emu_mbar_arrive_expect_tx(bar, bytes);
#endif
}

__device__ __forceinline__ void mbar_wait_parity(unsigned long long *bar, unsigned parity) {
#if defined(__CUDA_ARCH__)
  const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
  unsigned done;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"(b), "r"(parity) : "memory");
  } while (!done);
#elif !defined(__CUDACC__)
  while (!emu_mbar_try_wait_parity(bar, parity)) {}
#endif
}

// v -> CTA `rank`'s copy of *dst, 8 bytes counted on that CTA's copy of *bar (same shared-memory layout in every CTA)
__device__ __forceinline__ void dsmem_push(double *dst, double v, unsigned long long *bar, unsigned rank) {
#if defined(__CUDA_ARCH__)
  unsigned rd, rb;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rd) : "r"((unsigned)__cvta_generic_to_shared(dst)), "r"(rank));
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(rank));
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.f64 [%0], %1, [%2];" ::"r"(rd), "d"(v), "r"(rb) : "memory");
#elif !defined(__CUDACC__)
  emu_st_async(dst, v, bar, rank);
#endif
}

// One pass over this CTA's chunks at poses `P` -> row `rank` of every CTA's receive area, element f*PF_V + q.  Thread (rank, tid) owns chunk
// rank*PF_T + tid: CH consecutive edges of ONE frame (host pads each frame's run to a multiple of CH with
// frame -1), cached in shared memory (s_ed, SoA) when CACHED, so the LM trials never touch global memory.
// Which chunk thread (rank, tid) of the cluster owns when the chunks are cached in shared memory: consecutive WARPS of chunks go to
// consecutive CTAs (warp w of CTA r takes chunks 32 (w csize + r) ..), so that a problem with fewer chunks than threads — the PnP refit
// has ~500 edges for 4096 threads, the 5-frame BA ~2700 — keeps every SM of the cluster equally busy instead of filling CTA 0 first
// (the fp64 pass of 16 full warps costs ~2.5 K cycles on one SM).  A warp still holds 32 consecutive chunks: one frame, rarely two.
__device__ __forceinline__ int pf_chunk_of(unsigned rank, int tid, unsigned csize) {
  return ((((tid >> 5) * (int)csize) + (int)rank) << 5) + (tid & 31);
}

template <int CH, bool CACHED>
__device__ void pose_pass(const PoseArgs &a, int F, int nchunks, const double *P, const double *s_ed, const int *s_ef,
                          double *s_wacc /*[PF_NW][NV]*/, double *recv /*this round's receive area [csize][NV]*/,
                          unsigned long long *bar /*its barrier*/, unsigned rank, unsigned csize) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NV = F * PF_V;
  // s_wacc is all-zero on entry (cleared at kernel start and re-cleared by the reduction below)
  const int chunk = CACHED ? CH : a.chunk;
  const int stride = (int)csize * PF_T;
  for (int cbase = CACHED ? 0 : (int)rank * PF_T; cbase < (CACHED ? 1 : nchunks); cbase += CACHED ? 1 : stride) {      // one sweep when CACHED
    const int c = cbase + tid;
    double v[32];
#pragma unroll
    for (int q = 0; q < 32; ++q) v[q] = 0;
    int f = -1;
    if (CACHED) {
      f = s_ef[tid];
      if (f >= 0) {
        const double *Rt = P + 12 * f;
#pragma unroll
        for (int k = 0; k < CH; ++k) {
          const double *ed = s_ed + (size_t)k * 5 * PF_T + tid;
          const double ou = ed[3 * PF_T];
          if (ou > -1e290) edge_terms(a, Rt, ed[0], ed[PF_T], ed[2 * PF_T], ou, ed[4 * PF_T], v);   // -1e300 marks padding
        }
      }
    } else if (c < nchunks) {
      const int e0 = c * chunk;
      f = a.e_frame[e0];
      if (f >= 0) {
        const double *Rt = P + 12 * f;
        for (int e = e0; e < e0 + chunk; ++e) {
          if (a.e_frame[e] < 0) break;
          edge_terms(a, Rt, a.X[3 * e], a.X[3 * e + 1], a.X[3 * e + 2], a.obs[2 * e], a.obs[2 * e + 1], v);
        }
      }
    }
    // frame-segmented warp reduction: chunks are frame-major, so a warp spans one frame (rarely two)
    unsigned todo = __ballot_sync(0xffffffffu, f >= 0);
    if (todo) {                                  // the usual case: every active lane of the warp holds edges of the same frame
      const int fl = __shfl_sync(0xffffffffu, f, __ffs(todo) - 1);
      if (__ballot_sync(0xffffffffu, f >= 0 && f != fl) == 0) {
        const double tot = warp_fold32(v, lane);          // idle lanes contribute their zeros
        if (lane < PF_V) s_wacc[warp * NV + fl * PF_V + lane] += tot;
        todo = 0;
      }
    }
    while (todo) {
      const int leader = __ffs(todo) - 1;
      const int fl = __shfl_sync(0xffffffffu, f, leader);
      const bool mine = f == fl;
      const unsigned m = __ballot_sync(0xffffffffu, mine);
      double t[32];
#pragma unroll
      for (int q = 0; q < 32; ++q) t[q] = mine ? v[q] : 0.0;
      const double tot = warp_fold32(t, lane);
      if (lane < PF_V) s_wacc[warp * NV + fl * PF_V + lane] += tot;
      todo &= ~m;
    }
  }
  __syncthreads();
  for (int i = tid; i < NV; i += PF_T) {
    // all PF_NW loads first (independent, in flight together), then the clearing stores, then the sum in warp order
    double part[PF_NW];
#pragma unroll
    for (int w = 0; w < PF_NW; ++w) part[w] = s_wacc[w * NV + i];
#pragma unroll
    for (int w = 0; w < PF_NW; ++w) s_wacc[w * NV + i] = 0;
    double s2 = 0;
#pragma unroll
    for (int w = 0; w < PF_NW; ++w) s2 += part[w];
    for (unsigned r = 0; r < csize; ++r) dsmem_push(recv + rank * NV + i, s2, bar, r);      // this CTA's row of every receive area
  }
}

// BATCH: one independent LM per cluster (mvo_vo_pnp_batch_dev's refits), job j = cluster index; its edges are rows j * E of
// e_frame / X / obs, its pose and stats rows j * 12 * F and j * 16.  Each job keeps its own damping and stopping rule.
template <int CH, bool CACHED, bool STORE, bool BATCH = false>
__global__ void __launch_bounds__(PF_T, 1) k_ba_pose(PoseArgs a) {
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned rank = cluster.block_rank(), csize = cluster.num_blocks();
  if constexpr (BATCH) {
    const size_t j = blockIdx.x / csize;
    a.e_frame += j * a.E; a.X += j * a.E * 3; a.obs += j * a.E * 2;
    a.poses += j * 12 * a.F; a.stats += j * 16;
  }
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long t_start = clock64();       // cycles outside the trial loop, debug only (stats 4..7, 12, 13; s_c[3..6] on thread 0)
  pdl_wait();                                // PnP finish / the glue kernel wrote what this kernel reads (launch_pdl.cuh)
  pdl_launch_dependents();
  const long long t_run = clock64();
  extern __shared__ __align__(16) double sm[];
  __shared__ __align__(8) unsigned long long s_bar[2];     // one per receive area
  __shared__ int s_ef[PF_T];
  __shared__ double s_c[8];                  // 0 lambda, 2 chi (initial), 3..6 cycle counts (debug)
  __shared__ double s_fscale[2][BA_MAXF], s_fstep[2][BA_MAXF];     // by trial parity: a solve never overwrites what a
  __shared__ int s_okf[2][BA_MAXF];                                // slower warp is still reading for the previous decision
  __shared__ int s_fslot[BA_MAXF], s_fcnt[BA_MAXF], s_cstart[BA_MAXF + 1], s_F;
  int F = a.F, nchunks = CACHED ? a.E / CH : a.E / a.chunk;
  if (STORE) {
    // The window is described by the device-resident frame buffer: listed slots (newest first) that hold at
    // least min_links observations become the frames of the graph (vo.cpp:423-426); every CTA derives the same
    // layout from the same counters.  Frame f owns chunks [s_cstart[f], s_cstart[f+1]) of CH edges each.
    if (tid == 0) {
      int nf = 0, c = 0;
      if (*a.st.skip_flag == 0)
        for (int k = 0; k < a.st.nslots; ++k) {
          const int n = min(a.st.cnt[a.st.slot[k]], a.st.cap);
          if (n >= a.st.min_links) { s_fslot[nf] = a.st.slot[k]; s_fcnt[nf] = n; s_cstart[nf] = c; c += (n + CH - 1) / CH; ++nf; }
        }
      s_cstart[nf] = c;
      if (c > (int)csize * PF_T) nf = -1;     // cannot happen: the host sizes CH from upper bounds of the counters
      s_F = nf;
    }
    __syncthreads();
    F = s_F;
    nchunks = F > 0 ? s_cstart[F] : 0;
    if (F <= 0) {                              // nothing to optimise (PnP failed / BA disabled / no frame with links)
      if (rank == 0 && tid == 0) { a.st.out_info[0] = F; a.st.out_info[1] = 0; a.stats[0] = a.stats[1] = a.stats[2] = a.stats[3] = 0; a.stats[15] = 0; }
      return;                                  // every CTA of the cluster takes this branch together
    }
    if (rank == 0 && tid == 0) {
      a.st.out_info[0] = F;
      for (int f = 0; f < F; ++f) a.st.out_info[2 + f] = s_fslot[f];
      a.st.out_info[1] = 0;                   // edges to map points that still exist, counted after the cluster barrier below
    }
  }
  const int NV = F * PF_V;
  double *s_pose = sm;                       // F*12
  double *s_try = s_pose + F * 12;           // F*12
  double *s_lin0 = s_try + F * 12;           // NV  linearisations (current / trial), ping-pong
  double *s_lin1 = s_lin0 + NV;              // NV
  double *s_recv = s_lin1 + NV;              // [2][csize][NV]  partials of every CTA, by exchange parity
  double *s_wacc = s_recv + 2 * csize * NV;  // PF_NW * NV
  double *s_ed = s_wacc + PF_NW * NV;        // CH*5*PF_T (CACHED only)
  if (tid == 0) {
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    mbar_init_fence();
  }
  if (STORE) { for (int i = tid; i < F * 12; i += PF_T) s_pose[i] = a.st.pose[(size_t)s_fslot[i / 12] * 12 + i % 12]; }
  else { for (int i = tid; i < F * 12; i += PF_T) s_pose[i] = a.poses[i]; }
  for (int i = tid; i < PF_NW * NV; i += PF_T) s_wacc[i] = 0;
  int my_edges = 0;
  if (STORE) {                               // this thread's chunk: gather the (fixed) map points of its observations
    const int c = pf_chunk_of(rank, tid, csize);
    int f = -1;
    if (c < nchunks) { f = 0; while (c >= s_cstart[f + 1]) ++f; }
    s_ef[tid] = f;
    const int e0 = f >= 0 ? (c - s_cstart[f]) * CH : 0;
#pragma unroll
    for (int k = 0; k < CH; ++k) {
      double *ed = s_ed + (size_t)k * 5 * PF_T + tid;
      const bool real = f >= 0 && e0 + k < s_fcnt[f];
      double X0 = 0, X1 = 0, X2 = 1, ou = -1e300, ov = 0;
      if (real) {
        const size_t o = (size_t)s_fslot[f] * a.st.cap + e0 + k;
        const int id = a.st.edge_map[o];
        if (id >= 0 && id < a.st.n_ids && a.st.alive[id]) {       // deleted map points leave the graph (vo.cpp:438-440)
          const float *mp = a.st.map_pts + 3 * (size_t)id;
          const float2 ob = a.st.edge_obs[o];
          X0 = mp[0]; X1 = mp[1]; X2 = mp[2]; ou = ob.x; ov = ob.y;
          ++my_edges;
        }
      }
      ed[0] = X0; ed[PF_T] = X1; ed[2 * PF_T] = X2; ed[3 * PF_T] = ou; ed[4 * PF_T] = ov;
    }
  } else if (CACHED) {                       // this thread's chunk -> shared memory, once
    const int c = pf_chunk_of(rank, tid, csize);
    int f = -1;
    if (c < nchunks) f = a.e_frame[c * CH];
    s_ef[tid] = f;
#pragma unroll
    for (int k = 0; k < CH; ++k) {
      double *ed = s_ed + (size_t)k * 5 * PF_T + tid;
      const int e = c * CH + k;
      const bool real = f >= 0 && a.e_frame[e] >= 0;
      ed[0] = real ? a.X[3 * e] : 0; ed[PF_T] = real ? a.X[3 * e + 1] : 0; ed[2 * PF_T] = real ? a.X[3 * e + 2] : 1;
      ed[3 * PF_T] = real ? a.obs[2 * e] : -1e300; ed[4 * PF_T] = real ? a.obs[2 * e + 1] : 0;
    }
  }
  // The one cluster barrier before the exchanges: every CTA's barriers are initialised before any CTA pushes into them.
  cluster.sync();
  const long long t_setup = clock64();
  if (tid == 0) { s_c[3] = (double)(t_run - t_start); s_c[4] = (double)(t_setup - t_run); s_c[6] = (double)t_run; }
  // Exchange x (0: the initial pass, then one per trial) lands in receive area x & 1 and completes phase x >> 1 of barrier
  // x & 1.  Two areas suffice: a CTA pushes exchange x + 2 only after it has received every CTA's exchange x + 1, which each CTA
  // sends after it has finished reading exchange x.  Bytes may land before the receiver arms the phase: the transaction count
  // goes negative, and the phase cannot complete before the arrival that arms it.
  int xchg = 0;
  const unsigned xbytes = csize * (unsigned)NV * sizeof(double);
  auto recv_of = [&](int x) { return s_recv + (x & 1) * csize * NV; };
  // Sum the partials of all CTAs in rank order once they have landed.  Warp w writes the rows of frames w, w + PF_NW, .. of dst,
  // which only that warp's lane 0 reads (the solve of those frames), so no CTA barrier follows.  Every warp also sums the chi2
  // of each frame into lane f, the same sum as dst[f * PF_V + 27]: the LM decision is taken from registers.
  auto gather = [&](double *dst) -> double {
    const double *in = recv_of(xchg);
    unsigned long long *bar = &s_bar[xchg & 1];
    if (tid == 0) mbar_arrive_expect_tx(bar, xbytes);
    mbar_wait_parity(bar, (xchg >> 1) & 1);
    auto sum_ranks = [&](int i, int j, double &si, double &sj) {      // elements i and j (-1: none), all loads in flight together
      double v[PF_MAXC], u[PF_MAXC];
#pragma unroll
      for (unsigned r = 0; r < PF_MAXC; ++r) {
        v[r] = r < csize && i >= 0 ? in[r * NV + i] : 0.0;
        u[r] = r < csize && j >= 0 ? in[r * NV + j] : 0.0;
      }
      si = 0; sj = 0;
#pragma unroll
      for (unsigned r = 0; r < PF_MAXC; ++r) { si += v[r]; sj += u[r]; }       // fixed rank order: identical in every CTA
    };
    double chi_f, row, unused;
    if (warp < F) {                                                 // warp-uniform: the other warps issue only the chi2 loads
      sum_ranks(lane < F ? lane * PF_V + 27 : -1, lane < PF_V ? warp * PF_V + lane : -1, chi_f, row);
      if (lane < PF_V) dst[warp * PF_V + lane] = row;
    } else {
      sum_ranks(lane < F ? lane * PF_V + 27 : -1, -1, chi_f, unused);
    }
    for (int f = warp + PF_NW; f < F; f += PF_NW)                   // only when PF_NW < F
      if (lane < PF_V) { sum_ranks(f * PF_V + lane, -1, row, unused); dst[f * PF_V + lane] = row; }
    ++xchg;
    return chi_f;
  };
  double *s_cur = s_lin0, *s_new = s_lin1;
  double *p_cur = s_pose, *p_try = s_try;    // poses ping-pong like the linearisations
  pose_pass<CH, CACHED>(a, F, nchunks, p_cur, s_ed, s_ef, s_wacc, recv_of(xchg), &s_bar[xchg & 1], rank, csize);
  gather(s_cur);
  __syncthreads();                           // the initial chi2 and damping below read every frame's rows
  if (STORE) {                               // behind the cluster barrier above: out_info[1] has been zeroed
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) my_edges += __shfl_xor_sync(0xffffffffu, my_edges, o);
    if ((tid & 31) == 0 && my_edges) atomicAdd(&a.st.out_info[1], my_edges);
  }
  if (tid == 0) {
    double chi = 0, md = 0;
    for (int f = 0; f < F; ++f) {
      chi += s_cur[f * PF_V + 27];
      if (!(a.fix_first && f == 0)) {
        const double *h = s_cur + f * PF_V;
        md = fmax(md, fmax(fmax(fabs(h[0]), fabs(h[6])), fmax(fmax(fabs(h[11]), fabs(h[15])), fmax(fabs(h[18]), fabs(h[20])))));
      }
    }
    s_c[2] = chi;
    s_c[0] = 1e-5 * md;        // computeLambdaInit
  }
  __syncthreads();
  const double chi_init = s_c[2];
  int it = 0, trials = 0, rejected = 0;
  bool terminate = false;
  long long ph[4] = {0, 0, 0, 0}, tmark = clock64();
  if (tid == 0) s_c[5] = (double)(tmark - t_setup);
#define PF_MARK(i) do { const long long t_ = clock64(); ph[i] += t_ - tmark; tmark = t_; } while (0)
  // LM control state lives in registers, replicated in every thread (all compute the same values)
  double lambda = s_c[0], ni = 2, chi_cur = s_c[2];
  for (; it < a.iters && !terminate; ++it) {
    int qmax = 0;
    double rho = 0;
    bool accepted = false, tiny = false;
    do {
      // per-frame 6x6 solve + trial pose + this frame's share of the gain denominator (every CTA, identically), on lane 0 of
      // the warp that gathered the frame's rows
      const int b = trials & 1;
      __syncwarp();
      for (int f = warp; f < F; f += PF_NW) {
        if (lane != 0) continue;
        double d[6] = {0, 0, 0, 0, 0, 0};
        bool ok = true;
        const bool fixed = a.fix_first && f == 0;
        if (!fixed) {
          ok = chol6_solve(s_cur + f * PF_V, s_cur + f * PF_V + 21, lambda, d);
          if (ok) se3_update(d, p_cur + 12 * f, p_try + 12 * f);
        }
        if (!ok || fixed)
          for (int q = 0; q < 12; ++q) p_try[12 * f + q] = p_cur[12 * f + q];
        double sc = 0, ms = 0;
        if (ok && !fixed)
#pragma unroll
          for (int q = 0; q < 6; ++q) { sc += d[q] * (lambda * d[q] + s_cur[f * PF_V + 21 + q]); ms = fmax(ms, fabs(d[q])); }   // computeScale, CURRENT b
        s_fscale[b][f] = sc;
        s_fstep[b][f] = ms;
        s_okf[b][f] = ok;
      }
      __syncthreads();
      PF_MARK(0);
      pose_pass<CH, CACHED>(a, F, nchunks, p_try, s_ed, s_ef, s_wacc, recv_of(xchg), &s_bar[xchg & 1], rank, csize);
      PF_MARK(1);
      // gain ratio and LM control (OptimizationAlgorithmLevenberg::solve), computed by every thread.  Status, gain denominator and
      // step size of the frames depend on the solve alone: reduced while the partials of the other CTAs are in flight.
      bool ok = true;
      double scale = 0, mstep = 0;
      for (int f = 0; f < F; ++f) {
        ok = ok && s_okf[b][f];
        scale += s_fscale[b][f];
        mstep = fmax(mstep, s_fstep[b][f]);
      }
      const double rscale = ranged_rcp(scale + 1e-3);
      tiny = a.step_tol > 0 && ok && mstep < a.step_tol;
      const double chi_f = gather(s_new);
      PF_MARK(2);
      {
        double temp = 0;
        for (int f = 0; f < F; ++f) temp += __shfl_sync(0xffffffffu, chi_f, f);
        if (!ok) temp = 1.7976931348623157e308;
        rho = (chi_cur - temp) * rscale;
        accepted = rho > 0 && isfinite(temp);
        if (accepted) {
          const double tr = 2 * rho - 1;
          double alpha = 1. - tr * tr * tr;
          alpha = fmin(alpha, 2. / 3.);
          lambda *= fmax(1. / 3., alpha);
          ni = 2;
          chi_cur = temp;
          double *t = s_cur; s_cur = s_new; s_new = t;      // the trial state becomes current: pointer swaps only
          t = p_cur; p_cur = p_try; p_try = t;
        } else {
          lambda *= ni;
          ni *= 2;
          ++rejected;
        }
      }
      ++qmax;
      ++trials;
      PF_MARK(3);
    } while (rho < 0 && qmax < 10 && !tiny);
    if (qmax == 10 || rho == 0) terminate = true;
    // Optional early exit (step_tol > 0; the PnP refit and the tracker's BA): once a trial step is below step_tol
    // the remaining g2o trials can only apply steps that are smaller still (the damping grows after a rejection,
    // the iteration contracts after an acceptance), so the poses are final to within step_tol.  A rejected tiny
    // step is not applied, exactly as g2o would restore it.
    if (tiny) terminate = true;
  }
  const long long t_loop = clock64();
  cluster.sync();       // the last pushes of a CTA may still be landing in a peer: nobody leaves before every CTA has them
  const long long t_end = clock64();
  if (rank == 0) {
    if (STORE) { for (int i = tid; i < F * 12; i += PF_T) a.st.pose[(size_t)s_fslot[i / 12] * 12 + i % 12] = p_cur[i]; }
    else { for (int i = tid; i < F * 12; i += PF_T) a.poses[i] = p_cur[i]; }
    if (tid == 0) {
      a.stats[0] = chi_init; a.stats[1] = chi_cur; a.stats[2] = it; a.stats[3] = lambda; a.stats[15] = trials;
      for (int q = 0; q < 4; ++q) a.stats[8 + q] = (double)ph[q];
      a.stats[4] = s_c[4];                         // edge gather into shared memory and the start barrier
      a.stats[5] = s_c[5];                         // initial pass, exchange and damping
      a.stats[6] = (double)(t_end - t_loop);       // exit barrier
      a.stats[7] = rejected;
      a.stats[12] = s_c[3];                        // wait for the predecessor (programmatic dependent launch)
      a.stats[13] = (double)t_end - s_c[6];        // the whole kernel after that wait
    }
  }
}

constexpr size_t pose_smem_doubles(int F, int cached_ch, int csize) {
  return (size_t)F * 24 + 2 * (size_t)F * PF_V + 2 * (size_t)csize * F * PF_V + (size_t)PF_NW * F * PF_V + (size_t)cached_ch * 5 * PF_T;
}
// The H100 lets a block opt in to 227 KB of shared memory; k_ba_pose's static __shared__ arrays take less than 3 KB of it.
constexpr size_t PF_SMEM_MAX = 224 * 1024;
static_assert(pose_smem_doubles(BA_MAXF, 4, PF_MAXC) * sizeof(double) <= PF_SMEM_MAX, "largest pose LM does not fit shared memory");

}  // namespace

static int pose_cluster_size() {
  static const int env_cluster = getenv("MVO_BA_CLUSTER") ? atoi(getenv("MVO_BA_CLUSTER")) : BA_CLUSTER;
  return (env_cluster >= 1 && env_cluster <= PF_MAXC) ? env_cluster : BA_CLUSTER;
}

static int pose_launch(mvo_ctx *ctx, void (*kern)(PoseArgs), const PoseArgs &a, int csz, size_t smem, int n_clusters = 1) {
  if (smem > PF_SMEM_MAX) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "pose BA: shared memory %zu B", smem);
  MVO_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  {
    KTimer kt(ctx, KC_BA);
    // one cluster per LM; may start under its predecessor's tail
    MVO_CUDA(ctx, launch_pdl(ctx->stream, (unsigned)(n_clusters * csz), PF_T, smem, (unsigned)csz, kern, a));
  }
  ctx->launches++;
  return MVO_OK;
}

// Launch the pose-only LM on device-resident edge arrays (also used by the PnP refit).  n_jobs > 0: that many independent one-frame
// LMs in one launch (chunk 1), job j on rows j * E of the edge arrays, d_poses + 12 j and d_stats + 16 j; each job's sums run in
// the order of a single launch with the same E.
int mvo_ba_pose_launch(mvo_ctx *ctx, int F, int E, int chunk, const int32_t *d_eframe, const double *d_X, const double *d_obs, double fx, double fy,
                       double cx, double cy, const double *info, int iters, int use_huber, double huber, int fix_first,
                       double step_tol, double *d_poses, double *d_stats, int n_jobs = 0) {
  PoseArgs a;
  memset(&a, 0, sizeof a);
  a.chunk = chunk;
  a.F = F; a.E = E; a.iters = iters; a.fix_first = fix_first; a.use_huber = use_huber;
  a.fx = fx; a.fy = fy; a.cx = cx; a.cy = cy;
  a.i00 = info[0]; a.i01 = info[1]; a.i10 = info[2]; a.i11 = info[3];
  a.huber = huber; a.step_tol = step_tol;
  a.e_frame = d_eframe; a.X = d_X; a.obs = d_obs; a.poses = d_poses; a.stats = d_stats;
  const int csz = pose_cluster_size();
  const bool cached = chunk >= 1 && chunk <= 4 && E / chunk <= csz * PF_T;
  const size_t smem = pose_smem_doubles(F, cached ? chunk : 0, csz) * sizeof(double);
  if (n_jobs > 0) {
    if (F != 1 || chunk != 1) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "pose BA batch: one frame and chunk 1 per job");
    return pose_launch(ctx, cached ? k_ba_pose<1, true, false, true> : k_ba_pose<1, false, false, true>, a, csz, smem, n_jobs);
  }
  void (*kern)(PoseArgs) = k_ba_pose<1, false, false>;
  if (cached) {
    switch (chunk) {
      case 1: kern = k_ba_pose<1, true, false>; break;
      case 2: kern = k_ba_pose<2, true, false>; break;
      case 3: kern = k_ba_pose<3, true, false>; break;
      default: kern = k_ba_pose<4, true, false>; break;
    }
  }
  return pose_launch(ctx, kern, a, csz, smem);
}

// The same LM over the tracker's device-resident frame buffer (track.cu): the graph is assembled by the kernel
// from the per-frame observation lists and counters, nothing crosses PCIe.  e_upper = upper bound of the edge
// count (the host knows every counter except the newest frame's, which is bounded by its match count).
int mvo_ba_pose_store_launch(mvo_ctx *ctx, const MvoPoseStore &st, int e_upper, double fx, double fy, double cx, double cy,
                             const double *info, int iters, int use_huber, double huber, double step_tol, double *d_stats) {
  if (st.nslots < 1 || st.nslots > BA_MAXF) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "pose BA: %d frames (supported 1..%d)", st.nslots, BA_MAXF);
  const int csz = pose_cluster_size();
  int chunk = 1;
  while ((long)(e_upper + (long)st.nslots * (chunk - 1)) > (long)chunk * csz * PF_T && chunk <= 4) ++chunk;
  if (chunk > 4) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "pose BA: %d edges exceed the device-resident path", e_upper);
  PoseArgs a;
  memset(&a, 0, sizeof a);
  a.chunk = chunk;
  a.F = st.nslots; a.E = 0; a.iters = iters; a.fix_first = 0; a.use_huber = use_huber;
  a.fx = fx; a.fy = fy; a.cx = cx; a.cy = cy;
  a.i00 = info[0]; a.i01 = info[1]; a.i10 = info[2]; a.i11 = info[3];
  a.huber = huber; a.step_tol = step_tol;
  a.stats = d_stats;
  a.st = st;
  const size_t smem = pose_smem_doubles(st.nslots, chunk, csz) * sizeof(double);
  void (*kern)(PoseArgs) = nullptr;
  switch (chunk) {
    case 1: kern = k_ba_pose<1, true, true>; break;
    case 2: kern = k_ba_pose<2, true, true>; break;
    case 3: kern = k_ba_pose<3, true, true>; break;
    default: kern = k_ba_pose<4, true, true>; break;
  }
  return pose_launch(ctx, kern, a, csz, smem);
}

// Test entry (not part of the C ABI): the device-resident pose LM on a frame buffer given as host arrays.  Uploads them, runs
// mvo_ba_pose_store_launch as the tracker does, waits, and returns the whole ring of poses (ring x 12, in/out), out_info[0..17]
// and the 16 stats (both in/out: entries the kernel does not write keep the caller's values).  nslots may exceed 16 to reach
// the launcher's check; only the first 16 slots are copied.
extern "C" int mvo_test_ba_pose_store(mvo_ctx *ctx, const float *map_pts, const uint8_t *alive, int n_ids, const int32_t *edge_map,
                                      const float *edge_obs, const int32_t *cnt, double *pose, int ring, int cap, const int32_t *slots,
                                      int nslots, int min_links, int skip_flag, int e_upper, const double *K, const double *info,
                                      int iters, int use_huber, double huber, double step_tol, int32_t *out_info, double *stats) {
  if (!ctx || !map_pts || !alive || !edge_map || !edge_obs || !cnt || !pose || !slots || !K || !info || !out_info || !stats)
    return MVO_ERR_INVALID_ARG;
  if (n_ids < 0 || ring < 1 || cap < 1 || nslots < 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "pose BA test: bad sizes");
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t nrc = (size_t)ring * cap;
  size_t o = 0;
  const size_t o_map = o;  o = al(o + (size_t)n_ids * 12 + 12);
  const size_t o_alv = o;  o = al(o + (size_t)n_ids + 1);
  const size_t o_em = o;   o = al(o + nrc * 4);
  const size_t o_eo = o;   o = al(o + nrc * 8);
  const size_t o_cnt = o;  o = al(o + (size_t)ring * 4);
  const size_t o_pose = o; o = al(o + (size_t)ring * 96);
  const size_t o_flag = o; o = al(o + 4);
  const size_t o_info = o; o = al(o + 18 * 4);
  const size_t o_st = o;   o = al(o + 16 * 8);
  MVO_TRY(mvo_reserve(ctx, ctx->ba_buf, o));
  uint8_t *d = (uint8_t *)ctx->ba_buf.p;
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_map, map_pts, (size_t)n_ids * 12, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_alv, alive, (size_t)n_ids, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_em, edge_map, nrc * 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_eo, edge_obs, nrc * 8, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_cnt, cnt, (size_t)ring * 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_pose, pose, (size_t)ring * 96, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_flag, &skip_flag, 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_info, out_info, 18 * 4, cudaMemcpyHostToDevice, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(d + o_st, stats, 16 * 8, cudaMemcpyHostToDevice, ctx->stream));
  MvoPoseStore st;
  memset(&st, 0, sizeof st);
  st.map_pts = (const float *)(d + o_map); st.alive = d + o_alv; st.n_ids = n_ids;
  st.edge_map = (const int32_t *)(d + o_em); st.edge_obs = (const float2 *)(d + o_eo); st.cnt = (const int32_t *)(d + o_cnt);
  st.pose = (double *)(d + o_pose); st.cap = cap; st.nslots = nslots; st.min_links = min_links;
  for (int k = 0; k < nslots && k < 16; ++k) st.slot[k] = slots[k];
  st.skip_flag = (const int32_t *)(d + o_flag); st.out_info = (int32_t *)(d + o_info);
  // fy = fx, as the tracker passes it (g2o_ba.cpp ignores fy)
  const int rc = mvo_ba_pose_store_launch(ctx, st, e_upper, K[0], K[0], K[2], K[5], info, iters, use_huber, huber, step_tol,
                                          (double *)(d + o_st));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));      // the uploads above are done with the host arrays on every path
  if (rc != MVO_OK) return rc;
  MVO_CUDA(ctx, cudaMemcpyAsync(pose, d + o_pose, (size_t)ring * 96, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(out_info, d + o_info, 18 * 4, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(stats, d + o_st, 16 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MVO_OK;
}

// g2o_ba.cpp:183-190: camera->world T_w_c (4x4 row-major) -> world->camera [R|t] = (T_w_c)^-1 (R row-major, then t)
static void T_w_c_to_Rt(const double *T, double *q) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) q[i * 3 + j] = T[j * 4 + i];
    q[9 + i] = -(T[0 * 4 + i] * T[3] + T[1 * 4 + i] * T[7] + T[2 * 4 + i] * T[11]);
  }
}

// g2o_ba.cpp:298-305: world->camera [R|t] -> camera->world T_w_c
static void Rt_to_T_w_c(const double *p, double *T) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[i * 4 + j] = p[j * 3 + i];
    T[i * 4 + 3] = -(p[i] * p[9] + p[3 + i] * p[10] + p[6 + i] * p[11]);
  }
  T[12] = T[13] = T[14] = 0;
  T[15] = 1;
}

// Shared driver for bundleAdjustment and optimizeSingleFrame.
static int run_ba(mvo_ctx *ctx, double *poses_T_w_c, int F, float *points, int P, const int32_t *edge_frame,
                  const int32_t *edge_point, const float *obs, int E, const double *K, const double *info,
                  int fix_points, int update_points, int iterations, int use_huber, double *stats) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!poses_T_w_c || !K || !info || (P > 0 && !points) || (E > 0 && (!edge_frame || !edge_point || !obs)))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "bundleAdjustment: null pointer");
  if (F < 1 || F > BA_MAXF) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "bundleAdjustment: %d frames (supported 1..%d)", F, BA_MAXF);
  if (P < 0 || E < 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "bundleAdjustment: negative size");
  for (int k = 0; k < E; ++k)
    if (edge_frame[k] < 0 || edge_frame[k] >= F || edge_point[k] < 0 || edge_point[k] >= P)
      return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "bundleAdjustment: edge %d references frame %d / point %d", k, edge_frame[k], edge_point[k]);
  if (stats) stats[0] = stats[1] = stats[2] = stats[3] = 0;
  const int fix_first = ctx->prm.ba_fix_first_pose ? 1 : 0;
  const int nact = F - fix_first;
  if (E == 0 || iterations == 0 || (nact == 0 && fix_points)) return MVO_OK;      // nothing to optimise
  MVO_CUDA(ctx, cudaSetDevice(ctx->device));

  if (fix_points) {
    // ---- pose-only LM: edges frame-major (stable), each with its fixed 3-D point ----
    std::vector<int32_t> order(E), fstart(F + 1, 0);
    for (int k = 0; k < E; ++k) fstart[edge_frame[k] + 1]++;
    for (int f = 0; f < F; ++f) fstart[f + 1] += fstart[f];
    {
      std::vector<int32_t> cur(fstart.begin(), fstart.begin() + F);
      for (int k = 0; k < E; ++k) order[cur[edge_frame[k]]++] = k;
    }
    // chunk = edges per thread so that all chunks fit one sweep of the 8 x 512 threads
    const int csz = pose_cluster_size();
    int chunk = 1;
    while ((long)(E + (long)F * (chunk - 1)) > (long)chunk * csz * PF_T && chunk < 64) ++chunk;
    int Ep = 0;
    for (int f = 0; f < F; ++f) Ep += ((fstart[f + 1] - fstart[f] + chunk - 1) / chunk) * chunk;
    auto al2 = [](size_t v) { return (v + 255) & ~(size_t)255; };
    size_t o = 0;
    const size_t o_fr = o;   o = al2(o + (size_t)Ep * 4 + 4);
    const size_t o_X = o;    o = al2(o + (size_t)Ep * 24 + 24);
    const size_t o_obs = o;  o = al2(o + (size_t)Ep * 16 + 16);
    const size_t o_pose = o; o = al2(o + (size_t)F * 96);
    const size_t in_end = o;
    const size_t o_stats = o; o = al2(o + 256);
    MVO_TRY(mvo_reserve(ctx, ctx->ba_buf, o));
    MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_a, o + 256));
    uint8_t *h = (uint8_t *)ctx->h_a.p, *d = (uint8_t *)ctx->ba_buf.p;
    int32_t *hf = (int32_t *)(h + o_fr);
    double *hX = (double *)(h + o_X), *hobs = (double *)(h + o_obs), *hpose = (double *)(h + o_pose);
    {
      int w = 0;
      for (int f = 0; f < F; ++f) {
        for (int i = fstart[f]; i < fstart[f + 1]; ++i, ++w) {
          const int k = order[i];
          hf[w] = f;
          const float *p = points + 3 * (size_t)edge_point[k];
          hX[3 * w] = p[0]; hX[3 * w + 1] = p[1]; hX[3 * w + 2] = p[2];
          hobs[2 * w] = obs[2 * k]; hobs[2 * w + 1] = obs[2 * k + 1];
        }
        for (; w % chunk; ++w) { hf[w] = -1; hX[3 * w] = hX[3 * w + 1] = 0; hX[3 * w + 2] = 1; hobs[2 * w] = hobs[2 * w + 1] = 0; }
      }
    }
    for (int f = 0; f < F; ++f) T_w_c_to_Rt(poses_T_w_c + 16 * f, hpose + 12 * f);
    MVO_CUDA(ctx, cudaMemcpyAsync(d, h, in_end, cudaMemcpyHostToDevice, ctx->stream));
    MVO_TRY(mvo_ba_pose_launch(ctx, F, Ep, chunk, (const int32_t *)(d + o_fr), (const double *)(d + o_X), (const double *)(d + o_obs),
                               K[0], K[0], K[2], K[5], info, iterations, use_huber && ctx->prm.ba_huber_delta > 0,
                               ctx->prm.ba_huber_delta, fix_first, ctx->prm.ba_step_tol, (double *)(d + o_pose), (double *)(d + o_stats)));
    double *h_stats = (double *)(h + o_stats);
    MVO_CUDA(ctx, cudaMemcpyAsync(hpose, d + o_pose, (size_t)F * 96, cudaMemcpyDeviceToHost, ctx->stream));
    MVO_CUDA(ctx, cudaMemcpyAsync(h_stats, d + o_stats, 128, cudaMemcpyDeviceToHost, ctx->stream));
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int f = 0; f < F; ++f) Rt_to_T_w_c(hpose + 12 * f, poses_T_w_c + 16 * f);
    if (stats) memcpy(stats, h_stats, 32);
    if (getenv("MVO_BA_DEBUG"))
      fprintf(stderr, "k_ba_pose: F=%d E=%d Ep=%d chunk=%d cluster=%d it=%.0f trials=%.0f rejected=%.0f cycles solve=%.0f pass=%.0f "
              "gather=%.0f decide=%.0f | pdl_wait=%.0f setup=%.0f init=%.0f exit=%.0f kernel=%.0f\n", F, E, Ep, chunk, csz, h_stats[2],
              h_stats[15], h_stats[7], h_stats[8], h_stats[9], h_stats[10], h_stats[11], h_stats[12], h_stats[4], h_stats[5], h_stats[6],
              h_stats[13]);
    return MVO_OK;
  }

  // CSR by point, edges of a point ordered by frame (stable in the caller's order otherwise)
  std::vector<int32_t> pt_start(P + 2, 0), e_fr(E);
  std::vector<double> e_obs(2 * (size_t)E);
  {
    std::vector<int32_t> order(E);
    for (int k = 0; k < E; ++k) pt_start[edge_point[k] + 1]++;
    for (int p = 0; p < P; ++p) pt_start[p + 1] += pt_start[p];
    std::vector<int32_t> cur(pt_start.begin(), pt_start.begin() + P + 1);
    for (int k = 0; k < E; ++k) order[cur[edge_point[k]]++] = k;
    for (int p = 0; p < P; ++p)
      std::stable_sort(order.begin() + pt_start[p], order.begin() + pt_start[p + 1],
                       [&](int32_t x, int32_t y) { return edge_frame[x] < edge_frame[y]; });
    for (int i = 0; i < E; ++i) {
      e_fr[i] = edge_frame[order[i]];
      e_obs[2 * i] = obs[2 * order[i]];
      e_obs[2 * i + 1] = obs[2 * order[i] + 1];
    }
  }
  std::vector<double> pose12((size_t)F * 12), pts_d(3 * (size_t)std::max(P, 1));
  for (int f = 0; f < F; ++f) T_w_c_to_Rt(poses_T_w_c + 16 * f, pose12.data() + 12 * f);
  for (int i = 0; i < 3 * P; ++i) pts_d[i] = points[i];

  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  size_t o = 0;
  const size_t o_start = o; o = al(o + (size_t)(P + 1) * 4);
  const size_t o_fr = o;    o = al(o + (size_t)E * 4);
  const size_t o_obs = o;   o = al(o + (size_t)E * 16);
  const size_t o_pose = o;  o = al(o + (size_t)F * 96);
  const size_t o_pa = o;    o = al(o + (size_t)P * 24 + 24);
  const size_t in_end = o;
  const size_t o_pb = o;    o = al(o + (size_t)P * 24 + 24);
  const size_t o_hll = o;   o = al(o + (size_t)P * 48 + 48);
  const size_t o_bl = o;    o = al(o + (size_t)P * 24 + 24);
  const size_t o_hinv = o;  o = al(o + (size_t)P * 48 + 48);
  const size_t o_wd = o;    o = al(o + (size_t)P * F * 144 + 144);
  const size_t o_stats = o; o = al(o + 256);
  MVO_TRY(mvo_reserve(ctx, ctx->ba_buf, o));
  MVO_TRY(mvo_reserve_pinned(ctx, ctx->h_a, in_end + 4096));
  uint8_t *h = (uint8_t *)ctx->h_a.p, *d = (uint8_t *)ctx->ba_buf.p;
  memcpy(h + o_start, pt_start.data(), (size_t)(P + 1) * 4);
  memcpy(h + o_fr, e_fr.data(), (size_t)E * 4);
  memcpy(h + o_obs, e_obs.data(), (size_t)E * 16);
  memcpy(h + o_pose, pose12.data(), (size_t)F * 96);
  memcpy(h + o_pa, pts_d.data(), (size_t)P * 24);
  MVO_CUDA(ctx, cudaMemcpyAsync(d, h, in_end, cudaMemcpyHostToDevice, ctx->stream));

  BaArgs a;
  a.F = F; a.P = P; a.E = E; a.iters = iterations; a.fix_first = fix_first;
  a.use_huber = use_huber && ctx->prm.ba_huber_delta > 0;
  a.f = K[0]; a.cx = K[2]; a.cy = K[5];                      // g2o_ba.cpp:219-220: fy is ignored
  a.i00 = info[0]; a.i01 = info[1]; a.i10 = info[2]; a.i11 = info[3];
  a.huber = ctx->prm.ba_huber_delta;
  a.pt_start = (const int32_t *)(d + o_start); a.e_frame = (const int32_t *)(d + o_fr); a.obs = (const double *)(d + o_obs);
  a.poses = (double *)(d + o_pose); a.pts_a = (double *)(d + o_pa); a.pts_b = (double *)(d + o_pb);
  a.Hll = (double *)(d + o_hll); a.bl = (double *)(d + o_bl); a.Hinv = (double *)(d + o_hinv); a.Wd = (double *)(d + o_wd);
  // stats[7]: rejected trials, stats[8..15]: phase cycles and trials (debug)
  a.stats = (double *)(d + o_stats); a.pts_sel = (int32_t *)(d + o_stats + 32);
  // staging chunk for the Schur products: <= 64 KB of shared memory
  int pc = (int)(65536 / ((size_t)F * 36 * 8 + 24));
  pc = std::max(1, std::min(pc, 64));
  a.pc = pc;
  const size_t smem = ba_smem_doubles(F, nact, pc) * sizeof(double);
  if (smem > 220 * 1024) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "bundleAdjustment: shared memory %zu B", smem);
  MVO_CUDA(ctx, cudaFuncSetAttribute(k_ba, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(BA_CLUSTER);
  cfg.blockDim = dim3(BA_T);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = BA_CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  {
    KTimer kt(ctx, KC_BA);
    MVO_CUDA(ctx, cudaLaunchKernelEx(&cfg, k_ba, a));
  }
  ctx->launches++;
  // results
  double *h_pose = (double *)(h + o_pose), *h_stats = (double *)(h + in_end);
  MVO_CUDA(ctx, cudaMemcpyAsync(h_pose, a.poses, (size_t)F * 96, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaMemcpyAsync(h_stats, a.stats, 128, cudaMemcpyDeviceToHost, ctx->stream));
  MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (update_points && P > 0) {
    const int sel = *(int32_t *)((uint8_t *)h_stats + 32);
    MVO_CUDA(ctx, cudaMemcpyAsync(h + o_pa, sel ? a.pts_b : a.pts_a, (size_t)P * 24, cudaMemcpyDeviceToHost, ctx->stream));
    MVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const double *pd = (const double *)(h + o_pa);
    for (int i = 0; i < 3 * P; ++i) points[i] = (float)pd[i];      // g2o_ba.cpp:313-315
  }
  for (int f = 0; f < F; ++f) Rt_to_T_w_c(h_pose + 12 * f, poses_T_w_c + 16 * f);
  if (stats) memcpy(stats, h_stats, 32);
  if (getenv("MVO_BA_DEBUG")) {
    fprintf(stderr, "k_ba: F=%d P=%d E=%d pc=%d per=%d nact=%d smem=%zu it=%.0f trials=%.0f rejected=%.0f cycles A=%.0f B=%.0f C=%.0f "
            "D=%.0f E=%.0f F=%.0f sync=%.0f\n", F, P, E, pc, (P + BA_CLUSTER - 1) / BA_CLUSTER, nact, smem, h_stats[2], h_stats[15],
            h_stats[7], h_stats[8], h_stats[9], h_stats[10], h_stats[11], h_stats[12], h_stats[13], h_stats[14]);
  }
  return MVO_OK;
}

extern "C" {

int mvo_bundle_adjustment(mvo_ctx *ctx, double *poses_T_w_c, int n_frames, float *points, int n_points,
                          const int32_t *edge_frame, const int32_t *edge_point, const float *obs, int n_edges,
                          const double *K, const double *information, int fix_points, int update_points, double *stats) {
  return run_ba(ctx, poses_T_w_c, n_frames, points, n_points, edge_frame, edge_point, obs, n_edges, K, information,
                fix_points, update_points, ctx ? ctx->prm.ba_iterations : 0, 1, stats);
}

int mvo_optimize_single_frame(mvo_ctx *ctx, double *pose_T_w_c, float *points, const float *obs, int n_points,
                              const double *K, int fix_points, int update_points) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (n_points < 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "optimizeSingleFrame: negative size");
  // g2o_ba.cpp:82-98: one edge per (point i, pose 0), identity information, no robust kernel
  std::vector<int32_t> ef(n_points, 0), ep(n_points);
  for (int i = 0; i < n_points; ++i) ep[i] = i;
  const double I2[4] = {1, 0, 0, 1};
  mvo_params saved = ctx->prm;
  ctx->prm.ba_fix_first_pose = 0;
  const int rc = run_ba(ctx, pose_T_w_c, 1, points, n_points, ef.data(), ep.data(), obs, n_points, K, I2, fix_points,
                        update_points, ctx->prm.ba_iterations, 0, nullptr);
  ctx->prm = saved;
  return rc;
}

}  // extern "C"
