// The kernels of the batched RANSAC PnP (P3P hypotheses, scoring, arg-max + consensus set) — the text nvcc compiles, in a
// header so that the CPU test tier can build it for the host (tests/cpp/pnp_emu.cpp through tests/cpp/cuda_emu.h).
// Included by pnp.cu inside its anonymous namespace.  PNP_DYN_SMEM(type, name) declares the scoring kernel's dynamic shared
// memory (`extern __shared__ type name[]` for nvcc).
#pragma once
#include "pdl_device.cuh"

struct PnpCam { double fx, fy, cx, cy; };

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

struct V3 { double x, y, z; };
__device__ __forceinline__ V3 v3(double x, double y, double z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 operator*(double s, V3 a) { return v3(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ V3 unit(V3 a) { return rsqrt(dot(a, a)) * a; }

// symmetric 3x3 stored as m00 m01 m02 m11 m12 m22
struct S3 { double a, b, c, d, e, f; };
__device__ __forceinline__ S3 adj(const S3 &m) {   // adjugate (also symmetric)
  S3 r;
  r.a = m.d * m.f - m.e * m.e;
  r.b = m.c * m.e - m.b * m.f;
  r.c = m.b * m.e - m.c * m.d;
  r.d = m.a * m.f - m.c * m.c;
  r.e = m.b * m.c - m.a * m.e;
  r.f = m.a * m.d - m.b * m.b;
  return r;
}
__device__ __forceinline__ double det(const S3 &m) {
  return m.a * (m.d * m.f - m.e * m.e) - m.b * (m.b * m.f - m.c * m.e) + m.c * (m.b * m.e - m.c * m.d);
}
__device__ __forceinline__ double trprod(const S3 &p, const S3 &q) {   // trace(P Q)
  return p.a * q.a + p.d * q.d + p.f * q.f + 2.0 * (p.b * q.b + p.c * q.c + p.e * q.e);
}

// real roots of c3 x^3 + c2 x^2 + c1 x + c0; returns count (1..3), Newton-polished
__device__ int cubic_roots(double c3, double c2, double c1, double c0, double *r) {
  int n = 0;
  const double scale = fabs(c3) + fabs(c2) + fabs(c1) + fabs(c0);
  if (!(scale > 0)) return 0;
  if (fabs(c3) < 1e-14 * scale) {            // quadratic / linear
    if (fabs(c2) < 1e-14 * scale) {
      if (fabs(c1) < 1e-14 * scale) return 0;
      r[0] = -c0 / c1;
      return 1;
    }
    const double disc = c1 * c1 - 4 * c2 * c0;
    if (disc < 0) return 0;
    const double q = -0.5 * (c1 + copysign(sqrt(disc), c1));
    r[n++] = q / c2;
    if (q != 0) r[n++] = c0 / q;
    return n;
  }
  const double a = c2 / c3, b = c1 / c3, c = c0 / c3;
  const double Q = (a * a - 3 * b) / 9, R = (2 * a * a * a - 9 * a * b + 27 * c) / 54;
  if (R * R < Q * Q * Q) {
    const double th = acos(fmax(-1.0, fmin(1.0, R / sqrt(Q * Q * Q)))), sq = -2 * sqrt(Q);
    r[0] = sq * cos(th / 3) - a / 3;
    r[1] = sq * cos((th + 6.283185307179586) / 3) - a / 3;
    r[2] = sq * cos((th - 6.283185307179586) / 3) - a / 3;
    n = 3;
  } else {
    const double A = -copysign(cbrt(fabs(R) + sqrt(fmax(R * R - Q * Q * Q, 0.0))), R);
    const double B = A != 0 ? Q / A : 0;
    r[0] = A + B - a / 3;
    n = 1;
  }
  for (int i = 0; i < n; ++i) {
    double x = r[i];
    for (int it = 0; it < 3; ++it) {
      const double fx = ((c3 * x + c2) * x + c1) * x + c0, dfx = (3 * c3 * x + 2 * c2) * x + c1;
      if (dfx != 0) x -= fx / dfx;
    }
    r[i] = x;
  }
  return n;
}

struct Pose { double R[9]; double t[3]; };

__device__ __forceinline__ double reproj_err2(const Pose &P, const PnpCam &cam, V3 X, double u, double v) {
  const double x = P.R[0] * X.x + P.R[1] * X.y + P.R[2] * X.z + P.t[0];
  const double y = P.R[3] * X.x + P.R[4] * X.y + P.R[5] * X.z + P.t[1];
  const double z = P.R[6] * X.x + P.R[7] * X.y + P.R[8] * X.z + P.t[2];
  if (!(z > 1e-9)) return 1e300;       // behind the camera never counts as an inlier
  const double iz = 1.0 / z;
  const double du = cam.fx * x * iz + cam.cx - u, dv = cam.fy * y * iz + cam.cy - v;
  return du * du + dv * dv;
}

// P3P: up to 4 poses mapping world X[0..2] onto unit bearings f[0..2]
__device__ int p3p(const V3 *X, const V3 *f, Pose *out) {
  const double a = dot(X[1] - X[2], X[1] - X[2]), b = dot(X[0] - X[2], X[0] - X[2]), c = dot(X[0] - X[1], X[0] - X[1]);
  const double ca = dot(f[1], f[2]), cb = dot(f[0], f[2]), cg = dot(f[0], f[1]);
  if (!(a > 1e-18 && b > 1e-18 && c > 1e-18)) return 0;
  // conics in (u, v, 1) with u = s2/s1, v = s3/s1 (depth ratios):
  //   C1: b(u^2 + v^2 - 2uv ca) - a(1 + v^2 - 2v cb) = 0
  //   C2: b(1 + u^2 - 2u cg)    - c(1 + v^2 - 2v cb) = 0
  S3 C1, C2;
  C1.a = b;  C1.b = -b * ca; C1.c = 0;       C1.d = b - a; C1.e = a * cb; C1.f = -a;
  C2.a = b;  C2.b = 0;       C2.c = -b * cg; C2.d = -c;    C2.e = c * cb; C2.f = b - c;
  const S3 A1 = adj(C1), A2 = adj(C2);
  double roots[3];
  const int nr = cubic_roots(det(C2), trprod(C1, A2), trprod(A1, C2), det(C1), roots);
  // pick the pencil member that is the best-conditioned REAL line pair
  S3 D, AD;
  double best = 0;
  int bi = -1;
  for (int i = 0; i < nr; ++i) {
    const double g = roots[i];
    S3 Di;
    Di.a = C1.a + g * C2.a; Di.b = C1.b + g * C2.b; Di.c = C1.c + g * C2.c;
    Di.d = C1.d + g * C2.d; Di.e = C1.e + g * C2.e; Di.f = C1.f + g * C2.f;
    const S3 Ai = adj(Di);
    const double nrm = fabs(Di.a) + fabs(Di.b) + fabs(Di.c) + fabs(Di.d) + fabs(Di.e) + fabs(Di.f);
    const double m = fmax(fmax(-Ai.a, -Ai.d), -Ai.f) / (nrm * nrm + 1e-300);
    if (m > best) { best = m; bi = i; D = Di; AD = Ai; }
  }
  if (bi < 0) return 0;
  // p = l x m from adj(D) = -(p p^T)
  double p0, p1, p2;
  if (-AD.a >= -AD.d && -AD.a >= -AD.f) { const double s = sqrt(-AD.a); p0 = -AD.a / s; p1 = -AD.b / s; p2 = -AD.c / s; }
  else if (-AD.d >= -AD.f)              { const double s = sqrt(-AD.d); p0 = -AD.b / s; p1 = -AD.d / s; p2 = -AD.e / s; }
  else                                   { const double s = sqrt(-AD.f); p0 = -AD.c / s; p1 = -AD.e / s; p2 = -AD.f / s; }
  // N = D + [p]_x = 2 m l^T : rows are multiples of one line, columns of the other
  const double N[3][3] = {{D.a, D.b - p2, D.c + p1}, {D.b + p2, D.d, D.e - p0}, {D.c - p1, D.e + p0, D.f}};
  int ri = 0, cj = 0;
  double bm = -1;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      if (fabs(N[i][j]) > bm) { bm = fabs(N[i][j]); ri = i; cj = j; }
  if (!(bm > 0)) return 0;
  const double lines[2][3] = {{N[ri][0], N[ri][1], N[ri][2]}, {N[0][cj], N[1][cj], N[2][cj]}};
  int ns = 0;
  for (int li = 0; li < 2; ++li) {
    const double L0 = lines[li][0], L1 = lines[li][1], L2 = lines[li][2];
    const bool solve_v = fabs(L0) >= fabs(L1);      // u = al*v + be   (else v = al*u + be)
    const double den = solve_v ? L0 : L1;
    if (!(fabs(den) > 0)) continue;
    const double al = -(solve_v ? L1 : L0) / den, be = -L2 / den;
    // substitute into C2
    double q2, q1, q0;
    if (solve_v) {
      q2 = C2.a * al * al + 2 * C2.b * al + C2.d;
      q1 = 2 * (C2.a * al * be + C2.b * be + C2.c * al + C2.e);
      q0 = C2.a * be * be + 2 * C2.c * be + C2.f;
    } else {
      q2 = C2.d * al * al + 2 * C2.b * al + C2.a;
      q1 = 2 * (C2.d * al * be + C2.b * be + C2.e * al + C2.c);
      q0 = C2.d * be * be + 2 * C2.e * be + C2.f;
    }
    double w[2];
    int nw = 0;
    if (fabs(q2) < 1e-14 * (fabs(q1) + fabs(q0))) { if (q1 != 0) w[nw++] = -q0 / q1; }
    else {
      const double disc = q1 * q1 - 4 * q2 * q0;
      if (disc >= 0) {
        const double q = -0.5 * (q1 + copysign(sqrt(disc), q1));
        w[nw++] = q / q2;
        if (q != 0) w[nw++] = q0 / q;
      }
    }
    for (int k = 0; k < nw && ns < 4; ++k) {
      const double u = solve_v ? al * w[k] + be : w[k];
      const double v = solve_v ? w[k] : al * w[k] + be;
      if (!(u > 0 && v > 0)) continue;
      const double dn = 1 + v * v - 2 * v * cb;
      if (!(dn > 1e-18)) continue;
      const double s1 = sqrt(b / dn), s2 = u * s1, s3 = v * s1;
      const V3 P1 = s1 * f[0], P2 = s2 * f[1], P3 = s3 * f[2];
      // rigid transform from the two orthonormal triads
      const V3 e1 = unit(X[1] - X[0]), e3 = unit(cross(e1, X[2] - X[0])), e2 = cross(e3, e1);
      const V3 g1 = unit(P2 - P1), g3 = unit(cross(g1, P3 - P1)), g2 = cross(g3, g1);
      Pose &T = out[ns];
      T.R[0] = g1.x * e1.x + g2.x * e2.x + g3.x * e3.x; T.R[1] = g1.x * e1.y + g2.x * e2.y + g3.x * e3.y; T.R[2] = g1.x * e1.z + g2.x * e2.z + g3.x * e3.z;
      T.R[3] = g1.y * e1.x + g2.y * e2.x + g3.y * e3.x; T.R[4] = g1.y * e1.y + g2.y * e2.y + g3.y * e3.y; T.R[5] = g1.y * e1.z + g2.y * e2.z + g3.y * e3.z;
      T.R[6] = g1.z * e1.x + g2.z * e2.x + g3.z * e3.x; T.R[7] = g1.z * e1.y + g2.z * e2.y + g3.z * e3.y; T.R[8] = g1.z * e1.z + g2.z * e2.z + g3.z * e3.z;
      T.t[0] = P1.x - (T.R[0] * X[0].x + T.R[1] * X[0].y + T.R[2] * X[0].z);
      T.t[1] = P1.y - (T.R[3] * X[0].x + T.R[4] * X[0].y + T.R[5] * X[0].z);
      T.t[2] = P1.z - (T.R[6] * X[0].x + T.R[7] * X[0].y + T.R[8] * X[0].z);
      bool ok = true;
      for (int q = 0; q < 9; ++q) ok = ok && isfinite(T.R[q]);
      for (int q = 0; q < 3; ++q) ok = ok && isfinite(T.t[q]);
      if (ok) ++ns;
    }
  }
  return ns;
}

// The batch form of these kernels (BATCH = true, mvo_vo_pnp_batch_dev) runs one RANSAC per job of a map-matches batch: job j's
// correspondences are rows j * n of p3 / p2 (n = the batch's cap), its hypotheses and counts rows j * H.  Its count reaches the
// scoring and finish kernels through n_dev (one entry per job), as the tracker's device count does.
struct PnpJobs {
  const mvo_map_matches_result *mm;       // the map-matches records: status and n_matches of every job
  const double *T_prev;                   // 16 per job: the previous frame's T_w_c
  int min_pts;                            // mvo_track_params::min_pnp_points
  int32_t *n, *status;                    // out: the job's effective count and status, written by block (0, j)
};

// Job j's status and the count its RANSAC runs on: 0 for a failed job (every hypothesis is then invalid) and for one below
// min_pts (no solvePnPRansac call, vo.cpp:304-311).  Each check comes before anything is read through the value it checks.
__device__ __forceinline__ void pnp_job_count(const PnpJobs &jb, int j, int cap, int *status, int *count) {
  const mvo_map_matches_result r = jb.mm[j];
  int st = r.status, c = 0;
  if (st == MVO_OK && (r.n_matches < 0 || r.n_matches > cap)) st = MVO_ERR_INVALID_ARG;
  if (st == MVO_OK)
    for (int q = 0; q < 16; ++q)
      if (!isfinite(jb.T_prev[(size_t)j * 16 + q])) st = MVO_ERR_INVALID_ARG;
  if (st == MVO_OK && r.n_matches >= jb.min_pts) c = r.n_matches;
  *status = st;
  *count = c;
}

template <bool BATCH = false>
__global__ void __launch_bounds__(128)
k_pnp_hypotheses(const float *__restrict__ p3, const float *__restrict__ p2, int n, const int32_t *__restrict__ n_dev,
                 PnpCam cam, uint64_t seed, int H, double *__restrict__ poses, int32_t *__restrict__ valid, PnpJobs jb = PnpJobs()) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  pdl_wait();                             // the predecessor (match filter) wrote n_dev / p3 / p2
  pdl_launch_dependents();
  if constexpr (BATCH) {                  // grid (ceil(H / 128), n_jobs); n = cap
    const int j = blockIdx.y;
    int st, cnt;
    pnp_job_count(jb, j, n, &st, &cnt);
    if (blockIdx.x == 0 && threadIdx.x == 0) { jb.n[j] = cnt; jb.status[j] = st; }
    p3 += (size_t)j * n * 3; p2 += (size_t)j * n * 2;
    poses += (size_t)j * H * 12; valid += (size_t)j * H;
    n = cnt;
  }
  if (h >= H) return;
  if (n_dev) n = min(n, *n_dev);          // device-resident tracker: the pair count never visited the host
  if (n < 4) { valid[h] = 0; return; }
  int idx[4];
  uint64_t ctr = 0;
  for (int k = 0; k < 4; ++k) {
    for (int attempt = 0; attempt < 64; ++attempt) {
      const uint64_t r = splitmix64(seed ^ splitmix64(((uint64_t)h << 20) ^ ctr++));
      int cand = (int)(r % (uint64_t)n);
      bool dup = false;
      for (int q = 0; q < k; ++q) dup |= idx[q] == cand;
      idx[k] = cand;
      if (!dup) break;
    }
  }
  V3 X[4], f[3];
  double u4 = 0, v4 = 0;
  for (int k = 0; k < 4; ++k) {
    X[k] = v3(p3[3 * idx[k]], p3[3 * idx[k] + 1], p3[3 * idx[k] + 2]);
    const double u = p2[2 * idx[k]], v = p2[2 * idx[k] + 1];
    if (k < 3) f[k] = unit(v3((u - cam.cx) / cam.fx, (v - cam.cy) / cam.fy, 1.0));
    else { u4 = u; v4 = v; }
  }
  Pose sol[4];
  const int ns = p3p(X, f, sol);
  int bi = -1;
  double be = 1e300;
  for (int s = 0; s < ns; ++s) {
    // all three sample points must be in front of the camera and reproject onto themselves
    const double e4 = reproj_err2(sol[s], cam, X[3], u4, v4);
    if (e4 < be) { be = e4; bi = s; }
  }
  double *o = poses + (size_t)h * 12;
  if (bi >= 0 && be < 1e299) {
    for (int q = 0; q < 9; ++q) o[q] = sol[bi].R[q];
    for (int q = 0; q < 3; ++q) o[9 + q] = sol[bi].t[q];
    valid[h] = 1;
  } else {
    for (int q = 0; q < 12; ++q) o[q] = 0;
    valid[h] = 0;
  }
}

// Scoring: count(err^2 <= thr^2) per hypothesis, the count an fp64 evaluation gives, at fp32 cost.  Every point is
// first reprojected in fp32 together with a bound M on the fp32 error of err^2 (inputs are exact floats; R, t, K are
// rounded once; 3 FMAs, one approximate reciprocal, 2 FMAs — see the derivation at delta below).  Only points whose
// err^2 lies within M of the threshold (or whose depth is within the bound of zero) are re-evaluated in fp64 — a
// fraction of a percent — so the counts are identical to the all-fp64 kernel this replaces, while the fp64 pipe
// (64 lanes/clk/SM, division included) no longer bounds the stage.  One hypothesis per warp, points staged once
// per CTA in shared memory.
// BATCH: grid (x, n_jobs), job j = blockIdx.y, its correspondences staged in the n (= cap) rows of shared memory.
template <bool BATCH = false>
__global__ void __launch_bounds__(256)
k_pnp_score(const float *__restrict__ p3, const float *__restrict__ p2, int n, const int32_t *__restrict__ n_dev, PnpCam cam,
            double thr2, int H, const double *__restrict__ poses, const int32_t *__restrict__ valid, int32_t *__restrict__ counts) {
  PNP_DYN_SMEM(float, s_pts);      // [n][5]: X Y Z u v
  __shared__ float s_wmax[8];
  if constexpr (BATCH) {
    const int j = blockIdx.y;
    p3 += (size_t)j * n * 3; p2 += (size_t)j * n * 2; n_dev += j;
    poses += (size_t)j * H * 12; valid += (size_t)j * H; counts += (size_t)j * H;
  }
  pdl_wait();
  pdl_launch_dependents();
  if (n_dev) n = min(n, *n_dev);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  float mloc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float X = p3[3 * i], Y = p3[3 * i + 1], Z = p3[3 * i + 2];
    s_pts[5 * i] = X; s_pts[5 * i + 1] = Y; s_pts[5 * i + 2] = Z;
    s_pts[5 * i + 3] = p2[2 * i]; s_pts[5 * i + 4] = p2[2 * i + 1];
    mloc = fmaxf(mloc, fabsf(X) + fabsf(Y) + fabsf(Z));
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, d));
  if (lane == 0) s_wmax[warp] = mloc;
  __syncthreads();
  float mmax = 0.f;
  for (int w = 0; w < wpb; ++w) mmax = fmaxf(mmax, s_wmax[w]);
  const float EPS = 1.1920929e-7f;      // 2^-23
  const float fxf = (float)cam.fx, fyf = (float)cam.fy, cxf = (float)cam.cx, cyf = (float)cam.cy, thr2f = (float)thr2;
  for (int h = blockIdx.x * wpb + warp; h < H; h += gridDim.x * wpb) {
    if (!valid[h]) { if (lane == 0) counts[h] = -1; continue; }
    Pose P;
    const double *o = poses + (size_t)h * 12;
    for (int q = 0; q < 9; ++q) P.R[q] = o[q];
    for (int q = 0; q < 3; ++q) P.t[q] = o[9 + q];
    float Rf[9], tf[3];
#pragma unroll
    for (int q = 0; q < 9; ++q) Rf[q] = (float)P.R[q];
#pragma unroll
    for (int q = 0; q < 3; ++q) tf[q] = (float)P.t[q];
    // |fl(x) - x| <= 4 EPS (max|R_ij| (|X|+|Y|+|Z|) + |t|) for each camera coordinate (coefficient rounding + 3 FMAs,
    // twice the worst case); ca = that bound times the focal length
    float rmax = 1.f;
#pragma unroll
    for (int q = 0; q < 9; ++q) rmax = fmaxf(rmax, fabsf(Rf[q]));
    const float a = 4.f * EPS * (rmax * mmax + fmaxf(fabsf(tf[0]), fmaxf(fabsf(tf[1]), fabsf(tf[2]))));
    const float ca = fmaxf(fxf, fyf) * a;
    const float c0 = 2.f * EPS * (fabsf(cxf) + fabsf(cyf));
    int c = 0;
    for (int i = lane; i < n; i += 32) {
      const float *s = s_pts + 5 * i;
      const float X = s[0], Y = s[1], Z = s[2], u = s[3], v = s[4];
      const float x = fmaf(Rf[0], X, fmaf(Rf[1], Y, fmaf(Rf[2], Z, tf[0])));
      const float y = fmaf(Rf[3], X, fmaf(Rf[4], Y, fmaf(Rf[5], Z, tf[1])));
      const float z = fmaf(Rf[6], X, fmaf(Rf[7], Y, fmaf(Rf[8], Z, tf[2])));
      const float iz = __fdividef(1.f, z);
      const float xz = x * iz, yz = y * iz;
      const float up = fxf * xz, vp = fyf * yz;
      const float du = (up + cxf) - u, dv = (vp + cyf) - v;
      const float e2 = fmaf(du, du, dv * dv);
      // delta bounds the fp32 error of either projected coordinate:
      //   f * (a + |x/z| a) / |z|   (errors of x, y, z)  +  5 EPS |f x/z|  (reciprocal, products, focal rounding)  +  2 EPS |c|
      const float delta = fmaf(ca * fabsf(iz), 2.f + fabsf(xz) + fabsf(yz), fmaf(5.f * EPS, fabsf(up) + fabsf(vp), c0));
      const float M = 2.f * (fmaf(2.f * (fabsf(du) + fabsf(dv)), delta, 2.f * delta * delta) + 4.f * EPS * (e2 + thr2f));
      const bool front = z > 2.f * a + 1e-6f;                    // fp64 rule: z > 1e-9
      const bool behind = z < -(2.f * a + 1e-6f);
      const bool in = front && (e2 + M <= thr2f), out = behind || (front && (e2 - M > thr2f));
      bool inl = in;
      if (!in && !out) inl = reproj_err2(P, cam, v3(X, Y, Z), u, v) <= thr2;      // too close to call in fp32
      c += inl;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if (lane == 0) counts[h] = c;
  }
}

constexpr int FIN_T = 1024;

#include "pnp_cv_kernels.cuh"   // mvo_params::pnp_mode = 1 (cv::solvePnPRansac's flow)


// out: [0..8] R, [9..11] t, then int32 n_inliers at out_i[0], best hypothesis at out_i[1],
// inlier indices in inl[] and the one-frame edge list (ex, eo, ef) for the pose-only LM refit.
// mode 0: arg-max + consensus set; mode 1: every point is an inlier, pose_io holds the start pose; mode 2: cv::solvePnPRansac's
// flow (pnp_cv_kernels.cuh): the model RANSACPointSetRegistrator::run ends with + its consensus set under the float rule.
// BATCH: one CTA per job (j = blockIdx.x); every row of the job at its offset, out_i 4 and pose_io 12 per job.
template <bool BATCH = false>
__global__ void __launch_bounds__(FIN_T)
k_pnp_finish(const float *__restrict__ p3, const float *__restrict__ p2, int n, const int32_t *__restrict__ n_dev, PnpCam cam,
             double thr2, int H, const double *__restrict__ poses, const int32_t *__restrict__ counts, int mode, int max_iters,
             double *__restrict__ pose_io, int32_t *__restrict__ out_i, int32_t *__restrict__ inl,
             double *__restrict__ ex, double *__restrict__ eo, int32_t *__restrict__ ef) {
  __shared__ double s_red[32 * 28];
  __shared__ double s_pose[12];
  __shared__ int s_best, s_cnt[32];
  if constexpr (BATCH) {
    const int j = blockIdx.x;
    p3 += (size_t)j * n * 3; p2 += (size_t)j * n * 2; n_dev += j;
    poses += (size_t)j * H * 12; counts += (size_t)j * H;
    pose_io += (size_t)j * 12; out_i += (size_t)j * 4; inl += (size_t)j * n;
    ex += (size_t)j * n * 3; eo += (size_t)j * n * 2; ef += (size_t)j * n;
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_upper = n;                 // the refit is launched for this many edge slots
  pdl_wait();
  pdl_launch_dependents();
  if (n_dev) n = min(n, *n_dev);
  int n_in = 0;
  const bool cv_rule = mode == 2;
  const float thr2f = (float)thr2;
  if (mode == 0 || mode == 2) {
    // this thread's chunk of points: loaded first so that the L2 round trip overlaps the arg-max
    constexpr int MAXPER = 4;             // n <= 4096 on the register path; beyond that the points are re-read
    const int per = (n + FIN_T - 1) / FIN_T, b0 = tid * per, e0 = min(b0 + per, n);
    float px[MAXPER][5];
    if (per <= MAXPER) {
#pragma unroll
      for (int k = 0; k < MAXPER; ++k) {
        const int i = b0 + k;
        if (i < e0) { px[k][0] = p3[3 * i]; px[k][1] = p3[3 * i + 1]; px[k][2] = p3[3 * i + 2]; px[k][3] = p2[2 * i]; px[k][4] = p2[2 * i + 1]; }
      }
    }
    // arg-max of the inlier count, ties -> lowest hypothesis index
    long long best = -1;
    for (int h = tid; h < (cv_rule ? 0 : H); h += FIN_T) {
      const long long key = ((long long)counts[h] << 20) | (long long)(0xFFFFF - h);
      best = key > best ? key : best;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) { const long long o = __shfl_xor_sync(0xffffffffu, best, d); best = o > best ? o : best; }
    long long *s_k = reinterpret_cast<long long *>(s_red);
    if (lane == 0) s_k[warp] = best;
    __syncthreads();
    if (tid == 0) {
      long long b = -1;
      for (int w = 0; w < 32; ++w) b = s_k[w] > b ? s_k[w] : b;
      const int cnt = (int)(b >> 20);
      s_best = cnt >= 4 ? (int)(0xFFFFF - (b & 0xFFFFF)) : -1;
      if (cv_rule) { int iters_run = 0; s_best = cvp_replay(counts, H, n, 0.999, &iters_run); out_i[3] = iters_run; }
    }
    __syncthreads();
    if (s_best < 0) {
      if (tid == 0) { out_i[0] = 0; out_i[1] = -1; out_i[2] = 0; }
      for (int j = tid; j < n_upper; j += FIN_T) ef[j] = -1;
      if (tid < 12) pose_io[tid] = (tid == 0 || tid == 4 || tid == 8) ? 1.0 : 0.0;
      return;
    }
    if (tid < 12) s_pose[tid] = poses[(size_t)s_best * 12 + tid];
    __syncthreads();
    // ordered compaction of the consensus set (contiguous chunk per thread)
    Pose P;
    for (int q = 0; q < 9; ++q) P.R[q] = s_pose[q];
    for (int q = 0; q < 3; ++q) P.t[q] = s_pose[9 + q];
    // one evaluation per point: the chunk's points and verdicts stay in registers between the count and the write
    unsigned flags = 0;
    int mine = 0;
    if (per <= MAXPER) {
#pragma unroll
      for (int k = 0; k < MAXPER; ++k) {
        const int i = b0 + k;
        if (i < e0 && (cv_rule ? cvp_is_inlier(P, cam, v3(px[k][0], px[k][1], px[k][2]), px[k][3], px[k][4], thr2f)
                               : reproj_err2(P, cam, v3(px[k][0], px[k][1], px[k][2]), px[k][3], px[k][4]) <= thr2)) { flags |= 1u << k; ++mine; }
      }
    } else {
      for (int i = b0; i < e0; ++i)
        mine += cv_rule ? cvp_is_inlier(P, cam, v3(p3[3 * i], p3[3 * i + 1], p3[3 * i + 2]), p2[2 * i], p2[2 * i + 1], thr2f)
                        : reproj_err2(P, cam, v3(p3[3 * i], p3[3 * i + 1], p3[3 * i + 2]), p2[2 * i], p2[2 * i + 1]) <= thr2;
    }
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
    if (lane == 31) s_cnt[warp] = incl;
    __syncthreads();
    int off = incl - mine;
    for (int w = 0; w < 32; ++w) { if (w < warp) off += s_cnt[w]; n_in += s_cnt[w]; }
    // consensus set in ascending order + the one-frame edge list for the pose-only LM refit (ba.cu: k_ba_pose)
    if (per <= MAXPER) {
#pragma unroll
      for (int k = 0; k < MAXPER; ++k)
        if (flags & (1u << k)) {
          inl[off] = b0 + k;
          ex[3 * off] = px[k][0]; ex[3 * off + 1] = px[k][1]; ex[3 * off + 2] = px[k][2];
          eo[2 * off] = px[k][3]; eo[2 * off + 1] = px[k][4];
          ef[off] = 0;
          ++off;
        }
    } else {
      for (int i = b0; i < e0; ++i)
        if (cv_rule ? cvp_is_inlier(P, cam, v3(p3[3 * i], p3[3 * i + 1], p3[3 * i + 2]), p2[2 * i], p2[2 * i + 1], thr2f)
                    : reproj_err2(P, cam, v3(p3[3 * i], p3[3 * i + 1], p3[3 * i + 2]), p2[2 * i], p2[2 * i + 1]) <= thr2) {
          inl[off] = i;
          ex[3 * off] = p3[3 * i]; ex[3 * off + 1] = p3[3 * i + 1]; ex[3 * off + 2] = p3[3 * i + 2];
          eo[2 * off] = p2[2 * i]; eo[2 * off + 1] = p2[2 * i + 1];
          ef[off] = 0;
          ++off;
        }
    }
  } else {
    n_in = n;
    if (tid < 12) s_pose[tid] = pose_io[tid];
    __syncthreads();
    // refine-only entry: every point is an edge
    for (int j = tid; j < n_in; j += FIN_T) {
      ex[3 * j] = p3[3 * j]; ex[3 * j + 1] = p3[3 * j + 1]; ex[3 * j + 2] = p3[3 * j + 2];
      eo[2 * j] = p2[2 * j]; eo[2 * j + 1] = p2[2 * j + 1];
      ef[j] = 0;
    }
  }

  for (int j = n_in + tid; j < n_upper; j += FIN_T) ef[j] = -1;       // masked out of the refit
  const int it = 0;
  if (tid < 12) pose_io[tid] = s_pose[tid];
  if (tid == 0) { out_i[0] = n_in; out_i[1] = mode != 1 ? s_best : -1; out_i[2] = it; }
}

