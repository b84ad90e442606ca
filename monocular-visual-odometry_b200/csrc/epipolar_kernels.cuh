// The kernels of the two-view stage (essential matrix, triangulation, homography): the text nvcc compiles, kept in a header
// so that the CPU test tier can build the same kernels for the host and run them one OS thread per CUDA thread
// (tests/cpp/two_view_emu.cpp).  Included by epipolar.cu inside its anonymous namespace, after epipolar_math.cuh.
// EPI_DYN_SMEM(type, name) declares the dynamic shared-memory array of a kernel (`extern __shared__ type name[]` for nvcc).
#pragma once

__device__ __forceinline__ uint64_t splitmix64e(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

struct EpiCam { double f, cx, cy; };      // findEssentialMat(focal, pp): one focal length (epipolar_geometry.cpp:26-27)

// The kernel bodies below are device functions of one pair; the kernels of the batch sections run them for every pair (one pair
// per blockIdx.y, or one cluster per pair for the finish).  A single-pair call is a batch of one (epipolar.cu).

// hypothesis h: counter-based minimal sample of 8 distinct correspondences, epi::essential_from_8
__device__ __forceinline__ void epi_hypothesis(const float *__restrict__ p1, const float *__restrict__ p2, int n, EpiCam cam, uint64_t seed,
                                               int h, double *__restrict__ Es, int32_t *__restrict__ valid) {
  int idx[8];
  uint64_t ctr = 0;
  for (int k = 0; k < 8; ++k)
    for (int attempt = 0; attempt < 64; ++attempt) {
      const uint64_t r = splitmix64e(seed ^ splitmix64e(((uint64_t)h << 20) ^ ctr++));
      const int cand = (int)(r % (uint64_t)n);
      bool dup = false;
      for (int q = 0; q < k; ++q) dup |= idx[q] == cand;
      idx[k] = cand;
      if (!dup) break;
    }
  double a[16], b[16];
  const double inv = 1.0 / cam.f;
  for (int k = 0; k < 8; ++k) {
    a[2 * k] = ((double)p1[2 * idx[k]] - cam.cx) * inv; a[2 * k + 1] = ((double)p1[2 * idx[k] + 1] - cam.cy) * inv;
    b[2 * k] = ((double)p2[2 * idx[k]] - cam.cx) * inv; b[2 * k + 1] = ((double)p2[2 * idx[k] + 1] - cam.cy) * inv;
  }
  double E[9];
  int reason = 0;
  const bool ok = epi::essential_from_8(a, b, E, &reason);
  for (int q = 0; q < 9; ++q) Es[(size_t)h * 9 + q] = ok ? E[q] : 0.0;
  valid[h] = ok ? 1 : -reason;             // <= 0: rejected sample (the reason is kept for MVO_EPI_DEBUG)
}

// Sampson consensus of hypotheses cta * warps + warp, strided by ncta * warps; the CTA stages the n points once
__device__ __forceinline__ void epi_score_run(const float *__restrict__ p1, const float *__restrict__ p2, int n, EpiCam cam, double thr2, int H,
                                              const double *__restrict__ Es, const int32_t *__restrict__ valid, int32_t *__restrict__ counts,
                                              int cta, int ncta) {
  EPI_DYN_SMEM(double, s_pt);         // [n][4] calibrated coordinates x1 y1 x2 y2
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    s_pt[4 * i] = ((double)p1[2 * i] - cam.cx) / cam.f; s_pt[4 * i + 1] = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
    s_pt[4 * i + 2] = ((double)p2[2 * i] - cam.cx) / cam.f; s_pt[4 * i + 3] = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  for (int h = cta * wpb + warp; h < H; h += ncta * wpb) {
    if (valid[h] <= 0) { if (lane == 0) counts[h] = -1; continue; }
    double E[9];
    for (int q = 0; q < 9; ++q) E[q] = Es[(size_t)h * 9 + q];
    int c = 0;
    for (int i = lane; i < n; i += 32) c += epi::sampson_err(E, s_pt[4 * i], s_pt[4 * i + 1], s_pt[4 * i + 2], s_pt[4 * i + 3]) <= thr2;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if (lane == 0) counts[h] = c;
  }
}

constexpr int EFIN_T = 256;       // 255 registers per thread: the 20 (54) Gauss-Newton accumulators stay in registers (1024 threads = 64 registers spilled them)
constexpr int EPI_LO_ROUNDS = 3, EPI_GN_ITERS = 8;

__device__ __forceinline__ void skew_times(const double *t, const double *R, double *E) {      // E = [t]x R
  for (int j = 0; j < 3; ++j) {
    E[0 * 3 + j] = -t[2] * R[1 * 3 + j] + t[1] * R[2 * 3 + j];
    E[1 * 3 + j] = t[2] * R[0 * 3 + j] - t[0] * R[2 * 3 + j];
    E[2 * 3 + j] = -t[1] * R[0 * 3 + j] + t[0] * R[1 * 3 + j];
  }
}

// exp of a rotation vector.  Below 0.1 rad the two coefficients come from their Taylor series (remainder < 1e-19: the Gauss-Newton
// steps and the 1e-6 probing rotations all live there), above from sin / cos.
__device__ __forceinline__ void so3_exp(const double *w, double *R) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  double A, B;
  if (th2 < 1e-2) {
    A = 1 - th2 * (1.0 / 6) * (1 - th2 * (1.0 / 20) * (1 - th2 * (1.0 / 42) * (1 - th2 * (1.0 / 72) * (1 - th2 * (1.0 / 110)))));
    B = 0.5 * (1 - th2 * (1.0 / 12) * (1 - th2 * (1.0 / 30) * (1 - th2 * (1.0 / 56) * (1 - th2 * (1.0 / 90) * (1 - th2 * (1.0 / 132))))));
  } else {
    const double th = sqrt(th2);
    A = sin(th) / th; B = (1 - cos(th)) / th2;
  }
  const double x = w[0], y = w[1], z = w[2];
  R[0] = 1 - B * (y * y + z * z); R[1] = -A * z + B * x * y;      R[2] = A * y + B * x * z;
  R[3] = A * z + B * x * y;       R[4] = 1 - B * (x * x + z * z); R[5] = -A * x + B * y * z;
  R[6] = -A * y + B * x * z;      R[7] = A * x + B * y * z;       R[8] = 1 - B * (x * x + y * y);
}

// The estimate the Gauss-Newton iteration of epi_finish_run moves: R, the unit translation t and an orthonormal basis (b1, b2) of
// the tangent plane of the unit sphere at t.  A step d = (rotation increment on the right, two tangent-plane components).
struct EpiPose { double R[9], t[3], b1[3], b2[3]; };

__device__ __forceinline__ void epi_tangent_basis(EpiPose &P) {
  double a[3] = {1, 0, 0};
  if (fabs(P.t[0]) >= 0.9) { a[0] = 0; a[1] = 1; }
  epi::cross3(P.t, a, P.b1);
  const double in1 = 1.0 / sqrt(P.b1[0] * P.b1[0] + P.b1[1] * P.b1[1] + P.b1[2] * P.b1[2]);
  for (int i = 0; i < 3; ++i) P.b1[i] *= in1;
  epi::cross3(P.t, P.b1, P.b2);
}

__device__ __forceinline__ void epi_apply_step(EpiPose &P, const double *d) {
  double dR[9], Ro[9];
  so3_exp(d, dR);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Ro[i * 3 + j] = P.R[i * 3] * dR[j] + P.R[i * 3 + 1] * dR[3 + j] + P.R[i * 3 + 2] * dR[6 + j];
  for (int i = 0; i < 9; ++i) P.R[i] = Ro[i];
  double n = 0;
  for (int i = 0; i < 3; ++i) { P.t[i] = P.t[i] + d[3] * P.b1[i] + d[4] * P.b2[i]; n += P.t[i] * P.t[i]; }
  const double in = 1.0 / sqrt(n);
  for (int i = 0; i < 3; ++i) P.t[i] *= in;
  epi_tangent_basis(P);
}

// E at the estimate (k = 0) or at the estimate moved by 1e-6 along tangent direction k - 1 (k = 1..5): a rotation about axis
// k - 1 (k <= 3), a move of t along b1 / b2 (k = 4, 5)
__device__ __forceinline__ void epi_probe_E(const EpiPose &P, int k, double *E) {
  double Rk[9], tk[3];
  for (int i = 0; i < 9; ++i) Rk[i] = P.R[i];
  for (int i = 0; i < 3; ++i) tk[i] = P.t[i];
  if (k >= 1 && k <= 3) {
    double d[3] = {0, 0, 0}, dR[9];
    d[k - 1] = 1e-6;
    so3_exp(d, dR);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Rk[i * 3 + j] = P.R[i * 3] * dR[j] + P.R[i * 3 + 1] * dR[3 + j] + P.R[i * 3 + 2] * dR[6 + j];
  } else if (k >= 4) {
    const double *b = k == 4 ? P.b1 : P.b2;
    double n = 0;
    for (int i = 0; i < 3; ++i) { tk[i] = P.t[i] + 1e-6 * b[i]; n += tk[i] * tk[i]; }
    const double in = 1.0 / sqrt(n);
    for (int i = 0; i < 3; ++i) tk[i] *= in;
  }
  skew_times(tk, Rk, E);
}

// (J^T J + eps I) dx = -J^T r for the 5 x 5 system in sum[0..14] (upper triangle, row-major) / sum[15..19] (J^T r).  The damped
// matrix is symmetric positive definite: elimination without pivoting, every index static (the 30 entries stay in registers; the
// pivoting version indexed rows dynamically and ran out of local memory).  false: a non-positive pivot or a non-finite step.
__device__ __forceinline__ bool epi_solve5(const double *sum, double *dx, double *mx_out) {
  double A[5][6];
  int q = 0;
#pragma unroll
  for (int r = 0; r < 5; ++r)
#pragma unroll
    for (int c = r; c < 5; ++c) { A[r][c] = sum[q]; A[c][r] = sum[q]; ++q; }
  double tr = 0;
#pragma unroll
  for (int r = 0; r < 5; ++r) tr += A[r][r];
#pragma unroll
  for (int r = 0; r < 5; ++r) { A[r][r] += 1e-12 * tr + 1e-300; A[r][5] = -sum[15 + r]; }
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    if (!(A[k][k] > 0)) ok = false;
    const double ip = 1.0 / A[k][k];
#pragma unroll
    for (int r = k + 1; r < 5; ++r) {
      const double f = A[r][k] * ip;
#pragma unroll
      for (int c = k + 1; c < 6; ++c) A[r][c] -= f * A[k][c];
    }
#pragma unroll
    for (int c = k + 1; c < 6; ++c) A[k][c] *= ip;                 // row k of the unit upper triangle
  }
  double mx = 0;
#pragma unroll
  for (int r = 4; r >= 0; --r) {
    double v = A[r][5];
#pragma unroll
    for (int c = r + 1; c < 5; ++c) v -= A[r][c] * dx[c];
    dx[r] = v;
  }
#pragma unroll
  for (int r = 0; r < 5; ++r) { if (!isfinite(dx[r])) ok = false; mx = fmax(mx, fabs(dx[r])); }
  *mx_out = mx;
  return ok;
}

__device__ __forceinline__ double sampson_signed(const double *E, double x1, double y1, double x2, double y2) {
  const double Ex0 = E[0] * x1 + E[1] * y1 + E[2], Ex1 = E[3] * x1 + E[4] * y1 + E[5], Ex2 = E[6] * x1 + E[7] * y1 + E[8];
  const double Et0 = E[0] * x2 + E[3] * y2 + E[6], Et1 = E[1] * x2 + E[4] * y2 + E[7];
  return (x2 * Ex0 + y2 * Ex1 + Ex2) * rsqrt(Ex0 * Ex0 + Ex1 * Ex1 + Et0 * Et0 + Et1 * Et1);
}

// out_d: [0..8] E (scaled so that E[8] = 1, epipolar_geometry.cpp:37), [9..17] R1, [18..26] R2, [27..29] t of
// decomposeEssentialMat; out_i: [0] inliers, [1] best hypothesis, [3] consensus of the best minimal model, [4] consensus after the
// local optimisation, [5] Gauss-Newton iterations run, [8..11] cheirality votes (k_epi_vote_batch)
//
// After the arg-max the best minimal model is locally optimised (LO-RANSAC style): EPI_LO_ROUNDS times its consensus
// set is re-selected and (R, t/|t|) is re-estimated on it by Gauss-Newton on the signed Sampson residual (5 degrees of
// freedom, forward-difference Jacobian).  OpenCV returns the minimal five-point model as it is; the eight-point
// minimal models used here are noisier, and the local optimisation more than makes up for it (pose errors against
// synthetic truth ~10x below cv2's on the test scenes).  The reported inliers are the consensus set of the final model.
//
// One thread-block CLUSTER of EFIN_C CTAs (round 2; before: one CTA): a Gauss-Newton iteration is ~500 fp64 instructions per
// correspondence, which kept ONE SM busy for every iteration (16 iterations per call).  Every CTA owns a slice of the
// correspondences; the partial normal equations meet through distributed shared memory — each CTA reads all partials in rank
// order, so all of them hold bit-identical sums, take the same step and need no broadcast (the scheme of k_ba_pose).  All block
// state lives in DYNAMIC shared memory (the CPU test tier gives every block of a cluster its own copy of that).
constexpr int EFIN_C = 8;

struct EpiFinSmem {
  long long k[EFIN_T / 32];
  double E[9], R1[9], R2[9], t[3], R[9], E0[9];
  double Ek[6][9], red[EFIN_T / 32][20], part[2][20], sumv[20];
  int cnt[EFIN_T / 32], best, stop, ipart[4];
};

__device__ __forceinline__ void epi_finish_run(const float *__restrict__ p1, const float *__restrict__ p2, int n, EpiCam cam, double thr2, int H,
                                               const double *__restrict__ Es, const int32_t *__restrict__ counts, double *__restrict__ out_d,
                                               int32_t *__restrict__ out_i, int32_t *__restrict__ inl) {
  EPI_DYN_SMEM(double, smraw);
  EpiFinSmem &S = *reinterpret_cast<EpiFinSmem *>(smraw);
  cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
  const unsigned rank = cluster.block_rank(), csize = cluster.num_blocks();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // arg-max over the hypotheses: every CTA for itself (identical result)
  long long best = -1;
  for (int h = tid; h < H; h += EFIN_T) {
    const long long key = ((long long)counts[h] << 20) | (long long)(0xFFFFF - h);
    best = key > best ? key : best;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { const long long o = __shfl_xor_sync(0xffffffffu, best, d); best = o > best ? o : best; }
  if (lane == 0) S.k[warp] = best;
  __syncthreads();
  if (tid == 0) {
    long long b = -1;
    for (int w = 0; w < EFIN_T / 32; ++w) b = S.k[w] > b ? S.k[w] : b;
    S.best = (int)(b >> 20) >= 8 ? (int)(0xFFFFF - (b & 0xFFFFF)) : -1;
    if (rank == 0) out_i[3] = (int)(b >> 20);
  }
  __syncthreads();
  if (S.best < 0) {                                                  // every CTA takes this branch together
    if (rank == 0 && tid == 0) { out_i[0] = 0; out_i[1] = -1; out_i[2] = 0; }
    return;
  }
  if (tid == 0) {
    for (int q = 0; q < 9; ++q) S.E[q] = Es[(size_t)S.best * 9 + q];
    epi::decompose_essential(S.E, S.R1, S.R2, S.t);
    for (int q = 0; q < 9; ++q) { S.R[q] = S.R1[q]; S.E0[q] = S.E[q]; }      // either rotation of the twisted pair spans the same E = [t]x R (up to sign)
    skew_times(S.t, S.R, S.E);
  }
  __syncthreads();
  // this thread's correspondences: a contiguous chunk, ascending over (rank, tid)
  const int nthr = (int)csize * EFIN_T, g = (int)rank * EFIN_T + tid;
  const int per = (n + nthr - 1) / nthr, b0 = min(g * per, n), e0 = min(b0 + per, n);
  int parity = 0, gn_total = 0;
  // cluster-wide sum of NV doubles whose per-warp partials sit in S.red: every CTA ends up with the same sums in `sum`
  auto cluster_sums = [&](double *sum, int NV) {
    if (tid < NV) { double v = 0; for (int w = 0; w < EFIN_T / 32; ++w) v += S.red[w][tid]; S.part[parity][tid] = v; }
    cluster.sync();                                                  // partials of every CTA are in place (and the previous round's have been read)
    if (tid < NV) {                                                  // one entry per thread, the remote loads in flight together
      double v[EFIN_C];
#pragma unroll
      for (unsigned r = 0; r < EFIN_C; ++r) v[r] = r < csize ? *cluster.map_shared_rank(&S.part[parity][tid], r) : 0.0;
      double t = 0;
#pragma unroll
      for (unsigned r = 0; r < EFIN_C; ++r) t += v[r];               // rank order: identical in every CTA
      S.sumv[tid] = t;
    }
    parity ^= 1;
    __syncthreads();
    for (int q = 0; q < NV; ++q) sum[q] = S.sumv[q];
  };
  // ---- local optimisation ----
  // Per Gauss-Newton iteration: one pass over the points (every thread its chunk, warp-reduced partial sums), the cluster-wide
  // sums, then lanes 0..5 of warp 0 of every CTA solve the 5 x 5 system (redundantly: identical inputs, identical result), apply
  // the step to the estimate they hold in registers and evaluate E there (lane 0) / at its five forward probes (lanes 1..5).
  // That serial stretch is what an iteration costs (one warp, dependent fp64 chains): it is kept short — static-index solve, series
  // for the small rotations, reciprocals instead of divisions.
  EpiPose P;
  for (int q = 0; q < 9; ++q) P.R[q] = S.R[q];
  for (int q = 0; q < 3; ++q) P.t[q] = S.t[q];
  epi_tangent_basis(P);
#pragma unroll 1      // one copy of the loop body: unrolled, the 8 x 3 copies (29k instructions) missed the instruction cache every iteration
  for (int round = 0; round < EPI_LO_ROUNDS; ++round) {
    double Esel[9];
    for (int q = 0; q < 9; ++q) Esel[q] = S.E[q];          // consensus set of this round: fixed during its GN iterations
    if (tid < 6) epi_probe_E(P, tid, S.Ek[tid]);
    if (tid == 0) S.stop = 0;
    __syncthreads();
#pragma unroll 1
    for (int it = 0; it < EPI_GN_ITERS; ++it) {
      ++gn_total;
      double acc[20];
#pragma unroll
      for (int q = 0; q < 20; ++q) acc[q] = 0;
      for (int i = b0; i < e0; ++i) {
        const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
        const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
        if (!(epi::sampson_err(Esel, x1, y1, x2, y2) <= thr2)) continue;
        const double r0 = sampson_signed(S.Ek[0], x1, y1, x2, y2);
        double J[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) J[k] = (sampson_signed(S.Ek[k + 1], x1, y1, x2, y2) - r0) * 1e6;
        int q = 0;
#pragma unroll
        for (int r = 0; r < 5; ++r)
#pragma unroll
          for (int c = r; c < 5; ++c) acc[q++] += J[r] * J[c];
#pragma unroll
        for (int r = 0; r < 5; ++r) acc[15 + r] += J[r] * r0;
      }
#pragma unroll
      for (int q = 0; q < 20; ++q) {
        double v = acc[q];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
        if (lane == 0) S.red[warp][q] = v;
      }
      __syncthreads();
      double sum[20];
      cluster_sums(sum, 20);
      if (warp == 0) {
        double dx[5] = {0, 0, 0, 0, 0}, mx = 0;
        const bool ok = epi_solve5(sum, dx, &mx);
        if (ok && mx < 0.5) epi_apply_step(P, dx);            // a Gauss-Newton step of half a radian is not a refinement: keep the estimate
        // forward-difference Jacobian (1e-6 probes): the Gauss-Newton steps bottom out around 1e-9; 1e-8 rad is four orders
        // below what 0.5 px of keypoint noise leaves in the pose (was 1e-10: never reached, 8 iterations every round)
        const bool stop = !ok || mx < (round + 1 < EPI_LO_ROUNDS ? 1e-6 : 1e-8) || mx >= 0.5;      // the last round polishes; the earlier ones only have to settle the consensus set
        if (lane == 0) S.stop = stop ? 1 : 0;
        if (lane < 6 && !stop) epi_probe_E(P, lane, S.Ek[lane]);
      }
      __syncthreads();
      if (S.stop) break;
    }
    if (tid == 0) skew_times(P.t, P.R, S.E);
    __syncthreads();
  }
  // the local optimisation must not lose support: otherwise the minimal model stands
  {
    int c = 0;
    for (int i = b0; i < e0; ++i) {
      const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
      const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
      c += epi::sampson_err(S.E, x1, y1, x2, y2) <= thr2;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if (lane == 0) S.red[warp][0] = (double)c;
    __syncthreads();
    double tot[1];
    cluster_sums(tot, 1);
    if (tid == 0) {
      const int total = (int)tot[0];
      if (rank == 0) { out_i[4] = total; out_i[5] = gn_total; }
      long long b = -1;
      for (int w = 0; w < EFIN_T / 32; ++w) b = S.k[w] > b ? S.k[w] : b;
      if (!(total >= (int)(b >> 20))) {
        for (int q = 0; q < 9; ++q) S.E[q] = S.E0[q];                  // R1, R2, t of the minimal model are still in place
      } else {
        // decomposeEssentialMat of E = [t]x R without another SVD: the twisted pair is {R, (2 t t^T - I) R} (a half turn about t)
        for (int i = 0; i < 3; ++i)
          for (int j = 0; j < 3; ++j) {
            S.R1[i * 3 + j] = P.R[i * 3 + j];
            S.R2[i * 3 + j] = 2 * P.t[i] * (P.t[0] * P.R[j] + P.t[1] * P.R[3 + j] + P.t[2] * P.R[6 + j]) - P.R[i * 3 + j];
          }
        for (int q = 0; q < 3; ++q) S.t[q] = P.t[q];
      }
    }
    __syncthreads();
  }
  // ---- consensus set of the final model, ascending (the mask of findEssentialMat, epipolar_geometry.cpp:40-47) ----
  double E[9];
  for (int q = 0; q < 9; ++q) E[q] = S.E[q];
  int mine = 0;
  for (int i = b0; i < e0; ++i) {
    const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
    const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
    mine += epi::sampson_err(E, x1, y1, x2, y2) <= thr2;
  }
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
  if (lane == 31) S.cnt[warp] = incl;
  __syncthreads();                                   // also publishes R1, R2, t
  int off = incl - mine, cta_total = 0;
  for (int w = 0; w < EFIN_T / 32; ++w) { if (w < warp) off += S.cnt[w]; cta_total += S.cnt[w]; }
  if (tid == 0) S.ipart[0] = cta_total;
  cluster.sync();
  int n_in = 0;
  for (unsigned r = 0; r < csize; ++r) {
    const int c = *cluster.map_shared_rank(&S.ipart[0], r);
    if (r < rank) off += c;
    n_in += c;
  }
  // the consensus set, ascending; the cheirality vote of recoverPose runs in k_epi_vote_batch (all SMs), the pick in epi::recover_pose_pick
  for (int i = b0; i < e0; ++i) {
    const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
    const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
    if (epi::sampson_err(E, x1, y1, x2, y2) <= thr2) inl[off++] = i;
  }
  if (rank == 0 && tid == 0) {
    const double e22 = S.E[8];
    for (int q = 0; q < 9; ++q) { out_d[q] = S.E[q] / e22; out_d[9 + q] = S.R1[q]; out_d[18 + q] = S.R2[q]; }       // E /= E(2,2) (:37)
    for (int q = 0; q < 3; ++q) out_d[27 + q] = S.t[q];
    out_i[0] = n_in; out_i[1] = S.best;
    out_i[8] = out_i[9] = out_i[10] = out_i[11] = 0;                      // votes, accumulated by k_epi_vote_batch
  }
  cluster.sync();                                    // no CTA leaves while another still reads its shared memory
}

// recoverPose (calib3d five-point.cpp): triangulate every inlier with [I|0] and each of (R1,t) (R2,t) (R1,-t) (R2,-t); a point
// votes for a candidate when its depth is in (0, 50) in both cameras.  One thread per (inlier, candidate); out_i[8 + c] += votes.
__device__ __forceinline__ void epi_vote_run(const float *__restrict__ p1, const float *__restrict__ p2, EpiCam cam, const double *__restrict__ out_d,
                                             int32_t *__restrict__ out_i, const int32_t *__restrict__ inl, int cta) {
  const int n_in = out_i[0];
  const int j = cta * 64 + (threadIdx.x >> 2), c = threadIdx.x & 3;
  bool ok = false;
  if (j < n_in) {
    const int i = inl[j];
    const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
    const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
    const double *R = out_d + ((c & 1) ? 18 : 9);
    const double sg = c < 2 ? 1.0 : -1.0;
    const double P0[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    double P[12];
    for (int r = 0; r < 3; ++r) { P[4 * r] = R[3 * r]; P[4 * r + 1] = R[3 * r + 1]; P[4 * r + 2] = R[3 * r + 2]; P[4 * r + 3] = sg * out_d[27 + r]; }
    double X[4];
    epi::triangulate_dlt(P0, P, x1, y1, x2, y2, X);
    ok = X[2] * X[3] > 0;                            // mask = Q.z * Q.w > 0
    const double z1 = X[2] / X[3];
    ok = ok && z1 < 50.0;                            // distanceThresh
    const double z2 = (P[8] * X[0] + P[9] * X[1] + P[10] * X[2] + P[11] * X[3]) / X[3];
    ok = ok && z2 > 0 && z2 < 50.0;
  }
  const unsigned m = __ballot_sync(0xffffffffu, ok);
  const int lane = threadIdx.x & 31;
  if (lane < 4) {                                    // lanes c, c + 4, ... hold candidate c
    const int votes = __popc(m & (0x11111111u << lane));
    if (votes) atomicAdd(&out_i[8 + lane], votes);
  }
}

// doTriangulation of correspondence i into row j of out
__device__ __forceinline__ void epi_triangulate_one(const float *__restrict__ np1, const float *__restrict__ np2, int i,
                                                    const double *__restrict__ Rt /* 9 + 3 */, float *__restrict__ out, int j) {
  const double P0[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  double P[12];
  for (int r = 0; r < 3; ++r) { P[4 * r] = Rt[3 * r]; P[4 * r + 1] = Rt[3 * r + 1]; P[4 * r + 2] = Rt[3 * r + 2]; P[4 * r + 3] = Rt[9 + r]; }
  double X[4];
  epi::triangulate_dlt(P0, P, np1[2 * i], np1[2 * i + 1], np2[2 * i], np2[2 * i + 1], X);
  // pts4d is CV_32F for float input points; the reference divides by the fourth coordinate in float (:161-168)
  const float x = (float)X[0], y = (float)X[1], z = (float)X[2], w = (float)X[3];
  out[3 * j] = x / w; out[3 * j + 1] = y / w; out[3 * j + 2] = z / w;
}

__global__ void __launch_bounds__(128)
k_triangulate(const float *__restrict__ np1, const float *__restrict__ np2, const int32_t *__restrict__ inl, int n_in,
              const double *__restrict__ Rt /* 9 + 3 */, float *__restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_in) return;
  const int i = inl ? inl[j] : j;                 // no list: every correspondence (mvo_epi_essential_ex)
  epi_triangulate_one(np1, np2, i, Rt, out, j);
}

// ------------------------------------------------------------------------------------ batch of frame pairs
// The essential-matrix kernels for n_pairs matched frame pairs at once (a single-pair call: one pair, cap = n).  Pair p's scratch
// rows: points at p * cap, hypotheses at p * H, finish outputs at p * EPIB_OUT_D / p * EPIB_OUT_I.  pn[p] (written by k_epi_gather,
// or uploaded with the points): the pair's correspondence count, or MVO_ERR_INVALID_ARG; every later kernel skips a pair whose pn
// is below 8.
constexpr int EPIB_OUT_D = 32, EPIB_OUT_I = 16;

// One CTA per pair: checks the frame indices, the match count and every match's keypoint indices before reading through them,
// then writes pts1 / pts2 (pixels) and, for the triangulation, the normalised-plane points of two_view.cpp (pixel2CamNormPlane).
__global__ void __launch_bounds__(256)
k_epi_gather(const mvo_keypoint *__restrict__ kpts, const int32_t *__restrict__ kcounts, int batch, int cap, const int2 *__restrict__ pairs,
             const mvo_dmatch *__restrict__ matches, const int32_t *__restrict__ n_matches, double fx, double fy, double cx, double cy,
             float *__restrict__ p1, float *__restrict__ p2, float *__restrict__ np1, float *__restrict__ np2, int32_t *__restrict__ pn) {
  __shared__ int s_bad;
  const int pair = blockIdx.x;
  const int2 fr = pairs[pair];
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  if (fr.x < 0 || fr.x >= batch || fr.y < 0 || fr.y >= batch) { if (threadIdx.x == 0) pn[pair] = MVO_ERR_INVALID_ARG; return; }
  const int n = n_matches[pair];
  if (n < 0 || n > cap) { if (threadIdx.x == 0) pn[pair] = MVO_ERR_INVALID_ARG; return; }
  const int cq = min(max(kcounts[fr.x], 0), cap), ct = min(max(kcounts[fr.y], 0), cap);
  const mvo_keypoint *kq = kpts + (size_t)fr.x * cap, *kt = kpts + (size_t)fr.y * cap;
  const size_t o = (size_t)pair * cap * 2;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const mvo_dmatch m = matches[(size_t)pair * cap + i];
    if (m.query_idx < 0 || m.query_idx >= cq || m.train_idx < 0 || m.train_idx >= ct) { atomicOr(&s_bad, 1); continue; }
    const float x1 = kq[m.query_idx].x, y1 = kq[m.query_idx].y, x2 = kt[m.train_idx].x, y2 = kt[m.train_idx].y;
    p1[o + 2 * i] = x1; p1[o + 2 * i + 1] = y1; p2[o + 2 * i] = x2; p2[o + 2 * i + 1] = y2;
    if (np1) {
      np1[o + 2 * i] = (float)(((double)x1 - cx) / fx); np1[o + 2 * i + 1] = (float)(((double)y1 - cy) / fy);
      np2[o + 2 * i] = (float)(((double)x2 - cx) / fx); np2[o + 2 * i + 1] = (float)(((double)y2 - cy) / fy);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) pn[pair] = s_bad ? MVO_ERR_INVALID_ARG : n;
}

__global__ void __launch_bounds__(128)
k_epi_hypotheses_batch(const float *__restrict__ p1, const float *__restrict__ p2, const int32_t *__restrict__ pn, int cap, EpiCam cam,
                       uint64_t seed, int H, double *__restrict__ Es, int32_t *__restrict__ valid) {
  const int pair = blockIdx.y, h = blockIdx.x * blockDim.x + threadIdx.x, n = pn[pair];
  if (h >= H || n < 8) return;
  epi_hypothesis(p1 + (size_t)pair * cap * 2, p2 + (size_t)pair * cap * 2, n, cam, seed, h, Es + (size_t)pair * H * 9, valid + (size_t)pair * H);
}

// gridDim.x CTAs per pair (blockIdx.y); each stages only its own pair's points
__global__ void __launch_bounds__(256)
k_epi_score_batch(const float *__restrict__ p1, const float *__restrict__ p2, const int32_t *__restrict__ pn, int cap, EpiCam cam, double thr2,
                  int H, const double *__restrict__ Es, const int32_t *__restrict__ valid, int32_t *__restrict__ counts) {
  const int pair = blockIdx.y, n = pn[pair];
  if (n < 8) return;
  const size_t oh = (size_t)pair * H;
  epi_score_run(p1 + (size_t)pair * cap * 2, p2 + (size_t)pair * cap * 2, n, cam, thr2, H, Es + oh * 9, valid + oh, counts + oh, blockIdx.x, gridDim.x);
}

// one cluster per pair: CTAs [pair * csize, (pair + 1) * csize) along x
__global__ void __launch_bounds__(EFIN_T)
k_epi_finish_batch(const float *__restrict__ p1, const float *__restrict__ p2, const int32_t *__restrict__ pn, int cap, EpiCam cam, double thr2,
                   int H, const double *__restrict__ Es, const int32_t *__restrict__ counts, double *__restrict__ out_d,
                   int32_t *__restrict__ out_i, int32_t *__restrict__ inl) {
  const int pair = blockIdx.x / cooperative_groups::this_cluster().num_blocks(), n = pn[pair];
  if (n < 8) return;                                 // the whole cluster
  const size_t op = (size_t)pair * cap, oh = (size_t)pair * H;
  epi_finish_run(p1 + op * 2, p2 + op * 2, n, cam, thr2, H, Es + oh * 9, counts + oh, out_d + (size_t)pair * EPIB_OUT_D,
                 out_i + (size_t)pair * EPIB_OUT_I, inl + op);
}

__global__ void __launch_bounds__(256)
k_epi_vote_batch(const float *__restrict__ p1, const float *__restrict__ p2, const int32_t *__restrict__ pn, int cap, EpiCam cam,
                 const double *__restrict__ out_d, int32_t *__restrict__ out_i, const int32_t *__restrict__ inl) {
  const int pair = blockIdx.y;
  if (pn[pair] < 8) return;
  const size_t op = (size_t)pair * cap;
  epi_vote_run(p1 + op * 2, p2 + op * 2, cam, out_d + (size_t)pair * EPIB_OUT_D, out_i + (size_t)pair * EPIB_OUT_I, inl + op, blockIdx.x);
}

// recoverPose's pick (epi::recover_pose_pick, which mvo_epi_essential_end runs on the host) of every pair: one thread per pair; a
// failed pair gets its status and nothing else.
__global__ void __launch_bounds__(128)
k_epi_pick(const int32_t *__restrict__ pn, int n_pairs, const double *__restrict__ out_d, const int32_t *__restrict__ out_i,
           mvo_two_view_result *__restrict__ res) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= n_pairs) return;
  const int n = pn[pair];
  mvo_two_view_result &r = res[pair];
  if (n < 0) { r.status = n; return; }
  const int32_t *oi = out_i + (size_t)pair * EPIB_OUT_I;
  if (n < 8 || oi[0] < 8) { r.status = MVO_ERR_DEGENERATE; return; }
  r.votes = epi::recover_pose_pick(out_d + (size_t)pair * EPIB_OUT_D, oi + 8, r.E, r.R, r.t);
  r.status = MVO_OK; r.n_matches = n; r.n_inliers = oi[0];
}

// doTriangulation of every pair's inliers with that pair's (R, t)
__global__ void __launch_bounds__(128)
k_triangulate_batch(const float *__restrict__ np1, const float *__restrict__ np2, const mvo_two_view_result *__restrict__ res, int cap,
                    const int32_t *__restrict__ inl, float *__restrict__ out) {
  const int pair = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  const mvo_two_view_result &r = res[pair];
  if (r.status != MVO_OK || j >= r.n_inliers) return;
  double Rt[12];
  for (int q = 0; q < 9; ++q) Rt[q] = r.R[q];
  for (int q = 0; q < 3; ++q) Rt[9 + q] = r.t[q];
  const size_t op = (size_t)pair * cap;
  epi_triangulate_one(np1 + op * 2, np2 + op * 2, inl[op + j], Rt, out + op * 3, j);
}

// ---------------------------------------------------------------------------------------------------- homography
// estiMotionByHomography (reference src/geometry/epipolar_geometry.cpp:90-128): cv::findHomography(pts1, pts2, RANSAC,
// 3.0, mask) + H /= H(2,2) + inliers from the mask + cv::decomposeHomographyMat(H, K) + t /= |t|.  Same batched design
// as the essential-matrix path: H four-point hypotheses, forward transfer error consensus (the error OpenCV
// thresholds), local optimisation of the best one by Gauss-Newton on the transfer error over its consensus set
// (OpenCV refines its RANSAC result with LM on the same cost).  All three kernels work in isotropically scaled pixel
// coordinates ((u - cx) / f, (v - cy) / f, f = mean focal length): errors scale by 1 / f, the conditioning of the
// 4-point systems and of the normal equations does not depend on the image size.  The decomposition itself is a few
// hundred flops and runs on the host (the same epipolar_math.cuh routine); for a batch of pairs it runs in the combine kernel of
// two_view_batch.cu, compiled without contraction like the host code.
struct HomoCam { double f, cx, cy; };

// hypothesis h: counter-based minimal sample of 4 distinct correspondences, epi::homography_from_4
__device__ __forceinline__ void homo_hypothesis(const float *__restrict__ p1, const float *__restrict__ p2, int n, HomoCam cam, uint64_t seed,
                                                int h, double *__restrict__ Hs, int32_t *__restrict__ valid) {
  int idx[4];
  uint64_t ctr = 0;
  for (int k = 0; k < 4; ++k)
    for (int attempt = 0; attempt < 64; ++attempt) {
      const uint64_t r = splitmix64e(seed ^ splitmix64e(((uint64_t)h << 20) ^ (0x5bd1e995ull + ctr++)));
      const int cand = (int)(r % (uint64_t)n);
      bool dup = false;
      for (int q = 0; q < k; ++q) dup |= idx[q] == cand;
      idx[k] = cand;
      if (!dup) break;
    }
  double a[8], b[8];
  const double inv = 1.0 / cam.f;
  for (int k = 0; k < 4; ++k) {
    a[2 * k] = ((double)p1[2 * idx[k]] - cam.cx) * inv; a[2 * k + 1] = ((double)p1[2 * idx[k] + 1] - cam.cy) * inv;
    b[2 * k] = ((double)p2[2 * idx[k]] - cam.cx) * inv; b[2 * k + 1] = ((double)p2[2 * idx[k] + 1] - cam.cy) * inv;
  }
  double Hm[9];
  const bool ok = epi::homography_from_4(a, b, Hm);
  for (int q = 0; q < 9; ++q) Hs[(size_t)h * 9 + q] = ok ? Hm[q] : 0.0;
  valid[h] = ok ? 1 : 0;
}

// forward transfer error consensus of hypotheses cta * warps + warp, strided by ncta * warps; the CTA stages the n points once
__device__ __forceinline__ void homo_score_run(const float *__restrict__ p1, const float *__restrict__ p2, int n, HomoCam cam, double thr2, int H,
                                               const double *__restrict__ Hs, const int32_t *__restrict__ valid, int32_t *__restrict__ counts,
                                               int cta, int ncta) {
  EPI_DYN_SMEM(double, s_pt);         // [n][4] scaled coordinates x1 y1 x2 y2
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    s_pt[4 * i] = ((double)p1[2 * i] - cam.cx) / cam.f; s_pt[4 * i + 1] = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
    s_pt[4 * i + 2] = ((double)p2[2 * i] - cam.cx) / cam.f; s_pt[4 * i + 3] = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  for (int h = cta * wpb + warp; h < H; h += ncta * wpb) {
    if (valid[h] <= 0) { if (lane == 0) counts[h] = -1; continue; }
    double Hm[9];
    for (int q = 0; q < 9; ++q) Hm[q] = Hs[(size_t)h * 9 + q];
    int c = 0;
    for (int i = lane; i < n; i += 32) c += epi::homography_transfer_err(Hm, s_pt[4 * i], s_pt[4 * i + 1], s_pt[4 * i + 2], s_pt[4 * i + 3]) <= thr2;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if (lane == 0) counts[h] = c;
  }
}

constexpr int HOMO_NV = epi::HOMO_GN_NV;    // 45 entries of J^T J (upper triangle) + 9 of J^T r

// epi::homography_gn_step evaluated by one WARP: lane r holds row r of the augmented 9 x 10 system in registers, the pivot search is a
// warp arg-max (first row among equals, like the serial scan), row swaps and the pivot row travel by shuffles, the back
// substitution broadcasts one unknown per step.  Every entry goes through the operations of the serial function in the same
// order: the results are bit-identical.  (The serial function indexes rows dynamically, i.e. runs out of local memory, on one
// thread.)  All 32 lanes call it; every lane returns the same flag and the same H.
__device__ __forceinline__ bool homography_gn_step_warp(const double *sum, double *H) {
  const int lane = threadIdx.x & 31, r = lane < 9 ? lane : 8;
  double row[10];
#pragma unroll
  for (int c = 0; c < 9; ++c) {
    const int lo = r < c ? r : c, hi = r < c ? c : r;
    row[c] = sum[lo * 9 - (lo * (lo - 1)) / 2 + (hi - lo)];
  }
  double mxd = 0;
#pragma unroll
  for (int q = 0, d = 0; d < 9; q += 9 - d, ++d) mxd = fmax(mxd, sum[q]);          // the diagonal entries
#pragma unroll
  for (int c = 0; c < 9; ++c) if (c == r) row[c] += 1e-9 * mxd + 1e-300;
  row[9] = -sum[45 + r];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    double bv = (lane >= k && lane < 9) ? fabs(row[k]) : -1.0;
    int br = lane;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, bv, d);
      const int orow = __shfl_xor_sync(0xffffffffu, br, d);
      if (ov > bv || (ov == bv && orow < br)) { bv = ov; br = orow; }
    }
    if (!(bv > 0)) return true;
    if (br != k) {                                                     // uniform
      const int src = lane == k ? br : (lane == br ? k : lane);
#pragma unroll
      for (int c = 0; c < 10; ++c) row[c] = __shfl_sync(0xffffffffu, row[c], src);
    }
    double pk[10];
#pragma unroll
    for (int c = k; c < 10; ++c) pk[c] = __shfl_sync(0xffffffffu, row[c], k);
    if (lane > k && lane < 9) {
      const double f = row[k] / pk[k];
#pragma unroll
      for (int c = k; c < 10; ++c) row[c] -= f * pk[c];
    }
  }
  double dx[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) dx[q] = 0;
#pragma unroll
  for (int q = 8; q >= 0; --q) {
    double vq = row[9];
#pragma unroll
    for (int c = q + 1; c < 9; ++c) vq -= row[c] * dx[c];
    vq = vq / row[q];
    dx[q] = __shfl_sync(0xffffffffu, vq, q);
  }
  double mx = 0;
  bool bad = false;
#pragma unroll
  for (int q = 0; q < 9; ++q) { if (!epi::finite_d(dx[q])) bad = true; mx = fmax(mx, fabs(dx[q])); }
  if (bad || mx >= 0.5) return true;
  double nrm = 0;
#pragma unroll
  for (int q = 0; q < 9; ++q) { H[q] += dx[q]; nrm += H[q] * H[q]; }
  nrm = sqrt(nrm);
#pragma unroll
  for (int q = 0; q < 9; ++q) H[q] /= nrm;
  return mx < 1e-11;
}

// out_d: [0..8] H in pixel coordinates scaled so that H[8] = 1; out_i: [0] inliers, [1] best hypothesis,
// [3] consensus of the best minimal model, [4] consensus after the local optimisation, [5] Gauss-Newton iterations run
// One cluster of EFIN_C CTAs like epi_finish_run: every CTA owns a slice of the correspondences, the partial normal equations are
// summed in rank order through distributed shared memory (bit-identical in every CTA), thread 0 of every CTA takes the step.
struct HomoFinSmem {
  long long k[EFIN_T / 32];
  double H[9], H0[9], red[EFIN_T / 32][HOMO_NV], part[2][HOMO_NV], sum[HOMO_NV];
  int cnt[EFIN_T / 32], best, stop, ipart[4];
};

__device__ __forceinline__ void homo_finish_run(const float *__restrict__ p1, const float *__restrict__ p2, int n, HomoCam cam, double thr2, int H,
                                                const double *__restrict__ Hs, const int32_t *__restrict__ counts, double *__restrict__ out_d,
                                                int32_t *__restrict__ out_i, int32_t *__restrict__ inl) {
  EPI_DYN_SMEM(double, smraw);
  HomoFinSmem &S = *reinterpret_cast<HomoFinSmem *>(smraw);
  cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
  const unsigned rank = cluster.block_rank(), csize = cluster.num_blocks();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long best = -1;
  for (int h = tid; h < H; h += EFIN_T) {
    const long long key = ((long long)counts[h] << 20) | (long long)(0xFFFFF - h);
    best = key > best ? key : best;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) { const long long o = __shfl_xor_sync(0xffffffffu, best, d); best = o > best ? o : best; }
  if (lane == 0) S.k[warp] = best;
  __syncthreads();
  if (tid == 0) {
    long long b = -1;
    for (int w = 0; w < EFIN_T / 32; ++w) b = S.k[w] > b ? S.k[w] : b;
    S.best = (int)(b >> 20) >= 4 ? (int)(0xFFFFF - (b & 0xFFFFF)) : -1;
    S.ipart[1] = (int)(b >> 20);
    if (rank == 0) out_i[3] = (int)(b >> 20);
  }
  __syncthreads();
  if (S.best < 0) {                                                  // every CTA takes this branch together
    if (rank == 0 && tid == 0) { out_i[0] = 0; out_i[1] = -1; out_i[4] = 0; }
    return;
  }
  if (tid < 9) { const double v = Hs[(size_t)S.best * 9 + tid]; S.H[tid] = v; S.H0[tid] = v; }
  __syncthreads();
  const int nthr = (int)csize * EFIN_T, g = (int)rank * EFIN_T + tid;
  const int per = (n + nthr - 1) / nthr, b0 = min(g * per, n), e0 = min(b0 + per, n);
  int parity = 0, gn_total = 0;
  // cluster-wide sums of the NV per-warp partials in S.red -> S.sum (the same bits in every CTA)
  auto cluster_sums = [&](int NV) {
    if (tid < NV) { double v = 0; for (int w = 0; w < EFIN_T / 32; ++w) v += S.red[w][tid]; S.part[parity][tid] = v; }
    cluster.sync();
    if (tid < NV) {
      double v = 0;
      for (unsigned r = 0; r < csize; ++r) v += *cluster.map_shared_rank(&S.part[parity][tid], r);
      S.sum[tid] = v;
    }
    parity ^= 1;
    __syncthreads();
  };
  // ---- local optimisation: Gauss-Newton on the transfer error, additive update of the 9 entries (the scale of H is a
  // null direction of the normal equations: a small damping fixes the gauge, H is renormalised after every step) ----
#pragma unroll 1      // one copy of the loop body: unrolled, the 8 x 3 copies (29k instructions) missed the instruction cache every iteration
  for (int round = 0; round < EPI_LO_ROUNDS; ++round) {
    double Hsel[9];
    for (int q = 0; q < 9; ++q) Hsel[q] = S.H[q];
#pragma unroll 1
    for (int it = 0; it < EPI_GN_ITERS; ++it) {
      double Hc[9];
      for (int q = 0; q < 9; ++q) Hc[q] = S.H[q];
      double acc[HOMO_NV];
#pragma unroll
      for (int q = 0; q < HOMO_NV; ++q) acc[q] = 0;
      for (int i = b0; i < e0; ++i) {
        const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
        const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
        if (!(epi::homography_transfer_err(Hsel, x1, y1, x2, y2) <= thr2)) continue;
        epi::homography_gn_accumulate(Hc, x1, y1, x2, y2, acc);
      }
#pragma unroll
      for (int q = 0; q < HOMO_NV; ++q) {
        double vq = acc[q];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) vq += __shfl_xor_sync(0xffffffffu, vq, d);
        if (lane == 0) S.red[warp][q] = vq;
      }
      __syncthreads();
      cluster_sums(HOMO_NV);
      ++gn_total;
      if (warp == 0) {
        double Hn[9];
        for (int q = 0; q < 9; ++q) Hn[q] = S.H[q];
        const bool stop = homography_gn_step_warp(S.sum, Hn);
        __syncwarp();                                         // every lane has read S.H
        if (lane == 0) { S.stop = stop ? 1 : 0; for (int q = 0; q < 9; ++q) S.H[q] = Hn[q]; }
      }
      __syncthreads();
      if (S.stop) break;
    }
  }
  // the local optimisation must not lose support: otherwise the minimal model stands
  {
    int c = 0;
    for (int i = b0; i < e0; ++i) {
      const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
      const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
      c += epi::homography_transfer_err(S.H, x1, y1, x2, y2) <= thr2;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if (lane == 0) S.red[warp][0] = (double)c;
    __syncthreads();
    cluster_sums(1);
    if (tid == 0) {
      const int tot = (int)S.sum[0];
      if (rank == 0) { out_i[4] = tot; out_i[5] = gn_total; }
      if (!(tot >= S.ipart[1])) for (int q = 0; q < 9; ++q) S.H[q] = S.H0[q];
    }
    __syncthreads();
  }
  // ---- consensus set of the final model, ascending (the mask of findHomography, epipolar_geometry.cpp:108-116) ----
  double Hf[9];
  for (int q = 0; q < 9; ++q) Hf[q] = S.H[q];
  int mine = 0;
  for (int i = b0; i < e0; ++i) {
    const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
    const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
    mine += epi::homography_transfer_err(Hf, x1, y1, x2, y2) <= thr2;
  }
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
  if (lane == 31) S.cnt[warp] = incl;
  __syncthreads();
  int off = incl - mine, cta_total = 0;
  for (int w = 0; w < EFIN_T / 32; ++w) { if (w < warp) off += S.cnt[w]; cta_total += S.cnt[w]; }
  if (tid == 0) S.ipart[0] = cta_total;
  cluster.sync();
  int n_in = 0;
  for (unsigned r = 0; r < csize; ++r) {
    const int c = *cluster.map_shared_rank(&S.ipart[0], r);
    if (r < rank) off += c;
    n_in += c;
  }
  for (int i = b0; i < e0; ++i) {
    const double x1 = ((double)p1[2 * i] - cam.cx) / cam.f, y1 = ((double)p1[2 * i + 1] - cam.cy) / cam.f;
    const double x2 = ((double)p2[2 * i] - cam.cx) / cam.f, y2 = ((double)p2[2 * i + 1] - cam.cy) / cam.f;
    if (epi::homography_transfer_err(Hf, x1, y1, x2, y2) <= thr2) inl[off++] = i;
  }
  if (rank == 0 && tid == 0) {
    // back to pixel coordinates: x_scaled = S x_pix with S = [1/f 0 -cx/f; 0 1/f -cy/f; 0 0 1]  =>  H_pix = S^-1 H S
    const double f = cam.f, cx = cam.cx, cy = cam.cy;
    const double Sm[9] = {1 / f, 0, -cx / f, 0, 1 / f, -cy / f, 0, 0, 1}, Si[9] = {f, 0, cx, 0, f, cy, 0, 0, 1};
    double T[9], Hp[9];
    epi::mat3_mul(Hf, Sm, T);
    epi::mat3_mul(Si, T, Hp);
    for (int q = 0; q < 9; ++q) out_d[q] = Hp[q] / Hp[8];                       // H /= H(2,2) (:107)
    out_i[0] = n_in; out_i[1] = S.best;
  }
  cluster.sync();                                    // no CTA leaves while another still reads its shared memory
}

// ------------------------------------------------------------------------- homography for a batch of frame pairs
// The three homography kernels over the pairs of the essential batch (same pn, same point rows; in
// mvo_estimate_relative_poses_batch_dev the hypotheses reuse the essential half's hypothesis rows, which are free once
// k_epi_finish_batch has run), or over the one pair of a single call.  Pair p's finish outputs at p * EPIB_OUT_D / p * EPIB_OUT_I:
// k_homo_hypotheses_batch zeroes them (CTA 0 of each pair), so a pair without any model reads 0 inliers.  A pair is skipped below
// 4 correspondences, the minimal sample (a single call accepts 4 to 7; in a batch such a pair fails in the essential half).
__global__ void __launch_bounds__(128)
k_homo_hypotheses_batch(const float *__restrict__ p1, const float *__restrict__ p2, const int32_t *__restrict__ pn, int cap, HomoCam cam,
                        uint64_t seed, int H, double *__restrict__ Hs, int32_t *__restrict__ valid, double *__restrict__ out_d,
                        int32_t *__restrict__ out_i) {
  const int pair = blockIdx.y, h = blockIdx.x * blockDim.x + threadIdx.x, n = pn[pair];
  if (blockIdx.x == 0 && threadIdx.x < EPIB_OUT_D) {
    out_d[(size_t)pair * EPIB_OUT_D + threadIdx.x] = 0.0;
    if (threadIdx.x < EPIB_OUT_I) out_i[(size_t)pair * EPIB_OUT_I + threadIdx.x] = 0;
  }
  if (h >= H || n < 4) return;
  homo_hypothesis(p1 + (size_t)pair * cap * 2, p2 + (size_t)pair * cap * 2, n, cam, seed, h, Hs + (size_t)pair * H * 9, valid + (size_t)pair * H);
}

// gridDim.x CTAs per pair (blockIdx.y), sized as k_epi_score_batch
__global__ void __launch_bounds__(256)
k_homo_score_batch(const float *__restrict__ p1, const float *__restrict__ p2, const int32_t *__restrict__ pn, int cap, HomoCam cam, double thr2,
                   int H, const double *__restrict__ Hs, const int32_t *__restrict__ valid, int32_t *__restrict__ counts) {
  const int pair = blockIdx.y, n = pn[pair];
  if (n < 4) return;
  const size_t oh = (size_t)pair * H;
  homo_score_run(p1 + (size_t)pair * cap * 2, p2 + (size_t)pair * cap * 2, n, cam, thr2, H, Hs + oh * 9, valid + oh, counts + oh, blockIdx.x, gridDim.x);
}

// one EFIN_C-CTA cluster per pair, as k_epi_finish_batch
__global__ void __launch_bounds__(EFIN_T, 1)
k_homo_finish_batch(const float *__restrict__ p1, const float *__restrict__ p2, const int32_t *__restrict__ pn, int cap, HomoCam cam, double thr2,
                    int H, const double *__restrict__ Hs, const int32_t *__restrict__ counts, double *__restrict__ out_d,
                    int32_t *__restrict__ out_i, int32_t *__restrict__ inl) {
  const int pair = blockIdx.x / cooperative_groups::this_cluster().num_blocks(), n = pn[pair];
  if (n < 4) return;                                 // the whole cluster
  const size_t op = (size_t)pair * cap, oh = (size_t)pair * H;
  homo_finish_run(p1 + op * 2, p2 + op * 2, n, cam, thr2, H, Hs + oh * 9, counts + oh, out_d + (size_t)pair * EPIB_OUT_D,
                  out_i + (size_t)pair * EPIB_OUT_I, inl + op);
}

// doTriangulation of solution s (blockIdx.y) of pair blockIdx.z, with the (R, t) the combine step kept from before basics::invRt
// (mvo_estimate_relative_poses triangulates first and inverts afterwards): rt[(pair * 5 + s) * 12] = R | t, inlier row
// (pair * 5 + s) * cap of the caller's array
__global__ void __launch_bounds__(128)
k_triangulate_solutions_batch(const float *__restrict__ np1, const float *__restrict__ np2, const mvo_relative_poses_result *__restrict__ res,
                              const double *__restrict__ rt, int cap, const int32_t *__restrict__ inl, float *__restrict__ out) {
  const int pair = blockIdx.z, s = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  const mvo_relative_poses_result &r = res[pair];
  if (r.status != MVO_OK || s >= r.sol.num_solutions || j >= r.sol.n_inliers[s]) return;
  double Rt[12];
  for (int q = 0; q < 12; ++q) Rt[q] = rt[((size_t)pair * 5 + s) * 12 + q];
  const size_t op = (size_t)pair * cap, orow = ((size_t)pair * 5 + s) * cap;
  epi_triangulate_one(np1 + op * 2, np2 + op * 2, inl[orow + j], Rt, out + orow * 3, j);
}
