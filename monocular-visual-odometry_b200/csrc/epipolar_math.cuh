// Small dense numerics of the two-view stage (SURVEY.md §8f-1), written once for host and device: the CUDA kernels in
// epipolar.cu call these from one thread per hypothesis / per point, and tests/cpp/epipolar_math_host.cpp compiles the
// very same functions with g++ so that they are checked against numpy / cv2 on the CPU-only test tier.
//   sym_eigen_jacobi<N>      cyclic Jacobi eigen-decomposition of a symmetric NxN matrix (N = 3, 4)
//   null_vector_8x9          the 1-dimensional null space of an 8x9 system by Gaussian elimination with complete pivoting
//   svd3                     3x3 SVD from the eigen-decomposition of M^T M
//   essential_from_8         eight-point essential matrix on calibrated coordinates, projected onto the essential manifold
//   sampson_err              the squared Sampson distance OpenCV's findEssentialMat scores with (five-point.cpp)
//   decompose_essential      R1, R2, t of cv::decomposeEssentialMat
//   triangulate_dlt          one point of cv::triangulatePoints (the 4x4 homogeneous DLT, triangulate.cpp)
//   recover_pose_pick        recoverPose's choice among the four (R, t) of an essential matrix, t /= |t|
//   homography_motions       cv::decomposeHomographyMat(H, K), t /= |t|
// fp64 throughout, no dynamic memory, fixed loop bounds.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define EPI_HD __host__ __device__ __forceinline__
// the three routines with nested loops over local arrays are real calls on the device: inlining them into each other
// (essential_from_8 -> null_vector_8x9 / svd3 -> sym_eigen_jacobi) bloats every caller and, with nvcc 12.9, once
// produced wrong singular values inside essential_from_8 although each routine is correct on its own
// (tests/test_epipolar_gpu.py::test_device_math_equals_host_build).  `inline` for the linkage only: more than one translation
// unit includes this header (epipolar.cu, two_view_batch.cu)
#define EPI_HD_CALL __host__ __device__ __noinline__ inline
#else
#define EPI_HD inline
#define EPI_HD_CALL inline
#endif

namespace epi {

// A (symmetric, row-major, destroyed) -> eigenvalues w[N] (unsorted) and eigenvectors as COLUMNS of V
template <int N>
EPI_HD_CALL void sym_eigen_jacobi(double *A, double *w, double *V) {
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) V[i * N + j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 12; ++sweep) {
    double off = 0;
    for (int i = 0; i < N; ++i)
      for (int j = i + 1; j < N; ++j) off += A[i * N + j] * A[i * N + j];
    double diag = 0;
    for (int i = 0; i < N; ++i) diag += A[i * N + i] * A[i * N + i];
    if (off <= 1e-32 * diag || off == 0) break;
    for (int p = 0; p < N; ++p)
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p * N + q];
        if (apq == 0) continue;
        const double theta = (A[q * N + q] - A[p * N + p]) / (2 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1));
        const double c = 1 / sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < N; ++k) {               // columns p, q of A
          const double akp = A[k * N + p], akq = A[k * N + q];
          A[k * N + p] = c * akp - s * akq;
          A[k * N + q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {               // rows p, q of A
          const double apk = A[p * N + k], aqk = A[q * N + k];
          A[p * N + k] = c * apk - s * aqk;
          A[q * N + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < N; ++k) {
          const double vkp = V[k * N + p], vkq = V[k * N + q];
          V[k * N + p] = c * vkp - s * vkq;
          V[k * N + q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < N; ++i) w[i] = A[i * N + i];
}

// Null vector x (unit norm) of the 8x9 system M x = 0 (M row-major, destroyed).  Returns false when the system is
// rank deficient beyond one dimension (degenerate sample).
EPI_HD_CALL bool null_vector_8x9(double *M, double *x) {
  int perm[9];
  for (int j = 0; j < 9; ++j) perm[j] = j;
  for (int k = 0; k < 8; ++k) {
    int pr = k, pc = k;                              // complete pivoting
    double best = 0;
    for (int i = k; i < 8; ++i)
      for (int j = k; j < 9; ++j) {
        const double a = fabs(M[i * 9 + j]);
        if (a > best) { best = a; pr = i; pc = j; }
      }
    if (!(best > 1e-12)) return false;
    if (pr != k) for (int j = 0; j < 9; ++j) { const double t = M[k * 9 + j]; M[k * 9 + j] = M[pr * 9 + j]; M[pr * 9 + j] = t; }
    if (pc != k) {
      for (int i = 0; i < 8; ++i) { const double t = M[i * 9 + k]; M[i * 9 + k] = M[i * 9 + pc]; M[i * 9 + pc] = t; }
      const int t = perm[k]; perm[k] = perm[pc]; perm[pc] = t;
    }
    const double inv = 1.0 / M[k * 9 + k];
    for (int i = k + 1; i < 8; ++i) {
      const double f = M[i * 9 + k] * inv;
      if (f == 0) continue;
      for (int j = k; j < 9; ++j) M[i * 9 + j] -= f * M[k * 9 + j];
    }
  }
  double y[9];
  y[8] = 1.0;                                        // the free variable
  for (int k = 7; k >= 0; --k) {
    double s = 0;
    for (int j = k + 1; j < 9; ++j) s += M[k * 9 + j] * y[j];
    y[k] = -s / M[k * 9 + k];
  }
  double nrm = 0;
  for (int j = 0; j < 9; ++j) nrm += y[j] * y[j];
  nrm = sqrt(nrm);
  if (!(nrm > 0) || !(nrm - nrm == 0.0)) return false;
  for (int j = 0; j < 9; ++j) x[perm[j]] = y[j] / nrm;
  return true;
}

EPI_HD void cross3(const double *a, const double *b, double *c) {
  c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
EPI_HD double det3(const double *M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// M = U diag(s) V^T, s sorted descending, U and V orthogonal (columns), row-major 3x3.
EPI_HD_CALL void svd3(const double *M, double *U, double *s, double *V) {
  double A[9], w[3], Q[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i * 3 + j] = M[0 * 3 + i] * M[0 * 3 + j] + M[1 * 3 + i] * M[1 * 3 + j] + M[2 * 3 + i] * M[2 * 3 + j];
  sym_eigen_jacobi<3>(A, w, Q);
  int o[3] = {0, 1, 2};                               // order by eigenvalue, descending
  for (int a = 0; a < 3; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (w[o[b]] > w[o[a]]) { const int t = o[a]; o[a] = o[b]; o[b] = t; }
  for (int k = 0; k < 3; ++k) {
    s[k] = sqrt(w[o[k]] > 0 ? w[o[k]] : 0.0);
    for (int i = 0; i < 3; ++i) V[i * 3 + k] = Q[i * 3 + o[k]];
  }
  // U columns: M v_k / s_k for the two leading directions, the third completes a right-handed frame
  double u[3][3];
  for (int k = 0; k < 2; ++k) {
    double n = 0;
    for (int i = 0; i < 3; ++i) { u[k][i] = M[i * 3] * V[0 * 3 + k] + M[i * 3 + 1] * V[1 * 3 + k] + M[i * 3 + 2] * V[2 * 3 + k]; n += u[k][i] * u[k][i]; }
    n = sqrt(n);
    if (n > 0) for (int i = 0; i < 3; ++i) u[k][i] /= n;
  }
  {                                                   // re-orthogonalise u1 against u0 (nearly equal singular values)
    const double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
    double n = 0;
    for (int i = 0; i < 3; ++i) { u[1][i] -= d * u[0][i]; n += u[1][i] * u[1][i]; }
    n = sqrt(n);
    if (n > 0) for (int i = 0; i < 3; ++i) u[1][i] /= n;
  }
  cross3(u[0], u[1], u[2]);
  for (int k = 0; k < 3; ++k)
    for (int i = 0; i < 3; ++i) U[i * 3 + k] = u[k][i];
  // keep M = U S V^T for the third direction: flip v2 if needed (s2 >= 0 by construction, the sign lives in V)
  double mv[3];
  for (int i = 0; i < 3; ++i) mv[i] = M[i * 3] * V[0 * 3 + 2] + M[i * 3 + 1] * V[1 * 3 + 2] + M[i * 3 + 2] * V[2 * 3 + 2];
  if (mv[0] * u[2][0] + mv[1] * u[2][1] + mv[2] * u[2][2] < 0)
    for (int i = 0; i < 3; ++i) V[i * 3 + 2] = -V[i * 3 + 2];
}

// Essential matrix from 8 correspondences in calibrated coordinates (x1 -> x2, x2^T E x1 = 0), projected onto the
// essential manifold (singular values 1, 1, 0).  xy1 / xy2: 8 x 2.  Returns false for degenerate samples.
EPI_HD bool finite_d(double v) { return v - v == 0.0; }      // false for NaN and +-inf, no library call

// reason (optional): 0 ok, 1 singular sample, 2 rank-one null vector, 3 non-finite result
EPI_HD_CALL bool essential_from_8(const double *xy1, const double *xy2, double *E, int *reason = nullptr) {
  if (reason) *reason = 0;
  double M[72];
  for (int k = 0; k < 8; ++k) {
    const double x1 = xy1[2 * k], y1 = xy1[2 * k + 1], x2 = xy2[2 * k], y2 = xy2[2 * k + 1];
    double *r = M + 9 * k;
    r[0] = x2 * x1; r[1] = x2 * y1; r[2] = x2; r[3] = y2 * x1; r[4] = y2 * y1; r[5] = y2; r[6] = x1; r[7] = y1; r[8] = 1.0;
  }
  double f[9];
  if (!null_vector_8x9(M, f)) { if (reason) *reason = 1; return false; }
  double U[9], s[3], V[9];
  svd3(f, U, s, V);
  if (!(s[1] > 1e-9 * s[0])) { if (reason) *reason = 2; return false; }            // rank one: not an essential matrix
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) E[i * 3 + j] = U[i * 3] * V[j * 3] + U[i * 3 + 1] * V[j * 3 + 1];      // U diag(1,1,0) V^T
  for (int i = 0; i < 9; ++i)
    if (!finite_d(E[i])) { if (reason) *reason = 3; return false; }
  return true;
}

// Squared Sampson distance of (x1, y1) <-> (x2, y2) under E (calibrated coordinates)
EPI_HD double sampson_err(const double *E, double x1, double y1, double x2, double y2) {
  const double Ex0 = E[0] * x1 + E[1] * y1 + E[2], Ex1 = E[3] * x1 + E[4] * y1 + E[5], Ex2 = E[6] * x1 + E[7] * y1 + E[8];
  const double Et0 = E[0] * x2 + E[3] * y2 + E[6], Et1 = E[1] * x2 + E[4] * y2 + E[7];
  const double x2tEx1 = x2 * Ex0 + y2 * Ex1 + Ex2;
  return x2tEx1 * x2tEx1 / (Ex0 * Ex0 + Ex1 * Ex1 + Et0 * Et0 + Et1 * Et1);
}

// cv::decomposeEssentialMat: E = U diag(1,1,0) V^T, det(U), det(V) forced positive, W = [0 1 0; -1 0 0; 0 0 1],
// R1 = U W V^T, R2 = U W^T V^T, t = U[:, 2]
EPI_HD_CALL void decompose_essential(const double *E, double *R1, double *R2, double *t) {
  double U[9], s[3], V[9];
  svd3(E, U, s, V);
  if (det3(U) < 0) for (int i = 0; i < 9; ++i) U[i] = -U[i];
  if (det3(V) < 0) for (int i = 0; i < 9; ++i) V[i] = -V[i];
  // U W = [-u1, u0, u2] (columns), U W^T = [u1, -u0, u2]
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double a = -U[i * 3 + 1] * V[j * 3 + 0] + U[i * 3 + 0] * V[j * 3 + 1] + U[i * 3 + 2] * V[j * 3 + 2];
      const double b = U[i * 3 + 1] * V[j * 3 + 0] - U[i * 3 + 0] * V[j * 3 + 1] + U[i * 3 + 2] * V[j * 3 + 2];
      R1[i * 3 + j] = a;
      R2[i * 3 + j] = b;
    }
  for (int i = 0; i < 3; ++i) t[i] = U[i * 3 + 2];
}

// One point of cv::triangulatePoints: P1, P2 3x4 row-major, (x1, y1), (x2, y2) in the units of the projection
// matrices; X = right singular vector of the 4x4 DLT system for its smallest singular value (homogeneous, unit norm).
EPI_HD_CALL void triangulate_dlt(const double *P1, const double *P2, double x1, double y1, double x2, double y2, double *X) {
  double A[16];
  for (int j = 0; j < 4; ++j) {
    A[0 * 4 + j] = x1 * P1[2 * 4 + j] - P1[0 * 4 + j];
    A[1 * 4 + j] = y1 * P1[2 * 4 + j] - P1[1 * 4 + j];
    A[2 * 4 + j] = x2 * P2[2 * 4 + j] - P2[0 * 4 + j];
    A[3 * 4 + j] = y2 * P2[2 * 4 + j] - P2[1 * 4 + j];
  }
  double AtA[16], w[4], V[16];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) AtA[i * 4 + j] = A[0 * 4 + i] * A[0 * 4 + j] + A[1 * 4 + i] * A[1 * 4 + j] + A[2 * 4 + i] * A[2 * 4 + j] + A[3 * 4 + i] * A[3 * 4 + j];
  sym_eigen_jacobi<4>(AtA, w, V);
  int m = 0;
  for (int k = 1; k < 4; ++k) if (w[k] < w[m]) m = k;
  for (int i = 0; i < 4; ++i) X[i] = V[i * 4 + m];
}

// ---- homography (estiMotionByHomography, reference src/geometry/epipolar_geometry.cpp:90-128) ----------------------

// H (x2 ~ H x1, row-major 3x3, unit Frobenius norm) from 4 correspondences; any coordinate units.  False for
// degenerate samples (three collinear points make the 8x9 system rank deficient).
EPI_HD_CALL bool homography_from_4(const double *xy1, const double *xy2, double *H) {
  double M[72];
  for (int k = 0; k < 4; ++k) {
    const double x1 = xy1[2 * k], y1 = xy1[2 * k + 1], x2 = xy2[2 * k], y2 = xy2[2 * k + 1];
    double *r = M + 18 * k;
    r[0] = -x1; r[1] = -y1; r[2] = -1; r[3] = 0; r[4] = 0; r[5] = 0; r[6] = x2 * x1; r[7] = x2 * y1; r[8] = x2;
    r[9] = 0; r[10] = 0; r[11] = 0; r[12] = -x1; r[13] = -y1; r[14] = -1; r[15] = y2 * x1; r[16] = y2 * y1; r[17] = y2;
  }
  if (!null_vector_8x9(M, H)) return false;
  for (int i = 0; i < 9; ++i)
    if (!finite_d(H[i])) return false;
  return true;
}

// squared forward transfer error |x2 - H x1|^2 (the error cv::findHomography's RANSAC thresholds), +inf at w = 0
EPI_HD double homography_transfer_err(const double *H, double x1, double y1, double x2, double y2) {
  const double w = H[6] * x1 + H[7] * y1 + H[8];
  if (!(fabs(w) > 1e-300)) return 1e300;
  const double du = (H[0] * x1 + H[1] * y1 + H[2]) / w - x2, dv = (H[3] * x1 + H[4] * y1 + H[5]) / w - y2;
  return du * du + dv * dv;
}

// ---- Gauss-Newton on the forward transfer error, additive update of the 9 entries of H (unit Frobenius norm) ----
// One correspondence's contribution to the normal equations: acc[0..44] += upper triangle of J^T J (row-major),
// acc[45..53] += J^T r, with r = (u - x2, v - y2), (u, v) = H x1 dehomogenised.  Points at w ~ 0 contribute nothing.
constexpr int HOMO_GN_NV = 54;
EPI_HD void homography_gn_accumulate(const double *Hc, double x1, double y1, double x2, double y2, double *acc) {
  const double w = Hc[6] * x1 + Hc[7] * y1 + Hc[8];
  if (!(fabs(w) > 1e-12)) return;
  const double iw = 1.0 / w, u = (Hc[0] * x1 + Hc[1] * y1 + Hc[2]) * iw, v = (Hc[3] * x1 + Hc[4] * y1 + Hc[5]) * iw;
  const double ru = u - x2, rv = v - y2;
  const double Ju[9] = {x1 * iw, y1 * iw, iw, 0, 0, 0, -u * x1 * iw, -u * y1 * iw, -u * iw};
  const double Jv[9] = {0, 0, 0, x1 * iw, y1 * iw, iw, -v * x1 * iw, -v * y1 * iw, -v * iw};
  int q = 0;
  for (int r = 0; r < 9; ++r)
    for (int c = r; c < 9; ++c) acc[q++] += Ju[r] * Ju[c] + Jv[r] * Jv[c];
  for (int r = 0; r < 9; ++r) acc[45 + r] += Ju[r] * ru + Jv[r] * rv;
}

// Solve the accumulated normal equations and apply the step to H (renormalised to unit Frobenius norm).  The scale of H
// is a null direction of J^T J: a small damping of the diagonal fixes the gauge.  Returns true when the iteration
// should STOP: singular / non-finite system, a step below 1e-11 (converged) or above 0.5 (half the norm of H is not a
// refinement; H is left untouched in that case).
EPI_HD_CALL bool homography_gn_step(const double *sum, double *H) {
  double A[9][10];
  int q = 0;
  for (int r = 0; r < 9; ++r)
    for (int c = r; c < 9; ++c) { A[r][c] = sum[q]; A[c][r] = sum[q]; ++q; }
  double mxd = 0;
  for (int r = 0; r < 9; ++r) mxd = fmax(mxd, A[r][r]);
  for (int r = 0; r < 9; ++r) { A[r][r] += 1e-9 * mxd + 1e-300; A[r][9] = -sum[45 + r]; }
  for (int k = 0; k < 9; ++k) {                                  // Gaussian elimination with partial pivoting
    int pr = k;
    for (int r = k + 1; r < 9; ++r) if (fabs(A[r][k]) > fabs(A[pr][k])) pr = r;
    if (!(fabs(A[pr][k]) > 0)) return true;
    if (pr != k) for (int c = 0; c < 10; ++c) { const double t_ = A[k][c]; A[k][c] = A[pr][c]; A[pr][c] = t_; }
    for (int r = k + 1; r < 9; ++r) { const double f = A[r][k] / A[k][k]; for (int c = k; c < 10; ++c) A[r][c] -= f * A[k][c]; }
  }
  double dx[9], mx = 0;
  for (int r = 0; r < 9; ++r) dx[r] = 0;
  for (int r = 8; r >= 0; --r) { double vq = A[r][9]; for (int c = r + 1; c < 9; ++c) vq -= A[r][c] * dx[c]; dx[r] = vq / A[r][r]; }
  for (int r = 0; r < 9; ++r) { if (!finite_d(dx[r])) return true; mx = fmax(mx, fabs(dx[r])); }
  if (mx >= 0.5) return true;
  double nrm = 0;
  for (int r = 0; r < 9; ++r) { H[r] += dx[r]; nrm += H[r] * H[r]; }
  nrm = sqrt(nrm);
  for (int r = 0; r < 9; ++r) H[r] /= nrm;
  return mx < 1e-11;
}

EPI_HD void mat3_mul(const double *A, const double *B, double *C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}

// cv::decomposeHomographyMat on a calibrated homography Hn = K^-1 H K (any scale, any sign): Hn ~ R + t n^T with t in
// units of the plane distance.  Up to 4 solutions, in pairs (R, t, n), (R, -t, -n); one solution (R = Hn, t = n = 0)
// for a pure rotation.  Method: Ma, Soatto, Kosecka, Sastry, "An Invitation to 3-D Vision", section 5.3.3 (the
// eigenvectors of Hn^T Hn); OpenCV's analytical method (Malis & Vargas) yields the same solution set.
// Rs: 4 x 9, ts: 4 x 3, ns: 4 x 3.  Returns the number of solutions (0 for a singular input).
EPI_HD_CALL int decompose_homography(const double *Hin, double *Rs, double *ts, double *ns) {
  double H[9], U[9], sv[3], V[9];
  svd3(Hin, U, sv, V);
  if (!(sv[1] > 0) || !finite_d(sv[1])) return 0;
  const double sgn = det3(Hin) < 0 ? -1.0 : 1.0;                // the camera stays on one side of the plane: det(R + t n^T) > 0
  for (int i = 0; i < 9; ++i) H[i] = sgn * Hin[i] / sv[1];     // middle singular value -> 1
  const double s1 = sv[0] / sv[1], s3 = sv[2] / sv[1];
  const double a2 = 1 - s3 * s3, b2 = s1 * s1 - 1;             // both >= 0
  if (a2 + b2 < 1e-12) {                                         // H^T H = I: pure rotation
    for (int i = 0; i < 9; ++i) Rs[i] = H[i];
    for (int i = 0; i < 3; ++i) { ts[i] = 0; ns[i] = 0; }
    return 1;
  }
  double v1[3], v2[3], v3[3];
  for (int i = 0; i < 3; ++i) { v1[i] = V[i * 3]; v2[i] = V[i * 3 + 1]; v3[i] = V[i * 3 + 2]; }
  if (det3(V) < 0) for (int i = 0; i < 3; ++i) v3[i] = -v3[i];
  const double a = sqrt(a2 > 0 ? a2 : 0.0), b = sqrt(b2 > 0 ? b2 : 0.0), c = 1.0 / sqrt(a2 + b2);
  for (int k = 0; k < 2; ++k) {
    const double sg = k == 0 ? 1.0 : -1.0;
    double u[3], Nn[3], Hv2[3], Hu[3], HN[3], Um[9], Wm[9], R[9];
    for (int i = 0; i < 3; ++i) u[i] = (a * v1[i] + sg * b * v3[i]) * c;
    cross3(v2, u, Nn);
    for (int i = 0; i < 3; ++i) {
      Hv2[i] = H[i * 3] * v2[0] + H[i * 3 + 1] * v2[1] + H[i * 3 + 2] * v2[2];
      Hu[i] = H[i * 3] * u[0] + H[i * 3 + 1] * u[1] + H[i * 3 + 2] * u[2];
    }
    cross3(Hv2, Hu, HN);
    for (int i = 0; i < 3; ++i) {                               // U = [v2, u, v2 x u], W = [H v2, H u, H v2 x H u] (columns)
      Um[i * 3] = v2[i]; Um[i * 3 + 1] = u[i]; Um[i * 3 + 2] = Nn[i];
      Wm[i * 3] = Hv2[i]; Wm[i * 3 + 1] = Hu[i]; Wm[i * 3 + 2] = HN[i];
    }
    for (int i = 0; i < 3; ++i)                                  // R = W U^T
      for (int j = 0; j < 3; ++j) R[i * 3 + j] = Wm[i * 3] * Um[j * 3] + Wm[i * 3 + 1] * Um[j * 3 + 1] + Wm[i * 3 + 2] * Um[j * 3 + 2];
    double T[3];
    for (int i = 0; i < 3; ++i)
      T[i] = (H[i * 3] - R[i * 3]) * Nn[0] + (H[i * 3 + 1] - R[i * 3 + 1]) * Nn[1] + (H[i * 3 + 2] - R[i * 3 + 2]) * Nn[2];
    for (int pm = 0; pm < 2; ++pm) {
      const int o = 2 * k + pm;
      const double f = pm == 0 ? 1.0 : -1.0;
      for (int i = 0; i < 9; ++i) Rs[o * 9 + i] = R[i];
      for (int i = 0; i < 3; ++i) { ts[o * 3 + i] = f * T[i]; ns[o * 3 + i] = f * Nn[i]; }
    }
  }
  return 4;
}

// cv::decomposeHomographyMat(H, K) and t /= |t| (epipolar_geometry.cpp:119-126): Hn = K^-1 H K with K^-1 written out, then every
// solution's t scaled to unit length; a pure rotation keeps t = 0 (the reference divides by zero there).  Returns the number of
// solutions.  Both callers compile it without contraction (the host's g++ for x86-64, two_view_batch.cu with --fmad=false), so they
// get the same bits.
EPI_HD int homography_motions(const double *H, const double *K, double *Rs, double *ts, double *ns) {
  const double fx = K[0], fy = K[4], cx = K[2], cy = K[5];
  const double Km[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1}, Ki[9] = {1 / fx, 0, -cx / fx, 0, 1 / fy, -cy / fy, 0, 0, 1};
  double T[9], Hn[9];
  mat3_mul(H, Km, T);
  mat3_mul(Ki, T, Hn);
  const int n_sol = decompose_homography(Hn, Rs, ts, ns);
  for (int s = 0; s < n_sol; ++s) {
    double *t = ts + 3 * s;
    const double nt = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    if (nt > 0) for (int q = 0; q < 3; ++q) t[q] /= nt;
  }
  return n_sol;
}

// recoverPose's choice among (R1,t) (R2,t) (R1,-t) (R2,-t) of an essential-matrix finish output block od (E at 0, R1 at 9, R2 at 18,
// t at 27) with the four vote counts g: the first candidate whose count is a maximum (OpenCV's tie order), then t /= |t|
// (epipolar_geometry.cpp:54-55).  Writes E, R, t and returns the pick's vote count.  |t| rounds each product and sum on its own on
// both sides, so the device returns the host's bits; only its spelling differs.
EPI_HD int recover_pose_pick(const double *od, const int32_t *g, double *E, double *R, double *t) {
  int pick = 3;
  if (g[0] >= g[1] && g[0] >= g[2] && g[0] >= g[3]) pick = 0;
  else if (g[1] >= g[0] && g[1] >= g[2] && g[1] >= g[3]) pick = 1;
  else if (g[2] >= g[0] && g[2] >= g[1] && g[2] >= g[3]) pick = 2;
  const double *tt = od + 27, *Rp = od + ((pick & 1) ? 18 : 9), sg = pick < 2 ? 1.0 : -1.0;
#ifdef __CUDA_ARCH__
  const double nt = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(tt[0], tt[0]), __dmul_rn(tt[1], tt[1])), __dmul_rn(tt[2], tt[2])));
#else
  const double nt = sqrt(tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2]);
#endif
  for (int q = 0; q < 9; ++q) { E[q] = od[q]; R[q] = Rp[q]; }
  for (int q = 0; q < 3; ++q) t[q] = sg * tt[q] / nt;
  return g[pick];
}

// cv::filterHomographyDecompByVisibleRefpoints (removeWrongRtOfHomography, epipolar_geometry.cpp:59-88): a solution
// survives when every reference point lies in front of the plane normal in both views.
// np1 / np2: n x 2 points on the normalised image planes; keep[s] = 1 for the surviving solutions.  Host and device.
EPI_HD int filter_homography_solutions(const double *Rs, const double *ns, int n_sol, const float *np1, const float *np2,
                                       const int *inliers, int n_in, int *keep) {
  int kept = 0;
  for (int s = 0; s < n_sol; ++s) {
    const double *R = Rs + 9 * s, *nv = ns + 3 * s;
    const double m0 = R[0] * nv[0] + R[1] * nv[1] + R[2] * nv[2], m1 = R[3] * nv[0] + R[4] * nv[1] + R[5] * nv[2],
                 m2 = R[6] * nv[0] + R[7] * nv[1] + R[8] * nv[2];
    bool ok = true;
    for (int j = 0; j < n_in && ok; ++j) {
      const int i = inliers ? inliers[j] : j;
      const double d1 = nv[0] * np1[2 * i] + nv[1] * np1[2 * i + 1] + nv[2];
      const double d2 = m0 * np2[2 * i] + m1 * np2[2 * i + 1] + m2;
      ok = d1 > 0 && d2 > 0;
    }
    keep[s] = ok ? 1 : 0;
    kept += ok;
  }
  return kept;
}

}  // namespace epi
