// Host build of csrc/epipolar_math.cuh (the same functions the CUDA kernels call) behind a C interface for ctypes,
// so that the numerics of the two-view stage are checked against numpy / cv2 on the CPU-only test tier.
#include "epipolar_math.cuh"

extern "C" {
int epi_essential_from_8(const double *xy1, const double *xy2, double *E) { return epi::essential_from_8(xy1, xy2, E) ? 1 : 0; }
double epi_sampson(const double *E, double x1, double y1, double x2, double y2) { return epi::sampson_err(E, x1, y1, x2, y2); }
void epi_decompose(const double *E, double *R1, double *R2, double *t) { epi::decompose_essential(E, R1, R2, t); }
void epi_triangulate(const double *P1, const double *P2, double x1, double y1, double x2, double y2, double *X) {
  epi::triangulate_dlt(P1, P2, x1, y1, x2, y2, X);
}
void epi_svd3(const double *M, double *U, double *s, double *V) { epi::svd3(M, U, s, V); }
int epi_homography_from_4(const double *xy1, const double *xy2, double *H) { return epi::homography_from_4(xy1, xy2, H) ? 1 : 0; }
double epi_transfer_err(const double *H, double x1, double y1, double x2, double y2) { return epi::homography_transfer_err(H, x1, y1, x2, y2); }
int epi_decompose_homography(const double *H, double *Rs, double *ts, double *ns) { return epi::decompose_homography(H, Rs, ts, ns); }
int epi_filter_homography(const double *Rs, const double *ns, int n_sol, const float *np1, const float *np2, const int *inl, int n_in, int *keep) {
  return epi::filter_homography_solutions(Rs, ns, n_sol, np1, np2, inl, n_in, keep);
}
// the local optimisation of k_homo_finish_batch, serially: `rounds` times re-select the consensus set of the current H (scaled
// coordinates, squared threshold thr2), then up to `iters` Gauss-Newton steps on it (csrc/epipolar_kernels.cuh, homo_finish_run)
int epi_homography_lo(const double *xy1, const double *xy2, int n, double thr2, int rounds, int iters, double *H) {
  int steps = 0;
  for (int round = 0; round < rounds; ++round) {
    double Hsel[9];
    for (int q = 0; q < 9; ++q) Hsel[q] = H[q];
    for (int it = 0; it < iters; ++it) {
      double acc[epi::HOMO_GN_NV];
      for (int q = 0; q < epi::HOMO_GN_NV; ++q) acc[q] = 0;
      for (int i = 0; i < n; ++i) {
        if (!(epi::homography_transfer_err(Hsel, xy1[2 * i], xy1[2 * i + 1], xy2[2 * i], xy2[2 * i + 1]) <= thr2)) continue;
        epi::homography_gn_accumulate(H, xy1[2 * i], xy1[2 * i + 1], xy2[2 * i], xy2[2 * i + 1], acc);
      }
      ++steps;
      if (epi::homography_gn_step(acc, H)) break;
    }
  }
  return steps;
}
int epi_null_8x9(const double *M, double *x) { double T[72]; for (int i = 0; i < 72; ++i) T[i] = M[i]; return epi::null_vector_8x9(T, x) ? 1 : 0; }
}
