// TEST INFRASTRUCTURE (CPU tier): the two-view kernels (csrc/epipolar_kernels.cuh — essential matrix, triangulation,
// homography) built for the host with tests/cpp/cuda_emu.h and launched the way csrc/epipolar.cu launches them
// (mvo_esti_motion_by_essential, mvo_esti_motion_by_homography, mvo_do_triangulation: the batch kernels with one pair and
// cap = n, same thresholds, recoverPose's pick by the same epi::recover_pose_pick).  The essential-matrix kernels have run on hardware; the homography kernels have not — this is their
// first execution of any kind.
#include "cuda_emu.h"

#include "epipolar_math.cuh"
#include "mvo.h"
namespace {
#define EPI_DYN_SMEM(type, name) type *name = (type *)g_dyn_smem
#define EPI_NOINLINE
#include "epipolar_kernels.cuh"
}  // namespace

extern "C" {

// out_i: [0] inliers [1] best hypothesis [2] votes [3] consensus of the best minimal model [4] after the local optimisation
int emu_essential(const float *p1, const float *p2, int n, const double *K, double threshold, int H, uint64_t seed, double *E, double *R,
                  double *t, int32_t *inliers, int32_t *out_i) {
  EpiCam cam;
  cam.f = (K[0] + K[4]) / 2; cam.cx = K[2]; cam.cy = K[5];
  const double thr2 = (threshold / cam.f) * (threshold / cam.f);
  std::vector<double> Es((size_t)H * 9), out(64, 0.0);
  std::vector<int32_t> valid((size_t)H), counts((size_t)H), oi(64, 0);
  const int32_t pn[1] = {n};
  run_grid((unsigned)((H + 127) / 128), 1, 1, 128, 0, [&] { k_epi_hypotheses_batch(p1, p2, pn, n, cam, seed, H, Es.data(), valid.data()); });
  const int grid = std::min((H + 7) / 8, 64);                    // any grid covers all hypotheses (grid-stride loop)
  run_grid((unsigned)grid, 1, 1, 256, (size_t)n * 32, [&] { k_epi_score_batch(p1, p2, pn, n, cam, thr2, H, Es.data(), valid.data(), counts.data()); });
  run_clusters(EFIN_C, EFIN_C, EFIN_T, sizeof(EpiFinSmem),
               [&] { k_epi_finish_batch(p1, p2, pn, n, cam, thr2, H, Es.data(), counts.data(), out.data(), oi.data(), inliers); });
  run_grid((unsigned)((n + 63) / 64), 1, 1, 256, 0, [&] { k_epi_vote_batch(p1, p2, pn, n, cam, out.data(), oi.data(), inliers); });
  oi[2] = epi::recover_pose_pick(out.data(), oi.data() + 8, E, R, t);
  memcpy(out_i, oi.data(), 5 * sizeof(int32_t));
  if (getenv("MVO_EPI_DEBUG")) fprintf(stderr, "emu_essential: n %d inliers %d GN iterations %d\n", n, oi[0], oi[5]);
  return oi[0];
}

int emu_homography(const float *p1, const float *p2, int n, const double *K, double threshold, int H, uint64_t seed, double *Hout,
                   int32_t *inliers, int32_t *out_i) {
  HomoCam cam;
  cam.f = (K[0] + K[4]) / 2; cam.cx = K[2]; cam.cy = K[5];
  const double thr2 = (threshold / cam.f) * (threshold / cam.f);
  std::vector<double> Hs((size_t)H * 9), out(64, 0.0);
  std::vector<int32_t> valid((size_t)H), counts((size_t)H), oi(64, 0);
  const int32_t pn[1] = {n};
  run_grid((unsigned)((H + 127) / 128), 1, 1, 128, 0,
           [&] { k_homo_hypotheses_batch(p1, p2, pn, n, cam, seed, H, Hs.data(), valid.data(), out.data(), oi.data()); });
  const int grid = std::min((H + 7) / 8, 64);
  run_grid((unsigned)grid, 1, 1, 256, (size_t)n * 32, [&] { k_homo_score_batch(p1, p2, pn, n, cam, thr2, H, Hs.data(), valid.data(), counts.data()); });
  run_clusters(EFIN_C, EFIN_C, EFIN_T, sizeof(HomoFinSmem),
               [&] { k_homo_finish_batch(p1, p2, pn, n, cam, thr2, H, Hs.data(), counts.data(), out.data(), oi.data(), inliers); });
  if (getenv("MVO_EPI_DEBUG")) fprintf(stderr, "emu_homography: n %d inliers %d GN iterations %d\n", n, oi[0], oi[5]);
  memcpy(Hout, out.data(), 72);
  memcpy(out_i, oi.data(), 5 * sizeof(int32_t));
  return oi[0];
}

int emu_triangulate(const float *np1, const float *np2, const int32_t *inl, int n_in, const double *R, const double *t, float *out) {
  double Rt[12];
  memcpy(Rt, R, 72); memcpy(Rt + 9, t, 24);
  run_grid((unsigned)((n_in + 127) / 128), 1, 1, 128, 0, [&] { k_triangulate(np1, np2, inl, n_in, Rt, out); });
  return 0;
}

}  // extern "C"
