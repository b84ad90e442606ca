// The per-correspondence numerics of ORB-SLAM's E / H scores (reference src/geometry/motion_estimation.cpp:501-664), written once
// for the host (motion_host.cpp: mvo_check_essential_score / mvo_check_homography_score, g++) and the device (two_view_batch.cu:
// mvo_estimate_relative_poses_batch_dev, compiled without contraction so that every product and sum rounds as on the host).
// What stays with the callers is the order of the sum: thScore - chi is added point by point in inlier-list order.
#pragma once
#include "epipolar_math.cuh"

namespace epi {

constexpr double EH_ESSENTIAL_TH = 3.841, EH_ESSENTIAL_TH_SCORE = 5.991;   // checkEssentialScore (:524-527)
constexpr double EH_HOMOGRAPHY_TH = 5.991;                                  // checkHomographyScore (:613-614)

// 3x3 inverse by cofactors; false when the determinant is zero or not a number
EPI_HD bool inv3(const double *M, double *I) {
  const double c0 = M[4] * M[8] - M[5] * M[7], c1 = M[5] * M[6] - M[3] * M[8], c2 = M[3] * M[7] - M[4] * M[6];
  const double det = M[0] * c0 + M[1] * c1 + M[2] * c2;
  if (!(fabs(det) > 0)) return false;
  const double id = 1.0 / det;
  I[0] = c0 * id; I[1] = (M[2] * M[7] - M[1] * M[8]) * id; I[2] = (M[1] * M[5] - M[2] * M[4]) * id;
  I[3] = c1 * id; I[4] = (M[0] * M[8] - M[2] * M[6]) * id; I[5] = (M[2] * M[3] - M[0] * M[5]) * id;
  I[6] = c2 * id; I[7] = (M[1] * M[6] - M[0] * M[7]) * id; I[8] = (M[0] * M[4] - M[1] * M[3]) * id;
  return true;
}

// F21 = K^-T E21 K^-1 (:507-509) from K^-1
EPI_HD void essential_score_F(const double *E21, const double *Ki, double *F) {
  double KiT[9], T[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) KiT[i * 3 + j] = Ki[j * 3 + i];
  mat3_mul(E21, Ki, T);
  mat3_mul(KiT, T, F);
}

// checkEssentialScore for one correspondence (pixels): chi1 of x2 against l2 = F21 x1 (:543-557), chi2 of x1 against
// l1 = x2^T F21 (:559-573)
EPI_HD void essential_score_chi(const double *F, double u1, double v1, double u2, double v2, double invSigmaSquare, double *chi1, double *chi2) {
  const double a2 = F[0] * u1 + F[1] * v1 + F[2], b2 = F[3] * u1 + F[4] * v1 + F[5], c2 = F[6] * u1 + F[7] * v1 + F[8];
  const double num2 = a2 * u2 + b2 * v2 + c2;
  *chi1 = num2 * num2 / (a2 * a2 + b2 * b2) * invSigmaSquare;
  const double a1 = F[0] * u2 + F[3] * v2 + F[6], b1 = F[1] * u2 + F[4] * v2 + F[7], c1 = F[2] * u2 + F[5] * v2 + F[8];
  const double num1 = a1 * u1 + b1 * v1 + c1;
  *chi2 = num1 * num1 / (a1 * a1 + b1 * b1) * invSigmaSquare;
}

// checkHomographyScore for one correspondence (pixels): chi1 of x2 mapped into image 1 by H12 (:628-640), chi2 of x1 mapped
// into image 2 by H21 (:642-656)
EPI_HD void homography_score_chi(const double *H21, const double *H12, double u1, double v1, double u2, double v2, double invSigmaSquare,
                                 double *chi1, double *chi2) {
  const double wi = 1.0 / (H12[6] * u2 + H12[7] * v2 + H12[8]);
  const double u2in1 = (H12[0] * u2 + H12[1] * v2 + H12[2]) * wi, v2in1 = (H12[3] * u2 + H12[4] * v2 + H12[5]) * wi;
  *chi1 = ((u1 - u2in1) * (u1 - u2in1) + (v1 - v2in1) * (v1 - v2in1)) * invSigmaSquare;
  const double wj = 1.0 / (H21[6] * u1 + H21[7] * v1 + H21[8]);
  const double u1in2 = (H21[0] * u1 + H21[1] * v1 + H21[2]) * wj, v1in2 = (H21[3] * u1 + H21[4] * v1 + H21[5]) * wj;
  *chi2 = ((u2 - u1in2) * (u2 - u1in2) + (v2 - v1in2) * (v2 - v1in2)) * invSigmaSquare;
}

// The E / H choice (:134-154): ratio = score_h / (score_e + score_h) (:137); above the threshold, among the num_h homography
// solutions (indices 1..num_h, h_normals = num_h x 3) the one whose plane normal is most frontal, otherwise solution 0 (the
// essential one, motion_estimation.cpp:60-103).  Returns the ratio.
EPI_HD double eh_choose(double score_e, double score_h, const double *h_normals, int num_h, double threshold, int *best_sol) {
  const double ratio = score_h / (score_e + score_h);
  int best = 0;
  if (ratio > threshold && num_h > 0) {
    best = 1;
    double largest = fabs(h_normals[2]);
    for (int i = 2; i <= num_h; ++i) {
      const double nz = fabs(h_normals[3 * (i - 1) + 2]);
      if (nz > largest) { largest = nz; best = i; }
    }
  }
  *best_sol = best;
  return ratio;
}

}  // namespace epi
