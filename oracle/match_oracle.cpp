// TEST ORACLE — CPU restatement of the reference's descriptor-matching path.
// Not linked into libmvo.so; only tests/, smoke() and bench.py's cpu_baseline use it.
//
// Restates (reference paths relative to the reference repo root):
//   orc_select_uniform_kpts_by_grid   src/geometry/feature_match.cpp:51-84
//   orc_match_radius_bf               src/geometry/feature_match.cpp:86-124
//   orc_match_features                src/geometry/feature_match.cpp:126-239
//   orc_remove_duplicated_matches     src/geometry/feature_match.cpp:241-260
//   orc_hamming_nn / orc_hamming_knn2 cv::BFMatcher(NORM_HAMMING) match / knnMatch(k=2) as
//       called at feature_match.cpp:162 (exact form of the LSH search) and :208.  OpenCV is a
//       third-party dependency absent from the reference tree; its tie rule (lowest train
//       index first, strict '<' insertion) is pinned against cv2 4.13 in tests/test_match_oracle.py.
//   orc_retain_best                   cv::KeyPointsFilter::retainBest (OpenCV keypoint.cpp),
//       used by cv::ORB::detect per level (SURVEY.md App. A.4).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

extern "C" {

struct OrcKeyPoint { float x, y, size, angle, response; int32_t octave, class_id; };
struct OrcDMatch { int32_t queryIdx, trainIdx, imgIdx; float distance; };

static inline int hamming32(const uint8_t *a, const uint8_t *b) {
  int d = 0;
  for (int k = 0; k < 32; ++k) d += __builtin_popcount((unsigned)(a[k] ^ b[k]));
  return d;
}

// BFMatcher.match: best train per query, ties -> lowest trainIdx.
void orc_hamming_nn(const uint8_t *d1, int n1, const uint8_t *d2, int n2, OrcDMatch *out) {
  for (int i = 0; i < n1; ++i) {
    int best = -1, bj = -1;
    for (int j = 0; j < n2; ++j) {
      int d = hamming32(d1 + 32 * i, d2 + 32 * j);
      if (bj < 0 || d < best) { best = d; bj = j; }
    }
    out[i] = OrcDMatch{i, bj, 0, (float)best};
  }
}

// BFMatcher.knnMatch(k=2): sorted insertion with strict '<'.
void orc_hamming_knn2(const uint8_t *d1, int n1, const uint8_t *d2, int n2, OrcDMatch *out) {
  for (int i = 0; i < n1; ++i) {
    int b0 = 1 << 30, j0 = -1, b1 = 1 << 30, j1 = -1;
    for (int j = 0; j < n2; ++j) {
      int d = hamming32(d1 + 32 * i, d2 + 32 * j);
      if (d < b0) { b1 = b0; j1 = j0; b0 = d; j0 = j; }
      else if (d < b1) { b1 = d; j1 = j; }
    }
    out[2 * i] = OrcDMatch{i, j0, 0, (float)b0};
    out[2 * i + 1] = OrcDMatch{i, j1, 0, (float)b1};
  }
}

// feature_match.cpp:86-124.  Returns the number of matches written.
int orc_match_radius_bf(const float *xy1, const float *xy2, const uint8_t *d1, const uint8_t *d2,
                        int N1, int N2, float max_matching_pixel_dist, OrcDMatch *out) {
  int n = 0;
  float r2 = max_matching_pixel_dist * max_matching_pixel_dist;
  for (int i = 0; i < N1; i++) {
    bool is_matched = false;
    float x = xy1[2 * i], y = xy1[2 * i + 1];
    double min_feature_dist = 99999999.0, target_idx = 0;
    for (int j = 0; j < N2; j++) {
      float x2 = xy2[2 * j], y2 = xy2[2 * j + 1];
      if ((x - x2) * (x - x2) + (y - y2) * (y - y2) <= r2) {
        // cv::absdiff + cv::sum over the 32 bytes, divided by cols
        double s = 0;
        for (int k = 0; k < 32; ++k) s += std::abs((int)d1[32 * i + k] - (int)d2[32 * j + k]);
        double feature_dist = s / 32;
        if (feature_dist < min_feature_dist) {
          min_feature_dist = feature_dist;
          target_idx = j;
          is_matched = true;
        }
      }
    }
    if (is_matched) out[n++] = OrcDMatch{i, (int)target_idx, -1, static_cast<float>(min_feature_dist)};
  }
  return n;
}

// feature_match.cpp:241-260 (std::sort is unstable: same libstdc++ as the product build).
int orc_remove_duplicated_matches(OrcDMatch *m, int n) {
  std::vector<OrcDMatch> matches(m, m + n);
  std::sort(matches.begin(), matches.end(),
            [](const OrcDMatch &m1, const OrcDMatch &m2) { return m1.trainIdx < m2.trainIdx; });
  std::vector<OrcDMatch> res;
  if (!matches.empty()) res.push_back(matches[0]);
  for (size_t i = 1; i < matches.size(); i++)
    if (matches[i].trainIdx != matches[i - 1].trainIdx) res.push_back(matches[i]);
  std::memcpy(m, res.data(), res.size() * sizeof(OrcDMatch));
  return (int)res.size();
}

// feature_match.cpp:126-239 with method 1 = exact Hamming NN (what FLANN-LSH approximates).
// ratios are the values after the reference's Config::get<int> rounding (2 and 1).
// Returns the number of matches, or -1 for a wrong method index (reference throws).
int orc_match_features(const uint8_t *d1, int n1, const uint8_t *d2, int n2, int method_index,
                       const float *xy1, const float *xy2, float max_matching_pixel_dist,
                       double xiang_gao_ratio, double lowe_ratio, OrcDMatch *out) {
  std::vector<OrcDMatch> matches;
  double min_dis = 9999999, max_dis = 0, distance_threshold = -1;
  if (method_index == 1 || method_index == 3) {
    std::vector<OrcDMatch> all(n1 > 0 ? n1 : 1);
    int na;
    if (method_index == 3) na = orc_match_radius_bf(xy1, xy2, d1, d2, n1, n2, max_matching_pixel_dist, all.data());
    else { if (n2 > 0) { orc_hamming_nn(d1, n1, d2, n2, all.data()); na = n1; } else na = 0; }
    for (int i = 0; i < na; i++) {
      double dist = all[i].distance;
      if (dist < min_dis) min_dis = dist;
      if (dist > max_dis) max_dis = dist;
    }
    distance_threshold = std::max<float>(min_dis * xiang_gao_ratio, 30.0);
    for (int i = 0; i < na; i++)
      if (all[i].distance < distance_threshold) matches.push_back(all[i]);
  } else if (method_index == 2) {
    std::vector<OrcDMatch> knn(2 * (size_t)(n1 > 0 ? n1 : 1));
    orc_hamming_knn2(d1, n1, d2, n2, knn.data());
    for (int i = 0; i < n1; i++) {
      double dist = knn[2 * i].distance;
      if (dist < lowe_ratio * knn[2 * i + 1].distance) matches.push_back(knn[2 * i]);
    }
  } else {
    return -1;
  }
  int n = (int)matches.size();
  if (n) std::memcpy(out, matches.data(), n * sizeof(OrcDMatch));
  return orc_remove_duplicated_matches(out, n);
}

// feature_match.cpp:179-196 + :229 applied to an externally computed nearest-neighbour list
// (lets the CPU baseline use cv::BFMatcher — bit-identical to orc_hamming_nn — for the search).
int orc_threshold_and_dedup(OrcDMatch *all, int na, double xiang_gao_ratio) {
  double min_dis = 9999999, max_dis = 0;
  for (int i = 0; i < na; i++) {
    double dist = all[i].distance;
    if (dist < min_dis) min_dis = dist;
    if (dist > max_dis) max_dis = dist;
  }
  double distance_threshold = std::max<float>(min_dis * xiang_gao_ratio, 30.0);
  int n = 0;
  for (int i = 0; i < na; i++)
    if (all[i].distance < distance_threshold) all[n++] = all[i];
  return orc_remove_duplicated_matches(all, n);
}

// feature_match.cpp:51-84 (grid dims from this call's image size).
int orc_select_uniform_kpts_by_grid(OrcKeyPoint *kp, int n, int image_rows, int image_cols,
                                    int max_num_keypoints, int grid_size, int max_pts_per_grid) {
  int rows = image_rows / grid_size, cols = image_cols / grid_size;
  std::vector<std::vector<int>> grid(rows, std::vector<int>(cols, 0));
  std::vector<OrcKeyPoint> tmp;
  int cnt = 0;
  for (int i = 0; i < n; ++i) {
    const OrcKeyPoint &kpt = kp[i];
    int row = ((int)kpt.y) / grid_size, col = ((int)kpt.x) / grid_size;
    // reference: out-of-bounds UB for a keypoint in the strip right of / below the last whole cell (image size not a multiple of
    // grid_size, strip wider than the 31-px ORB border); the project's reading, shared by the library's device and host paths: skipped
    if (row < 0 || row >= rows || col < 0 || col >= cols) continue;
    if (grid[row][col] < max_pts_per_grid) {
      tmp.push_back(kpt);
      grid[row][col]++;
      cnt++;
      if (cnt > max_num_keypoints) break;
    }
  }
  if (!tmp.empty()) std::memcpy(kp, tmp.data(), tmp.size() * sizeof(OrcKeyPoint));
  return (int)tmp.size();
}

// cv::KeyPointsFilter::retainBest on (response, payload index) pairs; returns new size.
// idx[] is permuted exactly as the keypoint vector would be.
int orc_retain_best(float *response, int32_t *idx, int n, int n_points) {
  struct E { float r; int32_t i; };
  std::vector<E> v(n);
  for (int k = 0; k < n; ++k) v[k] = E{response[k], idx[k]};
  if (n_points >= 0 && (int)v.size() > n_points) {
    if (n_points == 0) { return 0; }
    std::nth_element(v.begin(), v.begin() + n_points - 1, v.end(),
                     [](const E &a, const E &b) { return a.r > b.r; });
    float ambiguous = v[n_points - 1].r;
    auto new_end = std::partition(v.begin() + n_points, v.end(),
                                  [ambiguous](const E &e) { return e.r >= ambiguous; });
    v.resize(new_end - v.begin());
  }
  for (size_t k = 0; k < v.size(); ++k) { response[k] = v[k].r; idx[k] = v[k].i; }
  return (int)v.size();
}

}  // extern "C"
