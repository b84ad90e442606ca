// The per-point numerics of the VO initialisation (reference src/vo/vo.cpp:53-244), written once for the host (vo_host.cpp,
// vo_pipeline.cpp: g++) and the device (vo_init_batch.cu: mvo_vo_init_candidates_batch_dev, compiled without contraction so that
// every product and sum rounds as on the host):
//   mul44 / trans_coord             the 4x4 product and basics::transCoord of estimateMotionAnd3DPoints_
//   triangulation_angle             one angle of retainGoodTriangulationResult_ (vo.cpp:206-214)
//   pixel_dist                      one term of computeMeanDistBetweenKeypoints (feature_match.cpp:262-279)
//   nth_element_d / sort_d          libstdc++'s std::nth_element and std::sort on doubles with operator<, step for step
// What stays with the callers is the order of every sum over points: sequential, in list order.
#pragma once
#include <math.h>
#include <string.h>

#if defined(__CUDACC__)
#define VOI_HD __host__ __device__ __forceinline__
#define VOI_HD_CALL __host__ __device__ __noinline__ inline
#else
#define VOI_HD inline
#define VOI_HD_CALL inline
#endif

namespace voi {

VOI_HD void mul44(const double *A, const double *B, double *C) {        // C may alias A or B
  double r[16];
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) {
    double a = 0;
    for (int k = 0; k < 4; ++k) a += A[i * 4 + k] * B[k * 4 + j];
    r[i * 4 + j] = a;
  }
  memcpy(C, r, sizeof r);
}

// basics::transCoord (opencv_funcs.cpp:121-125): R * p + t in double, narrowed to Point3f
VOI_HD void trans_coord(const float *p, const double *R, const double *t, float *out) {
  for (int r = 0; r < 3; ++r) out[r] = (float)(R[r * 3] * (double)p[0] + R[r * 3 + 1] * (double)p[1] + R[r * 3 + 2] * (double)p[2] + t[r]);
}

// The triangulation angle in degrees of a point given in the current camera: basics::preTranslatePoint3f(p, T_w_c_curr) (double
// accumulation, narrowed to Point3f, back to double, :208-209), the vectors to both camera centres (:210-211),
// calcAngleBetweenTwoVectors (opencv_funcs.cpp:176-190) and the reference's truncated pi (:213).  acos is the platform's: glibc on
// the host, CUDA's on the device (2 ulp), so only this call can make the device differ from the host.
VOI_HD double triangulation_angle(const float *p, const double *T_w_c_curr, const double *T_w_c_ref) {
  const double p0 = p[0], p1 = p[1], p2 = p[2];
  double pw[3];
  for (int r = 0; r < 3; ++r) {
    double acc = 0;
    acc += T_w_c_curr[r * 4] * p0; acc += T_w_c_curr[r * 4 + 1] * p1; acc += T_w_c_curr[r * 4 + 2] * p2; acc += T_w_c_curr[r * 4 + 3] * 1.0;
    pw[r] = (double)(float)acc;
  }
  double v1[3], v2[3], dot = 0, n1 = 0, n2 = 0;
  for (int r = 0; r < 3; ++r) {
    v1[r] = T_w_c_curr[r * 4 + 3] - pw[r];
    v2[r] = T_w_c_ref[r * 4 + 3] - pw[r];
    dot += v1[r] * v2[r]; n1 += v1[r] * v1[r]; n2 += v2[r] * v2[r];
  }
  const double angle = acos(dot / (sqrt(n1) * sqrt(n2)));
  return angle / 3.1415926 * 180.0;
}

// the distance between a keypoint of the reference frame and its match in the current frame: the differences are float
// subtractions, widened afterwards (feature_match.cpp:270-274)
VOI_HD double pixel_dist(float x_ref, float y_ref, float x_curr, float y_curr) {
  const double dx = x_ref - x_curr, dy = y_ref - y_curr;
  return sqrt(dx * dx + dy * dy);
}

// ---- libstdc++'s selection and sort (bits/stl_algo.h, bits/stl_heap.h) on doubles with operator< ----
// With a NaN among the values, std::nth_element and std::sort leave an order that depends on their exact steps (a NaN is neither
// less nor greater than anything).  These restate those steps so that the value they leave at a position is libstdc++'s.  The
// unguarded insertion sort reads below the range only when a NaN breaks the partition's ordering; that read is undefined on the
// host and stops at the first element here.

VOI_HD void stl_swap(double *a, double *b) { const double t = *a; *a = *b; *b = t; }

VOI_HD int stl_lg(int n) { int k = 0; while (n > 1) { n >>= 1; ++k; } return k; }         // std::__lg

VOI_HD void stl_adjust_heap(double *f, int hole, int len, double value) {              // std::__adjust_heap + std::__push_heap
  const int top = hole;
  int second = hole;
  while (second < (len - 1) / 2) {
    second = 2 * (second + 1);
    if (f[second] < f[second - 1]) second--;
    f[hole] = f[second];
    hole = second;
  }
  if ((len & 1) == 0 && second == (len - 2) / 2) {
    second = 2 * (second + 1);
    f[hole] = f[second - 1];
    hole = second - 1;
  }
  int parent = (hole - 1) / 2;
  while (hole > top && f[parent] < value) {
    f[hole] = f[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  f[hole] = value;
}

VOI_HD void stl_make_heap(double *f, int len) {
  if (len < 2) return;
  for (int parent = (len - 2) / 2;; --parent) {
    stl_adjust_heap(f, parent, len, f[parent]);
    if (parent == 0) return;
  }
}

VOI_HD void stl_pop_heap(double *f, int len, double *result) {                        // std::__pop_heap(first, first + len, result)
  const double value = *result;
  *result = f[0];
  stl_adjust_heap(f, 0, len, value);
}

VOI_HD void stl_heap_select(double *f, int middle, int last) {
  stl_make_heap(f, middle);
  for (int i = middle; i < last; ++i)
    if (f[i] < f[0]) stl_pop_heap(f, middle, f + i);
}

VOI_HD void stl_move_median_to_first(double *result, double *a, double *b, double *c) {
  if (*a < *b) {
    if (*b < *c) stl_swap(result, b);
    else if (*a < *c) stl_swap(result, c);
    else stl_swap(result, a);
  } else if (*a < *c) stl_swap(result, a);
  else if (*b < *c) stl_swap(result, c);
  else stl_swap(result, b);
}

// std::__unguarded_partition_pivot on [first, last): returns the cut
VOI_HD int stl_partition_pivot(double *v, int first, int last) {
  const int mid = first + (last - first) / 2;
  stl_move_median_to_first(v + first, v + first + 1, v + mid, v + last - 1);
  const double pivot = v[first];
  int lo = first + 1, hi = last;
  while (true) {
    while (v[lo] < pivot) ++lo;
    --hi;
    while (pivot < v[hi]) --hi;
    if (!(lo < hi)) return lo;
    stl_swap(v + lo, v + hi);
    ++lo;
  }
}

VOI_HD void stl_insertion_sort(double *v, int first, int last) {
  if (first == last) return;
  for (int i = first + 1; i != last; ++i) {
    const double val = v[i];
    if (val < v[first]) {
      for (int k = i; k > first; --k) v[k] = v[k - 1];
      v[first] = val;
    } else {
      int hole = i;
      while (hole - 1 >= first && val < v[hole - 1]) { v[hole] = v[hole - 1]; --hole; }
      v[hole] = val;
    }
  }
}

// std::nth_element(v, v + nth, v + n)
VOI_HD_CALL void nth_element_d(double *v, int nth, int n) {
  if (n == 0 || nth == n) return;
  int first = 0, last = n, depth = stl_lg(n) * 2;
  while (last - first > 3) {
    if (depth == 0) {
      stl_heap_select(v + first, nth - first + 1, last - first);
      stl_swap(v + first, v + nth);
      return;
    }
    --depth;
    const int cut = stl_partition_pivot(v, first, last);
    if (cut <= nth) first = cut;
    else last = cut;
  }
  stl_insertion_sort(v, first, last);
}

// std::sort(v, v + n): __introsort_loop + __final_insertion_sort.  The loop's recursion on the right part becomes the pending
// left parts on an explicit stack (the parts are disjoint, so the order they are taken up in does not matter): stack holds
// SORT_STACK (first, last, depth) triples, enough for the depth limit 2 floor(log2 n) of any int n.
constexpr int SORT_STACK = 64;
VOI_HD_CALL void sort_d(double *v, int n, int *stack) {
  if (n == 0) return;
  int *stack_first = stack, *stack_last = stack + SORT_STACK, *stack_depth = stack + 2 * SORT_STACK, top = 0;
  stack_first[0] = 0; stack_last[0] = n; stack_depth[0] = stl_lg(n) * 2; top = 1;
  while (top > 0) {
    --top;
    int first = stack_first[top], last = stack_last[top], depth = stack_depth[top];
    while (last - first > 16) {
      if (depth == 0) {                                          // std::__partial_sort(first, last, last)
        stl_heap_select(v + first, last - first, last - first);
        for (int l = last - first; l > 1; --l) stl_pop_heap(v + first, l - 1, v + first + l - 1);
        break;
      }
      --depth;
      const int cut = stl_partition_pivot(v, first, last);
      stack_first[top] = first; stack_last[top] = cut; stack_depth[top] = depth; ++top;
      first = cut;
    }
  }
  if (n > 16) {
    stl_insertion_sort(v, 0, 16);
    for (int i = 16; i < n; ++i) {                               // __unguarded_insertion_sort
      const double val = v[i];
      int hole = i;
      while (hole > 0 && val < v[hole - 1]) { v[hole] = v[hole - 1]; --hole; }
      v[hole] = val;
    }
  } else {
    stl_insertion_sort(v, 0, n);
  }
}

}  // namespace voi
