// The match-list filter kernels (k_match_filter: thresholds of matchFeatures + removeDuplicatedMatches restated on the device,
// see the comment in track.cu; k_match_filter_batch: the same body once per frame pair of mvo_match_features_batch_dev;
// k_map_match_filter: once per (frame, guess pose) job of mvo_vo_map_matches_batch_dev) and the projection helpers they share
// with the other tracking kernels — the text nvcc
// compiles, in a header so that the CPU test tier can build it for the host (tests/cpp/track_filter_emu.cpp, through
// tests/cpp/cuda_emu.h).  Included by track.cu inside an anonymous namespace.
// MVO_DYN_SMEM(type, name) declares the kernel's dynamic shared memory (`extern __shared__ __align__(16) type name[]` for nvcc).
#pragma once
#include "pdl_device.cuh"

struct Rt12 { double v[12]; };   // R row-major (9) + t (3), world->camera

// getMappointsInCurrentView_ (vo.cpp:16-49) for one map point: true when it is in front of the camera and inside the image
__device__ __forceinline__ bool project_point(const float *__restrict__ map_pts, int i, const Rt12 &Tcw, double fx, double fy, double cx,
                                              double cy, float fcols, float frows, float2 &uv) {
  // basics::preTranslatePoint3f (opencv_funcs.cpp:67-78): double accumulation of T(row, j) * p[j], j = 0..3,
  // narrowed to float.  Explicit _rn intrinsics: no FMA contraction, so the visibility decision is the one the
  // host arithmetic of the reference takes.
  const double p0 = map_pts[3 * i], p1 = map_pts[3 * i + 1], p2 = map_pts[3 * i + 2];
  double q[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    double acc = __dmul_rn(Tcw.v[3 * r], p0);
    acc = __dadd_rn(acc, __dmul_rn(Tcw.v[3 * r + 1], p1));
    acc = __dadd_rn(acc, __dmul_rn(Tcw.v[3 * r + 2], p2));
    acc = __dadd_rn(acc, Tcw.v[9 + r]);
    q[r] = acc;
  }
  const float xc = (float)q[0], yc = (float)q[1], zc = (float)q[2];
  // geometry::cam2pixel: K(0,0) * p.x / p.z + K(0,2) in double, narrowed to Point2f
  const float u = (float)__dadd_rn(__ddiv_rn(__dmul_rn(fx, (double)xc), (double)zc), cx);
  const float v = (float)__dadd_rn(__ddiv_rn(__dmul_rn(fy, (double)yc), (double)zc), cy);
  uv = make_float2(u, v);
  return !(zc < 0) && (u > 0 && v > 0 && u < fcols && v < frows);
}

// T_c_w = inv_rigid(T_w_c) (mvo_internal.h) as the 12 values project_point takes: the same products and sums in the same order,
// each rounded on its own, so that the pose is the host's to the bit whatever the translation unit's contraction setting
__device__ __forceinline__ Rt12 tcw_of_twc(const double *__restrict__ T) {
  Rt12 r;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) r.v[3 * i + j] = T[4 * j + i];
    r.v[9 + i] = -__dadd_rn(__dadd_rn(__dmul_rn(T[i], T[3]), __dmul_rn(T[4 + i], T[7])), __dmul_rn(T[8 + i], T[11]));
  }
  return r;
}

constexpr int MF_T = 1024;
constexpr int MF_MAXN = 8192;        // match-list / keypoint capacity of the device path (host path beyond)

struct FilterArgs {
  const uint32_t *keys;     // [nmap * W]
  uint8_t *vis;             // [nmap] in (project == 0) or out (project == 1)
  int nmap, nk, method, n_cap;
  double xg_ratio, lowe_ratio;
  int2 *pairs;              // out: (map index, keypoint index), sorted by keypoint index
  int32_t *info;            // out: the record of MvoFilterInfo (FI_PAIRS, FI_CANDIDATES, FI_STATUS, then the debug counters)
  // project == 1: getMappointsInCurrentView_ is evaluated here (methods 1/2: the matcher does not need the projections)
  int project;
  const float *map_pts;
  Rt12 Tcw;
  const double *d_Tcw;      // optional: the guess pose is read from device memory (a slot of the tracker's pose ring) instead of Tcw
  double fx, fy, cx, cy;
  float fcols, frows;
  // optional (p3 != nullptr): the 3d-2d pairs of poseEstimationPnP_ (vo.cpp:293-301) go straight into the PnP input arrays
  const mvo_keypoint *kpts;
  float *p3, *p2;
};

__device__ __forceinline__ int block_excl_scan(int v, int *s_warp, int &total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
  __syncthreads();                       // s_warp may still be read from a previous call
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  // every warp scans the 32 warp totals itself (one load + a shuffle scan instead of a serial loop)
  int w = s_warp[lane];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
  total = __shfl_sync(0xffffffffu, w, 31);
  const int before = __shfl_sync(0xffffffffu, w, warp) - __shfl_sync(0xffffffffu, s_warp[lane], warp);
  return before + incl - v;
}

// std::__adjust_heap (+ the std::__push_heap it ends with) on h[0, len), comp(x, y) = keypoint index of x < keypoint index of y
__device__ __forceinline__ void mf_adjust_heap(uint32_t *h, int hole, int len, uint32_t value) {
  const int top = hole;
  int child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if ((h[child] >> 16) < (h[child - 1] >> 16)) --child;
    h[hole] = h[child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    h[hole] = h[child - 1];
    hole = child - 1;
  }
  int parent = (hole - 1) / 2;
  while (hole > top && (h[parent] >> 16) < (value >> 16)) {
    h[hole] = h[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  h[hole] = value;
}

// What __introsort_loop does with a segment at its depth limit: std::__partial_sort(first, last, last) = __heap_select with an
// empty tail (= std::__make_heap) followed by std::__sort_heap.  Sequential by nature: one thread per segment.
__device__ __forceinline__ void mf_heapsort(uint32_t *h, int len) {
  if (len < 2) return;
  for (int parent = (len - 2) / 2;; --parent) {
    mf_adjust_heap(h, parent, len, h[parent]);
    if (parent == 0) break;
  }
  for (int last = len - 1; last > 0; --last) {          // __pop_heap(first, last, last)
    const uint32_t value = h[last];
    h[last] = h[0];
    mf_adjust_heap(h, 0, last, value);
  }
}

constexpr int MF_DFS_LEN = 40;       // segments up to this length are finished (their whole subtree, <= 3 partitions) by one warp, without block barriers
constexpr int MF_STACK = 40;         // per-warp stack of the depth-first phase (>= 2 lg(MF_MAXN) + a margin)

// std::__unguarded_partition_pivot(first, last, by keypoint index) evaluated by one warp; returns the cut (uniform over the warp).
// The stop positions of the left scan (Lo) and of the right scan (Ro) are properties of the range before any swap, the k-th swap pairs
// Lo[k] with Ro[k] while Lo[k] < Ro[k], the cut is min(Lo[K], Ro[K-1]).
__device__ __forceinline__ int mf_partition_warp(uint32_t *arr, uint16_t *Ls, uint16_t *Rs, int first, int last) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) {                         // __move_median_to_first(first, first+1, mid, last-1)
    const int ia = first + 1, ib = first + (last - first) / 2, ic = last - 1;
    const uint32_t ka = arr[ia] >> 16, kb = arr[ib] >> 16, kc = arr[ic] >> 16;
    int pick;
    if (ka < kb) pick = (kb < kc) ? ib : ((ka < kc) ? ic : ia);
    else pick = (ka < kc) ? ia : ((kb < kc) ? ic : ib);
    const uint32_t t = arr[first]; arr[first] = arr[pick]; arr[pick] = t;
  }
  __syncwarp();
  const uint32_t pivot = arr[first] >> 16;
  const int lo = first + 1, len = last - lo;
  const unsigned below = (1u << lane) - 1u;
  int nL = 0, nR = 0;
  for (int base = 0; base < len; base += 64) {                         // two 32-element groups per trip: four independent loads in flight
    const int i0 = base + lane, i1 = i0 + 32;
    const bool in0 = i0 < len, in1 = i1 < len;
    const uint32_t xl0 = in0 ? arr[lo + i0] >> 16 : 0u, xr0 = in0 ? arr[last - 1 - i0] >> 16 : 0u;
    const uint32_t xl1 = in1 ? arr[lo + i1] >> 16 : 0u, xr1 = in1 ? arr[last - 1 - i1] >> 16 : 0u;
    const bool ge0 = in0 && xl0 >= pivot, le0 = in0 && xr0 <= pivot;   // !(x < pivot): the left scan stops; !(pivot < x): the right scan stops
    const bool ge1 = in1 && xl1 >= pivot, le1 = in1 && xr1 <= pivot;
    const unsigned bg0 = __ballot_sync(0xffffffffu, ge0), bl0 = __ballot_sync(0xffffffffu, le0);
    const unsigned bg1 = __ballot_sync(0xffffffffu, ge1), bl1 = __ballot_sync(0xffffffffu, le1);
    const int cg0 = __popc(bg0), cl0 = __popc(bl0);
    if (ge0) Ls[lo + nL + __popc(bg0 & below)] = (uint16_t)(lo + i0);
    if (le0) Rs[lo + nR + __popc(bl0 & below)] = (uint16_t)(last - 1 - i0);
    if (ge1) Ls[lo + nL + cg0 + __popc(bg1 & below)] = (uint16_t)(lo + i1);
    if (le1) Rs[lo + nR + cl0 + __popc(bl1 & below)] = (uint16_t)(last - 1 - i1);
    nL += cg0 + __popc(bg1);
    nR += cl0 + __popc(bl1);
  }
  __syncwarp();
  const int nmin = min(nL, nR);
  int K = 0;
  for (int base = 0; base < nmin; base += 32) {
    const int j = base + lane;
    const bool sw = j < nmin && Ls[lo + j] < Rs[lo + j];
    const unsigned b = __ballot_sync(0xffffffffu, sw);
    if (sw) { const int x = Ls[lo + j], y = Rs[lo + j]; const uint32_t t = arr[x]; arr[x] = arr[y]; arr[y] = t; }
    const int c = __popc(b);
    K += c;
    if (c < 32) break;
  }
  __syncwarp();
  int cut;
  if (K == 0) cut = nL > 0 ? (int)Ls[lo] : last;                      // Lo[0] exists after the median step
  else { cut = (int)Rs[lo + K - 1]; if (K < nL) cut = min(cut, (int)Ls[lo + K]); }
  return cut;
}

// The body of the filter, run by one CTA of MF_T threads over one match list.  kAllVisible: every query takes part (a.vis and
// a.project are not read; the batched matchFeatures tail).  emit(o, query, train) writes the o-th surviving pair.
template <bool kAllVisible, class Emit>
__device__ __forceinline__ void match_filter_run(const FilterArgs &a, uint8_t *smraw, Emit emit) {
  const int cap = a.n_cap;
  uint32_t *arr = (uint32_t *)smraw;                    // [cap]  (train << 16) | position in the match list
  uint32_t *best = arr + cap;                           // [cap]  per keypoint: leftmost (position << 16 | list index)
  uint16_t *amap = (uint16_t *)(best + cap);            // [cap]  map index of list entry i
  uint16_t *Ls = amap + cap;                            // [cap]  Lo lists, segment [first,last) uses Ls[first..last)
  uint16_t *Rs = Ls + cap;                              // [cap]
  uint32_t *segA = (uint32_t *)(Rs + cap);              // [cap/16 + 2] segments of the current level (first | last << 16)
  uint32_t *segB = segA + cap / 16 + 2;
  uint32_t *dfs_seg = segB + cap / 16 + 2;              // [cap/16 + 2] segments of the depth-first phase
  uint8_t *dfs_lvl = (uint8_t *)(dfs_seg + cap / 16 + 2);   // [cap/16 + 2] their partition depth
  __shared__ int s_warp[MF_T / 32];
  __shared__ unsigned s_min;
  __shared__ int s_nseg[2], s_status, s_heap_segs, s_heap_max, s_ndfs;
  __shared__ uint32_t dfs_stack[(MF_T / 32) * MF_STACK];
  __shared__ uint8_t dfs_stack_lvl[(MF_T / 32) * MF_STACK];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nmap = a.nmap;
  const bool sad = a.method == 3;
  if (tid == 0) { s_min = 0xFFFFFFFFu; s_status = 0; s_nseg[0] = s_nseg[1] = 0; s_heap_segs = 0; s_heap_max = 0; s_ndfs = 0; }
  pdl_wait();                       // first kernel of a tracked frame's chain (see launch_pdl.cuh)
  pdl_launch_dependents();
  long long tph = clock64();        // phase cycle counters (thread 0) -> info[FI_CYC_PROLOGUE + i]: prologue, sort levels, epilogue
#define MF_MARK(i) do { if (tid == 0) { const long long t_ = clock64(); a.info[4 + (i)] = (int32_t)(t_ - tph); tph = t_; } } while (0)
  __syncthreads();
  // ---- thresholds (feature_match.cpp:179-196 for methods 1/3, :210-217 for method 2), ordered compaction ----
  const int per = (nmap + MF_T - 1) / MF_T, q0 = min(tid * per, nmap), q1 = min(q0 + per, nmap);
  auto visible = [&](int q) -> bool { return kAllVisible || a.vis[q] != 0; };
  if (!kAllVisible && a.project) {          // every thread reads back only the flags it wrote itself
    Rt12 Tcw = a.Tcw;
    if (a.d_Tcw) {          // enqueued ahead of time: the reference keyframe's pose as the bundle adjustment of the previous frame left it
#pragma unroll
      for (int q = 0; q < 12; ++q) Tcw.v[q] = a.d_Tcw[q];
    }
    for (int q = q0; q < q1; ++q) { float2 uv; a.vis[q] = project_point(a.map_pts, q, Tcw, a.fx, a.fy, a.cx, a.cy, a.fcols, a.frows, uv) ? 1 : 0; }
  }
  int nvis = 0;
  if (a.method != 2) {
    unsigned m = 0xFFFFFFFFu;
    for (int q = q0; q < q1; ++q) {
      if (!visible(q)) continue;
      ++nvis;
      const uint32_t k = a.keys[q];
      if (k != 0xFFFFFFFFu) m = min(m, k >> 16);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0 && m != 0xFFFFFFFFu) atomicMin(&s_min, m);
  } else {
    for (int q = q0; q < q1; ++q) nvis += visible(q);
  }
  __syncthreads();
  double thr = 0;
  if (a.method != 2) {
    // min_dis = 9999999 when nothing matched; distance is a float (Hamming count, or SAD/32 through double)
    const double min_dis = s_min == 0xFFFFFFFFu ? 9999999.0 : (sad ? (double)(float)((double)s_min / 32.0) : (double)(float)s_min);
    thr = (double)fmaxf((float)(min_dis * a.xg_ratio), 30.0f);        // std::max<float>(min_dis * ratio, 30.0)
  }
  auto passes = [&](int q, uint32_t &train) -> bool {
    if (!visible(q)) return false;
    if (a.method != 2) {
      const uint32_t k = a.keys[q];
      if (k == 0xFFFFFFFFu) return false;
      const uint32_t d = k >> 16;
      const float dist = sad ? (float)((double)d / 32.0) : (float)d;
      train = k & 0xFFFFu;
      return (double)dist < thr;
    }
    const uint32_t k0 = a.keys[2 * q], k1 = a.keys[2 * q + 1];
    if (k0 == 0xFFFFFFFFu) return false;
    train = k0 & 0xFFFFu;
    return (double)(float)(k0 >> 16) < a.lowe_ratio * (double)(float)(k1 >> 16);
  };
  int cnt = 0;
  for (int q = q0; q < q1; ++q) { uint32_t tr; cnt += passes(q, tr); }
  int n = 0, ncand = 0;
  int pos = block_excl_scan(cnt, s_warp, n);
  (void)block_excl_scan(nvis, s_warp, ncand);
  if (n > cap || a.nk > cap) {                          // beyond the device path's capacity
    if (tid == 0) { a.info[0] = 0; a.info[1] = ncand; a.info[2] = 1; }
    return;
  }
  for (int q = q0; q < q1; ++q) {
    uint32_t tr;
    if (passes(q, tr)) { arr[pos] = (tr << 16) | (uint32_t)pos; amap[pos] = (uint16_t)q; ++pos; }
  }
  for (int i = tid; i < a.nk; i += MF_T) best[i] = 0xFFFFFFFFu;
  if (tid == 0 && n > 16) { segA[0] = 0u | ((uint32_t)n << 16); s_nseg[0] = 1; }
  __syncthreads();
  MF_MARK(0);
  // ---- quicksort phase of std::sort ----
  // Level by level while segments are long (a list per level, one warp per segment); a segment of at most MF_DFS_LEN elements goes
  // to the list of the depth-first phase, where one warp finishes its whole subtree without a block barrier: the stragglers of
  // unbalanced partitions no longer cost a level (two block barriers, ~1600 cycles) each.  (Measured and dropped: whole-CTA
  // partitions of the long segments — five block barriers, 3300 cycles for 700 elements against 2900 by one warp — and depth-first
  // subtrees from 128 elements, which serialise ~12 partitions in one warp.)
  int depth_limit = 0;
  for (int m = n; m > 1; m >>= 1) ++depth_limit;        // std::__lg(n)
  depth_limit *= 2;
  uint32_t *cur = segA, *nxt = segB;
  int level = 0, which = 0;
  long long tlev = clock64();
  // [first, last) at partition depth lv: to the next level's list, to the depth-first list, or (<= 16) left to the final insertion sort
  auto push = [&](int f, int l, int lv, int nxt_list) {
    if (l - f <= 16) return;
    const uint32_t seg = (uint32_t)f | ((uint32_t)l << 16);
    if (l - f <= MF_DFS_LEN) { const int k = atomicAdd(&s_ndfs, 1); dfs_seg[k] = seg; dfs_lvl[k] = (uint8_t)min(lv, 255); }
    else nxt[atomicAdd(&s_nseg[nxt_list], 1)] = seg;
  };
  while (true) {
    const int nseg = s_nseg[which];
    if (nseg == 0) break;
    if (level >= depth_limit) {                         // libstdc++ heapsorts what is left: one thread per segment
      int big = 0;
      for (int sg = tid; sg < nseg; sg += MF_T) {
        const int first = (int)(cur[sg] & 0xFFFFu), last = (int)(cur[sg] >> 16);
        mf_heapsort(arr + first, last - first);
        big = max(big, last - first);
      }
      if (big) atomicMax(&s_heap_max, big);
      if (tid == 0) atomicAdd(&s_heap_segs, nseg);
      break;
    }
    // __introsort_loop recurses on [cut, last) and continues with [first, cut): both are pushed
    for (int sg = warp; sg < nseg; sg += MF_T / 32) {   // one warp per segment
      const int first = (int)(cur[sg] & 0xFFFFu), last = (int)(cur[sg] >> 16);
      const int cut = mf_partition_warp(arr, Ls, Rs, first, last);
      if (lane == 0) { push(cut, last, level + 1, which ^ 1); push(first, cut, level + 1, which ^ 1); }
    }
    __syncthreads();
    if (tid == 0) {
      if (level < 7) { const long long t_ = clock64(); a.info[9 + 2 * level] = (int32_t)(t_ - tlev); a.info[10 + 2 * level] = nseg; tlev = t_; }
      s_nseg[which] = 0;
    }
    which ^= 1;
    uint32_t *t = cur; cur = nxt; nxt = t;
    ++level;
    __syncthreads();
  }
  __syncthreads();
  // ---- depth-first phase: one warp per listed segment, explicit stack in shared memory ----
  {
    const int ndfs = s_ndfs;
    uint32_t *stk = dfs_stack + warp * MF_STACK;
    uint8_t *stl = dfs_stack_lvl + warp * MF_STACK;
    int heap_segs = 0, heap_max = 0;
    for (int sg = warp; sg < ndfs; sg += MF_T / 32) {
      int sp = 0;
      int first = (int)(dfs_seg[sg] & 0xFFFFu), last = (int)(dfs_seg[sg] >> 16), lv = dfs_lvl[sg];
      while (true) {
        // std::__introsort_loop(first, last, depth): while (last - first > 16) { depth limit -> heapsort; partition; recurse right; last = cut }
        while (last - first > 16) {
          if (lv >= depth_limit || sp >= MF_STACK) {   // (the stack bound cannot bind before the depth limit does)
            if (lane == 0) mf_heapsort(arr + first, last - first);
            __syncwarp();
            ++heap_segs; heap_max = max(heap_max, last - first);
            break;
          }
          const int cut = mf_partition_warp(arr, Ls, Rs, first, last);
          ++lv;
          if (last - cut > 16) { if (lane == 0) { stk[sp] = (uint32_t)cut | ((uint32_t)last << 16); stl[sp] = (uint8_t)min(lv, 255); } ++sp; }
          last = cut;
        }
        if (sp == 0) break;
        --sp;
        __syncwarp();
        first = (int)(stk[sp] & 0xFFFFu); last = (int)(stk[sp] >> 16); lv = stl[sp];
      }
    }
    if (lane == 0 && heap_segs) { atomicAdd(&s_heap_segs, heap_segs); atomicMax(&s_heap_max, heap_max); }
  }
  __syncthreads();
  if (s_status != 0) {
    if (tid == 0) { a.info[0] = 0; a.info[1] = ncand; a.info[2] = 1; }
    return;
  }
  MF_MARK(1);
  if (tid == 0) { a.info[8] = level; a.info[3] = s_heap_segs; a.info[7] = s_heap_max; }     // FI_LEVELS, FI_HEAP_SEGS, FI_HEAP_MAX
  // ---- final insertion sort is stable: of every run of equal keypoint indices the leftmost element survives ----
  for (int p = tid; p < n; p += MF_T) atomicMin(&best[arr[p] >> 16], ((uint32_t)p << 16) | (arr[p] & 0xFFFFu));
  __syncthreads();
  const int pk = (a.nk + MF_T - 1) / MF_T, t0 = min(tid * pk, a.nk), t1 = min(t0 + pk, a.nk);
  int c2 = 0;
  for (int t = t0; t < t1; ++t) c2 += best[t] != 0xFFFFFFFFu;
  int np = 0;
  int o = block_excl_scan(c2, s_warp, np);
  for (int t = t0; t < t1; ++t)
    if (best[t] != 0xFFFFFFFFu) {
      emit(o, (int)amap[best[t] & 0xFFFFu], t);
      ++o;
    }
  if (tid == 0) { a.info[0] = np; a.info[1] = ncand; a.info[2] = 0; }
  MF_MARK(2);
#undef MF_MARK
}

// The tracker's filter: map points (queries) in view of the guess pose against the frame's keypoints (trains); the pairs and,
// optionally, the PnP input arrays
__global__ void __launch_bounds__(MF_T, 1) k_match_filter(FilterArgs a) {
  MVO_DYN_SMEM(uint8_t, smraw);
  match_filter_run<false>(a, smraw, [&](int o, int mi, int t) {
    a.pairs[o] = make_int2(mi, t);
    if (a.p3) {
      a.p3[3 * o] = a.map_pts[3 * mi]; a.p3[3 * o + 1] = a.map_pts[3 * mi + 1]; a.p3[3 * o + 2] = a.map_pts[3 * mi + 2];
      a.p2[2 * o] = a.kpts[t].x; a.p2[2 * o + 1] = a.kpts[t].y;
    }
  });
}

// The tail of geometry::matchFeatures for a batch of frame pairs (mvo_match_features_batch_dev): one CTA per pair over the packed
// keys of match_batch_kernel (match.cu), every query visible, the surviving matches written as cv::DMatch records.  Per pair:
// n_out[p] = number of matches, or MVO_ERR_INVALID_ARG (no writes to out) for a frame index outside [0, batch) or a method-2 pair
// whose train frame has fewer than 2 keypoints.
struct FilterBatchArgs {
  const uint32_t *keys;     // [n_pairs][cap][W]
  const int32_t *counts;    // [batch]
  const int2 *pairs;        // [n_pairs] (query frame, train frame)
  int batch, cap, method, n_cap;
  double xg_ratio, lowe_ratio;
  mvo_dmatch *out;          // [n_pairs][cap]
  int32_t *n_out;           // [n_pairs]
};

__global__ void __launch_bounds__(MF_T, 1) k_match_filter_batch(FilterBatchArgs b) {
  MVO_DYN_SMEM(uint8_t, smraw);
  __shared__ int32_t s_info[24];
  // match_filter_run waits again: griddepcontrol.wait returns at once when the predecessor has already been waited for
  pdl_wait();
  pdl_launch_dependents();
  const int p = blockIdx.x;
  const int2 pr = b.pairs[p];
  const int W = b.method == 2 ? 2 : 1;
  if (pr.x < 0 || pr.x >= b.batch || pr.y < 0 || pr.y >= b.batch) {
    if (threadIdx.x == 0) b.n_out[p] = MVO_ERR_INVALID_ARG;
    return;
  }
  const int n1 = min(max(b.counts[pr.x], 0), b.cap), n2 = min(max(b.counts[pr.y], 0), b.cap);
  if (b.method == 2 && n2 < 2) {            // knnMatch(k = 2) needs two trains: mvo_match_features fails there
    if (threadIdx.x == 0) b.n_out[p] = MVO_ERR_INVALID_ARG;
    return;
  }
  if (n1 == 0 || n2 == 0) {                 // no query, or BFMatcher / the radius search over an empty train set: no matches
    if (threadIdx.x == 0) b.n_out[p] = 0;
    return;
  }
  FilterArgs a = {};
  a.keys = b.keys + (size_t)p * b.cap * W;
  a.nmap = n1; a.nk = n2; a.method = b.method; a.n_cap = b.n_cap;
  a.xg_ratio = b.xg_ratio; a.lowe_ratio = b.lowe_ratio;
  a.info = s_info;
  const uint32_t *keys = a.keys;
  mvo_dmatch *out = b.out + (size_t)p * b.cap;
  const int method = b.method;
  match_filter_run<true>(a, smraw, [&](int o, int qi, int t) {
    // unpack() of match_host.cpp: the best key of the query; method 3's distance is the SAD / 32 through double, img_idx -1
    const uint32_t d = keys[(size_t)qi * W] >> 16;
    mvo_dmatch m;
    m.query_idx = qi;
    m.train_idx = t;
    m.img_idx = method == 3 ? -1 : 0;
    m.distance = method == 3 ? (float)((double)d / 32.0) : (float)d;
    out[o] = m;
  });
  if (threadIdx.x == 0) b.n_out[p] = s_info[2] == 0 ? s_info[0] : MVO_ERR_UNSUPPORTED;   // s_info: written by this thread
}

// The step of poseEstimationPnP_ before solvePnPRansac (vo_pipeline.cpp: pose_estimation_pnp) for a batch of (frame, guess pose)
// jobs against one map (mvo_vo_map_matches_batch_dev): one CTA per job.  The CTA projects the map with T_c_w of the guess
// (getMappointsInCurrentView_), runs the filter over the keys of match_batch_kernel<MODE, true> with the in-view flags, and writes
// the candidate list, the DMatch records and the PnP inputs.  The candidate rows are written only once the filter has finished,
// so that a job it cannot finish writes its status alone; until then a record's query_idx holds the map index, which is turned
// into the candidate rank by a binary search of the (increasing) candidate row.
struct MapFilterArgs {
  const uint32_t *keys;         // [n_jobs][n_map][W]
  uint8_t *vis;                 // [n_jobs][n_map] scratch: in-view flags
  const mvo_keypoint *kpts;     // [batch][cap] (only read for d_pts2d)
  const int32_t *counts;        // [batch]
  const int32_t *frames;        // [n_jobs]
  const double *T_w_c;          // [n_jobs][16]
  const float *map_pts;         // [n_map][3]
  int batch, cap, n_map, method, n_cap;
  double xg_ratio, lowe_ratio;
  double fx, fy, cx, cy;
  float fcols, frows;
  mvo_map_matches_result *out;  // [n_jobs]
  int32_t *cand;                // [n_jobs][n_map]
  float *cand_xy;               // [n_jobs][n_map][2] or null
  mvo_dmatch *matches;          // [n_jobs][cap]
  float *p3, *p2;               // [n_jobs][cap][3] / [2] or null
};

__global__ void __launch_bounds__(MF_T, 1) k_map_match_filter(MapFilterArgs b) {
  MVO_DYN_SMEM(uint8_t, smraw);
  __shared__ int32_t s_info[24];
  __shared__ int s_scan[MF_T / 32];
  // match_filter_run waits again: griddepcontrol.wait returns at once when the predecessor has already been waited for
  pdl_wait();
  pdl_launch_dependents();
  const int j = blockIdx.x, tid = threadIdx.x;
  const int f = b.frames[j];
  const double *T = b.T_w_c + (size_t)j * 16;
  bool bad = f < 0 || f >= b.batch;
  for (int q = 0; q < 16; ++q) bad = bad || !isfinite(T[q]);
  if (bad) {
    if (tid == 0) b.out[j].status = MVO_ERR_INVALID_ARG;
    return;
  }
  const int nk = min(max(b.counts[f], 0), b.cap), nmap = b.n_map, method = b.method;
  const Rt12 Tcw = tcw_of_twc(T);
  uint8_t *vis = b.vis + (size_t)j * nmap;
  // the thread ranges of match_filter_run: every thread reads back only the flags it wrote itself
  const int per = (nmap + MF_T - 1) / MF_T, q0 = min(tid * per, nmap), q1 = min(q0 + per, nmap);
  int nv = 0;
  for (int q = q0; q < q1; ++q) {
    float2 uv;
    const bool in = project_point(b.map_pts, q, Tcw, b.fx, b.fy, b.cx, b.cy, b.fcols, b.frows, uv);
    vis[q] = in ? 1 : 0;
    nv += in;
  }
  int ncand = 0;
  const int rank0 = block_excl_scan(nv, s_scan, ncand);
  int np = 0;
  mvo_dmatch *mo = b.matches + (size_t)j * b.cap;
  if (ncand > 0 && nk > 0 && !(method == 2 && nk < 2)) {     // match_into skips the matcher otherwise
    const int W = method == 2 ? 2 : 1;
    FilterArgs a = {};
    a.keys = b.keys + (size_t)j * nmap * W;
    a.vis = vis;
    a.nmap = nmap; a.nk = nk; a.method = method; a.n_cap = b.n_cap;
    a.xg_ratio = b.xg_ratio; a.lowe_ratio = b.lowe_ratio;
    a.info = s_info;
    const uint32_t *keys = a.keys;
    const float *map_pts = b.map_pts;
    float *p3 = b.p3 ? b.p3 + (size_t)j * b.cap * 3 : nullptr, *p2 = b.p2 ? b.p2 + (size_t)j * b.cap * 2 : nullptr;
    const mvo_keypoint *kp = p2 ? b.kpts + (size_t)f * b.cap : nullptr;
    match_filter_run<false>(a, smraw, [&](int o, int mi, int t) {
      // unpack() of match_host.cpp, as k_match_filter_batch writes it; query_idx is the map index until the rank is known
      const uint32_t d = keys[(size_t)mi * W] >> 16;
      mvo_dmatch m;
      m.query_idx = mi;
      m.train_idx = t;
      m.img_idx = method == 3 ? -1 : 0;
      m.distance = method == 3 ? (float)((double)d / 32.0) : (float)d;
      mo[o] = m;
      if (p3) {                                             // vo.cpp:293-301
        p3[3 * o] = map_pts[3 * mi]; p3[3 * o + 1] = map_pts[3 * mi + 1]; p3[3 * o + 2] = map_pts[3 * mi + 2];
        p2[2 * o] = kp[t].x; p2[2 * o + 1] = kp[t].y;
      }
    });
    __syncthreads();                                        // s_info: written by thread 0 on every way out of the filter
    if (s_info[2] != 0) {
      if (tid == 0) b.out[j].status = MVO_ERR_UNSUPPORTED;
      return;
    }
    np = s_info[0];
  }
  int32_t *cand = b.cand + (size_t)j * nmap;
  float *cxy = b.cand_xy ? b.cand_xy + (size_t)j * nmap * 2 : nullptr;
  int r = rank0;
  for (int q = q0; q < q1; ++q) {
    if (!vis[q]) continue;
    cand[r] = q;
    if (cxy) {
      float2 uv;
      (void)project_point(b.map_pts, q, Tcw, b.fx, b.fy, b.cx, b.cy, b.fcols, b.frows, uv);
      cxy[2 * r] = uv.x; cxy[2 * r + 1] = uv.y;
    }
    ++r;
  }
  __syncthreads();                                          // the candidate row, for the ranks
  for (int o = tid; o < np; o += MF_T) {
    const int mi = mo[o].query_idx;
    int lo = 0, hi = ncand;                                 // the first candidate >= mi: mi itself
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (cand[mid] < mi) lo = mid + 1; else hi = mid; }
    mo[o].query_idx = lo;
  }
  if (tid == 0) {
    mvo_map_matches_result res;
    res.status = MVO_OK; res.n_candidates = ncand; res.n_matches = np; res.pad = 0;
    b.out[j] = res;
  }
}

// The projected pixels of every map point for every job (mvo_vo_map_matches_batch_dev, method 3: the radius gate of the matcher
// needs them before the filter has run); grid.y = jobs.  A job with a non-finite pose writes pixels nobody reads.
__global__ void __launch_bounds__(256) k_project_map_batch(const float *__restrict__ map_pts, int nmap, const double *__restrict__ T_w_c,
                                                           double fx, double fy, double cx, double cy, float fcols, float frows,
                                                           float2 *__restrict__ xy) {
  pdl_wait();
  pdl_launch_dependents();
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= nmap) return;
  const Rt12 Tcw = tcw_of_twc(T_w_c + (size_t)j * 16);
  float2 uv;
  (void)project_point(map_pts, i, Tcw, fx, fy, cx, cy, fcols, frows, uv);
  xy[(size_t)j * nmap + i] = uv;
}
