// Programmatic dependent launch (PDL) for the chain of small dependent kernels a tracked frame is (match filter -> PnP hypotheses ->
// scores -> finish -> refit -> glue -> window BA).  A kernel launched through launch_pdl may start while its predecessor in the stream
// is still running: its CTAs become resident as soon as every CTA of the predecessor has executed pdl_launch_dependents() (or has
// exited), run their prologue, and block in pdl_wait() until the predecessor's grid has completed and its writes are visible.  What is
// saved per boundary is the launch latency and the prologue (a few microseconds of a ~20 us kernel).
// Rules kept in this code base: every kernel launched through launch_pdl calls pdl_wait() before it touches global memory, and
// pdl_launch_dependents() right after; kernels without these calls are never launched with the attribute.
// MVO_PDL=0 launches the same kernels without the attribute (A/B hook).  The CPU test tier launches them as plain (cluster) kernels.
#pragma once
#include <stdlib.h>
#include <utility>

#include "pdl_device.cuh"

// grid x block threads, `cluster` CTAs per cluster (0 = no cluster attribute).  A kernel that uses cluster instructions (distributed
// shared memory, st.async, cluster barriers) needs the attribute even for a cluster of one CTA: without it the first of them faults
// with an illegal instruction.
template <class... P, class... A>
static inline cudaError_t launch_pdl(cudaStream_t stream, unsigned grid, unsigned block, size_t smem, unsigned cluster, void (*kernel)(P...), A &&...args) {
  static const bool pdl_on = !(getenv("MVO_PDL") && atoi(getenv("MVO_PDL")) == 0);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned na = 0;
  if (cluster > 0) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
#ifdef __CUDACC__
  if (pdl_on) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
#else
  (void)pdl_on;
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return emu_cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
#endif
}

// the same for kernels with multi-dimensional grids (the extraction chain: gray -> pyramid -> FAST -> select -> Harris -> retainBest ->
// grid selection -> blur -> describe -> pre-match); no clusters there
template <class... P, class... A>
static inline cudaError_t launch_pdl3(cudaStream_t stream, dim3 grid, dim3 block, size_t smem, void (*kernel)(P...), A &&...args) {
#ifdef __CUDACC__
  static const bool pdl_on = !(getenv("MVO_PDL") && atoi(getenv("MVO_PDL")) == 0) && !(getenv("MVO_PDL_ORB") && atoi(getenv("MVO_PDL_ORB")) == 0);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  unsigned na = 0;
  if (pdl_on) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
#else
  (void)stream;
  emu_launch(grid, block, smem, [&] { kernel(args...); });
  return cudaSuccess;
#endif
}
