// TEST INFRASTRUCTURE (CPU tier): the VO state machine (csrc/vo_pipeline.cpp, csrc/two_view.cpp) compiled a second time into its own
// shared object in which the GPU stages it calls are replaced by forwarders to function pointers the test installs
// (tests/test_vo_pipeline_host.py points them at the oracle stages).  This checks the HOST logic of the state machine —
// containers, bookkeeping, index plumbing — frame by frame against oracle/vo_pipeline_oracle.py without a GPU.
// Nothing here is part of libmvo.so; the product has no such indirection.
#include <stdarg.h>
#include "mvo_internal.h"

int mvo_fail(mvo_ctx *ctx, int code, const char *fmt, ...) {
  if (ctx) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    ctx->err = buf;
  }
  return code;
}

extern "C" {

struct HostcheckStages {
  int (*orb_extract)(const uint8_t *image, int rows, int cols, int channels, size_t stride, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc);
  int (*match_features)(const uint8_t *d1, int n1, const uint8_t *d2, int n2, int method, const float *xy1, const float *xy2, float radius,
                        mvo_dmatch *out, int *n_out);
  int (*esti_motion_by_homography)(const float *p1, const float *p2, int n, const double *K, double threshold, double *H, double *Rs, double *ts,
                                   double *normals, int *n_solutions, int32_t *inliers, int *n_inliers);
  int (*remove_wrong_rt_of_homography)(const float *np1, const float *np2, int n, const int32_t *inliers, int n_inliers, double *Rs, double *ts,
                                       double *normals, int *n_solutions);
  int (*esti_motion_by_essential)(const float *p1, const float *p2, int n, const double *K, double threshold, double *E, double *R, double *t,
                                  int32_t *inliers, int *n_inliers);
  int (*do_triangulation)(const float *np1, const float *np2, int n, const double *R, const double *t, const int32_t *inliers, int n_inliers,
                          float *pts3d);
  int (*solve_pnp_ransac)(const float *pts3d, const float *pts2d, int n, const double *K, double *rvec, double *tvec, int32_t *inliers,
                          int *n_inliers);
  int (*bundle_adjustment)(double *poses, int n_frames, float *points, int n_points, const int32_t *ef, const int32_t *ep, const float *obs,
                           int n_edges, const double *K, const double *information, int fix_points, int update_points);
};
static HostcheckStages g_stages;

void hostcheck_set_stages(const HostcheckStages *s) { g_stages = *s; }
mvo_ctx *hostcheck_ctx_new(int max_keypoints) {
  mvo_ctx *c = new mvo_ctx();
  mvo_default_params(&c->prm);
  c->prm.max_keypoints = max_keypoints;
  return c;
}
void hostcheck_ctx_free(mvo_ctx *c) { delete c; }
// for the my_slam adapter layer, which creates its own context (my_slam_adapter/mvo_context.cpp)
int mvo_create(mvo_ctx **out, int, const mvo_params *params) {
  mvo_ctx *c = new mvo_ctx();
  if (params) c->prm = *params; else mvo_default_params(&c->prm);
  *out = c;
  return MVO_OK;
}
void mvo_destroy(mvo_ctx *c) { delete c; }
const char *mvo_last_error(const mvo_ctx *c) { return c ? c->err.c_str() : ""; }

int mvo_orb_extract(mvo_ctx *, const uint8_t *image, int rows, int cols, int channels, size_t stride, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc) {
  return g_stages.orb_extract(image, rows, cols, channels, stride, kpts, n_kpts, desc);
}
// The host check covers the host-array mode of the state machine: the device-resident tracker reports itself unavailable, so
// mvo_vo_create selects the host-array path (mvo_trk_device_mode == 0) and none of the other tracker entry points is reached.
int mvo_tracker_create(mvo_ctx *, const double *, int, int, const mvo_track_params *, mvo_tracker **out) { *out = (mvo_tracker *)nullptr; return MVO_OK; }
void mvo_tracker_destroy(mvo_tracker *) {}
int mvo_tracker_prefetch(mvo_tracker *, const uint8_t *, int, size_t, int) { return MVO_ERR_UNSUPPORTED; }
int mvo_tracker_reset(mvo_tracker *, const double *) { return MVO_ERR_UNSUPPORTED; }
int mvo_tracker_frame_pose(const mvo_tracker *, int, double *) { return MVO_ERR_UNSUPPORTED; }
uint64_t mvo_tracker_kernel_launches(const mvo_tracker *) { return 0; }
int mvo_tracker_timing_enable(mvo_tracker *, uint32_t) { return MVO_ERR_UNSUPPORTED; }
int mvo_tracker_timing_read(mvo_tracker *, double *, uint64_t *) { return MVO_ERR_UNSUPPORTED; }
uint64_t mvo_kernel_launches(const mvo_ctx *) { return 0; }
int mvo_timing_enable(mvo_ctx *, uint32_t) { return MVO_ERR_UNSUPPORTED; }
int mvo_timing_read(mvo_ctx *, double *, uint64_t *) { return MVO_ERR_UNSUPPORTED; }
int mvo_match_features(mvo_ctx *, const uint8_t *d1, int n1, const uint8_t *d2, int n2, int method_index, const float *xy1, const float *xy2,
                       float radius, mvo_dmatch *out, int *n_out) {
  return g_stages.match_features(d1, n1, d2, n2, method_index, xy1, xy2, radius, out, n_out);
}
// mvo_estimate_relative_poses itself is the product's csrc/two_view.cpp, compiled into this object next to vo_pipeline.cpp
int mvo_esti_motion_by_homography(mvo_ctx *, const float *p1, const float *p2, int n, const double *K, double threshold, double *H, double *Rs,
                                  double *ts, double *normals, int *n_solutions, int32_t *inliers, int *n_inliers) {
  return g_stages.esti_motion_by_homography(p1, p2, n, K, threshold, H, Rs, ts, normals, n_solutions, inliers, n_inliers);
}
int mvo_remove_wrong_rt_of_homography(mvo_ctx *, const float *np1, const float *np2, int n, const int32_t *inliers, int n_inliers, double *Rs,
                                      double *ts, double *normals, int *n_solutions) {
  return g_stages.remove_wrong_rt_of_homography(np1, np2, n, inliers, n_inliers, Rs, ts, normals, n_solutions);
}
int mvo_esti_motion_by_essential(mvo_ctx *, const float *p1, const float *p2, int n, const double *K, double threshold, double *E, double *R,
                                 double *t, int32_t *inliers, int *n_inliers) {
  return g_stages.esti_motion_by_essential(p1, p2, n, K, threshold, E, R, t, inliers, n_inliers);
}
int mvo_do_triangulation(mvo_ctx *, const float *np1, const float *np2, int n, const double *R, const double *t, const int32_t *inliers,
                         int n_inliers, float *pts3d) {
  return g_stages.do_triangulation(np1, np2, n, R, t, inliers, n_inliers, pts3d);
}
int mvo_solve_pnp_ransac(mvo_ctx *, const float *pts3d, const float *pts2d, int n, const double *K, double *rvec, double *tvec, int32_t *inliers,
                         int *n_inliers) {
  return g_stages.solve_pnp_ransac(pts3d, pts2d, n, K, rvec, tvec, inliers, n_inliers);
}
int mvo_bundle_adjustment(mvo_ctx *, double *poses, int n_frames, float *points, int n_points, const int32_t *ef, const int32_t *ep,
                          const float *obs, int n_edges, const double *K, const double *information, int fix_points, int update_points, double *) {
  return g_stages.bundle_adjustment(poses, n_frames, points, n_points, ef, ep, obs, n_edges, K, information, fix_points, update_points);
}

}  // extern "C"

// never reached in the host check (only device images are copied back); libmvo.so links the CUDA runtime statically
extern "C" cudaError_t cudaMemcpy2D(void *, size_t, const void *, size_t, size_t, size_t, cudaMemcpyKind) { return cudaErrorNotSupported; }
extern "C" const char *cudaGetErrorString(cudaError_t) { return "host check: no CUDA runtime"; }

// C++ linkage, as declared in mvo_internal.h
int mvo_orb_extract_ex(mvo_ctx *, const uint8_t *image, int rows, int cols, int channels, size_t stride, int, mvo_keypoint *kpts, int *n_kpts, uint8_t *desc) {
  return g_stages.orb_extract(image, rows, cols, channels, stride, kpts, n_kpts, desc);
}
// csrc/two_view.cpp runs the two RANSACs as begin / end pairs (side by side on two streams in the product); here the pair forwards to the
// installed stage when it is collected
static struct { const float *p1, *p2; int n; const double *K; double thr; } g_e_job, g_h_job;
cudaStream_t mvo_side_stream(mvo_ctx *) { return nullptr; }
int mvo_epi_essential_begin(mvo_ctx *, const float *p1, const float *p2, int n, const double *K, double threshold, int, const float *, const float *,
                            const double *, const double *, bool, MvoEpiJob *) {
  g_e_job = {p1, p2, n, K, threshold};
  return MVO_OK;
}
int mvo_epi_essential_end(mvo_ctx *, MvoEpiJob *, double *E, double *R, double *t, int32_t *inliers, int *n_inliers, float *) {
  return g_stages.esti_motion_by_essential(g_e_job.p1, g_e_job.p2, g_e_job.n, g_e_job.K, g_e_job.thr, E, R, t, inliers, n_inliers);
}
int mvo_epi_homography_begin(mvo_ctx *, const float *p1, const float *p2, int n, const double *K, double threshold, MvoEpiJob *) {
  g_h_job = {p1, p2, n, K, threshold};
  return MVO_OK;
}
int mvo_epi_homography_end(mvo_ctx *, MvoEpiJob *, const double *, double *H, double *Rs, double *ts, double *normals, int *n_solutions, int32_t *inliers,
                           int *n_inliers) {
  return g_stages.esti_motion_by_homography(g_h_job.p1, g_h_job.p2, g_h_job.n, g_h_job.K, g_h_job.thr, H, Rs, ts, normals, n_solutions, inliers, n_inliers);
}
int mvo_do_triangulation_multi(mvo_ctx *, const float *np1, const float *np2, int n, int nsol, const double *const *R, const double *const *t,
                               const int32_t *const *inliers, const int *n_inliers, float *const *pts3d) {
  for (int s = 0; s < nsol; ++s) {
    const int rc = g_stages.do_triangulation(np1, np2, n, R[s], t[s], inliers[s], n_inliers[s], pts3d[s]);
    if (rc != MVO_OK) return rc;
  }
  return MVO_OK;
}
int mvo_epi_essential_ex(mvo_ctx *, const float *, const float *, int, const double *, double, double *, double *, double *, int32_t *, int *, int, const float *,
                         const float *, const double *, const double *, float *) { return MVO_ERR_UNSUPPORTED; }
int mvo_match_filter_keys(mvo_ctx *, int, const uint32_t *, int, mvo_dmatch *, int *) { return MVO_ERR_UNSUPPORTED; }
int mvo_trk_keyframe_fetch(mvo_tracker *, int, int, int, int, int, int, MvoKfFetch *) { return MVO_ERR_UNSUPPORTED; }
int mvo_trk_set_ref_desc(mvo_tracker *, int, int) { return MVO_ERR_UNSUPPORTED; }
int mvo_trk_device_mode(const mvo_tracker *) { return 0; }
void mvo_trk_configure(mvo_tracker *, int, int) {}
int mvo_trk_acquire(mvo_tracker *, const uint8_t *, int, size_t, int, int *, int *) { return MVO_ERR_UNSUPPORTED; }
void mvo_trk_release(mvo_tracker *, int) {}
int mvo_trk_fetch(mvo_tracker *, int, mvo_keypoint *, uint8_t *, uint8_t *) { return MVO_ERR_UNSUPPORTED; }
unsigned mvo_trk_slot_serial(const mvo_tracker *, int) { return 0; }
int mvo_trk_set_map_ids(mvo_tracker *, const float *, const uint8_t *, const int32_t *, int, int) { return MVO_ERR_UNSUPPORTED; }
int mvo_trk_push_frame(mvo_tracker *, const double *, const int32_t *, const int32_t *, const float *, int) { return MVO_ERR_UNSUPPORTED; }
int mvo_trk_append_links(mvo_tracker *, int, const int32_t *, const int32_t *, const float *, int) { return MVO_ERR_UNSUPPORTED; }
int mvo_trk_links(mvo_tracker *, int, int32_t *, int32_t *, int, int *) { return MVO_ERR_UNSUPPORTED; }
int mvo_trk_track(mvo_tracker *, int, const double *, const double *, double *, mvo_track_result *, int, int) { return MVO_ERR_UNSUPPORTED; }
