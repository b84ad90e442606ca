// The VisualOdometry state machine of the reference (SURVEY.md §8f-2) as host C++ over the C-ABI stages of this library:
//   addFrame                        reference src/vo/vo_addFrame.cpp:10-142
//   estimateMotionAnd3DPoints_      src/vo/vo.cpp:53-111   -> mvo_estimate_relative_poses, mvo_retain_good_triangulation,
//                                                             mvo_normalize_init_depth
//   isVoGoodToInit_                 src/vo/vo.cpp:113-172  -> mvo_is_vo_good_to_init
//   poseEstimationPnP_              src/vo/vo.cpp:267-381  -> mvo_match_features, mvo_solve_pnp_ransac
//   callBundleAdjustment_           src/vo/vo.cpp:384-478  -> mvo_bundle_adjustment
//   addKeyFrame_ / optimizeMap_ / pushCurrPointsToMap_ / getViewAngle_   src/vo/vo.cpp:482-584
//   keyframe branch                 vo_addFrame.cpp:93-124 -> mvo_esti_motion_by_essential (helperFindInlierMatchesByEpipolarCons,
//                                                             motion_estimation.cpp:180-196), mvo_do_triangulation
//                                                             (helperTriangulatePoints, :200-240)
// Frames, map points and their graph live in the same containers as in the reference (Frame / MapPoint / Map,
// include/my_slam/vo/*.h): the map and the per-frame keypoint -> map point links are std::unordered_map<int, ...> and are
// walked in container order, so the candidate order handed to the matcher is the reference's.  Every numeric stage runs on
// the GPU through the entry points named above; this file holds no arithmetic beyond 4x4 products and the bookkeeping.
//
// Where the reference would abort (an OpenCV assertion below 5 matched points in findEssentialMat; an empty rvec after a
// failed solvePnPRansac) the frame is skipped / the PnP is reported as failed instead.
//
// Two modes, selected by mvo_vo_params::track.device_resident:
//   * device-resident (default; shipped configuration = fixed map points): the tracking branch (vo_addFrame.cpp:71-91) runs
//     through the device-resident tracker (tracker.cpp): the map (in THIS file's container order, re-uploaded whenever a
//     keyframe changes it), the frame buffer and the BA graph stay in HBM, a tracked frame costs one host synchronisation,
//     and MapPoint::visible_times_ / matched_times_ are accumulated on the device and read back when optimizeMap_ needs
//     them.  Keypoints, descriptors and connections of a tracked frame are only copied to the host when the frame becomes
//     a keyframe (or the caller asks for them).  Initialisation and keyframe insertion fetch the frame (a keyframe also its
//     connections and the counters) with its match against the reference keyframe in one synchronisation
//     (mvo_trk_keyframe_fetch); a keyframe's essential-matrix RANSAC and its triangulation share one submission.
//   * host arrays (device_resident = 0, and always with free map points): every stage through its public entry point,
//     four host round trips per tracked frame, as a maintainer who only swaps the bodies of the reference functions gets it.
// Both give the same states, counts and keyframes; poses agree to the summation order of the BA (tests/test_vo_pipeline_gpu.py).
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <deque>
#include <memory>
#include <unordered_map>
#include <vector>
#include "mvo_internal.h"
#include "vo_init_math.cuh"

namespace {

// MVO_VO_DEBUG=1: host wall time of the stages of the initialisation / keyframe branches, printed per frame (stderr)
struct StageClock {
  bool on;
  double t0, acc[12];
  const char *name[12];
  int n;
  static double now() { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
  StageClock() : on(getenv("MVO_VO_DEBUG") != nullptr), t0(0), n(0) { if (on) t0 = now(); }
  void mark(const char *what) { if (!on || n >= 12) return; const double t = now(); name[n] = what; acc[n++] = t - t0; t0 = t; }
  void report(const char *head, int frame) {
    if (!on) return;
    fprintf(stderr, "%s frame %d:", head, frame);
    for (int i = 0; i < n; ++i) fprintf(stderr, " %s %.0f", name[i], acc[i]);
    fprintf(stderr, " us\n");
  }
};

enum { VO_BLANK = 0, VO_DOING_INITIALIZATION = 1, VO_DOING_TRACKING = 2, VO_LOST = 3 };   // vo.h:52-58

struct PtConn { int pt_ref_idx, pt_map_idx; };                   // frame.h:14-18

struct VoFrame {                                                 // vo::Frame (frame.h:20-98)
  int id = 0;
  std::vector<mvo_keypoint> kpts;
  std::vector<uint8_t> desc;                                     // n x 32
  std::vector<uint8_t> colors;                                   // n x 3, r g b (kpts_colors_)
  std::vector<float> xy;                                         // n x 2, keypoints_[i].pt
  double T_w_c[16];
  std::vector<mvo_dmatch> matches_with_ref, inliers_matches_with_ref, inliers_matches_for_3d, matches_with_map;
  std::vector<float> inliers_pts3d;                              // 3 per point, in this camera's frame
  std::vector<double> triangulation_angles;
  std::unordered_map<int, PtConn> conn;                          // inliers_to_mappt_connections_
  // device-resident mode: keypoints / descriptors / connections of a tracked frame stay on the GPU until somebody needs them
  bool host_ready = true, conn_ready = true;
  int nk = 0, slot = -1;
  unsigned serial = 0;
  int n() const { return host_ready ? (int)kpts.size() : nk; }
};
typedef std::shared_ptr<VoFrame> FramePtr;

struct VoMapPoint {                                              // vo::MapPoint (mappoint.h, mappoint.cpp:12-20)
  int id = 0;
  float pos[3];
  double norm[3];
  uint8_t desc[32];
  uint8_t rgb[3];
  int visible_times = 1, matched_times = 1;
};

using voi::mul44;
using voi::trans_coord;
void rodrigues_to_R(const double *w, double *R) {                // cv::Rodrigues(rvec -> R)
  const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (th < 1e-300) { R[0] = R[4] = R[8] = 1; R[1] = R[2] = R[3] = R[5] = R[6] = R[7] = 0; return; }
  const double c = cos(th), s = sin(th), c1 = 1 - c, x = w[0] / th, y = w[1] / th, z = w[2] / th;
  R[0] = c + c1 * x * x;     R[1] = c1 * x * y - s * z; R[2] = c1 * x * z + s * y;
  R[3] = c1 * x * y + s * z; R[4] = c + c1 * y * y;     R[5] = c1 * y * z - s * x;
  R[6] = c1 * x * z - s * y; R[7] = c1 * y * z + s * x; R[8] = c + c1 * z * z;
}

}  // namespace

struct mvo_vo {
  mvo_ctx *ctx = nullptr;
  mvo_vo_params prm;
  double K[9];
  int rows = 0, cols = 0;
  int state = VO_BLANK;
  std::unordered_map<int, VoMapPoint> map_points;                // vo::Map::map_points_ (map.h:21)
  std::unordered_map<int, FramePtr> keyframes;                   // vo::Map::keyframes_
  std::deque<FramePtr> buff;                                     // frames_buff_ (vo.h:70)
  FramePtr curr, prev, ref, prev_ref;
  int frame_factory_id = 0, point_factory_id = 0;                // Frame::factory_id_, MapPoint::factory_id_ (per instance here)
  double map_point_erase_ratio = 0.1;                            // function-local static of optimizeMap_ (vo.cpp:490-491)
  // scratch
  std::vector<float> p1, p2, np1, np2, pts3d, cand_xy, p3d, p2d, ba_ob, ba_pts;
  std::vector<uint8_t> cand_desc;
  std::vector<int32_t> inl, keep, cand_id, ba_ef, ba_ep, ba_used;
  std::vector<double> angles, ba_poses;
  std::vector<mvo_dmatch> matches;
  // device-resident mode
  mvo_tracker *trk = nullptr;
  bool dev = false;
  std::vector<int32_t> dev_order;                                // map point ids in the order of the last upload (container order)
  const uint8_t *cur_image = nullptr;                            // the frame being added (host pointer, or device pointer + scratch copy)
  int cur_channels = 0, cur_on_device = 0;
  size_t cur_stride = 0;
  std::vector<uint8_t> img_scratch;
  std::vector<int32_t> new_ids, new_kp;
  std::vector<float> new_obs, up_pts, tri_all;
  std::vector<uint8_t> up_desc;
};

namespace {

int match_into(mvo_vo *v, const uint8_t *d1, const float *xy1, int n1, const VoFrame &f2, int method, float radius,
               std::vector<mvo_dmatch> *out) {
  out->clear();
  if (n1 <= 0 || f2.n() <= 0 || (method == 2 && f2.n() < 2)) return MVO_OK;
  out->resize((size_t)n1);
  int nm = 0;
  const int rc = mvo_match_features(v->ctx, d1, n1, f2.desc.data(), f2.n(), method, xy1, f2.xy.data(), radius, out->data(), &nm);
  if (rc != MVO_OK) { out->clear(); return rc; }
  out->resize((size_t)nm);
  return MVO_OK;
}

// pixel colours of Frame::calcDescriptors (frame.h:80-84) from a HOST image
void sample_colors(VoFrame *f, const uint8_t *image, int channels, size_t stride) {
  const int n = (int)f->kpts.size();
  f->colors.resize((size_t)n * 3);
  for (int i = 0; i < n; ++i) {
    const int x = (int)floorf(f->kpts[i].x), y = (int)floorf(f->kpts[i].y);
    const uint8_t *px = image + (size_t)y * stride + (size_t)x * channels;
    if (channels == 3) { f->colors[3 * i] = px[2]; f->colors[3 * i + 1] = px[1]; f->colors[3 * i + 2] = px[0]; }   // getPixelAt: {r, g, b}
    else { f->colors[3 * i] = f->colors[3 * i + 1] = f->colors[3 * i + 2] = px[0]; }
  }
}

// the image of the frame being added as a host pointer (an image handed over in device memory is copied once, on demand)
int host_image(mvo_vo *v, const uint8_t **img, size_t *stride) {
  if (!v->cur_on_device) { *img = v->cur_image; *stride = v->cur_stride; return MVO_OK; }
  const size_t row = (size_t)v->cols * v->cur_channels;
  if (v->img_scratch.size() != row * v->rows) {
    v->img_scratch.resize(row * v->rows);
    MVO_CUDA(v->ctx, cudaMemcpy2D(v->img_scratch.data(), row, v->cur_image, v->cur_stride, row, v->rows, cudaMemcpyDeviceToHost));
  }
  *img = v->img_scratch.data();
  *stride = row;
  return MVO_OK;
}

// Frame::calcKeyPoints + calcDescriptors (frame.h:73-86), host-array mode
int extract(mvo_vo *v, VoFrame *f, const uint8_t *image, int channels, size_t stride, int on_device) {
  const int cap = v->ctx->prm.max_keypoints + 8;
  f->kpts.resize((size_t)cap);
  f->desc.resize((size_t)cap * 32);
  int n = cap;
  MVO_TRY(mvo_orb_extract_ex(v->ctx, image, v->rows, v->cols, channels, stride, on_device, f->kpts.data(), &n, f->desc.data()));
  f->kpts.resize((size_t)n);
  f->desc.resize((size_t)n * 32);
  f->xy.resize((size_t)n * 2);
  for (int i = 0; i < n; ++i) { f->xy[2 * i] = f->kpts[i].x; f->xy[2 * i + 1] = f->kpts[i].y; }
  const uint8_t *himg = nullptr;
  size_t hstride = 0;
  MVO_TRY(host_image(v, &himg, &hstride));
  sample_colors(f, himg, channels, hstride);
  return MVO_OK;
}

// device-resident mode: keypoints / descriptors of a frame whose extraction slot still holds it -> host
int ensure_host(mvo_vo *v, VoFrame *f) {
  if (f->host_ready) return MVO_OK;
  if (f->slot < 0 || mvo_trk_slot_serial(v->trk, f->slot) != f->serial)
    return mvo_fail(v->ctx, MVO_ERR_INVALID_ARG, "vo: frame %d has left the device (its keypoints are kept for two frames unless it is a keyframe)", f->id);
  f->kpts.resize((size_t)f->nk);
  f->desc.resize((size_t)f->nk * 32);
  f->colors.assign((size_t)f->nk * 3, 0);
  const bool cur = f == v->curr.get() && v->cur_image;
  // an image in device memory: the colours are gathered there (a few KB) instead of copying the image back
  MVO_TRY(mvo_trk_fetch(v->trk, f->slot, f->kpts.data(), f->desc.data(), cur && v->cur_on_device ? f->colors.data() : nullptr));
  f->xy.resize((size_t)f->nk * 2);
  for (int i = 0; i < f->nk; ++i) { f->xy[2 * i] = f->kpts[i].x; f->xy[2 * i + 1] = f->kpts[i].y; }
  if (cur && !v->cur_on_device) sample_colors(f, v->cur_image, v->cur_channels, v->cur_stride);
  f->host_ready = true;
  return MVO_OK;
}

// device-resident mode: inliers_to_mappt_connections_ of the k-th newest buffered frame -> host (insertion order = PnP inlier
// order, the order the host-array mode inserts them in, so the container order is the same)
int ensure_conn(mvo_vo *v, VoFrame *f, int k) {
  if (f->conn_ready) return MVO_OK;
  const int cap = v->ctx->prm.max_keypoints + 8;
  std::vector<int32_t> ids((size_t)cap), kp((size_t)cap);
  int n = 0;
  MVO_TRY(mvo_trk_links(v->trk, k, ids.data(), kp.data(), cap, &n));
  for (int i = 0; i < n; ++i) f->conn[kp[(size_t)i]] = PtConn{-1, ids[(size_t)i]};
  f->conn_ready = true;
  return MVO_OK;
}

// device-resident mode: the map in container order -> tracker (positions, descriptors, ids)
int upload_map(mvo_vo *v) {
  const size_t n = v->map_points.size();
  v->up_pts.resize(n * 3 + 3); v->up_desc.resize(n * 32 + 32); v->dev_order.resize(n);
  size_t k = 0;
  for (auto &kv : v->map_points) {
    const VoMapPoint &mp = kv.second;
    memcpy(&v->up_pts[3 * k], mp.pos, 12);
    memcpy(&v->up_desc[32 * k], mp.desc, 32);
    v->dev_order[k] = mp.id;
    ++k;
  }
  return mvo_trk_set_map_ids(v->trk, v->up_pts.data(), v->up_desc.data(), v->dev_order.data(), (int)n, 0);
}

// the increments of one keyframe fetch (positions = the order of the last upload) folded into the map
void fold_counters(mvo_vo *v, const int32_t *vis, const int32_t *matched, int n) {
  for (int k = 0; k < n && k < (int)v->dev_order.size(); ++k) {
    if (vis[k] == 0 && matched[k] == 0) continue;
    auto it = v->map_points.find(v->dev_order[(size_t)k]);
    if (it == v->map_points.end()) continue;
    it->second.visible_times += vis[k];
    it->second.matched_times += matched[k];
  }
}

// device-resident mode: a frame that did not go through the tracking step enters the tracker's frame buffer
int push_frame_to_tracker(mvo_vo *v, const VoFrame &f) {
  std::vector<int32_t> ids, kp;
  std::vector<float> obs;
  for (auto &kc : f.conn) {
    ids.push_back(kc.second.pt_map_idx);
    kp.push_back(kc.first);
    obs.push_back(f.xy[2 * (size_t)kc.first]); obs.push_back(f.xy[2 * (size_t)kc.first + 1]);
  }
  return mvo_trk_push_frame(v->trk, f.T_w_c, ids.data(), kp.data(), obs.data(), (int)ids.size());
}

void add_keyframe(mvo_vo *v, const FramePtr &f) {                // addKeyFrame_ (vo.cpp:482-486), Map::insertKeyFrame
  v->keyframes[f->id] = f;
  v->ref = f;
}

// retainGoodTriangulationResult_ (vo.cpp:181-244)
int retain_good_triangulation(mvo_vo *v) {
  VoFrame &c = *v->curr;
  const int n = (int)(c.inliers_pts3d.size() / 3);
  if (n == 0) return MVO_OK;
  v->keep.resize((size_t)n);
  v->angles.resize((size_t)n);
  int nk = 0;
  MVO_TRY(mvo_retain_good_triangulation(c.inliers_pts3d.data(), n, c.T_w_c, v->ref->T_w_c, v->prm.min_triang_angle,
                                        v->prm.max_ratio_angle_to_median, v->keep.data(), v->angles.data(), &nk));
  std::vector<float> kept((size_t)nk * 3);
  for (int i = 0; i < nk; ++i) {
    c.inliers_matches_for_3d.push_back(c.inliers_matches_with_ref[(size_t)v->keep[i]]);
    memcpy(&kept[3 * (size_t)i], &c.inliers_pts3d[3 * (size_t)v->keep[i]], 12);
    c.triangulation_angles.push_back(v->angles[i]);
  }
  c.inliers_pts3d.swap(kept);
  return MVO_OK;
}

// estimateMotionAnd3DPoints_ (vo.cpp:53-111).  *usable = 0 when the two-view problem is degenerate (see the file header).
int estimate_motion_and_3d_points(mvo_vo *v, mvo_vo_frame_info *info, int *usable) {
  VoFrame &c = *v->curr;
  const VoFrame &r = *v->ref;
  *usable = 0;
  const int n = (int)c.matches_with_ref.size();
  if (n < 8) return MVO_OK;
  v->p1.resize((size_t)n * 2); v->p2.resize((size_t)n * 2);
  for (int i = 0; i < n; ++i) {
    const mvo_dmatch &m = c.matches_with_ref[i];
    v->p1[2 * i] = r.xy[2 * m.query_idx]; v->p1[2 * i + 1] = r.xy[2 * m.query_idx + 1];
    v->p2[2 * i] = c.xy[2 * m.train_idx]; v->p2[2 * i + 1] = c.xy[2 * m.train_idx + 1];
  }
  mvo_two_view_solutions sol;
  v->inl.resize((size_t)5 * n);
  v->pts3d.resize((size_t)5 * n * 3);
  // the initialisation uses the configured findEssentialMat_threshold like the keyframe branch does (vo.cpp:60-70)
  const double saved_thr = v->ctx->prm.essential_threshold;
  v->ctx->prm.essential_threshold = v->prm.essential_threshold;
  const int rc = mvo_estimate_relative_poses(v->ctx, v->p1.data(), v->p2.data(), n, v->K, v->prm.init_calc_homography, 1, &sol,
                                             v->inl.data(), v->pts3d.data());
  v->ctx->prm.essential_threshold = saved_thr;
  if (rc == MVO_ERR_DEGENERATE) return MVO_OK;
  if (rc != MVO_OK) return rc;
  const int best = sol.best, ni = sol.n_inliers[best];
  info->best_sol = best;
  info->score_e = sol.score_e; info->score_h = sol.score_h; info->eh_ratio = sol.ratio;
  const double *R = sol.R[best];
  double t[3] = {sol.t[best][0], sol.t[best][1], sol.t[best][2]};
  const int32_t *inl = v->inl.data() + (size_t)best * n;
  const float *p3 = v->pts3d.data() + (size_t)best * n * 3;
  c.inliers_matches_with_ref.resize((size_t)ni);
  c.inliers_pts3d.resize((size_t)ni * 3);
  for (int i = 0; i < ni; ++i) {
    mvo_dmatch m = c.matches_with_ref[(size_t)inl[i]];
    m.img_idx = -1;                                              // cv::DMatch(queryIdx, trainIdx, distance) (motion_estimation.cpp:104-106)
    c.inliers_matches_with_ref[(size_t)i] = m;
    trans_coord(p3 + 3 * (size_t)i, R, t, &c.inliers_pts3d[3 * (size_t)i]);          // points in the current camera (vo.cpp:84-86)
  }
  double Trt[16], Tinv[16];
  rt_to_T(R, t, Trt);
  inv_rigid(Trt, Tinv);
  mul44(r.T_w_c, Tinv, c.T_w_c);                                 // vo.cpp:91
  MVO_TRY(retain_good_triangulation(v));
  *usable = 1;
  const int N = (int)(c.inliers_pts3d.size() / 3);
  if (N < 20) return MVO_OK;                                     // vo.cpp:97-101
  MVO_TRY(mvo_normalize_init_depth(c.inliers_pts3d.data(), N, t, v->prm.assumed_mean_depth_init, nullptr));     // :104-108
  rt_to_T(R, t, Trt);
  inv_rigid(Trt, Tinv);
  mul44(r.T_w_c, Tinv, c.T_w_c);                                 // :110
  return MVO_OK;
}

// isVoGoodToInit_ (vo.cpp:113-172)
int is_vo_good_to_init(mvo_vo *v, mvo_vo_frame_info *info, int *good) {
  VoFrame &c = *v->curr;
  const VoFrame &r = *v->ref;
  const int n = (int)c.inliers_matches_for_3d.size();
  v->p1.resize((size_t)std::max(n, 1) * 2); v->p2.resize((size_t)std::max(n, 1) * 2);
  for (int i = 0; i < n; ++i) {
    const mvo_dmatch &m = c.inliers_matches_for_3d[i];
    v->p1[2 * i] = r.xy[2 * m.query_idx]; v->p1[2 * i + 1] = r.xy[2 * m.query_idx + 1];
    v->p2[2 * i] = c.xy[2 * m.train_idx]; v->p2[2 * i + 1] = c.xy[2 * m.train_idx + 1];
  }
  info->n_inliers = n;
  const int na = (int)c.triangulation_angles.size();
  return mvo_is_vo_good_to_init(v->p1.data(), v->p2.data(), n, na ? c.triangulation_angles.data() : nullptr, na, v->prm.min_inlier_matches,
                                v->prm.min_pixel_dist, v->prm.min_median_triangulation_angle, good, &info->init_mean_pixel_dist,
                                &info->init_median_angle);
}

// pushCurrPointsToMap_ (vo.cpp:528-576)
void push_curr_points_to_map(mvo_vo *v) {
  VoFrame &c = *v->curr;
  VoFrame &r = *v->ref;
  const double cam[3] = {c.T_w_c[3], c.T_w_c[7], c.T_w_c[11]};   // Frame::getCamCenter
  const int n = (int)c.inliers_matches_for_3d.size();
  for (int i = 0; i < n; ++i) {
    const mvo_dmatch &dm = c.inliers_matches_for_3d[i];
    const int pt_idx = dm.train_idx;
    int map_point_id;
    auto it = r.conn.find(dm.query_idx);
    if (it != r.conn.end()) {
      map_point_id = it->second.pt_map_idx;                      // triangulated before: reuse (vo.cpp:548-551)
    } else {
      VoMapPoint mp;
      pre_translate(&c.inliers_pts3d[3 * (size_t)i], c.T_w_c, mp.pos);
      double d[3] = {(double)mp.pos[0] - cam[0], (double)mp.pos[1] - cam[1], (double)mp.pos[2] - cam[2]};
      const double len = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);        // basics::getNormalizedMat
      for (int q = 0; q < 3; ++q) mp.norm[q] = d[q] / len;
      memcpy(mp.desc, &c.desc[(size_t)pt_idx * 32], 32);
      memcpy(mp.rgb, &c.colors[(size_t)pt_idx * 3], 3);
      mp.id = v->point_factory_id++;
      map_point_id = mp.id;
      v->map_points[mp.id] = mp;                                 // Map::insertMapPoint
    }
    if (c.conn.insert({pt_idx, PtConn{dm.query_idx, map_point_id}}).second && v->dev) {
      v->new_ids.push_back(map_point_id);
      v->new_kp.push_back(pt_idx);
      v->new_obs.push_back(c.xy[2 * (size_t)pt_idx]); v->new_obs.push_back(c.xy[2 * (size_t)pt_idx + 1]);
    }
  }
}

// the test of Frame::isInFrame (frame.cpp:31-38) and getMappointsInCurrentView_ (vo.cpp:28-36)
bool project_in_frame(const mvo_vo *v, const double *T_c_w, const float *pos, float *u, float *w) {
  float pc[3];
  pre_translate(pos, T_c_w, pc);
  if (pc[2] < 0) return false;
  *u = (float)(v->K[0] * pc[0] / pc[2] + v->K[2]);               // geometry::cam2pixel (camera.cpp:23-28)
  *w = (float)(v->K[4] * pc[1] / pc[2] + v->K[5]);
  return *u > 0 && *w > 0 && *u < (float)v->cols && *w < (float)v->rows;
}

// optimizeMap_ (vo.cpp:488-526)
void optimize_map(mvo_vo *v) {
  const VoFrame &c = *v->curr;
  double Tcw[16];
  inv_rigid(c.T_w_c, Tcw);
  const double cam[3] = {c.T_w_c[3], c.T_w_c[7], c.T_w_c[11]};
  for (auto it = v->map_points.begin(); it != v->map_points.end();) {
    const VoMapPoint &mp = it->second;
    float u, w;
    if (!project_in_frame(v, Tcw, mp.pos, &u, &w)) { it = v->map_points.erase(it); continue; }
    const float match_ratio = float(mp.matched_times) / mp.visible_times;
    if (match_ratio < v->map_point_erase_ratio) { it = v->map_points.erase(it); continue; }
    double d[3] = {(double)mp.pos[0] - cam[0], (double)mp.pos[1] - cam[1], (double)mp.pos[2] - cam[2]};        // getViewAngle_ (vo.cpp:578-584)
    const double len = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    // angle = acos(x) > pi/4 (vo.cpp:515-519).  acos is monotonic, so the comparison is decided by x against cos(pi/4) except in a
    // 1e-12 band around it (and for |x| > 1, where acos is NaN and the reference keeps the point): only there acos is evaluated
    const double x = d[0] / len * mp.norm[0] + d[1] / len * mp.norm[1] + d[2] / len * mp.norm[2];
    const double cq = 0.70710678118654752440;
    bool too_oblique;
    if (x >= -1.0 && x < cq - 1e-12) too_oblique = true;
    else if (x > cq + 1e-12) too_oblique = false;
    else too_oblique = acos(x) > M_PI / 4.;
    if (too_oblique) { it = v->map_points.erase(it); continue; }
    ++it;
  }
  if (v->map_points.size() > 1000) v->map_point_erase_ratio += 0.05;
  else v->map_point_erase_ratio = 0.1;
}

// poseEstimationPnP_ (vo.cpp:267-381)
int pose_estimation_pnp(mvo_vo *v, mvo_vo_frame_info *info, bool *good) {
  VoFrame &c = *v->curr;
  // getMappointsInCurrentView_ (vo.cpp:16-49): container order
  double Tcw[16];
  inv_rigid(c.T_w_c, Tcw);
  const size_t nmap = v->map_points.size();
  v->cand_id.clear(); v->cand_xy.clear(); v->cand_desc.clear();
  v->cand_id.reserve(nmap); v->cand_xy.reserve(nmap * 2); v->cand_desc.reserve(nmap * 32);
  for (auto &kv : v->map_points) {
    VoMapPoint &mp = kv.second;
    float u, w;
    if (!project_in_frame(v, Tcw, mp.pos, &u, &w)) continue;
    v->cand_id.push_back(mp.id);
    v->cand_xy.push_back(u); v->cand_xy.push_back(w);
    v->cand_desc.insert(v->cand_desc.end(), mp.desc, mp.desc + 32);
    mp.visible_times++;
  }
  const int nc = (int)v->cand_id.size();
  info->n_candidates = nc;
  MVO_TRY(match_into(v, v->cand_desc.data(), v->cand_xy.data(), nc, c, v->prm.track.match_method, v->prm.track.match_radius, &c.matches_with_map));
  const int nm = (int)c.matches_with_map.size();
  info->n_matches = nm;
  v->p3d.resize((size_t)std::max(nm, 1) * 3); v->p2d.resize((size_t)std::max(nm, 1) * 2);
  for (int i = 0; i < nm; ++i) {                                 // vo.cpp:293-301
    const mvo_dmatch &m = c.matches_with_map[i];
    memcpy(&v->p3d[3 * (size_t)i], v->map_points[v->cand_id[(size_t)m.query_idx]].pos, 12);
    v->p2d[2 * i] = c.xy[2 * m.train_idx]; v->p2d[2 * i + 1] = c.xy[2 * m.train_idx + 1];
  }
  bool ok = nm >= v->prm.track.min_pnp_points;
  if (ok) {
    double rvec[3], tvec[3];
    v->inl.resize((size_t)nm);
    int ni = nm;
    const int rc = mvo_solve_pnp_ransac(v->ctx, v->p3d.data(), v->p2d.data(), nm, v->K, rvec, tvec, v->inl.data(), &ni);
    if (rc == MVO_ERR_DEGENERATE) ok = false;
    else if (rc != MVO_OK) return rc;
    if (ok) {
      std::vector<mvo_dmatch> kept((size_t)ni);
      for (int i = 0; i < ni; ++i) {                             // vo.cpp:333-354
        const mvo_dmatch &m = c.matches_with_map[(size_t)v->inl[i]];
        kept[(size_t)i] = m;
        VoMapPoint &mp = v->map_points[v->cand_id[(size_t)m.query_idx]];
        mp.matched_times++;
        c.conn[m.train_idx] = PtConn{-1, mp.id};
      }
      c.matches_with_map.swap(kept);
      info->n_inliers = ni;
      double R[9], Tc[16];
      rodrigues_to_R(rvec, R);
      rt_to_T(R, tvec, Tc);
      inv_rigid(Tc, c.T_w_c);                                  // vo.cpp:357
      if (trans_dist(c.T_w_c, v->prev->T_w_c) >= v->prm.track.max_dist_to_prev) ok = false;      // vo.cpp:360-369
    }
  }
  if (!ok) memcpy(c.T_w_c, v->prev->T_w_c, sizeof c.T_w_c);      // vo.cpp:376-379
  info->pnp_ok = ok;
  memcpy(info->T_w_c_pnp, c.T_w_c, sizeof c.T_w_c);
  *good = ok;
  return MVO_OK;
}

// callBundleAdjustment_ (vo.cpp:384-478)
int call_bundle_adjustment(mvo_vo *v, mvo_vo_frame_info *info) {
  const mvo_track_params &tp = v->prm.track;
  if (!tp.ba_enable) return MVO_OK;
  const int total = (int)v->buff.size();
  const int nba = std::min(tp.ba_window, total - 1);
  std::vector<VoFrame *> sel;
  v->ba_ef.clear(); v->ba_ep.clear(); v->ba_ob.clear(); v->ba_poses.clear(); v->ba_used.clear();
  std::unordered_map<int, int> slot;                             // map point id -> vertex (um_pts_3d_in_prev_frames)
  for (int b = total - 1; b >= total - nba; --b) {               // newest first (vo.cpp:417-419)
    VoFrame &f = *v->buff[(size_t)b];
    if ((int)f.conn.size() < 3) continue;                        // vo.cpp:423-426
    const int fi = (int)sel.size();
    sel.push_back(&f);
    v->ba_poses.insert(v->ba_poses.end(), f.T_w_c, f.T_w_c + 16);
    for (auto &kc : f.conn) {                                    // container order (vo.cpp:435-452)
      const int mappt_idx = kc.second.pt_map_idx;
      auto mit = v->map_points.find(mappt_idx);
      if (mit == v->map_points.end()) continue;                  // point has been deleted
      auto s = slot.find(mappt_idx);
      int vid;
      if (s == slot.end()) { vid = (int)v->ba_used.size(); slot[mappt_idx] = vid; v->ba_used.push_back(mappt_idx); }
      else vid = s->second;
      v->ba_ef.push_back(fi);
      v->ba_ep.push_back(vid);
      v->ba_ob.push_back(f.xy[2 * (size_t)kc.first]);
      v->ba_ob.push_back(f.xy[2 * (size_t)kc.first + 1]);
    }
  }
  if (sel.empty() || v->ba_ef.empty()) return MVO_OK;
  v->ba_pts.resize(v->ba_used.size() * 3);
  for (size_t k = 0; k < v->ba_used.size(); ++k) memcpy(&v->ba_pts[3 * k], v->map_points[v->ba_used[k]].pos, 12);
  const int fix = tp.ba_fix_points ? 1 : 0;
  const double saved_tol = v->ctx->prm.ba_step_tol;
  v->ctx->prm.ba_step_tol = tp.ba_step_tol;
  const int rc = mvo_bundle_adjustment(v->ctx, v->ba_poses.data(), (int)sel.size(), v->ba_pts.data(), (int)v->ba_used.size(), v->ba_ef.data(),
                                       v->ba_ep.data(), v->ba_ob.data(), (int)v->ba_ef.size(), v->K, tp.information, fix, !fix, nullptr);
  v->ctx->prm.ba_step_tol = saved_tol;
  if (rc != MVO_OK) return rc;
  for (size_t k = 0; k < sel.size(); ++k) memcpy(sel[k]->T_w_c, &v->ba_poses[16 * k], 16 * sizeof(double));
  if (!fix)
    for (size_t k = 0; k < v->ba_used.size(); ++k) memcpy(v->map_points[v->ba_used[k]].pos, &v->ba_pts[3 * k], 12);
  info->ba_frames = (int)sel.size();
  info->ba_edges = (int)v->ba_ef.size();
  return MVO_OK;
}

// device-resident mode: keypoints / descriptors / colours of a one-submission fetch become the frame's host copy
void adopt_fetched(mvo_vo *v, VoFrame *f, const MvoKfFetch &kf) {
  if (f->host_ready) return;
  const bool cur = f == v->curr.get() && v->cur_image;
  f->kpts.assign(kf.kpts, kf.kpts + kf.n_kpts);
  f->desc.assign(kf.desc, kf.desc + (size_t)kf.n_kpts * 32);
  f->xy.resize((size_t)kf.n_kpts * 2);
  for (int i = 0; i < kf.n_kpts; ++i) { f->xy[2 * i] = f->kpts[(size_t)i].x; f->xy[2 * i + 1] = f->kpts[(size_t)i].y; }
  if (kf.rgb) f->colors.assign(kf.rgb, kf.rgb + (size_t)kf.n_kpts * 3);
  else { f->colors.assign((size_t)kf.n_kpts * 3, 0); if (cur) sample_colors(f, v->cur_image, v->cur_channels, v->cur_stride); }
  f->host_ready = true;
}

// the keyframe branch of addFrame (vo_addFrame.cpp:93-124)
int insert_keyframe(mvo_vo *v, mvo_vo_frame_info *info) {
  VoFrame &c = *v->curr;
  const VoFrame &r = *v->ref;
  StageClock clk;
  const int method = v->prm.track.match_method;
  bool matched = false;
  if (v->dev) {
    // the frame's keypoints, descriptors, colours and connections, the visible / matched increments and the match against the
    // reference keyframe (whose descriptors stayed on the device): one submission, one synchronisation
    MvoKfFetch kf;
    const bool cur = v->cur_image != nullptr;
    MVO_TRY(mvo_trk_keyframe_fetch(v->trk, c.slot, cur && v->cur_on_device, 1, (int)v->dev_order.size(), r.id,
                                   method == 1 ? 0 : (method == 2 ? 1 : -1), &kf));
    adopt_fetched(v, &c, kf);
    if (!c.conn_ready) {
      for (int i = 0; i < kf.n_links; ++i) c.conn[kf.link_kp[i]] = PtConn{-1, kf.link_ids[i]};
      c.conn_ready = true;
    }
    fold_counters(v, kf.vis, kf.matched, kf.n_counters);          // visible_times_ / matched_times_ as of this frame
    clk.mark("fetch+match");
    if (kf.n_ref > 0 && kf.n_ref == r.n()) {
      c.matches_with_ref.resize((size_t)kf.n_ref);
      int nm = 0;
      MVO_TRY(mvo_match_filter_keys(v->ctx, method, kf.keys, kf.n_ref, c.matches_with_ref.data(), &nm));
      c.matches_with_ref.resize((size_t)nm);
      matched = true;
    }
  }
  if (!matched) MVO_TRY(match_into(v, r.desc.data(), r.xy.data(), r.n(), c, method, v->prm.max_match_dist_triangulation, &c.matches_with_ref));
  clk.mark("match");
  const int n = (int)c.matches_with_ref.size();
  info->kf_matches = n;
  if (n < 8) return MVO_OK;                                      // see the file header
  v->p1.resize((size_t)n * 2); v->p2.resize((size_t)n * 2);
  for (int i = 0; i < n; ++i) {
    const mvo_dmatch &m = c.matches_with_ref[i];
    v->p1[2 * i] = r.xy[2 * m.query_idx]; v->p1[2 * i + 1] = r.xy[2 * m.query_idx + 1];
    v->p2[2 * i] = c.xy[2 * m.train_idx]; v->p2[2 * i + 1] = c.xy[2 * m.train_idx + 1];
  }
  // helperTriangulatePoints with the known motion getMotionFromFrame1to2(curr_, ref_) = curr^-1 * ref (vo_commons.cpp:9-15)
  double Tci[16], T[16], R[9], t[3];
  inv_rigid(c.T_w_c, Tci);
  mul44(Tci, r.T_w_c, T);
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[i * 3 + j] = T[i * 4 + j]; t[i] = T[i * 4 + 3]; }
  auto to_norm_plane = [&](const mvo_dmatch &m, float *a, float *b) {        // pixel2CamNormPlane (camera.cpp:10-15)
    a[0] = (float)(((double)r.xy[2 * m.query_idx] - v->K[2]) / v->K[0]); a[1] = (float)(((double)r.xy[2 * m.query_idx + 1] - v->K[5]) / v->K[4]);
    b[0] = (float)(((double)c.xy[2 * m.train_idx] - v->K[2]) / v->K[0]); b[1] = (float)(((double)c.xy[2 * m.train_idx + 1] - v->K[5]) / v->K[4]);
  };
  // helperFindInlierMatchesByEpipolarCons (motion_estimation.cpp:180-196): the inliers of the essential-matrix RANSAC.  The
  // reference passes dummy R / t here, so only the consensus set is computed; in device-resident mode the triangulation of every
  // correspondence (its motion is known beforehand) rides in the same submission and the inliers' rows are picked below.
  double E[9], Re[9], te[3];
  v->inl.resize((size_t)n);
  int ni = n;
  int rc;
  if (v->dev) {
    v->np1.resize((size_t)n * 2); v->np2.resize((size_t)n * 2);
    for (int i = 0; i < n; ++i) to_norm_plane(c.matches_with_ref[(size_t)i], &v->np1[2 * (size_t)i], &v->np2[2 * (size_t)i]);
    v->tri_all.resize((size_t)n * 3);
    rc = mvo_epi_essential_ex(v->ctx, v->p1.data(), v->p2.data(), n, v->K, v->prm.essential_threshold, E, Re, te, v->inl.data(), &ni, 0,
                              v->np1.data(), v->np2.data(), R, t, v->tri_all.data());
  } else {
    rc = mvo_esti_motion_by_essential(v->ctx, v->p1.data(), v->p2.data(), n, v->K, v->prm.essential_threshold, E, Re, te, v->inl.data(), &ni);
  }
  if (rc == MVO_ERR_DEGENERATE) return MVO_OK;
  if (rc != MVO_OK) return rc;
  clk.mark("essential");
  c.inliers_matches_with_ref.resize((size_t)ni);
  for (int i = 0; i < ni; ++i) {
    mvo_dmatch m = c.matches_with_ref[(size_t)v->inl[i]];
    m.img_idx = -1;
    c.inliers_matches_with_ref[(size_t)i] = m;
  }
  v->pts3d.resize((size_t)std::max(ni, 1) * 3);
  if (v->dev) {
    for (int i = 0; i < ni; ++i) memcpy(&v->pts3d[3 * (size_t)i], &v->tri_all[3 * (size_t)v->inl[i]], 12);
  } else {
    v->np1.resize((size_t)ni * 2); v->np2.resize((size_t)ni * 2);
    for (int i = 0; i < ni; ++i) to_norm_plane(c.inliers_matches_with_ref[(size_t)i], &v->np1[2 * (size_t)i], &v->np2[2 * (size_t)i]);
    std::vector<int32_t> all((size_t)ni);
    for (int i = 0; i < ni; ++i) all[(size_t)i] = i;
    if (ni > 0) MVO_TRY(mvo_do_triangulation(v->ctx, v->np1.data(), v->np2.data(), ni, R, t, all.data(), ni, v->pts3d.data()));
  }
  c.inliers_pts3d.resize((size_t)ni * 3);
  for (int i = 0; i < ni; ++i) trans_coord(&v->pts3d[3 * (size_t)i], R, t, &c.inliers_pts3d[3 * (size_t)i]);
  clk.mark("triangulate");
  MVO_TRY(retain_good_triangulation(v));
  info->kf_new_points = (int)c.inliers_matches_for_3d.size();
  v->new_ids.clear(); v->new_kp.clear(); v->new_obs.clear();
  push_curr_points_to_map(v);
  clk.mark("retain+push");
  optimize_map(v);
  clk.mark("optimize_map");
  if (v->dev) {
    MVO_TRY(mvo_trk_set_ref_desc(v->trk, c.slot, c.id));         // this frame is the reference keyframe from now on
    MVO_TRY(upload_map(v));
    MVO_TRY(mvo_trk_append_links(v->trk, 0, v->new_ids.data(), v->new_kp.data(), v->new_obs.data(), (int)v->new_ids.size()));
  }
  clk.mark("upload");
  add_keyframe(v, v->curr);
  info->keyframe = 1;
  clk.report("keyframe", c.id);
  return MVO_OK;
}

}  // namespace

extern "C" {

void mvo_vo_default_params(mvo_vo_params *p) {
  if (!p) return;
  memset(p, 0, sizeof *p);
  mvo_default_track_params(&p->track);
  p->match_method_init = 1;                  // feature_match_method_index_initialization (config.yaml)
  p->max_match_dist_init = 100.f;            // max_matching_pixel_dist_in_initialization
  p->max_match_dist_triangulation = 100.f;   // max_matching_pixel_dist_in_triangulation
  p->essential_threshold = 1.0;              // findEssentialMat_threshold
  p->init_calc_homography = 1;               // is_calc_homo = true (vo.cpp:68)
  p->min_inlier_matches = 15;
  p->min_triang_angle = 1.0;
  p->max_ratio_angle_to_median = 20.0;       // max_ratio_between_max_angle_and_median_angle
  p->min_pixel_dist = 50.0;
  p->min_median_triangulation_angle = 2.0;
  p->assumed_mean_depth_init = 0.8;          // assumed_mean_pts_depth_during_vo_init
}

int mvo_vo_create(mvo_ctx *ctx, const double *K, int rows, int cols, const mvo_vo_params *params, mvo_vo **out) {
  if (!ctx || !out) return MVO_ERR_INVALID_ARG;
  *out = nullptr;
  if (!K || rows <= 0 || cols <= 0) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo: bad K / image size");
  mvo_vo_params p;
  if (params) p = *params; else mvo_vo_default_params(&p);
  if (p.match_method_init < 1 || p.match_method_init > 3 || p.track.match_method < 1 || p.track.match_method > 3 || p.track.ba_window < 1 ||
      p.track.ba_window > 16 || p.track.buffer_size < 2 || !(p.track.ba_step_tol >= 0))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo: bad parameters");
  mvo_vo *v = new mvo_vo();
  v->ctx = ctx;
  v->prm = p;
  memcpy(v->K, K, sizeof v->K);
  v->rows = rows; v->cols = cols;
  if (p.track.device_resident) {
    const int rc = mvo_tracker_create(ctx, K, rows, cols, &p.track, &v->trk);
    if (rc != MVO_OK) { delete v; return rc; }
    v->dev = mvo_trk_device_mode(v->trk) != 0;                   // fixed map points and a BA window the cluster kernel holds
    if (v->dev) mvo_trk_configure(v->trk, 1, 1);
    else { mvo_tracker_destroy(v->trk); v->trk = nullptr; }
  }
  *out = v;
  return MVO_OK;
}

void mvo_vo_destroy(mvo_vo *v) {
  if (!v) return;
  if (v->trk) mvo_tracker_destroy(v->trk);
  delete v;
}

int mvo_vo_device_resident(const mvo_vo *v) { return v && v->dev ? 1 : 0; }

int mvo_vo_reset(mvo_vo *v) {
  if (!v) return MVO_ERR_INVALID_ARG;
  v->state = VO_BLANK;
  std::unordered_map<int, VoMapPoint>().swap(v->map_points);     // fresh containers: the iteration order depends on the bucket history
  std::unordered_map<int, FramePtr>().swap(v->keyframes);
  v->buff.clear();
  v->curr.reset(); v->prev.reset(); v->ref.reset(); v->prev_ref.reset();
  v->frame_factory_id = v->point_factory_id = 0;
  v->map_point_erase_ratio = 0.1;
  v->dev_order.clear();
  if (v->trk) {
    double I[16];
    set_identity(I);
    MVO_TRY(mvo_tracker_reset(v->trk, I));
    MVO_TRY(mvo_trk_set_map_ids(v->trk, nullptr, nullptr, nullptr, 0, 1));
  }
  return MVO_OK;
}

int mvo_vo_prefetch(mvo_vo *v, const uint8_t *image, int channels, size_t stride, int image_on_device) {
  if (!v) return MVO_ERR_INVALID_ARG;
  if (!image || (channels != 1 && channels != 3) || stride < (size_t)v->cols * channels)
    return mvo_fail(v->ctx, MVO_ERR_INVALID_ARG, "vo: bad image arguments");
  if (!v->dev) return MVO_OK;                                    // host-array mode extracts inside add_frame
  return mvo_tracker_prefetch(v->trk, image, channels, stride, image_on_device);
}

uint64_t mvo_vo_kernel_launches(const mvo_vo *v) {
  if (!v) return 0;
  return v->trk ? mvo_tracker_kernel_launches(v->trk) : mvo_kernel_launches(v->ctx);
}

int mvo_vo_timing_enable(mvo_vo *v, uint32_t mask) {
  if (!v) return MVO_ERR_INVALID_ARG;
  return v->trk ? mvo_tracker_timing_enable(v->trk, mask) : mvo_timing_enable(v->ctx, mask);
}

int mvo_vo_timing_read(mvo_vo *v, double *ms, uint64_t *counts) {
  if (!v) return MVO_ERR_INVALID_ARG;
  return v->trk ? mvo_tracker_timing_read(v->trk, ms, counts) : mvo_timing_read(v->ctx, ms, counts);
}

int mvo_vo_add_frame(mvo_vo *v, const uint8_t *image, int channels, size_t stride, double *T_w_c_out, mvo_vo_frame_info *info_out) {
  return mvo_vo_add_frame_ex(v, image, channels, stride, 0, T_w_c_out, info_out);
}

int mvo_vo_add_frame_ex(mvo_vo *v, const uint8_t *image, int channels, size_t stride, int image_on_device, double *T_w_c_out,
                        mvo_vo_frame_info *info_out) {
  if (!v) return MVO_ERR_INVALID_ARG;
  if (!image || (channels != 1 && channels != 3) || stride < (size_t)v->cols * channels)
    return mvo_fail(v->ctx, MVO_ERR_INVALID_ARG, "vo: bad image arguments");
  mvo_vo_frame_info info;
  memset(&info, 0, sizeof info);
  info.best_sol = -1;
  FramePtr frame = std::make_shared<VoFrame>();
  frame->id = v->frame_factory_id;
  set_identity(frame->T_w_c);
  v->cur_image = image; v->cur_channels = channels; v->cur_stride = stride; v->cur_on_device = image_on_device;
  v->img_scratch.clear();
  // Frame::calcKeyPoints + calcDescriptors, before any state changes: an extraction error leaves the VO untouched
  int slot = -1;
  if (v->dev) {
    MVO_TRY(mvo_trk_acquire(v->trk, image, channels, stride, image_on_device, &slot, &frame->nk));
    frame->host_ready = false;
    frame->slot = slot;
    frame->serial = mvo_trk_slot_serial(v->trk, slot);
  } else {
    MVO_TRY(extract(v, frame.get(), image, channels, stride, image_on_device));
  }
  struct Release { mvo_vo *v; int slot; ~Release() { if (slot >= 0) mvo_trk_release(v->trk, slot); v->cur_image = nullptr; } } release{v, slot};
  v->frame_factory_id++;
  v->buff.push_back(frame);                                      // pushFrameToBuff_ (vo.h:81-86)
  if ((int)v->buff.size() > v->prm.track.buffer_size) v->buff.pop_front();
  v->curr = frame;
  info.frame_id = frame->id;
  info.state_in = v->state;
  info.n_keypoints = frame->n();
  v->prev_ref = v->ref;
  int rc = MVO_OK;
  if (v->state == VO_BLANK) {                                    // vo_addFrame.cpp:29-34
    if (v->dev) rc = ensure_host(v, frame.get());
    if (rc == MVO_OK) {
      v->state = VO_DOING_INITIALIZATION;
      add_keyframe(v, frame);
      info.keyframe = 1;
      if (v->dev) rc = mvo_trk_set_ref_desc(v->trk, slot, frame->id);
      if (rc == MVO_OK && v->dev) rc = push_frame_to_tracker(v, *frame);
    }
  } else if (v->state == VO_DOING_INITIALIZATION) {              // :35-69
    const VoFrame &r = *v->ref;
    bool matched = false;
    const int mi = v->prm.match_method_init;
    if (v->dev) {                       // the frame's host copy and its match against the first keyframe in one synchronisation
      MvoKfFetch kf;
      rc = mvo_trk_keyframe_fetch(v->trk, slot, v->cur_on_device, 0, 0, r.id, mi == 1 ? 0 : (mi == 2 ? 1 : -1), &kf);
      if (rc == MVO_OK) {
        adopt_fetched(v, frame.get(), kf);
        if (kf.n_ref > 0 && kf.n_ref == r.n()) {
          frame->matches_with_ref.resize((size_t)kf.n_ref);
          int nm = 0;
          rc = mvo_match_filter_keys(v->ctx, mi, kf.keys, kf.n_ref, frame->matches_with_ref.data(), &nm);
          frame->matches_with_ref.resize((size_t)nm);
          matched = rc == MVO_OK;
        }
      }
    }
    if (rc == MVO_OK && !matched)
      rc = match_into(v, r.desc.data(), r.xy.data(), r.n(), *frame, mi, v->prm.max_match_dist_init, &frame->matches_with_ref);
    int usable = 0, good = 0;
    if (rc == MVO_OK) { info.n_matches = (int)frame->matches_with_ref.size(); rc = estimate_motion_and_3d_points(v, &info, &usable); }
    if (rc == MVO_OK && usable) rc = is_vo_good_to_init(v, &info, &good);
    if (rc == MVO_OK && good) {
      v->new_ids.clear(); v->new_kp.clear(); v->new_obs.clear();
      push_curr_points_to_map(v);
      add_keyframe(v, frame);
      v->state = VO_DOING_TRACKING;
      info.keyframe = 1;
      if (v->dev) rc = mvo_trk_set_ref_desc(v->trk, slot, frame->id);
      if (rc == MVO_OK && v->dev) rc = upload_map(v);
    } else {
      memcpy(frame->T_w_c, v->ref->T_w_c, sizeof frame->T_w_c);  // :64-68
    }
    if (rc == MVO_OK && v->dev) rc = push_frame_to_tracker(v, *frame);
  } else if (v->state == VO_DOING_TRACKING && v->dev) {          // :70-125 through the device-resident tracker
    frame->conn_ready = false;
    mvo_track_result r;
    // where the reference keyframe sits in the frame buffer (this frame = 0), and whether this frame is likely to become a keyframe
    // (then the tracker does not enqueue the next frame's chain head ahead of time: the keyframe would invalidate it)
    int ref_k = -1;
    for (int k = 1; k < (int)v->buff.size(); ++k)
      if (v->buff[v->buff.size() - 1 - (size_t)k] == v->ref) { ref_k = k; break; }
    int allow_spec = 0;
    {
      const double d_prev = trans_dist(v->prev->T_w_c, v->ref->T_w_c);
      const double step = v->buff.size() >= 3 ? trans_dist(v->prev->T_w_c, v->buff[v->buff.size() - 3]->T_w_c) : 0.0;
      allow_spec = d_prev + 1.1 * step < v->prm.track.min_dist_keyframe;
    }
    rc = mvo_trk_track(v->trk, slot, v->ref->T_w_c, v->prev->T_w_c, frame->T_w_c, &r, ref_k, allow_spec);
    if (rc != MVO_OK) {                                          // the tracker has dropped the frame again: so do we
      v->buff.pop_back();
      v->curr = v->prev;
      v->frame_factory_id--;
      return rc;
    }
    info.n_candidates = r.n_candidates; info.n_matches = r.n_matches; info.n_inliers = r.n_inliers; info.pnp_ok = r.pnp_ok;
    info.ba_frames = r.ba_frames; info.ba_edges = r.ba_edges;
    memcpy(info.T_w_c_pnp, r.T_w_c_pnp, sizeof info.T_w_c_pnp);
    // bundle adjustment has moved the newest frames of the buffer (g2o_ba.cpp:298-305 writes the poses back in place)
    const int total = (int)v->buff.size(), nba = r.ba_frames > 0 ? std::min(v->prm.track.ba_window, total - 1) : 0;
    for (int k = 1; k < nba && rc == MVO_OK; ++k) rc = mvo_tracker_frame_pose(v->trk, k, v->buff[(size_t)(total - 1 - k)]->T_w_c);
    if (rc == MVO_OK && r.pnp_ok) {
      int large = 0;
      rc = mvo_check_large_move(frame->T_w_c, v->ref->T_w_c, v->prm.track.min_dist_keyframe, &large, nullptr, nullptr);
      if (rc == MVO_OK && large) rc = insert_keyframe(v, &info);
    }
  } else if (v->state == VO_DOING_TRACKING) {                    // :70-125, host arrays
    memcpy(frame->T_w_c, v->ref->T_w_c, sizeof frame->T_w_c);
    bool pnp_good = false;
    rc = pose_estimation_pnp(v, &info, &pnp_good);
    if (rc == MVO_OK && pnp_good) {
      rc = call_bundle_adjustment(v, &info);
      int large = 0;
      if (rc == MVO_OK) rc = mvo_check_large_move(frame->T_w_c, v->ref->T_w_c, v->prm.track.min_dist_keyframe, &large, nullptr, nullptr);
      if (rc == MVO_OK && large) rc = insert_keyframe(v, &info);
    }
  }
  if (rc != MVO_OK && !info.keyframe && !v->buff.empty() && v->buff.back() == frame) {
    // a stage failed (a CUDA error, an unsupported size): the frame leaves the buffer again, in both modes, so that
    // mvo_vo_frame_pose(k) keeps addressing the frames whose mvo_vo_add_frame call succeeded
    v->buff.pop_back();
    v->curr = v->prev;
    v->frame_factory_id--;
    return rc;
  }
  v->prev = frame;                                               // :141
  info.state_out = v->state;
  info.map_points = (int)v->map_points.size();
  if (T_w_c_out) memcpy(T_w_c_out, frame->T_w_c, 16 * sizeof(double));
  if (info_out) *info_out = info;
  return rc;
}

// run_vo.cpp:107-140 over images in memory (see mvo.h)
int mvo_vo_run_sequence(mvo_vo *v, const uint8_t *const *images, int n_frames, int channels, size_t stride, int images_on_device,
                        double *T_w_c_out, mvo_vo_frame_info *infos, int *n_done) {
  if (!v) return MVO_ERR_INVALID_ARG;
  if (n_done) *n_done = 0;
  if (n_frames < 0 || (n_frames > 0 && (!images || !T_w_c_out))) return mvo_fail(v->ctx, MVO_ERR_INVALID_ARG, "vo: bad sequence arguments");
  for (int i = 0; i < n_frames; ++i)
    if (!images[i]) return mvo_fail(v->ctx, MVO_ERR_INVALID_ARG, "vo: image %d is null", i);
  // two frames of look-ahead when the device-resident tracker extracts them (its extraction contexts work side by side): frame i
  // is added while frames i + 1 and i + 2 are in flight (three extraction slots: one held by the frame being added)
  const int ahead = v->dev ? 2 : 1;
  for (int k = 0; k <= ahead && k < n_frames; ++k) MVO_TRY(mvo_vo_prefetch(v, images[k], channels, stride, images_on_device));
  for (int i = 0; i < n_frames; ++i) {
    MVO_TRY(mvo_vo_add_frame_ex(v, images[i], channels, stride, images_on_device, T_w_c_out + 16 * (size_t)i, infos ? infos + i : nullptr));
    if (i + ahead + 1 < n_frames) MVO_TRY(mvo_vo_prefetch(v, images[i + ahead + 1], channels, stride, images_on_device));
    if (n_done) *n_done = i + 1;
  }
  return MVO_OK;
}

int mvo_vo_is_initialized(const mvo_vo *v) { return v && v->state == VO_DOING_TRACKING; }      // vo.cpp:174-177
int mvo_vo_map_size(const mvo_vo *v) { return v ? (int)v->map_points.size() : 0; }
int mvo_vo_num_keyframes(const mvo_vo *v) { return v ? (int)v->keyframes.size() : 0; }

int mvo_vo_get_map(const mvo_vo *v, int32_t *ids, float *pts3d, uint8_t *desc, uint8_t *rgb, int cap, int *n) {
  if (!v || !n) return MVO_ERR_INVALID_ARG;
  *n = (int)v->map_points.size();
  if (cap < *n) return MVO_ERR_CAPACITY;
  int k = 0;
  for (auto &kv : v->map_points) {                               // container order, as getMappointsInCurrentView_ walks it
    const VoMapPoint &mp = kv.second;
    if (ids) ids[k] = mp.id;
    if (pts3d) memcpy(pts3d + 3 * (size_t)k, mp.pos, 12);
    if (desc) memcpy(desc + 32 * (size_t)k, mp.desc, 32);
    if (rgb) memcpy(rgb + 3 * (size_t)k, mp.rgb, 3);
    ++k;
  }
  return MVO_OK;
}

int mvo_vo_has_keyframe(const mvo_vo *v, int frame_id) { return v && v->keyframes.count(frame_id) ? 1 : 0; }      // Map::hasKeyFrame

int mvo_vo_frame_data(const mvo_vo *v, int which, int what, void *out, int cap, int *n) {
  if (!v || !n) return MVO_ERR_INVALID_ARG;
  const VoFrame *f = nullptr;
  if (which == -1) f = v->prev_ref.get();                        // VisualOdometry::getPrevRef
  else if (which >= 0 && which < (int)v->buff.size()) f = v->buff[v->buff.size() - 1 - (size_t)which].get();
  if (!f) return MVO_ERR_INVALID_ARG;
  if (v->dev && (!f->host_ready || !f->conn_ready) && what != MVO_VO_FRAME_ID && which >= 0) {
    // device-resident mode: a tracked frame's keypoints / descriptors / PnP inliers are brought over on request
    mvo_vo *mv = const_cast<mvo_vo *>(v);
    VoFrame *mf = const_cast<VoFrame *>(f);
    if (what == MVO_VO_KEYPOINTS || what == MVO_VO_DESCRIPTORS) MVO_TRY(ensure_host(mv, mf));
    if (what == MVO_VO_MATCHES_WITH_MAP && mf->matches_with_map.empty()) {
      MVO_TRY(ensure_conn(mv, mf, which));
      // the PnP inliers (vo.cpp:333-354) as (map point id, keypoint index): the candidate-list index and the descriptor
      // distance of the reference's DMatch are not kept in this mode
      for (auto &kc : mf->conn)
        if (kc.second.pt_ref_idx < 0) mf->matches_with_map.push_back(mvo_dmatch{kc.second.pt_map_idx, kc.first, 0, 0.f});
    }
  }
  const void *src = nullptr;
  size_t count = 0, elem = 0;
  switch (what) {
    case MVO_VO_KEYPOINTS: src = f->kpts.data(); count = f->kpts.size(); elem = sizeof(mvo_keypoint); break;
    case MVO_VO_DESCRIPTORS: src = f->desc.data(); count = f->desc.size() / 32; elem = 32; break;
    case MVO_VO_MATCHES_WITH_REF: src = f->matches_with_ref.data(); count = f->matches_with_ref.size(); elem = sizeof(mvo_dmatch); break;
    case MVO_VO_MATCHES_WITH_MAP: src = f->matches_with_map.data(); count = f->matches_with_map.size(); elem = sizeof(mvo_dmatch); break;
    case MVO_VO_INLIERS_PTS3D: src = f->inliers_pts3d.data(); count = f->inliers_pts3d.size() / 3; elem = 12; break;
    case MVO_VO_FRAME_ID: {
      *n = 1;
      if (cap < 1 || !out) return MVO_ERR_CAPACITY;
      *(int32_t *)out = f->id;
      return MVO_OK;
    }
    default: return MVO_ERR_INVALID_ARG;
  }
  *n = (int)count;
  if ((int)count > cap || (count > 0 && !out)) return MVO_ERR_CAPACITY;
  if (count > 0) memcpy(out, src, count * elem);
  return MVO_OK;
}

int mvo_vo_frame_pose(const mvo_vo *v, int k, double *T_w_c) {
  if (!v || !T_w_c || k < 0 || k >= (int)v->buff.size()) return MVO_ERR_INVALID_ARG;
  memcpy(T_w_c, v->buff[v->buff.size() - 1 - (size_t)k]->T_w_c, 16 * sizeof(double));
  return MVO_OK;
}

}  // extern "C"

// The kernel of mvo_vo_init_candidates_batch_dev lives in vo_init_batch.cu, a translation unit of its own that is compiled without
// contraction (Makefile).  libmvo.so always links it; a library assembled from a subset of the units without it reports
// MVO_ERR_UNSUPPORTED for the call.
int mvo_vo_init_candidates_launch(mvo_ctx *ctx, const MvoInitCandidates &a) __attribute__((weak));

// mvo_vo_init_candidates_batch_dev (mvo.h): the call-level checks here, everything per pair in one launch (vo_init_batch.cu)
extern "C" int mvo_vo_init_candidates_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                                const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches,
                                                const int32_t *d_n_matches, const mvo_relative_poses_result *d_rp,
                                                const int32_t *d_rp_inliers, const float *d_rp_pts3d, const double *T_w_c_ref,
                                                const mvo_vo_params *vp, mvo_init_candidate_result *d_out, mvo_dmatch *d_kept,
                                                float *d_kept_pts3d, double *d_kept_angles) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!d_kpts || !d_counts || !d_pairs || !d_matches || !d_n_matches || !d_rp || !d_rp_inliers || !d_rp_pts3d || !T_w_c_ref || !vp ||
      !d_out || !d_kept || !d_kept_pts3d || !d_kept_angles)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo init candidates batch: null pointer");
  if (!mvo_vo_init_candidates_launch)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "vo init candidates batch: the library was built without vo_init_batch.cu");
  if (n_pairs < 0 || batch < 1 || cap < 1)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo init candidates batch: n_pairs=%d batch=%d cap=%d", n_pairs, batch, cap);
  for (int q = 0; q < 16; ++q)
    if (!std::isfinite(T_w_c_ref[q])) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo init candidates batch: T_w_c_ref is not finite");
  const double thr[5] = {vp->min_triang_angle, vp->max_ratio_angle_to_median, vp->min_pixel_dist, vp->min_median_triangulation_angle,
                         vp->assumed_mean_depth_init};
  for (double x : thr)
    if (!std::isfinite(x)) return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo init candidates batch: a threshold of vp is not finite");
  if (cap > 6400) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "vo init candidates batch: cap %d above 6400 correspondences", cap);
  if (n_pairs > 65535) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "vo init candidates batch: %d pairs, at most 65535 per call", n_pairs);
  if (n_pairs == 0) return MVO_OK;
  MvoInitCandidates a;
  a.kpts = d_kpts; a.counts = d_counts; a.pairs = d_pairs; a.n_matches = d_n_matches; a.rp_inliers = d_rp_inliers; a.matches = d_matches;
  a.rp = d_rp; a.rp_pts3d = d_rp_pts3d;
  a.batch = batch; a.cap = cap; a.n_pairs = n_pairs; a.min_inlier_matches = vp->min_inlier_matches;
  memcpy(a.T_ref, T_w_c_ref, sizeof a.T_ref);
  a.min_triang_angle = thr[0]; a.max_ratio_angle_to_median = thr[1]; a.min_pixel_dist = thr[2]; a.min_median_triangulation_angle = thr[3];
  a.assumed_mean_depth_init = thr[4];
  a.out = d_out; a.kept = d_kept; a.kept_pts3d = d_kept_pts3d; a.kept_angles = d_kept_angles;
  return mvo_vo_init_candidates_launch(ctx, a);
}

// The first and last kernels of mvo_vo_keyframe_points_batch_dev live in vo_init_batch.cu as well (the triangulation between them
// in epipolar.cu); a library without that unit reports MVO_ERR_UNSUPPORTED for the call.
int mvo_vo_keyframe_points_launch(mvo_ctx *ctx, const MvoKeyframePoints &a) __attribute__((weak));

// mvo_vo_keyframe_points_batch_dev (mvo.h): the call-level checks here, everything per pair in three launches
extern "C" int mvo_vo_keyframe_points_batch_dev(mvo_ctx *ctx, const mvo_keypoint *d_kpts, const int32_t *d_counts, int batch, int cap,
                                                const int32_t *d_pairs, int n_pairs, const mvo_dmatch *d_matches,
                                                const int32_t *d_n_matches, const mvo_two_view_result *d_ess,
                                                const int32_t *d_ess_inliers, const double *d_T_w_c, const double *K,
                                                const mvo_vo_params *vp, mvo_keyframe_points_result *d_out, mvo_dmatch *d_kept,
                                                float *d_kept_pts3d, double *d_kept_angles, float *d_kept_world, double *d_kept_norm) {
  if (!ctx) return MVO_ERR_INVALID_ARG;
  if (!d_kpts || !d_counts || !d_pairs || !d_matches || !d_n_matches || !d_ess || !d_ess_inliers || !d_T_w_c || !K || !vp || !d_out ||
      !d_kept || !d_kept_pts3d || !d_kept_angles)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo keyframe points batch: null pointer");
  if (!mvo_vo_keyframe_points_launch)
    return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "vo keyframe points batch: the library was built without vo_init_batch.cu");
  if (n_pairs < 0 || batch < 1 || cap < 1)
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo keyframe points batch: n_pairs=%d batch=%d cap=%d", n_pairs, batch, cap);
  if (!(std::isfinite(K[0]) && K[0] > 0 && std::isfinite(K[4]) && K[4] > 0))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo keyframe points batch: fx and fy must be finite and positive");
  if (!std::isfinite(vp->min_triang_angle) || !std::isfinite(vp->max_ratio_angle_to_median))
    return mvo_fail(ctx, MVO_ERR_INVALID_ARG, "vo keyframe points batch: a threshold of vp is not finite");
  if (cap > 6400) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "vo keyframe points batch: cap %d above 6400 correspondences", cap);
  if (n_pairs > 65535) return mvo_fail(ctx, MVO_ERR_UNSUPPORTED, "vo keyframe points batch: %d pairs, at most 65535 per call", n_pairs);
  if (n_pairs == 0) return MVO_OK;
  MvoKeyframePoints a;
  a.kpts = d_kpts; a.counts = d_counts; a.pairs = d_pairs; a.n_matches = d_n_matches; a.ess_inliers = d_ess_inliers; a.matches = d_matches;
  a.ess = d_ess; a.T_w_c = d_T_w_c;
  a.batch = batch; a.cap = cap; a.n_pairs = n_pairs;
  a.fx = K[0]; a.fy = K[4]; a.cx = K[2]; a.cy = K[5];
  a.min_triang_angle = vp->min_triang_angle; a.max_ratio_angle_to_median = vp->max_ratio_angle_to_median;
  a.out = d_out; a.kept = d_kept; a.kept_pts3d = d_kept_pts3d; a.kept_world = d_kept_world; a.kept_angles = d_kept_angles;
  a.kept_norm = d_kept_norm;
  return mvo_vo_keyframe_points_launch(ctx, a);
}
