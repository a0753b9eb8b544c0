// voxel_ba_shim.hpp — header-only C++ shim that re-creates the reference's call surface on top of the C-ABI (include/vxs.h),
// so voxelslam.cpp keeps compiling against the same names:
//
//   LidarFactor                (voxel_map.hpp:109-290)   -> vxs_shim::LidarFactor          (host staging + device factor)
//   Lidar_BA_Optimizer         (voxel_map.hpp:293-444)   -> vxs_shim::Lidar_BA_Optimizer
//   LI_BA_Optimizer            (voxel_map.hpp:450-655)   -> vxs_shim::LI_BA_Optimizer
//   LI_BA_OptimizerGravity     (voxel_map.hpp:658-864)   -> vxs_shim::LI_BA_OptimizerGravity
//
// Two layers:
//   * a plain layer (no Eigen): flat arrays in, flat arrays out — compile-tested in this repository (tests/test_abi.py);
//   * an Eigen/reference-typed layer behind VXS_SHIM_WITH_REFERENCE_TYPES: include it AFTER the reference's tools.hpp, preintegration.hpp and
//     voxel_map.hpp (it uses their IMUST, PointCluster, IMU_PRE, DIM, pointVar, PVecPtr, SlideWindow, Keyframe).  tests/test_abi.py compiles
//     this layer against the reference's REAL headers from the reference checkout (with stand-in headers for the Eigen / PCL /
//     ROS headers this image lacks) and, on boxes without the reference, against tests/shim_stubs/reference_stubs.hpp.
#pragma once
#include <cstring>
#include <deque>
#include <new>
#include <stdexcept>
#include <string>
#include <algorithm>
#include <vector>
#include "../../../include/vxs.h"

namespace vxs_shim {

inline void check(vxs_ctx* ctx, int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + (ctx ? vxs_ctx_last_error(ctx) : "libvxs error"));
}

// One context per calling thread (local mapping thread, global mapping thread).
class Context {
 public:
  explicit Context(int device = 0) { int rc = vxs_ctx_create(device, &ctx_); if (rc) throw std::runtime_error("vxs_ctx_create failed: no CUDA device, and libvxs has no CPU fallback"); }
  ~Context() { vxs_ctx_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  vxs_ctx* get() const { return ctx_; }
 private:
  vxs_ctx* ctx_ = nullptr;
};

// `LidarFactor voxhess(win_size);` (voxel_map.hpp:120) keeps compiling: one lazily created context per calling thread
inline Context& default_context() { static thread_local Context c(0); return c; }

// page-locked std::vector storage for the bulk of the staged factor, so that vxs_factor_push_voxels_async really overlaps PCIe and compute
template <class T>
struct PinnedAllocator {
  using value_type = T;
  PinnedAllocator() = default;
  template <class U> PinnedAllocator(const PinnedAllocator<U>&) {}
  T* allocate(size_t n) { void* p = nullptr; if (vxs_host_alloc(&p, uint64_t(n) * sizeof(T)) != 0 || !p) throw std::bad_alloc(); return static_cast<T*>(p); }
  void deallocate(T* p, size_t) { vxs_host_free(p); }
  template <class U> bool operator==(const PinnedAllocator<U>&) const { return true; }
  template <class U> bool operator!=(const PinnedAllocator<U>&) const { return false; }
};

// LidarFactor: push_voxel() stages on the host exactly like the reference's vectors; the first solver call uploads the batch.
class LidarFactor {
 public:
  int win_size;
  // read-back mirrors of the reference members the callers touch after a solve (voxel_map.hpp:1217-1222, voxelslam.cpp:651-655)
  std::vector<double> eig12;   // [V][12]  eig_values | eig_vectors (row-major, eigenvectors in columns)
  std::vector<double> sum10;   // [V][10]  pcr_adds

  LidarFactor(Context& c, int w) : win_size(w), ctx_(c.get()) { check(ctx_, vxs_factor_create(ctx_, w, &dev_), "vxs_factor_create"); }
  explicit LidarFactor(int w) : LidarFactor(default_context(), w) {}   // the reference's constructor (voxel_map.hpp:120)
  ~LidarFactor() { vxs_factor_destroy(dev_); }
  LidarFactor(const LidarFactor&) = delete;
  LidarFactor& operator=(const LidarFactor&) = delete;

  // voxel_map.hpp:122-130.  clusters10: win_size x 10 (N==0 => frame absent); fix10/eig12/sum10 as in vxs.h
  void push_voxel(const double* clusters10, const double* fix10, double coe, const double* eig, const double* sum) {
    for (int i = 0; i < win_size; i++) {
      const double* c = clusters10 + 10 * i;
      if (c[9] != 0.0) { frame_.push_back(i); cl_.insert(cl_.end(), c, c + 10); }
    }
    ptr_.push_back(int64_t(frame_.size()));
    fix_.insert(fix_.end(), fix10, fix10 + 10); coe_.push_back(coe);
    eig12.insert(eig12.end(), eig, eig + 12); sum10.insert(sum10.end(), sum, sum + 10);
    dirty_ = true;
  }
  void clear() {  // voxel_map.hpp:281-286
    ptr_.assign(1, 0); frame_.clear(); cl_.clear(); fix_.clear(); coe_.clear(); eig12.clear(); sum10.clear();
    check(ctx_, vxs_factor_clear(dev_), "vxs_factor_clear");
    dirty_ = false; device_filled_ = false;
  }
  size_t size() const {
    if (!device_filled_) return ptr_.size() - 1;
    int64_t v = 0; vxs_factor_counts(dev_, &v, nullptr, nullptr); return size_t(v);
  }
  // the factor was filled on the device (vxs_map_push_scan / vxs_build_*_factor): nothing is staged on the host, and margi reads the cached
  // eig / pcr_adds in place, so no read-back happens either
  vxs_factor* device_fill_target() { ptr_.assign(1, 0); frame_.clear(); cl_.clear(); fix_.clear(); coe_.clear(); eig12.clear(); sum10.clear(); dirty_ = false; device_filled_ = true; return dev_; }

  vxs_factor* device() {  // flush staged voxels
    if (dirty_) {
      check(ctx_, vxs_factor_clear(dev_), "vxs_factor_clear");
      check(ctx_, vxs_factor_set_win_size(dev_, win_size), "vxs_factor_set_win_size");
      // asynchronous: the solver's first Hessian build runs behind the upload chunks; the staged vectors stay untouched until it returns
      check(ctx_, vxs_factor_push_voxels_async(dev_, int64_t(size()), ptr_.data(), frame_.data(), cl_.data(), fix_.data(), coe_.data(), eig12.data(), sum10.data()),
            "vxs_factor_push_voxels_async");
      dirty_ = false;
    }
    return dev_;
  }
  void sync_back() {
    if (device_filled_) { const size_t v = size(); eig12.resize(v * 12); sum10.resize(v * 10); }
    if (size()) check(ctx_, vxs_factor_read_back(dev_, eig12.data(), sum10.data()), "vxs_factor_read_back");
  }
  vxs_ctx* ctx() const { return ctx_; }

 private:
  vxs_ctx* ctx_;
  vxs_factor* dev_ = nullptr;
  std::vector<int64_t> ptr_{0};
  std::vector<int32_t, PinnedAllocator<int32_t>> frame_;
  std::vector<double, PinnedAllocator<double>> cl_;
  std::vector<double> fix_, coe_;
  bool dirty_ = false, device_filled_ = false;
};

// Lidar_BA_Optimizer (flat layer): poses12 = W x 12 in/out, hess = (6W)^2 column-major out (may be null), resis gets 2 entries appended
class Lidar_BA_Optimizer {
 public:
  int thd_num = 2;
  bool damping_iter(double* poses12, LidarFactor& voxhess, double* hess, std::vector<double>& resis, int max_iter = 3) {
    double r[2] = {0, 0}; int conv = 0;
    int rc = vxs_lidar_ba(voxhess.ctx(), voxhess.device(), poses12, max_iter, thd_num, hess, r, &conv, nullptr, 0, nullptr);
    check(voxhess.ctx(), rc, "vxs_lidar_ba");
    resis.push_back(r[0]); resis.push_back(r[1]);
    voxhess.sync_back();
    return conv != 0;
  }
};

// LI_BA_Optimizer / LI_BA_OptimizerGravity (flat layer): states24 = W x 24, hooks wrap the caller's IMU_PRE objects
class LI_BA_Optimizer {
 public:
  double imu_coef = 1e-4;   // voxel_map.hpp:446
  void damping_iter(double* states24, LidarFactor& voxhess, const vxs_imu_hooks& imu, double* hess) {
    double r[2];
    check(voxhess.ctx(), vxs_li_ba(voxhess.ctx(), voxhess.device(), states24, 0, 3, imu_coef, &imu, hess, r, nullptr, 0, nullptr), "vxs_li_ba");
    voxhess.sync_back();
  }
};
class LI_BA_OptimizerGravity {
 public:
  double imu_coef = 1e-4;
  void damping_iter(double* states24, LidarFactor& voxhess, const vxs_imu_hooks& imu, std::vector<double>& resis, double* hess, int max_iter = 2) {
    double r[2] = {0, 0};
    check(voxhess.ctx(), vxs_li_ba(voxhess.ctx(), voxhess.device(), states24, 1, max_iter, imu_coef, &imu, hess, r, nullptr, 0, nullptr), "vxs_li_ba");
    resis.push_back(r[0]); resis.push_back(r[1]);
    voxhess.sync_back();
  }
};

}  // namespace vxs_shim

// ------------------------------------------------------------------------------------------------------------------------------
#if defined(VXS_SHIM_WITH_REFERENCE_TYPES)
// Requires the reference's tools.hpp (IMUST, PointCluster, DIM) and preintegration.hpp (IMU_PRE) to be included first.
namespace vxs_shim {

inline void pack_cluster(const PointCluster& c, double* o) {
  o[0] = c.P(0, 0); o[1] = c.P(0, 1); o[2] = c.P(0, 2); o[3] = c.P(1, 1); o[4] = c.P(1, 2); o[5] = c.P(2, 2);
  o[6] = c.v[0]; o[7] = c.v[1]; o[8] = c.v[2]; o[9] = double(c.N);
}
inline void pack_state(const IMUST& x, double* s) {
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) s[3 * r + c] = x.R(r, c);
  for (int k = 0; k < 3; k++) { s[9 + k] = x.p[k]; s[12 + k] = x.v[k]; s[15 + k] = x.bg[k]; s[18 + k] = x.ba[k]; s[21 + k] = x.g[k]; }
}
inline void unpack_state(const double* s, IMUST& x) {
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) x.R(r, c) = s[3 * r + c];
  for (int k = 0; k < 3; k++) { x.p[k] = s[9 + k]; x.v[k] = s[12 + k]; x.bg[k] = s[15 + k]; x.ba[k] = s[18 + k]; x.g[k] = s[21 + k]; }
}

// LidarFactor::push_voxel with the reference's argument list (voxel_map.hpp:122)
inline void push_voxel(LidarFactor& f, std::vector<PointCluster>& vec_orig, PointCluster& fix, double coe, Eigen::Vector3d& eig_value, Eigen::Matrix3d& eig_vector, PointCluster& pcr_add) {
  std::vector<double> cl(size_t(f.win_size) * 10);
  for (int i = 0; i < f.win_size; i++) pack_cluster(vec_orig[i], &cl[10 * i]);
  double fx[10], e[12], s[10];
  pack_cluster(fix, fx); pack_cluster(pcr_add, s);
  for (int k = 0; k < 3; k++) e[k] = eig_value[k];
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) e[3 + 3 * r + c] = eig_vector(r, c);
  f.push_voxel(cl.data(), fx, coe, e, s);
}

// the IMU factor stays the reference's own code: these hooks call IMU_PRE::give_evaluate(_g) / update_state on the caller's deque
struct ImuAdapter {
  std::deque<IMU_PRE*>* imus;
  static int eval(void* u, const double* states24, int W, int with_g, int want_jac, double* blocks, double* gvec, double* cost) {
    auto* self = static_cast<ImuAdapter*>(u);
    const int bs = with_g ? 33 : 30;
    Eigen::MatrixXd jtj(bs, bs); Eigen::VectorXd gg(bs);
    std::vector<IMUST> xs(W);
    for (int i = 0; i < W; i++) unpack_state(states24 + 24 * i, xs[i]);
    double c = 0;
    for (int i = 0; i + 1 < W; i++) {
      jtj.setZero(); gg.setZero();
      c += with_g ? (*self->imus)[i]->give_evaluate_g(xs[i], xs[i + 1], jtj, gg, want_jac != 0) : (*self->imus)[i]->give_evaluate(xs[i], xs[i + 1], jtj, gg, want_jac != 0);
      if (want_jac) { std::memcpy(blocks + size_t(i) * bs * bs, jtj.data(), sizeof(double) * bs * bs); std::memcpy(gvec + size_t(i) * bs, gg.data(), sizeof(double) * bs); }
    }
    *cost = c;
    return 0;
  }
  static int update(void* u, const double* dxi, int W) {
    auto* self = static_cast<ImuAdapter*>(u);
    for (int j = 0; j + 1 < W; j++) (*self->imus)[j]->update_state(Eigen::Map<const Eigen::Matrix<double, DIM, 1>>(dxi + DIM * j));
    return 0;
  }
  static int rollback(void* u) {
    auto* self = static_cast<ImuAdapter*>(u);
    for (IMU_PRE* p : *self->imus) { p->dbg = p->dbg_buf; p->dba = p->dba_buf; }
    return 0;
  }
  vxs_imu_hooks hooks() { vxs_imu_hooks h; h.user = this; h.eval = &eval; h.update = &update; h.rollback = &rollback; return h; }
};

// LI_BA_Optimizer::damping_iter(x_stats, voxhess, imus_factor, hess)  — voxelslam.cpp:1652-1653 call site
inline void li_ba_damping_iter(std::vector<IMUST>& x_stats, LidarFactor& voxhess, std::deque<IMU_PRE*>& imus_factor, Eigen::MatrixXd* hess, double imu_coef) {
  const int W = voxhess.win_size;
  std::vector<double> st(size_t(W) * 24);
  for (int i = 0; i < W; i++) pack_state(x_stats[i], &st[24 * i]);
  hess->resize(W * DIM, W * DIM);
  ImuAdapter ad{&imus_factor};
  LI_BA_Optimizer opt; opt.imu_coef = imu_coef;
  opt.damping_iter(st.data(), voxhess, ad.hooks(), hess->data());
  for (int i = 0; i < W; i++) unpack_state(&st[24 * i], x_stats[i]);
}
// Lidar_BA_Optimizer::damping_iter(xs, voxhess, &hess, resis, up, is_display) — voxelslam.cpp:2381-2384 call site
inline bool lidar_ba_damping_iter(std::vector<IMUST>& x_stats, LidarFactor& voxhess, Eigen::MatrixXd* hess, std::vector<double>& resis, int max_iter, int thd_num) {
  const int W = voxhess.win_size;
  std::vector<double> p(size_t(W) * 12), st(24);
  for (int i = 0; i < W; i++) { pack_state(x_stats[i], st.data()); std::memcpy(&p[12 * i], st.data(), 96); }
  hess->resize(6 * W, 6 * W);
  Lidar_BA_Optimizer opt; opt.thd_num = thd_num;
  bool conv = opt.damping_iter(p.data(), voxhess, hess->data(), resis, max_iter);
  for (int i = 0; i < W; i++) { for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) x_stats[i].R(r, c) = p[12 * i + 3 * r + c]; for (int k = 0; k < 3; k++) x_stats[i].p[k] = p[12 * i + 9 + k]; }
  return conv;
}

// down_sampling_voxel(pl_feat, voxel_size) — tools.hpp:201 (call sites voxelslam.cpp:1146, 2118, 2440).  PointType is
// pcl::PointXYZINormal (48 bytes, x,y,z first): the cloud goes up as it is, the surviving points keep the fields of the first point of
// their cell and get curvature = points in the cell, exactly like the reference; only the ORDER of the output differs (cell order
// instead of unordered_map order).
inline void down_sampling_voxel(Context& ctx, pcl::PointCloud<PointType>& pl_feat, double voxel_size) {
  const int64_t n = int64_t(pl_feat.size());
  std::vector<float> xyz(size_t(n) * 3), cnt(n);
  std::vector<int64_t> first(n);
  int64_t m = 0;
  check(ctx.get(), vxs_down_sampling_voxel(ctx.get(), reinterpret_cast<const float*>(pl_feat.points.data()), int(sizeof(PointType) / sizeof(float)), n, voxel_size,
                                           xyz.data(), cnt.data(), first.data(), n, &m), "vxs_down_sampling_voxel");
  if (m < 0) return;
  pcl::PointCloud<PointType> out;
  out.reserve(size_t(m));
  for (int64_t i = 0; i < m; i++) {
    PointType pp = pl_feat.points[size_t(first[i])];
    pp.x = xyz[3 * i]; pp.y = xyz[3 * i + 1]; pp.z = xyz[3 * i + 2]; pp.curvature = cnt[i];
    out.push_back(pp);
  }
  pl_feat.swap(out);
}
// down_sampling_pvec(pvec, voxel_size, pl_keep) — voxel_map.hpp:23 (call sites voxelslam.cpp:1146-1148 scan pre-processing).
// pointVar = { Vector3d pnt; Matrix3d var } = 12 doubles, handed to the device as it is.
inline void down_sampling_pvec(Context& ctx, PVec& pvec, double voxel_size, pcl::PointCloud<PointType>& pl_keep) {
  static_assert(sizeof(pointVar) % sizeof(double) == 0, "pointVar is a plain fp64 record");
  const int64_t n = int64_t(pvec.size());
  std::vector<float> xyz(size_t(n) * 3), vd(size_t(n) * 3);
  int64_t m = 0;
  check(ctx.get(), vxs_down_sampling_pvec(ctx.get(), reinterpret_cast<const double*>(pvec.data()), int(sizeof(pointVar) / sizeof(double)), n, voxel_size,
                                          xyz.data(), vd.data(), nullptr, nullptr, n, &m), "vxs_down_sampling_pvec");
  pcl::PointCloud<PointType>().swap(pl_keep);
  pl_keep.reserve(size_t(m));
  PointType ap;
  for (int64_t i = 0; i < m; i++) {
    ap.x = xyz[3 * i]; ap.y = xyz[3 * i + 1]; ap.z = xyz[3 * i + 2];
    ap.normal_x = vd[3 * i]; ap.normal_y = vd[3 * i + 1]; ap.normal_z = vd[3 * i + 2];
    pl_keep.push_back(ap);
  }
}
// down_sampling_close(pl_feat, voxel_size) — tools.hpp:240
inline void down_sampling_close(Context& ctx, pcl::PointCloud<PointType>& pl_feat, double voxel_size) {
  const int64_t n = int64_t(pl_feat.size());
  std::vector<int64_t> pick(n);
  int64_t m = 0;
  check(ctx.get(), vxs_down_sampling_close(ctx.get(), reinterpret_cast<const float*>(pl_feat.points.data()), int(sizeof(PointType) / sizeof(float)), n, voxel_size,
                                           nullptr, nullptr, pick.data(), n, &m), "vxs_down_sampling_close");
  if (m < 0) return;
  pcl::PointCloud<PointType> out;
  out.reserve(size_t(m));
  for (int64_t i = 0; i < m; i++) out.push_back(pl_feat.points[size_t(pick[i])]);
  pl_feat.swap(out);
}

// Submap merge at the end of HBA_add_edge (voxelslam.cpp:2428-2447): smps[i]->plptr clouds -> *plptr in the frame of xs[0], down-sampled
// at voxel_size / 8, intensity = map id of the keyframe the surviving point came from.
template <class KeyframePtrVec>
inline void submap_merge(Context& ctx, const std::vector<IMUST>& xs, const KeyframePtrVec& smps, double voxel_size, pcl::PointCloud<PointType>& out) {
  const int W = int(xs.size());
  std::vector<int64_t> off(size_t(W) + 1, 0);
  for (int i = 0; i < W; i++) off[i + 1] = off[i] + int64_t(smps[i]->plptr->size());
  std::vector<PointType> all; all.reserve(size_t(off[W]));
  for (int i = 0; i < W; i++) all.insert(all.end(), smps[i]->plptr->points.begin(), smps[i]->plptr->points.end());
  std::vector<double> p(size_t(W) * 12), st(24);
  for (int i = 0; i < W; i++) { pack_state(xs[i], st.data()); std::memcpy(&p[12 * size_t(i)], st.data(), 96); }
  const int64_t n = off[W];
  std::vector<float> xyz(size_t(n) * 3), cnt(n);
  std::vector<int64_t> first(n);
  int64_t m = 0;
  check(ctx.get(), vxs_submap_merge(ctx.get(), reinterpret_cast<const float*>(all.data()), int(sizeof(PointType) / sizeof(float)), off.data(), p.data(), W, voxel_size / 8,
                                    xyz.data(), cnt.data(), first.data(), n, &m), "vxs_submap_merge");
  out.clear(); out.reserve(size_t(m));
  for (int64_t k = 0; k < m; k++) {
    PointType pp = all[size_t(first[k])];
    const int kf = int(std::upper_bound(off.begin(), off.end(), first[k]) - off.begin()) - 1;
    pp.x = xyz[3 * k]; pp.y = xyz[3 * k + 1]; pp.z = xyz[3 * k + 2]; pp.curvature = cnt[k]; pp.intensity = smps[kf]->mp;
    out.push_back(pp);
  }
}

// LI_BA_OptimizerGravity::damping_iter(x_stats, voxhess, imus_factor, resis, hess, max_iter) — voxel_map.hpp:775, call sites voxelslam.cpp:632-634, 1643-1645
inline void li_ba_gravity_damping_iter(std::vector<IMUST>& x_stats, LidarFactor& voxhess, std::deque<IMU_PRE*>& imus_factor, std::vector<double>& resis, Eigen::MatrixXd* hess,
                                       int max_iter, double imu_coef) {
  const int W = voxhess.win_size;
  std::vector<double> st(size_t(W) * 24);
  for (int i = 0; i < W; i++) pack_state(x_stats[i], &st[24 * i]);
  hess->resize(W * DIM + 3, W * DIM + 3);
  ImuAdapter ad{&imus_factor};
  LI_BA_OptimizerGravity opt; opt.imu_coef = imu_coef;
  opt.damping_iter(st.data(), voxhess, ad.hooks(), resis, hess->data(), max_iter);
  for (int i = 0; i < W; i++) unpack_state(&st[24 * i], x_stats[i]);     // g is broadcast to every state by the solver (voxel_map.hpp:821)
}

// ---------------------------------------------------------------- the per-scan map calls of thd_odometry_localmapping on the device-resident map
// SurfMap stands for BOTH `surf_map` and `surf_map_slide` (unordered_map<VOXEL_LOC, OctoTree*>, voxelslam.hpp): the octree, the slide windows
// and the resident scans live in HBM (vxs_map).  The three reference calls keep their names and argument lists:
//   cut_voxel_multi(surf_map, pvec_buf[win_count-1], win_count-1, surf_map_slide, win_size, pwld, sws);      voxelslam.cpp:1612
//   multi_recut(surf_map_slide, win_count, x_buf, voxhess, sws);                                              voxelslam.cpp:1615
//   multi_margi(surf_map_slide, jour, win_count, x_buf, voxhess, sws[0]);                                     voxelslam.cpp:1669
// cut + recut are one device call (vxs_map_push_scan), so cut_voxel_multi only notes the scan and multi_recut does the work; multi_margi also
// rotates the slot ring, so the caller's `mp[i] += mgsize` loop (voxelslam.cpp:1689-1693) becomes a no-op on an unused array.
class SurfMap {
 public:
  SurfMap(Context& c, const vxs_map_params& p, int win_size, int max_pts = 100) : ctx_(c.get()) { check(ctx_, vxs_map_create(ctx_, &p, win_size, max_pts, &m_), "vxs_map_create"); }
  SurfMap(const vxs_map_params& p, int win_size, int max_pts = 100) : SurfMap(default_context(), p, win_size, max_pts) {}
  ~SurfMap() { vxs_map_destroy(m_); }
  SurfMap(const SurfMap&) = delete;
  SurfMap& operator=(const SurfMap&) = delete;
  vxs_map* get() const { return m_; }
  vxs_ctx* ctx() const { return ctx_; }
  PVecPtr pending;          // the scan cut_voxel_multi was called with, consumed by multi_recut
 private:
  vxs_ctx* ctx_; vxs_map* m_ = nullptr;
};
inline void cut_voxel_multi(SurfMap& feat_map, PVecPtr pvec, int /*win_count*/, SurfMap& /*feat_tem_map*/, int /*wdsize*/, PLV(3)& /*pwld: recomputed on the device, bit-exact*/,
                            std::vector<std::vector<SlideWindow*>>& /*sws*/) { feat_map.pending = pvec; }
inline void cut_voxel(SurfMap& feat_map, PVecPtr pvec, int /*win_count*/, SurfMap& /*feat_tem_map*/, int /*wdsize*/, PLV(3)& /*pwld*/, std::vector<SlideWindow*>& /*sws*/) { feat_map.pending = pvec; }
inline void multi_recut(SurfMap& feat_map, int win_count, std::vector<IMUST>& xs, LidarFactor& voxopt, std::vector<std::vector<SlideWindow*>>& /*sws*/) {
  static_assert(sizeof(pointVar) == 12 * sizeof(double), "pointVar = { Vector3d pnt; Matrix3d var } is handed to the device as 12 doubles (var is symmetric: storage order is irrelevant)");
  std::vector<double> p(size_t(win_count) * 12), st(24);
  for (int i = 0; i < win_count; i++) { pack_state(xs[i], st.data()); std::memcpy(&p[12 * size_t(i)], st.data(), 96); }
  const PVecPtr& pv = feat_map.pending;
  check(feat_map.ctx(), vxs_map_push_scan(feat_map.get(), pv ? reinterpret_cast<const double*>(pv->data()) : nullptr, pv ? int64_t(pv->size()) : 0, p.data(), win_count,
                                          voxopt.device_fill_target()), "vxs_map_push_scan");
  feat_map.pending.reset();
}
inline void multi_margi(SurfMap& feat_map, double /*jour*/, int win_count, std::vector<IMUST>& xs, LidarFactor& voxopt, std::vector<SlideWindow*>& /*sw*/) {
  std::vector<double> p(size_t(win_count) * 12), st(24);
  for (int i = 0; i < win_count; i++) { pack_state(xs[i], st.data()); std::memcpy(&p[12 * size_t(i)], st.data(), 96); }
  check(feat_map.ctx(), vxs_map_margi(feat_map.get(), p.data(), win_count, 1 /* multi_margi hard-codes margi(win_cnt, 1, ...), voxelslam.cpp:1360 */, voxopt.device()), "vxs_map_margi");
}

// ---------------------------------------------------------------- the map rebuild of an HBA pass (voxelslam.cpp:2374-2379)
//   OctreeGBA::cut_voxel(oct_map, xs[i], smps[i]->plptr, i, wdsize);   loop_refine.hpp:446      -> notes the keyframe
//   OctreeGBA_multi_recut(oct_map, voxhess, thread_num);               loop_refine.hpp:483      -> one vxs_build_gba_factor over all of them
class GbaMap {
 public:
  explicit GbaMap(const vxs_map_params& p) : params(p) {}
  vxs_map_params params;
  std::vector<pcl::PointCloud<PointType>::Ptr> clouds;
  std::vector<double> poses12;
  void clear() { clouds.clear(); poses12.clear(); }
};
inline void OctreeGBA_cut_voxel(GbaMap& feat_map, IMUST& xc, pcl::PointCloud<PointType>::Ptr plptr, int win_count, int /*wdsize*/) {
  if (int(feat_map.clouds.size()) <= win_count) { feat_map.clouds.resize(size_t(win_count) + 1); feat_map.poses12.resize((size_t(win_count) + 1) * 12); }
  feat_map.clouds[size_t(win_count)] = plptr;
  double st[24]; pack_state(xc, st);
  std::memcpy(&feat_map.poses12[12 * size_t(win_count)], st, 96);
}
inline void OctreeGBA_multi_recut(GbaMap& feat_map, LidarFactor& voxhess, int /*thd_num*/) {
  const int W = int(feat_map.clouds.size());
  std::vector<int64_t> off(size_t(W) + 1, 0);
  for (int i = 0; i < W; i++) off[size_t(i) + 1] = off[size_t(i)] + int64_t(feat_map.clouds[size_t(i)] ? feat_map.clouds[size_t(i)]->size() : 0);
  std::vector<PointType, PinnedAllocator<PointType>> all; all.reserve(size_t(off[size_t(W)]));
  for (int i = 0; i < W; i++) if (feat_map.clouds[size_t(i)]) all.insert(all.end(), feat_map.clouds[size_t(i)]->points.begin(), feat_map.clouds[size_t(i)]->points.end());
  int64_t nv = 0;
  check(voxhess.ctx(), vxs_build_gba_factor(voxhess.ctx(), &feat_map.params, reinterpret_cast<const float*>(all.data()), int(sizeof(PointType) / sizeof(float)), off.data(),
                                            feat_map.poses12.data(), W, voxhess.device_fill_target(), nullptr, 0, &nv), "vxs_build_gba_factor");
  feat_map.clear();          // the reference consumes (deletes) the octrees here too (loop_refine.hpp:503-509)
}

// ---------------------------------------------------------------- scan pre-processing and odometry association (voxelslam.hpp:187-214, voxelslam.cpp:876-918)
//   var_init(extrin_para, pl_down, pptr, dept_err, beam_err);   voxelslam.cpp:1246, 1584      pvec_update(pptr, x_curr, pwld);   voxelslam.cpp:611, 1250, 1594
// The records also stay on the device (the ctx's resident scan): the EKF passes and the later vxs_map_push_scan can take them from there.
inline void var_init(Context& ctx, IMUST& ext, pcl::PointCloud<PointType>& pl_cur, PVecPtr pptr, double dept_err, double beam_err) {
  static_assert(sizeof(pointVar) == 12 * sizeof(double), "pointVar is handed over as 12 doubles");
  const int64_t n = int64_t(pl_cur.size());
  pptr->clear(); pptr->resize(size_t(n));
  double R[9], p[3];
  for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) R[3 * r + c] = ext.R(r, c); p[r] = ext.p[r]; }
  std::vector<double> rec(size_t(n) * 12);
  check(ctx.get(), vxs_var_init(ctx.get(), reinterpret_cast<const float*>(pl_cur.points.data()), int(sizeof(PointType) / sizeof(float)), n, R, p, dept_err, beam_err, rec.data()), "vxs_var_init");
  for (int64_t i = 0; i < n; i++) {          // var comes back row-major; pointVar::var is an Eigen matrix (symmetric, so the storage order does not matter, but stay explicit)
    pointVar& pv = (*pptr)[size_t(i)];
    const double* q = &rec[12 * size_t(i)];
    pv.pnt = Eigen::Vector3d(q[0], q[1], q[2]);
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) pv.var(r, c) = q[3 + 3 * r + c];
  }
}
inline void pvec_update(Context& ctx, PVecPtr pptr, IMUST& x_curr, PLV(3)& pwld) {
  const int64_t n = int64_t(pptr->size());
  std::vector<double> rec(size_t(n) * 12), out(size_t(n) * 12), pw(size_t(n) * 3);
  for (int64_t i = 0; i < n; i++) { const pointVar& pv = (*pptr)[size_t(i)]; double* q = &rec[12 * size_t(i)]; for (int k = 0; k < 3; k++) q[k] = pv.pnt[k]; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) q[3 + 3 * r + c] = pv.var(r, c); }
  double st[24], rv[9], tv[9];
  pack_state(x_curr, st);
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { rv[3 * r + c] = x_curr.cov(r, c); tv[3 * r + c] = x_curr.cov(3 + r, 3 + c); }
  check(ctx.get(), vxs_pvec_update(ctx.get(), rec.data(), n, st, rv, tv, out.data(), pw.data()), "vxs_pvec_update");
  for (int64_t i = 0; i < n; i++) {
    pointVar& pv = (*pptr)[size_t(i)];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) pv.var(r, c) = out[12 * size_t(i) + 3 + 3 * r + c];
    pwld.push_back(Eigen::Vector3d(pw[3 * size_t(i)], pw[3 * size_t(i) + 1], pw[3 * size_t(i) + 2]));
  }
}
// the per-point loop of one EKF iteration (voxelslam.cpp:876-918) against the resident map: HTH, HTz, nnt, match_num.  first_pass uploads the scan, later passes reuse it.
inline int odom_accumulate(SurfMap& surf_map, PVecPtr pptr, IMUST& x_curr, bool first_pass, Eigen::Matrix<double, 6, 6>& HTH, Eigen::Matrix<double, 6, 1>& HTz, Eigen::Matrix3d& nnt) {
  const int64_t n = int64_t(pptr->size());
  std::vector<double> rec;
  if (first_pass) { rec.resize(size_t(n) * 12); for (int64_t i = 0; i < n; i++) { const pointVar& pv = (*pptr)[size_t(i)]; double* q = &rec[12 * size_t(i)]; for (int k = 0; k < 3; k++) q[k] = pv.pnt[k]; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) q[3 + 3 * r + c] = pv.var(r, c); } }
  double st[24], rv[9], tv[9], h[36], z[6], nn[9];
  pack_state(x_curr, st);
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { rv[3 * r + c] = x_curr.cov(r, c); tv[3 * r + c] = x_curr.cov(3 + r, 3 + c); }
  int64_t m = 0;
  check(surf_map.ctx(), vxs_map_odom_accumulate(surf_map.get(), first_pass ? rec.data() : nullptr, n, st, rv, tv, h, z, nn, &m, nullptr), "vxs_map_odom_accumulate");
  for (int r = 0; r < 6; r++) { for (int c = 0; c < 6; c++) HTH(r, c) = h[6 * r + c]; HTz[r] = z[r]; }
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) nnt(r, c) = nn[3 * r + c];
  return int(m);
}

// ---------------------------------------------------------------- bottom level of the hierarchical global BA in one call (thd_globalmapping, voxelslam.cpp:2484-2557)
// every window w solves HBA_add_edge(xs, smp_local, gba_edges1, mps, 1, 2, plptr) on keyframes win_first[w] .. +win_size-1; poses_out[w] are the window's refined xs
template <class KeyframePtrVec>
inline void hba_bottom_batch(Context& ctx, const vxs_map_params& fine, const KeyframePtrVec& keyframes, const std::vector<int32_t>& win_first, int win_size,
                             std::vector<std::vector<IMUST>>& poses_out, std::vector<int32_t>& status) {
  const int K = int(keyframes.size()), nwin = int(win_first.size());
  std::vector<int64_t> off(size_t(K) + 1, 0);
  for (int i = 0; i < K; i++) off[size_t(i) + 1] = off[size_t(i)] + int64_t(keyframes[i]->plptr->size());
  std::vector<PointType, PinnedAllocator<PointType>> all; all.reserve(size_t(off[size_t(K)]));
  std::vector<double> p(size_t(K) * 12), st(24), out(size_t(nwin) * win_size * 12);
  for (int i = 0; i < K; i++) { all.insert(all.end(), keyframes[i]->plptr->points.begin(), keyframes[i]->plptr->points.end()); pack_state(keyframes[i]->x0, st.data()); std::memcpy(&p[12 * size_t(i)], st.data(), 96); }
  status.assign(size_t(nwin), 0);
  check(ctx.get(), vxs_hba_bottom_batch(ctx.get(), &fine, reinterpret_cast<const float*>(all.data()), int(sizeof(PointType) / sizeof(float)), off.data(), p.data(), K, win_first.data(), nwin, win_size,
                                        2, 0, out.data(), nullptr, status.data(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr), "vxs_hba_bottom_batch");
  poses_out.assign(size_t(nwin), std::vector<IMUST>(size_t(win_size)));
  for (int w = 0; w < nwin; w++)
    for (int j = 0; j < win_size; j++) {
      poses_out[size_t(w)][size_t(j)] = keyframes[win_first[size_t(w)] + j]->x0;
      double s24[24] = {0}; std::memcpy(s24, &out[(size_t(w) * win_size + j) * 12], 96);
      IMUST& x = poses_out[size_t(w)][size_t(j)];
      for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) x.R(r, c) = s24[3 * r + c]; x.p[r] = s24[9 + r]; }
    }
}

}  // namespace vxs_shim
#endif  // VXS_SHIM_WITH_REFERENCE_TYPES
