// REFERENCE BUILD — TEST INFRASTRUCTURE ONLY.  This translation unit #includes the reference's OWN hot-path sources where they lie
// (Voxel-SLAM/VoxelSLAM/src/{tools,preintegration,voxel_map,loop_refine}.hpp, unmodified, never copied into this repository) and exposes
// them through the same C entry points as the hand-written oracle (vxo_capi.cpp, prefix vxr_ instead of vxo_), so that the oracle can be
// pinned against the reference's real control flow, constants and formulas (tests/test_ref_pin.py) and the CUDA path can be checked against
// the reference directly (tests/test_gpu_ref.py).  Eigen / PCL / ROS / GTSAM are absent from this image: they are replaced by the stand-in
// headers of oracle/ref_standin/ (only the third-party arithmetic is restated there — see Eigen/Core).  Output: oracle/_ref/libvxref.so
// (git-ignored, travels to the GPU box like the other built libraries).
//
// Pieces of voxelslam.cpp (one 2600-line ROS translation unit that cannot be compiled here) that drive these classes are restated in a few
// lines each where a test needs them, each with its file:line: the from-scratch build sequence (:611-625), the per-scan map sequence
// (:1599-1615, 1669-1712; multi_recut :1398-1453 and multi_margi :1321-1395 are the reference's own member functions, see below) and the EKF accumulation loop
// (:876-918).  Everything numerical they call is the reference's own code.
// Two pieces are NOT restated but cut out of their files at build time (oracle/Makefile) and compiled as they are: calcBodyVar / var_init / pvec_update
// (voxelslam.hpp:163-214) and the member functions HBA_add_edge (voxelslam.cpp:2319-2482), multi_margi / multi_recut (:1321-1453) and lio_state_estimation (:856-954).
#include <chrono>
#include <cstdint>
#include <cstring>
#include <deque>
#include "../include/vxs.h"
#include "voxel_map.hpp"      // -I $VXS_REFERENCE_SRC  (pulls tools.hpp, preintegration.hpp)
#include "loop_refine.hpp"
#include "../tests/harness/synth.hpp"   // the seeded IMU sample generator shared with the harness (so both arms integrate the same samples)
#ifndef DEG2RAD
#define DEG2RAD(x) ((x)*0.017453293)   // pcl/pcl_macros.h (PCL 1.10), used by calcBodyVar
#endif
#include "_ref/vh_pointvar.inc"         // calcBodyVar / var_init / pvec_update cut out of voxelslam.hpp:163-214 by the Makefile (see there)
struct RefHbaHost {                     // stands for the reference's node class around its member function HBA_add_edge (voxelslam.cpp:2319-2482)
  int thread_num = 1;                   // the node's thread count (voxelslam.cpp:805 reads it from the launch file); 1 = deterministic push order
#include "_ref/vc_hba_add_edge.inc"     // cut out of voxelslam.cpp by the Makefile (see there)
#include "_ref/vc_multi_margi_recut.inc"   // multi_margi + multi_recut (voxelslam.cpp:1321-1453), likewise
  IMUST x_curr;                            // the node's current state and its map, as lio_state_estimation uses them (voxelslam.cpp:737, 741)
  unordered_map<VOXEL_LOC, OctoTree*> surf_map;
#include "_ref/vc_lio_state_estimation.inc"   // lio_state_estimation (voxelslam.cpp:856-954), likewise
};

namespace {

IMUST state_from12(const double* p) {
  IMUST x;
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) x.R(r, c) = p[3 * r + c];
  for (int k = 0; k < 3; k++) x.p[k] = p[9 + k];
  x.g = Eigen::Vector3d(0, 0, -G_m_s2);
  return x;
}
IMUST state_from24(const double* s) {
  IMUST x = state_from12(s);
  for (int k = 0; k < 3; k++) { x.v[k] = s[12 + k]; x.bg[k] = s[15 + k]; x.ba[k] = s[18 + k]; x.g[k] = s[21 + k]; }
  return x;
}
void state_to24(const IMUST& x, double* s) {
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) s[3 * r + c] = x.R(r, c);
  for (int k = 0; k < 3; k++) { s[9 + k] = x.p[k]; s[12 + k] = x.v[k]; s[15 + k] = x.bg[k]; s[18 + k] = x.ba[k]; s[21 + k] = x.g[k]; }
}
vector<IMUST> states12(const double* p, int W) { vector<IMUST> xs(W); for (int i = 0; i < W; i++) xs[i] = state_from12(p + 12 * i); return xs; }
PointCluster pc_unpack(const double* c) {
  PointCluster pc;
  pc.P(0, 0) = c[0]; pc.P(0, 1) = pc.P(1, 0) = c[1]; pc.P(0, 2) = pc.P(2, 0) = c[2]; pc.P(1, 1) = c[3]; pc.P(1, 2) = pc.P(2, 1) = c[4]; pc.P(2, 2) = c[5];
  pc.v = Eigen::Vector3d(c[6], c[7], c[8]); pc.N = int(c[9]);
  return pc;
}
void pc_pack(const PointCluster& pc, double* c) {
  c[0] = pc.P(0, 0); c[1] = pc.P(0, 1); c[2] = pc.P(0, 2); c[3] = pc.P(1, 1); c[4] = pc.P(1, 2); c[5] = pc.P(2, 2); c[6] = pc.v[0]; c[7] = pc.v[1]; c[8] = pc.v[2]; c[9] = pc.N;
}
void eig12_pack(const Eigen::Vector3d& w, const Eigen::Matrix3d& U, double* o) { for (int k = 0; k < 3; k++) o[k] = w[k]; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) o[3 + 3 * r + c] = U(r, c); }

// the reference keeps its map parameters in globals (voxel_map.hpp:82-89, loop_refine.hpp:269-271); voxelslam.cpp:805-833 fills them
int g_ring[4096];
void set_local_params(const vxs_map_params* p, int max_pts = 100) {
  voxel_size = p->voxel_size; min_eigen_value = p->min_eigen_value; max_layer = p->max_layer; max_points = max_pts;
  min_point << p->min_point[0], p->min_point[1], p->min_point[2], p->min_point[3];
  plane_eigen_value_thre.assign(8, p->plane_thre[3]);
  for (int k = 0; k < 4; k++) plane_eigen_value_thre[k] = p->plane_thre[k];
  for (int i = 0; i < 4096; i++) g_ring[i] = i;
  mp = g_ring;
}
void set_gba_params(const vxs_map_params* p) {
  gba_voxel_size = p->voxel_size; gba_min_eigen_value = p->min_eigen_value; max_layer = p->max_layer;
  gba_eigen_value_array.assign(8, p->plane_thre[3]);
  for (int k = 0; k < 4; k++) gba_eigen_value_array[k] = p->plane_thre[k];
}

struct RefFactor { LidarFactor f; vector<vxs_voxel_id> ids; explicit RefFactor(int w) : f(w) {} };

// identity (root cell, layer, octant path) of the leaves that tras_opt pushed, through opt_state (voxel_map.hpp:1320)
void collect_ids(OctoTree* o, const VOXEL_LOC& root, int path, vector<vxs_voxel_id>& ids) {
  if (o->octo_state == 0) {
    if (o->opt_state >= 0) {
      if (int(ids.size()) <= o->opt_state) ids.resize(size_t(o->opt_state) + 1);
      vxs_voxel_id id; id.x = root.x; id.y = root.y; id.z = root.z; id.layer = o->layer; id.path = path;
      ids[size_t(o->opt_state)] = id;
    }
    return;
  }
  for (int i = 0; i < 8; i++) if (o->leaves[i]) collect_ids(o->leaves[i], root, path * 8 + i, ids);
}
void free_tree(OctoTree* o) { for (int i = 0; i < 8; i++) if (o->leaves[i]) free_tree(o->leaves[i]); delete o->sw; delete o; }   // the reference leaks / recycles; tests free
void free_map(unordered_map<VOXEL_LOC, OctoTree*>& m) { for (auto& kv : m) free_tree(kv.second); m.clear(); }

PVecPtr make_pvec(const double* pts, int64_t n, double var_diag) {
  PVecPtr pv(new PVec(size_t(n)));
  for (int64_t k = 0; k < n; k++) { (*pv)[size_t(k)].pnt = Eigen::Vector3d(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2]); (*pv)[size_t(k)].var.setZero(); for (int d = 0; d < 3; d++) (*pv)[size_t(k)].var(d, d) = var_diag; }
  return pv;
}

}  // namespace

extern "C" {

int vxr_standin_eigen(void) { return VXREF_EIGEN_STANDIN; }
// var_init / pvec_update: the reference's own functions (voxelslam.hpp:187-214)
void vxr_var_init(const float* pts, int stride, int64_t n, const double* ext_R9, const double* ext_p3, double dept_err_, double beam_err_, double* pv12) {
  IMUST ext;
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) ext.R(r, c) = ext_R9[3 * r + c];
  for (int k = 0; k < 3; k++) ext.p[k] = ext_p3[k];
  pcl::PointCloud<PointType> pl;
  for (int64_t i = 0; i < n; i++) { PointType ap; ap.x = pts[size_t(i) * stride]; ap.y = pts[size_t(i) * stride + 1]; ap.z = pts[size_t(i) * stride + 2]; pl.push_back(ap); }
  PVecPtr pptr(new PVec);
  var_init(ext, pl, pptr, dept_err_, beam_err_);
  for (int64_t i = 0; i < n; i++) { const pointVar& pv = (*pptr)[size_t(i)]; for (int k = 0; k < 3; k++) pv12[12 * i + k] = pv.pnt[k]; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) pv12[12 * i + 3 + 3 * r + c] = pv.var(r, c); }
}
void vxr_pvec_update(double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, double* pwld_out) {
  PVecPtr pptr(new PVec(size_t(n)));
  for (int64_t i = 0; i < n; i++) { pointVar& pv = (*pptr)[size_t(i)]; pv.pnt = Eigen::Vector3d(pv12[12 * i], pv12[12 * i + 1], pv12[12 * i + 2]); for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) pv.var(r, c) = pv12[12 * i + 3 + 3 * r + c]; }
  IMUST x = state_from12(pose12);
  x.cov.setZero();
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { x.cov(r, c) = rot_var9[3 * r + c]; x.cov(3 + r, 3 + c) = tsl_var9[3 * r + c]; }
  PLV(3) pwld;
  pvec_update(pptr, x, pwld);
  for (int64_t i = 0; i < n; i++) { const pointVar& pv = (*pptr)[size_t(i)]; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) pv12[12 * i + 3 + 3 * r + c] = pv.var(r, c); for (int k = 0; k < 3; k++) pwld_out[3 * i + k] = pwld[size_t(i)][k]; }
}


// ---------------------------------------------------------------- primitives
void vxr_eig3(const double* A9_rowmajor, double* w3, double* U9_rowmajor) {
  Eigen::Matrix3d A;
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) A(r, c) = A9_rowmajor[3 * r + c];
  Eigen::SelfAdjointEigenSolver<Eigen::Matrix3d> saes(A);
  for (int k = 0; k < 3; k++) w3[k] = saes.eigenvalues()[k];
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) U9_rowmajor[3 * r + c] = saes.eigenvectors()(r, c);
}
// quantisation + hash as cut_voxel does them (voxel_map.hpp:1511-1518, tools.hpp:39-48): every point is cut into an empty map, the key of
// the root cell it creates is read back and hashed with std::hash<VOXEL_LOC>
void vxr_voxel_keys(const double* pw, int64_t n, double vs, int64_t* xyz, uint64_t* hash) {
  vxs_map_params p{}; p.voxel_size = vs; p.min_eigen_value = 0.0025; p.max_layer = 2; for (int k = 0; k < 4; k++) { p.min_point[k] = 5; p.plane_thre[k] = 0.25; }
  set_local_params(&p);
  vector<SlideWindow*> sws;
  for (int64_t i = 0; i < n; i++) {
    unordered_map<VOXEL_LOC, OctoTree*> m, ms;
    PVecPtr pv = make_pvec(pw + 3 * i, 1, 0.0);
    PLV(3) pwld; pwld.push_back((*pv)[0].pnt);
    cut_voxel(m, pv, 0, ms, 1, pwld, sws);
    const VOXEL_LOC& k = m.begin()->first;
    xyz[3 * i] = k.x; xyz[3 * i + 1] = k.y; xyz[3 * i + 2] = k.z;
    if (hash) hash[i] = uint64_t(std::hash<VOXEL_LOC>()(k));
    free_map(m);
  }
  for (SlideWindow* s : sws) delete s;
}
void vxr_cluster_from_points(const double* pts, int64_t n, double* c10) { PointCluster c; for (int64_t i = 0; i < n; i++) c.push(Eigen::Vector3d(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2])); pc_pack(c, c10); }
void vxr_cluster_transform(const double* c10, const double* pose12, double* out10) { PointCluster o; o.transform(pc_unpack(c10), state_from12(pose12)); pc_pack(o, out10); }
void vxr_so3_exp(const double* w, double* R9) { Eigen::Matrix3d R = Exp(Eigen::Vector3d(w[0], w[1], w[2])); for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) R9[3 * r + c] = R(r, c); }
int vxr_ldlt_solve(const double* A_colmajor, const double* b, int n, double* x) {     // the stand-in's LDLT (Eigen's published kernel), see Eigen/Core
  Eigen::MatrixXd A(n, n); Eigen::VectorXd bb(n);
  for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) A(i, j) = A_colmajor[size_t(j) * n + i];
  for (int i = 0; i < n; i++) bb[i] = b[i];
  Eigen::VectorXd xx = A.ldlt().solve(bb);
  for (int i = 0; i < n; i++) x[i] = xx[i];
  return 0;
}

// ---------------------------------------------------------------- LidarFactor (voxel_map.hpp:109-290)
void* vxr_factor_create(int W) { return new RefFactor(W); }
void vxr_factor_destroy(void* h) { delete static_cast<RefFactor*>(h); }
int64_t vxr_factor_size(void* h) { return int64_t(static_cast<RefFactor*>(h)->f.plvec_voxels.size()); }
int vxr_factor_win(void* h) { return static_cast<RefFactor*>(h)->f.win_size; }
void vxr_factor_push_dense(void* h, int64_t n, const double* clusters10, const double* fix10, const double* coe, const double* eig12, const double* sum10) {
  LidarFactor& f = static_cast<RefFactor*>(h)->f;
  const int W = f.win_size;
  for (int64_t v = 0; v < n; v++) {
    vector<PointCluster> pcs(W);
    for (int i = 0; i < W; i++) pcs[i] = pc_unpack(clusters10 + (size_t(v) * W + i) * 10);
    PointCluster fix = fix10 ? pc_unpack(fix10 + size_t(v) * 10) : PointCluster();
    Eigen::Vector3d w(eig12[12 * v], eig12[12 * v + 1], eig12[12 * v + 2]);
    Eigen::Matrix3d U; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) U(r, c) = eig12[12 * v + 3 + 3 * r + c];
    PointCluster add = pc_unpack(sum10 + size_t(v) * 10);
    f.push_voxel(pcs, fix, coe ? coe[v] : 1.0, w, U, add);
  }
}
void vxr_factor_export(void* h, double* clusters10, double* fix10, double* coe, double* eig12, double* sum10, vxs_voxel_id* ids) {
  RefFactor* rf = static_cast<RefFactor*>(h);
  LidarFactor& f = rf->f;
  const int W = f.win_size;
  for (size_t v = 0; v < f.plvec_voxels.size(); v++) {
    if (clusters10) for (int i = 0; i < W; i++) pc_pack(f.plvec_voxels[v][i], clusters10 + (v * W + i) * 10);
    if (fix10) pc_pack(f.sig_vecs[v], fix10 + v * 10);
    if (coe) coe[v] = f.coeffs[v];
    if (eig12) eig12_pack(f.eig_values[v], f.eig_vectors[v], eig12 + v * 12);
    if (sum10) pc_pack(f.pcr_adds[v], sum10 + v * 10);
    if (ids && v < rf->ids.size()) ids[v] = rf->ids[v];
  }
}
double vxr_factor_residual(void* h, const double* poses12) {
  LidarFactor& f = static_cast<RefFactor*>(h)->f;
  vector<IMUST> xs = states12(poses12, f.win_size);
  double r = 0; f.evaluate_only_residual(xs, 0, int(f.plvec_voxels.size()), r);
  return r;
}
double vxr_factor_hessian(void* h, const double* poses12, double* hess, double* jact) {
  LidarFactor& f = static_cast<RefFactor*>(h)->f;
  const int n = 6 * f.win_size;
  vector<IMUST> xs = states12(poses12, f.win_size);
  Eigen::MatrixXd H(n, n); Eigen::VectorXd J(n); double r = 0;
  f.acc_evaluate2(xs, 0, int(f.plvec_voxels.size()), H, J, r);
  if (hess) for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) hess[size_t(j) * n + i] = H(i, j);
  if (jact) for (int i = 0; i < n; i++) jact[i] = J[i];
  return r;
}
// timing of the reference's own threaded passes (Lidar_BA_Optimizer::divide_thread / only_residual with thd_num threads); seconds per pass
double vxr_time_hessian(void* h, const double* poses12, int threads, int reps, double* r_out) {
  LidarFactor& f = static_cast<RefFactor*>(h)->f;
  vector<IMUST> xs = states12(poses12, f.win_size);
  Lidar_BA_Optimizer opt; opt.thd_num = threads; opt.win_size = f.win_size; opt.jac_leng = 6 * f.win_size;
  Eigen::MatrixXd H(opt.jac_leng, opt.jac_leng); Eigen::VectorXd J(opt.jac_leng);
  auto t0 = std::chrono::steady_clock::now();
  double r = 0;
  for (int i = 0; i < reps; i++) r = opt.divide_thread(xs, f, H, J);
  const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (r_out) *r_out = r;
  return s / reps;
}
double vxr_time_residual(void* h, const double* poses12, int threads, int reps, double* r_out) {
  LidarFactor& f = static_cast<RefFactor*>(h)->f;
  vector<IMUST> xs = states12(poses12, f.win_size);
  Lidar_BA_Optimizer opt; opt.thd_num = threads; opt.win_size = f.win_size; opt.jac_leng = 6 * f.win_size;
  auto t0 = std::chrono::steady_clock::now();
  double r = 0;
  for (int i = 0; i < reps; i++) r = opt.only_residual(xs, f);
  const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (r_out) *r_out = r;
  return s / reps;
}

// ---------------------------------------------------------------- LM drivers
// Lidar_BA_Optimizer::damping_iter (voxel_map.hpp:367-442).  The reference keeps no per-iteration trace: *trace_len = 0.
int vxr_lidar_ba(void* h, double* poses12, int max_iter, int thd_num, double* hess_out, double* resis2, int* is_converge, vxs_lm_trace*, int, int* trace_len) {
  LidarFactor& f = static_cast<RefFactor*>(h)->f;
  const int W = f.win_size, n = 6 * W;
  if (int(f.plvec_voxels.size()) < thd_num) return VXS_ERR_TOO_FEW_VOXELS;   // the reference would printf + exit(0) (voxel_map.hpp:345-348)
  vector<IMUST> xs = states12(poses12, W);
  Lidar_BA_Optimizer opt; opt.thd_num = thd_num;
  Eigen::MatrixXd hess; vector<double> resis;
  const bool conv = opt.damping_iter(xs, f, &hess, resis, max_iter, false);
  for (int i = 0; i < W; i++) { double s[24]; state_to24(xs[i], s); std::memcpy(poses12 + 12 * i, s, 12 * 8); }
  if (hess_out && hess.rows() == n) for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) hess_out[size_t(j) * n + i] = hess(i, j);
  if (resis2) { resis2[0] = resis.size() > 0 ? resis[0] : 0; resis2[1] = resis.size() > 1 ? resis[1] : 0; }
  if (is_converge) *is_converge = conv ? 1 : 0;
  if (trace_len) *trace_len = 0;
  return 0;
}

// W-1 real IMU_PRE objects fed with the harness's seeded samples (tests/harness/synth.hpp ImuWindow::build draws the same sequence)
struct RefImu { deque<IMU_PRE*> pre, initial; ~RefImu() { for (auto p : pre) delete p; for (auto p : initial) delete p; } };
void* vxr_imu_create(const double* poses12_true, int W, double T, int samples, double gyr_noise, double acc_noise, uint64_t seed) {
  noiseMeas.setZero(); noiseWalk.setZero();                        // voxelslam.cpp:828-833 with config/avia.yaml:39-42
  for (int i = 0; i < 3; i++) { noiseMeas(i, i) = 0.01; noiseMeas(3 + i, 3 + i) = 1.0; noiseWalk(i, i) = 1e-4; noiseWalk(3 + i, 3 + i) = 1e-4; }
  imupre_scale_gravity = 1.0;
  RefImu* h = new RefImu();
  vxh::SplitMix64 g(seed);
  for (int i = 0; i + 1 < W; i++) {
    IMU_PRE* pre = new IMU_PRE();
    const double *Ri = poses12_true + 12 * i, *Rj = poses12_true + 12 * (i + 1);
    double RiT[9], dR[9], w[3];
    vxh::mat3_t(Ri, RiT); vxh::mat3_mul(RiT, Rj, dR); vxh::log3(dR, w);
    const double dt = T / samples;
    double Rcur[9];
    std::memcpy(Rcur, Ri, 72);
    for (int s = 0; s < samples; s++) {
      double gw[3] = {0, 0, 9.8}, acc[3], gyr[3];
      vxh::mat3_tvec(Rcur, gw, acc);
      for (int k = 0; k < 3; k++) { gyr[k] = w[k] / T + gyr_noise * g.gauss(); acc[k] += acc_noise * g.gauss(); }
      Eigen::Vector3d cur_gyr(gyr[0], gyr[1], gyr[2]), cur_acc(acc[0], acc[1], acc[2]);
      pre->add_imu(cur_gyr, cur_acc, dt);                            // preintegration.hpp:75-135 (bg = ba = 0 here, as in the harness)
      double wd[3] = {w[0] / T * dt, w[1] / T * dt, w[2] / T * dt}, E[9], Rn[9];
      vxh::exp3(wd, E); vxh::mat3_mul(Rcur, E, Rn); std::memcpy(Rcur, Rn, 72);
    }
    h->pre.push_back(pre);
    h->initial.push_back(new IMU_PRE(*pre));
  }
  return h;
}
void vxr_imu_destroy(void* h) { delete static_cast<RefImu*>(h); }
void vxr_imu_reset(void* hh) { RefImu* h = static_cast<RefImu*>(hh); for (size_t i = 0; i < h->pre.size(); i++) *h->pre[i] = *h->initial[i]; }
// sum over the factors of IMU_PRE::give_evaluate(_g) — same outputs as vxs_imu_hooks::eval (blocks bs x bs column-major per factor)
int vxr_imu_eval(void* hh, const double* states24, int W, int with_gravity, int want_jac, double* blocks, double* gvec, double* cost) {
  RefImu* h = static_cast<RefImu*>(hh);
  const int bs = with_gravity ? 33 : 30;
  double c = 0;
  for (int i = 0; i + 1 < W; i++) {
    IMUST a = state_from24(states24 + 24 * i), b = state_from24(states24 + 24 * (i + 1));
    Eigen::MatrixXd jtj(bs, bs); Eigen::VectorXd gg(bs);
    jtj.setZero(); gg.setZero();
    c += with_gravity ? h->pre[size_t(i)]->give_evaluate_g(a, b, jtj, gg, want_jac != 0) : h->pre[size_t(i)]->give_evaluate(a, b, jtj, gg, want_jac != 0);
    if (want_jac) { for (int q = 0; q < bs; q++) for (int p = 0; p < bs; p++) blocks[size_t(i) * bs * bs + size_t(q) * bs + p] = jtj(p, q); for (int p = 0; p < bs; p++) gvec[size_t(i) * bs + p] = gg[p]; }
  }
  *cost = c;
  return 0;
}
// LI_BA_Optimizer::damping_iter (voxel_map.hpp:562-653, 3 iterations hard-coded) / LI_BA_OptimizerGravity::damping_iter (:775-862)
int vxr_li_ba(void* h, double* states24, int with_gravity, int max_iter, double coef, void* imu, double* hess_out, double* resis2, vxs_lm_trace*, int, int* trace_len) {
  LidarFactor& f = static_cast<RefFactor*>(h)->f;
  RefImu* im = static_cast<RefImu*>(imu);
  const int W = f.win_size, n = 15 * W + (with_gravity ? 3 : 0);
  imu_coef = coef;
  vector<IMUST> xs(W);
  for (int i = 0; i < W; i++) xs[i] = state_from24(states24 + 24 * i);
  Eigen::MatrixXd hess; vector<double> resis;
  if (with_gravity) { LI_BA_OptimizerGravity opt; opt.damping_iter(xs, f, im->pre, resis, &hess, max_iter); }
  else { LI_BA_Optimizer opt; opt.damping_iter(xs, f, im->pre, &hess); }
  for (int i = 0; i < W; i++) state_to24(xs[i], states24 + 24 * i);
  if (hess_out && hess.rows() == n) for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) hess_out[size_t(j) * n + i] = hess(i, j);
  if (resis2) { resis2[0] = resis.size() > 0 ? resis[0] : 0; resis2[1] = resis.size() > 1 ? resis[1] : 0; }
  if (trace_len) *trace_len = 0;
  return 0;
}

// ---------------------------------------------------------------- voxel map, build from scratch (voxelslam.cpp:611-625: cut_voxel per scan, then recut + tras_opt per root)
void* vxr_build_window_factor(const vxs_map_params* mpar, const double* pts_body, const int64_t* scan_offsets, const double* poses12, int W, const double* fix_pts, int64_t n_fix,
                              int /*threads*/, double var_diag, double* seconds) {
  set_local_params(mpar);
  vector<IMUST> xs = states12(poses12, W);
  RefFactor* rf = new RefFactor(W);
  unordered_map<VOXEL_LOC, OctoTree*> surf_map, surf_map_slide;
  vector<SlideWindow*> sws;
  auto t0 = std::chrono::steady_clock::now();
  if (fix_pts && n_fix > 0) { PVecPtr fx = make_pvec(fix_pts, n_fix, var_diag); cut_voxel(surf_map, *fx, W, 0.0); }   // voxel_map.hpp:1641-1671
  for (int i = 0; i < W; i++) {
    PVecPtr pv = make_pvec(pts_body + 3 * scan_offsets[i], scan_offsets[i + 1] - scan_offsets[i], var_diag);
    PLV(3) pwld;
    for (pointVar& p : *pv) pwld.push_back(xs[i].R * p.pnt + xs[i].p);                                               // voxelslam.cpp:616
    cut_voxel(surf_map, pv, i, surf_map_slide, W, pwld, sws);
  }
  rf->f.clear(); rf->f.win_size = W;
  for (auto iter = surf_map.begin(); iter != surf_map.end(); ++iter) { iter->second->recut(W, xs, sws); iter->second->tras_opt(rf->f); }   // :620-624
  if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  for (auto& kv : surf_map) collect_ids(kv.second, kv.first, 0, rf->ids);
  rf->ids.resize(rf->f.plvec_voxels.size());
  free_map(surf_map);
  for (SlideWindow* s : sws) delete s;
  return rf;
}
// OctreeGBA::cut_voxel for every keyframe + OctreeGBA_multi_recut (loop_refine.hpp:446-479, 483-537).  No voxel identities (the GBA tree keeps
// no back reference): callers match voxels by their point sums.
void* vxr_build_gba_factor(const vxs_map_params* mpar, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, int W, int threads, double* seconds) {
  set_gba_params(mpar);
  vector<IMUST> xs = states12(poses12, W);
  RefFactor* rf = new RefFactor(W);
  unordered_map<VOXEL_LOC, OctreeGBA*> oct_map;
  auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < W; i++) {
    pcl::PointCloud<PointType>::Ptr pl(new pcl::PointCloud<PointType>());
    for (int64_t k = kf_offsets[i]; k < kf_offsets[i + 1]; k++) { PointType ap; ap.x = xyz[size_t(k) * stride_floats]; ap.y = xyz[size_t(k) * stride_floats + 1]; ap.z = xyz[size_t(k) * stride_floats + 2]; pl->push_back(ap); }
    OctreeGBA::cut_voxel(oct_map, xs[i], pl, i, W);
  }
  OctreeGBA_multi_recut(oct_map, rf->f, threads);
  if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return rf;
}

// The reference's own HBA_add_edge on W keyframe clouds (body frame) and poses: the outer coarse -> fine loop, the PGO edges of the final Hessian and (want_submap) the
// merged, down-sampled submap cloud in the frame of keyframe 0.  The function optimises a private copy of the poses (voxelslam.cpp:2326-2348): they are visible through
// the edges' relative poses only.  Returns the number of edges (all in map 0); *n_submap = points of the merged cloud.
int64_t vxr_hba_add_edge(const vxs_map_params* coarse, const vxs_map_params* fine, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, int W, int max_iter,
                         int thread_num, int want_submap, int64_t edge_cap, int32_t* eij, double* v6, double* rot, double* tra, int64_t sub_cap, float* sub_xyz, int64_t* n_submap) {
  set_gba_params(coarse);
  voxel_size = fine->voxel_size; min_eigen_value = fine->min_eigen_value;        // the globals the last outer iteration switches to (:2368-2371)
  plane_eigen_value_thre.assign(8, fine->plane_thre[3]);
  for (int k = 0; k < 4; k++) plane_eigen_value_thre[k] = fine->plane_thre[k];
  vector<IMUST> xs = states12(poses12, W);
  vector<Keyframe*> smps;
  for (int i = 0; i < W; i++) {
    Keyframe* kf = new Keyframe(xs[i]);
    kf->id = i; kf->mp = 0;
    for (int64_t k = kf_offsets[i]; k < kf_offsets[i + 1]; k++) { PointType ap; ap.x = xyz[size_t(k) * stride_floats]; ap.y = xyz[size_t(k) * stride_floats + 1]; ap.z = xyz[size_t(k) * stride_floats + 2]; kf->plptr->push_back(ap); }
    smps.push_back(kf);
  }
  PGO_Edges edges;
  vector<int> maps = {0};
  pcl::PointCloud<PointType>::Ptr sub;
  if (want_submap) sub.reset(new pcl::PointCloud<PointType>());
  RefHbaHost host;
  host.HBA_add_edge(xs, smps, edges, maps, max_iter, thread_num, sub);
  int64_t m = 0;
  for (PGO_Edge& e : edges.edges) for (size_t k = 0; k < e.ids1.size(); k++, m++) {
    if (m >= edge_cap) continue;
    eij[2 * m] = e.ids1[k]; eij[2 * m + 1] = e.ids2[k];
    for (int a = 0; a < 6; a++) v6[6 * m + a] = e.covs[k][a];
    for (int a = 0; a < 3; a++) { tra[3 * m + a] = e.tras[k][a]; for (int b = 0; b < 3; b++) rot[9 * m + 3 * a + b] = e.rots[k](a, b); }
  }
  if (n_submap) *n_submap = sub ? int64_t(sub->size()) : 0;
  if (sub) for (int64_t i = 0; i < int64_t(sub->size()) && i < sub_cap; i++) { const PointType& p = (*sub)[size_t(i)]; sub_xyz[3 * i] = p.x; sub_xyz[3 * i + 1] = p.y; sub_xyz[3 * i + 2] = p.z; }
  for (Keyframe* kf : smps) delete kf;
  return m;
}

// ---------------------------------------------------------------- down-sampling (tools.hpp:201-302, voxel_map.hpp:23-64); the cloud's first point index rides in `intensity`
int64_t vxr_down_sampling(int mode, const float* pts, int stride, int64_t n, double vs, float* xyz_out, float* cnt_out, int64_t* idx_out, int64_t cap) {
  if (vs < 0.001) return -1;
  pcl::PointCloud<PointType> pl;
  for (int64_t i = 0; i < n; i++) { PointType ap; ap.x = pts[size_t(i) * stride]; ap.y = pts[size_t(i) * stride + 1]; ap.z = pts[size_t(i) * stride + 2]; ap.curvature = 0; std::memcpy(&ap.data_c[2], &i, 8); pl.push_back(ap); }
  if (mode == 0) down_sampling_voxel(pl, vs); else down_sampling_close(pl, vs);
  for (int64_t i = 0; i < int64_t(pl.size()) && i < cap; i++) {
    const PointType& p = pl[size_t(i)];
    xyz_out[3 * i] = p.x; xyz_out[3 * i + 1] = p.y; xyz_out[3 * i + 2] = p.z;
    std::memcpy(&idx_out[i], &p.data_c[2], 8);
    cnt_out[i] = p.curvature;          // down_sampling_voxel: points in the cell; down_sampling_close keeps the picked point untouched (0)
  }
  return int64_t(pl.size());
}
int64_t vxr_down_sampling_pvec(const double* pv, int stride, int64_t n, double vs, float* xyz_out, float* nrm_out, float* cnt_out, int64_t* idx_out, int64_t cap) {
  PVec pvec; pvec.resize(size_t(n));
  for (int64_t i = 0; i < n; i++) { const double* p = pv + size_t(i) * stride; pvec[size_t(i)].pnt = Eigen::Vector3d(p[0], p[1], p[2]); for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) pvec[size_t(i)].var(r, c) = p[3 + 3 * r + c]; }
  pcl::PointCloud<PointType> keep;
  down_sampling_pvec(pvec, vs, keep);
  for (int64_t i = 0; i < int64_t(keep.size()) && i < cap; i++) {
    const PointType& p = keep[size_t(i)];
    xyz_out[3 * i] = p.x; xyz_out[3 * i + 1] = p.y; xyz_out[3 * i + 2] = p.z; nrm_out[3 * i] = p.normal_x; nrm_out[3 * i + 1] = p.normal_y; nrm_out[3 * i + 2] = p.normal_z;
    cnt_out[i] = 0; idx_out[i] = -1;   // the reference keeps neither the count nor an index here: callers match cells by position
  }
  return int64_t(keep.size());
}

// ---------------------------------------------------------------- stateful local map: margi / plane_update / match (voxel_map.hpp:1118-1146, 1196-1305, 1335-1392, 1674-1698)
struct RefLocalMap { unordered_map<VOXEL_LOC, OctoTree*> map, slide; vxs_map_params mp; int W; LidarFactor f; vector<SlideWindow*> sws; RefLocalMap(int w) : W(w), f(w) {} ~RefLocalMap() { free_map(map); for (auto s : sws) delete s; } };
void* vxr_local_map_build(const vxs_map_params* mpar, const double* pts_body, const int64_t* scan_offsets, const double* poses12, int W, double var_diag, int mgsize) {
  if (mgsize != 1) return nullptr;     // multi_margi hard-codes margi(win_cnt, 1, ...) (voxelslam.cpp:1360)
  RefLocalMap* h = new RefLocalMap(W);
  h->mp = *mpar;
  set_local_params(mpar);
  vector<IMUST> xs = states12(poses12, W);
  for (int i = 0; i < W; i++) {
    PVecPtr pv = make_pvec(pts_body + 3 * scan_offsets[i], scan_offsets[i + 1] - scan_offsets[i], var_diag);
    PLV(3) pwld;
    for (pointVar& p : *pv) pwld.push_back(xs[i].R * p.pnt + xs[i].p);
    cut_voxel(h->map, pv, i, h->slide, W, pwld, h->sws);
  }
  for (auto& kv : h->map) { kv.second->recut(W, xs, h->sws); kv.second->tras_opt(h->f); }
  for (auto& kv : h->map) kv.second->margi(W, 1, xs, h->f);
  return h;
}
void vxr_local_map_free(void* h) { delete static_cast<RefLocalMap*>(h); }
static void collect_planes(OctoTree* o, vector<OctoTree*>& out) {
  if (o->octo_state == 0) { if (o->plane.is_plane && o->plane.radius > 0) out.push_back(o); return; }
  for (int i = 0; i < 8; i++) if (o->leaves[i]) collect_planes(o->leaves[i], out);
}
int64_t vxr_local_map_planes(void* hh, double* rows52, int64_t cap) {
  RefLocalMap* h = static_cast<RefLocalMap*>(hh);
  vector<OctoTree*> pl;
  for (auto& kv : h->map) collect_planes(kv.second, pl);
  for (int64_t i = 0; i < int64_t(pl.size()) && i < cap; i++) {
    double* r = rows52 + 52 * i; OctoTree* o = pl[size_t(i)];
    for (int k = 0; k < 3; k++) { r[k] = o->plane.center[k]; r[3 + k] = o->plane.normal[k]; r[44 + k] = o->voxel_center[k]; r[49 + k] = o->eig_value[k]; }
    for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) r[6 + 6 * a + b] = o->plane.plane_var(a, b);
    r[42] = o->plane.radius; r[43] = o->pcr_add.N; r[47] = double(o->quater_length) * 2;
    double t = 0; for (int k = 0; k < 9; k++) t += o->cov_add(k, k);
    r[48] = t;
  }
  return int64_t(pl.size());
}
// the per-point loop of lio_state_estimation (voxelslam.cpp:876-918) around the reference's match()
static int odom_accum_impl(unordered_map<VOXEL_LOC, OctoTree*>& the_map, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, int passes, double* HTH36, double* HTz6,
                                  double* nnt9, int32_t* flags) {
  IMUST x_curr = state_from12(pose12);
  Eigen::Matrix3d rot_var, tsl_var;
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { rot_var(r, c) = rot_var9[3 * r + c]; tsl_var(r, c) = tsl_var9[3 * r + c]; }
  vector<OctoTree*> octos(size_t(n), nullptr);
  int match_num = 0;
  for (int pass = 0; pass < passes; pass++) {
    Eigen::Matrix<double, 6, 6> HTH; HTH.setZero();
    Eigen::Matrix<double, 6, 1> HTz; HTz.setZero();
    Eigen::Matrix3d nnt; nnt.setZero();
    match_num = 0;
    for (int64_t i = 0; i < n; i++) {
      pointVar pv; const double* p = pv12 + 12 * i;
      pv.pnt = Eigen::Vector3d(p[0], p[1], p[2]);
      for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) pv.var(r, c) = p[3 + 3 * r + c];
      Eigen::Matrix3d phat = hat(pv.pnt);
      Eigen::Matrix3d var_world = x_curr.R * pv.var * x_curr.R.transpose() + phat * rot_var * phat.transpose() + tsl_var;
      Eigen::Vector3d wld = x_curr.R * pv.pnt + x_curr.p;
      double sigma_d = 0;
      Plane* pla = nullptr;
      int flag = 0;
      if (octos[size_t(i)] != nullptr && octos[size_t(i)]->inside(wld)) { double max_prob = 0; flag = octos[size_t(i)]->match(wld, pla, max_prob, var_world, sigma_d, octos[size_t(i)]); }
      else flag = match(the_map, wld, pla, var_world, sigma_d, octos[size_t(i)]);
      if (flags && pass == passes - 1) flags[i] = flag;
      if (flag) {
        Plane& pp = *pla;
        double R_inv = 1.0 / (0.0005 + sigma_d);
        double resi = pp.normal.dot(wld - pp.center);
        Eigen::Matrix<double, 6, 1> jac;
        jac.head(3) = phat * x_curr.R.transpose() * pp.normal;
        jac.tail(3) = pp.normal;
        HTH += R_inv * jac * jac.transpose();
        HTz -= R_inv * jac * resi;
        nnt += pp.normal * pp.normal.transpose();
        match_num++;
      }
    }
    for (int a = 0; a < 6; a++) { for (int b = 0; b < 6; b++) HTH36[6 * a + b] = HTH(a, b); HTz6[a] = HTz[a]; }
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) nnt9[3 * a + b] = nnt(a, b);
  }
  return match_num;
}

int vxr_local_map_odom_accumulate(void* hh, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, int passes, double* HTH36, double* HTz6,
                                  double* nnt9, int32_t* flags) {
  RefLocalMap* h = static_cast<RefLocalMap*>(hh);
  set_local_params(&h->mp);
  return odom_accum_impl(h->map, pv12, n, pose12, rot_var9, tsl_var9, passes, HTH36, HTz6, nnt9, flags);
}

// The reference's own lio_state_estimation (up to 4 EKF iterations: association with the per-point leaf cache, 15x15 update, re-match rule, degeneracy test on nnt)
// on the local map.  state24 = R | p | v | bg | ba | g, cov225 row-major; both updated in place.  Returns the function's bool (1 = not degenerate).
int vxr_local_map_lio_state_estimation(void* hh, const double* pv12, int64_t n, double* state24, double* cov225) {
  RefLocalMap* h = static_cast<RefLocalMap*>(hh);
  set_local_params(&h->mp);
  PVecPtr pv(new PVec(size_t(n)));
  for (int64_t k = 0; k < n; k++) { const double* p = pv12 + 12 * k; (*pv)[size_t(k)].pnt = Eigen::Vector3d(p[0], p[1], p[2]); for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) (*pv)[size_t(k)].var(r, c) = p[3 + 3 * r + c]; }
  RefHbaHost host;
  host.x_curr = state_from24(state24);
  for (int r = 0; r < DIM; r++) for (int c = 0; c < DIM; c++) host.x_curr.cov(r, c) = cov225[DIM * r + c];
  host.surf_map.swap(h->map);
  const bool ok = host.lio_state_estimation(pv);
  host.surf_map.swap(h->map);
  state_to24(host.x_curr, state24);
  for (int r = 0; r < DIM; r++) for (int c = 0; c < DIM; c++) cov225[DIM * r + c] = host.x_curr.cov(r, c);
  return ok ? 1 : 0;
}

// ---------------------------------------------------------------- the per-scan map sequence of thd_odometry_localmapping (voxelslam.cpp:1599-1615, 1669-1712), poses given
struct RefSlidingSim {
  vxs_map_params mp; int win_size, mgsize, max_pts;
  vector<int> ring;
  unordered_map<VOXEL_LOC, OctoTree*> surf_map, surf_map_slide;
  vector<IMUST> x_buf;
  int win_count = 0, win_base = 0;
  LidarFactor voxhess;
  vector<SlideWindow*> sws;
  RefSlidingSim(const vxs_map_params& m, int w, int mg, int mxp) : mp(m), win_size(w), mgsize(mg), max_pts(mxp), ring(size_t(w)), voxhess(w) { for (int i = 0; i < w; i++) ring[size_t(i)] = i; }
  ~RefSlidingSim() { free_map(surf_map); for (auto s : sws) delete s; }
  void bind() { set_local_params(&mp, max_pts); mp_bind(); }
  void mp_bind() { ::mp = ring.data(); }
};
void* vxr_sliding_sim_create(const vxs_map_params* mpar, int win_size, int mgsize, int max_pts) { return mgsize == 1 ? new RefSlidingSim(*mpar, win_size, mgsize, max_pts) : nullptr; }
void vxr_sliding_sim_free(void* h) { delete static_cast<RefSlidingSim*>(h); }
static void ref_sim_add(RefSlidingSim* s, PVecPtr pv, const double* pose12, int ba_iters);
void vxr_sliding_sim_add_scan(void* hh, const double* pts_body, int64_t n, const double* pose12, double var_diag) { ref_sim_add(static_cast<RefSlidingSim*>(hh), make_pvec(pts_body, n, var_diag), pose12, 0); }
void vxr_sliding_sim_add_scan_pv(void* hh, const double* pv12, int64_t n, const double* pose12, int ba_iters) {
  PVecPtr pv(new PVec(size_t(n)));
  for (int64_t k = 0; k < n; k++) { const double* p = pv12 + 12 * k; (*pv)[size_t(k)].pnt = Eigen::Vector3d(p[0], p[1], p[2]); for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) (*pv)[size_t(k)].var(r, c) = p[3 + 3 * r + c]; }
  ref_sim_add(static_cast<RefSlidingSim*>(hh), pv, pose12, ba_iters);
}
void* vxr_sliding_sim_factor(void* hh) { RefSlidingSim* s = static_cast<RefSlidingSim*>(hh); RefFactor* rf = new RefFactor(s->win_size); rf->f = s->voxhess; return rf; }
static void ref_sim_add(RefSlidingSim* s, PVecPtr pv, const double* pose12, int ba_iters) {
  s->bind();
  IMUST x = state_from12(pose12);
  s->win_count++; s->x_buf.push_back(x);                                                   // :1599-1601
  s->voxhess.clear(); s->voxhess.win_size = s->win_size;                                   // :1609
  PLV(3) pwld;
  for (pointVar& p : *pv) pwld.push_back(x.R * p.pnt + x.p);
  cut_voxel(s->surf_map, pv, s->win_count - 1, s->surf_map_slide, s->win_size, pwld, s->sws);   // :1611 (the single-thread form of :1612)
  RefHbaHost host;                                                                          // thread_num = 1
  { vector<vector<SlideWindow*>> sws(1); sws[0].swap(s->sws); host.multi_recut(s->surf_map_slide, s->win_count, s->x_buf, s->voxhess, sws); s->sws.swap(sws[0]); }   // :1615, the reference's own function
  if (s->win_count >= s->win_size) {
    if (ba_iters > 0 && s->voxhess.plvec_voxels.size() >= 2) {                               // the BA between recut and margi (:1637-1654), pose-only flavour
      Lidar_BA_Optimizer opt; opt.thd_num = 2;
      Eigen::MatrixXd hess; vector<double> resis;
      opt.damping_iter(s->x_buf, s->voxhess, &hess, resis, ba_iters, false);
    }
    host.multi_margi(s->surf_map_slide, 0.0, s->win_count, s->x_buf, s->voxhess, s->sws);         // :1669, the reference's own function (jour only stamps the octrees)
    for (int i = 0; i < s->win_size; i++) { s->ring[size_t(i)] += s->mgsize; if (s->ring[size_t(i)] >= s->win_size) s->ring[size_t(i)] -= s->win_size; }                              // :1689-1693
    for (int i = s->mgsize; i < s->win_count; i++) s->x_buf[size_t(i - s->mgsize)] = s->x_buf[size_t(i)];                                                                             // :1695-1701
    for (int i = s->win_count - s->mgsize; i < s->win_count; i++) s->x_buf.pop_back();
    s->win_base += s->mgsize; s->win_count -= s->mgsize;
  }
}
static void collect_leaves(OctoTree* o, vector<OctoTree*>& out) {
  if (o->octo_state == 0) { out.push_back(o); return; }
  for (int i = 0; i < 8; i++) if (o->leaves[i]) collect_leaves(o->leaves[i], out);
}
int64_t vxr_sliding_sim_state(void* hh, int32_t* head, double* poses12, double* rows, int64_t cap) {
  RefSlidingSim* s = static_cast<RefSlidingSim*>(hh);
  const int W = s->win_size;
  head[0] = s->win_count; head[1] = s->win_base;
  for (int i = 0; i < W; i++) head[2 + i] = s->ring[size_t(i)];
  for (int i = 0; i < s->win_count; i++) { double st[24]; state_to24(s->x_buf[size_t(i)], st); std::memcpy(poses12 + 12 * i, st, 96); }
  vector<OctoTree*> lv; vector<char> in_slide;
  for (auto& kv : s->surf_map) { collect_leaves(kv.second, lv); in_slide.resize(lv.size(), s->surf_map_slide.count(kv.first) ? 1 : 0); }
  const int rw = 32 + 10 * W;
  for (int64_t t = 0; t < int64_t(lv.size()) && t < cap; t++) {
    double* r = rows + size_t(t) * rw; OctoTree* o = lv[size_t(t)];
    for (int k = 0; k < 3; k++) r[k] = o->voxel_center[k];
    r[3] = double(o->quater_length) * 2; r[4] = o->layer; r[5] = o->plane.is_plane; r[6] = o->isexist; r[7] = o->sw != nullptr; r[8] = in_slide[size_t(t)]; r[9] = o->opt_state; r[10] = o->last_num;
    r[11] = double(o->point_fix.size());
    pc_pack(o->pcr_add, r + 12); pc_pack(o->pcr_fix, r + 22);
    for (int i = 0; i < W; i++) { if (o->sw) pc_pack(o->sw->pcrs_local[size_t(s->ring[size_t(i)])], r + 32 + 10 * i); else for (int k = 0; k < 10; k++) r[32 + 10 * i + k] = 0; }
  }
  return int64_t(lv.size());
}

int64_t vxr_sliding_sim_planes(void* hh, double* rows52, int64_t cap) {
  RefSlidingSim* s = static_cast<RefSlidingSim*>(hh);
  vector<OctoTree*> pl;
  for (auto& kv : s->surf_map) collect_planes(kv.second, pl);
  for (int64_t i = 0; i < int64_t(pl.size()) && i < cap; i++) {
    double* r = rows52 + 52 * i; OctoTree* o = pl[size_t(i)];
    for (int k = 0; k < 3; k++) { r[k] = o->plane.center[k]; r[3 + k] = o->plane.normal[k]; r[44 + k] = o->voxel_center[k]; r[49 + k] = o->eig_value[k]; }
    for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) r[6 + 6 * a + b] = o->plane.plane_var(a, b);
    r[42] = o->plane.radius; r[43] = o->pcr_add.N; r[47] = double(o->quater_length) * 2;
    double t = 0; for (int k = 0; k < 9; k++) t += o->cov_add(k, k);
    r[48] = t;
  }
  return int64_t(pl.size());
}
int vxr_sliding_sim_odom_accumulate(void* hh, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, double* HTH36, double* HTz6, double* nnt9,
                                    int32_t* flags) {
  RefSlidingSim* s = static_cast<RefSlidingSim*>(hh);
  s->bind();
  return odom_accum_impl(s->surf_map, pv12, n, pose12, rot_var9, tsl_var9, 1, HTH36, HTz6, nnt9, flags);
}

}  // extern "C"
