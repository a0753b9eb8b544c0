// ORACLE — TEST INFRASTRUCTURE ONLY (see vxo_core.hpp header; parity unpinned).
//
// Voxel-map side of the hot path, restated from Voxel-SLAM/VoxelSLAM/src/:
//   voxel_map.hpp:1511-1518 (= loop_refine.hpp:452-459)  float quantisation      -> voxel_key
//   tools.hpp:24-49          VOXEL_LOC + hash                                    -> VoxelLoc, voxel_hash
//   voxel_map.hpp:896-930    SlideWindow
//   voxel_map.hpp:935-1333   OctoTree: push/push_fix*/plane_judge/allocate/allocate_fix/fix_divide/
//                            subdivide/recut/tras_opt
//   voxel_map.hpp:66-81, 1118-1146, 1196-1305, 1335-1392, 1471-1480, 1674-1698
//                            Plane, plane_update, margi, match, inside   (SURVEY 8f ranks 1 and 3: oracle only, no CUDA path yet)
//   voxelslam.cpp:876-918    one accumulation pass of the odometry EKF (HTH, HTz, nnt, match count)
//   voxel_map.hpp:1504-1540  cut_voxel (window)   :1641-1671 cut_voxel (fixed map points)
//   voxelslam.cpp:600-628    build-from-scratch sequence (cut all scans, then recut + tras_opt)
//   loop_refine.hpp:273-537  OctreeGBA, OctreeGBA_multi_recut
//   voxelslam.cpp:2360-2427  HBA_add_edge BA loop + PGO edge extraction
//   tools.hpp:201-302        down_sampling_voxel / down_sampling_close
#pragma once
#include <unordered_map>
#include "vxo_core.hpp"

namespace vxo {

struct VoxelLoc {
  int64_t x, y, z;
  bool operator==(const VoxelLoc& o) const { return x == o.x && y == o.y && z == o.z; }
};
// tools.hpp:39-48 with HASH_P=116101, MAX_N=10000000000 (tools.hpp:9-10); size_t wrap-around arithmetic
inline uint64_t voxel_hash(const VoxelLoc& s) {
  const uint64_t HP = 116101ull, MN = 10000000000ull;
  return (((uint64_t(s.z) * HP) % MN + uint64_t(s.y)) * HP) % MN + uint64_t(s.x);
}
struct VoxelLocHash { size_t operator()(const VoxelLoc& s) const { return size_t(voxel_hash(s)); } };

// voxel_map.hpp:1511-1518: float loc = pw/voxel_size; if(loc<0) loc -= 1; (int64_t)loc   (trap B#1)
inline VoxelLoc voxel_key(const V3& pw, double voxel_size) {
  int64_t k[3];
  for (int j = 0; j < 3; j++) {
    float loc = float(pw[j] / voxel_size);
    if (loc < 0) loc -= 1;
    k[j] = int64_t(loc);
  }
  return VoxelLoc{k[0], k[1], k[2]};
}

struct MapParams {
  double voxel_size = 1.0;           // voxel_map.hpp:87
  double min_eigen_value = 0.0025;   // voxel_map.hpp:84
  int max_layer = 2;                 // voxel_map.hpp:85
  double min_point[4] = {5, 5, 5, 5};              // voxelslam.cpp:812
  double plane_thre[8] = {.25, .25, .25, .25, .25, .25, .25, .25};  // plane_eigen_value_thre (already inverted, voxelslam.cpp:825)
  bool with_cov_add = false;         // voxel_map.hpp:990-992 by-product used only by plane_update (odometry)
  int max_points = 100;              // voxel_map.hpp:86
  const int* ring = nullptr;         // voxel_map.hpp:934 `int* mp`: logical window position -> slide-window slot (null = identity: from-scratch builds)
  int slot(int i) const { return ring ? ring[i] : i; }
};

// voxel_map.hpp:66-81 (is_plane lives on the OctoTree in this restatement)
struct Plane {
  V3 center = v3(0, 0, 0), normal = v3(0, 0, 0);
  double plane_var[36];   // row-major 6x6: [normal | center]
  float radius = 0;
  Plane() { for (double& x : plane_var) x = 0; }
};

struct PV { V3 pnt; M3 var; };  // voxel_map.hpp:14-19 pointVar

// voxel_map.hpp:91-106
inline void bf_var(const PV& pv, double bcov[81], const V3& vec) {
  double Bi[6][3] = {{2 * vec[0], 0, 0}, {vec[1], vec[0], 0}, {vec[2], 0, vec[0]}, {0, 2 * vec[1], 0}, {0, vec[2], vec[1]}, {0, 0, 2 * vec[2]}};
  double Biup[6][3];
  for (int r = 0; r < 6; r++) for (int c = 0; c < 3; c++) Biup[r][c] = (Bi[r][0] * pv.var(0, c) + Bi[r][1] * pv.var(1, c)) + Bi[r][2] * pv.var(2, c);
  for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) bcov[r * 9 + c] = (Biup[r][0] * Bi[c][0] + Biup[r][1] * Bi[c][1]) + Biup[r][2] * Bi[c][2];
  for (int r = 0; r < 6; r++) for (int c = 0; c < 3; c++) { bcov[r * 9 + 6 + c] = Biup[r][c]; bcov[(6 + c) * 9 + r] = Biup[r][c]; }
  for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) bcov[(6 + r) * 9 + 6 + c] = pv.var(r, c);
}

struct SlideWindow {  // voxel_map.hpp:896-930
  std::vector<std::vector<PV>> points;
  std::vector<PC> pcrs_local;
  explicit SlideWindow(int w) : points(w), pcrs_local(w) { for (auto& p : points) p.reserve(20); }
  void clear() { for (auto& p : points) p.clear(); for (auto& c : pcrs_local) c.clear(); }
};

// identification of a factor voxel for order-independent comparison in tests
struct VoxelId { int64_t x, y, z; int layer; int path; };  // path = sum leafnum_l * 8^(l-1)

struct OctoTree {  // voxel_map.hpp:935-1502
  SlideWindow* sw = nullptr;
  PC pcr_add;
  double cov_add[81];
  PC pcr_fix;
  std::vector<PV> point_fix;
  int layer, octo_state = 0, wdsize;
  OctoTree* leaves[8];
  double voxel_center[3];
  float quater_length;
  bool is_plane = false, isexist = false;
  V3 eig_value; M3 eig_vector;
  int opt_state = -1;
  int last_num = 0;
  Plane plane;
  VoxelLoc root{0, 0, 0}; int path = 0;  // bookkeeping for tests only

  OctoTree(int l, int w) : layer(l), wdsize(w) { for (auto& p : leaves) p = nullptr; std::memset(cov_add, 0, sizeof cov_add); }
  ~OctoTree() { for (auto p : leaves) delete p; delete sw; }

  void push(int ord, const PV& pv, const V3& pw, const MapParams& mp_) {  // :969-994 (the slide-window pool `sws` is an allocation detail)
    if (!sw) sw = new SlideWindow(wdsize);
    isexist = true;
    const int mord = mp_.slot(ord);
    if (layer < mp_.max_layer) sw->points[mord].push_back(pv);
    sw->pcrs_local[mord].push(pv.pnt);
    pcr_add.push(pw);
    if (mp_.with_cov_add) { double Bi[81]; bf_var(pv, Bi, pw); for (int i = 0; i < 81; i++) cov_add[i] += Bi[i]; }
  }
  void push_fix(const PV& pv, const MapParams& mp_) {  // :996-1005
    if (layer < mp_.max_layer) point_fix.push_back(pv);
    pcr_fix.push(pv.pnt); pcr_add.push(pv.pnt);
    if (mp_.with_cov_add) { double Bi[81]; bf_var(pv, Bi, pv.pnt); for (int i = 0; i < 81; i++) cov_add[i] += Bi[i]; }
  }
  void push_fix_novar(const PV& pv, const MapParams& mp_) {  // :1007-1013
    if (layer < mp_.max_layer) point_fix.push_back(pv);
    pcr_fix.push(pv.pnt); pcr_add.push(pv.pnt);
  }
  bool plane_judge(const V3& ev, const MapParams& mp_) const {  // :1015-1019
    return ev[0] < mp_.min_eigen_value && (ev[0] / ev[2]) < mp_.plane_thre[layer];
  }
  OctoTree* child_for(const V3& pw) {  // :1029-1041 (same code at :1056-1068, :1078-1089, :1101-1112)
    int xyz[3] = {0, 0, 0};
    for (int k = 0; k < 3; k++) if (pw[k] > voxel_center[k]) xyz[k] = 1;
    int leafnum = 4 * xyz[0] + 2 * xyz[1] + xyz[2];
    if (!leaves[leafnum]) {
      OctoTree* c = new OctoTree(layer + 1, wdsize);
      for (int k = 0; k < 3; k++) c->voxel_center[k] = voxel_center[k] + (2 * xyz[k] - 1) * quater_length;  // int*float -> float, then double +
      c->quater_length = quater_length / 2;
      c->root = root; c->path = path * 8 + leafnum;
      leaves[leafnum] = c;
    }
    return leaves[leafnum];
  }
  void allocate(int ord, const PV& pv, const V3& pw, const MapParams& mp_) {  // :1021-1046
    if (octo_state == 0) push(ord, pv, pw, mp_);
    else child_for(pw)->allocate(ord, pv, pw, mp_);
  }
  void allocate_fix(const PV& pv, const MapParams& mp_) {  // :1048-1072
    if (octo_state == 0) push_fix_novar(pv, mp_);
    else if (layer < mp_.max_layer) child_for(pv.pnt)->allocate_fix(pv, mp_);
  }
  void fix_divide(const MapParams& mp_) { for (const PV& pv : point_fix) child_for(pv.pnt)->push_fix(pv, mp_); }  // :1074-1094
  void subdivide(int si, const State& xx, const MapParams& mp_) {  // :1096-1116 — world point re-derived with the CURRENT pose
    for (const PV& pv : sw->points[mp_.slot(si)]) {
      V3 pw = xx.R * pv.pnt + xx.p;
      child_for(pw)->push(si, pv, pw, mp_);
    }
  }
  void recut(int win_count, const std::vector<State>& x_buf, const MapParams& mp_) {  // :1148-1194
    if (octo_state == 0) {
      if (layer >= 0) {
        opt_state = -1;
        if (pcr_add.N <= mp_.min_point[layer]) { is_plane = false; return; }
        if (!isexist || sw == nullptr) return;
        eig3_sym(pcr_add.cov(), eig_value, eig_vector);
        is_plane = plane_judge(eig_value, mp_);
        if (is_plane) return;
        else if (layer >= mp_.max_layer) return;
      }
      if (pcr_fix.N != 0) { fix_divide(mp_); std::vector<PV>().swap(point_fix); }
      for (int i = 0; i < win_count; i++) subdivide(i, x_buf[i], mp_);
      sw->clear(); delete sw; sw = nullptr;
      octo_state = 1;
    }
    for (auto c : leaves) if (c) c->recut(win_count, x_buf, mp_);
  }
  // voxel_map.hpp:1118-1146: plane centre, normal and their 6x6 covariance propagated from cov_add (the 9x9 covariance of the
  // cluster parameters [P(6) | v(3)] accumulated by bf_var) through d(normal)/d(cluster) = sum_k u_k f_kl / (N (lambda_l - lambda_k))
  void plane_update() {
    const double N = pcr_add.N;
    plane.center = v3(pcr_add.v[0] / N, pcr_add.v[1] / N, pcr_add.v[2] / N);
    const int l = 0;
    V3 u[3];
    for (int k = 0; k < 3; k++) u[k] = v3(eig_vector(0, k), eig_vector(1, k), eig_vector(2, k));
    const double nv = 1.0 / N;
    double u_c[3][9];
    for (auto& r : u_c) for (double& x : r) x = 0;
    for (int k = 0; k < 3; k++) {
      if (k == l) continue;
      double ukl[3][3];
      for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) ukl[a][b] = u[k][a] * u[l][b];
      double fkl[9] = {ukl[0][0], ukl[1][0] + ukl[0][1], ukl[2][0] + ukl[0][2], ukl[1][1], ukl[1][2] + ukl[2][1], ukl[2][2], 0, 0, 0};
      const double dk = dot(u[k], plane.center), dl = dot(u[l], plane.center);
      for (int a = 0; a < 3; a++) fkl[6 + a] = -(dk * u[l][a] + dl * u[k][a]);
      const double s = nv / (eig_value[l] - eig_value[k]);
      for (int a = 0; a < 3; a++) for (int c = 0; c < 9; c++) u_c[a][c] += s * u[k][a] * fkl[c];
    }
    double Jc[3][9];
    for (int a = 0; a < 3; a++) for (int c = 0; c < 9; c++) { double t = 0; for (int m = 0; m < 9; m++) t += u_c[a][m] * cov_add[m * 9 + c]; Jc[a][c] = t; }
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
      double t = 0; for (int m = 0; m < 9; m++) t += Jc[a][m] * u_c[b][m];
      plane.plane_var[a * 6 + b] = t;
      const double jn = nv * Jc[a][6 + b];
      plane.plane_var[a * 6 + 3 + b] = jn;
      plane.plane_var[(3 + b) * 6 + a] = jn;
      plane.plane_var[(3 + a) * 6 + 3 + b] = nv * nv * cov_add[(6 + a) * 9 + 6 + b];
    }
    plane.normal = u[0];
    plane.radius = float(eig_value[2]);
  }
  // voxel_map.hpp:1196-1305: marginalise the oldest `mgsize` scans of the window out of every leaf.  mp[] = logical window position ->
  // slide-window slot (voxel_map.hpp:934).  The "opt_state >= size" printf+exit of the reference is an assert-like guard (returns false).
  bool margi(int win_count, int mgsize, const std::vector<State>& x_buf, const LidarFactor& vox_opt, const std::vector<int>& mp, const MapParams& mp_) {
    if (octo_state == 0 && layer >= 0) {
      if (!isexist || sw == nullptr) return true;
      std::vector<PC> pcrs_world(wdsize);
      if (opt_state >= int(vox_opt.pcr_adds.size())) return false;
      if (opt_state >= 0) {
        pcr_add = vox_opt.pcr_adds[opt_state];
        eig_value = vox_opt.eig_values[opt_state];
        eig_vector = vox_opt.eig_vectors[opt_state];
        opt_state = -1;
        for (int i = 0; i < mgsize; i++)
          if (sw->pcrs_local[mp[i]].N != 0) pcrs_world[i].transform(sw->pcrs_local[mp[i]], x_buf[i].R, x_buf[i].p);
      } else {
        pcr_add = pcr_fix;
        for (int i = 0; i < win_count; i++)
          if (sw->pcrs_local[mp[i]].N != 0) { pcrs_world[i].transform(sw->pcrs_local[mp[i]], x_buf[i].R, x_buf[i].p); pcr_add += pcrs_world[i]; }
        if (is_plane) eig3_sym(pcr_add.cov(), eig_value, eig_vector);
      }
      if (pcr_fix.N < mp_.max_points && is_plane)
        if (pcr_add.N - last_num >= 5 || last_num <= 10) { plane_update(); last_num = int(pcr_add.N); }
      if (pcr_fix.N < mp_.max_points) {
        for (int i = 0; i < mgsize; i++)
          if (pcrs_world[i].N != 0) {
            pcr_fix += pcrs_world[i];
            for (PV pv : sw->points[mp[i]]) { pv.pnt = x_buf[i].R * pv.pnt + x_buf[i].p; point_fix.push_back(pv); }
          }
      } else {
        for (int i = 0; i < mgsize; i++) if (pcrs_world[i].N != 0) pcr_add -= pcrs_world[i];
        if (!point_fix.empty()) std::vector<PV>().swap(point_fix);
      }
      for (int i = 0; i < mgsize; i++)
        if (sw->pcrs_local[mp[i]].N != 0) { sw->pcrs_local[mp[i]].clear(); sw->points[mp[i]].clear(); }
      isexist = !(pcr_fix.N >= pcr_add.N);
      return true;
    }
    isexist = false;
    bool ok = true;
    for (auto c : leaves) if (c) { ok = c->margi(win_count, mgsize, x_buf, vox_opt, mp, mp_) && ok; isexist = isexist || c->isexist; }
    return ok;
  }
  bool inside(const V3& wld) const {  // voxel_map.hpp:1471-1480
    const double hl = quater_length * 2;
    for (int k = 0; k < 3; k++) if (!(wld[k] >= voxel_center[k] - hl && wld[k] <= voxel_center[k] + hl)) return false;
    return true;
  }
  // voxel_map.hpp:1335-1392: descend to the leaf that contains wld; accept its plane if the point lies within 3 sqrt(radius) of the
  // centre (in-plane) and within 3 sigma of the plane, sigma^2 = J plane_var J^T + n^T var_wld n.  float intermediates as in the reference.
  int match(const V3& wld, const Plane*& pla, const M3& var_wld, double& sigma_d, OctoTree*& oc) {
    int flag = 0;
    if (octo_state == 0) {
      if (is_plane) {
        const V3 d = wld - plane.center;
        const float dis_to_plane = float(std::fabs(dot(plane.normal, d)));
        const float dis_to_center = float(dot(d, d));
        const float range_dis = dis_to_center - dis_to_plane * dis_to_plane;
        if (range_dis <= 3 * 3 * plane.radius) {
          const double J[6] = {d[0], d[1], d[2], -plane.normal[0], -plane.normal[1], -plane.normal[2]};
          double sigma_l = 0;
          for (int a = 0; a < 6; a++) { double t = 0; for (int b = 0; b < 6; b++) t += plane.plane_var[a * 6 + b] * J[b]; sigma_l += J[a] * t; }
          sigma_l += dot(plane.normal, var_wld * plane.normal);
          if (dis_to_plane < 3 * std::sqrt(sigma_l)) { oc = this; sigma_d = sigma_l; pla = &plane; flag = 1; }
        }
      }
    } else {
      int xyz[3] = {0, 0, 0};
      for (int k = 0; k < 3; k++) if (wld[k] > voxel_center[k]) xyz[k] = 1;
      const int leafnum = 4 * xyz[0] + 2 * xyz[1] + xyz[2];
      if (leaves[leafnum] != nullptr) flag = leaves[leafnum]->match(wld, pla, var_wld, sigma_d, oc);
    }
    return flag;
  }
  void tras_opt(LidarFactor& vox_opt, std::vector<VoxelId>* ids, const int* ring_ = nullptr) {  // :1308-1333
    if (octo_state == 0) {
      if (layer >= 0 && isexist && is_plane && sw != nullptr) {
        if (eig_value[0] / eig_value[1] > 0.12) return;
        std::vector<PC> pcrs(wdsize);
        for (int i = 0; i < wdsize; i++) pcrs[i] = sw->pcrs_local[ring_ ? ring_[i] : i];   // :1317-1319 pcrs[i] = sw->pcrs_local[mp[i]]
        opt_state = int(vox_opt.size());
        vox_opt.push_voxel(pcrs, pcr_fix, 1.0, eig_value, eig_vector, pcr_add);
        if (ids) ids->push_back(VoxelId{root.x, root.y, root.z, layer, path});
      }
    } else
      for (auto c : leaves) if (c) c->tras_opt(vox_opt, ids, ring_);
  }
  void clear_slwd() {  // :1482-1500 (the windows go back to a pool in the reference; here they are freed)
    if (octo_state != 0) for (auto c : leaves) if (c) c->clear_slwd();
    if (sw) { delete sw; sw = nullptr; }
  }
};

using LocalMap = std::unordered_map<VoxelLoc, OctoTree*, VoxelLocHash>;
inline void local_map_free(LocalMap& m) { for (auto& kv : m) delete kv.second; m.clear(); }

// voxel_map.hpp:1674-1698: root-cell lookup, then OctoTree::match
inline int match(LocalMap& feat_map, const V3& wld, const Plane*& pla, const M3& var_wld, double& sigma_d, OctoTree*& oc, double voxel_size) {
  auto it = feat_map.find(voxel_key(wld, voxel_size));
  if (it == feat_map.end()) return 0;
  return it->second->match(wld, pla, var_wld, sigma_d, oc);
}
// voxelslam.cpp:876-918: one pass over the scan inside the odometry EKF iteration.  octos: per-point cache of the matched leaf
// (voxelslam.cpp:866-867, 892-900).  HTH 6x6 row-major, HTz 6, nnt 3x3 row-major.  Returns the number of matched points.
inline int odom_accumulate(LocalMap& surf_map, const std::vector<PV>& pvec, const State& x, const M3& rot_var, const M3& tsl_var, double voxel_size,
                           std::vector<OctoTree*>& octos, double HTH[36], double HTz[6], double nnt[9]) {
  for (int i = 0; i < 36; i++) HTH[i] = 0;
  for (int i = 0; i < 6; i++) HTz[i] = 0;
  for (int i = 0; i < 9; i++) nnt[i] = 0;
  int match_num = 0;
  octos.resize(pvec.size(), nullptr);
  const M3 Rt = tr(x.R);
  for (size_t i = 0; i < pvec.size(); i++) {
    const PV& pv = pvec[i];
    const M3 phat = hat(pv.pnt);
    const M3 var_world = (x.R * pv.var * Rt + phat * rot_var * tr(phat)) + tsl_var;
    const V3 wld = x.R * pv.pnt + x.p;
    double sigma_d = 0;
    const Plane* pla = nullptr;
    int flag;
    if (octos[i] != nullptr && octos[i]->inside(wld)) flag = octos[i]->match(wld, pla, var_world, sigma_d, octos[i]);
    else flag = match(surf_map, wld, pla, var_world, sigma_d, octos[i], voxel_size);
    if (!flag) continue;
    const double R_inv = 1.0 / (0.0005 + sigma_d);
    const double resi = dot(pla->normal, wld - pla->center);
    const V3 jh = phat * (Rt * pla->normal);
    const double jac[6] = {jh[0], jh[1], jh[2], pla->normal[0], pla->normal[1], pla->normal[2]};
    for (int a = 0; a < 6; a++) { for (int b = 0; b < 6; b++) HTH[a * 6 + b] += R_inv * jac[a] * jac[b]; HTz[a] -= R_inv * jac[a] * resi; }
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) nnt[a * 3 + b] += pla->normal[a] * pla->normal[b];
    match_num++;
  }
  return match_num;
}

// voxelslam.hpp:163-184 calcBodyVar: range / bearing noise of one point in the sensor frame.  The reference's float intermediates are kept
// (`const float range_inc, degree_inc` parameters, `float range`, `float range_var`); DEG2RAD(x) = ((x)*0.017453293) (pcl_macros.h).
inline void calc_body_var(V3& pb, const float range_inc, const float degree_inc, M3& var) {
  if (pb[2] == 0) pb[2] = 0.0001;
  float range = std::sqrt(pb[0] * pb[0] + pb[1] * pb[1] + pb[2] * pb[2]);
  float range_var = range_inc * range_inc;
  const double dv = std::pow(std::sin(degree_inc * 0.017453293), 2);
  const double nrm = std::sqrt((pb[0] * pb[0] + pb[1] * pb[1]) + pb[2] * pb[2]);
  const V3 direction = v3(pb[0] / nrm, pb[1] / nrm, pb[2] / nrm);
  const M3 direction_hat = hat(direction);
  V3 b1 = v3(1, 1, -(direction[0] + direction[1]) / direction[2]);
  { const double l = std::sqrt((b1[0] * b1[0] + b1[1] * b1[1]) + b1[2] * b1[2]); b1 = v3(b1[0] / l, b1[1] / l, b1[2] / l); }
  V3 b2 = v3(b1[1] * direction[2] - b1[2] * direction[1], b1[2] * direction[0] - b1[0] * direction[2], b1[0] * direction[1] - b1[1] * direction[0]);   // base_vector1.cross(direction)
  { const double l = std::sqrt((b2[0] * b2[0] + b2[1] * b2[1]) + b2[2] * b2[2]); b2 = v3(b2[0] / l, b2[1] / l, b2[2] / l); }
  // A = range * direction_hat * N,  N = [b1 b2] (3 x 2)
  double A[3][2];
  for (int a = 0; a < 3; a++) {
    A[a][0] = ((double(range) * direction_hat(a, 0)) * b1[0] + (double(range) * direction_hat(a, 1)) * b1[1]) + (double(range) * direction_hat(a, 2)) * b1[2];
    A[a][1] = ((double(range) * direction_hat(a, 0)) * b2[0] + (double(range) * direction_hat(a, 1)) * b2[1]) + (double(range) * direction_hat(a, 2)) * b2[2];
  }
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) var(a, b) = (direction[a] * double(range_var)) * direction[b] + ((A[a][0] * dv) * A[b][0] + (A[a][1] * dv) * A[b][1]);
}
// voxelslam.hpp:187-203 var_init: pts = x, y, z float (PointType), stride floats apart
inline void var_init(const M3& ext_R, const V3& ext_p, const float* pts, int stride, int64_t n, double dept_err, double beam_err, std::vector<PV>& out) {
  out.resize(size_t(n));
  for (int64_t i = 0; i < n; i++) {
    PV& pv = out[size_t(i)];
    pv.pnt = v3(pts[size_t(i) * stride], pts[size_t(i) * stride + 1], pts[size_t(i) * stride + 2]);
    calc_body_var(pv.pnt, float(dept_err), float(beam_err), pv.var);
    pv.pnt = ext_R * pv.pnt + ext_p;
    pv.var = ext_R * pv.var * tr(ext_R);
  }
}
// voxelslam.hpp:205-214 pvec_update
inline void pvec_update(std::vector<PV>& pvec, const State& x, const M3& rot_var, const M3& tsl_var, std::vector<V3>& pwld) {
  for (PV& pv : pvec) {
    const M3 phat = hat(pv.pnt);
    pv.var = (x.R * pv.var * tr(x.R) + phat * rot_var * tr(phat)) + tsl_var;
    pwld.push_back(x.R * pv.pnt + x.p);
  }
}

// voxel_map.hpp:1504-1540 (feat_tem_map bookkeeping dropped: in a from-scratch build slide map == map)
inline void cut_voxel(LocalMap& feat_map, const std::vector<PV>& pvec, int win_count, int wdsize, const std::vector<V3>& pwld, const MapParams& mp_) {
  for (size_t i = 0; i < pvec.size(); i++) {
    VoxelLoc position = voxel_key(pwld[i], mp_.voxel_size);
    auto it = feat_map.find(position);
    if (it != feat_map.end()) { it->second->allocate(win_count, pvec[i], pwld[i], mp_); it->second->isexist = true; }
    else {
      OctoTree* ot = new OctoTree(0, wdsize);
      ot->root = position;
      ot->allocate(win_count, pvec[i], pwld[i], mp_);
      ot->voxel_center[0] = (0.5 + position.x) * mp_.voxel_size;
      ot->voxel_center[1] = (0.5 + position.y) * mp_.voxel_size;
      ot->voxel_center[2] = (0.5 + position.z) * mp_.voxel_size;
      ot->quater_length = float(mp_.voxel_size / 4.0);
      feat_map[position] = ot;
    }
  }
}
// voxel_map.hpp:1641-1671 — fixed (already-world) map points
inline void cut_voxel_fix(LocalMap& feat_map, const std::vector<PV>& pvec, int wdsize, const MapParams& mp_) {
  for (const PV& pv : pvec) {
    VoxelLoc position = voxel_key(pv.pnt, mp_.voxel_size);
    auto it = feat_map.find(position);
    if (it != feat_map.end()) it->second->allocate_fix(pv, mp_);
    else {
      OctoTree* ot = new OctoTree(0, wdsize);
      ot->root = position;
      ot->push_fix_novar(pv, mp_);
      ot->voxel_center[0] = (0.5 + position.x) * mp_.voxel_size;
      ot->voxel_center[1] = (0.5 + position.y) * mp_.voxel_size;
      ot->voxel_center[2] = (0.5 + position.z) * mp_.voxel_size;
      ot->quater_length = float(mp_.voxel_size / 4.0);
      feat_map[position] = ot;
    }
  }
}

// voxelslam.cpp:600-628 (motion_init) / :1171-1180 (loop_update): cut every scan of the window with the
// current poses, then recut(win_size) + tras_opt on every root.  `threads`>1 mirrors multi_recut
// (voxelslam.cpp:1398-1453: roots split into ranges, recut in threads, serial tras_opt).
inline void build_window_factor(LocalMap& map, const std::vector<std::vector<PV>>& scans, const std::vector<State>& xs, const MapParams& mp_,
                                int threads, LidarFactor& out, std::vector<VoxelId>* ids) {
  const int W = int(scans.size());
  std::vector<V3> pwld;
  for (int i = 0; i < W; i++) {
    pwld.resize(scans[i].size());
    for (size_t k = 0; k < scans[i].size(); k++) pwld[k] = xs[i].R * scans[i][k].pnt + xs[i].p;  // voxelslam.cpp:616
    cut_voxel(map, scans[i], i, W, pwld, mp_);
  }
  std::vector<OctoTree*> roots;
  for (auto& kv : map) roots.push_back(kv.second);
  if (threads <= 1 || int(roots.size()) < threads) {
    for (auto r : roots) r->recut(W, xs, mp_);
  } else {
    std::vector<std::vector<OctoTree*>> octss(threads);
    double part = 1.0 * roots.size() / threads;
    int cnt = 0;
    for (auto r : roots) { octss[cnt].push_back(r); if (octss[cnt].size() >= part && cnt < threads - 1) cnt++; }
    std::vector<std::thread> th;
    for (int i = 1; i < threads; i++) th.emplace_back([&, i] { for (auto r : octss[i]) r->recut(W, xs, mp_); });
    for (auto r : octss[0]) r->recut(W, xs, mp_);
    for (auto& t : th) t.join();
  }
  for (auto r : roots) r->tras_opt(out, ids);
}

// ------------------------------------------------------------------ global-BA map  loop_refine.hpp:269-537
struct GbaParams {
  double voxel_size = 1.0;          // gba_voxel_size
  double min_eigen_value = 0.01;    // gba_min_eigen_value
  double eigen_value_array[8] = {.25, .25, .25, .25, .25, .25, .25, .25};  // gba_eigen_value_array (inverted, voxelslam.cpp:2490)
  int max_layer = 2;                // shares the global max_layer (loop_refine.hpp:391)
};

struct OctreeGBA {  // loop_refine.hpp:273-481
  std::vector<std::vector<V3>> locals, worlds;
  PC pcr_add;
  int layer, octo_state = 0, wdsize;
  OctreeGBA* leaves[8];
  double voxel_center[3];
  float quater_length;
  bool is_plane = false;
  VoxelLoc root{0, 0, 0}; int path = 0;
  OctreeGBA(int l, int w) : locals(w), worlds(w), layer(l), wdsize(w) { for (auto& p : leaves) p = nullptr; }
  ~OctreeGBA() { for (auto p : leaves) delete p; }
  void push(int ord, const V3& local, const V3& world) { locals[ord].push_back(local); worlds[ord].push_back(world); pcr_add.push(world); }  // :316-321
  void subdivide() {  // :323-356 — uses the STORED world points
    for (int i = 0; i < wdsize; i++)
      for (size_t j = 0; j < locals[i].size(); j++) {
        const V3& pw = worlds[i][j];
        int xyz[3] = {0, 0, 0};
        for (int k = 0; k < 3; k++) if (pw[k] > voxel_center[k]) xyz[k] = 1;
        int leafnum = 4 * xyz[0] + 2 * xyz[1] + xyz[2];
        if (!leaves[leafnum]) {
          OctreeGBA* c = new OctreeGBA(layer + 1, wdsize);
          for (int k = 0; k < 3; k++) c->voxel_center[k] = voxel_center[k] + (2 * xyz[k] - 1) * quater_length;
          c->quater_length = quater_length / 2;
          c->root = root; c->path = path * 8 + leafnum;
          leaves[leafnum] = c;
        }
        leaves[leafnum]->push(i, locals[i][j], pw);
      }
  }
  void recut(LidarFactor& vox_opt, const GbaParams& gp, std::vector<VoxelId>* ids) {  // :358-405
    if (pcr_add.N <= 10) return;
    V3 ev; M3 evec;
    eig3_sym(pcr_add.cov(), ev, evec);
    is_plane = ev[0] < gp.min_eigen_value && (ev[0] / ev[2]) < gp.eigen_value_array[layer];
    if (is_plane) {
      if (pcr_add.N < 10) return;
      int exi = 0;
      for (int i = 0; i < wdsize; i++) if (!locals[i].empty()) exi++;
      if (exi <= 1) return;
      if (ev[0] / ev[1] > 0.12) return;
      std::vector<PC> pcrs(wdsize);
      for (int i = 0; i < wdsize; i++) for (const V3& v : locals[i]) pcrs[i].push(v);
      PC pcr_fix;
      vox_opt.push_voxel(pcrs, pcr_fix, 1.0, ev, evec, pcr_add);
      if (ids) ids->push_back(VoxelId{root.x, root.y, root.z, layer, path});
      return;
    } else if (layer >= gp.max_layer) return;
    else { subdivide(); octo_state = 1; }
    for (auto c : leaves) if (c) c->recut(vox_opt, gp, ids);
  }
};
using GbaMap = std::unordered_map<VoxelLoc, OctreeGBA*, VoxelLocHash>;

// loop_refine.hpp:446-479.  xyz are the keyframe's float points (pcl::PointXYZINormal x,y,z).
inline void gba_cut_voxel(GbaMap& feat_map, const State& xc, const float* xyz, size_t npts, int win_count, int wdsize, const GbaParams& gp) {
  for (size_t k = 0; k < npts; k++) {
    V3 local = v3(xyz[3 * k], xyz[3 * k + 1], xyz[3 * k + 2]);
    V3 world = xc.R * local + xc.p;
    VoxelLoc position = voxel_key(world, gp.voxel_size);
    auto it = feat_map.find(position);
    if (it != feat_map.end()) it->second->push(win_count, local, world);
    else {
      OctreeGBA* ot = new OctreeGBA(0, wdsize);
      ot->root = position;
      ot->push(win_count, local, world);
      ot->voxel_center[0] = (0.5 + position.x) * gp.voxel_size;
      ot->voxel_center[1] = (0.5 + position.y) * gp.voxel_size;
      ot->voxel_center[2] = (0.5 + position.z) * gp.voxel_size;
      ot->quater_length = float(gp.voxel_size / 4.0);
      feat_map[position] = ot;
    }
  }
}
// loop_refine.hpp:483-537: roots split into ranges, thread-private factors concatenated in thread order; the map is consumed.
inline void gba_multi_recut(GbaMap& feat_map, LidarFactor& voxhess, int thd_num, const GbaParams& gp, std::vector<VoxelId>* ids) {
  std::vector<std::vector<OctreeGBA*>> octss(thd_num);
  std::vector<LidarFactor> facs(thd_num, LidarFactor(voxhess.win_size));
  std::vector<std::vector<VoxelId>> idss(thd_num);
  double part = 1.0 * feat_map.size() / thd_num;
  int cnt = 0;
  for (auto& kv : feat_map) { octss[cnt].push_back(kv.second); if (octss[cnt].size() >= part && cnt < thd_num - 1) cnt++; }
  auto fn = [&](int i) { for (OctreeGBA* oc : octss[i]) { oc->recut(facs[i], gp, ids ? &idss[i] : nullptr); delete oc; } };
  std::vector<std::thread> th;
  for (int i = 1; i < thd_num; i++) th.emplace_back(fn, i);
  fn(0);
  for (auto& t : th) t.join();
  feat_map.clear();
  for (int i = 0; i < thd_num; i++) {
    for (size_t a = 0; a < facs[i].size(); a++)
      voxhess.push_voxel(facs[i].plvec_voxels[a], facs[i].sig_vecs[a], facs[i].coeffs[a], facs[i].eig_values[a], facs[i].eig_vectors[a], facs[i].pcr_adds[a]);
    if (ids) ids->insert(ids->end(), idss[i].begin(), idss[i].end());
  }
}

struct Keyframes {  // the cloud of each keyframe (float xyz, as PointXYZINormal stores them)
  std::vector<const float*> xyz;
  std::vector<size_t> npts;
};
struct PgoEdge { int i, j; double rot[9], tra[3], v6[6]; };

// voxelslam.cpp:2360-2427 — the BA loop of HBA_add_edge (coarse-to-fine switch to the LocalBA voxel parameters) and the
// PGO edge extraction from the last raw Hessian.  `fine` = {voxel_size, plane_eigen_value_thre, min_eigen_value} of LocalBA.
inline int hba_window(std::vector<State>& xs, const Keyframes& kf, GbaParams gp, const GbaParams& fine, int max_iter, int thread_num, Mat& hess,
                      std::vector<PgoEdge>* edges, std::vector<double>* resis_log) {
  const int wdsize = int(xs.size());
  int up = 4, converge_flag = 0, iters_run = 0;
  double converge_thre = 0.05;
  for (int iterCnt = 0; iterCnt < max_iter; iterCnt++) {
    if (converge_flag == 1 || iterCnt == max_iter - 1) {
      gp.voxel_size = fine.voxel_size; gp.min_eigen_value = fine.min_eigen_value;
      for (int k = 0; k < 8; k++) gp.eigen_value_array[k] = fine.eigen_value_array[k];
    }
    GbaMap oct_map;
    for (int i = 0; i < wdsize; i++) gba_cut_voxel(oct_map, xs[i], kf.xyz[i], kf.npts[i], i, wdsize, gp);
    LidarFactor voxhess(wdsize);
    gba_multi_recut(oct_map, voxhess, thread_num, gp, nullptr);
    std::vector<double> resis;
    int status = 0;
    bool is_converge = lidar_ba_damping_iter(xs, voxhess, &hess, resis, up, thread_num, nullptr, &status);
    iters_run++;
    if (status != 0) return -1;
    if (resis_log) { resis_log->push_back(resis[0]); resis_log->push_back(resis[1]); }
    if ((std::fabs(resis[0] - resis[1]) / resis[0] < converge_thre && is_converge) || (iterCnt == max_iter - 2 && converge_flag == 0)) {
      converge_thre = 0.01;
      if (converge_flag == 0) converge_flag = 1;
      else if (converge_flag == 1) break;
    }
  }
  if (edges) {
    for (int i = 0; i < wdsize - 1; i++)
      for (int j = i + 1; j < wdsize; j++) {
        bool isAdd = true;
        PgoEdge e; e.i = i; e.j = j;
        for (int k = 0; k < 6; k++) {
          double hc = std::fabs(hess(6 * i + k, 6 * j + k));
          if (hc < 1e-6) { isAdd = false; break; }
          e.v6[k] = 1.0 / hc;
        }
        if (!isAdd) continue;
        V3 t = tr(xs[i].R) * (xs[j].p - xs[i].p);
        M3 r = tr(xs[i].R) * xs[j].R;
        for (int a = 0; a < 3; a++) { e.tra[a] = t[a]; for (int b = 0; b < 3; b++) e.rot[3 * a + b] = r(a, b); }
        edges->push_back(e);
      }
  }
  return iters_run;
}


// ---------------------------------------------------------------- tools.hpp:201-302 voxel-grid down-sampling (float point clouds)
struct DsPoint { float x, y, z, cnt; int64_t idx; };
// float quantisation of a FLOAT coordinate (tools.hpp:210-215): loc = p / voxel_size (double division, stored as float); loc < 0: loc -= 1.0
inline VoxelLoc voxel_key_f(const float* p, double voxel_size) {
  int64_t k[3];
  for (int j = 0; j < 3; j++) {
    float loc = float(double(p[j]) / voxel_size);
    if (loc < 0) loc = float(double(loc) - 1.0);
    k[j] = int64_t(loc);
  }
  return VoxelLoc{k[0], k[1], k[2]};
}
// tools.hpp:201-238.  Returns false when voxel_size < 0.001 (cloud untouched).  out order = the map's iteration order (unspecified in
// the reference as well); idx = input index of the first point of the cell (the reference keeps that point's other fields), cnt = curvature.
inline bool down_sampling_voxel(const float* pts, int stride, int64_t n, double voxel_size, std::vector<DsPoint>& out) {
  out.clear();
  if (voxel_size < 0.001) return false;
  std::unordered_map<VoxelLoc, DsPoint, VoxelLocHash> feat_map;
  for (int64_t i = 0; i < n; i++) {
    const float* p = pts + size_t(i) * stride;
    const VoxelLoc position = voxel_key_f(p, voxel_size);
    auto it = feat_map.find(position);
    if (it == feat_map.end()) feat_map[position] = DsPoint{p[0], p[1], p[2], 1.0f, i};
    else {
      DsPoint& pp = it->second;                       // float arithmetic throughout (PointType fields are float)
      pp.x = (pp.x * pp.cnt + p[0]) / (pp.cnt + 1);
      pp.y = (pp.y * pp.cnt + p[1]) / (pp.cnt + 1);
      pp.z = (pp.z * pp.cnt + p[2]) / (pp.cnt + 1);
      pp.cnt += 1;
    }
  }
  for (auto& kv : feat_map) out.push_back(kv.second);
  return true;
}
// tools.hpp:240-302: the input point nearest to the cell's float centroid; idx = its input index
inline bool down_sampling_close(const float* pts, int stride, int64_t n, double voxel_size, std::vector<DsPoint>& out) {
  out.clear();
  if (voxel_size < 0.001) return false;
  std::unordered_map<VoxelLoc, std::vector<int64_t>, VoxelLocHash> feat_map;
  for (int64_t i = 0; i < n; i++) feat_map[voxel_key_f(pts + size_t(i) * stride, voxel_size)].push_back(i);
  for (auto& kv : feat_map) {
    const std::vector<int64_t>& pl = kv.second;
    const int plsize = int(pl.size());
    const float* p0 = pts + size_t(pl[0]) * stride;
    float bx = p0[0], by = p0[1], bz = p0[2];
    for (int i = 1; i < plsize; i++) { const float* pp = pts + size_t(pl[i]) * stride; bx += pp[0]; by += pp[1]; bz += pp[2]; }
    bx /= plsize; by /= plsize; bz /= plsize;
    double ndis = 100;
    int mnum = 0;
    for (int i = 0; i < plsize; i++) {
      const float* pp = pts + size_t(pl[i]) * stride;
      const double xx = bx - pp[0], yy = by - pp[1], zz = bz - pp[2];   // float differences, widened afterwards (tools.hpp:285-287)
      const double dis = xx * xx + yy * yy + zz * zz;
      if (dis < ndis) { mnum = i; ndis = dis; }
    }
    const float* pb = pts + size_t(pl[mnum]) * stride;
    out.push_back(DsPoint{pb[0], pb[1], pb[2], float(plsize), pl[mnum]});
  }
  return true;
}

// voxel_map.hpp:23-64 down_sampling_pvec: running fp64 mean of pnt and var per cell; pl_keep gets float(pnt) and float(diag(var)).
// pv records `stride` doubles apart: pnt [0..2], var [3..11].  out.{x,y,z} = point, nrm = the three diagonal variances, idx = first point.
struct DsPvec { float x, y, z, nx, ny, nz, cnt; int64_t idx; };
inline void down_sampling_pvec(const double* pv, int stride, int64_t n, double voxel_size, std::vector<DsPvec>& out) {
  struct Acc { double pnt[3]; double var[9]; int cnt; int64_t first; };
  std::unordered_map<VoxelLoc, Acc, VoxelLocHash> feat_map;
  for (int64_t i = 0; i < n; i++) {
    const double* p = pv + size_t(i) * stride;
    const VoxelLoc position = voxel_key(v3(p[0], p[1], p[2]), voxel_size);
    auto it = feat_map.find(position);
    if (it == feat_map.end()) {
      Acc a; for (int k = 0; k < 3; k++) a.pnt[k] = p[k]; for (int k = 0; k < 9; k++) a.var[k] = p[3 + k]; a.cnt = 1; a.first = i;
      feat_map[position] = a;
    } else {
      Acc& a = it->second;
      for (int k = 0; k < 3; k++) a.pnt[k] = (a.pnt[k] * a.cnt + p[k]) / (a.cnt + 1);
      for (int k = 0; k < 9; k++) a.var[k] = (a.var[k] * a.cnt + p[3 + k]) / (a.cnt + 1);
      a.cnt += 1;
    }
  }
  out.clear();
  for (auto& kv : feat_map) {
    const Acc& a = kv.second;
    out.push_back(DsPvec{float(a.pnt[0]), float(a.pnt[1]), float(a.pnt[2]), float(a.var[0]), float(a.var[4]), float(a.var[8]), float(a.cnt), a.first});
  }
}

// voxelslam.cpp:2428-2447: submap merge of HBA_add_edge.  xs: W poses (R row-major, p); clouds concatenated with kf_offsets.
// merged (n x 3 float) receives the transformed points; then down_sampling_voxel(voxel_size) (the caller passes voxel_size / 8).
inline bool submap_merge(const float* pts, int stride, const int64_t* kf_offsets, const double* poses12, int W, double voxel_size, std::vector<float>& merged,
                         std::vector<DsPoint>& out) {
  const int64_t n = kf_offsets[W];
  merged.assign(size_t(n) * 3, 0.0f);
  const double* P0 = poses12;
  for (int i = 0; i < W; i++) {
    const double* Pi = poses12 + 12 * size_t(i);
    double dR[9], dp[3];
    const double d[3] = {Pi[9] - P0[9], Pi[10] - P0[10], Pi[11] - P0[11]};
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) dR[3 * r + c] = (P0[r] * Pi[c] + P0[3 + r] * Pi[3 + c]) + P0[6 + r] * Pi[6 + c];   // xc.R.transpose() * xs[i].R
      dp[r] = (P0[r] * d[0] + P0[3 + r] * d[1]) + P0[6 + r] * d[2];                                                  // xc.R.transpose() * (xs[i].p - xc.p)
    }
    for (int64_t k = kf_offsets[i]; k < kf_offsets[i + 1]; k++) {
      const float* p = pts + size_t(k) * stride;
      const double x = p[0], y = p[1], z = p[2];
      for (int r = 0; r < 3; r++) merged[3 * size_t(k) + r] = float(((dR[3 * r] * x + dR[3 * r + 1] * y) + dR[3 * r + 2] * z) + dp[r]);    // v3 = dR * v3 + dp; ap.x = v3[0]
    }
  }
  return down_sampling_voxel(merged.data(), 3, n, voxel_size, out);
}

// ------------------------------------------------------------------ sliding-window local mapping, map side only
// voxelslam.cpp:1599-1686 without the odometry, the IMU and the BA solve (poses are given): per scan cut_voxel into the map and the
// slide map, multi_recut (+ tras_opt) on the slide map, and once the window is full multi_margi(mgsize), erase of the dead roots from
// the slide map, rotation of the slot ring and shift of the pose buffer.  Single-threaded (the thread split of multi_recut / multi_margi
// only partitions the roots).  The state after every scan is what the next round's device map has to reproduce.
struct SlidingWindowSim {
  MapParams mp_;
  int win_size, mgsize;
  std::vector<int> ring;
  LocalMap surf_map;                                   // owns the trees
  std::unordered_map<VoxelLoc, OctoTree*, VoxelLocHash> slide;   // roots touched inside the current window (not owning)
  std::vector<State> x_buf;
  int win_count = 0, win_base = 0;
  LidarFactor voxhess;
  SlidingWindowSim(const MapParams& m, int w, int mg) : mp_(m), win_size(w), mgsize(mg), ring(w), voxhess(w) {
    for (int i = 0; i < w; i++) ring[i] = i;
    mp_.with_cov_add = true;
    mp_.ring = ring.data();
  }
  ~SlidingWindowSim() { local_map_free(surf_map); }
  SlidingWindowSim(const SlidingWindowSim&) = delete;
  SlidingWindowSim& operator=(const SlidingWindowSim&) = delete;

  // ba_iters > 0: a pose-only BA (Lidar_BA_Optimizer::damping_iter) runs between tras_opt and margi once the window is full, as the LI-BA does in
  // the reference loop (voxelslam.cpp:1637-1654): x_buf moves and the factor's cached eig / pcr_adds are overwritten before margi reads them
  void add_scan(const std::vector<PV>& scan, const State& x, int ba_iters = 0) {
    win_count++;
    x_buf.push_back(x);
    voxhess.clear(); voxhess.win_size = win_size;
    for (const PV& pv : scan) {                        // cut_voxel, voxel_map.hpp:1504-1540
      const V3 pw = x.R * pv.pnt + x.p;
      const VoxelLoc position = voxel_key(pw, mp_.voxel_size);
      auto it = surf_map.find(position);
      OctoTree* ot;
      if (it != surf_map.end()) { ot = it->second; ot->allocate(win_count - 1, pv, pw, mp_); ot->isexist = true; }
      else {
        ot = new OctoTree(0, win_size);
        ot->root = position;
        ot->allocate(win_count - 1, pv, pw, mp_);
        for (int k = 0; k < 3; k++) ot->voxel_center[k] = (0.5 + (k == 0 ? position.x : k == 1 ? position.y : position.z)) * mp_.voxel_size;
        ot->quater_length = float(mp_.voxel_size / 4.0);
        surf_map[position] = ot;
      }
      slide[position] = ot;
    }
    for (auto& kv : slide) kv.second->recut(win_count, x_buf, mp_);            // multi_recut, voxelslam.cpp:1398-1446
    for (auto& kv : slide) kv.second->tras_opt(voxhess, nullptr, ring.data());
    if (win_count >= win_size) {
      if (ba_iters > 0 && int(voxhess.size()) >= 2) { Mat hess; std::vector<double> resis; int status = 0; lidar_ba_damping_iter(x_buf, voxhess, &hess, resis, ba_iters, 2, nullptr, &status); }
      std::vector<int> rg(ring);
      for (auto& kv : slide) kv.second->margi(win_count, mgsize, x_buf, voxhess, rg, mp_);   // multi_margi, :1321-1395
      for (auto it = slide.begin(); it != slide.end();) { if (it->second->isexist) ++it; else { it->second->clear_slwd(); it = slide.erase(it); } }
      for (int i = 0; i < win_size; i++) { ring[i] += mgsize; if (ring[i] >= win_size) ring[i] -= win_size; }   // :1658-1662
      for (int i = mgsize; i < win_count; i++) x_buf[i - mgsize] = x_buf[i];
      for (int i = 0; i < mgsize; i++) x_buf.pop_back();
      win_base += mgsize; win_count -= mgsize;
    }
  }
};

}  // namespace vxo
