// ORACLE — TEST INFRASTRUCTURE ONLY.  Never linked into, imported by, or executed from the product
// path (voxel_slam_b200/).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may use it.
//
// PARITY UNPINNED: the reference (hku-mars/Voxel-SLAM) ships no tests, golden vectors or fixtures
// for this path and cannot be compiled here (needs Eigen 3.3.7 / PCL / ROS, none present).  This
// file is a dependency-free CPU restatement of the reference algorithm; it is pinned instead by
// finite-difference checks, numpy.linalg.eigh / scipy cross-checks and metamorphic properties
// (tests/test_oracle_*.py).
//
// Restates (file:line are into Voxel-SLAM/VoxelSLAM/src/):
//   tools.hpp:51-66      Exp            -> so3_exp
//   tools.hpp:304-365    PointCluster   -> PC (push / cov / += / -= / transform)
//   voxel_map.hpp:109-290  LidarFactor  -> LidarFactor (push_voxel, acc_evaluate2, evaluate_only_residual)
//   voxel_map.hpp:293-444  Lidar_BA_Optimizer      -> lidar_ba_damping_iter
//   voxel_map.hpp:450-655  LI_BA_Optimizer         -> li_ba_damping_iter(gravity=false)
//   voxel_map.hpp:658-864  LI_BA_OptimizerGravity  -> li_ba_damping_iter(gravity=true)
// Third-party arithmetic restated from its published algorithm (Eigen 3.3.7, README.md:28):
//   SelfAdjointEigenSolver<Matrix3d>  -> eig3_sym (cyclic Jacobi, ascending; eigenvector signs free)
//   LDLT<MatrixXd,Lower>              -> ldlt_solve (left-looking, pivot = largest |diag| of the
//                                        not-yet-eliminated ORIGINAL diagonal, lower triangle only)
// Floating point canon: plain fp64, left-to-right sums, compile with -ffp-contract=off.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

namespace vxo {

// ------------------------------------------------------------------ small fixed-size algebra
struct V3 {
  double d[3];
  double& operator[](int i) { return d[i]; }
  const double& operator[](int i) const { return d[i]; }
};
struct M3 {  // row-major
  double m[3][3];
  double& operator()(int r, int c) { return m[r][c]; }
  const double& operator()(int r, int c) const { return m[r][c]; }
};

inline V3 v3(double a, double b, double c) { return V3{{a, b, c}}; }
inline V3 operator+(const V3& a, const V3& b) { return v3(a[0] + b[0], a[1] + b[1], a[2] + b[2]); }
inline V3 operator-(const V3& a, const V3& b) { return v3(a[0] - b[0], a[1] - b[1], a[2] - b[2]); }
inline V3 operator*(double s, const V3& a) { return v3(s * a[0], s * a[1], s * a[2]); }
inline double dot(const V3& a, const V3& b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
inline M3 m3_zero() { M3 r; std::memset(&r, 0, sizeof r); return r; }
inline M3 m3_eye() { M3 r = m3_zero(); r(0, 0) = r(1, 1) = r(2, 2) = 1.0; return r; }
inline M3 operator+(const M3& a, const M3& b) { M3 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r(i, j) = a(i, j) + b(i, j); return r; }
inline M3 operator-(const M3& a, const M3& b) { M3 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r(i, j) = a(i, j) - b(i, j); return r; }
inline M3 operator*(double s, const M3& a) { M3 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r(i, j) = s * a(i, j); return r; }
inline M3 operator*(const M3& a, const M3& b) {
  M3 r;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r(i, j) = (a(i, 0) * b(0, j) + a(i, 1) * b(1, j)) + a(i, 2) * b(2, j);
  return r;
}
inline V3 operator*(const M3& a, const V3& x) {
  return v3((a(0, 0) * x[0] + a(0, 1) * x[1]) + a(0, 2) * x[2], (a(1, 0) * x[0] + a(1, 1) * x[1]) + a(1, 2) * x[2],
            (a(2, 0) * x[0] + a(2, 1) * x[1]) + a(2, 2) * x[2]);
}
inline M3 tr(const M3& a) { M3 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r(i, j) = a(j, i); return r; }
inline M3 outer(const V3& a, const V3& b) { M3 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r(i, j) = a[i] * b[j]; return r; }
inline M3 hat(const V3& v) {  // tools.hpp:93-100 / SKEW_SYM_MATRX tools.hpp:11
  M3 r = m3_zero();
  r(0, 1) = -v[2]; r(0, 2) = v[1]; r(1, 0) = v[2]; r(1, 2) = -v[0]; r(2, 0) = -v[1]; r(2, 1) = v[0];
  return r;
}

// tools.hpp:51-66 — Rodrigues; identity below |w| < 1e-11
inline M3 so3_exp(const V3& w) {
  double n = std::sqrt(dot(w, w));
  if (n >= 1e-11) {
    V3 ax = (1.0 / n) * w;
    // reference divides (ang / ang_norm); keep the division form for closeness
    ax = v3(w[0] / n, w[1] / n, w[2] / n);
    M3 K = hat(ax);
    return m3_eye() + std::sin(n) * K + (1.0 - std::cos(n)) * (K * K);
  }
  return m3_eye();
}

// ------------------------------------------------------------------ state at the boundary
// tools.hpp:135-199 IMUST, pose part + the dofs the LI solvers touch.  24 doubles:
// R (row-major 9) | p | v | bg | ba | g
struct State {
  M3 R; V3 p, v, bg, ba, g;
};
constexpr int STATE_DOUBLES = 24;
inline State state_from(const double* s) {
  State x;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) x.R(i, j) = s[3 * i + j];
  for (int i = 0; i < 3; i++) { x.p[i] = s[9 + i]; x.v[i] = s[12 + i]; x.bg[i] = s[15 + i]; x.ba[i] = s[18 + i]; x.g[i] = s[21 + i]; }
  return x;
}
inline void state_to(const State& x, double* s) {
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) s[3 * i + j] = x.R(i, j);
  for (int i = 0; i < 3; i++) { s[9 + i] = x.p[i]; s[12 + i] = x.v[i]; s[15 + i] = x.bg[i]; s[18 + i] = x.ba[i]; s[21 + i] = x.g[i]; }
}

// ------------------------------------------------------------------ PointCluster  tools.hpp:304-365
struct PC {
  M3 P; V3 v; int N;
  PC() { clear(); }
  void clear() { P = m3_zero(); v = v3(0, 0, 0); N = 0; }
  void push(const V3& p) { N++; P = P + outer(p, p); v = v + p; }  // tools.hpp:326-331
  M3 cov() const {                                                  // tools.hpp:333-337
    V3 c = v3(v[0] / N, v[1] / N, v[2] / N);
    M3 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r(i, j) = P(i, j) / N - c[i] * c[j];
    return r;
  }
  PC& operator+=(const PC& o) { P = P + o.P; v = v + o.v; N += o.N; return *this; }
  PC& operator-=(const PC& o) { P = P - o.P; v = v - o.v; N -= o.N; return *this; }
  void transform(const PC& s, const M3& R, const V3& p) {  // tools.hpp:357-363
    N = s.N;
    V3 Rv = R * s.v;
    v = Rv + double(N) * p;
    M3 rp = outer(Rv, p);
    P = ((R * s.P) * tr(R) + rp + tr(rp)) + double(N) * outer(p, p);
  }
};
// packed boundary form: Pxx Pxy Pxz Pyy Pyz Pzz vx vy vz N  (10 doubles)
inline void pc_pack(const PC& c, double* o) {
  o[0] = c.P(0, 0); o[1] = c.P(0, 1); o[2] = c.P(0, 2); o[3] = c.P(1, 1); o[4] = c.P(1, 2); o[5] = c.P(2, 2);
  o[6] = c.v[0]; o[7] = c.v[1]; o[8] = c.v[2]; o[9] = double(c.N);
}
inline PC pc_unpack(const double* o) {
  PC c;
  c.P(0, 0) = o[0]; c.P(0, 1) = c.P(1, 0) = o[1]; c.P(0, 2) = c.P(2, 0) = o[2];
  c.P(1, 1) = o[3]; c.P(1, 2) = c.P(2, 1) = o[4]; c.P(2, 2) = o[5];
  c.v = v3(o[6], o[7], o[8]); c.N = int(o[9]);
  return c;
}

// ------------------------------------------------------------------ 3x3 symmetric eigensolver
// Stand-in for Eigen::SelfAdjointEigenSolver<Matrix3d> (voxel_map.hpp:267,1161; loop_refine.hpp:363):
// reads the lower triangle, eigenvalues ascending, eigenvectors in the COLUMNS of U.
// Cyclic Jacobi with Rutishauser's update; converges to full fp64 accuracy (checked vs numpy eigh).
inline void eig3_sym(const M3& A, V3& w, M3& U) {
  double a[3][3];
  for (int i = 0; i < 3; i++) for (int j = 0; j <= i; j++) a[i][j] = a[j][i] = A(i, j);
  double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 64; sweep++) {
    double dmax = std::fmax(std::fabs(a[0][0]), std::fmax(std::fabs(a[1][1]), std::fabs(a[2][2])));
    double omax = std::fmax(std::fabs(a[0][1]), std::fmax(std::fabs(a[0][2]), std::fabs(a[1][2])));
    if (omax == 0.0 || omax <= 1e-22 * dmax) break;
    for (int p = 0; p < 2; p++)
      for (int q = p + 1; q < 3; q++) {
        double apq = a[p][q];
        if (apq == 0.0) continue;
        double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
        double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c);
        double h = t * apq;
        a[p][p] -= h; a[q][q] += h; a[p][q] = a[q][p] = 0.0;
        int r = 3 - p - q;
        double g = a[r][p], hh = a[r][q];
        a[r][p] = a[p][r] = g - s * (hh + g * tau);
        a[r][q] = a[q][r] = hh + s * (g - hh * tau);
        for (int k = 0; k < 3; k++) {
          double vp = V[k][p], vq = V[k][q];
          V[k][p] = vp - s * (vq + vp * tau);
          V[k][q] = vq + s * (vp - vq * tau);
        }
      }
  }
  int idx[3] = {0, 1, 2};
  double ev[3] = {a[0][0], a[1][1], a[2][2]};
  for (int i = 0; i < 2; i++) for (int j = 0; j < 2 - i; j++) if (ev[idx[j]] > ev[idx[j + 1]]) { int t = idx[j]; idx[j] = idx[j + 1]; idx[j + 1] = t; }
  for (int k = 0; k < 3; k++) { w[k] = ev[idx[k]]; for (int r = 0; r < 3; r++) U(r, k) = V[r][idx[k]]; }
}

// ------------------------------------------------------------------ dense column-major matrix
struct Mat {
  int r = 0, c = 0;
  std::vector<double> a;
  Mat() {}
  Mat(int r_, int c_) : r(r_), c(c_), a(size_t(r_) * c_, 0.0) {}
  void resize(int r_, int c_) { r = r_; c = c_; a.assign(size_t(r_) * c_, 0.0); }
  void zero() { std::fill(a.begin(), a.end(), 0.0); }
  double& operator()(int i, int j) { return a[size_t(j) * r + i]; }
  const double& operator()(int i, int j) const { return a[size_t(j) * r + i]; }
};

// Eigen 3.3.7 LDLT<MatrixXd, Lower>::compute + solve, restated (unblocked left-looking kernel:
// at step k the pivot is the largest |diagonal| among rows k..n-1 — those diagonal entries have not
// been updated yet, so the pivot order is by ORIGINAL diagonal magnitude; symmetric swap; column k
// is then updated from the already finished columns).  Used at voxel_map.hpp:403,597,811.
// A is overwritten.  Returns false if a zero pivot was met (Eigen would keep going with zeros).
inline bool ldlt_solve(Mat& A, const std::vector<double>& b, std::vector<double>& x) {
  const int n = A.r;
  std::vector<int> tr_(n);
  std::vector<double> temp(n);
  bool ok = true;
  for (int k = 0; k < n; k++) {
    int p = k; double big = std::fabs(A(k, k));
    for (int i = k + 1; i < n; i++) { double v = std::fabs(A(i, i)); if (v > big) { big = v; p = i; } }
    tr_[k] = p;
    if (p != k) {
      for (int j = 0; j < k; j++) std::swap(A(k, j), A(p, j));
      for (int i = p + 1; i < n; i++) std::swap(A(i, k), A(i, p));
      std::swap(A(k, k), A(p, p));
      for (int i = k + 1; i < p; i++) std::swap(A(i, k), A(p, i));
    }
    int rs = n - k - 1;
    if (k > 0) {
      double s = 0;
      for (int j = 0; j < k; j++) { temp[j] = A(j, j) * A(k, j); s += A(k, j) * temp[j]; }
      A(k, k) -= s;
      for (int j = 0; j < k; j++) {
        double tj = temp[j];
        const double* col = &A(k + 1, j);
        double* dst = &A(k + 1, k);
        for (int i = 0; i < rs; i++) dst[i] -= col[i] * tj;
      }
    }
    double akk = A(k, k);
    if (std::fabs(akk) > 0) { for (int i = k + 1; i < n; i++) A(i, k) /= akk; }
    else ok = false;
  }
  x = b;
  for (int k = 0; k < n; k++) if (tr_[k] != k) std::swap(x[k], x[tr_[k]]);
  for (int j = 0; j < n; j++) { double xj = x[j]; for (int i = j + 1; i < n; i++) x[i] -= A(i, j) * xj; }
  for (int i = 0; i < n; i++) { double d = A(i, i); x[i] = (std::fabs(d) > 2.2250738585072014e-308) ? x[i] / d : 0.0; }
  for (int j = n - 1; j >= 0; j--) { double s = x[j]; for (int i = j + 1; i < n; i++) s -= A(i, j) * x[i]; x[j] = s; }
  for (int k = n - 1; k >= 0; k--) if (tr_[k] != k) std::swap(x[k], x[tr_[k]]);
  return ok;
}

// ------------------------------------------------------------------ LidarFactor  voxel_map.hpp:109-290
struct LidarFactor {
  std::vector<PC> sig_vecs;                    // fix clusters
  std::vector<std::vector<PC>> plvec_voxels;   // [voxel][win_size] body-frame clusters (dense, as the reference)
  std::vector<double> coeffs;
  std::vector<V3> eig_values;
  std::vector<M3> eig_vectors;
  std::vector<PC> pcr_adds;
  int win_size;
  explicit LidarFactor(int w) : win_size(w) {}

  void push_voxel(const std::vector<PC>& vec_orig, const PC& fix, double coe, const V3& ev, const M3& evec, const PC& pcr_add) {  // :122-130
    plvec_voxels.push_back(vec_orig); sig_vecs.push_back(fix); coeffs.push_back(coe);
    eig_values.push_back(ev); eig_vectors.push_back(evec); pcr_adds.push_back(pcr_add);
  }
  void clear() { sig_vecs.clear(); plvec_voxels.clear(); eig_values.clear(); eig_vectors.clear(); pcr_adds.clear(); coeffs.clear(); }  // :281-286
  size_t size() const { return plvec_voxels.size(); }

  // voxel_map.hpp:132-241.  Hess is (6W x 6W) column-major, JacT 6W.  Uses the CACHED eig / pcr_adds.
  void acc_evaluate2(const std::vector<State>& xs, int head, int end, Mat& Hess, std::vector<double>& JacT, double& residual) const {
    Hess.zero(); std::fill(JacT.begin(), JacT.end(), 0.0); residual = 0;
    const int W = win_size;
    std::vector<V3> viRiTuk(W);
    std::vector<M3> viRiTukukT(W);
    std::vector<double> Auk(size_t(W) * 18);  // [i][3][6] row-major
    auto A = [&](int i, int r, int c) -> double& { return Auk[size_t(i) * 18 + r * 6 + c]; };

    for (int a = head; a < end; a++) {
      const std::vector<PC>& sig_orig = plvec_voxels[a];
      double coe = coeffs[a];
      V3 lmbd = eig_values[a];
      const M3& U = eig_vectors[a];
      int NN = pcr_adds[a].N;
      V3 vBar = v3(pcr_adds[a].v[0] / NN, pcr_adds[a].v[1] / NN, pcr_adds[a].v[2] / NN);
      V3 u[3];
      for (int k = 0; k < 3; k++) u[k] = v3(U(0, k), U(1, k), U(2, k));
      const V3& uk = u[0];
      M3 ukukT = outer(uk, uk);
      M3 umumT = m3_zero();
      for (int i = 1; i < 3; i++) umumT = umumT + (2.0 / (lmbd[0] - lmbd[i])) * outer(u[i], u[i]);

      for (int i = 0; i < W; i++) if (sig_orig[i].N != 0) {
        const M3& Pi = sig_orig[i].P; const V3& vi = sig_orig[i].v; const M3& Ri = xs[i].R;
        double ni = sig_orig[i].N;
        M3 vihat = hat(vi);
        V3 RiTuk = tr(Ri) * uk;
        M3 RiTukhat = hat(RiTuk);
        V3 PiRiTuk = Pi * RiTuk;
        viRiTuk[i] = vihat * RiTuk;
        viRiTukukT[i] = outer(viRiTuk[i], uk);
        V3 ti_v = xs[i].p - vBar;
        double ukTti_v = dot(uk, ti_v);
        M3 combo1 = hat(PiRiTuk) + ukTti_v * vihat;
        V3 combo2 = Ri * vi + ni * ti_v;
        M3 left = (Ri * Pi + outer(ti_v, vi)) * RiTukhat - Ri * combo1;
        M3 right = outer(combo2, uk) + dot(combo2, uk) * m3_eye();
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { A(i, r, c) = left(r, c) / NN; A(i, r, c + 3) = right(r, c) / NN; }

        double jjt[6];
        for (int c = 0; c < 6; c++) jjt[c] = (A(i, 0, c) * uk[0] + A(i, 1, c) * uk[1]) + A(i, 2, c) * uk[2];
        for (int c = 0; c < 6; c++) JacT[6 * i + c] += coe * jjt[c];

        M3 HRt = (2.0 / NN * (1.0 - ni / NN)) * viRiTukukT[i];
        double Hb[6][6];
        {  // Auk^T * umumT * Auk
          double MA[3][6];
          for (int r = 0; r < 3; r++) for (int c = 0; c < 6; c++) MA[r][c] = (umumT(r, 0) * A(i, 0, c) + umumT(r, 1) * A(i, 1, c)) + umumT(r, 2) * A(i, 2, c);
          for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Hb[r][c] = (A(i, 0, r) * MA[0][c] + A(i, 1, r) * MA[1][c]) + A(i, 2, r) * MA[2][c];
        }
        M3 rr = (2.0 / NN) * ((combo1 - RiTukhat * Pi) * RiTukhat) - (2.0 / NN / NN) * outer(viRiTuk[i], viRiTuk[i]) - 0.5 * hat(v3(jjt[0], jjt[1], jjt[2]));
        double ttc = 2.0 / NN * (ni - ni * ni / NN);
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) {
          Hb[r][c] += rr(r, c); Hb[r][c + 3] += HRt(r, c); Hb[r + 3][c] += HRt(c, r); Hb[r + 3][c + 3] += ttc * ukukT(r, c);
        }
        for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Hess(6 * i + r, 6 * i + c) += coe * Hb[r][c];
      }

      for (int i = 0; i < W - 1; i++) if (sig_orig[i].N != 0) {
        double ni = sig_orig[i].N;
        double MAi[6][3];  // Auk_i^T * umumT
        for (int r = 0; r < 6; r++) for (int c = 0; c < 3; c++) MAi[r][c] = (A(i, 0, r) * umumT(0, c) + A(i, 1, r) * umumT(1, c)) + A(i, 2, r) * umumT(2, c);
        for (int j = i + 1; j < W; j++) if (sig_orig[j].N != 0) {
          double nj = sig_orig[j].N;
          double Hb[6][6];
          for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Hb[r][c] = (MAi[r][0] * A(j, 0, c) + MAi[r][1] * A(j, 1, c)) + MAi[r][2] * A(j, 2, c);
          double c0 = -2.0 / NN / NN, c1 = -2.0 * nj / NN / NN, c2 = -2.0 * ni / NN / NN, c3 = -2.0 * ni * nj / NN / NN;
          for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) {
            Hb[r][c] += c0 * viRiTuk[i][r] * viRiTuk[j][c];
            Hb[r][c + 3] += c1 * viRiTukukT[i](r, c);
            Hb[r + 3][c] += c2 * viRiTukukT[j](c, r);
            Hb[r + 3][c + 3] += c3 * ukukT(r, c);
          }
          for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Hess(6 * i + r, 6 * j + c) += coe * Hb[r][c];
        }
      }
      residual += coe * lmbd[0];
    }
    for (int i = 1; i < W; i++) for (int j = 0; j < i; j++)
      for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Hess(6 * i + r, 6 * j + c) = Hess(6 * j + c, 6 * i + r);
  }

  // voxel_map.hpp:243-279.  Overwrites the cached eig / pcr_adds (also when the LM step is rejected later).
  void evaluate_only_residual(const std::vector<State>& xs, int head, int end, double& residual) {
    residual = 0;
    PC pcr;
    for (int a = head; a < end; a++) {
      const std::vector<PC>& sig_orig = plvec_voxels[a];
      PC sig = sig_vecs[a];
      for (int i = 0; i < win_size; i++) if (sig_orig[i].N != 0) { pcr.transform(sig_orig[i], xs[i].R, xs[i].p); sig += pcr; }
      V3 w; M3 U;
      eig3_sym(sig.cov(), w, U);
      eig_values[a] = w; eig_vectors[a] = U; pcr_adds[a] = sig;
      residual += coeffs[a] * w[0];
    }
  }
};

// ------------------------------------------------------------------ thread fan-out shared by the 3 solvers
// voxel_map.hpp:298-335 / 465-523 — per-thread dense Hessians, serial sum after join; range bounds are
// double products truncated to int (trap B#10).
inline double lidar_hessian_threads(const std::vector<State>& xs, const LidarFactor& f, int thd_num, Mat& Hess, std::vector<double>& JacT) {
  const int n = f.win_size * 6;
  Hess.zero(); std::fill(JacT.begin(), JacT.end(), 0.0);
  int tthd = thd_num;
  int g_size = int(f.size());
  if (g_size < tthd) tthd = 1;
  std::vector<Mat> hs(tthd, Mat(n, n));
  std::vector<std::vector<double>> js(tthd, std::vector<double>(n));
  std::vector<double> rs(tthd, 0.0);
  double part = 1.0 * g_size / tthd;
  std::vector<std::thread> th;
  for (int i = 1; i < tthd; i++) th.emplace_back([&, i] { f.acc_evaluate2(xs, int(part * i), int(part * (i + 1)), hs[i], js[i], rs[i]); });
  f.acc_evaluate2(xs, 0, int(part), hs[0], js[0], rs[0]);
  double residual = 0;
  for (int i = 0; i < tthd; i++) {
    if (i) th[i - 1].join();
    for (size_t k = 0; k < Hess.a.size(); k++) Hess.a[k] += hs[i].a[k];
    for (int k = 0; k < n; k++) JacT[k] += js[i][k];
    residual += rs[i];
  }
  return residual;
}
inline double lidar_residual_threads(const std::vector<State>& xs, LidarFactor& f, int thd_num) {  // voxel_map.hpp:337-365
  int g_size = int(f.size());
  std::vector<double> rs(thd_num, 0.0);
  double part = 1.0 * g_size / thd_num;
  std::vector<std::thread> th;
  for (int i = 1; i < thd_num; i++) th.emplace_back([&, i] { f.evaluate_only_residual(xs, int(part * i), int(part * (i + 1)), rs[i]); });
  f.evaluate_only_residual(xs, 0, int(part), rs[0]);
  double r = 0;
  for (int i = 0; i < thd_num; i++) { if (i) th[i - 1].join(); r += rs[i]; }
  return r;
}

struct LmTrace { double r1, r2, u, v, q1; int accepted; };

// voxel_map.hpp:367-442  Lidar_BA_Optimizer::damping_iter.  status: 0 ok, -1 = reference would exit(0) ("Too Less Voxel").
inline bool lidar_ba_damping_iter(std::vector<State>& x_stats, LidarFactor& voxhess, Mat* hess, std::vector<double>& resis, int max_iter,
                                  int thd_num, std::vector<LmTrace>* trace, int* status) {
  const int W = voxhess.win_size, n = 6 * W;
  if (status) *status = 0;
  double u = 0.01, v = 2;
  Mat Hess(n, n), M(n, n);
  std::vector<double> JacT(n), dxi(n), D(n), rhs(n);
  hess->resize(n, n);
  double residual1 = 0, residual2 = 0, q;
  bool is_calc_hess = true, is_converge = true;
  std::vector<State> x_temp = x_stats;
  for (int i = 0; i < max_iter; i++) {
    if (is_calc_hess) { residual1 = lidar_hessian_threads(x_stats, voxhess, thd_num, Hess, JacT); *hess = Hess; }
    if (i == 0) resis.push_back(residual1);
    for (int r = 0; r < 6; r++) for (int c = 0; c < n; c++) { Hess(r, c) = 0; Hess(c, r) = 0; }
    for (int r = 0; r < 6; r++) { Hess(r, r) = 1.0; JacT[r] = 0; }
    for (int k = 0; k < n; k++) D[k] = Hess(k, k);
    M = Hess;
    for (int k = 0; k < n; k++) { M(k, k) += u * D[k]; rhs[k] = -JacT[k]; }
    ldlt_solve(M, rhs, dxi);
    for (int j = 0; j < W; j++) {
      x_temp[j].R = x_stats[j].R * so3_exp(v3(dxi[6 * j], dxi[6 * j + 1], dxi[6 * j + 2]));
      x_temp[j].p = x_stats[j].p + v3(dxi[6 * j + 3], dxi[6 * j + 4], dxi[6 * j + 5]);
    }
    double q1 = 0;
    for (int k = 0; k < n; k++) q1 += dxi[k] * (u * D[k] * dxi[k] - JacT[k]);
    q1 *= 0.5;
    if (int(voxhess.size()) < thd_num) { if (status) *status = -1; return false; }  // voxel_map.hpp:345-348 exit(0)
    residual2 = lidar_residual_threads(x_temp, voxhess, thd_num);
    q = residual1 - residual2;
    int acc = q > 0;
    if (trace) trace->push_back(LmTrace{residual1, residual2, u, v, q1, acc});
    if (q > 0) {
      x_stats = x_temp;
      double one_three = 1.0 / 3;
      q = q / q1; v = 2; q = 1 - std::pow(2 * q - 1, 3);
      u *= (q < one_three ? one_three : q);
      is_calc_hess = true;
    } else { u = u * v; v = 2 * v; is_calc_hess = false; is_converge = false; }
    if (std::fabs((residual1 - residual2) / residual1) < 1e-6) break;
  }
  resis.push_back(residual2);
  return is_converge;
}

// IMU side of the LI solvers stays outside (preintegration.hpp is not on the path): the caller supplies it.
//   eval(states, want_jac, blocks, gvec) -> sum of the W-1 factor costs r^T cov^-1 r (unscaled).
//     want_jac: blocks[(W-1)][bs*bs] column-major and gvec[(W-1)][bs], bs = 30 (33 with gravity:
//     the trailing 3 rows/cols are the gravity dofs)            == IMU_PRE::give_evaluate(_g)  preintegration.hpp:137,214
//   update(dxi)  == IMU_PRE::update_state for factor j with dxi.block<15,1>(15 j)                preintegration.hpp:296
//   rollback()   == dbg = dbg_buf; dba = dba_buf                                                 voxel_map.hpp:639-643
struct ImuHooks {
  std::function<double(const std::vector<State>&, bool, double*, double*)> eval;
  std::function<void(const double*)> update;
  std::function<void()> rollback;
};

// voxel_map.hpp:562-653 (gravity=false; fixed 3 iterations, gauge = 15 dofs of pose 0) and
// voxel_map.hpp:775-862 (gravity=true; n = 15W+3, gauge = 6 dofs).  imu_coef voxel_map.hpp:446.
inline void li_ba_damping_iter(std::vector<State>& x_stats, LidarFactor& voxhess, ImuHooks& imu, double imu_coef, bool gravity, int max_iter,
                               Mat* hess, std::vector<double>* resis, std::vector<LmTrace>* trace) {
  const int W = voxhess.win_size, DIMS = 15, n = W * DIMS + (gravity ? 3 : 0), nl = 6 * W;
  const int bs = gravity ? 33 : 30;
  const int thd_num = 5;
  double u = 0.01, v = 2;
  Mat Hess(n, n), M(n, n), hl(nl, nl);
  std::vector<double> JacT(n), dxi(n), D(n), rhs(n), jl(nl);
  std::vector<double> blocks(size_t(W - 1) * bs * bs), gvec(size_t(W - 1) * bs);
  hess->resize(n, n);
  double residual1 = 0, residual2 = 0, q;
  bool is_calc_hess = true;
  std::vector<State> x_temp = x_stats;
  // LI_BA_Optimizer hard-codes 3 iterations (voxel_map.hpp:581); a SMALLER max_iter steps fewer (single-iteration parity / timing), as vxs_li_ba does
  const int iters = gravity ? max_iter : (max_iter < 3 ? max_iter : 3);
  for (int it = 0; it < iters; it++) {
    if (is_calc_hess) {
      // divide_thread  voxel_map.hpp:465-523 / 673-736 (IMU part on the calling thread, then hess_plus)
      Hess.zero(); std::fill(JacT.begin(), JacT.end(), 0.0);
      double r_imu = imu.eval(x_stats, true, blocks.data(), gvec.data());
      for (int i = 0; i < W - 1; i++) {
        const double* B = &blocks[size_t(i) * bs * bs];
        const double* g = &gvec[size_t(i) * bs];
        auto gi = [&](int k) { return k < 30 ? i * DIMS + k : n - 3 + (k - 30); };
        for (int c = 0; c < bs; c++) { for (int r = 0; r < bs; r++) Hess(gi(r), gi(c)) += B[size_t(c) * bs + r]; JacT[gi(c)] += g[c]; }
      }
      for (double& h : Hess.a) h *= imu_coef;
      for (double& g : JacT) g *= imu_coef;
      double residual = r_imu * (imu_coef * 0.5);
      residual += lidar_hessian_threads(x_stats, voxhess, thd_num, hl, jl);
      for (int i = 0; i < W; i++) {  // hess_plus voxel_map.hpp:455-463
        for (int k = 0; k < 6; k++) JacT[i * DIMS + k] += jl[i * 6 + k];
        for (int j = 0; j < W; j++) for (int r = 0; r < 6; r++) for (int c = 0; c < 6; c++) Hess(i * DIMS + r, j * DIMS + c) += hl(i * 6 + r, j * 6 + c);
      }
      residual1 = residual;
      *hess = Hess;
    }
    if (gravity && it == 0 && resis) resis->push_back(residual1);
    const int gf = gravity ? 6 : DIMS;
    for (int r = 0; r < gf; r++) for (int c = 0; c < n; c++) { Hess(r, c) = 0; Hess(c, r) = 0; }
    for (int r = 0; r < gf; r++) { Hess(r, r) = 1.0; JacT[r] = 0; }
    for (int k = 0; k < n; k++) D[k] = Hess(k, k);
    M = Hess;
    for (int k = 0; k < n; k++) { M(k, k) += u * D[k]; rhs[k] = -JacT[k]; }
    ldlt_solve(M, rhs, dxi);
    if (gravity) x_temp[0].g = x_temp[0].g + v3(dxi[n - 3], dxi[n - 2], dxi[n - 1]);  // voxel_map.hpp:813 (accumulates on x_temp, as written)
    for (int j = 0; j < W; j++) {
      const double* d = &dxi[DIMS * j];
      x_temp[j].R = x_stats[j].R * so3_exp(v3(d[0], d[1], d[2]));
      x_temp[j].p = x_stats[j].p + v3(d[3], d[4], d[5]);
      x_temp[j].v = x_stats[j].v + v3(d[6], d[7], d[8]);
      x_temp[j].bg = x_stats[j].bg + v3(d[9], d[10], d[11]);
      x_temp[j].ba = x_stats[j].ba + v3(d[12], d[13], d[14]);
      if (gravity) x_temp[j].g = x_temp[0].g;
    }
    imu.update(dxi.data());
    double q1 = 0;
    for (int k = 0; k < n; k++) q1 += dxi[k] * (u * D[k] * dxi[k] - JacT[k]);
    q1 *= 0.5;
    // only_residual  voxel_map.hpp:525-560 / 738-773
    double ri = imu.eval(x_temp, false, nullptr, nullptr) * (imu_coef * 0.5);
    int tn = int(voxhess.size()) < thd_num ? 1 : thd_num;
    residual2 = ri + lidar_residual_threads(x_temp, voxhess, tn);
    q = residual1 - residual2;
    int acc = q > 0;
    if (trace) trace->push_back(LmTrace{residual1, residual2, u, v, q1, acc});
    if (q > 0) {
      x_stats = x_temp;
      double one_three = 1.0 / 3;
      q = q / q1; v = 2; q = 1 - std::pow(2 * q - 1, 3);
      u *= (q < one_three ? one_three : q);
      is_calc_hess = true;
    } else { u = u * v; v = 2 * v; is_calc_hess = false; imu.rollback(); }
    if (std::fabs((residual1 - residual2) / residual1) < 1e-6) break;
  }
  if (gravity && resis) resis->push_back(residual2);
}

}  // namespace vxo
