// Per-voxel / per-entry math of the BA hot path, written for the GPU (register-resident fp64, no local arrays
// with dynamic indexing) but compilable as plain C++ so tests can exercise it on the CPU (tests/test_host_math.py).
//
// What it restates (reference = Voxel-SLAM/VoxelSLAM/src/):
//   tools.hpp:357-363        PointCluster::transform            -> cluster_transform_acc
//   voxel_map.hpp:264-273    cov + SelfAdjointEigenSolver        -> cov_from_sum, eig3_jacobi
//   voxel_map.hpp:163-234    acc_evaluate2 per observing frame   -> entry_jacobian  (rank-3 + block-diagonal form,
//                            SURVEY.md App. A.3:  H_voxel = sum_m alpha_m b^m b^m^T + blockdiag(D_i))
//   tools.hpp:51-66          Exp                                 -> so3_exp
#pragma once
#include <math.h>
#if defined(__CUDACC__)
#define VXS_HD __host__ __device__ __forceinline__
#else
#define VXS_HD inline
#endif

namespace vxs {

struct d3 { double x, y, z; };
VXS_HD d3 mk3(double x, double y, double z) { d3 r; r.x = x; r.y = y; r.z = z; return r; }
VXS_HD d3 operator+(d3 a, d3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
VXS_HD d3 operator-(d3 a, d3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
VXS_HD d3 operator*(double s, d3 a) { return mk3(s * a.x, s * a.y, s * a.z); }
VXS_HD double dot(d3 a, d3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
VXS_HD d3 cross(d3 a, d3 b) { return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

struct sym3 { double xx, xy, xz, yy, yz, zz; };
VXS_HD d3 mul(const sym3& P, d3 v) { return mk3(P.xx * v.x + P.xy * v.y + P.xz * v.z, P.xy * v.x + P.yy * v.y + P.yz * v.z, P.xz * v.x + P.yz * v.y + P.zz * v.z); }

struct rot3 { double r00, r01, r02, r10, r11, r12, r20, r21, r22; };  // row-major
VXS_HD d3 mul(const rot3& R, d3 v) { return mk3(R.r00 * v.x + R.r01 * v.y + R.r02 * v.z, R.r10 * v.x + R.r11 * v.y + R.r12 * v.z, R.r20 * v.x + R.r21 * v.y + R.r22 * v.z); }
VXS_HD d3 mulT(const rot3& R, d3 v) { return mk3(R.r00 * v.x + R.r10 * v.y + R.r20 * v.z, R.r01 * v.x + R.r11 * v.y + R.r21 * v.z, R.r02 * v.x + R.r12 * v.y + R.r22 * v.z); }

struct cluster { sym3 P; d3 v; double n; };  // n = point count (as double)

VXS_HD rot3 load_rot(const double* p) { rot3 R; R.r00 = p[0]; R.r01 = p[1]; R.r02 = p[2]; R.r10 = p[3]; R.r11 = p[4]; R.r12 = p[5]; R.r20 = p[6]; R.r21 = p[7]; R.r22 = p[8]; return R; }

// acc += transform(c; R, t)      tools.hpp:357-363:  v' = R v + N t ;  P' = R P R^T + (Rv) t^T + t (Rv)^T + N t t^T
VXS_HD void cluster_transform_acc(const cluster& c, const rot3& R, d3 t, cluster& acc) {
  d3 Rv = mul(R, c.v);
  // rows of R*P (P symmetric)
  d3 a0 = mul(c.P, mk3(R.r00, R.r01, R.r02));  // (R P) row 0 = (P R_row0^T)^T
  d3 a1 = mul(c.P, mk3(R.r10, R.r11, R.r12));
  d3 a2 = mul(c.P, mk3(R.r20, R.r21, R.r22));
  d3 r0 = mk3(R.r00, R.r01, R.r02), r1 = mk3(R.r10, R.r11, R.r12), r2 = mk3(R.r20, R.r21, R.r22);
  double n = c.n;
  acc.P.xx += dot(a0, r0) + 2.0 * Rv.x * t.x + n * t.x * t.x;
  acc.P.xy += dot(a0, r1) + (Rv.x * t.y + Rv.y * t.x) + n * t.x * t.y;
  acc.P.xz += dot(a0, r2) + (Rv.x * t.z + Rv.z * t.x) + n * t.x * t.z;
  acc.P.yy += dot(a1, r1) + 2.0 * Rv.y * t.y + n * t.y * t.y;
  acc.P.yz += dot(a1, r2) + (Rv.y * t.z + Rv.z * t.y) + n * t.y * t.z;
  acc.P.zz += dot(a2, r2) + 2.0 * Rv.z * t.z + n * t.z * t.z;
  acc.v.x += Rv.x + n * t.x; acc.v.y += Rv.y + n * t.y; acc.v.z += Rv.z + n * t.z;
  acc.n += n;
}

// tools.hpp:333-337  cov = P/N - c c^T  (c = v/N)
VXS_HD sym3 cov_from_sum(const cluster& s) {
  double N = s.n;
  d3 c = mk3(s.v.x / N, s.v.y / N, s.v.z / N);
  sym3 C;
  C.xx = s.P.xx / N - c.x * c.x; C.xy = s.P.xy / N - c.x * c.y; C.xz = s.P.xz / N - c.x * c.z;
  C.yy = s.P.yy / N - c.y * c.y; C.yz = s.P.yz / N - c.y * c.z; C.zz = s.P.zz / N - c.z * c.z;
  return C;
}

// One Jacobi rotation in the (p,q) plane of a symmetric 3x3 held in scalars.  app,aqq diagonal, apq the pivot,
// arp,arq the two remaining off-diagonals (r = third index).  vXp/vXq: columns p,q of the eigenvector matrix.
VXS_HD void jacobi_rot(double& app, double& aqq, double& apq, double& arp, double& arq, double& v0p, double& v0q, double& v1p, double& v1q,
                       double& v2p, double& v2q) {
  if (apq == 0.0) return;
  double theta = (aqq - app) / (2.0 * apq);
  double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
  double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c);
  double h = t * apq;
  app -= h; aqq += h; apq = 0.0;
  double g = arp, hh = arq;
  arp = g - s * (hh + g * tau); arq = hh + s * (g - hh * tau);
  g = v0p; hh = v0q; v0p = g - s * (hh + g * tau); v0q = hh + s * (g - hh * tau);
  g = v1p; hh = v1q; v1p = g - s * (hh + g * tau); v1q = hh + s * (g - hh * tau);
  g = v2p; hh = v2q; v2p = g - s * (hh + g * tau); v2q = hh + s * (g - hh * tau);
}

// Symmetric 3x3 eigen-decomposition, fp64 cyclic Jacobi, eigenvalues ascending, eigenvectors = columns (u0,u1,u2).
// Replaces Eigen::SelfAdjointEigenSolver<Matrix3d> (voxel_map.hpp:267,1161; loop_refine.hpp:363).  A closed-form
// (trigonometric) solve is NOT accurate enough here: cov is formed in world coordinates, lambda0/lambda2 ~ 1e-6 and
// lambda1 ~ lambda2 is the normal case, so the smallest eigenvalue needs the relative accuracy Jacobi gives.
VXS_HD void eig3_jacobi(const sym3& C, double w[3], d3& u0, d3& u1, d3& u2) {
  double a00 = C.xx, a11 = C.yy, a22 = C.zz, a01 = C.xy, a02 = C.xz, a12 = C.yz;
  double v00 = 1, v01 = 0, v02 = 0, v10 = 0, v11 = 1, v12 = 0, v20 = 0, v21 = 0, v22 = 1;
  for (int sweep = 0; sweep < 24; sweep++) {
    double dmax = fmax(fabs(a00), fmax(fabs(a11), fabs(a22)));
    double omax = fmax(fabs(a01), fmax(fabs(a02), fabs(a12)));
    if (omax == 0.0 || omax <= 1e-22 * dmax) break;
    jacobi_rot(a00, a11, a01, a02, a12, v00, v01, v10, v11, v20, v21);  // (0,1), r=2: a[2][0]=a02, a[2][1]=a12
    jacobi_rot(a00, a22, a02, a01, a12, v00, v02, v10, v12, v20, v22);  // (0,2), r=1: a[1][0]=a01, a[1][2]=a12
    jacobi_rot(a11, a22, a12, a01, a02, v01, v02, v11, v12, v21, v22);  // (1,2), r=0: a[0][1]=a01, a[0][2]=a02
  }
  // sort ascending (3-element network), carrying the columns
  d3 c0 = mk3(v00, v10, v20), c1 = mk3(v01, v11, v21), c2 = mk3(v02, v12, v22);
  double e0 = a00, e1 = a11, e2 = a22;
  if (e0 > e1) { double t = e0; e0 = e1; e1 = t; d3 tc = c0; c0 = c1; c1 = tc; }
  if (e1 > e2) { double t = e1; e1 = e2; e2 = t; d3 tc = c1; c1 = c2; c2 = tc; }
  if (e0 > e1) { double t = e0; e0 = e1; e1 = t; d3 tc = c0; c0 = c1; c1 = tc; }
  w[0] = e0; w[1] = e1; w[2] = e2; u0 = c0; u1 = c1; u2 = c2;
}

// tools.hpp:51-66
VXS_HD rot3 so3_exp(d3 w) {
  double n = sqrt(dot(w, w));
  rot3 R;
  if (n >= 1e-11) {
    d3 a = mk3(w.x / n, w.y / n, w.z / n);
    double s = sin(n), c = 1.0 - cos(n);
    // K = hat(a); K*K = a a^T - I (|a| = 1 up to rounding; expand exactly as K*K)
    double kk00 = -(a.z * a.z) - a.y * a.y, kk11 = -(a.z * a.z) - a.x * a.x, kk22 = -(a.y * a.y) - a.x * a.x;
    double kk01 = a.x * a.y, kk02 = a.x * a.z, kk12 = a.y * a.z;
    R.r00 = 1.0 + c * kk00; R.r01 = -s * a.z + c * kk01; R.r02 = s * a.y + c * kk02;
    R.r10 = s * a.z + c * kk01; R.r11 = 1.0 + c * kk11; R.r12 = -s * a.x + c * kk12;
    R.r20 = -s * a.y + c * kk02; R.r21 = s * a.x + c * kk12; R.r22 = 1.0 + c * kk22;
  } else {
    R.r00 = R.r11 = R.r22 = 1.0; R.r01 = R.r02 = R.r10 = R.r12 = R.r20 = R.r21 = 0.0;
  }
  return R;
}
VXS_HD rot3 rot_mul(const rot3& A, const rot3& B) {
  rot3 C;
  C.r00 = A.r00 * B.r00 + A.r01 * B.r10 + A.r02 * B.r20; C.r01 = A.r00 * B.r01 + A.r01 * B.r11 + A.r02 * B.r21; C.r02 = A.r00 * B.r02 + A.r01 * B.r12 + A.r02 * B.r22;
  C.r10 = A.r10 * B.r00 + A.r11 * B.r10 + A.r12 * B.r20; C.r11 = A.r10 * B.r01 + A.r11 * B.r11 + A.r12 * B.r21; C.r12 = A.r10 * B.r02 + A.r11 * B.r12 + A.r12 * B.r22;
  C.r20 = A.r20 * B.r00 + A.r21 * B.r10 + A.r22 * B.r20; C.r21 = A.r20 * B.r01 + A.r21 * B.r11 + A.r22 * B.r21; C.r22 = A.r20 * B.r02 + A.r21 * B.r12 + A.r22 * B.r22;
  return C;
}

// Per-voxel constants of acc_evaluate2 (voxel_map.hpp:163-174), from the cached eig / summed cluster.
struct voxel_consts {
  d3 u0, u1, u2;     // eigenvectors, u0 = plane normal (kk = 0)
  d3 vbar;           // pcr_add.v / NN
  double NN;         // pcr_add.N
  double invN;       // 1 / NN
  double s1, s2, s3; // sqrt(-coe*alpha_m): alpha1 = 2/(l0-l1), alpha2 = 2/(l0-l2), alpha3 = -2/NN^2  (all <= 0)
  double coe;
};
VXS_HD voxel_consts make_voxel_consts(const double lam[3], d3 u0, d3 u1, d3 u2, d3 sumv, double NN, double coe) {
  voxel_consts k;
  k.u0 = u0; k.u1 = u1; k.u2 = u2; k.NN = NN; k.invN = 1.0 / NN; k.coe = coe;
  k.vbar = mk3(sumv.x / NN, sumv.y / NN, sumv.z / NN);
  k.s1 = sqrt(coe * (2.0 / (lam[1] - lam[0])));
  k.s2 = sqrt(coe * (2.0 / (lam[2] - lam[0])));
  k.s3 = sqrt(coe * 2.0) / NN;
  return k;
}

// Output of one (voxel, frame) entry.
//   g[6]      : Auk^T u0                       (voxel_map.hpp:202)            -> JacT += coe*g
//   x[18]     : rows sqrt(-coe*alpha_m) * b^m, m=1..3, 6 each                  -> H -= sum_m x^m x^m^T over frame pairs
//   Drr[9],Drt[9],Dtt[6] : block-diagonal remainder D_i (row-major 3x3, 3x3, symmetric 3x3 packed xx xy xz yy yz zz),
//               already multiplied by coe.  H_ii += [[Drr, Drt],[Drt^T, Dtt]]
struct entry_out { double g[6]; double x[18]; double Drr[9]; double Drt[9]; double Dtt[6]; };

// b(y) = Auk^T y for an arbitrary direction y (no 3x6 matrix is formed):
//   top    = z x r + Pr x ry + s (v x ry),   ry = R^T y,  z = P ry + (tau.y) v
//   bottom = u (c2.y) + (c2.u) y
VXS_HD void auk_t_times(d3 y, const cluster& c, const rot3& R, d3 r, d3 Pr, d3 tau, double s, d3 c2, d3 u, double c2u, double invN, double out[6]) {
  d3 ry = mulT(R, y);
  d3 z = mul(c.P, ry) + dot(tau, y) * c.v;
  d3 top = cross(z, r) + cross(Pr, ry) + s * cross(c.v, ry);
  double c2y = dot(c2, y);
  out[0] = invN * top.x; out[1] = invN * top.y; out[2] = invN * top.z;
  out[3] = invN * (u.x * c2y + c2u * y.x); out[4] = invN * (u.y * c2y + c2u * y.y); out[5] = invN * (u.z * c2y + c2u * y.z);
}

VXS_HD void entry_jacobian(const voxel_consts& k, const cluster& c, const rot3& R, d3 t, entry_out& o) {
  const d3 u = k.u0;
  const double invN = k.invN, ni = c.n;
  d3 r = mulT(R, u);                 // RiTuk
  d3 w = cross(c.v, r);              // viRiTuk = hat(vi) * RiTuk
  d3 Pr = mul(c.P, r);               // PiRiTuk
  d3 tau = t - k.vbar;               // ti_v
  double s = dot(u, tau);            // ukTti_v
  d3 c2 = mul(R, c.v) + ni * tau;    // combo2
  double c2u = dot(c2, u);

  auk_t_times(u, c, R, r, Pr, tau, s, c2, u, c2u, invN, o.g);
  double b1[6], b2[6];
  auk_t_times(k.u1, c, R, r, Pr, tau, s, c2, u, c2u, invN, b1);
  auk_t_times(k.u2, c, R, r, Pr, tau, s, c2, u, c2u, invN, b2);
  for (int i = 0; i < 6; i++) { o.x[i] = k.s1 * b1[i]; o.x[6 + i] = k.s2 * b2[i]; }
  o.x[12] = k.s3 * w.x; o.x[13] = k.s3 * w.y; o.x[14] = k.s3 * w.z;
  o.x[15] = k.s3 * ni * u.x; o.x[16] = k.s3 * ni * u.y; o.x[17] = k.s3 * ni * u.z;

  // D_rr = (2/N) (C1 - hat(r) P) hat(r) - 1/2 hat(g_theta),  C1 = hat(Pr) + s hat(v)     (voxel_map.hpp:196,207)
  //   rows of Y = C1 - hat(r) P :  (hat(a))_row_i = e_i x a (as a row vector: e_i^T hat(a) = (a x e_i)^T ... ) — written out below.
  // hat(a) = [[0,-az,ay],[az,0,-ax],[-ay,ax,0]]
  d3 q = Pr + s * c.v;  // C1 = hat(q)
  // hat(r) P : row i = (hat(r) row i) * P
  d3 hr0 = mk3(0.0, -r.z, r.y), hr1 = mk3(r.z, 0.0, -r.x), hr2 = mk3(-r.y, r.x, 0.0);
  d3 hp0 = mul(c.P, hr0), hp1 = mul(c.P, hr1), hp2 = mul(c.P, hr2);  // P symmetric: (row * P)^T = P * row^T
  d3 y0 = mk3(0.0, -q.z, q.y) - hp0, y1 = mk3(q.z, 0.0, -q.x) - hp1, y2 = mk3(-q.y, q.x, 0.0) - hp2;
  // (Y hat(r)) row i = y_i x r   (m^T hat(r) = (m x r)^T)
  d3 z0 = cross(y0, r), z1 = cross(y1, r), z2 = cross(y2, r);
  const double f = 2.0 * invN * k.coe, hg = 0.5 * k.coe;
  o.Drr[0] = f * z0.x;               o.Drr[1] = f * z0.y + hg * o.g[2]; o.Drr[2] = f * z0.z - hg * o.g[1];
  o.Drr[3] = f * z1.x - hg * o.g[2]; o.Drr[4] = f * z1.y;               o.Drr[5] = f * z1.z + hg * o.g[0];
  o.Drr[6] = f * z2.x + hg * o.g[1]; o.Drr[7] = f * z2.y - hg * o.g[0]; o.Drr[8] = f * z2.z;
  // D_rt = (2/N) w u^T ; D_tt = (2 n_i / N) u u^T
  o.Drt[0] = f * w.x * u.x; o.Drt[1] = f * w.x * u.y; o.Drt[2] = f * w.x * u.z;
  o.Drt[3] = f * w.y * u.x; o.Drt[4] = f * w.y * u.y; o.Drt[5] = f * w.y * u.z;
  o.Drt[6] = f * w.z * u.x; o.Drt[7] = f * w.z * u.y; o.Drt[8] = f * w.z * u.z;
  const double ft = f * ni;
  o.Dtt[0] = ft * u.x * u.x; o.Dtt[1] = ft * u.x * u.y; o.Dtt[2] = ft * u.x * u.z; o.Dtt[3] = ft * u.y * u.y; o.Dtt[4] = ft * u.y * u.z; o.Dtt[5] = ft * u.z * u.z;
}

}  // namespace vxs
