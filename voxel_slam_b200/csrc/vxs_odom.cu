// Odometry association + EKF normal-equation accumulation on the device (SURVEY.md §8f rank 3):
//   match()            voxel_map.hpp:1674-1698  root-cell lookup
//   OctoTree::match()  voxel_map.hpp:1335-1392  descent to the leaf, 3-sigma gates, sigma_d
//   the per-point loop of the EKF update, voxelslam.cpp:876-918: HTH += R_inv jac jac^T, HTz -= R_inv jac resi, nnt += n n^T, match_num++
//
// The octree itself stays where the reference keeps it (host) until the stateful map moves to the device (§8f rank 1): after every
// marginalisation the caller exports the plane leaves once (vxs_odom_set_planes: cube centre + layer, plane centre / normal / 6x6
// covariance / radius — the fields plane_update writes, voxel_map.hpp:1118-1146) and every EKF iteration is then one kernel over the
// scan.  Leaves partition space, so "descend from the root" == "probe the sorted leaf table with the (root cell, layer, octant path)
// key of every layer"; the octant path follows the reference's comparisons and float quarter lengths exactly (same routine as the map
// build), so the point -> leaf assignment is bit-exact.
// What is bit-exact against the reference: var_init's points, the world points, their root cells and leaves, and the per-point match
// flags (the gate operands are rounded as the reference rounds them, see vxs_odom_math.cuh).  What is held to a tolerance: var_init's
// and pvec_update's variances, sigma_l, and the HTH / HTz / nnt sums (fp64 atomics in warp-tree order).
// The whole iterated update, lio_state_estimation (voxelslam.cpp:856-958), is here too: vxs_lio_run enqueues k_lio_init and 4 x (association
// pass, k_lio_step) for both association paths (vxs_odom_lio_update, vxs_map_lio_update); its passes sum in a fixed order, not through atomics.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include "vxs_internal.h"
#include "vxs_math.cuh"
#include "vxs_odom_math.cuh"

using namespace vxs;

namespace {

// ---- bit-exact cell arithmetic (same as vxs_voxelize.cu; kept local so that the validated map-build unit stays untouched)
__host__ __device__ inline long long od_quantise(double pw, double voxel_size) {
#ifdef __CUDA_ARCH__
  float loc = __double2float_rn(__ddiv_rn(pw, voxel_size));
  if (loc < 0.0f) loc = __fsub_rn(loc, 1.0f);
  return __float2ll_rz(loc);
#else
  float loc = float(pw / voxel_size);
  if (loc < 0) loc -= 1;
  return (long long)loc;
#endif
}
__device__ __forceinline__ double od_dot3(double a0, double a1, double a2, double x, double y, double z, double t) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, x), __dmul_rn(a1, y)), __dmul_rn(a2, z)), t);
}
// octants of the deeper layers, 3 bits per layer, layer 1 in the low bits (voxel_map.hpp:1029-1040)
__device__ __forceinline__ unsigned int od_octants(double wx, double wy, double wz, long long kx, long long ky, long long kz, double voxel_size, int max_layer) {
  double cx = __dmul_rn(__dadd_rn(0.5, (double)kx), voxel_size), cy = __dmul_rn(__dadd_rn(0.5, (double)ky), voxel_size), cz = __dmul_rn(__dadd_rn(0.5, (double)kz), voxel_size);
  float q = __double2float_rn(__ddiv_rn(voxel_size, 4.0));
  unsigned int bits = 0;
  for (int l = 0; l < max_layer; l++) {
    const int bx = wx > cx, by = wy > cy, bz = wz > cz;
    bits |= (unsigned int)(4 * bx + 2 * by + bz) << (3 * l);
    cx = __dadd_rn(cx, (double)__fmul_rn((float)(2 * bx - 1), q));
    cy = __dadd_rn(cy, (double)__fmul_rn((float)(2 * by - 1), q));
    cz = __dadd_rn(cz, (double)__fmul_rn((float)(2 * bz - 1), q));
    q = __fdiv_rn(q, 2.0f);
  }
  return bits;
}
// key of a node: linear root id | layer | path (path = octants most-significant first, as OctoTree numbers its children)
__host__ __device__ inline unsigned long long od_key(unsigned long long root_lin, int layer, unsigned int path) { return (root_lin << 12) | ((unsigned long long)layer << 9) | path; }
__device__ __forceinline__ unsigned int od_path_prefix(unsigned int bits, int depth) {
  unsigned int p = 0;
  for (int j = 0; j < depth; j++) p = p * 8 + ((bits >> (3 * j)) & 7u);
  return p;
}


struct OdomScratch {
  DevBuf<unsigned long long> keys;
  DevBuf<double> rows, pts, out, st;
  DevBuf<double> lio, parts;        // vxs_lio_run: the LioState block and the partial rows of the association passes
  DevBuf<int> flags;
  long long n_planes = 0, n_pts = 0;
  long long minx = 0, miny = 0, minz = 0, ex = 0, ey = 0, ez = 0;
  double voxel_size = 1.0;
  int max_layer = 0;
};

// kRows = false: the 34 sums go to `out` through fp64 atomics (vxs_odom_accumulate).  kRows = true (vxs_odom_lio_update): one partial row per
// block (od_flush_row), and the whole block returns at entry once the EKF step has set *stopped.
template <bool kRows>
__global__ void __launch_bounds__(OD_THREADS) k_odom_accumulate(const double* __restrict__ pv, long long n, const double* __restrict__ st /* R9 p3 rotvar9 tslvar9 */,
                                                                const unsigned long long* __restrict__ keys, const double* __restrict__ rows, long long n_planes, long long minx,
                                                                long long miny, long long minz, long long ex, long long ey, long long ez, double voxel_size, int max_layer,
                                                                double* __restrict__ out /* HTH 36 | HTz 6 | nnt 9 | count */, int* __restrict__ flags, const int* __restrict__ stopped) {
  if (kRows && *stopped) return;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double acc[34];
#pragma unroll
  for (int k = 0; k < 34; k++) acc[k] = 0.0;
  int hit = 0;
  if (i < n) {
    const double* p = pv + 12 * i;
    const double x = p[0], y = p[1], z = p[2];
    const double R[9] = {st[0], st[1], st[2], st[3], st[4], st[5], st[6], st[7], st[8]};
    const double wx = od_dot3(R[0], R[1], R[2], x, y, z, st[9]), wy = od_dot3(R[3], R[4], R[5], x, y, z, st[10]), wz = od_dot3(R[6], R[7], R[8], x, y, z, st[11]);
    const long long kx = od_quantise(wx, voxel_size), ky = od_quantise(wy, voxel_size), kz = od_quantise(wz, voxel_size);
    const long long rx = kx - minx, ry = ky - miny, rz = kz - minz;
    if (rx >= 0 && ry >= 0 && rz >= 0 && rx < ex && ry < ey && rz < ez) {
      const unsigned long long root_lin = ((unsigned long long)rx * (unsigned long long)ey + (unsigned long long)ry) * (unsigned long long)ez + (unsigned long long)rz;
      const unsigned int bits = od_octants(wx, wy, wz, kx, ky, kz, voxel_size, max_layer);
      long long found = -1;
      for (int l = 0; l <= max_layer && found < 0; l++) {
        const unsigned long long key = od_key(root_lin, l, od_path_prefix(bits, l));
        long long lo = 0, hi = n_planes;                       // first key >= wanted
        while (lo < hi) { const long long mid = (lo + hi) >> 1; if (keys[mid] < key) lo = mid + 1; else hi = mid; }
        if (lo < n_planes && keys[lo] == key) found = lo;
      }
      if (found >= 0) hit = od_contribution(rows + OD_ROW * found, x, y, z, wx, wy, wz, p, st, acc);
    }
    if (flags) flags[i] = hit;
  }
  if (kRows) od_flush_row(acc, out);
  else od_flush(acc, out);
}

// calcBodyVar + var_init (voxelslam.hpp:163-203): per point the range / bearing noise model in the sensor frame, then the extrinsic.
// The float intermediates of the reference are kept: `float range`, `float range_var = range_inc * range_inc` (:167-168); dir_var =
// pow(sin(DEG2RAD(degree_inc)), 2) is the same for every point and is computed on the host with the same libm calls.
__global__ void __launch_bounds__(256) k_var_init(const float* __restrict__ pts, int stride, long long n, const double* __restrict__ ext /* R9 p3 */, float range_inc, double dir_var,
                                                  double* __restrict__ pv) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* ap = pts + size_t(i) * stride;
  double pb[3] = {(double)ap[0], (double)ap[1], (double)ap[2]};
  if (pb[2] == 0) pb[2] = 0.0001;                                              // :165-166 (modifies pv.pnt itself)
  const double nn = (pb[0] * pb[0] + pb[1] * pb[1]) + pb[2] * pb[2];
  const float range = __double2float_rn(sqrt(nn));
  const float range_var = __fmul_rn(range_inc, range_inc);
  const double inv = sqrt(nn);
  const double d[3] = {pb[0] / inv, pb[1] / inv, pb[2] / inv};                 // direction.normalize()
  double b1[3] = {1.0, 1.0, -(d[0] + d[1]) / d[2]};
  { const double l = sqrt((b1[0] * b1[0] + b1[1] * b1[1]) + b1[2] * b1[2]); b1[0] /= l; b1[1] /= l; b1[2] /= l; }
  double b2[3] = {b1[1] * d[2] - b1[2] * d[1], b1[2] * d[0] - b1[0] * d[2], b1[0] * d[1] - b1[1] * d[0]};    // base_vector1.cross(direction)
  { const double l = sqrt((b2[0] * b2[0] + b2[1] * b2[1]) + b2[2] * b2[2]); b2[0] /= l; b2[1] /= l; b2[2] /= l; }
  // A = range * hat(direction) * [b1 b2]:  hat(d) v = d x v
  const double r = (double)range;
  const double A1[3] = {r * (d[1] * b1[2] - d[2] * b1[1]), r * (d[2] * b1[0] - d[0] * b1[2]), r * (d[0] * b1[1] - d[1] * b1[0])};
  const double A2[3] = {r * (d[1] * b2[2] - d[2] * b2[1]), r * (d[2] * b2[0] - d[0] * b2[2]), r * (d[0] * b2[1] - d[1] * b2[0])};
  double var[9];
  const double rv = (double)range_var;
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) var[3 * a + b] = d[a] * rv * d[b] + (A1[a] * dir_var * A1[b] + A2[a] * dir_var * A2[b]);
  // pv.pnt = ext.R * pv.pnt + ext.p;  pv.var = ext.R * pv.var * ext.R^T     (:199-200).  The point without FMA contraction: the map assigns
  // it to cells and leaves, so it must round as the reference's does; the variance only feeds sigma and is held to a tolerance.
  double* o = pv + 12 * i;
#pragma unroll
  for (int a = 0; a < 3; a++) o[a] = od_dot3(ext[3 * a], ext[3 * a + 1], ext[3 * a + 2], pb[0], pb[1], pb[2], ext[9 + a]);
  double t[9];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) t[3 * a + b] = (ext[3 * a] * var[b] + ext[3 * a + 1] * var[3 + b]) + ext[3 * a + 2] * var[6 + b];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) o[3 + 3 * a + b] = (t[3 * a] * ext[3 * b] + t[3 * a + 1] * ext[3 * b + 1]) + t[3 * a + 2] * ext[3 * b + 2];
}
// pvec_update (voxelslam.hpp:205-214): pv.var = R var R^T + phat rot_var phat^T + tsl_var (in place, pv.pnt stays in the body frame), pwld = R pnt + p
__global__ void __launch_bounds__(256) k_pvec_update(double* __restrict__ pv, long long n, const double* __restrict__ st /* R9 p3 rotvar9 tslvar9 */, double* __restrict__ pwld) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double* p = pv + 12 * i;
  const double x = p[0], y = p[1], z = p[2];
  const double ph[9] = {0.0, -z, y, z, 0.0, -x, -y, x, 0.0};
  double t[9], u[9];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) {
      t[3 * a + b] = (st[3 * a] * p[3 + b] + st[3 * a + 1] * p[6 + b]) + st[3 * a + 2] * p[9 + b];                       // R var
      u[3 * a + b] = (ph[3 * a] * st[12 + b] + ph[3 * a + 1] * st[15 + b]) + ph[3 * a + 2] * st[18 + b];                 // phat rot_var
    }
  double o[9];
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++)
      o[3 * a + b] = (((t[3 * a] * st[3 * b] + t[3 * a + 1] * st[3 * b + 1]) + t[3 * a + 2] * st[3 * b + 2]) + ((u[3 * a] * ph[3 * b] + u[3 * a + 1] * ph[3 * b + 1]) + u[3 * a + 2] * ph[3 * b + 2])) +
                     st[21 + 3 * a + b];
#pragma unroll
  for (int k = 0; k < 9; k++) p[3 + k] = o[k];
  if (pwld) {
    pwld[3 * i] = od_dot3(st[0], st[1], st[2], x, y, z, st[9]); pwld[3 * i + 1] = od_dot3(st[3], st[4], st[5], x, y, z, st[10]); pwld[3 * i + 2] = od_dot3(st[6], st[7], st[8], x, y, z, st[11]);
  }
}

// ---------------------------------------------------------------- the iterated EKF update, lio_state_estimation (voxelslam.cpp:856-958)
// The state of one vxs_*_lio_update call on the device: copied in once and read back once.  The association passes read st and stopped;
// the step kernel owns the rest.
struct LioState {
  double st[30];                 // R9 p3 of x_curr | rot_var9 tsl_var9 = x_curr.cov blocks (0,0), (3,3) (:874-875; fixed until the stop)
  double x[24], xp[24];          // x_curr, x_prop (state24 layout)
  double cov[225], cov_inv[225];   // row-major
  double trace[12];              // per iteration: match_num, |rot_add|, |tra_add|
  double match_num;              // of the last pass
  int stopped, iters, rematch, ok, err, pad;
};
#define LIO_THREADS 1024
#define LIO_GROUPS (LIO_THREADS / 34)

// The 15x15 algebra rounds as the reference's scalar code does: products and sums left to right, no FMA contraction.
__device__ __forceinline__ double lmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ladd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double lsub(double a, double b) { return __dsub_rn(a, b); }

// inv = a^-1 for the row-major 15x15 a (overwritten by its LU factors) as the reference's Matrix<double, 15, 15>::inverse() forms it
// (PartialPivLU): unblocked right-looking LU, the row pivot the first entry of largest magnitude in the column, the column divided by the
// pivot, the rank-1 update; then P I solved with the unit-lower and the upper factor, one column per thread.  Returns false to every thread
// when a pivot is exactly zero (the reference would go on with infinities).
__device__ bool lio_inverse15(double (*a)[15], double (*inv)[15], int* piv) {
  const int t = threadIdx.x;
  for (int k = 0; k < 15; k++) {
    if (t == 0) {
      int p = k; double big = fabs(a[k][k]);
      for (int i = k + 1; i < 15; i++) if (fabs(a[i][k]) > big) { big = fabs(a[i][k]); p = i; }
      piv[k] = big == 0.0 ? -1 : p;
    }
    __syncthreads();
    const int p = piv[k];
    if (p < 0) return false;
    if (p != k && t < 15) { const double v = a[k][t]; a[k][t] = a[p][t]; a[p][t] = v; }
    __syncthreads();
    if (t > k && t < 15) a[t][k] = a[t][k] / a[k][k];
    __syncthreads();
    const int r = 14 - k;
    if (t < r * r) { const int i = k + 1 + t / r, j = k + 1 + t % r; a[i][j] = lsub(a[i][j], lmul(a[i][k], a[k][j])); }
    __syncthreads();
  }
  if (t < 15) {
    for (int i = 0; i < 15; i++) inv[i][t] = i == t ? 1.0 : 0.0;
    for (int k = 0; k < 15; k++) if (piv[k] != k) { const double v = inv[k][t]; inv[k][t] = inv[piv[k]][t]; inv[piv[k]][t] = v; }
    for (int j = 0; j < 15; j++) { const double xj = inv[j][t]; for (int i = j + 1; i < 15; i++) inv[i][t] = lsub(inv[i][t], lmul(a[i][j], xj)); }
    for (int j = 14; j >= 0; j--) { inv[j][t] = inv[j][t] / a[j][j]; const double xj = inv[j][t]; for (int i = 0; i < j; i++) inv[i][t] = lsub(inv[i][t], lmul(a[i][j], xj)); }
  }
  __syncthreads();
  return true;
}

// cov_inv = x_curr.cov.inverse() (:872), once before the first pass.  A zero pivot stops the update before it starts (err).
__global__ void __launch_bounds__(LIO_THREADS) k_lio_init(LioState* __restrict__ s) {
  __shared__ double a[15][15], inv[15][15];
  __shared__ int piv[15];
  const int t = threadIdx.x;
  if (t < 225) a[t / 15][t % 15] = s->cov[t];
  __syncthreads();
  if (!lio_inverse15(a, inv, piv)) { if (t == 0) { s->err = 1; s->stopped = 1; } return; }
  if (t < 225) s->cov_inv[t] = inv[t / 15][t % 15];
}

// tools.hpp:86-91 Log and 51-66 Exp, in the reference's operation order
__device__ __forceinline__ void lio_log(const double* R, double* o) {
  const double tr = ladd(ladd(R[0], R[4]), R[8]);
  const double th = tr > 3.0 - 1e-6 ? 0.0 : acos(lmul(0.5, lsub(tr, 1.0)));
  const double K[3] = {lsub(R[7], R[5]), lsub(R[2], R[6]), lsub(R[3], R[1])};
  const double f = fabs(th) < 0.001 ? 0.5 : lmul(0.5, th) / sin(th);
  for (int k = 0; k < 3; k++) o[k] = lmul(f, K[k]);
}
__device__ __forceinline__ void lio_exp(const double* w, double* E) {
  const double nn = sqrt(ladd(ladd(lmul(w[0], w[0]), lmul(w[1], w[1])), lmul(w[2], w[2])));
  for (int k = 0; k < 9; k++) E[k] = (k % 4 == 0) ? 1.0 : 0.0;
  if (!(nn >= 1e-11)) return;
  const double r[3] = {w[0] / nn, w[1] / nn, w[2] / nn};
  const double K[9] = {0.0, -r[2], r[1], r[2], 0.0, -r[0], -r[1], r[0], 0.0};
  const double s = sin(nn), c = lsub(1.0, cos(nn));
  double cK[9];
  for (int k = 0; k < 9; k++) cK[k] = lmul(c, K[k]);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      double kk = lmul(cK[3 * i], K[j]);
      for (int q = 1; q < 3; q++) kk = ladd(kk, lmul(cK[3 * i + q], K[3 * q + j]));
      E[3 * i + j] = ladd(ladd(E[3 * i + j], lmul(s, K[3 * i + j])), kk);
    }
}

// One iteration of the EKF loop (voxelslam.cpp:873-948) against the partial rows of the pass before it; one CTA.  Returns at entry once
// the update has stopped.  The partial rows are summed in a fixed order, so the iteration is bit-reproducible.
__global__ void __launch_bounds__(LIO_THREADS) k_lio_step(LioState* __restrict__ s, const double* __restrict__ rows, int nrows) {
  if (s->stopped) return;
  __shared__ double red[LIO_GROUPS][34];
  __shared__ double sum[34], HTH[6][6], a[15][15], K1[15][15], G[15][6], vec[15], sol[15], ncov[225];
  __shared__ int piv[15], stop;
  const int t = threadIdx.x;
  // ---- the 34 sums: thread (group g, column k) adds rows g, g + G, ... with eight interleaved partial sums, then the groups in order
  if (t < 34 * LIO_GROUPS) {
    const int k = t % 34, g = t / 34;
    double p0 = 0, p1 = 0, p2 = 0, p3 = 0, p4 = 0, p5 = 0, p6 = 0, p7 = 0;
    int r = g;
    for (; r + 7 * LIO_GROUPS < nrows; r += 8 * LIO_GROUPS) {
      const double* q = rows + 34 * size_t(r) + k;
      p0 += q[0]; p1 += q[34 * LIO_GROUPS]; p2 += q[68 * LIO_GROUPS]; p3 += q[102 * LIO_GROUPS];
      p4 += q[136 * LIO_GROUPS]; p5 += q[170 * LIO_GROUPS]; p6 += q[204 * LIO_GROUPS]; p7 += q[238 * LIO_GROUPS];
    }
    for (; r < nrows; r += LIO_GROUPS) p0 += rows[34 * size_t(r) + k];
    red[g][k] = ((p0 + p1) + (p2 + p3)) + ((p4 + p5) + (p6 + p7));
  }
  __syncthreads();
  if (t < 34) {
    double v = red[0][t];
    for (int g = 1; g < LIO_GROUPS; g++) v += red[g][t];
    sum[t] = v;
  }
  __syncthreads();
  if (t < 36) {   // HTH from its upper triangle (row-major 21)
    const int i = t / 6, j = t % 6, lo = i < j ? i : j, hi = i < j ? j : i;
    HTH[i][j] = sum[lo * 6 - lo * (lo - 1) / 2 + (hi - lo)];
  }
  __syncthreads();
  // ---- K_1 = (H_T_H + cov_inv)^-1,  H_T_H.block<6,6>(0,0) = HTH  (:920-921)
  if (t < 225) { const int i = t / 15, j = t % 15; a[i][j] = (i < 6 && j < 6) ? ladd(HTH[i][j], s->cov_inv[t]) : s->cov_inv[t]; }
  __syncthreads();
  if (!lio_inverse15(a, K1, piv)) { if (t == 0) { s->err = 1; s->stopped = 1; } return; }
  // ---- G.block<15,6> = K_1.block<15,6> HTH;  vec = x_prop - x_curr (IMUST::operator-, tools.hpp:164-173)
  if (t < 90) {
    const int i = t / 6, c = t % 6;
    double v = lmul(K1[i][0], HTH[0][c]);
    for (int k = 1; k < 6; k++) v = ladd(v, lmul(K1[i][k], HTH[k][c]));
    G[i][c] = v;
  } else if (t == 96) {
    const double* R = s->x; const double* Rp = s->xp;
    double D[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) { double v = lmul(R[i], Rp[j]); for (int k = 1; k < 3; k++) v = ladd(v, lmul(R[3 * k + i], Rp[3 * k + j])); D[3 * i + j] = v; }   // x.R^T xp.R
    lio_log(D, vec);
    for (int k = 3; k < 15; k++) vec[k] = lsub(s->xp[6 + k], s->x[6 + k]);
  }
  __syncthreads();
  // ---- solution = K_1.block<15,6> HTz + vec - G.block<15,6> vec.head(6)  (:923)
  if (t < 15) {
    double u = lmul(K1[t][0], sum[21]), w = lmul(G[t][0], vec[0]);
    for (int k = 1; k < 6; k++) { u = ladd(u, lmul(K1[t][k], sum[21 + k])); w = ladd(w, lmul(G[t][k], vec[k])); }
    sol[t] = lsub(ladd(u, vec[t]), w);
  }
  __syncthreads();
  // ---- x_curr += solution (IMUST::operator+=, tools.hpp:154-162), the convergence test, rematch_num and the stop rule (:925-946)
  if (t == 0) {
    double E[9], R[9];
    lio_exp(sol, E);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) { double v = lmul(s->x[3 * i], E[j]); for (int k = 1; k < 3; k++) v = ladd(v, lmul(s->x[3 * i + k], E[3 * k + j])); R[3 * i + j] = v; }
    for (int k = 0; k < 9; k++) s->x[k] = R[k];
    for (int k = 3; k < 15; k++) s->x[6 + k] = ladd(s->x[6 + k], sol[k]);
    const double rn = sqrt(ladd(ladd(lmul(sol[0], sol[0]), lmul(sol[1], sol[1])), lmul(sol[2], sol[2])));
    const double tn = sqrt(ladd(ladd(lmul(sol[3], sol[3]), lmul(sol[4], sol[4])), lmul(sol[5], sol[5])));
    const int it = s->iters;
    const bool converged = lmul(rn, 57.3) < 0.01 && lmul(tn, 100.0) < 0.015;
    if (converged || (s->rematch == 0 && it == 4 - 2)) s->rematch++;
    stop = s->rematch >= 2 || it == 4 - 1;
    s->trace[3 * it] = sum[33]; s->trace[3 * it + 1] = rn; s->trace[3 * it + 2] = tn;
    s->match_num = sum[33];
    s->iters = it + 1;
    for (int k = 0; k < 12; k++) s->st[k] = s->x[k];       // R, p for the next pass; rot_var / tsl_var stay
  }
  __syncthreads();
  if (!stop) return;
  // ---- the stop: x_curr.cov = (I - G) x_curr.cov (:944), then the smallest eigenvalue of this iteration's nnt (:950-956)
  if (t < 225) {
    const int i = t / 15, j = t % 15;
    double v = 0.0;
    for (int k = 0; k < 15; k++) {
      const double m = k < 6 ? lsub(i == k ? 1.0 : 0.0, G[i][k]) : (i == k ? 1.0 : 0.0);   // (I - G)(i, k); G is zero beyond column 5
      v = k ? ladd(v, lmul(m, s->cov[15 * k + j])) : lmul(m, s->cov[j]);
    }
    ncov[t] = v;
  }
  __syncthreads();
  if (t < 225) s->cov[t] = ncov[t];
  if (t == 0) {
    sym3 C; C.xx = sum[27]; C.xy = sum[28]; C.xz = sum[29]; C.yy = sum[30]; C.yz = sum[31]; C.zz = sum[32];
    double w[3]; d3 u0, u1, u2;
    eig3_jacobi(C, w, u0, u1, u2);
    s->ok = !(w[0] < 14);
    s->stopped = 1;
  }
}

OdomScratch* odom_scratch(vxs_ctx* c) { if (!c->odom_scratch) c->odom_scratch = new OdomScratch(); return static_cast<OdomScratch*>(c->odom_scratch); }

}  // namespace

void vxs_odom_release(vxs_ctx* c) {
  if (!c->odom_scratch) return;
  OdomScratch* s = static_cast<OdomScratch*>(c->odom_scratch);
  s->keys.release(); s->rows.release(); s->pts.release(); s->out.release(); s->st.release(); s->flags.release(); s->lio.release(); s->parts.release();
  delete s;
  c->odom_scratch = nullptr;
}

extern "C" int vxs_odom_set_planes(vxs_ctx* ctx, const vxs_map_params* mp, int64_t n, const double* voxel_center, const int32_t* layer, const double* center, const double* normal,
                                   const double* plane_var36, const float* radius) {
  if (!ctx || !mp || n < 0 || (n > 0 && (!voxel_center || !layer || !center || !normal || !plane_var36 || !radius))) return VXS_ERR_ARG;
  if (mp->max_layer < 0 || mp->max_layer > 3 || !(mp->voxel_size > 0)) return vxs_fail(ctx, VXS_ERR_ARG, "max_layer must be 0..3 and voxel_size > 0");
  cudaSetDevice(ctx->device);
  OdomScratch* s = odom_scratch(ctx);
  s->n_planes = 0; s->voxel_size = mp->voxel_size; s->max_layer = mp->max_layer;
  if (n == 0) return VXS_OK;
  const double vs = mp->voxel_size;
  std::vector<long long> root(size_t(n) * 3);
  std::vector<unsigned int> path(n);
  long long mn[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, mx[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
  for (int64_t i = 0; i < n; i++) {
    if (layer[i] < 0 || layer[i] > mp->max_layer) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_odom_set_planes: layer outside 0..max_layer");
    const double* vc = voxel_center + 3 * i;
    long long k[3];
    for (int a = 0; a < 3; a++) { k[a] = od_quantise(vc[a], vs); root[3 * size_t(i) + a] = k[a]; mn[a] = std::min(mn[a], k[a]); mx[a] = std::max(mx[a], k[a]); }
    // replay the descent from the root cell to this cube (voxel_map.hpp:1029-1040): the cube centre picks its own octants
    double c[3] = {(0.5 + double(k[0])) * vs, (0.5 + double(k[1])) * vs, (0.5 + double(k[2])) * vs};
    float q = float(vs / 4.0);
    unsigned int pth = 0;
    for (int l = 0; l < layer[i]; l++) {
      int b[3];
      for (int a = 0; a < 3; a++) { b[a] = vc[a] > c[a]; c[a] = c[a] + double(float(2 * b[a] - 1) * q); }
      pth = pth * 8 + unsigned(4 * b[0] + 2 * b[1] + b[2]);
      q = q / 2.0f;
    }
    path[i] = pth;
  }
  const long double ex = (long double)mx[0] - mn[0] + 1, ey = (long double)mx[1] - mn[1] + 1, ez = (long double)mx[2] - mn[2] + 1;
  if (ex * ey * ez >= (long double)(1ull << 50)) return vxs_fail(ctx, VXS_ERR_RANGE, "plane table spans more than 2^50 root cells");
  s->minx = mn[0]; s->miny = mn[1]; s->minz = mn[2]; s->ex = (long long)ex; s->ey = (long long)ey; s->ez = (long long)ez;
  std::vector<unsigned long long> key(n);
  std::vector<int64_t> order(n);
  for (int64_t i = 0; i < n; i++) {
    const unsigned long long lin = ((unsigned long long)(root[3 * size_t(i)] - mn[0]) * (unsigned long long)s->ey + (unsigned long long)(root[3 * size_t(i) + 1] - mn[1])) * (unsigned long long)s->ez +
                                   (unsigned long long)(root[3 * size_t(i) + 2] - mn[2]);
    key[i] = od_key(lin, layer[i], path[i]);
    order[i] = i;
  }
  std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return key[a] < key[b]; });
  std::vector<unsigned long long> skey(n);
  std::vector<double> rows(size_t(n) * OD_ROW);
  for (int64_t t = 0; t < n; t++) {
    const int64_t i = order[t];
    skey[t] = key[i];
    if (t > 0 && skey[t] == skey[t - 1]) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_odom_set_planes: two planes in the same cube");
    double* r = rows.data() + size_t(t) * OD_ROW;
    for (int a = 0; a < 3; a++) { r[a] = center[3 * i + a]; r[3 + a] = normal[3 * i + a]; }
    int u = 6;
    for (int a = 0; a < 6; a++) for (int b = a; b < 6; b++) r[u++] = plane_var36[36 * i + 6 * a + b];
    r[27] = double(radius[i]);
  }
  VXS_CUDA(ctx, s->keys.reserve(size_t(n)));
  VXS_CUDA(ctx, s->rows.reserve(size_t(n) * OD_ROW));
  VXS_CUDA(ctx, cudaMemcpyAsync(s->keys.p, skey.data(), size_t(n) * 8, cudaMemcpyHostToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaMemcpyAsync(s->rows.p, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  s->n_planes = n;
  return VXS_OK;
}

extern "C" int vxs_odom_accumulate(vxs_ctx* ctx, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, double* HTH36, double* HTz6,
                                   double* nnt9, int64_t* match_num, int32_t* flags) {
  if (!ctx || n < 0 || !pose12 || !rot_var9 || !tsl_var9 || !HTH36 || !HTz6 || !nnt9 || !match_num) return VXS_ERR_ARG;
  cudaSetDevice(ctx->device);
  OdomScratch* s = odom_scratch(ctx);
  if (pv12) {   // NULL re-uses the scan of the previous call (the EKF loop re-associates the same scan up to four times)
    VXS_CUDA(ctx, s->pts.reserve(size_t(std::max<int64_t>(n, 1)) * 12));
    if (n) VXS_CUDA(ctx, cudaMemcpyAsync(s->pts.p, pv12, size_t(n) * 96, cudaMemcpyHostToDevice, ctx->stream));
    s->n_pts = n;
  } else if (n != s->n_pts) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_odom_accumulate: no resident scan of this size");
  double st[30];
  for (int k = 0; k < 12; k++) st[k] = pose12[k];
  for (int k = 0; k < 9; k++) { st[12 + k] = rot_var9[k]; st[21 + k] = tsl_var9[k]; }
  VXS_CUDA(ctx, s->st.reserve(30)); VXS_CUDA(ctx, s->out.reserve(34));
  VXS_CUDA(ctx, cudaMemcpyAsync(s->st.p, st, sizeof st, cudaMemcpyHostToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaMemsetAsync(s->out.p, 0, 34 * 8, ctx->stream));
  int* dflags = nullptr;
  if (flags) { VXS_CUDA(ctx, s->flags.reserve(size_t(std::max<int64_t>(n, 1)))); dflags = s->flags.p; }
  if (n > 0 && s->n_planes > 0)
    VXS_LAUNCH(ctx, "k_odom_accumulate", k_odom_accumulate<false>, unsigned((n + 255) / 256), 256, 0, s->pts.p, (long long)n, s->st.p, s->keys.p, s->rows.p, s->n_planes, s->minx, s->miny,
               s->minz, s->ex, s->ey, s->ez, s->voxel_size, s->max_layer, s->out.p, dflags, nullptr);
  else if (flags && n > 0) VXS_CUDA(ctx, cudaMemsetAsync(dflags, 0, size_t(n) * 4, ctx->stream));
  double out[34];
  VXS_CUDA(ctx, cudaMemcpyAsync(out, s->out.p, sizeof out, cudaMemcpyDeviceToHost, ctx->stream));
  if (flags && n > 0) VXS_CUDA(ctx, cudaMemcpyAsync(flags, dflags, size_t(n) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int u = 0;
  for (int a = 0; a < 6; a++) for (int b = a; b < 6; b++) { HTH36[6 * a + b] = out[u]; HTH36[6 * b + a] = out[u]; u++; }
  for (int a = 0; a < 6; a++) HTz6[a] = out[21 + a];
  const int sy[9] = {27, 28, 29, 28, 30, 31, 29, 31, 32};
  for (int k = 0; k < 9; k++) nnt9[k] = out[sy[k]];
  *match_num = int64_t(out[33] + 0.5);
  return VXS_OK;
}

// ---------------------------------------------------------------- the ctx's resident scan (shared with vxs_map.cu)
int vxs_odom_resident_scan(vxs_ctx* ctx, double** pv12_dev, long long* n) {
  OdomScratch* s = odom_scratch(ctx);
  *pv12_dev = s->pts.p; *n = s->n_pts;
  return VXS_OK;
}
int vxs_odom_set_resident_scan(vxs_ctx* ctx, const double* pv12_host, long long n) {
  OdomScratch* s = odom_scratch(ctx);
  VXS_CUDA(ctx, s->pts.reserve(size_t(std::max<long long>(n, 1)) * 12));
  if (n) VXS_CUDA(ctx, cudaMemcpyAsync(s->pts.p, pv12_host, size_t(n) * 96, cudaMemcpyHostToDevice, ctx->stream));
  s->n_pts = n;
  return VXS_OK;
}

extern "C" int vxs_var_init(vxs_ctx* ctx, const float* pts, int stride_floats, int64_t n, const double* ext_R9, const double* ext_p3, double dept_err, double beam_err, double* pv12_out) {
  if (!ctx || n < 0 || (n > 0 && !pts) || stride_floats < 3 || !ext_R9 || !ext_p3) return VXS_ERR_ARG;
  cudaSetDevice(ctx->device);
  OdomScratch* s = odom_scratch(ctx);
  VXS_CUDA(ctx, s->pts.reserve(size_t(std::max<int64_t>(n, 1)) * 12));
  VXS_CUDA(ctx, s->st.reserve(30));
  s->n_pts = n;
  if (n == 0) return VXS_OK;
  VXS_CUDA(ctx, ctx->stage.reserve((size_t(n) * stride_floats + 1) / 2 + 1));
  float* raw = reinterpret_cast<float*>(ctx->stage.p);
  VXS_CUDA(ctx, cudaMemcpyAsync(raw, pts, size_t(n) * stride_floats * 4, cudaMemcpyHostToDevice, ctx->stream));
  double ext[12];
  for (int k = 0; k < 9; k++) ext[k] = ext_R9[k];
  for (int k = 0; k < 3; k++) ext[9 + k] = ext_p3[k];
  VXS_CUDA(ctx, cudaMemcpyAsync(s->st.p, ext, sizeof ext, cudaMemcpyHostToDevice, ctx->stream));
  // calcBodyVar takes `const float range_inc, const float degree_inc` (:163): the doubles narrow at the call; DEG2RAD(x) = ((x)*0.017453293) (pcl_macros.h)
  const float range_inc = float(dept_err), degree_inc = float(beam_err);
  const double dir_var = std::pow(std::sin(double(degree_inc) * 0.017453293), 2);
  VXS_LAUNCH(ctx, "k_var_init", k_var_init, unsigned((n + 255) / 256), 256, 0, raw, stride_floats, (long long)n, s->st.p, range_inc, dir_var, s->pts.p);
  if (pv12_out) VXS_CUDA(ctx, cudaMemcpyAsync(pv12_out, s->pts.p, size_t(n) * 96, cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return VXS_OK;
}

extern "C" int vxs_pvec_update(vxs_ctx* ctx, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, double* pv12_out, double* pwld_out) {
  if (!ctx || n < 0 || !pose12 || !rot_var9 || !tsl_var9) return VXS_ERR_ARG;
  cudaSetDevice(ctx->device);
  OdomScratch* s = odom_scratch(ctx);
  if (pv12) { int rc = vxs_odom_set_resident_scan(ctx, pv12, n); if (rc) return rc; }
  else if (n != s->n_pts) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_pvec_update: no resident scan of this size");
  if (n == 0) return VXS_OK;
  double st[30];
  for (int k = 0; k < 12; k++) st[k] = pose12[k];
  for (int k = 0; k < 9; k++) { st[12 + k] = rot_var9[k]; st[21 + k] = tsl_var9[k]; }
  VXS_CUDA(ctx, s->st.reserve(30));
  VXS_CUDA(ctx, cudaMemcpyAsync(s->st.p, st, sizeof st, cudaMemcpyHostToDevice, ctx->stream));
  double* pw = nullptr;
  if (pwld_out) { VXS_CUDA(ctx, ctx->stage.reserve(size_t(n) * 3)); pw = ctx->stage.p; }
  VXS_LAUNCH(ctx, "k_pvec_update", k_pvec_update, unsigned((n + 255) / 256), 256, 0, s->pts.p, (long long)n, s->st.p, pw);
  if (pv12_out) VXS_CUDA(ctx, cudaMemcpyAsync(pv12_out, s->pts.p, size_t(n) * 96, cudaMemcpyDeviceToHost, ctx->stream));
  if (pwld_out) VXS_CUDA(ctx, cudaMemcpyAsync(pwld_out, pw, size_t(n) * 24, cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return VXS_OK;
}

// ---------------------------------------------------------------- lio_state_estimation on the device (voxelslam.cpp:856-958)
// Enqueued without a host round trip: cov_inv, then 4 x (association pass, step) unconditionally; the step that stops sets the stopped flag and
// every later launch returns at entry.  One read-back and one synchronisation per call.
int vxs_lio_run(vxs_ctx* ctx, const char* who, const double* pv12, int64_t n, bool has_map, const vxs_lio_assoc& assoc, double* state24, double* cov225, int32_t* ok,
                int32_t* iters, int64_t* match_num, double* trace12, int32_t* flags) {
  cudaSetDevice(ctx->device);
  OdomScratch* s = odom_scratch(ctx);
  if (pv12) { int rc = vxs_odom_set_resident_scan(ctx, pv12, n); if (rc) return rc; }
  else if (n != s->n_pts) return vxs_fail(ctx, VXS_ERR_ARG, (std::string(who) + ": no resident scan of this size").c_str());
  LioState h;
  std::memset(&h, 0, sizeof h);
  for (int k = 0; k < 12; k++) h.st[k] = state24[k];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) { h.st[12 + 3 * i + j] = cov225[15 * i + j]; h.st[21 + 3 * i + j] = cov225[15 * (3 + i) + 3 + j]; }
  for (int k = 0; k < 24; k++) h.x[k] = h.xp[k] = state24[k];
  for (int k = 0; k < 225; k++) h.cov[k] = cov225[k];
  const unsigned grid = (n > 0 && has_map) ? unsigned((n + OD_THREADS - 1) / OD_THREADS) : 0u;
  VXS_CUDA(ctx, s->lio.reserve((sizeof(LioState) + 7) / 8));
  VXS_CUDA(ctx, s->parts.reserve(size_t(std::max(grid, 1u)) * 34));
  int* dflags = nullptr;
  if (flags && n > 0) { VXS_CUDA(ctx, s->flags.reserve(size_t(n))); dflags = s->flags.p; }
  LioState* d = reinterpret_cast<LioState*>(s->lio.p);
  VXS_CUDA(ctx, cudaMemcpyAsync(d, &h, sizeof h, cudaMemcpyHostToDevice, ctx->stream));
  if (dflags && !grid) VXS_CUDA(ctx, cudaMemsetAsync(dflags, 0, size_t(n) * 4, ctx->stream));
  VXS_LAUNCH(ctx, "k_lio_init", k_lio_init, 1, LIO_THREADS, 0, d);
  for (int it = 0; it < 4; it++) {
    if (grid) { int rc = assoc(grid, s->pts.p, (long long)n, d->st, &d->stopped, s->parts.p, dflags); if (rc) return rc; }
    VXS_LAUNCH(ctx, "k_lio_step", k_lio_step, 1, LIO_THREADS, 0, d, s->parts.p, int(grid));
  }
  VXS_CUDA(ctx, cudaMemcpyAsync(&h, d, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
  if (dflags) VXS_CUDA(ctx, cudaMemcpyAsync(flags, dflags, size_t(n) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (h.err) return vxs_fail(ctx, VXS_ERR_ARG, (std::string(who) + ": exact zero pivot in the inverse of the covariance").c_str());
  for (int k = 0; k < 24; k++) state24[k] = h.x[k];
  for (int k = 0; k < 225; k++) cov225[k] = h.cov[k];
  *ok = h.ok; *iters = h.iters; *match_num = int64_t(h.match_num);
  if (trace12) for (int k = 0; k < 12; k++) trace12[k] = h.trace[k];
  return VXS_OK;
}

extern "C" int vxs_odom_lio_update(vxs_ctx* ctx, const double* pv12, int64_t n, double* state24, double* cov225, int32_t* ok, int32_t* iters, int64_t* match_num, double* trace12,
                                   int32_t* flags) {
  if (!ctx || n < 0 || !state24 || !cov225 || !ok || !iters || !match_num) return VXS_ERR_ARG;
  OdomScratch* s = odom_scratch(ctx);
  auto assoc = [&](unsigned grid, const double* pv, long long np, const double* st, const int* stopped, double* rows, int* fl) -> int {
    VXS_LAUNCH(ctx, "k_odom_accumulate_rows", k_odom_accumulate<true>, grid, OD_THREADS, 0, pv, np, st, s->keys.p, s->rows.p, s->n_planes, s->minx, s->miny, s->minz, s->ex, s->ey,
               s->ez, s->voxel_size, s->max_layer, rows, fl, stopped);
    return VXS_OK;
  };
  return vxs_lio_run(ctx, "vxs_odom_lio_update", pv12, n, s->n_planes > 0, assoc, state24, cov225, ok, iters, match_num, trace12, flags);
}
