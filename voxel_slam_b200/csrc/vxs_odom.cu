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
#include <algorithm>
#include <cmath>
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
  DevBuf<int> flags;
  long long n_planes = 0, n_pts = 0;
  long long minx = 0, miny = 0, minz = 0, ex = 0, ey = 0, ez = 0;
  double voxel_size = 1.0;
  int max_layer = 0;
};

__global__ void __launch_bounds__(256) k_odom_accumulate(const double* __restrict__ pv, long long n, const double* __restrict__ st /* R9 p3 rotvar9 tslvar9 */,
                                                         const unsigned long long* __restrict__ keys, const double* __restrict__ rows, long long n_planes, long long minx,
                                                         long long miny, long long minz, long long ex, long long ey, long long ez, double voxel_size, int max_layer,
                                                         double* __restrict__ out /* HTH 36 | HTz 6 | nnt 9 | count */, int* __restrict__ flags) {
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
  od_flush(acc, out);
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

OdomScratch* odom_scratch(vxs_ctx* c) { if (!c->odom_scratch) c->odom_scratch = new OdomScratch(); return static_cast<OdomScratch*>(c->odom_scratch); }

}  // namespace

void vxs_odom_release(vxs_ctx* c) {
  if (!c->odom_scratch) return;
  OdomScratch* s = static_cast<OdomScratch*>(c->odom_scratch);
  s->keys.release(); s->rows.release(); s->pts.release(); s->out.release(); s->st.release(); s->flags.release();
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
    VXS_LAUNCH(ctx, "k_odom_accumulate", k_odom_accumulate, unsigned((n + 255) / 256), 256, 0, s->pts.p, (long long)n, s->st.p, s->keys.p, s->rows.p, s->n_planes, s->minx, s->miny, s->minz,
               s->ex, s->ey, s->ez, s->voxel_size, s->max_layer, s->out.p, dflags);
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
