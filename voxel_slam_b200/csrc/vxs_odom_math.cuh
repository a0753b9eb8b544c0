// The per-point part of the EKF update once the leaf of a world point is known (shared by vxs_odom.cu — exported plane table — and
// vxs_map.cu — the resident map): OctoTree::match's 3-sigma gates in the reference's float arithmetic (voxel_map.hpp:1339-1363) and the
// HTH / HTz / nnt / match_num contributions of voxelslam.cpp:900-913.
// Bit-exact against the reference: the gate operands d, n.d and d.d (rounded intrinsics, no FMA), hence the range gate and, but for
// sigma_l, the 3-sigma gate.  Held to a tolerance: sigma_l (formed from the upper triangle of plane_var, in another order) and the
// accumulated sums.  sigma_l can only flip a flag where 3 sqrt(sigma_l) lies within its own rounding of float(|n.d|).
#pragma once
#define OD_ROW 28   // per plane: centre 3, normal 3, plane_var upper triangle 21, radius 1
// r: the 28-double plane row; (x, y, z) body point, (wx, wy, wz) world point, p = pointVar record (pnt 3 | var 9), st = R9 p3 rot_var9 tsl_var9.
// acc[34]: HTH upper triangle 21 | HTz 6 | nnt 6 | count.  Returns 1 when the point matched.
__device__ __forceinline__ int od_contribution(const double* r, double x, double y, double z, double wx, double wy, double wz, const double* __restrict__ p, const double* __restrict__ st,
                                               double* acc) {
  const double R[9] = {st[0], st[1], st[2], st[3], st[4], st[5], st[6], st[7], st[8]};
  const double c[3] = {r[0], r[1], r[2]}, nr[3] = {r[3], r[4], r[5]};
  // the gate operands in the reference's order and without FMA contraction (voxel_map.hpp:1339-1341): a contracted n.d or d.d rounds
  // differently, and a point within rounding of a gate then flips its flag
  const double d[3] = {__dsub_rn(wx, c[0]), __dsub_rn(wy, c[1]), __dsub_rn(wz, c[2])};
  const double nd = __dadd_rn(__dadd_rn(__dmul_rn(nr[0], d[0]), __dmul_rn(nr[1], d[1])), __dmul_rn(nr[2], d[2]));
  const float dis_to_plane = (float)fabs(nd);
  const float dis_to_center = (float)__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
  const float range_dis = __fsub_rn(dis_to_center, __fmul_rn(dis_to_plane, dis_to_plane));
  if (!(range_dis <= __fmul_rn(9.0f, (float)r[27]))) return 0;
  // sigma_l = J plane_var J^T + n^T var_world n,  J = [d | -n]
  const double J[6] = {d[0], d[1], d[2], -nr[0], -nr[1], -nr[2]};
  double sigma_l = 0.0;
  int t = 6;
#pragma unroll
  for (int a = 0; a < 6; a++)
#pragma unroll
    for (int b = a; b < 6; b++) { const double v = r[t++]; sigma_l += (a == b ? 1.0 : 2.0) * v * J[a] * J[b]; }
  // var_world = R var R^T + phat rot_var phat^T + tsl_var; only n^T (.) n is needed:  (R^T n)^T var (R^T n) + (phat^T n)^T rot_var (phat^T n) + n^T tsl_var n
  const double a1[3] = {R[0] * nr[0] + R[3] * nr[1] + R[6] * nr[2], R[1] * nr[0] + R[4] * nr[1] + R[7] * nr[2], R[2] * nr[0] + R[5] * nr[1] + R[8] * nr[2]};   // R^T n
  const double a2[3] = {-(z * nr[1] - y * nr[2]), -(x * nr[2] - z * nr[0]), -(y * nr[0] - x * nr[1])};   // phat^T n = -(p x n)
  const double* var = p + 3;
  const double* rv = st + 12; const double* tv = st + 21;
  double q = 0.0;
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) q += a1[a] * var[3 * a + b] * a1[b] + a2[a] * rv[3 * a + b] * a2[b] + nr[a] * tv[3 * a + b] * nr[b];
  sigma_l += q;
  if (!((double)dis_to_plane < 3.0 * sqrt(sigma_l))) return 0;
  const double R_inv = 1.0 / (0.0005 + sigma_l);
  // jac.head(3) = phat R^T n = p x (R^T n),  jac.tail(3) = n
  const double jac[6] = {y * a1[2] - z * a1[1], z * a1[0] - x * a1[2], x * a1[1] - y * a1[0], nr[0], nr[1], nr[2]};
  int u = 0;
#pragma unroll
  for (int a = 0; a < 6; a++)
#pragma unroll
    for (int b = a; b < 6; b++) acc[u++] = R_inv * jac[a] * jac[b];           // 21: upper triangle of HTH
#pragma unroll
  for (int a = 0; a < 6; a++) acc[21 + a] = -R_inv * jac[a] * nd;                // HTz
  acc[27] = nr[0] * nr[0]; acc[28] = nr[0] * nr[1]; acc[29] = nr[0] * nr[2]; acc[30] = nr[1] * nr[1]; acc[31] = nr[1] * nr[2]; acc[32] = nr[2] * nr[2];
  acc[33] = 1.0;
  return 1;
}
// warp reduction of the 34 sums, one fp64 RED per value and warp
__device__ __forceinline__ void od_flush(const double* acc, double* __restrict__ out) {
#pragma unroll
  for (int k = 0; k < 34; k++) {
    double v = acc[k];
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
    if ((threadIdx.x & 31) == 0 && v != 0.0) atomicAdd(out + k, v);
  }
}
// The same 34 sums without atomics, for the iterated EKF update whose branches they decide: the warp tree above, then the warps of the
// block in ascending order through shared memory, one partial row per block (row = out + 34 * blockIdx.x).  Bit-reproducible for a fixed
// grid.  Every thread of the block must reach it; blockDim.x == OD_THREADS.
#define OD_THREADS 256
__device__ __forceinline__ void od_flush_row(const double* acc, double* __restrict__ out) {
  __shared__ double red[OD_THREADS / 32][34];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 34; k++) {
    double v = acc[k];
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
    if (lane == 0) red[w][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 34) {
    double s = red[0][threadIdx.x];
#pragma unroll
    for (int j = 1; j < OD_THREADS / 32; j++) s += red[j][threadIdx.x];
    out[34 * size_t(blockIdx.x) + threadIdx.x] = s;
  }
}
