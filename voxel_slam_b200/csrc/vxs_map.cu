// Persistent, device-resident local voxel map of the sliding-window loop (SURVEY.md §8f rank 1): the state that the reference keeps
// in `surf_map` / `surf_map_slide` (unordered_map<VOXEL_LOC, OctoTree*>) across scans, and the per-scan functions around the BA:
//   cut_voxel / cut_voxel_multi     voxel_map.hpp:1504-1639   one NEW scan into the map (root-cell lookup / insert, descent, push)
//   OctoTree::push / push_fix / allocate / subdivide / fix_divide   :969-1116, Bf_var :91-106 (the 9x9 cov_add by-product)
//   multi_recut + OctoTree::recut   voxelslam.cpp:1398-1453, voxel_map.hpp:1148-1194   re-decide every leaf of the slide trees
//   OctoTree::tras_opt              :1308-1333   factor of the current window straight into the device CSR
//   multi_margi + OctoTree::margi   voxelslam.cpp:1321-1395, voxel_map.hpp:1196-1305   after the BA: take pcr_add / eig back from the
//                                   factor, move the oldest scan into pcr_fix / point_fix, plane_update :1118-1146, isexist, slide erase,
//                                   clear_slwd :1482-1500, ring rotation voxelslam.cpp:1689-1693
// so that a scan costs one upload of ITS points instead of the from-scratch rebuild of the whole window (vxs_build_window_factor).
//
// GPU formulation — no pointer octree, no per-voxel mutex:
//   * node table (SoA, append-only): root cell / layer / octant path / centre / quarter length / 8 child links / flags, pcr_add, pcr_fix,
//     the 45 unique entries of cov_add, eig, the plane row the odometry kernel reads; roots are found through an open-addressing hash
//     table over VOXEL_LOC; nodes are created with a claim-CAS and a second pass for the points that met a claim in flight;
//   * the slide windows (`SlideWindow`, W clusters per leaf) live in a block pool with a free list (the reference recycles them in `sws`);
//   * points never move: every resident scan keeps a leaf id per point (and the marginalised points that stay re-cuttable — point_fix —
//     sit in a pool with a leaf id); a subdivision re-labels the points of the subdivided leaves with the CURRENT poses
//     (voxel_map.hpp:1100, parity trap B#4) and re-accumulates them;
//   * every accumulation is a stable sort by (node, slot) + one thread group per node, so sums are deterministic;
//   * recut is level by level: one thread per leaf decides dead / plane / subdivide (fp64 Jacobi eigensolve), subdivisions are rare after
//     the first scans of a window.
// The reference's early-outs when there are fewer roots than threads (cut_voxel_multi :1597, multi_recut VS:1409, multi_margi VS:1343,
// parity trap B#16) are NOT reproduced: the work is always done.
#include <math.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "vxs_internal.h"
#include "vxs_math.cuh"
#include "vxs_sortscan.cuh"
#include "vxs_odom_math.cuh"

using namespace vxs;

namespace {

enum : unsigned int { F_INNER = 1u, F_EXIST = 2u, F_PLANE = 4u, F_SLIDE = 8u, F_MARK = 16u, F_DROP = 32u, F_KEEPFIX = 64u, F_KILLFIX = 128u };
#define MAP_RETRY (-2)
#define MAP_CLAIM 0xFFFFFFFFu
#define MAP_MAX_MG 4
#define PLANE_ROW 28          // centre 3 | normal 3 | upper triangle of the 6x6 plane_var (21) | radius — the row format of vxs_odom.cu

struct NodeView {
  size_t cap;
  int* root; int* child; unsigned int* flags; int* layer; int* path; int* sw; int* opt; int* last_num;
  long long* rkey; double* center; float* quater;
  double* add; double* fix; double* cov; double* eig; double* plane;
};

struct MapState;

}  // namespace

struct vxs_map {
  vxs_ctx* ctx = nullptr;
  vxs_map_params mp;
  int W = 0, max_points = 100;
  // nodes
  size_t ncap = 0; int n_nodes = 0;
  DevBuf<int> n_root, n_child, n_layer, n_path, n_sw, n_opt, n_last;
  DevBuf<unsigned int> n_flags;
  DevBuf<long long> n_rkey;
  DevBuf<double> n_center, n_add, n_fix, n_cov, n_eig, n_plane;
  DevBuf<float> n_quater;
  // root hash
  DevBuf<unsigned int> table; size_t tcap = 0;
  // counters on device: [0] node count, [1] sw bump, [2] free-list top, [3] marks, [4] fix count (appends), [5..] scratch
  DevBuf<int> counters;
  // slide-window block pool
  DevBuf<double> swp; size_t swcap = 0; int sw_bump = 0;
  DevBuf<int> sw_free;
  // resident scans, one per ring slot
  std::vector<DevBuf<double>*> scan_pv; std::vector<DevBuf<int>*> scan_leaf; std::vector<long long> scan_n;
  DevBuf<unsigned long long> scan_ptrs;     // [2][W+1] device pointers (pv12, leaf) per slot; entry W = fix pool
  // fix pool (point_fix of all leaves)
  DevBuf<double> fix_pv, fix_pv2; DevBuf<int> fix_leaf, fix_leaf2; long long fix_n = 0, fix_dead = 0;   // *2 = spare pool of the compaction (ping-pong)
  // ring: logical window position -> slot (voxel_map.hpp:934 `int* mp`)
  std::vector<int> ring;
  DevBuf<int> d_ring;        // [W] ring | [W+1] inverse (slot -> logical, entry W = W for the fix pseudo slot)
  DevBuf<double> d_poses;    // [W+1][12], entry W = identity
  DevBuf<long long> d_off;   // prefix of the virtual point index space
  // scratch
  SortScratch ss;
  DevBuf<unsigned long long> keysA, keysB, refs, rec_key;
  DevBuf<unsigned int> idxA, idxB, flagbuf, scanbuf, rec_start, node_of_rec, node_rec_start, nflag;
  DevBuf<unsigned int> sel, nent, voff, eoff;
  DevBuf<double> odom_st;    // pose / covariance block and the 34 sums of vxs_map_odom_accumulate
  int win_count = 0;
  long long bb[6] = {0, 0, 0, 0, 0, 0}; bool bb_valid = false;
};

namespace {

static NodeView view(vxs_map* m) {
  NodeView v;
  v.cap = m->ncap; v.root = m->n_root.p; v.child = m->n_child.p; v.flags = m->n_flags.p; v.layer = m->n_layer.p; v.path = m->n_path.p; v.sw = m->n_sw.p; v.opt = m->n_opt.p;
  v.last_num = m->n_last.p; v.rkey = m->n_rkey.p; v.center = m->n_center.p; v.quater = m->n_quater.p; v.add = m->n_add.p; v.fix = m->n_fix.p; v.cov = m->n_cov.p; v.eig = m->n_eig.p;
  v.plane = m->n_plane.p;
  return v;
}

// ---- bit-exact cell arithmetic (same routines as vxs_voxelize.cu)
__device__ __forceinline__ double dot3_rn(double a0, double a1, double a2, double x, double y, double z, double t) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, x), __dmul_rn(a1, y)), __dmul_rn(a2, z)), t);
}
__device__ __forceinline__ d3 world_point(const double* __restrict__ pose, d3 p) {
  return mk3(dot3_rn(pose[0], pose[1], pose[2], p.x, p.y, p.z, pose[9]), dot3_rn(pose[3], pose[4], pose[5], p.x, p.y, p.z, pose[10]),
             dot3_rn(pose[6], pose[7], pose[8], p.x, p.y, p.z, pose[11]));
}
__device__ __forceinline__ long long quantise(double pw, double voxel_size) {
  float loc = __double2float_rn(__ddiv_rn(pw, voxel_size));
  if (loc < 0.0f) loc = __fsub_rn(loc, 1.0f);
  return __float2ll_rz(loc);
}
__device__ __forceinline__ unsigned int table_hash(long long x, long long y, long long z) {
  unsigned long long h = (unsigned long long)x * 0x9E3779B97F4A7C15ull ^ ((unsigned long long)y * 0xC2B2AE3D27D4EB4Full + 0x165667B19E3779F9ull) ^ ((unsigned long long)z * 0xD6E8FEB86659FD93ull);
  h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 32;
  return (unsigned int)h;
}
__device__ __forceinline__ int octant_of(const NodeView& nv, int node, d3 w) {   // voxel_map.hpp:1029-1032
  const int bx = w.x > nv.center[node], by = w.y > nv.center[nv.cap + node], bz = w.z > nv.center[2 * nv.cap + node];
  return 4 * bx + 2 * by + bz;
}
__device__ __forceinline__ void init_common(const NodeView& nv, int idx, int root, int layer, int path) {
  nv.root[idx] = root; nv.layer[idx] = layer; nv.path[idx] = path; nv.sw[idx] = -1; nv.opt[idx] = -1; nv.last_num[idx] = 0; nv.flags[idx] = 0u;
}
// child creation (voxel_map.hpp:1034-1040): centre = parent centre + (2 b - 1) * quater_length (int * float -> float, then double +), quater halves
__device__ __forceinline__ void init_child(const NodeView& nv, int idx, int parent, int oct) {
  init_common(nv, idx, nv.root[parent], nv.layer[parent] + 1, nv.path[parent] * 8 + oct);
  const float q = nv.quater[parent];
  const int b[3] = {(oct >> 2) & 1, (oct >> 1) & 1, oct & 1};
  for (int k = 0; k < 3; k++) nv.center[k * nv.cap + idx] = __dadd_rn(nv.center[k * nv.cap + parent], (double)__fmul_rn((float)(2 * b[k] - 1), q));
  nv.quater[idx] = __fdiv_rn(q, 2.0f);
}
// returns the child of `node` for octant `oct`, creating it if needed; MAP_RETRY when another thread is creating it right now
__device__ __forceinline__ int child_find_or_create(const NodeView& nv, int node, int oct, int* count) {
  int* slot = nv.child + size_t(oct) * nv.cap + node;
  int c = *((volatile int*)slot);
  if (c == -1) {
    const int old = atomicCAS(slot, -1, MAP_RETRY);
    if (old == -1) {
      const int idx = atomicAdd(count, 1);
      init_child(nv, idx, node, oct);
      __threadfence();
      atomicExch(slot, idx);
      return idx;
    }
    c = old;
  }
  return c;     // >= 0 or MAP_RETRY
}

// ---------------------------------------------------------------- cut_voxel of the new scan: root lookup / insert + descent
__global__ void __launch_bounds__(256) k_map_locate(NodeView nv, unsigned int* __restrict__ table, unsigned int tmask, int* __restrict__ count, const double* __restrict__ pv12, long long n,
                                                    const double* __restrict__ pose, double voxel_size, int* __restrict__ leaf_out, int pass) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (pass > 0 && leaf_out[i] != MAP_RETRY) return;
  const double* p = pv12 + 12 * i;
  const d3 w = world_point(pose, mk3(p[0], p[1], p[2]));
  const long long kx = quantise(w.x, voxel_size), ky = quantise(w.y, voxel_size), kz = quantise(w.z, voxel_size);
  unsigned int h = table_hash(kx, ky, kz) & tmask;
  int node = -1;
  for (;;) {
    unsigned int v = *((volatile unsigned int*)(table + h));
    if (v == 0u) {
      const unsigned int old = atomicCAS(table + h, 0u, MAP_CLAIM);
      if (old == 0u) {
        const int idx = atomicAdd(count, 1);
        init_common(nv, idx, idx, 0, 0);
        nv.rkey[idx] = kx; nv.rkey[nv.cap + idx] = ky; nv.rkey[2 * nv.cap + idx] = kz;
        nv.center[idx] = __dmul_rn(__dadd_rn(0.5, (double)kx), voxel_size);              // (0.5 + position.x) * voxel_size   voxel_map.hpp:1530-1532
        nv.center[nv.cap + idx] = __dmul_rn(__dadd_rn(0.5, (double)ky), voxel_size);
        nv.center[2 * nv.cap + idx] = __dmul_rn(__dadd_rn(0.5, (double)kz), voxel_size);
        nv.quater[idx] = __double2float_rn(__ddiv_rn(voxel_size, 4.0));                  // :1533
        __threadfence();
        atomicExch(table + h, (unsigned int)idx + 1u);
        node = idx;
        break;
      }
      v = old;
    }
    if (v == MAP_CLAIM) { leaf_out[i] = MAP_RETRY; atomicAdd(count + 7, 1); return; }
    const int r = int(v - 1u);
    // the key of a root another block may have published in this launch: read it at L2 (__ldcg).  A plain load can hit an L1 line cached
    // before the publication (while probing its neighbours), miss the match, and the probe would then insert the same cell a second time.
    if (__ldcg(nv.rkey + r) == kx && __ldcg(nv.rkey + nv.cap + r) == ky && __ldcg(nv.rkey + 2 * nv.cap + r) == kz) { node = r; break; }
    h = (h + 1u) & tmask;
  }
  atomicOr(nv.flags + node, F_EXIST | F_SLIDE);          // iter->second->isexist = true; feat_tem_map[position] = ...   :1523-1526
  while (*((volatile unsigned int*)(nv.flags + node)) & F_INNER) {
    const int c = child_find_or_create(nv, node, octant_of(nv, node, w), count);
    if (c == MAP_RETRY) { leaf_out[i] = MAP_RETRY; atomicAdd(count + 7, 1); return; }
    node = c;
  }
  leaf_out[i] = node;
}

// refs / keys of the new scan for the accumulation: key = (leaf << 8) | slot
__global__ void __launch_bounds__(256) k_map_scan_keys(const int* __restrict__ leaf, long long n, int slot, unsigned long long* __restrict__ keys, unsigned int* __restrict__ idx,
                                                       unsigned long long* __restrict__ refs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = ((unsigned long long)(unsigned int)leaf[i] << 8) | (unsigned long long)slot;
  idx[i] = (unsigned int)i;
  refs[i] = ((unsigned long long)slot << 32) | (unsigned long long)i;
}

// ---------------------------------------------------------------- slide-window blocks
__device__ __forceinline__ int sw_alloc(int* counters, const int* __restrict__ sw_free) {
  for (;;) {   // pop the free list, else bump
    const int t = *((volatile int*)(counters + 2));
    if (t <= 0) break;
    if (atomicCAS(counters + 2, t, t - 1) == t) return sw_free[t - 1];
  }
  return atomicAdd(counters + 1, 1);
}
// one thread per node head of the sorted record list: a node that receives window points (slot < W) gets its SlideWindow (push :972-983) and isexist
__global__ void __launch_bounds__(128) k_map_alloc_sw(NodeView nv, const unsigned int* __restrict__ node_rec_start, const unsigned long long* __restrict__ rec_key, unsigned int Nn, int W,
                                                      int* counters, const int* __restrict__ sw_free) {
  const unsigned int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= Nn) return;
  const unsigned long long k = rec_key[node_rec_start[h]];       // records of a node are sorted by slot: the first one tells whether any is a window slot
  if (int(k & 255ull) >= W) return;
  const int node = int(k >> 8);
  if (nv.sw[node] < 0) nv.sw[node] = sw_alloc(counters, sw_free);
  nv.flags[node] |= F_EXIST;
}

// Bf_var (voxel_map.hpp:91-106), upper triangle of the symmetric 9x9 in row-major packed order (45 entries) added to acc
__device__ __forceinline__ void bf_var_acc(const double* __restrict__ var, d3 v, double* acc) {
  const double Bi[6][3] = {{2 * v.x, 0, 0}, {v.y, v.x, 0}, {v.z, 0, v.x}, {0, 2 * v.y, 0}, {0, v.z, v.y}, {0, 0, 2 * v.z}};
  double Bu[6][3];
#pragma unroll
  for (int r = 0; r < 6; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) Bu[r][c] = (Bi[r][0] * var[c] + Bi[r][1] * var[3 + c]) + Bi[r][2] * var[6 + c];
  int t = 0;
#pragma unroll
  for (int r = 0; r < 9; r++)
#pragma unroll
    for (int c = r; c < 9; c++) {
      double val;
      if (r < 6 && c < 6) val = (Bu[r][0] * Bi[c][0] + Bu[r][1] * Bi[c][1]) + Bu[r][2] * Bi[c][2];
      else if (r < 6) val = Bu[r][c - 6];
      else val = var[3 * (r - 6) + (c - 6)];
      acc[t++] += val;
    }
}

struct PointSrcs { const unsigned long long* ptrs; const int* inv_ring; const double* poses; int W; };   // ptrs[slot] = pv12 of the slot (W = fix pool)

// G lanes per node: every record (node, slot) of the node in turn — push (:985-992) / push_fix (:996-1005) of all its points:
//   slot < W : sw->pcrs_local[slot] += p_body p_body^T ...,  pcr_add += p_world ...,  cov_add += Bf_var(var, p_world)
//   slot = W : pcr_fix += p, pcr_add += p, cov_add += Bf_var(var, p)       (fixed points are already in world coordinates)
template <int G>
__global__ void __launch_bounds__(128) k_map_accum(NodeView nv, PointSrcs src, const unsigned int* __restrict__ vs, const unsigned long long* __restrict__ refs,
                                                   const unsigned int* __restrict__ rec_start, const unsigned long long* __restrict__ rec_key,
                                                   const unsigned int* __restrict__ node_rec_start, unsigned int Nn, double* __restrict__ swp, int with_cov) {
  const int lane = threadIdx.x & (G - 1);
  const unsigned int grp = (blockIdx.x * blockDim.x + threadIdx.x) / G, ngrp = (gridDim.x * blockDim.x) / G;
  const unsigned int iters = (Nn + ngrp - 1) / ngrp;
  const int W = src.W;
  for (unsigned int it = 0; it < iters; it++) {
    const unsigned int h = grp + it * ngrp;
    const bool valid = h < Nn;
    unsigned int rb = 0, re = 0;
    if (valid) { rb = node_rec_start[h]; re = node_rec_start[h + 1]; }
    double wsum[10], cv[45];
#pragma unroll
    for (int k = 0; k < 10; k++) wsum[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 45; k++) cv[k] = 0.0;
    int node = 0;
    for (unsigned int r = rb; r < re; r++) {
      const unsigned long long key = rec_key[r];
      node = int(key >> 8);
      const int slot = int(key & 255ull);
      const double* base = reinterpret_cast<const double*>(src.ptrs[slot]);
      const double* pose = src.poses + 12 * src.inv_ring[slot];
      double ls[10];
#pragma unroll
      for (int k = 0; k < 10; k++) ls[k] = 0.0;
      for (unsigned int j = rec_start[r] + lane; j < rec_start[r + 1]; j += G) {
        const unsigned long long ref = refs[vs[j]];
        const double* p = base + 12 * size_t(ref & 0xFFFFFFFFull);
        const d3 b = mk3(p[0], p[1], p[2]);
        const d3 w = slot < W ? world_point(pose, b) : b;
        ls[0] += b.x * b.x; ls[1] += b.x * b.y; ls[2] += b.x * b.z; ls[3] += b.y * b.y; ls[4] += b.y * b.z; ls[5] += b.z * b.z; ls[6] += b.x; ls[7] += b.y; ls[8] += b.z; ls[9] += 1.0;
        wsum[0] += w.x * w.x; wsum[1] += w.x * w.y; wsum[2] += w.x * w.z; wsum[3] += w.y * w.y; wsum[4] += w.y * w.z; wsum[5] += w.z * w.z; wsum[6] += w.x; wsum[7] += w.y; wsum[8] += w.z;
        wsum[9] += 1.0;
        if (with_cov) bf_var_acc(p + 3, w, cv);
      }
#pragma unroll
      for (int k = 0; k < 10; k++)
#pragma unroll
        for (int off = G / 2; off > 0; off >>= 1) ls[k] += __shfl_xor_sync(0xffffffffu, ls[k], off);
      if (lane == 0) {
        if (slot < W) { double* d = swp + (size_t(nv.sw[node]) * W + slot) * 10; for (int k = 0; k < 10; k++) d[k] += ls[k]; }
        else for (int k = 0; k < 10; k++) nv.fix[size_t(k) * nv.cap + node] += ls[k];
      }
    }
#pragma unroll
    for (int k = 0; k < 10; k++)
#pragma unroll
      for (int off = G / 2; off > 0; off >>= 1) wsum[k] += __shfl_xor_sync(0xffffffffu, wsum[k], off);
    if (with_cov) {
#pragma unroll
      for (int k = 0; k < 45; k++)
#pragma unroll
        for (int off = G / 2; off > 0; off >>= 1) cv[k] += __shfl_xor_sync(0xffffffffu, cv[k], off);
    }
    if (valid && lane == 0 && re > rb) {
      for (int k = 0; k < 10; k++) nv.add[size_t(k) * nv.cap + node] += wsum[k];
      if (with_cov) for (int k = 0; k < 45; k++) nv.cov[size_t(k) * nv.cap + node] += cv[k];
    }
  }
}

// ---------------------------------------------------------------- recut (voxel_map.hpp:1148-1172), one layer
struct DecideArgs { double min_eigen_value, thre, min_point; int layer, max_layer; };
__global__ void __launch_bounds__(128) k_map_decide(NodeView nv, int n_nodes, DecideArgs a, int* __restrict__ counters) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes) return;
  unsigned int f = nv.flags[nd];
  if ((f & F_INNER) || nv.layer[nd] != a.layer || !(nv.flags[nv.root[nd]] & F_SLIDE)) return;
  nv.opt[nd] = -1;
  cluster S;
  S.P.xx = nv.add[nd]; S.P.xy = nv.add[nv.cap + nd]; S.P.xz = nv.add[2 * nv.cap + nd]; S.P.yy = nv.add[3 * nv.cap + nd]; S.P.yz = nv.add[4 * nv.cap + nd]; S.P.zz = nv.add[5 * nv.cap + nd];
  S.v = mk3(nv.add[6 * nv.cap + nd], nv.add[7 * nv.cap + nd], nv.add[8 * nv.cap + nd]); S.n = nv.add[9 * nv.cap + nd];
  if (S.n <= a.min_point) { nv.flags[nd] = f & ~F_PLANE; return; }
  if (!(f & F_EXIST) || nv.sw[nd] < 0) return;
  double w[3]; d3 u0, u1, u2;
  eig3_jacobi(cov_from_sum(S), w, u0, u1, u2);
  const size_t c = nv.cap;
  nv.eig[nd] = w[0]; nv.eig[c + nd] = w[1]; nv.eig[2 * c + nd] = w[2];
  nv.eig[3 * c + nd] = u0.x; nv.eig[4 * c + nd] = u1.x; nv.eig[5 * c + nd] = u2.x; nv.eig[6 * c + nd] = u0.y; nv.eig[7 * c + nd] = u1.y; nv.eig[8 * c + nd] = u2.y;
  nv.eig[9 * c + nd] = u0.z; nv.eig[10 * c + nd] = u1.z; nv.eig[11 * c + nd] = u2.z;
  const bool plane = (w[0] < a.min_eigen_value) && (w[0] / w[2] < a.thre);                 // plane_judge :1015-1019
  if (plane) { nv.flags[nd] = f | F_PLANE; return; }
  f &= ~F_PLANE;
  if (a.layer < a.max_layer) { f |= F_MARK; atomicAdd(counters + 3, 1); }
  nv.flags[nd] = f;
}

// virtual index space over the window scans in logical order (entry wc = the fix pool): j -> (logical i, local index)
struct VirtPts { const long long* off; int nseg; };
__device__ __forceinline__ int seg_of(const VirtPts& v, long long j) {
  int lo = 0, hi = v.nseg;
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (v.off[mid] <= j) lo = mid; else hi = mid; }
  return lo;
}
// flag the points (window scans + fix pool) whose leaf is marked for subdivision
__global__ void __launch_bounds__(256) k_map_flag_marked(NodeView nv, VirtPts vp, const unsigned long long* __restrict__ leaf_ptrs, const int* __restrict__ ring, int wc, int W, long long total,
                                                         unsigned int* __restrict__ flag) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= total) return;
  const int s = seg_of(vp, j);
  const int slot = s < wc ? ring[s] : W;
  const int* lf = reinterpret_cast<const int*>(leaf_ptrs[slot]);
  const int l = lf[j - vp.off[s]];
  flag[j] = (l >= 0 && (nv.flags[l] & F_MARK)) ? 1u : 0u;
}
// subdivide (:1096-1116) / fix_divide (:1074-1094): new leaf of every flagged point, with the CURRENT pose of its scan
__global__ void __launch_bounds__(256) k_map_subdiv_assign(NodeView nv, VirtPts vp, PointSrcs src, const unsigned long long* __restrict__ leaf_ptrs, const int* __restrict__ ring, int wc, long long total,
                                                           const unsigned int* __restrict__ flag, const unsigned int* __restrict__ pos, int* __restrict__ count, int max_layer,
                                                           unsigned long long* __restrict__ keys, unsigned int* __restrict__ idx, unsigned long long* __restrict__ refs, int pass) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= total || !flag[j]) return;
  const unsigned int o = pos[j];
  if (pass > 0 && keys[o] != ~0ull) return;
  const int W = src.W;
  const int s = seg_of(vp, j);
  const int slot = s < wc ? ring[s] : W;
  const long long li = j - vp.off[s];
  int* lf = reinterpret_cast<int*>(leaf_ptrs[slot]);
  const int parent = lf[li];
  const double* p = reinterpret_cast<const double*>(src.ptrs[slot]) + 12 * size_t(li);
  const d3 b = mk3(p[0], p[1], p[2]);
  const d3 w = slot < W ? world_point(src.poses + 12 * s, b) : b;
  const int c = child_find_or_create(nv, parent, octant_of(nv, parent, w), count);
  idx[o] = o;
  refs[o] = ((unsigned long long)slot << 32) | (unsigned long long)li;
  if (c == MAP_RETRY) { keys[o] = ~0ull; atomicAdd(count + 7, 1); return; }
  keys[o] = ((unsigned long long)(unsigned int)c << 8) | (unsigned long long)slot;
  // fixed points are only kept re-cuttable below max_layer (push_fix :998-999); window points keep their leaf at every layer
  lf[li] = (slot == W && nv.layer[c] >= max_layer) ? -1 : c;
}
// the subdivided leaves become inner nodes: sw->clear(); sws.push_back(sw); sw = nullptr; octo_state = 1   (:1182-1185)
__global__ void __launch_bounds__(128) k_map_finish_subdiv(NodeView nv, int n_nodes, int W, double* __restrict__ swp, int* __restrict__ counters, int* __restrict__ sw_free) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes) return;
  const unsigned int f = nv.flags[nd];
  if (!(f & F_MARK)) return;
  nv.flags[nd] = (f | F_INNER) & ~F_MARK;
  const int b = nv.sw[nd];
  if (b >= 0) {
    double* d = swp + size_t(b) * W * 10;
    for (int k = 0; k < W * 10; k++) d[k] = 0.0;
    sw_free[atomicAdd(counters + 2, 1)] = b;
    nv.sw[nd] = -1;
  }
}

// ---------------------------------------------------------------- tras_opt (:1308-1333)
__global__ void __launch_bounds__(128) k_map_select(NodeView nv, int n_nodes, int W, const int* __restrict__ ring, const double* __restrict__ swp, unsigned int* __restrict__ sel,
                                                    unsigned int* __restrict__ nent) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes) return;
  const unsigned int f = nv.flags[nd];
  unsigned int take = 0, cnt = 0;
  if (!(f & F_INNER) && (f & F_EXIST) && (f & F_PLANE) && nv.sw[nd] >= 0 && (nv.flags[nv.root[nd]] & F_SLIDE)) {
    if (!(nv.eig[nd] / nv.eig[nv.cap + nd] > 0.12)) {
      take = 1;
      const double* d = swp + size_t(nv.sw[nd]) * W * 10;
      for (int i = 0; i < W; i++) if (d[ring[i] * 10 + 9] != 0.0) cnt++;
    }
  }
  sel[nd] = take; nent[nd] = cnt;
}
struct FactorOut { int32_t* ptr; int32_t* frame; int32_t* vox; double* cl; size_t Ecap; double* fix; double* coe; double* eig; double* sum; size_t Vcap; };
__global__ void __launch_bounds__(128) k_map_emit(NodeView nv, int n_nodes, int W, const int* __restrict__ ring, const double* __restrict__ swp, const unsigned int* __restrict__ sel,
                                                  const unsigned int* __restrict__ voff, const unsigned int* __restrict__ eoff, FactorOut fo) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes || !sel[nd]) return;
  const unsigned int v = voff[nd];
  unsigned int e = eoff[nd];
  fo.ptr[v] = int32_t(e);
  const double* d = swp + size_t(nv.sw[nd]) * W * 10;
  for (int i = 0; i < W; i++) {            // pcrs[i] = sw->pcrs_local[mp[i]]  :1317-1319; only N != 0 entries are stored (CSR)
    const double* c = d + ring[i] * 10;
    if (c[9] == 0.0) continue;
    fo.frame[e] = i; fo.vox[e] = int32_t(v);
    for (int k = 0; k < 10; k++) fo.cl[size_t(k) * fo.Ecap + e] = c[k];
    e++;
  }
  for (int k = 0; k < 10; k++) { fo.fix[size_t(k) * fo.Vcap + v] = nv.fix[size_t(k) * nv.cap + nd]; fo.sum[size_t(k) * fo.Vcap + v] = nv.add[size_t(k) * nv.cap + nd]; }
  for (int k = 0; k < 12; k++) fo.eig[size_t(k) * fo.Vcap + v] = nv.eig[size_t(k) * nv.cap + nd];
  fo.coe[v] = 1.0;
  nv.opt[nd] = int(v);                      // opt_state = vox_opt.plvec_voxels.size()  :1320
}
__global__ void k_map_last_ptr(int32_t* ptr, const unsigned int* totals) { ptr[totals[0]] = int32_t(totals[1]); }

// ---------------------------------------------------------------- margi (:1196-1305) + plane_update (:1118-1146)
__device__ __forceinline__ cluster load_node_cluster(const double* base, size_t cap, int nd) {
  cluster c;
  c.P.xx = base[nd]; c.P.xy = base[cap + nd]; c.P.xz = base[2 * cap + nd]; c.P.yy = base[3 * cap + nd]; c.P.yz = base[4 * cap + nd]; c.P.zz = base[5 * cap + nd];
  c.v = mk3(base[6 * cap + nd], base[7 * cap + nd], base[8 * cap + nd]); c.n = base[9 * cap + nd];
  return c;
}
__device__ __forceinline__ void store_node_cluster(double* base, size_t cap, int nd, const cluster& c) {
  base[nd] = c.P.xx; base[cap + nd] = c.P.xy; base[2 * cap + nd] = c.P.xz; base[3 * cap + nd] = c.P.yy; base[4 * cap + nd] = c.P.yz; base[5 * cap + nd] = c.P.zz;
  base[6 * cap + nd] = c.v.x; base[7 * cap + nd] = c.v.y; base[8 * cap + nd] = c.v.z; base[9 * cap + nd] = c.n;
}
__device__ __forceinline__ cluster zero_cluster() { cluster c; c.P.xx = c.P.xy = c.P.xz = c.P.yy = c.P.yz = c.P.zz = 0.0; c.v = mk3(0, 0, 0); c.n = 0.0; return c; }
__device__ __forceinline__ void cluster_add(cluster& a, const cluster& b, double s) {
  a.P.xx += s * b.P.xx; a.P.xy += s * b.P.xy; a.P.xz += s * b.P.xz; a.P.yy += s * b.P.yy; a.P.yz += s * b.P.yz; a.P.zz += s * b.P.zz;
  a.v.x += s * b.v.x; a.v.y += s * b.v.y; a.v.z += s * b.v.z; a.n += s * b.n;
}
__device__ __forceinline__ cluster load_slot(const double* d) { cluster c; c.P.xx = d[0]; c.P.xy = d[1]; c.P.xz = d[2]; c.P.yy = d[3]; c.P.yz = d[4]; c.P.zz = d[5]; c.v = mk3(d[6], d[7], d[8]); c.n = d[9]; return c; }

// plane.center / normal / plane_var / radius from pcr_add, eig and cov_add
__device__ void plane_update_dev(const NodeView& nv, int nd, const cluster& add, const double* w, const d3* u) {
  const size_t cap = nv.cap;
  const double N = add.n, nvv = 1.0 / N;
  const d3 center = mk3(add.v.x / N, add.v.y / N, add.v.z / N);
  double C[9][9];
  { int t = 0; for (int r = 0; r < 9; r++) for (int c = r; c < 9; c++) { const double v = nv.cov[size_t(t++) * cap + nd]; C[r][c] = v; C[c][r] = v; } }
  double uc[3][9];
  for (int a = 0; a < 3; a++) for (int c = 0; c < 9; c++) uc[a][c] = 0.0;
  const double ul[3] = {u[0].x, u[0].y, u[0].z};
  for (int k = 1; k < 3; k++) {
    const double uk[3] = {u[k].x, u[k].y, u[k].z};
    double ukl[3][3];
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) ukl[a][b] = uk[a] * ul[b];
    double fkl[9] = {ukl[0][0], ukl[1][0] + ukl[0][1], ukl[2][0] + ukl[0][2], ukl[1][1], ukl[1][2] + ukl[2][1], ukl[2][2], 0, 0, 0};
    const double dk = (uk[0] * center.x + uk[1] * center.y) + uk[2] * center.z, dl = (ul[0] * center.x + ul[1] * center.y) + ul[2] * center.z;
    for (int a = 0; a < 3; a++) fkl[6 + a] = -(dk * ul[a] + dl * uk[a]);
    const double s = nvv / (w[0] - w[k]);
    for (int a = 0; a < 3; a++) for (int c = 0; c < 9; c++) uc[a][c] += s * uk[a] * fkl[c];
  }
  double Jc[3][9];
  for (int a = 0; a < 3; a++) for (int c = 0; c < 9; c++) { double t = 0; for (int m = 0; m < 9; m++) t += uc[a][m] * C[m][c]; Jc[a][c] = t; }
  double V[6][6];
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
    double t = 0; for (int m = 0; m < 9; m++) t += Jc[a][m] * uc[b][m];
    V[a][b] = t;
    const double jn = nvv * Jc[a][6 + b];
    V[a][3 + b] = jn; V[3 + b][a] = jn;
    V[3 + a][3 + b] = nvv * nvv * C[6 + a][6 + b];
  }
  double* pl = nv.plane;
  pl[nd] = center.x; pl[cap + nd] = center.y; pl[2 * cap + nd] = center.z; pl[3 * cap + nd] = ul[0]; pl[4 * cap + nd] = ul[1]; pl[5 * cap + nd] = ul[2];
  int t = 6;
  for (int a = 0; a < 6; a++) for (int b = a; b < 6; b++) pl[size_t(t++) * cap + nd] = V[a][b];
  pl[27 * cap + nd] = (double)__double2float_rn(w[2]);      // plane.radius is a float (voxel_map.hpp:72)
}

struct MargiArgs { int win_count, mgsize, W, max_points; };
struct FactorCache { const double* sum; const double* eig; size_t Vcap; long long V; };
__global__ void __launch_bounds__(64) k_map_margi(NodeView nv, int n_nodes, MargiArgs a, const int* __restrict__ ring, const double* __restrict__ poses, double* __restrict__ swp,
                                                  FactorCache fc, int* __restrict__ status) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes) return;
  unsigned int f = nv.flags[nd];
  if ((f & F_INNER) || !(nv.flags[nv.root[nd]] & F_SLIDE)) return;
  if (!(f & F_EXIST) || nv.sw[nd] < 0) return;
  const size_t cap = nv.cap;
  double* sw = swp + size_t(nv.sw[nd]) * a.W * 10;
  cluster pw[MAP_MAX_MG];
  for (int i = 0; i < MAP_MAX_MG; i++) pw[i] = zero_cluster();
  cluster add;
  double w[3]; d3 u[3];
  const int opt = nv.opt[nd];
  if (opt >= fc.V) { atomicExch(status, 1); return; }                 // the reference printf + exit(0)s here (:1211-1215)
  if (opt >= 0) {
    add = load_node_cluster(fc.sum, fc.Vcap, opt);                    // pcr_add = vox_opt.pcr_adds[opt_state] ...  :1217-1221
    w[0] = fc.eig[opt]; w[1] = fc.eig[fc.Vcap + opt]; w[2] = fc.eig[2 * fc.Vcap + opt];
    for (int k = 0; k < 3; k++) u[k] = mk3(fc.eig[(3 + k) * fc.Vcap + opt], fc.eig[(6 + k) * fc.Vcap + opt], fc.eig[(9 + k) * fc.Vcap + opt]);
    nv.opt[nd] = -1;
    for (int i = 0; i < a.mgsize; i++) {
      const cluster c = load_slot(sw + ring[i] * 10);
      if (c.n != 0.0) cluster_transform_acc(c, load_rot(poses + 12 * i), mk3(poses[12 * i + 9], poses[12 * i + 10], poses[12 * i + 11]), pw[i]);
    }
  } else {
    add = load_node_cluster(nv.fix, cap, nd);                         // pcr_add = pcr_fix + sum over the window  :1231-1238
    for (int i = 0; i < a.win_count; i++) {
      const cluster c = load_slot(sw + ring[i] * 10);
      if (c.n == 0.0) continue;
      cluster t = zero_cluster();
      cluster_transform_acc(c, load_rot(poses + 12 * i), mk3(poses[12 * i + 9], poses[12 * i + 10], poses[12 * i + 11]), t);
      if (i < a.mgsize) pw[i] = t;
      cluster_add(add, t, 1.0);
    }
    w[0] = nv.eig[nd]; w[1] = nv.eig[cap + nd]; w[2] = nv.eig[2 * cap + nd];
    for (int k = 0; k < 3; k++) u[k] = mk3(nv.eig[(3 + k) * cap + nd], nv.eig[(6 + k) * cap + nd], nv.eig[(9 + k) * cap + nd]);
    if (f & F_PLANE) eig3_jacobi(cov_from_sum(add), w, u[0], u[1], u[2]);   // :1240-1245
  }
  // eig_value / eig_vector of the node follow the branch above
  nv.eig[nd] = w[0]; nv.eig[cap + nd] = w[1]; nv.eig[2 * cap + nd] = w[2];
  for (int k = 0; k < 3; k++) { nv.eig[(3 + k) * cap + nd] = u[k].x; nv.eig[(6 + k) * cap + nd] = u[k].y; nv.eig[(9 + k) * cap + nd] = u[k].z; }
  cluster fix = load_node_cluster(nv.fix, cap, nd);
  const bool room = fix.n < double(a.max_points);
  if (room && (f & F_PLANE)) {
    const int last = nv.last_num[nd];
    if (add.n - double(last) >= 5.0 || last <= 10) { plane_update_dev(nv, nd, add, w, u); nv.last_num[nd] = int(add.n); }   // :1249-1254
  }
  f &= ~(F_KEEPFIX | F_KILLFIX);
  if (room) {
    bool any = false;
    for (int i = 0; i < a.mgsize; i++) if (pw[i].n != 0.0) { cluster_add(fix, pw[i], 1.0); any = true; }   // pcr_fix += pcrs_world[i]; point_fix gets the slot's points  :1256-1269
    if (any) f |= F_KEEPFIX;
  } else {
    for (int i = 0; i < a.mgsize; i++) if (pw[i].n != 0.0) cluster_add(add, pw[i], -1.0);                  // :1271-1279
    f |= F_KILLFIX;
  }
  store_node_cluster(nv.fix, cap, nd, fix);
  store_node_cluster(nv.add, cap, nd, add);
  for (int i = 0; i < a.mgsize; i++) { double* d = sw + ring[i] * 10; if (d[9] != 0.0) for (int k = 0; k < 10; k++) d[k] = 0.0; }   // :1281-1286
  if (fix.n >= add.n) f &= ~F_EXIST; else f |= F_EXIST;                                                    // :1288-1291
  nv.flags[nd] = f;
}
// inner nodes: isexist = OR over the children (:1296-1303), one layer per launch, deepest first
__global__ void __launch_bounds__(128) k_map_inner_exist(NodeView nv, int n_nodes, int layer) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes) return;
  const unsigned int f = nv.flags[nd];
  if (!(f & F_INNER) || nv.layer[nd] != layer || !(nv.flags[nv.root[nd]] & F_SLIDE)) return;
  bool ex = false;
  for (int o = 0; o < 8; o++) { const int c = nv.child[size_t(o) * nv.cap + nd]; if (c >= 0 && (nv.flags[c] & F_EXIST)) ex = true; }
  nv.flags[nd] = ex ? (f | F_EXIST) : (f & ~F_EXIST);
}
// slide roots that ceased to exist leave the slide map; their trees hand their windows back (clear_slwd :1482-1500, voxelslam.cpp:1379-1388)
__global__ void __launch_bounds__(128) k_map_drop_roots(NodeView nv, int n_nodes) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes || nv.root[nd] != nd) return;
  const unsigned int f = nv.flags[nd];
  if ((f & F_SLIDE) && !(f & F_EXIST)) nv.flags[nd] = (f & ~F_SLIDE) | F_DROP;
}
__global__ void __launch_bounds__(128) k_map_clear_slwd(NodeView nv, int n_nodes, int W, double* __restrict__ swp, int* __restrict__ counters, int* __restrict__ sw_free) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes) return;
  if (!(nv.flags[nv.root[nd]] & F_DROP)) return;
  const int b = nv.sw[nd];
  if (b >= 0) {
    double* d = swp + size_t(b) * W * 10;
    for (int k = 0; k < W * 10; k++) d[k] = 0.0;
    sw_free[atomicAdd(counters + 2, 1)] = b;
    nv.sw[nd] = -1;
  }
}
__global__ void __launch_bounds__(128) k_map_clear_drop(NodeView nv, int n_nodes) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd < n_nodes && nv.root[nd] == nd) nv.flags[nd] &= ~F_DROP;
}
// points of the marginalised scan that stay re-cuttable: pv.pnt = x_buf[i].R * pv.pnt + x_buf[i].p; point_fix.push_back(pv)   (:1262-1266)
__global__ void __launch_bounds__(256) k_map_fix_flags(NodeView nv, const int* __restrict__ leaf, long long n, int max_layer, unsigned int* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = leaf[i];
  flag[i] = (l >= 0 && (nv.flags[l] & F_KEEPFIX) && nv.layer[l] < max_layer) ? 1u : 0u;
}
__global__ void __launch_bounds__(256) k_map_fix_append(const double* __restrict__ pv12, const int* __restrict__ leaf, long long n, const double* __restrict__ pose, const unsigned int* __restrict__ flag,
                                                        const unsigned int* __restrict__ pos, double* __restrict__ fix_pv, int* __restrict__ fix_leaf, long long base) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flag[i]) return;
  const double* p = pv12 + 12 * i;
  const d3 w = world_point(pose, mk3(p[0], p[1], p[2]));
  double* o = fix_pv + 12 * (base + pos[i]);
  o[0] = w.x; o[1] = w.y; o[2] = w.z;
  for (int k = 3; k < 12; k++) o[k] = p[k];
  fix_leaf[base + pos[i]] = leaf[i];
}
// leaves whose pcr_fix is full drop their point_fix (PVec().swap(point_fix), :1277-1278)
__global__ void __launch_bounds__(256) k_map_fix_kill(NodeView nv, int* __restrict__ fix_leaf, long long n, int* __restrict__ counters) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = fix_leaf[i];
  if (l >= 0 && (nv.flags[l] & F_KILLFIX)) { fix_leaf[i] = -1; atomicAdd(counters + 5, 1); }
}
__global__ void __launch_bounds__(256) k_map_fix_live(const int* __restrict__ fix_leaf, long long n, unsigned int* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = fix_leaf[i] >= 0 ? 1u : 0u;
}
__global__ void __launch_bounds__(256) k_map_fix_compact(const double* __restrict__ pv, const int* __restrict__ leaf, long long n, const unsigned int* __restrict__ flag, const unsigned int* __restrict__ pos,
                                                         double* __restrict__ pv_out, int* __restrict__ leaf_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flag[i]) return;
  for (int k = 0; k < 12; k++) pv_out[12 * size_t(pos[i]) + k] = pv[12 * i + k];
  leaf_out[pos[i]] = leaf[i];
}

// ---------------------------------------------------------------- read-back for tests / the odometry table
__global__ void __launch_bounds__(256) k_map_count_fix(const int* __restrict__ fix_leaf, long long n, int* __restrict__ cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && fix_leaf[i] >= 0) atomicAdd(cnt + fix_leaf[i], 1);
}
__global__ void __launch_bounds__(128) k_map_leaf_flags(NodeView nv, int n_nodes, unsigned int* __restrict__ flag) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd < n_nodes) flag[nd] = (nv.flags[nd] & F_INNER) ? 0u : 1u;
}
// row layout documented at vxs_map_read_leaves (include/vxs.h): 32 + 10 W doubles per leaf
__global__ void __launch_bounds__(128) k_map_leaf_rows(NodeView nv, int n_nodes, int W, const int* __restrict__ ring, const double* __restrict__ swp, const unsigned int* __restrict__ flag,
                                                       const unsigned int* __restrict__ pos, const int* __restrict__ fixcnt, double* __restrict__ rows) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes || !flag[nd]) return;
  double* r = rows + size_t(pos[nd]) * (32 + 10 * W);
  const size_t cap = nv.cap;
  const unsigned int f = nv.flags[nd];
  for (int k = 0; k < 3; k++) r[k] = nv.center[k * cap + nd];
  r[3] = double(nv.quater[nd]) * 2; r[4] = nv.layer[nd]; r[5] = (f & F_PLANE) ? 1 : 0; r[6] = (f & F_EXIST) ? 1 : 0; r[7] = nv.sw[nd] >= 0 ? 1 : 0;
  r[8] = (nv.flags[nv.root[nd]] & F_SLIDE) ? 1 : 0; r[9] = nv.opt[nd]; r[10] = nv.last_num[nd]; r[11] = fixcnt[nd];
  for (int k = 0; k < 10; k++) { r[12 + k] = nv.add[size_t(k) * cap + nd]; r[22 + k] = nv.fix[size_t(k) * cap + nd]; }
  const double* d = nv.sw[nd] >= 0 ? swp + size_t(nv.sw[nd]) * W * 10 : nullptr;
  for (int i = 0; i < W; i++) for (int k = 0; k < 10; k++) r[32 + 10 * i + k] = d ? d[ring[i] * 10 + k] : 0.0;
}
__global__ void __launch_bounds__(128) k_map_plane_flags(NodeView nv, int n_nodes, unsigned int* __restrict__ flag) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd < n_nodes) { const unsigned int f = nv.flags[nd]; flag[nd] = (!(f & F_INNER) && (f & F_PLANE) && nv.plane[27 * nv.cap + nd] > 0.0) ? 1u : 0u; }
}
// 52 doubles per plane leaf (vxs_map_read_planes): centre3 normal3 plane_var36 radius N voxel_center3 half cov-trace eig3
__global__ void __launch_bounds__(128) k_map_plane_rows(NodeView nv, int n_nodes, const unsigned int* __restrict__ flag, const unsigned int* __restrict__ pos, double* __restrict__ rows,
                                                        long long* __restrict__ ids) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes || !flag[nd]) return;
  double* r = rows + size_t(pos[nd]) * 52;
  const size_t cap = nv.cap;
  for (int k = 0; k < 6; k++) r[k] = nv.plane[size_t(k) * cap + nd];
  int t = 6;
  for (int a = 0; a < 6; a++) for (int b = a; b < 6; b++) { const double v = nv.plane[size_t(t++) * cap + nd]; r[6 + 6 * a + b] = v; r[6 + 6 * b + a] = v; }
  r[42] = nv.plane[27 * cap + nd]; r[43] = nv.add[9 * cap + nd];
  for (int k = 0; k < 3; k++) { r[44 + k] = nv.center[k * cap + nd]; r[49 + k] = nv.eig[size_t(k) * cap + nd]; }
  r[47] = double(nv.quater[nd]) * 2;
  double tr = 0; { int q = 0; for (int a = 0; a < 9; a++) for (int b = a; b < 9; b++) { if (a == b) tr += nv.cov[size_t(q) * cap + nd]; q++; } }
  r[48] = tr;
  if (ids) { const int rt = nv.root[nd]; long long* o = ids + 5 * size_t(pos[nd]); o[0] = nv.rkey[rt]; o[1] = nv.rkey[cap + rt]; o[2] = nv.rkey[2 * cap + rt]; o[3] = nv.layer[nd]; o[4] = nv.path[nd]; }
}
// rebuild of the root hash table after it grew
__global__ void __launch_bounds__(128) k_map_rehash(NodeView nv, int n_nodes, unsigned int* __restrict__ table, unsigned int tmask) {
  const int nd = blockIdx.x * blockDim.x + threadIdx.x;
  if (nd >= n_nodes || nv.root[nd] != nd) return;
  unsigned int h = table_hash(nv.rkey[nd], nv.rkey[nv.cap + nd], nv.rkey[2 * nv.cap + nd]) & tmask;
  while (atomicCAS(table + h, 0u, (unsigned int)nd + 1u) != 0u) h = (h + 1u) & tmask;
}

// ---------------------------------------------------------------- odometry association against the resident map (SURVEY.md §8f rank 3)
// match() (voxel_map.hpp:1674-1698): root cell of the world point through the root hash (surf_map holds EVERY root, also those that left the slide
// map), OctoTree::match (:1335-1392): descend by centre comparison while the node is inner (a missing child ends the search), at the leaf the
// 3-sigma gates on the plane row that plane_update left in the node — read in place, nothing is exported or re-sorted.
// kRows as k_odom_accumulate (vxs_odom.cu): atomic sums for vxs_map_odom_accumulate, partial rows + the stopped flag for vxs_map_lio_update.
template <bool kRows>
__global__ void __launch_bounds__(OD_THREADS) k_map_odom(NodeView nv, const unsigned int* __restrict__ table, unsigned int tmask, const double* __restrict__ pv, long long n,
                                                         const double* __restrict__ st /* R9 p3 rotvar9 tslvar9 */, double voxel_size, double* __restrict__ out, int* __restrict__ flags,
                                                         const int* __restrict__ stopped) {
  if (kRows && *stopped) return;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double acc[34];
#pragma unroll
  for (int k = 0; k < 34; k++) acc[k] = 0.0;
  if (i < n) {
    int hit = 0;
    const double* p = pv + 12 * i;
    const double x = p[0], y = p[1], z = p[2];
    const d3 w = world_point(st, mk3(x, y, z));
    const long long kx = quantise(w.x, voxel_size), ky = quantise(w.y, voxel_size), kz = quantise(w.z, voxel_size);
    unsigned int h = table_hash(kx, ky, kz) & tmask;
    int node = -1;
    for (;;) {
      const unsigned int v = table[h];
      if (v == 0u) break;
      const int r = int(v - 1u);
      if (nv.rkey[r] == kx && nv.rkey[nv.cap + r] == ky && nv.rkey[2 * nv.cap + r] == kz) { node = r; break; }
      h = (h + 1u) & tmask;
    }
    while (node >= 0 && (nv.flags[node] & F_INNER)) node = nv.child[size_t(octant_of(nv, node, w)) * nv.cap + node];     // leaves[leafnum] == nullptr -> no match
    if (node >= 0 && (nv.flags[node] & F_PLANE)) {
      double row[OD_ROW];
#pragma unroll
      for (int k = 0; k < OD_ROW; k++) row[k] = nv.plane[size_t(k) * nv.cap + node];
      hit = od_contribution(row, x, y, z, w.x, w.y, w.z, p, st, acc);
    }
    if (flags) flags[i] = hit;
  }
  if (kRows) od_flush_row(acc, out);
  else od_flush(acc, out);
}

// ---------------------------------------------------------------- host side
template <class T> static int grow_soa(vxs_ctx* ctx, DevBuf<T>& b, int rows, size_t oldcap, size_t newcap, int used, int fill) {
  T* np = nullptr;
  VXS_CUDA(ctx, cudaMalloc((void**)&np, size_t(rows) * newcap * sizeof(T)));
  VXS_CUDA(ctx, cudaMemsetAsync(np, fill, size_t(rows) * newcap * sizeof(T), ctx->stream));
  if (b.p && used > 0) VXS_CUDA(ctx, cudaMemcpy2DAsync(np, newcap * sizeof(T), b.p, oldcap * sizeof(T), size_t(used) * sizeof(T), size_t(rows), cudaMemcpyDeviceToDevice, ctx->stream));
  if (b.p) { VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); cudaFree(b.p); }
  b.p = np; b.cap = size_t(rows) * newcap;
  return VXS_OK;
}
static int map_reserve_nodes(vxs_map* m, size_t need) {
  vxs_ctx* ctx = m->ctx;
  if (need > m->ncap) {
    size_t nc = std::max<size_t>(m->ncap * 2, 1 << 16);
    while (nc < need) nc *= 2;
    const size_t oc = m->ncap; const int u = m->n_nodes;
    int rc;
    if ((rc = grow_soa(ctx, m->n_root, 1, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_child, 8, oc, nc, u, 0xFF)) || (rc = grow_soa(ctx, m->n_flags, 1, oc, nc, u, 0)) ||
        (rc = grow_soa(ctx, m->n_layer, 1, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_path, 1, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_sw, 1, oc, nc, u, 0xFF)) ||
        (rc = grow_soa(ctx, m->n_opt, 1, oc, nc, u, 0xFF)) || (rc = grow_soa(ctx, m->n_last, 1, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_rkey, 3, oc, nc, u, 0)) ||
        (rc = grow_soa(ctx, m->n_center, 3, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_quater, 1, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_add, 10, oc, nc, u, 0)) ||
        (rc = grow_soa(ctx, m->n_fix, 10, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_cov, 45, oc, nc, u, 0)) || (rc = grow_soa(ctx, m->n_eig, 12, oc, nc, u, 0)) ||
        (rc = grow_soa(ctx, m->n_plane, PLANE_ROW, oc, nc, u, 0)))
      return rc;
    m->ncap = nc;
  }
  // root hash table: at least 2 slots per possible node
  if (m->tcap < 2 * m->ncap) {
    size_t tc = 1; while (tc < 2 * m->ncap) tc *= 2;
    if (m->table.p) { cudaStreamSynchronize(ctx->stream); cudaFree(m->table.p); m->table.p = nullptr; m->table.cap = 0; }
    VXS_CUDA(ctx, m->table.reserve(tc));
    VXS_CUDA(ctx, cudaMemsetAsync(m->table.p, 0, tc * 4, ctx->stream));
    m->tcap = tc;
    if (m->n_nodes > 0) VXS_LAUNCH(ctx, "k_map_rehash", k_map_rehash, nblk(size_t(m->n_nodes), 128), 128, 0, view(m), m->n_nodes, m->table.p, (unsigned int)(tc - 1));
  }
  return VXS_OK;
}
static int map_reserve_sw(vxs_map* m, size_t need_blocks) {
  vxs_ctx* ctx = m->ctx;
  if (need_blocks <= m->swcap) return VXS_OK;
  size_t nc = std::max<size_t>(m->swcap * 2, 1 << 12);
  while (nc < need_blocks) nc *= 2;
  double* np = nullptr; int* nf = nullptr;
  const size_t bd = size_t(m->W) * 10;
  VXS_CUDA(ctx, cudaMalloc((void**)&np, nc * bd * 8));
  VXS_CUDA(ctx, cudaMemsetAsync(np, 0, nc * bd * 8, ctx->stream));
  VXS_CUDA(ctx, cudaMalloc((void**)&nf, nc * 4));
  if (m->swp.p) {
    VXS_CUDA(ctx, cudaMemcpyAsync(np, m->swp.p, m->swcap * bd * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    VXS_CUDA(ctx, cudaMemcpyAsync(nf, m->sw_free.p, m->swcap * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(m->swp.p); cudaFree(m->sw_free.p);
  }
  m->swp.p = np; m->swp.cap = nc * bd; m->sw_free.p = nf; m->sw_free.cap = nc; m->swcap = nc;
  return VXS_OK;
}
static int read_counters(vxs_map* m, int* out8) {
  vxs_ctx* ctx = m->ctx;
  VXS_CUDA(ctx, cudaMemcpyAsync(out8, m->counters.p, 8 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return VXS_OK;
}
// device copies of ring / inverse ring / poses / per-slot pointers for a window of `wc` scans
static int upload_window(vxs_map* m, const double* poses12, int wc) {
  vxs_ctx* ctx = m->ctx;
  const int W = m->W;
  std::vector<int> rg(size_t(2 * W + 1));
  for (int i = 0; i < W; i++) { rg[size_t(i)] = m->ring[size_t(i)]; rg[size_t(W + m->ring[size_t(i)])] = i; }
  rg[size_t(2 * W)] = W;
  std::vector<double> ps(size_t(W + 1) * 12, 0.0);
  memcpy(ps.data(), poses12, size_t(wc) * 96);
  const double ident[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
  memcpy(ps.data() + size_t(W) * 12, ident, 96);
  std::vector<unsigned long long> ptrs(size_t(2 * (W + 1)));
  for (int s = 0; s < W; s++) { ptrs[size_t(s)] = (unsigned long long)(uintptr_t)m->scan_pv[size_t(s)]->p; ptrs[size_t(W + 1 + s)] = (unsigned long long)(uintptr_t)m->scan_leaf[size_t(s)]->p; }
  ptrs[size_t(W)] = (unsigned long long)(uintptr_t)m->fix_pv.p; ptrs[size_t(2 * W + 1)] = (unsigned long long)(uintptr_t)m->fix_leaf.p;
  VXS_CUDA(ctx, cudaMemcpyAsync(m->d_ring.p, rg.data(), rg.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaMemcpyAsync(m->d_poses.p, ps.data(), ps.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaMemcpyAsync(m->scan_ptrs.p, ptrs.data(), ptrs.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));     // the host vectors go out of scope
  return VXS_OK;
}
static PointSrcs point_srcs(vxs_map* m) { PointSrcs s; s.ptrs = m->scan_ptrs.p; s.inv_ring = m->d_ring.p + m->W; s.poses = m->d_poses.p; s.W = m->W; return s; }

// sort `cnt` (key, idx) pairs, cut them into (node, slot) records and node heads, give windows to the nodes that need one, accumulate
static int accumulate_sorted(vxs_map* m, size_t cnt, int key_bits) {
  vxs_ctx* ctx = m->ctx;
  if (cnt == 0) return VXS_OK;
  cudaStream_t st = ctx->stream;
  unsigned long long* ks; unsigned int* vs;
  int rc = radix_sort(ctx, &m->ss, m->keysA.p, m->idxA.p, m->keysB.p, m->idxB.p, cnt, key_bits, &ks, &vs);
  if (rc) return rc;
  VXS_CUDA(ctx, m->flagbuf.reserve(cnt)); VXS_CUDA(ctx, m->scanbuf.reserve(cnt));
  VXS_LAUNCH(ctx, "k_flag_heads", k_flag_heads, nblk(cnt, 256), 256, 0, ks, cnt, m->flagbuf.p);
  rc = scan_u32(ctx, &m->ss, m->flagbuf.p, m->scanbuf.p, cnt, m->ss.totals.p + 0);
  if (rc) return rc;
  unsigned int R = 0;
  VXS_CUDA(ctx, cudaMemcpyAsync(&R, m->ss.totals.p + 0, 4, cudaMemcpyDeviceToHost, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  VXS_CUDA(ctx, m->rec_start.reserve(size_t(R) + 1)); VXS_CUDA(ctx, m->rec_key.reserve(size_t(R)));
  VXS_CUDA(ctx, m->node_of_rec.reserve(size_t(R))); VXS_CUDA(ctx, m->nflag.reserve(size_t(R) * 2)); VXS_CUDA(ctx, m->node_rec_start.reserve(size_t(R) + 1));
  VXS_LAUNCH(ctx, "k_write_records", k_write_records, nblk(cnt, 256), 256, 0, ks, m->flagbuf.p, m->scanbuf.p, cnt, m->rec_start.p, m->rec_key.p, m->ss.totals.p + 0);
  unsigned int* nflag = m->nflag.p; unsigned int* nex = m->nflag.p + R;
  VXS_LAUNCH(ctx, "k_flag_nodes", k_flag_nodes, nblk(R, 256), 256, 0, m->rec_key.p, size_t(R), 8, nflag);
  rc = scan_u32(ctx, &m->ss, nflag, nex, R, m->ss.totals.p + 1);
  if (rc) return rc;
  unsigned int Nn = 0;
  VXS_CUDA(ctx, cudaMemcpyAsync(&Nn, m->ss.totals.p + 1, 4, cudaMemcpyDeviceToHost, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  VXS_LAUNCH(ctx, "k_write_nodes", k_write_nodes, nblk(R, 256), 256, 0, nflag, nex, size_t(R), m->node_of_rec.p, m->node_rec_start.p, m->ss.totals.p + 1);
  rc = map_reserve_sw(m, size_t(m->sw_bump) + Nn);
  if (rc) return rc;
  VXS_LAUNCH(ctx, "k_map_alloc_sw", k_map_alloc_sw, nblk(Nn, 128), 128, 0, view(m), m->node_rec_start.p, m->rec_key.p, Nn, m->W, m->counters.p, m->sw_free.p);
  const double avg = double(cnt) / double(std::max(Nn, 1u));
  const unsigned grid = std::min<unsigned>(nblk(size_t(Nn) * 8, 128), unsigned(ctx->sm_count) * 16);
  if (avg > 24.0) { auto kp = k_map_accum<32>; VXS_LAUNCH(ctx, "k_map_accum", kp, std::min<unsigned>(nblk(size_t(Nn) * 32, 128), unsigned(ctx->sm_count) * 16), 128, 0, view(m), point_srcs(m), vs, m->refs.p, m->rec_start.p, m->rec_key.p, m->node_rec_start.p, Nn, m->swp.p, 1); }
  else if (avg > 3.0) { auto kp = k_map_accum<8>; VXS_LAUNCH(ctx, "k_map_accum", kp, grid, 128, 0, view(m), point_srcs(m), vs, m->refs.p, m->rec_start.p, m->rec_key.p, m->node_rec_start.p, Nn, m->swp.p, 1); }
  else { auto kp = k_map_accum<1>; VXS_LAUNCH(ctx, "k_map_accum", kp, std::min<unsigned>(nblk(size_t(Nn), 128), unsigned(ctx->sm_count) * 16), 128, 0, view(m), point_srcs(m), vs, m->refs.p, m->rec_start.p, m->rec_key.p, m->node_rec_start.p, Nn, m->swp.p, 1); }
  int c8[8];
  rc = read_counters(m, c8);
  if (rc) return rc;
  m->n_nodes = c8[0]; m->sw_bump = c8[1];
  return VXS_OK;
}

static int map_recut(vxs_map* m, int wc) {
  vxs_ctx* ctx = m->ctx;
  const int W = m->W;
  for (int layer = 0; layer <= m->mp.max_layer; layer++) {
    DecideArgs a; a.min_eigen_value = m->mp.min_eigen_value; a.thre = m->mp.plane_thre[std::min(layer, 3)]; a.min_point = m->mp.min_point[std::min(layer, 3)];
    a.layer = layer; a.max_layer = m->mp.max_layer;
    VXS_CUDA(ctx, cudaMemsetAsync(m->counters.p + 3, 0, 4, ctx->stream));
    VXS_LAUNCH(ctx, "k_map_decide", k_map_decide, nblk(size_t(m->n_nodes), 128), 128, 0, view(m), m->n_nodes, a, m->counters.p);
    if (layer == m->mp.max_layer) break;
    int c8[8];
    int rc = read_counters(m, c8);
    if (rc) return rc;
    if (c8[3] == 0) continue;
    // ---- subdivide the marked leaves
    std::vector<long long> off(size_t(wc) + 2, 0);
    for (int i = 0; i < wc; i++) off[size_t(i) + 1] = off[size_t(i)] + m->scan_n[size_t(m->ring[size_t(i)])];
    off[size_t(wc) + 1] = off[size_t(wc)] + m->fix_n;
    const long long total = off[size_t(wc) + 1];
    if (total == 0) continue;
    if (total >= (1ll << 32)) return vxs_fail(ctx, VXS_ERR_ARG, "more than 2^32 resident points");
    VXS_CUDA(ctx, m->d_off.reserve(size_t(W) + 3));
    VXS_CUDA(ctx, cudaMemcpyAsync(m->d_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    VirtPts vp; vp.off = m->d_off.p; vp.nseg = wc + 1;
    VXS_CUDA(ctx, m->flagbuf.reserve(size_t(total))); VXS_CUDA(ctx, m->scanbuf.reserve(size_t(total)));
    const unsigned long long* leaf_ptrs = m->scan_ptrs.p + (W + 1);
    VXS_LAUNCH(ctx, "k_map_flag_marked", k_map_flag_marked, nblk(size_t(total), 256), 256, 0, view(m), vp, leaf_ptrs, m->d_ring.p, wc, W, total, m->flagbuf.p);
    rc = scan_u32(ctx, &m->ss, m->flagbuf.p, m->scanbuf.p, size_t(total), m->ss.totals.p + 2);
    if (rc) return rc;
    unsigned int na = 0;
    VXS_CUDA(ctx, cudaMemcpyAsync(&na, m->ss.totals.p + 2, 4, cudaMemcpyDeviceToHost, ctx->stream));
    VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (na > 0) {
      rc = map_reserve_nodes(m, size_t(m->n_nodes) + na);
      if (rc) return rc;
      VXS_CUDA(ctx, m->keysA.reserve(na)); VXS_CUDA(ctx, m->keysB.reserve(na)); VXS_CUDA(ctx, m->idxA.reserve(na)); VXS_CUDA(ctx, m->idxB.reserve(na)); VXS_CUDA(ctx, m->refs.reserve(na));
      // the flag / scan buffers are reused by accumulate_sorted: keep the compaction positions in idxB until the assignment ran
      int c2[8];
      for (int pass = 0;; pass++) {
        VXS_CUDA(ctx, cudaMemsetAsync(m->counters.p + 7, 0, 4, ctx->stream));
        VXS_LAUNCH(ctx, "k_map_subdiv_assign", k_map_subdiv_assign, nblk(size_t(total), 256), 256, 0, view(m), vp, point_srcs(m), leaf_ptrs, m->d_ring.p, wc, total, m->flagbuf.p, m->scanbuf.p,
                   m->counters.p, int(m->mp.max_layer), m->keysA.p, m->idxA.p, m->refs.p, pass);
        if (pass == 0) continue;
        rc = read_counters(m, c2);
        if (rc) return rc;
        if (c2[7] == 0) break;
        if (pass > 64) return vxs_fail(ctx, VXS_ERR_CUDA, "vxs_map_push_scan: child creation did not settle");
      }
      m->n_nodes = c2[0];
      rc = accumulate_sorted(m, na, bits_for((unsigned long long)m->n_nodes) + 8);
      if (rc) return rc;
    }
    VXS_LAUNCH(ctx, "k_map_finish_subdiv", k_map_finish_subdiv, nblk(size_t(m->n_nodes), 128), 128, 0, view(m), m->n_nodes, W, m->swp.p, m->counters.p, m->sw_free.p);
  }
  return VXS_OK;
}

static int map_emit_factor(vxs_map* m, vxs_factor* out) {
  vxs_ctx* ctx = m->ctx;
  const int W = m->W;
  vxs_factor_clear(out);
  out->W = W;
  const size_t nn = size_t(m->n_nodes);
  if (nn == 0) return VXS_OK;
  VXS_CUDA(ctx, m->sel.reserve(nn)); VXS_CUDA(ctx, m->nent.reserve(nn)); VXS_CUDA(ctx, m->voff.reserve(nn)); VXS_CUDA(ctx, m->eoff.reserve(nn));
  VXS_LAUNCH(ctx, "k_map_select", k_map_select, nblk(nn, 128), 128, 0, view(m), m->n_nodes, W, m->d_ring.p, m->swp.p, m->sel.p, m->nent.p);
  int rc = scan_u32(ctx, &m->ss, m->sel.p, m->voff.p, nn, m->ss.totals.p + 4);
  if (rc) return rc;
  rc = scan_u32(ctx, &m->ss, m->nent.p, m->eoff.p, nn, m->ss.totals.p + 5);
  if (rc) return rc;
  unsigned int tot[2] = {0, 0};
  VXS_CUDA(ctx, cudaMemcpyAsync(tot, m->ss.totals.p + 4, 8, cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (tot[0] == 0) return VXS_OK;
  rc = vxs_factor_reserve(out, tot[0], tot[1]);
  if (rc) return rc;
  FactorOut fo; fo.ptr = out->ptr; fo.frame = out->frame; fo.vox = out->vox; fo.cl = out->cl; fo.Ecap = out->Ecap; fo.fix = out->fix; fo.coe = out->coe; fo.eig = out->eig; fo.sum = out->sum; fo.Vcap = out->Vcap;
  VXS_LAUNCH(ctx, "k_map_emit", k_map_emit, nblk(nn, 128), 128, 0, view(m), m->n_nodes, W, m->d_ring.p, m->swp.p, m->sel.p, m->voff.p, m->eoff.p, fo);
  VXS_LAUNCH(ctx, "k_map_last_ptr", k_map_last_ptr, 1, 1, 0, out->ptr, m->ss.totals.p + 4);
  out->V = tot[0]; out->E = tot[1]; out->has_fix = true;
  return VXS_OK;
}

}  // namespace

// ================================================================ C ABI
extern "C" int vxs_map_create(vxs_ctx* ctx, const vxs_map_params* mp, int win_size, int max_points, vxs_map** out) {
  if (!ctx || !mp || !out || win_size < 1 || win_size > 250 || mp->max_layer < 0 || mp->max_layer > 3 || !(mp->voxel_size > 0)) return VXS_ERR_ARG;
  cudaSetDevice(ctx->device);
  vxs_map* m = new vxs_map();
  m->ctx = ctx; m->mp = *mp; m->W = win_size; m->max_points = max_points > 0 ? max_points : 100;
  m->ring.resize(size_t(win_size));
  for (int i = 0; i < win_size; i++) m->ring[size_t(i)] = i;
  for (int s = 0; s < win_size; s++) { m->scan_pv.push_back(new DevBuf<double>()); m->scan_leaf.push_back(new DevBuf<int>()); m->scan_n.push_back(0); }
  int rc = VXS_OK;
  do {
    if (m->counters.reserve(8) != cudaSuccess || m->d_ring.reserve(size_t(2 * win_size + 1)) != cudaSuccess || m->d_poses.reserve(size_t(win_size + 1) * 12) != cudaSuccess ||
        m->scan_ptrs.reserve(size_t(2 * (win_size + 1))) != cudaSuccess || m->ss.totals.reserve(16) != cudaSuccess) { rc = VXS_ERR_NOMEM; break; }
    cudaMemsetAsync(m->counters.p, 0, 32, ctx->stream);
    rc = map_reserve_nodes(m, 1 << 16);
    if (rc) break;
    rc = map_reserve_sw(m, 1 << 12);
  } while (0);
  if (rc) { delete m; return rc; }
  *out = m;
  return VXS_OK;
}
extern "C" int vxs_map_destroy(vxs_map* m) {
  if (!m) return VXS_OK;
  if (m->ctx) { cudaSetDevice(m->ctx->device); cudaStreamSynchronize(m->ctx->stream); }
  for (auto b : m->scan_pv) { b->release(); delete b; }
  for (auto b : m->scan_leaf) { b->release(); delete b; }
  m->n_root.release(); m->n_child.release(); m->n_layer.release(); m->n_path.release(); m->n_sw.release(); m->n_opt.release(); m->n_last.release(); m->n_flags.release(); m->n_rkey.release();
  m->n_center.release(); m->n_add.release(); m->n_fix.release(); m->n_cov.release(); m->n_eig.release(); m->n_plane.release(); m->n_quater.release(); m->table.release(); m->counters.release();
  m->swp.release(); m->sw_free.release(); m->scan_ptrs.release(); m->fix_pv.release(); m->fix_leaf.release(); m->fix_pv2.release(); m->fix_leaf2.release(); m->d_ring.release(); m->d_poses.release(); m->d_off.release();
  m->ss.hist.release(); m->ss.blocksums.release(); m->ss.totals.release(); m->keysA.release(); m->keysB.release(); m->refs.release(); m->rec_key.release(); m->idxA.release(); m->idxB.release();
  m->flagbuf.release(); m->scanbuf.release(); m->rec_start.release(); m->node_of_rec.release(); m->node_rec_start.release(); m->nflag.release(); m->sel.release(); m->nent.release();
  m->voff.release(); m->eoff.release(); m->odom_st.release();
  delete m;
  return VXS_OK;
}

extern "C" int vxs_map_push_scan(vxs_map* m, const double* pv12, int64_t n, const double* poses12, int win_count, vxs_factor* out) {
  if (!m || !poses12 || n < 0 || win_count < 1 || win_count > m->W || (out && out->ctx != m->ctx)) return VXS_ERR_ARG;
  if (win_count != m->win_count + 1) return vxs_fail(m->ctx, VXS_ERR_ARG, "vxs_map_push_scan: win_count must be the number of resident scans + 1 (call vxs_map_margi when the window is full)");
  if (n >= (1ll << 31)) return vxs_fail(m->ctx, VXS_ERR_ARG, "more than 2^31 points in one scan");
  vxs_ctx* ctx = m->ctx;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int W = m->W, slot = m->ring[size_t(win_count - 1)];
  // ---- the new scan becomes resident in its ring slot
  DevBuf<double>& pv = *m->scan_pv[size_t(slot)]; DevBuf<int>& lf = *m->scan_leaf[size_t(slot)];
  VXS_CUDA(ctx, pv.reserve(size_t(std::max<int64_t>(n, 1)) * 12)); VXS_CUDA(ctx, lf.reserve(size_t(std::max<int64_t>(n, 1))));
  if (n && pv12) VXS_CUDA(ctx, cudaMemcpyAsync(pv.p, pv12, size_t(n) * 96, cudaMemcpyHostToDevice, st));
  else if (n) {   // pv12 == NULL: the scan that vxs_var_init / vxs_pvec_update left on the device (no host round trip)
    double* res = nullptr; long long nres = 0;
    vxs_odom_resident_scan(ctx, &res, &nres);
    if (nres != n || !res) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_map_push_scan: pv12 is NULL and there is no resident scan of this size (vxs_var_init / vxs_pvec_update)");
    VXS_CUDA(ctx, cudaMemcpyAsync(pv.p, res, size_t(n) * 96, cudaMemcpyDeviceToDevice, st));
  }
  m->scan_n[size_t(slot)] = n;
  m->win_count = win_count;
  int rc = map_reserve_nodes(m, size_t(m->n_nodes) + size_t(n));
  if (rc) return rc;
  rc = upload_window(m, poses12, win_count);
  if (rc) return rc;
  if (n) {
    // ---- cut_voxel: leaf of every point (two passes: the second one serves the points that met a node being created)
    const unsigned int tmask = (unsigned int)(m->tcap - 1);
    // a point that meets a node being created by another thread is served by a later pass; a later pass can create nodes itself (a root whose
    // hash slot was claimed for ANOTHER root in the pass before), so the passes repeat until no point is left over (2-3 in practice)
    int c8[8];
    for (int pass = 0;; pass++) {
      VXS_CUDA(ctx, cudaMemsetAsync(m->counters.p + 7, 0, 4, st));
      VXS_LAUNCH(ctx, "k_map_locate", k_map_locate, nblk(size_t(n), 256), 256, 0, view(m), m->table.p, tmask, m->counters.p, pv.p, (long long)n, m->d_poses.p + size_t(win_count - 1) * 12,
                 m->mp.voxel_size, lf.p, pass);
      if (pass == 0) continue;
      rc = read_counters(m, c8);
      if (rc) return rc;
      if (c8[7] == 0) break;
      if (pass > 64) return vxs_fail(ctx, VXS_ERR_CUDA, "vxs_map_push_scan: node creation did not settle");
    }
    m->n_nodes = c8[0];
    // ---- push: accumulate the scan into its leaves
    VXS_CUDA(ctx, m->keysA.reserve(size_t(n))); VXS_CUDA(ctx, m->keysB.reserve(size_t(n))); VXS_CUDA(ctx, m->idxA.reserve(size_t(n))); VXS_CUDA(ctx, m->idxB.reserve(size_t(n)));
    VXS_CUDA(ctx, m->refs.reserve(size_t(n)));
    VXS_LAUNCH(ctx, "k_map_scan_keys", k_map_scan_keys, nblk(size_t(n), 256), 256, 0, lf.p, (long long)n, slot, m->keysA.p, m->idxA.p, m->refs.p);
    rc = accumulate_sorted(m, size_t(n), bits_for((unsigned long long)m->n_nodes) + 8);
    if (rc) return rc;
  }
  // ---- multi_recut on the slide trees, then tras_opt
  rc = map_recut(m, win_count);
  if (rc) return rc;
  if (out) { rc = map_emit_factor(m, out); if (rc) return rc; }
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  return VXS_OK;
}

extern "C" int vxs_map_margi(vxs_map* m, const double* poses12, int win_count, int mgsize, vxs_factor* f) {
  if (!m || !poses12 || !f || f->ctx != m->ctx || win_count != m->win_count || mgsize < 1 || mgsize > MAP_MAX_MG || mgsize > win_count) return VXS_ERR_ARG;
  vxs_ctx* ctx = m->ctx;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int W = m->W;
  int rc = upload_window(m, poses12, win_count);
  if (rc) return rc;
  { int rcw = vxs_factor_wait_uploads(f); if (rcw) return rcw; }
  MargiArgs a; a.win_count = win_count; a.mgsize = mgsize; a.W = W; a.max_points = m->max_points;
  FactorCache fc; fc.sum = f->sum; fc.eig = f->eig; fc.Vcap = f->Vcap; fc.V = f->V;
  VXS_CUDA(ctx, cudaMemsetAsync(m->counters.p + 5, 0, 12, st));
  VXS_LAUNCH(ctx, "k_map_margi", k_map_margi, nblk(size_t(m->n_nodes), 64), 64, 0, view(m), m->n_nodes, a, m->d_ring.p, m->d_poses.p, m->swp.p, fc, m->counters.p + 6);
  // ---- point_fix: drop those of the full leaves, append the marginalised scans' points of the others
  if (m->fix_n) VXS_LAUNCH(ctx, "k_map_fix_kill", k_map_fix_kill, nblk(size_t(m->fix_n), 256), 256, 0, view(m), m->fix_leaf.p, m->fix_n, m->counters.p);
  for (int i = 0; i < mgsize; i++) {
    const int slot = m->ring[size_t(i)];
    const long long n = m->scan_n[size_t(slot)];
    if (n == 0) continue;
    VXS_CUDA(ctx, m->flagbuf.reserve(size_t(n))); VXS_CUDA(ctx, m->scanbuf.reserve(size_t(n)));
    VXS_LAUNCH(ctx, "k_map_fix_flags", k_map_fix_flags, nblk(size_t(n), 256), 256, 0, view(m), m->scan_leaf[size_t(slot)]->p, n, int(m->mp.max_layer), m->flagbuf.p);
    rc = scan_u32(ctx, &m->ss, m->flagbuf.p, m->scanbuf.p, size_t(n), m->ss.totals.p + 6);
    if (rc) return rc;
    unsigned int add = 0;
    VXS_CUDA(ctx, cudaMemcpyAsync(&add, m->ss.totals.p + 6, 4, cudaMemcpyDeviceToHost, st));
    VXS_CUDA(ctx, cudaStreamSynchronize(st));
    if (add) {
      if (size_t(m->fix_n + add) > m->fix_leaf.cap) {      // grow the pool, keeping its contents
        const size_t nc = std::max<size_t>(size_t(m->fix_n + add) * 2, 1 << 16);
        double* np = nullptr; int* nl = nullptr;
        VXS_CUDA(ctx, cudaMalloc((void**)&np, nc * 96)); VXS_CUDA(ctx, cudaMalloc((void**)&nl, nc * 4));
        if (m->fix_n) { VXS_CUDA(ctx, cudaMemcpyAsync(np, m->fix_pv.p, size_t(m->fix_n) * 96, cudaMemcpyDeviceToDevice, st)); VXS_CUDA(ctx, cudaMemcpyAsync(nl, m->fix_leaf.p, size_t(m->fix_n) * 4, cudaMemcpyDeviceToDevice, st)); }
        VXS_CUDA(ctx, cudaStreamSynchronize(st));
        if (m->fix_pv.p) cudaFree(m->fix_pv.p);
        if (m->fix_leaf.p) cudaFree(m->fix_leaf.p);
        m->fix_pv.p = np; m->fix_pv.cap = nc * 12; m->fix_leaf.p = nl; m->fix_leaf.cap = nc;
      }
      VXS_LAUNCH(ctx, "k_map_fix_append", k_map_fix_append, nblk(size_t(n), 256), 256, 0, m->scan_pv[size_t(slot)]->p, m->scan_leaf[size_t(slot)]->p, n, m->d_poses.p + size_t(i) * 12, m->flagbuf.p,
                 m->scanbuf.p, m->fix_pv.p, m->fix_leaf.p, m->fix_n);
      m->fix_n += add;
    }
    m->scan_n[size_t(slot)] = 0;       // sw->points[mp[i]].clear()
  }
  // ---- isexist of the inner nodes, slide erase, clear_slwd
  for (int layer = m->mp.max_layer - 1; layer >= 0; layer--) VXS_LAUNCH(ctx, "k_map_inner_exist", k_map_inner_exist, nblk(size_t(m->n_nodes), 128), 128, 0, view(m), m->n_nodes, layer);
  VXS_LAUNCH(ctx, "k_map_drop_roots", k_map_drop_roots, nblk(size_t(m->n_nodes), 128), 128, 0, view(m), m->n_nodes);
  VXS_LAUNCH(ctx, "k_map_clear_slwd", k_map_clear_slwd, nblk(size_t(m->n_nodes), 128), 128, 0, view(m), m->n_nodes, W, m->swp.p, m->counters.p, m->sw_free.p);
  VXS_LAUNCH(ctx, "k_map_clear_drop", k_map_clear_drop, nblk(size_t(m->n_nodes), 128), 128, 0, view(m), m->n_nodes);
  int c8[8];
  rc = read_counters(m, c8);
  if (rc) return rc;
  if (c8[6] != 0) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_map_margi: a leaf's opt_state points beyond the factor (the factor is not the one vxs_map_push_scan filled; voxel_map.hpp:1211-1215)");
  m->fix_dead += c8[5];
  // ---- compact the point_fix pool when most of it is dead
  if (m->fix_n > (1 << 16) && m->fix_dead * 2 > m->fix_n) {
    const size_t n = size_t(m->fix_n);
    VXS_CUDA(ctx, m->flagbuf.reserve(n)); VXS_CUDA(ctx, m->scanbuf.reserve(n));
    VXS_LAUNCH(ctx, "k_map_fix_live", k_map_fix_live, nblk(n, 256), 256, 0, m->fix_leaf.p, m->fix_n, m->flagbuf.p);
    rc = scan_u32(ctx, &m->ss, m->flagbuf.p, m->scanbuf.p, n, m->ss.totals.p + 7);
    if (rc) return rc;
    unsigned int live = 0;
    VXS_CUDA(ctx, cudaMemcpyAsync(&live, m->ss.totals.p + 7, 4, cudaMemcpyDeviceToHost, st));
    VXS_CUDA(ctx, cudaStreamSynchronize(st));
    // compact into the spare pool (same capacity as the live one, allocated once and kept) and swap: no cudaMalloc / cudaFree per compaction —
    // a 400 MB cudaFree + cudaMalloc pair every other scan cost ~80 ms of host time in the first version
    if (m->fix_pv2.cap < m->fix_pv.cap || m->fix_leaf2.cap < m->fix_leaf.cap) {
      m->fix_pv2.release(); m->fix_leaf2.release();
      VXS_CUDA(ctx, m->fix_pv2.reserve(m->fix_pv.cap)); VXS_CUDA(ctx, m->fix_leaf2.reserve(m->fix_leaf.cap));
    }
    VXS_LAUNCH(ctx, "k_map_fix_compact", k_map_fix_compact, nblk(n, 256), 256, 0, m->fix_pv.p, m->fix_leaf.p, m->fix_n, m->flagbuf.p, m->scanbuf.p, m->fix_pv2.p, m->fix_leaf2.p);
    std::swap(m->fix_pv.p, m->fix_pv2.p); std::swap(m->fix_pv.cap, m->fix_pv2.cap);
    std::swap(m->fix_leaf.p, m->fix_leaf2.p); std::swap(m->fix_leaf.cap, m->fix_leaf2.cap);
    m->fix_n = live; m->fix_dead = 0;
  }
  // ---- ring rotation (voxelslam.cpp:1689-1693); the caller shifts its pose buffer (:1695-1712)
  for (int i = 0; i < W; i++) { m->ring[size_t(i)] += mgsize; if (m->ring[size_t(i)] >= W) m->ring[size_t(i)] -= W; }
  m->win_count = win_count - mgsize;
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  return VXS_OK;
}

extern "C" int vxs_map_counts(const vxs_map* m, int64_t* n_nodes, int64_t* n_fix_points, int* win_count, int32_t* ring) {
  if (!m) return VXS_ERR_ARG;
  if (n_nodes) *n_nodes = m->n_nodes;
  if (n_fix_points) *n_fix_points = m->fix_n;
  if (win_count) *win_count = m->win_count;
  if (ring) for (int i = 0; i < m->W; i++) ring[i] = m->ring[size_t(i)];
  return VXS_OK;
}

// every leaf of the map in the row layout of the oracle's sliding-window simulator (32 + 10 W doubles); *n_out = number of leaves
extern "C" int vxs_map_read_leaves(vxs_map* m, double* rows, int64_t cap, int64_t* n_out) {
  if (!m || !n_out) return VXS_ERR_ARG;
  vxs_ctx* ctx = m->ctx;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  *n_out = 0;
  const size_t nn = size_t(m->n_nodes);
  if (nn == 0) return VXS_OK;
  const int W = m->W;
  std::vector<int> rg(size_t(2 * W + 1));
  for (int i = 0; i < W; i++) { rg[size_t(i)] = m->ring[size_t(i)]; rg[size_t(W + m->ring[size_t(i)])] = i; }
  rg[size_t(2 * W)] = W;
  VXS_CUDA(ctx, cudaMemcpyAsync(m->d_ring.p, rg.data(), rg.size() * 4, cudaMemcpyHostToDevice, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  VXS_CUDA(ctx, m->sel.reserve(nn)); VXS_CUDA(ctx, m->voff.reserve(nn)); VXS_CUDA(ctx, m->nent.reserve(nn));
  VXS_LAUNCH(ctx, "k_map_leaf_flags", k_map_leaf_flags, nblk(nn, 128), 128, 0, view(m), m->n_nodes, m->sel.p);
  int rc = scan_u32(ctx, &m->ss, m->sel.p, m->voff.p, nn, m->ss.totals.p + 8);
  if (rc) return rc;
  unsigned int nl = 0;
  VXS_CUDA(ctx, cudaMemcpyAsync(&nl, m->ss.totals.p + 8, 4, cudaMemcpyDeviceToHost, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  *n_out = nl;
  if (!rows || cap < int64_t(nl)) return VXS_OK;
  int* fixcnt = reinterpret_cast<int*>(m->nent.p);
  VXS_CUDA(ctx, cudaMemsetAsync(fixcnt, 0, nn * 4, st));
  if (m->fix_n) VXS_LAUNCH(ctx, "k_map_count_fix", k_map_count_fix, nblk(size_t(m->fix_n), 256), 256, 0, m->fix_leaf.p, m->fix_n, fixcnt);
  const size_t rw = size_t(32 + 10 * W);
  VXS_CUDA(ctx, ctx->stage.reserve(size_t(nl) * rw));
  VXS_LAUNCH(ctx, "k_map_leaf_rows", k_map_leaf_rows, nblk(nn, 128), 128, 0, view(m), m->n_nodes, W, m->d_ring.p, m->swp.p, m->sel.p, m->voff.p, fixcnt, ctx->stage.p);
  VXS_CUDA(ctx, cudaMemcpyAsync(rows, ctx->stage.p, size_t(nl) * rw * 8, cudaMemcpyDeviceToHost, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  return VXS_OK;
}

// plane leaves (is_plane, radius > 0): 52 doubles per plane (see k_map_plane_rows) + identity (root x, y, z, layer, path)
extern "C" int vxs_map_read_planes(vxs_map* m, double* rows52, int64_t* ids5, int64_t cap, int64_t* n_out) {
  if (!m || !n_out) return VXS_ERR_ARG;
  vxs_ctx* ctx = m->ctx;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  *n_out = 0;
  const size_t nn = size_t(m->n_nodes);
  if (nn == 0) return VXS_OK;
  VXS_CUDA(ctx, m->sel.reserve(nn)); VXS_CUDA(ctx, m->voff.reserve(nn));
  VXS_LAUNCH(ctx, "k_map_plane_flags", k_map_plane_flags, nblk(nn, 128), 128, 0, view(m), m->n_nodes, m->sel.p);
  int rc = scan_u32(ctx, &m->ss, m->sel.p, m->voff.p, nn, m->ss.totals.p + 9);
  if (rc) return rc;
  unsigned int np = 0;
  VXS_CUDA(ctx, cudaMemcpyAsync(&np, m->ss.totals.p + 9, 4, cudaMemcpyDeviceToHost, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  *n_out = np;
  if (!rows52 || cap < int64_t(np) || np == 0) return VXS_OK;
  VXS_CUDA(ctx, ctx->stage.reserve(size_t(np) * 52));
  VXS_CUDA(ctx, ctx->stage_i64.reserve(size_t(np) * 5));
  VXS_LAUNCH(ctx, "k_map_plane_rows", k_map_plane_rows, nblk(nn, 128), 128, 0, view(m), m->n_nodes, m->sel.p, m->voff.p, ctx->stage.p, (long long*)ctx->stage_i64.p);
  VXS_CUDA(ctx, cudaMemcpyAsync(rows52, ctx->stage.p, size_t(np) * 52 * 8, cudaMemcpyDeviceToHost, st));
  if (ids5) VXS_CUDA(ctx, cudaMemcpyAsync(ids5, ctx->stage_i64.p, size_t(np) * 5 * 8, cudaMemcpyDeviceToHost, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  return VXS_OK;
}

// The per-point loop of the EKF update (voxelslam.cpp:876-918) against the resident map: no plane table is exported (vxs_odom_set_planes is the
// host-octree path).  pv12 = NULL uses the scan that vxs_var_init / a previous call left on the device.
extern "C" int vxs_map_odom_accumulate(vxs_map* m, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, double* HTH36, double* HTz6,
                                       double* nnt9, int64_t* match_num, int32_t* flags) {
  if (!m || n < 0 || !pose12 || !rot_var9 || !tsl_var9 || !HTH36 || !HTz6 || !nnt9 || !match_num) return VXS_ERR_ARG;
  vxs_ctx* ctx = m->ctx;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  if (pv12) { int rc = vxs_odom_set_resident_scan(ctx, pv12, n); if (rc) return rc; }
  double* pv = nullptr; long long nres = 0;
  vxs_odom_resident_scan(ctx, &pv, &nres);
  if (nres != n) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_map_odom_accumulate: no resident scan of this size");
  double sth[30];
  for (int k = 0; k < 12; k++) sth[k] = pose12[k];
  for (int k = 0; k < 9; k++) { sth[12 + k] = rot_var9[k]; sth[21 + k] = tsl_var9[k]; }
  VXS_CUDA(ctx, m->odom_st.reserve(30 + 34));
  double* d_st = m->odom_st.p; double* d_out = m->odom_st.p + 30;
  VXS_CUDA(ctx, cudaMemcpyAsync(d_st, sth, sizeof sth, cudaMemcpyHostToDevice, st));
  VXS_CUDA(ctx, cudaMemsetAsync(d_out, 0, 34 * 8, st));
  int* dflags = nullptr;
  if (flags && n > 0) { VXS_CUDA(ctx, m->flagbuf.reserve(size_t(n))); dflags = reinterpret_cast<int*>(m->flagbuf.p); }
  if (n > 0 && m->n_nodes > 0)
    VXS_LAUNCH(ctx, "k_map_odom", k_map_odom<false>, nblk(size_t(n), 256), 256, 0, view(m), m->table.p, (unsigned int)(m->tcap - 1), pv, (long long)n, d_st, m->mp.voxel_size, d_out, dflags,
               nullptr);
  else if (dflags) VXS_CUDA(ctx, cudaMemsetAsync(dflags, 0, size_t(n) * 4, st));
  double out[34];
  VXS_CUDA(ctx, cudaMemcpyAsync(out, d_out, sizeof out, cudaMemcpyDeviceToHost, st));
  if (dflags) VXS_CUDA(ctx, cudaMemcpyAsync(flags, dflags, size_t(n) * 4, cudaMemcpyDeviceToHost, st));
  VXS_CUDA(ctx, cudaStreamSynchronize(st));
  int u = 0;
  for (int a = 0; a < 6; a++) for (int b = a; b < 6; b++) { HTH36[6 * a + b] = out[u]; HTH36[6 * b + a] = out[u]; u++; }
  for (int a = 0; a < 6; a++) HTz6[a] = out[21 + a];
  const int sy[9] = {27, 28, 29, 28, 30, 31, 29, 31, 32};
  for (int k = 0; k < 9; k++) nnt9[k] = out[sy[k]];
  *match_num = int64_t(out[33] + 0.5);
  return VXS_OK;
}

// lio_state_estimation (voxelslam.cpp:856-958) against the resident map: the driver and the step kernel are vxs_odom.cu's, the passes k_map_odom<true>.
extern "C" int vxs_map_lio_update(vxs_map* m, const double* pv12, int64_t n, double* state24, double* cov225, int32_t* ok, int32_t* iters, int64_t* match_num, double* trace12,
                                  int32_t* flags) {
  if (!m || n < 0 || !state24 || !cov225 || !ok || !iters || !match_num) return VXS_ERR_ARG;
  vxs_ctx* ctx = m->ctx;
  auto assoc = [&](unsigned grid, const double* pv, long long np, const double* st, const int* stopped, double* rows, int* fl) -> int {
    VXS_LAUNCH(ctx, "k_map_odom_rows", k_map_odom<true>, grid, OD_THREADS, 0, view(m), m->table.p, (unsigned int)(m->tcap - 1), pv, np, st, m->mp.voxel_size, rows, fl, stopped);
    return VXS_OK;
  };
  return vxs_lio_run(ctx, "vxs_map_lio_update", pv12, n, m->n_nodes > 0, assoc, state24, cov225, ok, iters, match_num, trace12, flags);
}
