// LidarFactor evaluation (sm_90a): the kernels of acc_evaluate2 (voxel_map.hpp:132-241), re-designed for the GPU, and the host drivers
// of both evaluations; evaluate_only_residual (voxel_map.hpp:243-279) is the streaming kernel of vxs_resid.cu.
//
//   k_jac           group per voxel, lane per entry: g_i, D_i and the three scaled rank-1 rows x^m_i (SURVEY App. A.3),
//                   rows stored for the SYRK, g/D accumulated with fp64 RED.                 k*80+176 B read, k*144 B written / voxel
//   k_syrk          H -= X^T X on the fp64 tensor cores (mma.sync.m16n8k4.f64 / DMMA.16x8x4): warp unit = 48x48 output (8x8 frames,
//                   6x6 tiles of 8x8, one MMA per pair of tile rows, 72 accumulators/lane), CTA = 2x2 units, X staged with cp.async (zero-fill), 3 stages;
//                   split over voxel chunks, fp64 RED epilogue.  fp64-bound for k >~ 4 (SURVEY §7.3).
//   k_lambda_sum    thread per voxel: residual of acc_evaluate2 from the cached eigenvalues, deterministic two-level reduction of
//                   sum coe*lambda0 ("last block" pattern).
//   k_pairs         sparse windows (k << W, top-level global BA): group per voxel, block pairs straight to RED.
//   k_assemble      dense n x n system from the block accumulators (+ the CPU-evaluated IMU 30x30 blocks), mirror of the lower triangle.
#include <algorithm>
#include <cstdlib>
#include "vxs_factor_view.cuh"

// deterministic block + grid reduction of one double per thread; result[0] written by the last block
__device__ __forceinline__ void block_grid_sum(double val, double* partial, unsigned int* counter, double* result) {
  __shared__ double sh[256];
  __shared__ bool is_last;
  const int tid = threadIdx.x;
  sh[tid] = val;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) { if (tid < s) sh[tid] += sh[tid + s]; __syncthreads(); }
  if (tid == 0) {
    partial[blockIdx.x] = sh[0];
    __threadfence();
    unsigned int t = atomicAdd(counter, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    double a = 0.0;
    for (unsigned int i = tid; i < gridDim.x; i += blockDim.x) a += __ldcg(partial + i);
    sh[tid] = a;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) { if (tid < s) sh[tid] += sh[tid + s]; __syncthreads(); }
    if (tid == 0) { result[0] = sh[0]; *counter = 0u; }
  }
}

// residual += coe * lmbd[kk] of acc_evaluate2 (voxel_map.hpp:234) from the cached eigenvalues
__global__ void __launch_bounds__(256) k_lambda_sum(FactorView f, double* partial, unsigned int* counter, double* result) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  block_grid_sum(v < f.V ? f.coe[v] * f.eig[v] : 0.0, partial, counter, result);
}

// per-voxel constants of acc_evaluate2 (voxel_map.hpp:163-174), once per voxel instead of once per (voxel, frame) lane:
// the two square roots and four divisions are ~25 % of a lane's instructions otherwise
__global__ void __launch_bounds__(256) k_voxel_consts(FactorView f, double* __restrict__ vc) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= f.V) return;
  const size_t st = f.Vcap;
  const double lam[3] = {f.eig[v], f.eig[st + v], f.eig[2 * st + v]};
  const double* s = f.sum + v;
  const voxel_consts k = make_voxel_consts(lam, mk3(0, 0, 0), mk3(0, 0, 0), mk3(0, 0, 0), mk3(s[6 * st], s[7 * st], s[8 * st]), s[9 * st], f.coe[v]);
  vc[v] = k.s1; vc[st + v] = k.s2; vc[2 * st + v] = k.s3; vc[3 * st + v] = k.invN; vc[4 * st + v] = k.vbar.x; vc[5 * st + v] = k.vbar.y; vc[6 * st + v] = k.vbar.z; vc[7 * st + v] = k.coe;
}
__device__ __forceinline__ voxel_consts load_voxel_consts(const FactorView& f, int v) {
  const size_t st = f.Vcap;
  const double* e = f.eig + v;
  voxel_consts k;
  k.u0 = mk3(__ldg(e + 3 * st), __ldg(e + 6 * st), __ldg(e + 9 * st));
  k.u1 = mk3(__ldg(e + 4 * st), __ldg(e + 7 * st), __ldg(e + 10 * st));
  k.u2 = mk3(__ldg(e + 5 * st), __ldg(e + 8 * st), __ldg(e + 11 * st));
  const double* c = f.vc + v;
  k.s1 = __ldg(c); k.s2 = __ldg(c + st); k.s3 = __ldg(c + 2 * st); k.invN = __ldg(c + 3 * st);
  k.vbar = mk3(__ldg(c + 4 * st), __ldg(c + 5 * st), __ldg(c + 6 * st)); k.coe = __ldg(c + 7 * st);
  k.NN = 0.0;
  return k;
}

// ------------------------------------------------------------------ Hessian part 1: per-entry Jacobian rows
// Dense-window layout of the scaled rank-3 rows, shaped for the fp64 tensor-core SYRK (k_syrk):
//   rows of X = (voxel, m) flattened, 3 per voxel; four voxels = 12 rows = three k-chunks of 4 rows;
//   XT[voxel_group][chunk 0..2][column 0..6W-1][kr 0..3]   (column = 6*frame + c)
// so that (a) one k-chunk of a range of frames is one contiguous run (bulk cp.async staging) and (b) a warp's mma fragment
// (lane l -> row l&3, column c0 + l>>2) is 32 consecutive doubles in shared memory.
__device__ __forceinline__ size_t xt_index(int v, int frame, int m, int c, int n) {
  const int r = 3 * (v & 3) + m;
  return ((size_t(v >> 2) * 3 + (r >> 2)) * n + 6 * frame + c) * 4 + (r & 3);
}
__device__ __forceinline__ void xt_store_zero(double* X, int v, int f0, int nframes, int n) {
  for (int f = f0; f < f0 + nframes; f++)
    for (int m = 0; m < 3; m++) {
      const size_t b = xt_index(v, f, m, 0, n);
#pragma unroll
      for (int c = 0; c < 6; c++) X[b + 4 * c] = 0.0;
    }
}

// Gradient / block-diagonal accumulation without per-entry atomics: a thread keeps the 30 sums of the frame it is currently
// looking at in registers and only flushes them (fp64 RED) when its frame changes.  In a sliding window the entry a lane
// handles has the same frame for (almost) every voxel, so the flush happens a handful of times per thread instead of once per
// entry; in sparse global-BA windows it degenerates gracefully to the per-entry scatter (where contention is low anyway).
template <int G, bool DENSE>
__global__ void __launch_bounds__(128, 3) k_jac(FactorView f, const double* __restrict__ poses, int pstride, double* __restrict__ X, double* __restrict__ gD,
                                                const int32_t* __restrict__ vwin, const int* __restrict__ build_mask) {   // batch: voxels of windows with build_mask == 0 are skipped
  __shared__ double acc[30][128];   // per-thread running sums for the thread's current frame (column = thread: conflict-free)
  const int tid = threadIdx.x;
  const int lane = tid & (G - 1);
  const int group = (blockIdx.x * blockDim.x + tid) / G;
  const int ngroups = (gridDim.x * blockDim.x) / G;
  const int W = f.W;
  double* gbuf = gD;
  double* Dbuf = gD + size_t(W) * 6;
  int cur_fr = -1;
#pragma unroll
  for (int i = 0; i < 30; i++) acc[i][tid] = 0.0;
  for (int v = group; v < f.V; v += ngroups) {
    if (build_mask && !build_mask[vwin[v]]) continue;
    const int beg = f.ptr[v], end = f.ptr[v + 1];
    if (DENSE && beg == end && lane == 0) xt_store_zero(X, v, 0, W, 6 * W);
    if (beg + lane >= end) continue;
    const voxel_consts kc = load_voxel_consts(f, v);
    for (int en = beg + lane; en < end; en += G) {
      cluster c = load_cluster_soa(f.cl, f.Ecap, size_t(en));
      const int fr = __ldg(f.frame + en);
      if (fr != cur_fr) {
        if (cur_fr >= 0) {
          double* g = gbuf + cur_fr * 6; double* D = Dbuf + cur_fr * 24;
#pragma unroll
          for (int i = 0; i < 6; i++) { atomicAdd(g + i, acc[i][tid]); acc[i][tid] = 0.0; }
#pragma unroll
          for (int i = 0; i < 24; i++) { atomicAdd(D + i, acc[6 + i][tid]); acc[6 + i][tid] = 0.0; }
        }
        cur_fr = fr;
      }
      rot3 R; d3 t;
      load_pose(poses, pstride, fr, R, t);
      entry_out o;
      entry_jacobian(kc, c, R, t, o);
      if (DENSE) {
#pragma unroll
        for (int m = 0; m < 3; m++) {
          const size_t b = xt_index(v, fr, m, 0, 6 * W);
#pragma unroll
          for (int cc = 0; cc < 6; cc++) X[b + 4 * cc] = o.x[6 * m + cc];
        }
        // zero the slots of frames that do not observe this voxel
        const int prev = (en > beg) ? __ldg(f.frame + en - 1) : -1;
        if (fr - prev > 1) xt_store_zero(X, v, prev + 1, fr - prev - 1, 6 * W);
        if (en == end - 1 && fr < W - 1) xt_store_zero(X, v, fr + 1, W - 1 - fr, 6 * W);
      } else {
        double2* x2 = reinterpret_cast<double2*>(X + size_t(en) * 18);
#pragma unroll
        for (int i = 0; i < 9; i++) x2[i] = make_double2(o.x[2 * i], o.x[2 * i + 1]);
      }
#pragma unroll
      for (int i = 0; i < 6; i++) acc[i][tid] += kc.coe * o.g[i];
#pragma unroll
      for (int i = 0; i < 9; i++) { acc[6 + i][tid] += o.Drr[i]; acc[15 + i][tid] += o.Drt[i]; }
#pragma unroll
      for (int i = 0; i < 6; i++) acc[24 + i][tid] += o.Dtt[i];
    }
  }
  if (cur_fr >= 0) {
    double* g = gbuf + cur_fr * 6; double* D = Dbuf + cur_fr * 24;
#pragma unroll
    for (int i = 0; i < 6; i++) atomicAdd(g + i, acc[i][tid]);
#pragma unroll
    for (int i = 0; i < 24; i++) atomicAdd(D + i, acc[6 + i][tid]);
  }
}

// Dense windows, W <= 128: same math as k_jac<.,true>, but a CTA owns whole voxel groups (4 voxels = one 12-row slab of XT),
// builds the slab in shared memory and writes it out with coalesced 16-B stores — XT sectors interleave rows of different
// voxels, so per-entry stores would be partial-sector writes from different warps.  Threads are 64-lane groups (lane = frame slot
// in a sliding window), two voxels per round, two rounds per group; gradient / D sums as in k_jac.
template <int LPV>   // lanes per voxel: 64 (W <= 64, two voxels per round) or 128 (W <= 128, one voxel per round) so that a lane keeps one frame slot
__global__ void __launch_bounds__(128, 3) k_jac_slab(FactorView f, const double* __restrict__ poses, int pstride, double* __restrict__ XT, double* __restrict__ gD, int g_first,
                                                     int ngroups_vox) {   // voxel groups [g_first, ngroups_vox)
  extern __shared__ __align__(16) double sm[];
  constexpr int VPR = 128 / LPV;                     // voxels per round
  const int tid = threadIdx.x, half = tid / LPV, lane = tid % LPV;
  const int W = f.W, n = 6 * W;
  const int slab = 3 * n * 4;                        // doubles per voxel group (global layout [chunk][col][kr])
  const int TW = 7 * W;                              // padded row length of the shared slab: [chunk][kr][7*frame + c] — a lane (frame)
  const int tslab = 12 * TW;                         // advances 7 doubles, so 16 lanes hit 32 distinct banks (6 would 4-way conflict)
  double* acc = sm;                                  // [30][128]
  double* T = sm + 30 * 128;
  double* sp = T + tslab;                            // [12][W] poses
  double* gbuf = gD;
  double* Dbuf = gD + size_t(W) * 6;
  int cur_fr = -1;
#pragma unroll
  for (int i = 0; i < 30; i++) acc[i * 128 + tid] = 0.0;
  stage_poses(sp, poses, pstride, W);
  for (int G = g_first + blockIdx.x; G < ngroups_vox; G += gridDim.x) {
    {   // pull the next group's entries and voxel constants towards L2 while this one is computed
      const int Gn = G + gridDim.x;
#pragma unroll
      for (int round = 0; round < 4 / VPR; round++) {
        const int vn = 4 * Gn + VPR * round + half;
        if (Gn < ngroups_vox && vn < f.V) {
          prefetch_entry(f, __ldg(f.ptr + vn) + lane);
          if (lane < 9) prefetch_l2(f.eig + size_t(3 + lane) * f.Vcap + vn); else if (lane < 17) prefetch_l2(f.vc + size_t(lane - 9) * f.Vcap + vn);
        }
      }
    }
    for (int i = tid; i < tslab / 2; i += 128) reinterpret_cast<double2*>(T)[i] = make_double2(0.0, 0.0);
    __syncthreads();
    for (int round = 0; round < 4 / VPR; round++) {
      const int v = 4 * G + VPR * round + half;
      if (v >= f.V) continue;
      const int beg = f.ptr[v], end = f.ptr[v + 1];
      if (beg + lane >= end) continue;
      const voxel_consts kc = load_voxel_consts(f, v);
      for (int en = beg + lane; en < end; en += LPV) {
        cluster c = load_cluster_soa(f.cl, f.Ecap, size_t(en));
        const int fr = __ldg(f.frame + en);
        if (fr != cur_fr) {
          if (cur_fr >= 0) {
            double* g = gbuf + cur_fr * 6; double* D = Dbuf + cur_fr * 24;
#pragma unroll
            for (int i = 0; i < 6; i++) { atomicAdd(g + i, acc[i * 128 + tid]); acc[i * 128 + tid] = 0.0; }
#pragma unroll
            for (int i = 0; i < 24; i++) { atomicAdd(D + i, acc[(6 + i) * 128 + tid]); acc[(6 + i) * 128 + tid] = 0.0; }
          }
          cur_fr = fr;
        }
        rot3 R; d3 t;
        load_pose_s(sp, W, fr, R, t);
        entry_out o;
        entry_jacobian(kc, c, R, t, o);
#pragma unroll
        for (int m = 0; m < 3; m++) {
          const int r = 3 * (v & 3) + m;     // row of the slab = (chunk r>>2, kr r&3)
          double* dst = T + size_t(r) * TW + 7 * fr;
#pragma unroll
          for (int cc = 0; cc < 6; cc++) dst[cc] = o.x[6 * m + cc];
        }
#pragma unroll
        for (int i = 0; i < 6; i++) acc[i * 128 + tid] += kc.coe * o.g[i];
#pragma unroll
        for (int i = 0; i < 9; i++) { acc[(6 + i) * 128 + tid] += o.Drr[i]; acc[(15 + i) * 128 + tid] += o.Drt[i]; }
#pragma unroll
        for (int i = 0; i < 6; i++) acc[(24 + i) * 128 + tid] += o.Dtt[i];
      }
    }
    __syncthreads();
    double2* dst = reinterpret_cast<double2*>(XT + size_t(G) * slab);
    for (int i = tid; i < 3 * n; i += 128) {        // i = chunk*n + col : gather the four kr values, write one 32-B sector
      const int ch = i / n, col = i - ch * n, fq = col / 6, cc = col - fq * 6;
      const double* src = T + size_t(4 * ch) * TW + 7 * fq + cc;
      dst[2 * i] = make_double2(src[0], src[TW]);
      dst[2 * i + 1] = make_double2(src[2 * TW], src[3 * TW]);
    }
    __syncthreads();
  }
  if (cur_fr >= 0) {
    double* g = gbuf + cur_fr * 6; double* D = Dbuf + cur_fr * 24;
#pragma unroll
    for (int i = 0; i < 6; i++) atomicAdd(g + i, acc[i * 128 + tid]);
#pragma unroll
    for (int i = 0; i < 24; i++) atomicAdd(D + i, acc[(6 + i) * 128 + tid]);
  }
}

// ------------------------------------------------------------------ Hessian part 2a: sparse windows, block pairs -> RED
template <int G>
__global__ void __launch_bounds__(128) k_pairs(FactorView f, const double* __restrict__ X, double* __restrict__ C) {
  const int lane = threadIdx.x & (G - 1);
  const int group = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int ngroups = (gridDim.x * blockDim.x) / G;
  const int nl = f.W * 6;
  for (int v = group; v < f.V; v += ngroups) {
    const int beg = f.ptr[v], k = f.ptr[v + 1] - beg;
    const int total = k * k * 36;
    for (int idx = lane; idx < total; idx += G) {
      const int a = idx / (36 * k), rem = idx - a * 36 * k, b = rem / 36, el = rem - b * 36;
      if (b < a) continue;
      const int r = el / 6, c = el - r * 6;
      const double* xa = X + size_t(beg + a) * 18 + r;
      const double* xb = X + size_t(beg + b) * 18 + c;
      const double val = xa[0] * xb[0] + xa[6] * xb[6] + xa[12] * xb[12];
      const int fa = __ldg(f.frame + beg + a), fb = __ldg(f.frame + beg + b);
      atomicAdd(C + size_t(6 * fb + c) * nl + 6 * fa + r, -val);
    }
  }
}

// Batch of independent windows (vxs_hba_bottom_batch): frames are global (window * WB + slot), a voxel only touches its own window, so the
// pair blocks go to that window's (6 WB)^2 block of a block-diagonal accumulator instead of a (6 W_total)^2 matrix.
template <int G>
__global__ void __launch_bounds__(128) k_pairs_bd(FactorView f, const double* __restrict__ X, double* __restrict__ Cbd, int WB, const int32_t* __restrict__ vwin, const int* __restrict__ build_mask) {
  const int lane = threadIdx.x & (G - 1);
  const int group = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int ngroups = (gridDim.x * blockDim.x) / G;
  const int nb = 6 * WB;
  for (int v = group; v < f.V; v += ngroups) {
    const int win = vwin[v];
    if (build_mask && !build_mask[win]) continue;
    const int beg = f.ptr[v], k = f.ptr[v + 1] - beg;
    const int total = k * k * 36;
    double* C = Cbd + size_t(win) * nb * nb;
    const int fbase = win * WB;
    for (int idx = lane; idx < total; idx += G) {
      const int a = idx / (36 * k), rem = idx - a * 36 * k, b = rem / 36, el = rem - b * 36;
      if (b < a) continue;
      const int r = el / 6, c = el - r * 6;
      const double* xa = X + size_t(beg + a) * 18 + r;
      const double* xb = X + size_t(beg + b) * 18 + c;
      const double val = xa[0] * xb[0] + xa[6] * xb[6] + xa[12] * xb[12];
      const int fa = __ldg(f.frame + beg + a) - fbase, fb = __ldg(f.frame + beg + b) - fbase;
      atomicAdd(C + size_t(6 * fb + c) * nb + 6 * fa + r, -val);
    }
  }
}
// zero the accumulators of the windows that are rebuilt: Cbd block, g (6 per frame), D (24 per frame)
__global__ void __launch_bounds__(256) k_bd_zero(double* __restrict__ Cbd, double* __restrict__ gD, int WB, int nwin, const int* __restrict__ build_mask) {
  const int win = blockIdx.x;
  if (build_mask && !build_mask[win]) return;
  const int nb = 6 * WB, Wt = nwin * WB;
  for (int i = threadIdx.x; i < nb * nb; i += blockDim.x) Cbd[size_t(win) * nb * nb + i] = 0.0;
  for (int i = threadIdx.x; i < WB * 6; i += blockDim.x) gD[size_t(win) * WB * 6 + i] = 0.0;
  for (int i = threadIdx.x; i < WB * 24; i += blockDim.x) gD[size_t(Wt) * 6 + size_t(win) * WB * 24 + i] = 0.0;
}

// ------------------------------------------------------------------ Hessian part 2b: dense windows, SYRK on the fp64 tensor cores
// H -= X^T X with X = (3V) x (6W).  With scalar DFMA the kernel is limited by the shared-memory -> register delivery
// (2 B per FMA at 72 accumulators/thread equals the 128 B/clk LSU limit at full FP64 rate), not by the FP64 pipe.
// mma.sync.m16n8k4.f64 (SASS DMMA.16x8x4, one of Hopper's fp64 tensor shapes) shares each operand across 8 lanes inside the tensor core.
// On an H100 80GB HBM3 (700 W power limit, 1980 MHz; tools/dmma_shapes.py) it runs at 66.5 TFLOP/s, twice Ampere's m8n8k4 (33.4);
// m16n8k8 / m16n8k16 measure the same 66.3 / 66.2, so the SYRK uses the k4 shape, whose fragments are the ones the XT layout stages.
//   * column blocks of 8 frames (48 columns), the remainder block (W mod 8 frames) FIRST so it only pairs with itself;
//   * warp unit = (row block a, column block b), a <= b: 6x6 tiles of 8x8, 72 fp64 accumulators per lane; one m16n8k4 covers the two
//     tiles (ti = 0, 1) of a tile column inside a piece (see SyPiece), its A fragment is exactly the two 8-column runs the XT layout stages;
//   * CTA = 2x2 units; k runs over (voxel, m) rows in chunks of 4; XT (see xt_index) is staged with 16-B cp.async,
//     3 stages of 4 voxels (12 rows); split over voxel chunks; fp64 RED epilogue into the upper block triangle.
#define SY_THREADS 128
#define SY_STAGES 3
#define SY_PCOLS 96                             // columns per part (2 blocks x 48)
#define SY_PART (3 * SY_PCOLS * 4)              // doubles per part per stage: 3 chunks x 96 cols x 4 rows
#define SY_STAGE_DOUBLES (2 * SY_PART)

__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gsrc, bool pred) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
  int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sa), "l"(gsrc), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }
// C[16x8] += A[16x4] B[4x8] (SASS DMMA.16x8x4).  Lane (g = lane/4, t = lane%4) holds a0 = A[g][t], a1 = A[g+8][t], b = B[t][g],
// c0, c1 = C[g][2t, 2t+1] and c2, c3 = C[g+8][2t, 2t+1].
__device__ __forceinline__ void dmma1684(double& c0, double& c1, double& c2, double& c3, double a0, double a1, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
               : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3) : "d"(a0), "d"(a1), "d"(b));
}

struct SyrkGeom { int r0, ngc, nbp, ntiles; };
__device__ inline int sy_gstart(const SyrkGeom& g, int grp) { return grp <= 0 ? 0 : g.r0 + 8 * (grp - 1); }
__device__ inline int sy_glen(const SyrkGeom& g, int grp) { return grp < 0 || grp >= g.ngc ? 0 : (grp == 0 ? g.r0 : 8); }
static SyrkGeom sy_geom(int W) {
  SyrkGeom g;
  g.r0 = (W % 8 == 0) ? 8 : (W % 8);
  g.ngc = (W - g.r0) / 8 + 1;
  g.nbp = (g.ngc + 1) / 2;
  g.ntiles = g.nbp * (g.nbp + 1) / 2;
  return g;
}

// A warp's share of a CTA tile: up to three "pieces", each = two 8-row mma tile rows x six 8-column tile columns (12 tiles)
// of one unit.  Splitting units into pieces and dealing the pieces round-robin keeps all four warps (= all four tensor pipes of
// the SM) busy on diagonal / remainder tiles, where a unit-per-warp mapping leaves one to three warps idle.
struct SyPiece { int offI, offJ, ntI, ntJ, rowbase, colbase, nvalI, nvalJ; unsigned mask; };   // mask: bit ti*6+tj = tile needed

// tile index -> (row part A, column part B), A <= B
__device__ inline void sy_tile_parts(const SyrkGeom& g, int tile, int& A, int& B) {
  int a = 0, rem = tile;
  while (rem >= g.nbp - a) { rem -= g.nbp - a; a++; }
  A = a; B = a + rem;
}

// The pieces of tile (A, B) that `warp` runs: the tile's pieces in a fixed order, piece q to warp q % 4 (warp-uniform, <= 3 per warp).
__device__ inline int sy_pieces(const SyrkGeom& g, int A, int B, int warp, SyPiece (&pc)[3]) {
  int npc = 0, q = 0;
  for (int u = 0; u < 4; u++) {
    const int wy = u >> 1, wx = u & 1, ga = 2 * A + wy, gb = 2 * B + wx;
    if (!(ga < g.ngc && gb < g.ngc && ga <= gb)) continue;
    const int nvalI = 6 * sy_glen(g, ga), nvalJ = 6 * sy_glen(g, gb);
    const int ntI = (nvalI + 7) >> 3, ntJ = (nvalJ + 7) >> 3;
    for (int t0 = 0; t0 < ntI; t0 += 2, q++) {
      if ((q & 3) != warp || npc >= 3) continue;
      SyPiece P;
      P.offI = (wy ? 6 * sy_glen(g, 2 * A) : 0) + 8 * t0;
      P.offJ = wx ? 6 * sy_glen(g, 2 * B) : 0;
      P.ntI = ntI - t0 < 2 ? ntI - t0 : 2; P.ntJ = ntJ;
      P.rowbase = 6 * sy_gstart(g, ga) + 8 * t0; P.colbase = 6 * sy_gstart(g, gb);
      P.nvalI = nvalI - 8 * t0; P.nvalJ = nvalJ;
      // tiles of a diagonal unit whose rows all belong to later frames than all of their columns hold only pairs with
      // frame(i) > frame(j): never stored (11 of the 36 tiles of a full diagonal unit)
      P.mask = 0u;
      for (int ti = 0; ti < P.ntI; ti++)
        for (int tj = 0; tj < P.ntJ; tj++)
          if (!(ga == gb && (8 * (t0 + ti)) / 6 > (8 * tj + 7) / 6)) P.mask |= 1u << (ti * 6 + tj);
      if (npc == 0) pc[0] = P; else if (npc == 1) pc[1] = P; else pc[2] = P;
      npc++;
    }
  }
  return npc;
}

// operand fragments of k-chunk kc of a piece (pI, pJ: the piece's row / column operands in the stage, lane offset included)
__device__ __forceinline__ void sy_frags(const double* pI, const double* pJ, int kc, double (&fa)[2], double (&fb)[6]) {
#pragma unroll
  for (int t = 0; t < 2; t++) fa[t] = pI[(kc * SY_PCOLS + 8 * t) * 4];
#pragma unroll
  for (int t = 0; t < 6; t++) fb[t] = pJ[(kc * SY_PCOLS + 8 * t) * 4];
}

// One k-chunk (4 rows of X) of a piece: one m16n8k4 per tile column tj covers both tile rows ti = 0, 1 (acc[2tj..] and acc[12+2tj..]).
// A column is skipped only when its ti = 0 tile is masked out: its ti = 1 tile (later frames) then is too.  A tile that is computed but
// masked out (ti = 1 of a diagonal column, or the missing second tile row of a one-row piece) is never stored: sy_epilogue tests the mask.
__device__ __forceinline__ void sy_mma_chunk(double* acc, unsigned mask, const double (&fa)[2], const double (&fb)[6]) {
  if ((mask & 0x3Fu) == 0x3Fu) {
#pragma unroll
    for (int tj = 0; tj < 6; tj++) dmma1684(acc[2 * tj], acc[2 * tj + 1], acc[12 + 2 * tj], acc[13 + 2 * tj], fa[0], fa[1], fb[tj]);
  } else {
#pragma unroll
    for (int tj = 0; tj < 6; tj++)
      if ((mask >> tj) & 1u) dmma1684(acc[2 * tj], acc[2 * tj + 1], acc[12 + 2 * tj], acc[13 + 2 * tj], fa[0], fa[1], fb[tj]);
  }
}

// all pieces of one staged voxel group (3 k-chunks)
__device__ __forceinline__ void sy_stage_mma(double (&acc)[72], const SyPiece (&pc)[3], int npc, const double* sI, const double* sJ) {
#pragma unroll
  for (int p = 0; p < 3; p++) {
    if (p < npc) {
      const double* pI = sI + size_t(pc[p].offI) * 4;
      const double* pJ = sJ + size_t(pc[p].offJ) * 4;
#pragma unroll
      for (int kc = 0; kc < 3; kc++) {
        double fa[2], fb[6];
        sy_frags(pI, pJ, kc, fa, fb);
        sy_mma_chunk(acc + p * 24, pc[p].mask, fa, fb);
      }
    }
  }
}

// lane holds C[8ti + lane/4][8tj + 2(lane%4) + {0,1}] of every tile of its pieces; H_ij -= x_i x_j^T for frame(i) <= frame(j), fp64 RED
__device__ __forceinline__ void sy_epilogue(const double (&acc)[72], const SyPiece (&pc)[3], int npc, int lane, double* __restrict__ C, int n) {
  const int rl = lane >> 2, cl = 2 * (lane & 3);
#pragma unroll
  for (int p = 0; p < 3; p++) {
    if (p < npc) {
#pragma unroll
      for (int ti = 0; ti < 2; ti++)
#pragma unroll
        for (int tj = 0; tj < 6; tj++) {
          const int r = 8 * ti + rl;
          if (((pc[p].mask >> (ti * 6 + tj)) & 1u) && r < pc[p].nvalI) {
            const int R = pc[p].rowbase + r;
#pragma unroll
            for (int e = 0; e < 2; e++) {
              const int c = 8 * tj + cl + e;
              const int Cc = pc[p].colbase + c;
              if (c < pc[p].nvalJ && (R / 6) <= (Cc / 6)) atomicAdd(C + size_t(Cc) * n + R, -acc[p * 24 + 2 * (ti * 6 + tj) + e]);
            }
          }
        }
    }
  }
}

// One CTA = one (tile, voxel chunk) work item: XT staged with 16-B cp.async (zero-fill past a part's columns), SY_STAGES stages of one
// voxel group each, one CTA barrier per stage, RED epilogue.
__global__ void __launch_bounds__(SY_THREADS, 2) k_syrk(const double* __restrict__ XT, double* __restrict__ C, int g_first, int ngroups_vox, int W, SyrkGeom g, int groups_per_chunk) {
  extern __shared__ __align__(16) double smem[];
  const int tile = int(blockIdx.x % g.ntiles), chunk = int(blockIdx.x / g.ntiles);
  const int g_begin = g_first + chunk * groups_per_chunk, g_end = min(ngroups_vox, g_begin + groups_per_chunk);   // voxel groups [g_first, ngroups_vox)
  if (g_begin >= g_end) return;
  int A, B;
  sy_tile_parts(g, tile, A, B);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = 6 * W;
  // part geometry: part I = blocks 2A, 2A+1 (contiguous frames), part J = blocks 2B, 2B+1
  const int colI0 = 6 * sy_gstart(g, 2 * A), ncolI = 6 * (sy_glen(g, 2 * A) + sy_glen(g, 2 * A + 1));
  const int colJ0 = 6 * sy_gstart(g, 2 * B), ncolJ = 6 * (sy_glen(g, 2 * B) + sy_glen(g, 2 * B + 1));
  SyPiece pc[3];
  const int npc = sy_pieces(g, A, B, warp, pc);

  double acc[72];
#pragma unroll
  for (int i = 0; i < 72; i++) acc[i] = 0.0;

  const int nsteps = g_end - g_begin;                  // one voxel group (4 voxels, 3 k-chunks) per step
  constexpr int CH_PER_RUN = SY_PCOLS * 2;             // 16-B chunks per (k-chunk, part) run: 96 cols x 32 B
  constexpr int CH_PER_STAGE = 3 * 2 * CH_PER_RUN;     // 1152
  constexpr int CH_PER_THREAD = CH_PER_STAGE / SY_THREADS;   // 9
  // the loader's address arithmetic does not depend on the step: do it once (source offset inside a voxel group, smem offset, predicate)
  int ld_src[CH_PER_THREAD], ld_dst[CH_PER_THREAD];
  unsigned ld_ok = 0;
#pragma unroll
  for (int j = 0; j < CH_PER_THREAD; j++) {
    const int ch = tid + j * SY_THREADS;
    const int run = ch / CH_PER_RUN, off = ch - run * CH_PER_RUN;      // run = part*3 + kchunk
    const int part = run / 3, kc = run - part * 3;
    const int col = off >> 1;                                            // column inside the part
    const bool ok = col < (part ? ncolJ : ncolI);
    ld_src[j] = (kc * n + (part ? colJ0 : colI0) + (ok ? col : 0)) * 4 + (off & 1) * 2;
    ld_dst[j] = part * SY_PART + (kc * SY_PCOLS + col) * 4 + (off & 1) * 2;
    ld_ok |= (ok ? 1u : 0u) << j;
  }
  const size_t group_stride = size_t(3) * n * 4;
  auto issue = [&](int step) {
    double* sbase = smem + size_t(step % SY_STAGES) * SY_STAGE_DOUBLES;
    const double* gbase = XT + size_t(g_begin + step) * group_stride;
#pragma unroll
    for (int j = 0; j < CH_PER_THREAD; j++) cp_async16_zfill(sbase + ld_dst[j], gbase + ld_src[j], (ld_ok >> j) & 1u);
  };
  for (int s = 0; s < SY_STAGES - 1; s++) { if (s < nsteps) issue(s); cp_async_commit(); }
  for (int step = 0; step < nsteps; step++) {
    cp_async_wait<SY_STAGES - 2>();
    __syncthreads();
    if (step + SY_STAGES - 1 < nsteps) issue(step + SY_STAGES - 1);
    cp_async_commit();
    const double* sI = smem + size_t(step % SY_STAGES) * SY_STAGE_DOUBLES + lane;
    sy_stage_mma(acc, pc, npc, sI, sI + SY_PART);
  }
  cp_async_wait<0>();
  sy_epilogue(acc, pc, npc, lane, C, n);
}

// ------------------------------------------------------------------ dense system assembly
// H (n x n col-major) from the lidar block accumulator C (upper block triangle), block-diagonal D, gradient g, and the
// host-evaluated IMU part (already summed over factors, unscaled).  S = dofs per frame (6 or 15); rows >= W*S are the gravity dofs.
// Mirrors hess_plus (voxel_map.hpp:455-463) + "Hess.block(6i,6j) = Hess.block(6j,6i)^T" (voxel_map.hpp:237-239).
__global__ void k_assemble(const double* __restrict__ C, const double* __restrict__ gD, const double* __restrict__ blocks, const double* __restrict__ gvec, int bs,
                           double imu_coef, int W, int S, int n, double* __restrict__ H, double* __restrict__ jact) {
  const size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= size_t(n) * n) return;
  const int row = int(idx % n), col = int(idx / n);
  const int nl = 6 * W, nfs = W * S;
  const double* Dbuf = gD + size_t(W) * 6;
  double val = 0.0;
  if (row < nfs && col < nfs) {
    const int fi = row / S, a = row - fi * S, fj = col / S, b = col - fj * S;
    if (a < 6 && b < 6) {
      if (fi < fj) val = C[size_t(6 * fj + b) * nl + 6 * fi + a];
      else if (fi > fj) val = C[size_t(6 * fi + a) * nl + 6 * fj + b];
      else {
        val = C[size_t(6 * fi + b) * nl + 6 * fi + a];
        const double* D = Dbuf + fi * 24;
        if (a < 3 && b < 3) val += D[3 * a + b];
        else if (a < 3) val += D[9 + 3 * a + (b - 3)];
        else if (b < 3) val += D[9 + 3 * b + (a - 3)];
        else {
          const int p = a - 3, q = b - 3, lo = p < q ? p : q, hi = p < q ? q : p;
          val += D[18 + (lo == 0 ? hi : (lo == 1 ? 2 + hi : 5))];
        }
      }
    }
  }
  if (blocks) {  // IMU factor i couples frames (i, i+1) [and the 3 gravity dofs]: voxel_map.hpp:493-499 / 701-712, then *= imu_coef
    const size_t bb = size_t(bs) * bs;
    double imu = 0.0;
    const bool rg = row >= nfs, cg = col >= nfs;
    if (!rg && !cg) {
      const int fi = row / S, a = row - fi * S, fj = col / S, b = col - fj * S;
      if (fi == fj) {
        if (fi >= 1) imu += blocks[size_t(fi - 1) * bb + size_t(15 + b) * bs + 15 + a];
        if (fi <= W - 2) imu += blocks[size_t(fi) * bb + size_t(b) * bs + a];
      } else if (fi + 1 == fj) imu += blocks[size_t(fi) * bb + size_t(15 + b) * bs + a];
      else if (fj + 1 == fi) imu += blocks[size_t(fj) * bb + size_t(b) * bs + 15 + a];
    } else if (rg && cg) {
      for (int i = 0; i < W - 1; i++) imu += blocks[size_t(i) * bb + size_t(30 + col - nfs) * bs + 30 + row - nfs];
    } else if (rg) {
      const int fj = col / S, b = col - fj * S, lr = 30 + row - nfs;
      if (fj >= 1) imu += blocks[size_t(fj - 1) * bb + size_t(15 + b) * bs + lr];
      if (fj <= W - 2) imu += blocks[size_t(fj) * bb + size_t(b) * bs + lr];
    } else {
      const int fi = row / S, a = row - fi * S, lc = 30 + col - nfs;
      if (fi >= 1) imu += blocks[size_t(fi - 1) * bb + size_t(lc) * bs + 15 + a];
      if (fi <= W - 2) imu += blocks[size_t(fi) * bb + size_t(lc) * bs + a];
    }
    val += imu_coef * imu;
  }
  H[idx] = val;
  if (col == 0) {
    double g = 0.0;
    if (row < nfs) { const int fi = row / S, a = row - fi * S; if (a < 6) g = gD[fi * 6 + a]; }
    if (gvec) {
      double gi = 0.0;
      if (row < nfs) {
        const int fi = row / S, a = row - fi * S;
        if (fi >= 1) gi += gvec[size_t(fi - 1) * bs + 15 + a];
        if (fi <= W - 2) gi += gvec[size_t(fi) * bs + a];
      } else {
        for (int i = 0; i < W - 1; i++) gi += gvec[size_t(i) * bs + 30 + row - nfs];
      }
      g += imu_coef * gi;
    }
    jact[row] = g;
  }
}

// ------------------------------------------------------------------ host drivers
static inline unsigned nblk(size_t n, unsigned b) { return unsigned((n + b - 1) / b); }

// k_syrk over voxel groups [g0, g1) as a (tile, voxel chunk) grid; n_up > 1 when the groups are one of the n_up upload chunks of a
// chunked first build, which share the waves.  Waves: CTA durations differ by 3x between tile kinds (full off-diagonal / diagonal /
// remainder) and the CTAs are dispatched in order, so the last wave leaves SMs idle for up to one CTA duration; ncu showed 68.6 % DMMA-pipe
// activity on average against 85.5 % on the busiest SM at 4 waves.  More, shorter CTAs shrink that tail (each pays one pipeline fill and
// one 96x96 RED epilogue); k_syrk measured at the metric shape (tools/dmma_shapes.py, H100 80GB HBM3, 700 W power limit, 1980 MHz):
// 4 waves 0.576 ms, 8: 0.552, 12: 0.557, 16: 0.568, 24: 0.598.
static int launch_syrk(vxs_ctx* ctx, vxs_factor* f, double* C, int W, int g0, int g1, int n_up) {
  const SyrkGeom g = sy_geom(W);
  const int ng = g1 - g0;
  const size_t smem = size_t(SY_STAGES) * SY_STAGE_DOUBLES * 8;
  VXS_CUDA(ctx, cudaFuncSetAttribute(k_syrk, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  const int target_ctas = std::max(1, ctx->sm_count * 2 * ctx->syrk_waves / n_up);
  int nchunks = std::max(1, std::min<int>(target_ctas / g.ntiles, (ng + 7) / 8));
  const int gpc = (ng + nchunks - 1) / nchunks;
  nchunks = (ng + gpc - 1) / gpc;
  VXS_LAUNCH(ctx, "k_syrk", k_syrk, unsigned(nchunks * g.ntiles), SY_THREADS, smem, f->X.p, C, g0, g1, W, g, gpc);
  return VXS_OK;
}
static int pick_group(const vxs_factor* f) {
  const double avg = f->V > 0 ? double(f->E) / double(f->V) : 1.0;
  return avg > 16.0 ? 32 : (avg > 8.0 ? 16 : 8);
}
static int pick_group_jac(const vxs_factor* f) {   // one lane per frame slot of the window when it fits (W <= 64)
  const double avg = f->V > 0 ? double(f->E) / double(f->V) : 1.0;
  if (avg > 24.0 && f->W > 32) return 64;
  return avg > 16.0 ? 32 : (avg > 8.0 ? 16 : 8);
}

// layout of the all-reducible accumulator block: [ C (6W)^2 | g 6W | D 24W | r1 ]
static size_t hess_block_doubles(int W) { return size_t(6 * W) * size_t(6 * W) + size_t(30) * W + 1; }

int vxs_eval_residual_dev(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pstride, double* residual_dev) {
  if (f->V == 0) {   // a rank of a voxel-sharded run may own no voxel at all: it still has to take part in the scalar all-reduce
    VXS_CUDA(ctx, cudaMemsetAsync(residual_dev, 0, 8, ctx->stream));
    if (ctx->nranks > 1) return vxs_comm_allreduce(ctx, residual_dev, 1);
    return VXS_OK;
  }
  { int rcw = vxs_factor_wait_uploads(f); if (rcw) return rcw; }
  { int rcs = vxs_residual_stream_launch(ctx, f, poses_dev, pstride, residual_dev); if (rcs) return rcs; }
  if (ctx->nranks > 1) return vxs_comm_allreduce(ctx, residual_dev, 1);
  return VXS_OK;
}

// Builds C / g / D / r1 in f->C (layout above).  Dense windows go through the SYRK, sparse ones through k_pairs.
int vxs_eval_hessian_dev(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pstride, double* /*unused*/) {
  const int W = f->W;
  const size_t nl = size_t(6) * W, tot = hess_block_doubles(W);
  VXS_CUDA(ctx, f->C.reserve(tot));
  double* C = f->C.p; double* gD = C + nl * nl; double* r1 = gD + size_t(30) * W;
  VXS_CUDA(ctx, cudaMemsetAsync(C, 0, tot * 8, ctx->stream));
  if (f->V > 0) {
    FactorView fv = make_view(f);
    const int G = pick_group(f);
    // dense-slot rows when the window is reasonably covered (SURVEY §5 "long-context" row): V*W*144 B vs E*144 B
    const bool dense = (double(f->V) * W <= 4.0 * double(f->E)) && (double(f->V) * W * 144.0 <= 24e9);
    const size_t vpad = (size_t(f->V) + 3) & ~size_t(3);
    const size_t xdoubles = dense ? vpad * W * 18 : size_t(f->E) * 18;
    VXS_CUDA(ctx, f->X.reserve(xdoubles));
    if (dense && W > 128 && (f->V & 3))   // rows of the padding voxels of the last group of 4 must be zero (k_jac_slab zero-fills itself)
      VXS_CUDA(ctx, cudaMemsetAsync(f->X.p + (vpad - 4) * W * 18, 0, size_t(4) * W * 18 * 8, ctx->stream));
    const unsigned blocks_v = nblk(size_t(f->V), 256);
    VXS_CUDA(ctx, f->partial.reserve(blocks_v));
    if (!f->counter.p) { VXS_CUDA(ctx, f->counter.reserve(4)); VXS_CUDA(ctx, cudaMemsetAsync(f->counter.p, 0, 16, ctx->stream)); }
    VXS_CUDA(ctx, f->vc.reserve(size_t(8) * f->Vcap));
    fv.vc = f->vc.p;
    VXS_LAUNCH(ctx, "k_voxel_consts", k_voxel_consts, nblk(size_t(f->V), 256), 256, 0, fv, f->vc.p);
    const int GJ = pick_group_jac(f);
    unsigned gridj = unsigned(std::min<size_t>((size_t(f->V) * GJ + 127) / 128, size_t(ctx->sm_count) * 8));
    unsigned grid = unsigned(std::min<size_t>((size_t(f->V) * G + 127) / 128, size_t(ctx->sm_count) * 16));
#define LAUNCH_JAC(GG, DD) { auto kp = k_jac<GG, DD>; VXS_LAUNCH(ctx, "k_jac", kp, gridj, 128, 0, fv, poses_dev, pstride, f->X.p, gD, (const int32_t*)nullptr, (const int*)nullptr); }
    // First build after vxs_factor_push_voxels_async: the clusters are still arriving in chunks of voxel groups; run the Jacobian and the
    // SYRK chunk by chunk behind the upload events so that the PCIe transfer overlaps them (both kernels only accumulate: RED into C, g, D).
    const bool chunked = f->up_pending > 0 && dense && W <= 128;
    if (!chunked) { int rcw = vxs_factor_wait_uploads(f); if (rcw) return rcw; }
    const int n_up = chunked ? f->up_n : 1;
    if (dense && W <= 128) {
      const int ngv = int((f->V + 3) / 4);
      const size_t smem = (size_t(30) * 128 + size_t(12) * 7 * W + size_t(12) * W) * 8;
      int g0 = 0;
      for (int uc = 0; uc < n_up; uc++) {
        const int g1 = chunked ? std::min(f->up_group_end[uc], ngv) : ngv;
        if (chunked) VXS_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, f->up_ev[uc], 0));
        if (g1 > g0) {
          const int ng = g1 - g0;
          const unsigned grids = unsigned(std::min<int>(ng, ctx->sm_count * 3 * 2));
          if (W <= 64) {
            auto kp = k_jac_slab<64>;
            VXS_CUDA(ctx, cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
            VXS_LAUNCH(ctx, "k_jac", kp, grids, 128, smem, fv, poses_dev, pstride, f->X.p, gD, g0, g1);
          } else {
            auto kp = k_jac_slab<128>;
            VXS_CUDA(ctx, cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
            VXS_LAUNCH(ctx, "k_jac", kp, grids, 128, smem, fv, poses_dev, pstride, f->X.p, gD, g0, g1);
          }
          int rcs = launch_syrk(ctx, f, C, W, g0, g1, n_up);   // SYRK over the same groups
          if (rcs) return rcs;
        }
        g0 = g1;
      }
      if (chunked) f->up_pending = 0;
    } else if (dense) {
      if (GJ == 64) LAUNCH_JAC(64, true) else if (GJ == 32) LAUNCH_JAC(32, true) else if (GJ == 16) LAUNCH_JAC(16, true) else LAUNCH_JAC(8, true)
      int rcs = launch_syrk(ctx, f, C, W, 0, int((f->V + 3) / 4), 1);   // voxel groups of 4 (12 rows of X each)
      if (rcs) return rcs;
    } else {
      if (GJ == 64) LAUNCH_JAC(64, false) else if (GJ == 32) LAUNCH_JAC(32, false) else if (GJ == 16) LAUNCH_JAC(16, false) else LAUNCH_JAC(8, false)
      if (G == 32) { auto kp = k_pairs<32>; VXS_LAUNCH(ctx, "k_pairs", kp, grid, 128, 0, fv, f->X.p, C); }
      else if (G == 16) { auto kp = k_pairs<16>; VXS_LAUNCH(ctx, "k_pairs", kp, grid, 128, 0, fv, f->X.p, C); }
      else { auto kp = k_pairs<8>; VXS_LAUNCH(ctx, "k_pairs", kp, grid, 128, 0, fv, f->X.p, C); }
    }
#undef LAUNCH_JAC
    VXS_LAUNCH(ctx, "k_lambda_sum", k_lambda_sum, blocks_v, 256, 0, fv, f->partial.p, f->counter.p, r1);
  }
  if (ctx->nranks > 1) return vxs_comm_allreduce(ctx, C, tot);
  return VXS_OK;
}

// Block-diagonal Hessian build of a batch of windows: Cbd = [nwin][(6 WB)^2] (upper block triangle, as C), gD = g [W_total][6] | D [W_total][24],
// both zeroed and rebuilt only for the windows with build_mask != 0 (device flags; nullptr = all).  Uses the cached eig / sum like acc_evaluate2.
int vxs_eval_hessian_bd_dev(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pstride, const int* build_mask_dev, double* Cbd, double* gD) {
  const int WB = f->block_W;
  if (WB <= 0 || !f->vwin.p) return vxs_fail(ctx, VXS_ERR_ARG, "not a batch factor");
  const int nwin = f->W / WB;
  VXS_LAUNCH(ctx, "k_bd_zero", k_bd_zero, unsigned(nwin), 256, 0, Cbd, gD, WB, nwin, build_mask_dev);
  if (f->V == 0) return VXS_OK;
  FactorView fv = make_view(f);
  VXS_CUDA(ctx, f->X.reserve(size_t(f->E) * 18));
  VXS_CUDA(ctx, f->vc.reserve(size_t(8) * f->Vcap));
  fv.vc = f->vc.p;
  VXS_LAUNCH(ctx, "k_voxel_consts", k_voxel_consts, nblk(size_t(f->V), 256), 256, 0, fv, f->vc.p);
  const int G = pick_group(f);
  const unsigned grid = unsigned(std::min<size_t>((size_t(f->V) * G + 127) / 128, size_t(ctx->sm_count) * 16));
#define LAUNCH_BD(GG) { auto kj = k_jac<GG, false>; VXS_LAUNCH(ctx, "k_jac", kj, grid, 128, 0, fv, poses_dev, pstride, f->X.p, gD, (const int32_t*)f->vwin.p, build_mask_dev); \
                        auto kp = k_pairs_bd<GG>; VXS_LAUNCH(ctx, "k_pairs", kp, grid, 128, 0, fv, f->X.p, Cbd, WB, (const int32_t*)f->vwin.p, build_mask_dev); }
  if (G == 32) LAUNCH_BD(32) else if (G == 16) LAUNCH_BD(16) else LAUNCH_BD(8)
#undef LAUNCH_BD
  return VXS_OK;
}

// assemble into ctx->Hraw / ctx->jact (n = W*S + extra).  Himu/gimu device pointers or null.
int vxs_assemble_dev(vxs_ctx* ctx, vxs_factor* f, int S, int n, const double* blocks, const double* gvec, int bs, double imu_coef) {
  const int W = f->W;
  const size_t nl = size_t(6) * W;
  VXS_CUDA(ctx, ctx->Hraw.reserve(size_t(n) * n));
  VXS_CUDA(ctx, ctx->jact.reserve(size_t(n)));
  const double* C = f->C.p; const double* gD = C + nl * nl;
  VXS_LAUNCH(ctx, "k_assemble", k_assemble, nblk(size_t(n) * n, 256), 256, 0, C, gD, blocks, gvec, bs, imu_coef, W, S, n, ctx->Hraw.p, ctx->jact.p);
  ctx->hraw_n = n; ctx->hraw_S = S;
  return VXS_OK;
}
double* vxs_hess_r1_dev(vxs_factor* f) { return f->C.p + size_t(6 * f->W) * size_t(6 * f->W) + size_t(30) * f->W; }

// ------------------------------------------------------------------ public evaluation entry points
extern "C" int vxs_factor_evaluate_residual(vxs_ctx* ctx, vxs_factor* f, const double* poses12, double* residual) {
  if (!ctx || !f || !poses12 || !residual || f->ctx != ctx) return VXS_ERR_ARG;
  cudaSetDevice(ctx->device);
  const int W = f->W;
  VXS_CUDA(ctx, ctx->states_a.reserve(size_t(W) * 24));
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->states_a.p, poses12, size_t(W) * 12 * 8, cudaMemcpyHostToDevice, ctx->stream));
  int rc = vxs_eval_residual_dev(ctx, f, ctx->states_a.p, 12, ctx->scal.p);
  if (rc) return rc;
  VXS_CUDA(ctx, cudaMemcpyAsync(residual, ctx->scal.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return VXS_OK;
}

extern "C" int vxs_factor_evaluate_hessian(vxs_ctx* ctx, vxs_factor* f, const double* poses12, double* hess, double* jact, double* residual) {
  if (!ctx || !f || !poses12 || f->ctx != ctx) return VXS_ERR_ARG;
  cudaSetDevice(ctx->device);
  const int W = f->W, n = 6 * W;
  VXS_CUDA(ctx, ctx->states_a.reserve(size_t(W) * 24));
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->states_a.p, poses12, size_t(W) * 12 * 8, cudaMemcpyHostToDevice, ctx->stream));
  int rc = vxs_eval_hessian_dev(ctx, f, ctx->states_a.p, 12, nullptr);
  if (rc) return rc;
  rc = vxs_assemble_dev(ctx, f, 6, n, nullptr, nullptr, 0, 0.0);
  if (rc) return rc;
  if (hess) VXS_CUDA(ctx, cudaMemcpyAsync(hess, ctx->Hraw.p, size_t(n) * n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (jact) VXS_CUDA(ctx, cudaMemcpyAsync(jact, ctx->jact.p, size_t(n) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (residual) VXS_CUDA(ctx, cudaMemcpyAsync(residual, vxs_hess_r1_dev(f), 8, cudaMemcpyDeviceToHost, ctx->stream));
  VXS_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return VXS_OK;
}
