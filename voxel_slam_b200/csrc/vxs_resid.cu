// evaluate_only_residual (voxel_map.hpp:243-279) as ONE streaming kernel (sm_90a):
//
//   k_residual_stream   persistent, RS_PER_SM = 3 CTAs per SM of RS_TE = 256 consumer threads + one producer warp, RS_STAGES = 2 stages each
//                       (tuned on the metric shape, see vxs_residual_stream_launch).  The producer warp streams the SoA cluster columns (80 B per (voxel, frame) entry, + the
//                       4-B frame index) of the CTA's voxel batches through a ring of shared-memory stages with 1-D bulk copies
//                       (cp.async.bulk + mbarrier complete_tx — TMA without a tensor map: every column of a tile is one contiguous run),
//                       so ~130 KB per SM are in flight whatever the consumers do.  TE / 32 consumer warps, per tile of TE entries:
//                         A  thread per entry: PointCluster::transform with the entry's pose (tools.hpp:357-363), result written back in place;
//                         B  thread per (voxel, component, quarter): fixed-order sum of the voxel's run inside the tile into the batch's
//                            accumulators in shared memory (the order depends only on the factor and the launch shape: bit-stable run to run);
//                       after the last tile of a batch, thread per voxel: + fix cluster, covariance, fp64 Jacobi eigensolve
//                       (SelfAdjointEigenSolver, voxel_map.hpp:264-268), store of pcr_add / eig_values / eig_vectors (:271-273) and
//                       coe * lambda_0 (:275), while the producer is already filling the stages with the next batch.
//                       Deterministic two-level reduction of the residual ("last block" pattern).
//
// Algorithmic bytes (SURVEY.md 8d): (k+1) * 80 B read + 176 B written per voxel; nothing is re-read: the summed cluster never goes
// back to HBM before the eigensolve.
#include <algorithm>
#include <cstdlib>
#include "vxs_factor_view.cuh"
#include "vxs_pipe.cuh"

// TE = entries per tile = consumer threads of a CTA (one per entry); + one producer warp.  Smaller CTAs, several per SM, overlap one CTA's
// reduction / eigensolve phases with another's transform phase (the phases of one CTA run in lock step).
#define RS_TE 256
#define RS_PER_SM 3                      // CTAs per SM the batches are cut for and the shared memory is budgeted for
#define RS_STAGES 2                      // stages of the bulk-copy ring
#define RS_COLPAD 2                      // doubles of padding between the columns of a stage (bank spread for phase B)
#define RS_COL (RS_TE + RS_COLPAD)
#define RS_STAGE_BYTES (10 * RS_COL * 8 + RS_TE * 4)

struct ResidPlan { int V, VB, nbatch, vbcap; };   // vbcap = VB rounded up to 8: sizes the accumulators / ptr window in shared memory

// SP: the poses are staged in shared memory ([12][W], see load_pose_s) instead of read from global memory; only their source differs
template <bool SP>
__global__ void __launch_bounds__(RS_TE + 32) k_residual_stream(FactorView f, const double* __restrict__ poses, int pstride, ResidPlan pl, double* __restrict__ partial,
                                                                unsigned int* __restrict__ counter, double* __restrict__ result, double* __restrict__ rvox) {
  constexpr int RS_CONS = RS_TE, RS_THREADS = RS_TE + 32;
  extern __shared__ __align__(128) unsigned char rs_smem[];
  __shared__ int s_va[2], s_vb[2];   // by tile parity: a fast warp writes the next tile's values while a slow one still reads this tile's
  // layout: stages | acc[vbcap][10] | sp_ptr[vbcap + 8] | red[RS_CONS] | barriers | poses [12][W]
  unsigned char* stage_base = rs_smem;
  double* acc = reinterpret_cast<double*>(rs_smem + size_t(RS_STAGES) * RS_STAGE_BYTES);
  int* sp_ptr = reinterpret_cast<int*>(acc + pl.vbcap * 10);
  double* red = reinterpret_cast<double*>(sp_ptr + pl.vbcap + 8);
  uint64_t* full = reinterpret_cast<uint64_t*>(red + RS_CONS);
  uint64_t* empty = full + RS_STAGES;
  double* sp = reinterpret_cast<double*>(empty + RS_STAGES);
  __shared__ bool is_last;

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < RS_STAGES; s++) { mbar_init(full + s, 1); mbar_init(empty + s, RS_CONS / 32); }
    mbar_fence_init();
  }
  if (SP) { for (int i = tid; i < 12 * f.W; i += RS_THREADS) { const int fr = i / 12, c = i - fr * 12; sp[c * f.W + fr] = __ldg(poses + size_t(fr) * pstride + c); } }
  __syncthreads();

  // this CTA's batches: [b0, b1), batch b = voxels [b * VB, min(V, (b + 1) * VB))
  const int b0 = int((long long)pl.nbatch * blockIdx.x / gridDim.x), b1 = int((long long)pl.nbatch * (blockIdx.x + 1) / gridDim.x);

  if (tid >= RS_CONS) {
    // ------------------------------------------------------------ producer warp (one lane issues; the others idle until the end)
    if (tid == RS_CONS) {
      unsigned int tc = 0;   // running tile counter of this CTA
      for (int b = b0; b < b1; b++) {
        const int vb0 = b * pl.VB, vb1 = min(pl.V, vb0 + pl.VB);
        const int B0 = __ldg(f.ptr + vb0), B1 = __ldg(f.ptr + vb1);
        const int A0 = B0 & ~3, Bend = (B1 + 3) & ~3;
        for (int t0 = A0; t0 < B1; t0 += RS_TE, tc++) {
          const int s = int(tc % unsigned(RS_STAGES));
          const unsigned int ph = (tc / unsigned(RS_STAGES)) & 1u;
          mbar_wait(empty + s, ph ^ 1u);
          const int cnt = min(RS_TE, Bend - t0);          // multiple of 4 entries: 32-B multiples for the fp64 columns, 16-B for the frames
          unsigned char* st = stage_base + size_t(s) * RS_STAGE_BYTES;
          mbar_arrive_expect_tx(full + s, unsigned(cnt) * 84u);
#pragma unroll
          for (int c = 0; c < 10; c++) bulk_g2s(st + size_t(c) * RS_COL * 8, f.cl + size_t(c) * f.Ecap + t0, unsigned(cnt) * 8u, full + s);
          bulk_g2s(st + size_t(10) * RS_COL * 8, f.frame + t0, unsigned(cnt) * 4u, full + s);
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers
    const int lane = tid & 31;
    unsigned int tc = 0;
    double rsum = 0.0;
    for (int b = b0; b < b1; b++) {
      const int vb0 = b * pl.VB, vb1 = min(pl.V, vb0 + pl.VB), nv = vb1 - vb0;
      for (int i = tid; i <= nv; i += RS_CONS) sp_ptr[i] = f.ptr[vb0 + i];
      for (int i = tid; i < nv * 10; i += RS_CONS) acc[i] = 0.0;
      named_bar_sync(1, RS_CONS);
      const int B0 = sp_ptr[0], B1 = sp_ptr[nv];
      const int A0 = B0 & ~3;
      for (int t0 = A0; t0 < B1; t0 += RS_TE, tc++) {
        const int s = int(tc % unsigned(RS_STAGES));
        const unsigned int ph = (tc / unsigned(RS_STAGES)) & 1u;
        double* col = reinterpret_cast<double*>(stage_base + size_t(s) * RS_STAGE_BYTES);
        const int* frs = reinterpret_cast<const int*>(col + 10 * RS_COL);
        if (lane == 0) mbar_wait(full + s, ph);      // one lane polls (a polling warp costs issue slots the working warps need), the rest of the warp parks at the warp barrier
        __syncwarp();
        // ---- phase A: transform the entry in place
        const int e = t0 + tid;
        if (e >= B0 && e < B1) {
          cluster c;
          c.P.xx = col[tid]; c.P.xy = col[RS_COL + tid]; c.P.xz = col[2 * RS_COL + tid]; c.P.yy = col[3 * RS_COL + tid]; c.P.yz = col[4 * RS_COL + tid]; c.P.zz = col[5 * RS_COL + tid];
          c.v = mk3(col[6 * RS_COL + tid], col[7 * RS_COL + tid], col[8 * RS_COL + tid]); c.n = col[9 * RS_COL + tid];
          rot3 R; d3 t;
          if (SP) load_pose_s(sp, f.W, frs[tid], R, t); else load_pose(poses, pstride, frs[tid], R, t);
          cluster o;
          o.P.xx = o.P.xy = o.P.xz = o.P.yy = o.P.yz = o.P.zz = 0.0; o.v = mk3(0, 0, 0); o.n = 0.0;
          cluster_transform_acc(c, R, t, o);
          col[tid] = o.P.xx; col[RS_COL + tid] = o.P.xy; col[2 * RS_COL + tid] = o.P.xz; col[3 * RS_COL + tid] = o.P.yy; col[4 * RS_COL + tid] = o.P.yz; col[5 * RS_COL + tid] = o.P.zz;
          col[6 * RS_COL + tid] = o.v.x; col[7 * RS_COL + tid] = o.v.y; col[8 * RS_COL + tid] = o.v.z; col[9 * RS_COL + tid] = o.n;
        }
        // first / last voxel of the batch with entries in this tile: the thread of voxel j tests its own range (exactly one hit each)
        const int tlo = max(B0, t0), thi = min(B1, t0 + RS_TE);
        for (int j = tid; j < nv; j += RS_CONS) {
          const int p0 = sp_ptr[j], p1 = sp_ptr[j + 1];
          if (p0 <= tlo && tlo < p1) s_va[tc & 1u] = j;
          if (p0 <= thi - 1 && thi - 1 < p1) s_vb[tc & 1u] = j;
        }
        named_bar_sync(1, RS_CONS);
        // ---- phase B: per (voxel, component, quarter) fixed-order partial sums of the tile into the batch accumulators
        const int va = s_va[tc & 1u], vbv = s_vb[tc & 1u];
        const int total = (vbv - va + 1) * 40;
        for (int base = 0; base < total; base += RS_CONS) {
          const int idx = base + tid;
          const bool ok = idx < total;              // total is a multiple of 4 and tid's quad is aligned: a quad is valid or not as a whole
          double sacc = 0.0;
          int v = 0, cc = 0, q = 0;
          if (ok) {
            const int vi = idx / 40, r = idx - vi * 40;
            cc = r >> 2; q = r & 3; v = va + vi;
            const int lo = max(sp_ptr[v], tlo), hi = min(sp_ptr[v + 1], thi), len = max(hi - lo, 0);
            const int qlo = lo + ((len * q) >> 2), qhi = lo + ((len * (q + 1)) >> 2);
            const double* src = col + cc * RS_COL - t0;
            for (int j = qlo; j < qhi; j++) sacc += src[j];
          }
          sacc += __shfl_xor_sync(0xffffffffu, sacc, 1);
          sacc += __shfl_xor_sync(0xffffffffu, sacc, 2);
          if (ok && q == 0) acc[v * 10 + cc] += sacc;
        }
        // the stage is rewritten by the async proxy next: order this thread's generic writes (phase A) before it, then release the stage
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + s);
        // phase B of the next tile must not start before everybody's phase B of this one is done with `acc`: the barrier after the next phase A orders them
      }
      named_bar_sync(1, RS_CONS);
      // ---- per voxel: + fix, covariance, eigensolve, cache, residual   (voxel_map.hpp:255, 264-275)
      if (tid < nv) {
        const int v = vb0 + tid;
        const size_t st = f.Vcap;
        cluster sg;
        const double* a = acc + tid * 10;
        sg.P.xx = a[0]; sg.P.xy = a[1]; sg.P.xz = a[2]; sg.P.yy = a[3]; sg.P.yz = a[4]; sg.P.zz = a[5]; sg.v = mk3(a[6], a[7], a[8]); sg.n = a[9];
        if (f.has_fix) {
          const cluster fx = load_cluster_soa(f.fix, st, size_t(v));
          sg.P.xx += fx.P.xx; sg.P.xy += fx.P.xy; sg.P.xz += fx.P.xz; sg.P.yy += fx.P.yy; sg.P.yz += fx.P.yz; sg.P.zz += fx.P.zz; sg.v = sg.v + fx.v; sg.n += fx.n;
        }
        double* so = f.sum + v;
        so[0] = sg.P.xx; so[st] = sg.P.xy; so[2 * st] = sg.P.xz; so[3 * st] = sg.P.yy; so[4 * st] = sg.P.yz; so[5 * st] = sg.P.zz;
        so[6 * st] = sg.v.x; so[7 * st] = sg.v.y; so[8 * st] = sg.v.z; so[9 * st] = sg.n;
        double w[3]; d3 u0, u1, u2;
        eig3_jacobi(cov_from_sum(sg), w, u0, u1, u2);
        double* eo = f.eig + v;
        eo[0] = w[0]; eo[st] = w[1]; eo[2 * st] = w[2];
        eo[3 * st] = u0.x; eo[4 * st] = u1.x; eo[5 * st] = u2.x; eo[6 * st] = u0.y; eo[7 * st] = u1.y; eo[8 * st] = u2.y; eo[9 * st] = u0.z; eo[10 * st] = u1.z; eo[11 * st] = u2.z;
        const double contrib = f.coe[v] * w[0];
        if (rvox) rvox[v] = contrib;              // per-voxel residual for the per-window sums of a batch (vxs_hba_bottom_batch)
        rsum += contrib;
      }
      named_bar_sync(1, RS_CONS);   // acc / sp_ptr are re-initialised for the next batch
    }
    red[tid] = rsum;
  }
  __syncthreads();
  // ---- deterministic block + grid reduction (fixed tree; the last CTA adds the per-CTA partials in index order)
  for (int s = RS_CONS / 2; s > 0; s >>= 1) { if (tid < s) red[tid] += red[tid + s]; __syncthreads(); }
  if (tid == 0) {
    partial[blockIdx.x] = red[0];
    __threadfence();
    const unsigned int t = atomicAdd(counter, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    double a = 0.0;
    if (tid < RS_CONS) { for (unsigned int i = tid; i < gridDim.x; i += RS_CONS) a += __ldcg(partial + i); red[tid] = a; }
    __syncthreads();
    for (int s = RS_CONS / 2; s > 0; s >>= 1) { if (tid < s) red[tid] += red[tid + s]; __syncthreads(); }
    if (tid == 0) { result[0] = red[0]; *counter = 0u; }
  }
}

// Launch shapes tried at the metric shape before the H100 port (us), TE x CTAs/SM x stages: 512 x 1 x 4: 98; 256 x 2 x 4: 81-85; 128 x 4 x 3: 79-81; 256 x 3 x 2: 76 (this one);
// 128 x 6 x 2: 99.  The bulk copies need 16-B aligned columns: vxs_factor_reserve keeps Ecap a multiple of 32.  Needs f->V > 0.
int vxs_residual_stream_launch(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pstride, double* residual_dev, double* rvox) {
  const int G = ctx->sm_count * RS_PER_SM;
  // batches: about 96 voxels each, an equal number per CTA
  const long long V = f->V;
  long long m = std::max<long long>(1, (V + (long long)G * 48) / ((long long)G * 96));
  long long VB = (V + (long long)G * m - 1) / ((long long)G * m);
  while (VB > RS_TE) { m++; VB = (V + (long long)G * m - 1) / ((long long)G * m); }
  VB = std::max<long long>(VB, 1);
  ResidPlan pl; pl.V = int(V); pl.VB = int(VB); pl.nbatch = int((V + VB - 1) / VB); pl.vbcap = int((VB + 7) & ~7ll);
  const size_t smem_gmem_poses = size_t(RS_STAGES) * RS_STAGE_BYTES + size_t(pl.vbcap) * 80 + size_t(pl.vbcap + 8) * 4 + size_t(RS_TE) * 8 + 2 * RS_STAGES * 8 + 128;
  const size_t budget = size_t(ctx->smem_optin) / RS_PER_SM - 1024;   // per-CTA share (1 KB per CTA is reserved by the driver)
  // the pose table goes to shared memory when it fits next to the rest (W <= 195 always does); otherwise the poses are read from global memory,
  // a plan that needs at most 57 664 B (VB <= 144) of the 76 458 B an H100 CTA gets
  const bool sp = smem_gmem_poses + size_t(12) * f->W * 8 <= budget;
  if (!sp && smem_gmem_poses > budget) return vxs_fail(ctx, VXS_ERR_CUDA, "k_residual_stream: not enough shared memory per CTA on this device");
  const size_t smem = smem_gmem_poses + (sp ? size_t(12) * f->W * 8 : 0);
  const unsigned grid = unsigned(std::min<long long>(G, pl.nbatch));
  VXS_CUDA(ctx, f->partial.reserve(std::max<size_t>(size_t(grid), size_t((V + 255) / 256))));
  if (!f->counter.p) { VXS_CUDA(ctx, f->counter.reserve(4)); VXS_CUDA(ctx, cudaMemsetAsync(f->counter.p, 0, 16, ctx->stream)); }
  FactorView fv = make_view(f);
  auto kp = sp ? k_residual_stream<true> : k_residual_stream<false>;
  VXS_CUDA(ctx, cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  VXS_LAUNCH(ctx, "k_residual_stream", kp, grid, RS_TE + 32, smem, fv, poses_dev, pstride, pl, f->partial.p, f->counter.p, residual_dev, rvox);
  return VXS_OK;
}
