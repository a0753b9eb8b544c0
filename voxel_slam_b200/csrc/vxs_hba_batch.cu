// Bottom level of the hierarchical global BA as ONE batch (SURVEY.md §8a12 / §8e(1)): thd_globalmapping calls HBA_add_edge(xs, smp_local, gba_edges1,
// mps, max_iter = 1, thread_num = 2, plptr) once per 10-keyframe window, stride 5 (voxelslam.cpp:2484-2557) — hundreds of independent 60-dof problems,
// each ~11 launches of 10-40 us per LM iteration when run one at a time.  Here a chunk of windows is ONE problem:
//   * one map build over the chunk's clouds (vxs_voxelize.cu, batch mode: every window owns a private copy of the cell space, so
//     OctreeGBA::cut_voxel + OctreeGBA_multi_recut, loop_refine.hpp:446-537, of all windows are the same sort / segment passes);
//   * Lidar_BA_Optimizer::damping_iter (voxel_map.hpp:367-442) for all windows in lock step, entirely on the device: block-diagonal Hessian
//     (k_jac + k_pairs_bd), one CTA per window for assembly + gauge fix + Eigen-ordered LDL^T of the 6W system in shared memory + retraction,
//     the streaming residual kernel over all voxels with per-voxel output, deterministic per-window sums, one thread per window for the
//     accept / reject bookkeeping.  No host synchronisation inside the `up` = 4 iterations;
//   * PGO edges of every window from its raw Hessian (voxelslam.cpp:2405-2427).
// The reference's outer loop runs exactly once for max_iter = 1 (iterCnt == max_iter - 1 switches to the fine parameters, :2362-2372), which is
// what the bottom level uses; other max_iter values go through vxs_hba_window one window at a time.
#include <algorithm>
#include <cstring>
#include <vector>
#include "vxs_internal.h"
#include "vxs_math.cuh"
#include "vxs_sortscan.cuh"

using namespace vxs;

// vxs_voxelize.cu
int vxs_build_gba_batch(vxs_ctx* ctx, const vxs_map_params* mp, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, const int32_t* win_first, int nwin,
                        int win_size, int kf_lo, int kf_hi, vxs_factor* out, const float* xyz_dev, int64_t dev_first_point);
int vxs_submap_merge_batch_impl(vxs_ctx* ctx, const float* xyz, const float* xyz_dev, int64_t dev_first_point, int stride_floats, const int64_t* kf_offsets, int K, const double* poses_win,
                                const int32_t* win_first, int nwin, int win_size, double voxel_size, int64_t max_points_per_chunk, float* xyz_out, float* count_out,
                                int64_t* first_index_out, int64_t cap, int64_t* win_offsets, int64_t* n_out, DevBuf<float>* dev_out);
int vxs_hba_window_impl(vxs_ctx* ctx, const vxs_map_params* coarse, const vxs_map_params* fine, const float* xyz, const float* xyz_dev, int stride_floats, const int64_t* kf_offsets,
                        double* poses12, int W, int max_iter, int thread_num, double* hess_out, double* resis_log, int* outer_iters, long long own_lo, long long own_hi);
int vxs_hba_top_routed(vxs_ctx* ctx, const vxs_map_params* coarse, const vxs_map_params* fine, const float* sub_mine, const int64_t* woff_host, int first_window, int nmine, int nwin,
                       double* poses12, int max_iter, int thread_num, double* resis_log, int* outer_iters, DevBuf<float>* sendbuf, DevBuf<float>* recvbuf);
int vxs_comm_allgatherv_f32(vxs_ctx* ctx, const float* mine, size_t my_count, float* all, const size_t* counts, const size_t* displs, float* pad, size_t slot);   // vxs_lm.cu

namespace {

#define HB_MAXN 96   // 6 * win_size <= 96 (win_size <= 16)

struct BdState {     // per-window LM state, SoA on the device
  double* x; double* xt;          // [nwin][WB][12]
  double* u; double* v; double* r1; double* r2; double* q1; double* resis;   // resis [nwin][2]
  int* calc; int* conv; int* done; int* iters; int* status; int* nvox;
  double* Hraw; double* dx;       // [nwin][n*n], [nwin][n]
};

__global__ void __launch_bounds__(256) k_bd_lambda(const double* __restrict__ eig, const double* __restrict__ coe, int V, double* __restrict__ rvox) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) rvox[v] = coe[v] * eig[v];          // residual += coe * lmbd[kk] from the cached eigenvalues (voxel_map.hpp:234)
}
// deterministic per-window sum of the per-voxel residuals (voxels of a window through the CSR built once per map)
__global__ void __launch_bounds__(128) k_bd_winsum(const double* __restrict__ rvox, const int* __restrict__ win_ptr, const unsigned int* __restrict__ win_vox, const int* __restrict__ mask, int use_calc,
                                                   double* __restrict__ out) {
  const int w = blockIdx.x;
  if (mask && ((use_calc && !mask[w]) || (!use_calc && mask[w]))) return;    // use_calc: only windows that rebuild (mask = calc); else: skip done windows (mask = done)
  __shared__ double sh[128];
  double a = 0.0;
  for (int i = win_ptr[w] + threadIdx.x; i < win_ptr[w + 1]; i += 128) a += rvox[win_vox[i]];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 64; s > 0; s >>= 1) { if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s]; __syncthreads(); }
  if (threadIdx.x == 0) out[w] = sh[0];
}

// One CTA per window: assemble the 6W x 6W system of a fresh build, gauge fix, D = diag, M = H + u D, Eigen's pivot order (descending |D|),
// LDL^T, solve, retraction, q1.      voxel_map.hpp:391-409
__global__ void __launch_bounds__(128) k_bd_solve(BdState S, const double* __restrict__ Cbd, const double* __restrict__ gD, int WB, int nwin) {
  const int w = blockIdx.x, tid = threadIdx.x;
  if (S.done[w]) return;
  const int n = 6 * WB, Wt = nwin * WB;
  extern __shared__ double sm[];
  double* M = sm;                        // [n][n + 1] row-major, permuted
  double* Dg = M + n * (n + 1);          // [n] diagonal of the gauge-fixed H
  double* rhs = Dg + n;                  // [n] -JacT (gauged), then the solution
  double* y = rhs + n;                   // [n] permuted work vector
  int* perm = reinterpret_cast<int*>(y + n);
  double* Hr = S.Hraw + size_t(w) * n * n;
  if (S.calc[w]) {
    // Hess from the block accumulators: upper block triangle of C + block-diagonal D, mirrored (voxel_map.hpp:237-239); JacT = g
    const double* C = Cbd + size_t(w) * n * n;
    const double* g = gD + size_t(w) * WB * 6;
    const double* Db = gD + size_t(Wt) * 6 + size_t(w) * WB * 24;
    for (int idx = tid; idx < n * n; idx += 128) {
      const int row = idx % n, col = idx / n;
      const int fi = row / 6, a = row - 6 * fi, fj = col / 6, b = col - 6 * fj;
      double val;
      if (fi < fj) val = C[size_t(6 * fj + b) * n + 6 * fi + a];
      else if (fi > fj) val = C[size_t(6 * fi + a) * n + 6 * fj + b];
      else {
        val = C[size_t(6 * fi + b) * n + 6 * fi + a];
        const double* D = Db + fi * 24;
        if (a < 3 && b < 3) val += D[3 * a + b];
        else if (a < 3) val += D[9 + 3 * a + (b - 3)];
        else if (b < 3) val += D[9 + 3 * b + (a - 3)];
        else { const int p = a - 3, q = b - 3, lo = p < q ? p : q, hi = p < q ? q : p; val += D[18 + (lo == 0 ? hi : (lo == 1 ? 2 + hi : 5))]; }
      }
      Hr[idx] = val;                     // raw (pre-gauge) Hessian of the last build: *hess (:391)
    }
    __syncthreads();
  }
  // gauge: first 6 rows / columns zero, identity block, JacT.head(6) = 0 (:397-400).  JacT = g of the last build: without a rebuild (after a
  // reject, :433) the accumulators still hold it, as the reference's JacT does
  __shared__ double jact_s[HB_MAXN];
  { const double* g = gD + size_t(w) * WB * 6; for (int k = tid; k < n; k += 128) jact_s[k] = g[k]; }
  __syncthreads();
  for (int k = tid; k < n; k += 128) { Dg[k] = k < 6 ? 1.0 : Hr[size_t(k) * n + k]; rhs[k] = k < 6 ? 0.0 : -jact_s[k]; }
  __syncthreads();
  // Eigen's LDLT pivots on the largest remaining ORIGINAL diagonal entry: a fixed permutation by descending |diag| of M = H + u D (ties by index)
  const double u = S.u[w];
  for (int k = tid; k < n; k += 128) {
    const double ak = fabs(Dg[k] + u * Dg[k]);
    int rank = 0;
    for (int j = 0; j < n; j++) { const double aj = fabs(Dg[j] + u * Dg[j]); rank += (aj > ak) || (aj == ak && j < k); }
    perm[rank] = k;
  }
  __syncthreads();
  for (int idx = tid; idx < n * n; idx += 128) {
    const int i = idx / n, j = idx - i * n;
    const int r = perm[i], c = perm[j];
    double val = (r < 6 || c < 6) ? ((r == c) ? 1.0 : 0.0) : Hr[size_t(c) * n + r];
    if (r == c) val += u * Dg[r];
    M[i * (n + 1) + j] = val;
  }
  for (int k = tid; k < n; k += 128) y[k] = rhs[perm[k]];
  __syncthreads();
  // right-looking LDL^T in place (lower triangle: L, diagonal: d), thread i owns row i
  __shared__ int sing;
  if (tid == 0) sing = 0;
  for (int k = 0; k < n; k++) {
    const double dk = M[k * (n + 1) + k];
    const double rk = dk != 0.0 ? 1.0 / dk : 0.0;
    if (tid == 0 && dk == 0.0) sing = 1;
    __syncthreads();
    if (tid > k && tid < n) {
      const double lik = M[tid * (n + 1) + k] * rk;
      for (int j = k + 1; j <= tid; j++) M[tid * (n + 1) + j] -= lik * M[j * (n + 1) + k];     // M[j][k] is still the unscaled column k (row j writes only its own row)
    }
    __syncthreads();
    if (tid > k && tid < n) M[tid * (n + 1) + k] *= rk;
    __syncthreads();
  }
  // forward L z = P b, D, backward L^T x = z   (sequential over k, parallel over rows)
  for (int k = 0; k < n; k++) {
    const double yk = y[k];
    __syncthreads();
    if (tid > k && tid < n) y[tid] -= M[tid * (n + 1) + k] * yk;
    __syncthreads();
  }
  for (int k = tid; k < n; k += 128) { const double d = M[k * (n + 1) + k]; y[k] = d != 0.0 ? y[k] / d : 0.0; }
  __syncthreads();
  for (int k = n - 1; k >= 0; k--) {
    const double yk = y[k];
    __syncthreads();
    if (tid < k) y[tid] -= M[k * (n + 1) + tid] * yk;
    __syncthreads();
  }
  for (int k = tid; k < n; k += 128) S.dx[size_t(w) * n + perm[k]] = y[k];
  __syncthreads();
  if (tid == 0 && sing && S.status[w] == 0) S.status[w] = VXS_WARN_SINGULAR;
  // x_temp = x [+] dx (:405-409), q1 = 0.5 dx . (u D dx - JacT) (:411)
  const double* dx = S.dx + size_t(w) * n;
  if (tid < WB) {
    const double* s = S.x + (size_t(w) * WB + tid) * 12; double* o = S.xt + (size_t(w) * WB + tid) * 12; const double* d = dx + 6 * tid;
    const rot3 Rn = rot_mul(load_rot(s), so3_exp(mk3(d[0], d[1], d[2])));
    o[0] = Rn.r00; o[1] = Rn.r01; o[2] = Rn.r02; o[3] = Rn.r10; o[4] = Rn.r11; o[5] = Rn.r12; o[6] = Rn.r20; o[7] = Rn.r21; o[8] = Rn.r22;
    for (int k = 0; k < 3; k++) o[9 + k] = s[9 + k] + d[3 + k];
  }
  if (tid == 0) {
    double q1 = 0.0;
    for (int k = 0; k < n; k++) q1 += dx[k] * (u * Dg[k] * dx[k] + rhs[k]);
    S.q1[w] = 0.5 * q1;
  }
}

// accept / reject bookkeeping of one LM iteration, one thread per window (:412-438)
__global__ void __launch_bounds__(128) k_bd_accept(BdState S, int nwin, int WB, int max_iter, int thd_num) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nwin || S.done[w]) return;
  if (S.nvox[w] < thd_num) {     // "Too Less Voxel" exit(0), voxel_map.hpp:345-348: damping_iter has recorded r1 and returns false
    S.resis[2 * w] = S.r1[w]; S.conv[w] = 0; S.status[w] = VXS_ERR_TOO_FEW_VOXELS; S.done[w] = 1; return;
  }
  const double r1 = S.r1[w], r2 = S.r2[w];
  if (S.iters[w] == 0) S.resis[2 * w] = r1;
  double q = r1 - r2;
  if (q > 0) {
    for (int k = 0; k < WB * 12; k++) S.x[size_t(w) * WB * 12 + k] = S.xt[size_t(w) * WB * 12 + k];
    const double one_three = 1.0 / 3;
    q = q / S.q1[w]; S.v[w] = 2; q = 1 - pow(2 * q - 1, 3);
    S.u[w] *= (q < one_three ? one_three : q);
    S.calc[w] = 1;
  } else { S.u[w] = S.u[w] * S.v[w]; S.v[w] = 2 * S.v[w]; S.calc[w] = 0; S.conv[w] = 0; }
  S.resis[2 * w + 1] = r2;
  S.iters[w] += 1;
  if (fabs((r1 - r2) / r1) < 1e-6 || S.iters[w] >= max_iter) { S.done[w] = 1; S.calc[w] = 0; }      // *hess stays the Hessian of the last build
}
// poses of all windows for the kernels that index poses by global frame: [nwin * WB][12] is exactly the layout of x / xt — nothing to do.

// PGO edges of every window (voxelslam.cpp:2405-2427): pair p = (i, j) in lexicographic order; valid when the six diagonal entries of block (i, j) are >= 1e-6
__global__ void __launch_bounds__(128) k_bd_edges(BdState S, int WB, int npairs, int* __restrict__ valid, double* __restrict__ v6, double* __restrict__ rot, double* __restrict__ tra) {
  const int w = blockIdx.x, n = 6 * WB;
  const double* H = S.Hraw + size_t(w) * n * n;
  for (int p = threadIdx.x; p < npairs; p += blockDim.x) {
    int i = 0, rem = p;
    while (rem >= WB - 1 - i) { rem -= WB - 1 - i; i++; }
    const int j = i + 1 + rem;
    bool ok = true; double vv[6];
    for (int k = 0; k < 6; k++) { const double hc = fabs(H[size_t(6 * j + k) * n + 6 * i + k]); if (hc < 1e-6) { ok = false; break; } vv[k] = 1.0 / hc; }
    const size_t o = size_t(w) * npairs + p;
    valid[o] = ok ? 1 : 0;
    if (!ok) continue;
    for (int k = 0; k < 6; k++) v6[o * 6 + k] = vv[k];
    const double* pi = S.x + (size_t(w) * WB + i) * 12; const double* pj = S.x + (size_t(w) * WB + j) * 12;
    const rot3 Ri = load_rot(pi), Rj = load_rot(pj);
    const d3 t = mulT(Ri, mk3(pj[9] - pi[9], pj[10] - pi[10], pj[11] - pi[11]));
    tra[o * 3] = t.x; tra[o * 3 + 1] = t.y; tra[o * 3 + 2] = t.z;
    const double a[9] = {Ri.r00, Ri.r01, Ri.r02, Ri.r10, Ri.r11, Ri.r12, Ri.r20, Ri.r21, Ri.r22}, b[9] = {Rj.r00, Rj.r01, Rj.r02, Rj.r10, Rj.r11, Rj.r12, Rj.r20, Rj.r21, Rj.r22};
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) rot[o * 9 + 3 * r + c] = a[r] * b[c] + a[3 + r] * b[3 + c] + a[6 + r] * b[6 + c];
  }
}

__global__ void __launch_bounds__(256) k_bd_vwin_keys(const int32_t* __restrict__ vwin, int V, unsigned long long* __restrict__ keys, unsigned int* __restrict__ idx) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V) { keys[v] = (unsigned long long)vwin[v]; idx[v] = (unsigned int)v; }
}
__global__ void __launch_bounds__(256) k_bd_win_ptr(const unsigned long long* __restrict__ skeys, int V, int nwin, int* __restrict__ win_ptr) {
  // win_ptr[w] = first position whose key >= w (binary search per window)
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w > nwin) return;
  int lo = 0, hi = V;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (skeys[mid] < (unsigned long long)w) lo = mid + 1; else hi = mid; }
  win_ptr[w] = lo;
}
__global__ void __launch_bounds__(128) k_bd_init(BdState S, const int* __restrict__ win_ptr, int nwin) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nwin) return;
  S.u[w] = 0.01; S.v[w] = 2; S.r1[w] = 0; S.r2[w] = 0; S.q1[w] = 0; S.resis[2 * w] = 0; S.resis[2 * w + 1] = 0;
  S.calc[w] = 1; S.conv[w] = 1; S.done[w] = 0; S.iters[w] = 0; S.status[w] = 0; S.nvox[w] = win_ptr[w + 1] - win_ptr[w];
}

struct BatchScratch {    // one per ctx, grow-only: a pass must not pay cudaMalloc / cudaFree of GB-sized buffers (each is a device-wide synchronisation)
  DevBuf<double> d; DevBuf<int> i; DevBuf<unsigned long long> kA, kB; DevBuf<unsigned int> iA, iB; DevBuf<double> rvox, Cbd, gD, out_d; DevBuf<int> out_i;
  SortScratch ss;
  DevBuf<float> pts, sub_mine, sub_all, sub_pad;   // vxs_hba_pass: this rank's keyframe clouds, its merged submaps, all ranks' submaps, the padded all-gather slots
  vxs_factor* f = nullptr;                // the chunk factor, kept between calls
  long long last_voxels = 0, last_entries = 0;   // plane voxels / (voxel, keyframe) clusters of the last bottom batch (all chunks)
};
BatchScratch* hba_scratch(vxs_ctx* c) { if (!c->hba_scratch) c->hba_scratch = new BatchScratch(); return static_cast<BatchScratch*>(c->hba_scratch); }

}  // namespace

void vxs_hba_release(vxs_ctx* c) {
  if (!c->hba_scratch) return;
  BatchScratch* B = static_cast<BatchScratch*>(c->hba_scratch);
  B->d.release(); B->i.release(); B->kA.release(); B->kB.release(); B->iA.release(); B->iB.release(); B->rvox.release(); B->Cbd.release(); B->gD.release(); B->out_d.release();
  B->out_i.release(); B->ss.hist.release(); B->ss.blocksums.release(); B->ss.totals.release(); B->pts.release(); B->sub_mine.release(); B->sub_all.release(); B->sub_pad.release();
  // B->f is owned by the ctx's factor list (released with it)
  delete B;
  c->hba_scratch = nullptr;
}

static int hba_bottom_batch_impl(vxs_ctx* ctx, const vxs_map_params* fine, const float* xyz, const float* xyz_dev, int64_t dev_first_point, int stride_floats, const int64_t* kf_offsets,
                                 const double* poses12, int K, const int32_t* win_first, int nwin, int win_size, int thread_num, int64_t max_points_per_chunk, double* poses_out, double* resis,
                                 int32_t* status, int32_t* is_converge, int32_t* lm_iters, int32_t* edge_valid, double* edge_v6, double* edge_rot, double* edge_tra, double* hess_out) {
  if (!ctx || !fine || !xyz || !kf_offsets || !poses12 || !win_first || K <= 0 || nwin <= 0 || win_size < 2 || 6 * win_size > HB_MAXN || stride_floats < 3 || !poses_out) return VXS_ERR_ARG;
  for (int w = 0; w < nwin; w++) if (win_first[w] < 0 || win_first[w] + win_size > K) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_hba_bottom_batch: a window reaches beyond the keyframes");
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int WB = win_size, n = 6 * WB, npairs = WB * (WB - 1) / 2, up = 4;
  if (max_points_per_chunk <= 0) max_points_per_chunk = 96ll << 20;
  BatchScratch& B = *hba_scratch(ctx);
  int rc = VXS_OK;
  if (!B.f) { rc = vxs_factor_create(ctx, WB, &B.f); if (rc) return rc; }
  vxs_factor* f = B.f;
  int warn = VXS_OK;
  B.last_voxels = 0; B.last_entries = 0;
  for (int w0 = 0; w0 < nwin;) {
    // ---- chunk of windows bounded by its number of (virtual) points
    int w1 = w0; int64_t vp = 0;
    while (w1 < nwin) {
      const int64_t np = kf_offsets[win_first[w1] + WB] - kf_offsets[win_first[w1]];
      if (w1 > w0 && vp + np > max_points_per_chunk) break;
      vp += np; w1++;
    }
    const int nw = w1 - w0;
    int kf_lo = K, kf_hi = 0;
    for (int w = w0; w < w1; w++) { kf_lo = std::min(kf_lo, int(win_first[w])); kf_hi = std::max(kf_hi, int(win_first[w]) + WB); }
    rc = vxs_build_gba_batch(ctx, fine, xyz, stride_floats, kf_offsets, poses12, win_first + w0, nw, WB, kf_lo, kf_hi, f, xyz_dev, dev_first_point);
    if (rc < 0) return rc;
    const int V = int(f->V);
    B.last_voxels += f->V; B.last_entries += f->E;
    // ---- per-window state
    const size_t nd = size_t(nw) * WB * 12 * 2 + size_t(nw) * 7 + size_t(nw) * n * n + size_t(nw) * n;
    VXS_CUDA(ctx, B.d.reserve(nd)); VXS_CUDA(ctx, B.i.reserve(size_t(nw) * 6 + size_t(nw) + 2));
    BdState S;
    double* p = B.d.p;
    S.x = p; p += size_t(nw) * WB * 12; S.xt = p; p += size_t(nw) * WB * 12; S.u = p; p += nw; S.v = p; p += nw; S.r1 = p; p += nw; S.r2 = p; p += nw; S.q1 = p; p += nw; S.resis = p; p += 2 * nw;
    S.Hraw = p; p += size_t(nw) * n * n; S.dx = p;
    int* q = B.i.p;
    S.calc = q; q += nw; S.conv = q; q += nw; S.done = q; q += nw; S.iters = q; q += nw; S.status = q; q += nw; S.nvox = q; q += nw;
    int* win_ptr = q;
    std::vector<double> xs(size_t(nw) * WB * 12);
    for (int w = 0; w < nw; w++) memcpy(xs.data() + size_t(w) * WB * 12, poses12 + size_t(win_first[w0 + w]) * 12, size_t(WB) * 96);
    VXS_CUDA(ctx, cudaMemcpyAsync(S.x, xs.data(), xs.size() * 8, cudaMemcpyHostToDevice, st));
    VXS_CUDA(ctx, cudaMemcpyAsync(S.xt, xs.data(), xs.size() * 8, cudaMemcpyHostToDevice, st));
    VXS_CUDA(ctx, cudaMemsetAsync(S.Hraw, 0, size_t(nw) * n * n * 8, st));
    // ---- voxels by window (CSR), once per map
    unsigned int* win_vox = nullptr;
    if (V > 0) {
      VXS_CUDA(ctx, B.kA.reserve(size_t(V))); VXS_CUDA(ctx, B.kB.reserve(size_t(V))); VXS_CUDA(ctx, B.iA.reserve(size_t(V))); VXS_CUDA(ctx, B.iB.reserve(size_t(V)));
      VXS_CUDA(ctx, B.ss.totals.reserve(16));
      VXS_LAUNCH(ctx, "k_bd_vwin_keys", k_bd_vwin_keys, unsigned((V + 255) / 256), 256, 0, (const int32_t*)f->vwin.p, V, B.kA.p, B.iA.p);
      unsigned long long* ks; unsigned int* vs;
      rc = radix_sort(ctx, &B.ss, B.kA.p, B.iA.p, B.kB.p, B.iB.p, size_t(V), bits_for((unsigned long long)nw), &ks, &vs);
      if (rc) return rc;
      win_vox = vs;
      VXS_LAUNCH(ctx, "k_bd_win_ptr", k_bd_win_ptr, unsigned((nw + 256) / 256), 256, 0, ks, V, nw, win_ptr);
    } else VXS_CUDA(ctx, cudaMemsetAsync(win_ptr, 0, size_t(nw + 1) * 4, st));
    VXS_LAUNCH(ctx, "k_bd_init", k_bd_init, unsigned((nw + 127) / 128), 128, 0, S, (const int*)win_ptr, nw);
    VXS_CUDA(ctx, B.rvox.reserve(size_t(std::max(V, 1))));
    VXS_CUDA(ctx, B.Cbd.reserve(size_t(nw) * n * n)); VXS_CUDA(ctx, B.gD.reserve(size_t(nw) * WB * 30));
    const size_t smem = (size_t(n) * (n + 1) + 3 * size_t(n)) * 8 + size_t(n) * 4 + 16;
    VXS_CUDA(ctx, cudaFuncSetAttribute(k_bd_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    // ---- Lidar_BA_Optimizer::damping_iter(xs, voxhess, &hess, resis, up) for all windows, no host synchronisation inside
    for (int it = 0; it < up && V > 0; it++) {
      rc = vxs_eval_hessian_bd_dev(ctx, f, S.x, 12, S.calc, B.Cbd.p, B.gD.p);      // windows with is_calc_hess (the others keep their accumulators)
      if (rc) return rc;
      VXS_LAUNCH(ctx, "k_bd_lambda", k_bd_lambda, unsigned((V + 255) / 256), 256, 0, (const double*)f->eig, (const double*)f->coe, V, B.rvox.p);
      VXS_LAUNCH(ctx, "k_bd_winsum", k_bd_winsum, unsigned(nw), 128, 0, (const double*)B.rvox.p, (const int*)win_ptr, (const unsigned int*)win_vox, (const int*)S.calc, 1, S.r1);
      VXS_LAUNCH(ctx, "k_bd_solve", k_bd_solve, unsigned(nw), 128, smem, S, (const double*)B.Cbd.p, (const double*)B.gD.p, WB, nw);
      rc = vxs_residual_stream_launch(ctx, f, S.xt, 12, ctx->scal.p, B.rvox.p);     // evaluate_only_residual at x_temp: overwrites the cached eig / pcr_adds (:271-273)
      if (rc) return rc;
      VXS_LAUNCH(ctx, "k_bd_winsum", k_bd_winsum, unsigned(nw), 128, 0, (const double*)B.rvox.p, (const int*)win_ptr, (const unsigned int*)win_vox, (const int*)S.done, 0, S.r2);
      VXS_LAUNCH(ctx, "k_bd_accept", k_bd_accept, unsigned((nw + 127) / 128), 128, 0, S, nw, WB, up, thread_num);
    }
    // ---- edges + read back
    VXS_CUDA(ctx, B.out_d.reserve(size_t(nw) * npairs * 18)); VXS_CUDA(ctx, B.out_i.reserve(size_t(nw) * npairs));
    double* d_v6 = B.out_d.p; double* d_rot = d_v6 + size_t(nw) * npairs * 6; double* d_tra = d_rot + size_t(nw) * npairs * 9;
    VXS_LAUNCH(ctx, "k_bd_edges", k_bd_edges, unsigned(nw), 128, 0, S, WB, npairs, B.out_i.p, d_v6, d_rot, d_tra);
    VXS_CUDA(ctx, cudaMemcpyAsync(poses_out + size_t(w0) * WB * 12, S.x, size_t(nw) * WB * 96, cudaMemcpyDeviceToHost, st));
    if (resis) VXS_CUDA(ctx, cudaMemcpyAsync(resis + 2 * size_t(w0), S.resis, size_t(nw) * 16, cudaMemcpyDeviceToHost, st));
    if (status) VXS_CUDA(ctx, cudaMemcpyAsync(status + w0, S.status, size_t(nw) * 4, cudaMemcpyDeviceToHost, st));
    if (is_converge) VXS_CUDA(ctx, cudaMemcpyAsync(is_converge + w0, S.conv, size_t(nw) * 4, cudaMemcpyDeviceToHost, st));
    if (lm_iters) VXS_CUDA(ctx, cudaMemcpyAsync(lm_iters + w0, S.iters, size_t(nw) * 4, cudaMemcpyDeviceToHost, st));
    if (edge_valid) VXS_CUDA(ctx, cudaMemcpyAsync(edge_valid + size_t(w0) * npairs, B.out_i.p, size_t(nw) * npairs * 4, cudaMemcpyDeviceToHost, st));
    if (edge_v6) VXS_CUDA(ctx, cudaMemcpyAsync(edge_v6 + size_t(w0) * npairs * 6, d_v6, size_t(nw) * npairs * 48, cudaMemcpyDeviceToHost, st));
    if (edge_rot) VXS_CUDA(ctx, cudaMemcpyAsync(edge_rot + size_t(w0) * npairs * 9, d_rot, size_t(nw) * npairs * 72, cudaMemcpyDeviceToHost, st));
    if (edge_tra) VXS_CUDA(ctx, cudaMemcpyAsync(edge_tra + size_t(w0) * npairs * 3, d_tra, size_t(nw) * npairs * 24, cudaMemcpyDeviceToHost, st));
    if (hess_out) VXS_CUDA(ctx, cudaMemcpyAsync(hess_out + size_t(w0) * n * n, S.Hraw, size_t(nw) * n * n * 8, cudaMemcpyDeviceToHost, st));
    VXS_CUDA(ctx, cudaStreamSynchronize(st));
    if (V == 0) for (int w = 0; w < nw; w++) {     // no LM iteration ran: r1 = 0 (no voxel), damping_iter returns false as above
      if (status) status[w0 + w] = VXS_ERR_TOO_FEW_VOXELS;
      if (is_converge) is_converge[w0 + w] = 0;
    }
    w0 = w1;
  }
  return warn;
}

extern "C" int vxs_hba_bottom_batch(vxs_ctx* ctx, const vxs_map_params* fine, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, int K,
                                    const int32_t* win_first, int nwin, int win_size, int thread_num, int64_t max_points_per_chunk, double* poses_out, double* resis, int32_t* status,
                                    int32_t* is_converge, int32_t* lm_iters, int32_t* edge_valid, double* edge_v6, double* edge_rot, double* edge_tra, double* hess_out) {
  return hba_bottom_batch_impl(ctx, fine, xyz, nullptr, 0, stride_floats, kf_offsets, poses12, K, win_first, nwin, win_size, thread_num, max_points_per_chunk, poses_out, resis, status,
                               is_converge, lm_iters, edge_valid, edge_v6, edge_rot, edge_tra, hess_out);
}

// One pass of the hierarchical global BA (thd_globalmapping, voxelslam.cpp:2484-2557) with everything between the keyframe clouds and the results on the device:
//   windows  w = 0 .. nwin-1 of win_size keyframes, first keyframe w * win_stride; rank r of n handles the contiguous share [nwin r / n, nwin (r+1) / n);
//   bottom   hba_bottom_batch_impl on the rank's windows (the keyframes it needs are uploaded ONCE), then the submap merge + down-sampling, output left on the device;
//   exchange the merged submaps go to every rank over NCCL (sizes by an all-reduce, clouds by grouped broadcasts), straight between device buffers;
//   top      HBA_add_edge over all submaps (W = nwin, max_iter = top_max_iter): voxel-sharded map + all-reduced Hessian + replicated solve, reading the device-resident clouds.
extern "C" int vxs_hba_pass(vxs_ctx* ctx, const vxs_map_params* coarse, const vxs_map_params* fine, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, int K,
                            int win_size, int win_stride, int bottom_thread_num, int top_thread_num, int top_max_iter, int64_t max_points_per_chunk, double* bottom_poses, double* bottom_resis,
                            int32_t* bottom_status, int32_t* bottom_edge_valid, double* bottom_edge_v6, double* bottom_edge_rot, double* bottom_edge_tra, int32_t* my_first_window,
                            int32_t* my_window_count, double* top_poses, double* top_resis_log, int* top_outer_iters, int64_t* submap_sizes, double* phase_ms) {
  if (!ctx || !coarse || !fine || !xyz || !kf_offsets || !poses12 || K <= 0 || win_size < 2 || win_stride < 1 || K < win_size || !bottom_poses || !top_poses) return VXS_ERR_ARG;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const int nwin = (K - win_size) / win_stride + 1;
  std::vector<int32_t> win_first(static_cast<size_t>(nwin));
  for (int w = 0; w < nwin; w++) win_first[size_t(w)] = w * win_stride;
  const int lo = int((long long)nwin * ctx->rank / ctx->nranks), hi = int((long long)nwin * (ctx->rank + 1) / ctx->nranks), nmine = hi - lo;
  if (my_first_window) *my_first_window = lo;
  if (my_window_count) *my_window_count = nmine;
  cudaEvent_t ev[5];
  for (auto& e : ev) cudaEventCreate(&e);
  auto cleanup = [&](int code) { for (auto& e : ev) cudaEventDestroy(e); return code; };
  BatchScratch& PB = *hba_scratch(ctx);
  DevBuf<float>& pts = PB.pts; DevBuf<float>& sub_mine = PB.sub_mine; DevBuf<float>& sub_all = PB.sub_all;
  int rc = VXS_OK;
  cudaEventRecord(ev[0], st);
  // ---- this rank's keyframes, uploaded once
  std::vector<int64_t> woff(size_t(nmine) + 1, 0);
  std::vector<double> sizes_d(static_cast<size_t>(nwin) + 1, 0.0);      // [nwin] = error flag: a rank whose bottom level failed must not leave its peers waiting in the exchange
  int my_err = 0;
  const bool multi = ctx->nranks > 1;
  if (nmine > 0) {
    const int kf_lo = win_first[size_t(lo)], kf_hi = win_first[size_t(hi) - 1] + win_size;
    const int64_t p0 = kf_offsets[kf_lo], np = kf_offsets[kf_hi] - p0;
    if (pts.reserve(size_t(std::max<int64_t>(np, 1)) * stride_floats) != cudaSuccess) {
      my_err = vxs_fail(ctx, VXS_ERR_NOMEM, "vxs_hba_pass: keyframe clouds do not fit");
      if (!multi) { return cleanup(my_err); }
    }
    if (!my_err && np > 0) cudaMemcpyAsync(pts.p, xyz + size_t(p0) * stride_floats, size_t(np) * stride_floats * 4, cudaMemcpyHostToDevice, st);
    if (!my_err) rc = hba_bottom_batch_impl(ctx, fine, xyz, pts.p, p0, stride_floats, kf_offsets, poses12, K, win_first.data() + lo, nmine, win_size, bottom_thread_num, max_points_per_chunk, bottom_poses,
                               bottom_resis, bottom_status, nullptr, nullptr, bottom_edge_valid, bottom_edge_v6, bottom_edge_rot, bottom_edge_tra, nullptr);
    if (rc < 0 && !my_err) { if (!multi) { return cleanup(rc); } my_err = rc; }
    cudaEventRecord(ev[1], st);
    int64_t ntot = 0;
    if (!my_err) rc = vxs_submap_merge_batch_impl(ctx, xyz, pts.p, p0, stride_floats, kf_offsets, K, bottom_poses, win_first.data() + lo, nmine, win_size, fine->voxel_size / 8, max_points_per_chunk, nullptr,
                                     nullptr, nullptr, 0, woff.data(), &ntot, &sub_mine);
    if (rc < 0 && !my_err) { if (!multi) { return cleanup(rc); } my_err = rc; }
    if (!my_err) for (int w = 0; w < nmine; w++) sizes_d[size_t(lo + w)] = double(woff[size_t(w) + 1] - woff[size_t(w)]);
    else sizes_d[size_t(nwin)] = 1.0;
  } else cudaEventRecord(ev[1], st);
  cudaEventRecord(ev[2], st);
  // ---- multi-GPU: either every point goes straight to the rank that owns its root cell (all-to-all, default), or the submaps of all ranks go to every rank (all-gather,
  //      VXS_HBA_ROUTE=0) and every rank picks its points out of all of them
  const bool routed = ctx->nranks > 1 && ctx->hba_route;
  const float* sub_dev = sub_mine.p;
  if (ctx->nranks > 1) {
    if (ctx->stage.reserve(size_t(nwin) + 1) != cudaSuccess) { return cleanup(VXS_ERR_NOMEM); }
    cudaMemcpyAsync(ctx->stage.p, sizes_d.data(), (size_t(nwin) + 1) * 8, cudaMemcpyHostToDevice, st);
    rc = vxs_comm_allreduce(ctx, ctx->stage.p, size_t(nwin) + 1);          // every rank contributed its own windows' sizes (+ its error flag), zeros elsewhere
    if (rc) { return cleanup(rc); }
    cudaMemcpyAsync(sizes_d.data(), ctx->stage.p, (size_t(nwin) + 1) * 8, cudaMemcpyDeviceToHost, st);
    cudaStreamSynchronize(st);
    if (sizes_d[size_t(nwin)] > 0.0) {       // all ranks leave together, before any further collective
      return cleanup(my_err ? my_err : vxs_fail(ctx, VXS_ERR_COMM, "vxs_hba_pass: the bottom level failed on another rank"));
    }
    if (!routed) {
    std::vector<size_t> counts(size_t(ctx->nranks), 0), displs(size_t(ctx->nranks), 0);
      size_t tot = 0;
      for (int r = 0; r < ctx->nranks; r++) {
        const int rlo = int((long long)nwin * r / ctx->nranks), rhi = int((long long)nwin * (r + 1) / ctx->nranks);
        size_t c = 0;
        for (int w = rlo; w < rhi; w++) c += size_t(sizes_d[size_t(w)]);
        counts[size_t(r)] = c * 3; displs[size_t(r)] = tot * 3; tot += c;
      }
      // head room of 1/8: the merged clouds differ by a few cells from pass to pass (the poses of the bottom level agree to rounding only), and a buffer that
      // is a few bytes short costs a cudaFree + cudaMalloc of gigabytes (measured: 370 ms once every few passes)
      if (sub_all.cap < std::max<size_t>(tot, 1) * 3 && sub_all.reserve((std::max<size_t>(tot, 1) + tot / 8) * 3) != cudaSuccess) { return cleanup(vxs_fail(ctx, VXS_ERR_NOMEM, "vxs_hba_pass: submaps do not fit")); }
      size_t slot = 0;
      for (size_t c : counts) slot = std::max(slot, c);
      slot = (slot + 3) & ~size_t(3);
      // the padded all-gather reads `slot` floats from this rank's buffer: make sure they exist
      const size_t slot_cap = std::max<size_t>(slot, 1) + slot / 8;
      if ((sub_mine.cap < std::max<size_t>(slot, 1) && sub_mine.reserve_keep(slot_cap, counts[size_t(ctx->rank)], st) != cudaSuccess) ||
          (PB.sub_pad.cap < std::max<size_t>(slot, 1) * size_t(ctx->nranks) && PB.sub_pad.reserve(slot_cap * size_t(ctx->nranks)) != cudaSuccess)) {
        return cleanup(vxs_fail(ctx, VXS_ERR_NOMEM, "vxs_hba_pass: exchange buffers do not fit"));
      }
      rc = vxs_comm_allgatherv_f32(ctx, sub_mine.p, counts[size_t(ctx->rank)], sub_all.p, counts.data(), displs.data(), PB.sub_pad.p, slot);
      if (rc) { return cleanup(rc); }
      sub_dev = sub_all.p;
    }
  }
  cudaEventRecord(ev[3], st);
  // ---- top level
  std::vector<int64_t> sub_off(size_t(nwin) + 1, 0);
  for (int w = 0; w < nwin; w++) { sub_off[size_t(w) + 1] = sub_off[size_t(w)] + int64_t(sizes_d[size_t(w)]); if (submap_sizes) submap_sizes[w] = int64_t(sizes_d[size_t(w)]); }
  for (int w = 0; w < nwin; w++) memcpy(top_poses + size_t(w) * 12, poses12 + size_t(win_first[size_t(w)]) * 12, 96);
  int outer = 0;
  if (routed)
    rc = vxs_hba_top_routed(ctx, coarse, fine, sub_mine.p, woff.data(), lo, nmine, nwin, top_poses, top_max_iter, top_thread_num, top_resis_log, &outer, &PB.sub_pad, &sub_all);
  else if (sub_off[size_t(nwin)] > 0)
    rc = vxs_hba_window_impl(ctx, coarse, fine, nullptr, sub_dev, 3, sub_off.data(), top_poses, nwin, top_max_iter, top_thread_num, nullptr, top_resis_log, &outer,
                             ctx->nranks > 1 ? (long long)sub_off[size_t(lo)] : -1, ctx->nranks > 1 ? (long long)sub_off[size_t(hi)] : -1);
  if (top_outer_iters) *top_outer_iters = outer;
  cudaEventRecord(ev[4], st);
  cudaStreamSynchronize(st);
  if (phase_ms) {
    for (int k = 0; k < 4; k++) { float ms = 0; cudaEventElapsedTime(&ms, ev[k], ev[k + 1]); phase_ms[k] = ms; }
    phase_ms[4] = double(PB.last_voxels); phase_ms[5] = double(PB.last_entries);
  }
  return cleanup(rc);
}
