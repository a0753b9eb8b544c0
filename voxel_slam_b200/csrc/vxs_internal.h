// Internal structures of libvxs (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include "../../include/vxs.h"

#define VXS_SM_COUNT_FALLBACK 132

struct vxs_stage {
  const char* name;
  double ms_total;
  int64_t calls;
};
struct vxs_pending_event {
  int stage;
  cudaEvent_t a, b;
};

template <typename T>
struct DevBuf {  // grow-only device buffer
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    // a buffer that has to grow AGAIN gets 25 % head room: sizes that creep up from call to call (record / node counts of successive map builds) must not
    // cost a cudaFree + cudaMalloc pair — each a device-wide synchronisation, hundreds of ms for GB-sized buffers — every time
    const size_t want = p ? n + n / 4 : n;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    cudaError_t e = cudaMalloc((void**)&p, want * sizeof(T));
    if (e != cudaSuccess && want > n) { cudaGetLastError(); e = cudaMalloc((void**)&p, n * sizeof(T)); if (e == cudaSuccess) cap = n; return e; }
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  // grow to n elements keeping the first `used` ones
  cudaError_t reserve_keep(size_t n, size_t used, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    size_t nc = cap ? cap : 1024;
    while (nc < n) nc *= 2;
    T* np = nullptr;
    cudaError_t e = cudaMalloc((void**)&np, nc * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p && used) { e = cudaMemcpyAsync(np, p, used * sizeof(T), cudaMemcpyDeviceToDevice, st); if (e == cudaSuccess) e = cudaStreamSynchronize(st); }
    if (p) cudaFree(p);
    p = np; cap = nc;
    return e;
  }
};

struct vxs_ctx {
  DevBuf<double> stage2;             // AoS staging of an asynchronous cluster upload (lives until its conversion kernels ran)
  void* odom_scratch = nullptr;      // vxs_odom.cu: plane table + resident scan
  long long* ldlt_prof = nullptr;   // vxs_diag_ldlt_phases: device stamp buffer, otherwise null
  int device = 0;
  int sm_count = VXS_SM_COUNT_FALLBACK;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_copy = nullptr;
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
  std::string err;
  int64_t launches = 0;
  // timing
  bool timing = false;
  std::vector<vxs_stage> stages;
  std::vector<vxs_pending_event> pending;
  std::vector<cudaEvent_t> event_pool;
  // NCCL
  void* comm = nullptr;
  int rank = 0, nranks = 1;
  // per-ctx (= per-device) launch configuration, filled once in vxs_ctx_create (a ctx is used by one thread at a time)
  int coop = -1;                  // cooperative launch of k_ldlt_all possible on this device (-1 = not probed yet)
  int ldlt_blocks_per_sm = 0;
  int ldlt_lookahead = 1;         // VXS_LDLT_LOOKAHEAD_CTA=0 keeps the look-ahead on CTA 0 (A/B switch)
  int syrk_waves = 12;            // VXS_SYRK_WAVES
  int syrk_only_tile = -1;        // VXS_SYRK_ONLY_TILE: diagnostic, run a single tile kind of k_syrk (results are then incomplete)
  int resid_stream = 1;           // VXS_RESID_STREAM=0: k_cluster_sum + k_eig_residual instead of the one streaming kernel (A/B switch)
  int resid_te = 256;             // VXS_RESID_TE: entries per tile (= consumer threads per CTA) of k_residual_stream: 512 (1 CTA/SM), 256 (2), 128 (4)
  int resid_stages = 2, resid_per_sm = 3;   // VXS_RESID_STAGES (2..4), VXS_RESID_PER_SM (CTAs per SM the batches are cut for; 0 = by tile size)
  int smem_optin = 0;             // cudaDevAttrMaxSharedMemoryPerBlockOptin
  int hba_route = 1;              // VXS_HBA_ROUTE=0: multi-GPU top level of vxs_hba_pass through the all-gather of the submaps instead of the owner-routed all-to-all
  int syrk_bulk = 0;              // VXS_SYRK_BULK=1: the bulk-copy / mbarrier form of k_syrk (A/B switch; measured 0.796 vs 0.737 ms for the cp.async form at the metric shape)
  int syrk_streamk = 0;           // VXS_SYRK_STREAMK=1: one-wave stream-K plan instead of the (tile, chunk) grid of k_syrk (A/B switch; measured SLOWER at the metric
                                  // shape, 1.06 vs 0.74 ms: tiles of one voxel chunk no longer run together, so every tile re-reads its XT columns from HBM instead of L2)
  // what ctx->Hraw currently holds (vxs_hba_edges refuses anything but a lidar-only 6W system)
  int hraw_n = 0, hraw_S = 0;
  // solver scratch (n = system size)
  DevBuf<double> Hraw, Mp, Lm, himu, gimu, jact, dvec, rhs, dx, dtmp, states_a, states_b;
  DevBuf<int> perm;
  DevBuf<double> scal;   // small scalar slots on device
  DevBuf<int> flags;
  DevBuf<double> stage;   // H2D/D2H staging for AoS<->SoA conversion
  DevBuf<int64_t> stage_i64;
  // pinned host staging
  double* h_pin = nullptr;
  size_t h_pin_cap = 0;
  // voxeliser scratch lives in vxs_voxelize.cu (opaque)
  void* vox_scratch = nullptr;
  void* hba_scratch = nullptr;       // vxs_hba_batch.cu: persistent buffers of the batched / hierarchical global-BA calls (grow-only, no malloc per pass)
  std::vector<struct vxs_factor*> factors;   // live factors created on this ctx (released with it)
};

struct vxs_factor {
  vxs_ctx* ctx = nullptr;
  int W = 0;
  int64_t V = 0, E = 0;
  size_t Vcap = 0, Ecap = 0;     // SoA strides
  int32_t* ptr = nullptr;        // [Vcap+1]
  int32_t* frame = nullptr;      // [Ecap]
  int32_t* vox = nullptr;        // [Ecap] entry -> voxel
  double* cl = nullptr;          // [10][Ecap] SoA clusters
  double* fix = nullptr;         // [10][Vcap]
  double* coe = nullptr;         // [Vcap]
  double* eig = nullptr;         // [12][Vcap]
  double* sum = nullptr;         // [10][Vcap]
  bool has_fix = false;
  // batch of independent windows (vxs_hba_bottom_batch): W = nwin * block_W global frames, voxel v belongs to window vwin[v] and only touches that window's frames
  int block_W = 0;
  DevBuf<int32_t> vwin;
  // evaluation workspaces (sized lazily)
  DevBuf<double> X;              // scaled rank-3 rows: dense-slot [V][W][18] or compact [E][18]
  DevBuf<double> C;              // lidar Hessian accumulator, (6W)^2 column-major, upper block triangle
  DevBuf<double> gD;             // [W][6] gradient + [W][24] block-diagonal remainder
  DevBuf<double> partial;        // block partial sums for the residual
  DevBuf<unsigned int> counter;
  DevBuf<double> vc;             // [8][Vcap] per-voxel constants for k_jac
  DevBuf<int> sk_tab;            // stream-K plan of k_syrk_sk: seg_ptr[nctas+1] | segments (tile, g_begin, g_end)
  int sk_key[4] = {-1, -1, -1, -1};   // (W, g0, g1, nctas) the plan was made for
  DevBuf<double> cache_copy;     // [22][Vcap] snapshot of eig | sum
  size_t cache_copy_V = 0;
  // asynchronous chunked upload (vxs_factor_push_voxels_async): the clusters arrive on ctx->copy_stream in up_n chunks of whole voxel
  // groups; up_ev[c] fires when chunk c (voxel groups < up_group_end[c]) is resident and converted to SoA.  up_pending > 0 until a
  // consumer has ordered ctx->stream behind the events.
  static const int UP_MAX = 8;
  int up_pending = 0, up_n = 0;
  int up_group_end[UP_MAX] = {0};
  cudaEvent_t up_ev[UP_MAX] = {nullptr};
  cudaEvent_t up_fence = nullptr;
};
void vxs_odom_release(vxs_ctx* c);
void vxs_hba_release(vxs_ctx* c);
int vxs_odom_resident_scan(vxs_ctx* ctx, double** pv12_dev, long long* n);            // the scan var_init / odom_accumulate / pvec_update left on the device
int vxs_odom_set_resident_scan(vxs_ctx* ctx, const double* pv12_host, long long n);
int vxs_factor_wait_uploads(vxs_factor* f);   // orders ctx->stream behind every pending upload chunk (device-side wait, no host sync)

inline int vxs_fail(vxs_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess) {
  if (c) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s%s%s", what, e != cudaSuccess ? ": " : "", e != cudaSuccess ? cudaGetErrorString(e) : "");
    c->err = buf;
  }
  return code;
}
#define VXS_CUDA(ctx, call)                                                   \
  do {                                                                        \
    cudaError_t _e = (call);                                                  \
    if (_e != cudaSuccess) return vxs_fail((ctx), VXS_ERR_CUDA, #call, _e);   \
  } while (0)

int vxs_stage_id(vxs_ctx* c, const char* name);
void vxs_stage_begin(vxs_ctx* c, int stage);
void vxs_stage_end(vxs_ctx* c);

// Launch a kernel on the ctx stream, count it, optionally bracket it with events under the given stage name.
#define VXS_LAUNCH(ctx, stage_name_, kern, grid, block, smem, ...)                    \
  do {                                                                               \
    if ((ctx)->timing) vxs_stage_begin((ctx), vxs_stage_id((ctx), stage_name_));     \
    kern<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);                    \
    (ctx)->launches++;                                                               \
    if ((ctx)->timing) vxs_stage_end((ctx));                                         \
    cudaError_t _le = cudaGetLastError();                                            \
    if (_le != cudaSuccess) return vxs_fail((ctx), VXS_ERR_CUDA, stage_name_, _le);  \
  } while (0)

// factor internals shared between translation units
int vxs_factor_reserve(vxs_factor* f, size_t Vneed, size_t Eneed);
int vxs_factor_finish_push(vxs_factor* f);  // builds entry->voxel map, sets flags

// evaluation (vxs_eval.cu): all device-side, results stay on device
struct vxs_eval_out {
  double* C;    // (6W)^2 lidar Hessian (upper block triangle valid, diag blocks full), column-major
  double* gD;   // [W][6] g, then [W][24] D
};
int vxs_eval_residual_dev(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pose_stride, double* residual_dev);
int vxs_eval_hessian_dev(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pose_stride, double* r1_dev);
int vxs_eval_hessian_bd_dev(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pstride, const int* build_mask_dev, double* Cbd, double* gD);
int vxs_comm_allreduce(vxs_ctx* ctx, double* buf, size_t n);
int vxs_residual_stream_launch(vxs_ctx* ctx, vxs_factor* f, const double* poses_dev, int pstride, double* residual_dev, int* ran, double* rvox = nullptr);   // vxs_resid.cu

// solver (vxs_solve.cu)
int vxs_solve_damped(vxs_ctx* ctx, const double* Hraw, const double* jact, int n, int gauge, double u, double* dx_dev, double* D_dev, double* rhs_dev, int* singular_flag_host);
