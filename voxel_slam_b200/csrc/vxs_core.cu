// Context, timing and the device-resident LidarFactor container (CSR over observing frames, SoA clusters).
// Reference: voxel_map.hpp:109-130,281-286 (LidarFactor members, push_voxel, clear).
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include "vxs_internal.h"

// ------------------------------------------------------------------ ctx
extern "C" int vxs_version(void) { return 100; }

extern "C" int vxs_ctx_create(int device, vxs_ctx** out) {
  if (!out) return VXS_ERR_ARG;
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    fprintf(stderr, "vxs_ctx_create: no CUDA device (%s) — libvxs has no CPU fallback\n", cudaGetErrorString(e));
    return VXS_ERR_CUDA;
  }
  if (device < 0 || device >= ndev) return VXS_ERR_ARG;
  vxs_ctx* c = new vxs_ctx();
  c->device = device;
  if (cudaSetDevice(device) != cudaSuccess) { delete c; return VXS_ERR_CUDA; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return VXS_ERR_CUDA; }
  cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&c->ev_copy, cudaEventDisableTiming);
  cudaEventCreate(&c->ev_t0); cudaEventCreate(&c->ev_t1);
  c->scal.reserve(64);
  c->flags.reserve(16);
  { const char* e = getenv("VXS_LDLT_LOOKAHEAD_CTA"); c->ldlt_lookahead = (e && e[0] == '0') ? 0 : 1; }
  { const char* e = getenv("VXS_SYRK_WAVES"); c->syrk_waves = e ? std::max(1, atoi(e)) : 8; }
  cudaDeviceGetAttribute(&c->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  { const char* e = getenv("VXS_HBA_ROUTE"); c->hba_route = (e && e[0] == '0') ? 0 : 1; }
  *out = c;
  return VXS_OK;
}

void vxs_voxelize_release(vxs_ctx* c);
static void vxs_factor_release_device(vxs_factor* f);

extern "C" int vxs_ctx_destroy(vxs_ctx* c) {
  if (!c) return VXS_OK;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  for (vxs_factor* f : c->factors) { vxs_factor_release_device(f); f->ctx = nullptr; }   // handles stay valid for vxs_factor_destroy
  c->factors.clear();
  vxs_ctx_comm_destroy(c);
  vxs_voxelize_release(c);
  vxs_odom_release(c);
  vxs_hba_release(c);
  for (auto& p : c->pending) { cudaEventDestroy(p.a); cudaEventDestroy(p.b); }
  for (auto ev : c->event_pool) cudaEventDestroy(ev);
  c->Hraw.release(); c->Mp.release(); c->Lm.release(); c->himu.release(); c->gimu.release(); c->jact.release(); c->dvec.release();
  c->rhs.release(); c->dx.release(); c->dtmp.release(); c->states_a.release(); c->states_b.release(); c->perm.release();
  c->scal.release(); c->flags.release(); c->stage.release(); c->stage2.release(); c->stage_i64.release();
  if (c->h_pin) cudaFreeHost(c->h_pin);
  if (c->ev_copy) cudaEventDestroy(c->ev_copy);
  if (c->ev_t0) cudaEventDestroy(c->ev_t0);
  if (c->ev_t1) cudaEventDestroy(c->ev_t1);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return VXS_OK;
}
extern "C" const char* vxs_ctx_last_error(const vxs_ctx* c) { return c ? c->err.c_str() : "null ctx"; }
extern "C" int64_t vxs_ctx_launch_count(const vxs_ctx* c) { return c ? c->launches : 0; }
extern "C" int vxs_host_alloc(void** out, uint64_t bytes) { return cudaHostAlloc(out, bytes, cudaHostAllocDefault) == cudaSuccess ? VXS_OK : VXS_ERR_NOMEM; }
extern "C" int vxs_host_free(void* p) { return cudaFreeHost(p) == cudaSuccess ? VXS_OK : VXS_ERR_CUDA; }

// ------------------------------------------------------------------ timing
int vxs_stage_id(vxs_ctx* c, const char* name) {
  for (size_t i = 0; i < c->stages.size(); i++) if (c->stages[i].name == name || strcmp(c->stages[i].name, name) == 0) return int(i);
  c->stages.push_back(vxs_stage{name, 0.0, 0});
  return int(c->stages.size()) - 1;
}
static cudaEvent_t vxs_get_event(vxs_ctx* c) {
  if (!c->event_pool.empty()) { cudaEvent_t e = c->event_pool.back(); c->event_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
void vxs_stage_begin(vxs_ctx* c, int stage) {
  vxs_pending_event p; p.stage = stage; p.a = vxs_get_event(c); p.b = vxs_get_event(c);
  cudaEventRecord(p.a, c->stream);
  c->pending.push_back(p);
}
void vxs_stage_end(vxs_ctx* c) { cudaEventRecord(c->pending.back().b, c->stream); }
static void vxs_timing_flush(vxs_ctx* c) {
  cudaStreamSynchronize(c->stream);
  for (auto& p : c->pending) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) { c->stages[p.stage].ms_total += ms; c->stages[p.stage].calls++; }
    c->event_pool.push_back(p.a); c->event_pool.push_back(p.b);
  }
  c->pending.clear();
}
extern "C" int vxs_ctx_timing_enable(vxs_ctx* c, int on) { if (!c) return VXS_ERR_ARG; if (!on && c->timing) vxs_timing_flush(c); c->timing = on != 0; return VXS_OK; }
extern "C" int vxs_ctx_timing_reset(vxs_ctx* c) { if (!c) return VXS_ERR_ARG; vxs_timing_flush(c); for (auto& s : c->stages) { s.ms_total = 0; s.calls = 0; } return VXS_OK; }
extern "C" int vxs_ctx_timing_read(vxs_ctx* c, int cap, const char** names, double* ms_total, int64_t* calls, int* n_out) {
  if (!c) return VXS_ERR_ARG;
  vxs_timing_flush(c);
  int n = std::min<int>(cap, int(c->stages.size()));
  for (int i = 0; i < n; i++) { names[i] = c->stages[i].name; ms_total[i] = c->stages[i].ms_total; calls[i] = c->stages[i].calls; }
  if (n_out) *n_out = n;
  return VXS_OK;
}

extern "C" int vxs_ctx_timer_start(vxs_ctx* c) {
  if (!c) return VXS_ERR_ARG;
  cudaSetDevice(c->device);
  VXS_CUDA(c, cudaStreamSynchronize(c->stream));
  VXS_CUDA(c, cudaEventRecord(c->ev_t0, c->stream));
  return VXS_OK;
}
extern "C" int vxs_ctx_timer_stop(vxs_ctx* c, double* ms) {
  if (!c || !ms) return VXS_ERR_ARG;
  VXS_CUDA(c, cudaEventRecord(c->ev_t1, c->stream));
  VXS_CUDA(c, cudaEventSynchronize(c->ev_t1));
  float f = 0;
  VXS_CUDA(c, cudaEventElapsedTime(&f, c->ev_t0, c->ev_t1));
  *ms = f;
  return VXS_OK;
}

// fp64 FMA peak: 8 independent chains per thread, enough warps to fill every SM
__global__ void __launch_bounds__(256) k_dfma_peak(double* out, int iters) {
  double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  const double b = 1.0000001, c = 1e-9;
  for (int i = 0; i < iters; i++) {
    a0 = fma(a0, b, c); a1 = fma(a1, b, c); a2 = fma(a2, b, c); a3 = fma(a3, b, c);
    a4 = fma(a4, b, c); a5 = fma(a5, b, c); a6 = fma(a6, b, c); a7 = fma(a7, b, c);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = ((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7));
}
extern "C" int vxs_diag_fp64_tflops(vxs_ctx* c, double* tflops) {
  if (!c || !tflops) return VXS_ERR_ARG;
  cudaSetDevice(c->device);
  const int blocks = c->sm_count * 8, iters = 20000;
  VXS_CUDA(c, c->stage.reserve(size_t(blocks) * 256));
  double best = 0;
  for (int rep = 0; rep < 4; rep++) {
    VXS_CUDA(c, cudaEventRecord(c->ev_t0, c->stream));
    VXS_LAUNCH(c, "k_dfma_peak", k_dfma_peak, blocks, 256, 0, c->stage.p, iters);
    VXS_CUDA(c, cudaEventRecord(c->ev_t1, c->stream));
    VXS_CUDA(c, cudaEventSynchronize(c->ev_t1));
    float ms = 0;
    VXS_CUDA(c, cudaEventElapsedTime(&ms, c->ev_t0, c->ev_t1));
    const double tf = double(blocks) * 256 * iters * 8 * 2 / (ms * 1e-3) / 1e12;
    if (rep > 0 && tf > best) best = tf;
  }
  *tflops = best;
  return VXS_OK;
}

// fp64 tensor-core (DMMA) peak of one mma.sync shape: 8 independent accumulator tiles per warp.
// SHAPE 0 = m8n8k4 (Ampere's shape, SASS DMMA.8x8x4), 1 = m16n8k4, 2 = m16n8k8, 3 = m16n8k16 (Hopper, DMMA.16x8x{4,8,16}).
constexpr int kDmmaShapes = 4;
constexpr int dmma_shape_fma(int shape) { return shape == 0 ? 8 * 8 * 4 : 16 * 8 * (4 << (shape - 1)); }
template <int SHAPE>
__global__ void __launch_bounds__(256) k_dmma_peak(double* out, int iters) {
  constexpr int NC = SHAPE == 0 ? 2 : 4;    // accumulator registers per tile
  double c[8 * NC];
#pragma unroll
  for (int i = 0; i < 8 * NC; i++) c[i] = 0.0;
  double a[8], b[4];
#pragma unroll
  for (int i = 0; i < 8; i++) a[i] = 1.0 + (threadIdx.x + i) * 1e-9;
#pragma unroll
  for (int i = 0; i < 4; i++) b[i] = 1.0 - (threadIdx.x + i) * 1e-9;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int t = 0; t < 8; t++) {
      double* d = c + NC * t;
      if (SHAPE == 0)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(d[0]), "+d"(d[1]) : "d"(a[0]), "d"(b[0]));
      else if (SHAPE == 1)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                     : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
      else if (SHAPE == 2)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                     : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
      else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                     : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8 * NC; i++) s += c[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// best of three timed launches after one warm-up; every shape does the same flops per launch
static int dmma_shape_tflops(vxs_ctx* c, int shape, double* tflops) {
  cudaSetDevice(c->device);
  const int blocks = c->sm_count * 4, iters = 4000 * dmma_shape_fma(0) / dmma_shape_fma(shape);
  void (*const kernels[kDmmaShapes])(double*, int) = {k_dmma_peak<0>, k_dmma_peak<1>, k_dmma_peak<2>, k_dmma_peak<3>};
  VXS_CUDA(c, c->stage.reserve(size_t(blocks) * 256));
  double best = 0;
  for (int rep = 0; rep < 4; rep++) {
    VXS_CUDA(c, cudaEventRecord(c->ev_t0, c->stream));
    VXS_LAUNCH(c, "k_dmma_peak", kernels[shape], blocks, 256, 0, c->stage.p, iters);
    VXS_CUDA(c, cudaEventRecord(c->ev_t1, c->stream));
    VXS_CUDA(c, cudaEventSynchronize(c->ev_t1));
    float ms = 0;
    VXS_CUDA(c, cudaEventElapsedTime(&ms, c->ev_t0, c->ev_t1));
    const double tf = double(blocks) * 8 /*warps*/ * iters * 8 /*mma*/ * dmma_shape_fma(shape) * 2 / (ms * 1e-3) / 1e12;
    if (rep > 0 && tf > best) best = tf;
  }
  *tflops = best;
  return VXS_OK;
}
// the shape k_syrk issues (m16n8k4), so that it is the ceiling of the kernel's own instruction
extern "C" int vxs_diag_dmma_tflops(vxs_ctx* c, double* tflops) {
  if (!c || !tflops) return VXS_ERR_ARG;
  return dmma_shape_tflops(c, 1, tflops);
}
extern "C" int vxs_diag_dmma_shapes(vxs_ctx* c, double tflops[4]) {
  if (!c || !tflops) return VXS_ERR_ARG;
  for (int s = 0; s < kDmmaShapes; s++) {
    int rc = dmma_shape_tflops(c, s, tflops + s);
    if (rc) return rc;
  }
  return VXS_OK;
}

// ------------------------------------------------------------------ factor container
extern "C" int vxs_factor_create(vxs_ctx* ctx, int win_size, vxs_factor** out) {
  if (!ctx || !out || win_size <= 0) return VXS_ERR_ARG;
  vxs_factor* f = new vxs_factor();
  f->ctx = ctx; f->W = win_size;
  ctx->factors.push_back(f);
  *out = f;
  return VXS_OK;
}
static void factor_free_arrays(vxs_factor* f) {
  cudaFree(f->ptr); cudaFree(f->frame); cudaFree(f->vox); cudaFree(f->cl); cudaFree(f->fix); cudaFree(f->coe); cudaFree(f->eig); cudaFree(f->sum);
  f->ptr = f->frame = f->vox = nullptr; f->cl = f->fix = f->coe = f->eig = f->sum = nullptr;
  f->Vcap = f->Ecap = 0;
}
static void vxs_factor_release_device(vxs_factor* f) {
  factor_free_arrays(f);
  f->vwin.release(); f->X.release(); f->C.release(); f->gD.release(); f->partial.release(); f->counter.release(); f->cache_copy.release(); f->vc.release();
  for (int c = 0; c < vxs_factor::UP_MAX; c++) if (f->up_ev[c]) { cudaEventDestroy(f->up_ev[c]); f->up_ev[c] = nullptr; }
  if (f->up_fence) { cudaEventDestroy(f->up_fence); f->up_fence = nullptr; }
  f->up_pending = f->up_n = 0;
  f->V = f->E = 0; f->cache_copy_V = 0;
}
extern "C" int vxs_factor_destroy(vxs_factor* f) {
  if (!f) return VXS_OK;
  if (f->ctx) {   // ctx still alive
    vxs_ctx* c = f->ctx;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    vxs_factor_release_device(f);
    for (size_t i = 0; i < c->factors.size(); i++) if (c->factors[i] == f) { c->factors.erase(c->factors.begin() + i); break; }
  }
  delete f;
  return VXS_OK;
}
extern "C" int vxs_factor_clear(vxs_factor* f) {
  if (!f || !f->ctx) return VXS_ERR_ARG;
  int rc = vxs_factor_wait_uploads(f);   // an upload still in flight targets the arrays the next push will write
  f->V = 0; f->E = 0; f->has_fix = false; f->block_W = 0;
  return rc;
}
extern "C" int vxs_factor_set_win_size(vxs_factor* f, int w) { if (!f || w <= 0 || f->V != 0) return VXS_ERR_ARG; f->W = w; return VXS_OK; }
extern "C" int vxs_factor_counts(const vxs_factor* f, int64_t* n_vox, int64_t* n_entries, int* win_size) {
  if (!f) return VXS_ERR_ARG;
  if (n_vox) *n_vox = f->V; if (n_entries) *n_entries = f->E; if (win_size) *win_size = f->W;
  return VXS_OK;
}

// grow SoA storage, preserving content
int vxs_factor_reserve(vxs_factor* f, size_t Vneed, size_t Eneed) {
  vxs_ctx* ctx = f->ctx;
  if (Vneed <= f->Vcap && Eneed <= f->Ecap) return VXS_OK;
  if (Eneed >= (size_t(1) << 31) || Vneed >= (size_t(1) << 31)) return vxs_fail(ctx, VXS_ERR_ARG, "factor too large for 32-bit offsets");
  size_t Vn = std::max(Vneed, f->Vcap), En = std::max(Eneed, f->Ecap);
  if (f->V > 0) { Vn = std::max(Vn, f->Vcap * 2); En = std::max(En, f->Ecap * 2); }  // amortise repeated appends
  Vn = (Vn + 31) & ~size_t(31); En = (En + 31) & ~size_t(31);  // keep every SoA row 256-byte aligned
  int32_t *ptr = nullptr, *frame = nullptr, *vox = nullptr;
  double *cl = nullptr, *fix = nullptr, *coe = nullptr, *eig = nullptr, *sum = nullptr;
  VXS_CUDA(ctx, cudaMalloc((void**)&ptr, (Vn + 1) * sizeof(int32_t)));
  VXS_CUDA(ctx, cudaMalloc((void**)&frame, En * sizeof(int32_t)));
  VXS_CUDA(ctx, cudaMalloc((void**)&vox, En * sizeof(int32_t)));
  VXS_CUDA(ctx, cudaMalloc((void**)&cl, 10 * En * sizeof(double)));
  VXS_CUDA(ctx, cudaMalloc((void**)&fix, 10 * Vn * sizeof(double)));
  VXS_CUDA(ctx, cudaMalloc((void**)&coe, Vn * sizeof(double)));
  VXS_CUDA(ctx, cudaMalloc((void**)&eig, 12 * Vn * sizeof(double)));
  VXS_CUDA(ctx, cudaMalloc((void**)&sum, 10 * Vn * sizeof(double)));
  cudaStream_t s = ctx->stream;
  if (f->V > 0) {
    size_t V = size_t(f->V), E = size_t(f->E);
    VXS_CUDA(ctx, cudaMemcpyAsync(ptr, f->ptr, (V + 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    VXS_CUDA(ctx, cudaMemcpyAsync(frame, f->frame, E * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    VXS_CUDA(ctx, cudaMemcpy2DAsync(cl, En * 8, f->cl, f->Ecap * 8, E * 8, 10, cudaMemcpyDeviceToDevice, s));
    VXS_CUDA(ctx, cudaMemcpy2DAsync(fix, Vn * 8, f->fix, f->Vcap * 8, V * 8, 10, cudaMemcpyDeviceToDevice, s));
    VXS_CUDA(ctx, cudaMemcpyAsync(coe, f->coe, V * 8, cudaMemcpyDeviceToDevice, s));
    VXS_CUDA(ctx, cudaMemcpy2DAsync(eig, Vn * 8, f->eig, f->Vcap * 8, V * 8, 12, cudaMemcpyDeviceToDevice, s));
    VXS_CUDA(ctx, cudaMemcpy2DAsync(sum, Vn * 8, f->sum, f->Vcap * 8, V * 8, 10, cudaMemcpyDeviceToDevice, s));
  }
  VXS_CUDA(ctx, cudaStreamSynchronize(s));
  factor_free_arrays(f);
  f->ptr = ptr; f->frame = frame; f->vox = vox; f->cl = cl; f->fix = fix; f->coe = coe; f->eig = eig; f->sum = sum;
  f->Vcap = Vn; f->Ecap = En;
  return VXS_OK;
}

// AoS [n][K] (linear) -> SoA rows dst[c*stride + off + i]
__global__ void k_aos_to_soa(const double* __restrict__ src, double* __restrict__ dst, size_t n, int K, size_t stride, size_t off) {
  size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n * K) return;
  size_t i = idx / K; int c = int(idx - i * K);
  dst[size_t(c) * stride + off + i] = src[idx];
}
__global__ void k_soa_to_aos(const double* __restrict__ src, double* __restrict__ dst, size_t n, int K, size_t stride) {
  size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n * K) return;
  size_t i = idx / K; int c = int(idx - i * K);
  dst[idx] = src[size_t(c) * stride + i];
}
__global__ void k_fill(double* dst, size_t n, double val) {
  size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx < n) dst[idx] = val;
}
__global__ void k_zero_rows(double* dst, size_t n, int K, size_t stride, size_t off) {
  size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n * K) return;
  size_t i = idx % n; int c = int(idx / n);
  dst[size_t(c) * stride + off + i] = 0.0;
}
__global__ void k_ptr_offset(const int64_t* __restrict__ src, int32_t* __restrict__ dst, size_t n_plus1, int64_t base) {
  size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx < n_plus1) dst[idx] = int32_t(src[idx] + base);
}
__global__ void k_entry_to_voxel(const int32_t* __restrict__ ptr, int32_t* __restrict__ vox, int64_t v0, int64_t V) {
  int64_t v = v0 + int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= V) return;
  for (int32_t e = ptr[v]; e < ptr[v + 1]; e++) vox[e] = int32_t(v);
}

static inline unsigned nblk(size_t n, unsigned b) { return unsigned((n + b - 1) / b); }

extern "C" int vxs_factor_push_voxels(vxs_factor* f, int64_t n_vox, const int64_t* entry_ptr, const int32_t* entry_frame,
                                      const double* entry_cluster10, const double* fix10, const double* coe, const double* eig12,
                                      const double* sum10) {
  if (!f || !f->ctx || n_vox < 0 || (n_vox > 0 && (!entry_ptr || !entry_frame || !entry_cluster10 || !eig12 || !sum10))) return VXS_ERR_ARG;
  if (n_vox == 0) return VXS_OK;
  vxs_ctx* ctx = f->ctx;
  cudaSetDevice(ctx->device);
  { int rcw = vxs_factor_wait_uploads(f); if (rcw) return rcw; }
  const int64_t n_ent = entry_ptr[n_vox] - entry_ptr[0];
  if (entry_ptr[0] != 0 || n_ent < 0) return vxs_fail(ctx, VXS_ERR_ARG, "entry_ptr must start at 0 and be non-decreasing");
  int rc = vxs_factor_reserve(f, size_t(f->V + n_vox), size_t(f->E + n_ent));
  if (rc) return rc;
  cudaStream_t s = ctx->stream;
  const size_t V0 = size_t(f->V), E0 = size_t(f->E), n = size_t(n_vox), ne = size_t(n_ent);
  VXS_CUDA(ctx, ctx->stage.reserve(std::max(ne * 10, n * 12)));
  VXS_CUDA(ctx, ctx->stage_i64.reserve(n + 1));
  // CSR structure
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage_i64.p, entry_ptr, (n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  VXS_LAUNCH(ctx, "k_ptr_offset", k_ptr_offset, nblk(n + 1, 256), 256, 0, ctx->stage_i64.p, f->ptr + V0, n + 1, int64_t(E0));
  if (ne) VXS_CUDA(ctx, cudaMemcpyAsync(f->frame + E0, entry_frame, ne * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  // clusters
  if (ne) {
    VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage.p, entry_cluster10, ne * 10 * 8, cudaMemcpyHostToDevice, s));
    VXS_LAUNCH(ctx, "k_aos_to_soa", k_aos_to_soa, nblk(ne * 10, 256), 256, 0, ctx->stage.p, f->cl, ne, 10, f->Ecap, E0);
  }
  // per-voxel records (the staging buffer is reused: stream order keeps each copy behind the previous kernel)
  if (fix10) {
    VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage.p, fix10, n * 10 * 8, cudaMemcpyHostToDevice, s));
    VXS_LAUNCH(ctx, "k_aos_to_soa", k_aos_to_soa, nblk(n * 10, 256), 256, 0, ctx->stage.p, f->fix, n, 10, f->Vcap, V0);
    bool any = false;
    for (size_t i = 0; i < n && !any; i++) any = fix10[i * 10 + 9] != 0.0;
    f->has_fix = f->has_fix || any;
  } else {
    VXS_LAUNCH(ctx, "k_zero_rows", k_zero_rows, nblk(n * 10, 256), 256, 0, f->fix, n, 10, f->Vcap, V0);
  }
  if (coe) VXS_CUDA(ctx, cudaMemcpyAsync(f->coe + V0, coe, n * 8, cudaMemcpyHostToDevice, s));
  else VXS_LAUNCH(ctx, "k_fill", k_fill, nblk(n, 256), 256, 0, f->coe + V0, n, 1.0);
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage.p, eig12, n * 12 * 8, cudaMemcpyHostToDevice, s));
  VXS_LAUNCH(ctx, "k_aos_to_soa", k_aos_to_soa, nblk(n * 12, 256), 256, 0, ctx->stage.p, f->eig, n, 12, f->Vcap, V0);
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage.p, sum10, n * 10 * 8, cudaMemcpyHostToDevice, s));
  VXS_LAUNCH(ctx, "k_aos_to_soa", k_aos_to_soa, nblk(n * 10, 256), 256, 0, ctx->stage.p, f->sum, n, 10, f->Vcap, V0);
  f->V += n_vox; f->E += n_ent;
  VXS_LAUNCH(ctx, "k_entry_to_voxel", k_entry_to_voxel, nblk(n, 128), 128, 0, f->ptr, f->vox, int64_t(V0), f->V);
  VXS_CUDA(ctx, cudaStreamSynchronize(s));  // host buffers may be reused by the caller on return
  return VXS_OK;
}

int vxs_factor_wait_uploads(vxs_factor* f) {
  if (!f || !f->ctx || f->up_pending == 0) return VXS_OK;
  vxs_ctx* ctx = f->ctx;
  for (int c = 0; c < f->up_n; c++) VXS_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, f->up_ev[c], 0));
  f->up_pending = 0;
  return VXS_OK;
}
extern "C" int vxs_factor_sync_uploads(vxs_factor* f) {
  if (!f || !f->ctx) return VXS_ERR_ARG;
  if (f->up_n > 0 && f->up_ev[f->up_n - 1]) VXS_CUDA(f->ctx, cudaEventSynchronize(f->up_ev[f->up_n - 1]));   // chunks complete in order on one stream
  VXS_CUDA(f->ctx, cudaStreamSynchronize(f->ctx->stream));
  return VXS_OK;
}

// Same contract as vxs_factor_push_voxels for an EMPTY factor, but nothing is waited for: the per-voxel records go up on the ctx stream,
// the clusters (the bulk: 80 B per entry) on the copy stream in chunks of whole voxel groups, each followed by its AoS -> SoA conversion
// and an event.  The first Hessian build then runs chunk by chunk behind those events, so the PCIe transfer of chunk c+1 overlaps the
// Jacobian / SYRK work on chunk c.  The host buffers must stay valid (and should be pinned) until a consuming call has returned.
extern "C" int vxs_factor_push_voxels_async(vxs_factor* f, int64_t n_vox, const int64_t* entry_ptr, const int32_t* entry_frame, const double* entry_cluster10,
                                            const double* fix10, const double* coe, const double* eig12, const double* sum10) {
  if (!f || !f->ctx || n_vox < 0 || (n_vox > 0 && (!entry_ptr || !entry_frame || !entry_cluster10 || !eig12 || !sum10))) return VXS_ERR_ARG;
  const int NCH = 4;
  if (f->V != 0 || n_vox < 64 * NCH) return vxs_factor_push_voxels(f, n_vox, entry_ptr, entry_frame, entry_cluster10, fix10, coe, eig12, sum10);
  vxs_ctx* ctx = f->ctx;
  cudaSetDevice(ctx->device);
  int rc = vxs_factor_wait_uploads(f);
  if (rc) return rc;
  const int64_t n_ent = entry_ptr[n_vox] - entry_ptr[0];
  if (entry_ptr[0] != 0 || n_ent < 0) return vxs_fail(ctx, VXS_ERR_ARG, "entry_ptr must start at 0 and be non-decreasing");
  rc = vxs_factor_reserve(f, size_t(n_vox), size_t(n_ent));
  if (rc) return rc;
  cudaStream_t s = ctx->stream, cs = ctx->copy_stream;
  const size_t n = size_t(n_vox), ne = size_t(n_ent);
  VXS_CUDA(ctx, ctx->stage.reserve(n * 12));
  VXS_CUDA(ctx, ctx->stage2.reserve(ne * 10));
  VXS_CUDA(ctx, ctx->stage_i64.reserve(n + 1));
  if (!f->up_fence) VXS_CUDA(ctx, cudaEventCreateWithFlags(&f->up_fence, cudaEventDisableTiming));
  for (int c = 0; c < NCH; c++) if (!f->up_ev[c]) VXS_CUDA(ctx, cudaEventCreateWithFlags(&f->up_ev[c], cudaEventDisableTiming));
  // the copy stream starts behind whatever the ctx stream still does with this factor's arrays
  VXS_CUDA(ctx, cudaEventRecord(f->up_fence, s));
  VXS_CUDA(ctx, cudaStreamWaitEvent(cs, f->up_fence, 0));
  // clusters + frame indices, chunked by voxel groups of 4 (the unit of the dense Jacobian / SYRK kernels)
  const int64_t ngv = (n_vox + 3) / 4;
  for (int c = 0; c < NCH; c++) {
    const int64_t g0 = ngv * c / NCH, g1 = ngv * (c + 1) / NCH;
    const int64_t v0 = std::min<int64_t>(4 * g0, n_vox), v1 = std::min<int64_t>(4 * g1, n_vox);
    const size_t e0 = size_t(entry_ptr[v0]), e1 = size_t(entry_ptr[v1]);
    if (e1 > e0) {
      VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage2.p + e0 * 10, entry_cluster10 + e0 * 10, (e1 - e0) * 80, cudaMemcpyHostToDevice, cs));
      VXS_CUDA(ctx, cudaMemcpyAsync(f->frame + e0, entry_frame + e0, (e1 - e0) * 4, cudaMemcpyHostToDevice, cs));
      k_aos_to_soa<<<nblk((e1 - e0) * 10, 256), 256, 0, cs>>>(ctx->stage2.p + e0 * 10, f->cl, e1 - e0, 10, f->Ecap, e0);
      ctx->launches++;
    }
    VXS_CUDA(ctx, cudaEventRecord(f->up_ev[c], cs));
    f->up_group_end[c] = int(g1);
  }
  f->up_n = NCH; f->up_pending = NCH;
  // CSR structure and per-voxel records on the ctx stream (small: 4 + 8 + 96 + 80 (+80) bytes per voxel)
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage_i64.p, entry_ptr, (n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  VXS_LAUNCH(ctx, "k_ptr_offset", k_ptr_offset, nblk(n + 1, 256), 256, 0, ctx->stage_i64.p, f->ptr, n + 1, int64_t(0));
  if (fix10) {
    VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage.p, fix10, n * 10 * 8, cudaMemcpyHostToDevice, s));
    VXS_LAUNCH(ctx, "k_aos_to_soa", k_aos_to_soa, nblk(n * 10, 256), 256, 0, ctx->stage.p, f->fix, n, 10, f->Vcap, size_t(0));
    bool any = false;
    for (size_t i = 0; i < n && !any; i++) any = fix10[i * 10 + 9] != 0.0;
    f->has_fix = f->has_fix || any;
  } else {
    VXS_LAUNCH(ctx, "k_zero_rows", k_zero_rows, nblk(n * 10, 256), 256, 0, f->fix, n, 10, f->Vcap, size_t(0));
  }
  if (coe) VXS_CUDA(ctx, cudaMemcpyAsync(f->coe, coe, n * 8, cudaMemcpyHostToDevice, s));
  else VXS_LAUNCH(ctx, "k_fill", k_fill, nblk(n, 256), 256, 0, f->coe, n, 1.0);
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage.p, eig12, n * 12 * 8, cudaMemcpyHostToDevice, s));
  VXS_LAUNCH(ctx, "k_aos_to_soa", k_aos_to_soa, nblk(n * 12, 256), 256, 0, ctx->stage.p, f->eig, n, 12, f->Vcap, size_t(0));
  VXS_CUDA(ctx, cudaMemcpyAsync(ctx->stage.p, sum10, n * 10 * 8, cudaMemcpyHostToDevice, s));
  VXS_LAUNCH(ctx, "k_aos_to_soa", k_aos_to_soa, nblk(n * 10, 256), 256, 0, ctx->stage.p, f->sum, n, 10, f->Vcap, size_t(0));
  f->V = n_vox; f->E = n_ent;
  VXS_LAUNCH(ctx, "k_entry_to_voxel", k_entry_to_voxel, nblk(n, 128), 128, 0, f->ptr, f->vox, int64_t(0), f->V);
  return VXS_OK;
}

extern "C" int vxs_factor_push_voxels_dense(vxs_factor* f, int64_t n_vox, const double* clusters10, const double* fix10, const double* coe,
                                            const double* eig12, const double* sum10) {
  if (!f || !f->ctx || n_vox < 0 || (n_vox > 0 && !clusters10)) return VXS_ERR_ARG;
  const int W = f->W;
  std::vector<int64_t> ptr(size_t(n_vox) + 1, 0);
  std::vector<int32_t> frame;
  std::vector<double> cl;
  frame.reserve(size_t(n_vox) * W); cl.reserve(size_t(n_vox) * W * 10);
  for (int64_t v = 0; v < n_vox; v++) {
    for (int i = 0; i < W; i++) {
      const double* c = clusters10 + (size_t(v) * W + i) * 10;
      if (c[9] != 0.0) { frame.push_back(i); cl.insert(cl.end(), c, c + 10); }  // voxel_map.hpp:178 "if(sig_orig[i].N != 0)"
    }
    ptr[size_t(v) + 1] = int64_t(frame.size());
  }
  return vxs_factor_push_voxels(f, n_vox, ptr.data(), frame.data(), cl.data(), fix10, coe, eig12, sum10);
}

extern "C" int vxs_factor_cache_save(vxs_factor* f) {
  if (!f || !f->ctx) return VXS_ERR_ARG;
  vxs_ctx* ctx = f->ctx;
  cudaSetDevice(ctx->device);
  const size_t V = size_t(f->V);
  if (V == 0) { f->cache_copy_V = 0; return VXS_OK; }
  { int rcw = vxs_factor_wait_uploads(f); if (rcw) return rcw; }
  VXS_CUDA(ctx, f->cache_copy.reserve(V * 22));
  VXS_CUDA(ctx, cudaMemcpy2DAsync(f->cache_copy.p, V * 8, f->eig, f->Vcap * 8, V * 8, 12, cudaMemcpyDeviceToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaMemcpy2DAsync(f->cache_copy.p + V * 12, V * 8, f->sum, f->Vcap * 8, V * 8, 10, cudaMemcpyDeviceToDevice, ctx->stream));
  f->cache_copy_V = V;
  return VXS_OK;
}
extern "C" int vxs_factor_cache_restore(vxs_factor* f) {
  if (!f || !f->ctx) return VXS_ERR_ARG;
  vxs_ctx* ctx = f->ctx;
  const size_t V = size_t(f->V);
  if (V == 0) return VXS_OK;
  if (f->cache_copy_V != V) return vxs_fail(ctx, VXS_ERR_ARG, "vxs_factor_cache_restore: no snapshot of this factor");
  cudaSetDevice(ctx->device);
  VXS_CUDA(ctx, cudaMemcpy2DAsync(f->eig, f->Vcap * 8, f->cache_copy.p, V * 8, V * 8, 12, cudaMemcpyDeviceToDevice, ctx->stream));
  VXS_CUDA(ctx, cudaMemcpy2DAsync(f->sum, f->Vcap * 8, f->cache_copy.p + V * 12, V * 8, V * 8, 10, cudaMemcpyDeviceToDevice, ctx->stream));
  return VXS_OK;
}

extern "C" int vxs_factor_read_back(vxs_factor* f, double* eig12, double* sum10) {
  if (!f || !f->ctx) return VXS_ERR_ARG;
  vxs_ctx* ctx = f->ctx;
  cudaSetDevice(ctx->device);
  const size_t n = size_t(f->V);
  if (n == 0) return VXS_OK;
  { int rcw = vxs_factor_wait_uploads(f); if (rcw) return rcw; }
  cudaStream_t s = ctx->stream;
  VXS_CUDA(ctx, ctx->stage.reserve(n * 22));
  if (eig12) {
    VXS_LAUNCH(ctx, "k_soa_to_aos", k_soa_to_aos, nblk(n * 12, 256), 256, 0, f->eig, ctx->stage.p, n, 12, f->Vcap);
    VXS_CUDA(ctx, cudaMemcpyAsync(eig12, ctx->stage.p, n * 12 * 8, cudaMemcpyDeviceToHost, s));
  }
  if (sum10) {
    VXS_LAUNCH(ctx, "k_soa_to_aos", k_soa_to_aos, nblk(n * 10, 256), 256, 0, f->sum, ctx->stage.p + n * 12, n, 10, f->Vcap);
    VXS_CUDA(ctx, cudaMemcpyAsync(sum10, ctx->stage.p + n * 12, n * 10 * 8, cudaMemcpyDeviceToHost, s));
  }
  VXS_CUDA(ctx, cudaStreamSynchronize(s));
  return VXS_OK;
}

extern "C" int vxs_factor_read_structure(vxs_factor* f, int64_t* entry_ptr, int32_t* entry_frame, double* entry_cluster10, double* fix10, double* coe) {
  if (!f || !f->ctx) return VXS_ERR_ARG;
  vxs_ctx* ctx = f->ctx;
  cudaSetDevice(ctx->device);
  const size_t n = size_t(f->V), ne = size_t(f->E);
  { int rcw = vxs_factor_wait_uploads(f); if (rcw) return rcw; }
  cudaStream_t s = ctx->stream;
  if (entry_ptr) {
    std::vector<int32_t> p32(n + 1, 0);
    if (n) VXS_CUDA(ctx, cudaMemcpyAsync(p32.data(), f->ptr, (n + 1) * 4, cudaMemcpyDeviceToHost, s));
    VXS_CUDA(ctx, cudaStreamSynchronize(s));
    for (size_t i = 0; i <= n; i++) entry_ptr[i] = p32[i];
  }
  if (n == 0) return VXS_OK;
  if (entry_frame && ne) VXS_CUDA(ctx, cudaMemcpyAsync(entry_frame, f->frame, ne * 4, cudaMemcpyDeviceToHost, s));
  VXS_CUDA(ctx, ctx->stage.reserve(std::max(ne * 10, n * 10)));
  if (entry_cluster10 && ne) {
    VXS_LAUNCH(ctx, "k_soa_to_aos", k_soa_to_aos, nblk(ne * 10, 256), 256, 0, f->cl, ctx->stage.p, ne, 10, f->Ecap);
    VXS_CUDA(ctx, cudaMemcpyAsync(entry_cluster10, ctx->stage.p, ne * 10 * 8, cudaMemcpyDeviceToHost, s));
    VXS_CUDA(ctx, cudaStreamSynchronize(s));
  }
  if (fix10) {
    VXS_LAUNCH(ctx, "k_soa_to_aos", k_soa_to_aos, nblk(n * 10, 256), 256, 0, f->fix, ctx->stage.p, n, 10, f->Vcap);
    VXS_CUDA(ctx, cudaMemcpyAsync(fix10, ctx->stage.p, n * 10 * 8, cudaMemcpyDeviceToHost, s));
  }
  if (coe) VXS_CUDA(ctx, cudaMemcpyAsync(coe, f->coe, n * 8, cudaMemcpyDeviceToHost, s));
  VXS_CUDA(ctx, cudaStreamSynchronize(s));
  return VXS_OK;
}
