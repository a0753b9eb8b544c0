// Device-side view of a vxs_factor (CSR over the frames that observe each voxel, SoA clusters) and the load helpers shared by the
// evaluation kernels (vxs_eval.cu, vxs_resid.cu).
#pragma once
#include "vxs_internal.h"
#include "vxs_math.cuh"

using namespace vxs;

struct FactorView {
  const int32_t* ptr; const int32_t* frame;
  const double* cl; size_t Ecap;
  const double* fix; const double* coe;
  double* eig; double* sum; size_t Vcap;
  const double* vc;     // [8][Vcap] per-voxel constants of acc_evaluate2 (k_voxel_consts)
  int V; int W; int has_fix;
};
static inline FactorView make_view(const vxs_factor* f) {
  FactorView v;
  v.ptr = f->ptr; v.frame = f->frame; v.cl = f->cl; v.Ecap = f->Ecap; v.fix = f->fix; v.coe = f->coe; v.eig = f->eig; v.sum = f->sum;
  v.Vcap = f->Vcap; v.V = int(f->V); v.W = f->W; v.has_fix = f->has_fix ? 1 : 0; v.vc = f->vc.p;
  return v;
}

__device__ __forceinline__ cluster load_cluster_soa(const double* __restrict__ base, size_t stride, size_t i) {
  cluster c;
  c.P.xx = __ldg(base + i); c.P.xy = __ldg(base + stride + i); c.P.xz = __ldg(base + 2 * stride + i);
  c.P.yy = __ldg(base + 3 * stride + i); c.P.yz = __ldg(base + 4 * stride + i); c.P.zz = __ldg(base + 5 * stride + i);
  c.v.x = __ldg(base + 6 * stride + i); c.v.y = __ldg(base + 7 * stride + i); c.v.z = __ldg(base + 8 * stride + i);
  c.n = __ldg(base + 9 * stride + i);
  return c;
}
__device__ __forceinline__ void load_pose(const double* __restrict__ poses, int stride, int fr, rot3& R, d3& t) {
  const double* p = poses + size_t(fr) * stride;
  R.r00 = __ldg(p); R.r01 = __ldg(p + 1); R.r02 = __ldg(p + 2); R.r10 = __ldg(p + 3); R.r11 = __ldg(p + 4); R.r12 = __ldg(p + 5);
  R.r20 = __ldg(p + 6); R.r21 = __ldg(p + 7); R.r22 = __ldg(p + 8);
  t = mk3(__ldg(p + 9), __ldg(p + 10), __ldg(p + 11));
}

// Poses staged once per CTA in shared memory, component-major [12][W]: lanes of a group read consecutive frames, so each of the 12
// reads is one conflict-free wavefront instead of a 96-byte-strided global gather (the LSU, not DRAM, bounds these kernels).
__device__ __forceinline__ void stage_poses(double* sp, const double* __restrict__ poses, int pstride, int W) {
  for (int i = threadIdx.x; i < 12 * W; i += blockDim.x) { const int fr = i / 12, c = i - fr * 12; sp[c * W + fr] = __ldg(poses + size_t(fr) * pstride + c); }
  __syncthreads();
}
__device__ __forceinline__ void load_pose_s(const double* sp, int W, int fr, rot3& R, d3& t) {
  R.r00 = sp[fr]; R.r01 = sp[W + fr]; R.r02 = sp[2 * W + fr]; R.r10 = sp[3 * W + fr]; R.r11 = sp[4 * W + fr]; R.r12 = sp[5 * W + fr];
  R.r20 = sp[6 * W + fr]; R.r21 = sp[7 * W + fr]; R.r22 = sp[8 * W + fr];
  t = mk3(sp[9 * W + fr], sp[10 * W + fr], sp[11 * W + fr]);
}

// L2 prefetch of the cluster columns (and frame index) of entry e: the evaluation kernels are latency-bound at their register-limited
// occupancy (ncu: long-scoreboard stalls dominate), so each group pulls the entries of its NEXT voxel towards L2 one iteration ahead.
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_entry(const FactorView& f, int e) {
  if (size_t(e) >= f.Ecap) return;
#pragma unroll
  for (int c = 0; c < 10; c++) prefetch_l2(f.cl + size_t(c) * f.Ecap + e);
  prefetch_l2(f.frame + e);
}

