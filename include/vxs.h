/* vxs.h — C-ABI of the H100-native Voxel-SLAM bundle-adjustment hot path (libvxs.so).
 *
 * The reference (hku-mars/Voxel-SLAM, one ROS C++ executable) has no plugin/FFI layer: the boundary of this path is
 * the C++ call surface used by VoxelSLAM/src/voxelslam.cpp.  Every entry point below names the reference interface it
 * replaces (file:line into Voxel-SLAM/VoxelSLAM/src/).  A header-only C++ shim with the reference's class names
 * on top of this ABI is in voxel_slam_b200/csrc/shim/voxel_ba_shim.hpp; INTEGRATION.md shows the binding.
 *
 * Conventions
 *  - plain C types only; all pointers are HOST pointers unless the name says _dev; caller owns every buffer.
 *  - every function returns an int status (VXS_OK = 0, <0 error, >0 warning); nothing ever calls exit()
 *    (the reference printf+exit(0)s, voxel_map.hpp:345-348, 1211-1215).
 *  - one vxs_ctx per calling thread (the reference runs local BA and global BA on two threads concurrently,
 *    voxelslam.cpp:2617-2619); a ctx owns its CUDA stream(s) and scratch memory; calls on one ctx are synchronous.
 *  - there is NO CPU fallback: without a CUDA device vxs_ctx_create fails with VXS_ERR_CUDA.
 *  - layouts: pose12 = R row-major (9) | p (3).  state24 = R (9) | p | v | bg | ba | g  (tools.hpp:135-145 IMUST without t, cov).
 *    cluster10 = Pxx Pxy Pxz Pyy Pyz Pzz vx vy vz N  (tools.hpp:304-310 PointCluster, symmetric P packed, N as double).
 *    eig12 = lambda0..2 (ascending) | U row-major 3x3, eigenvectors in COLUMNS (Eigen convention, voxel_map.hpp:163-168).
 *    Hessians are column-major n x n like Eigen::MatrixXd.
 */
#ifndef VXS_H
#define VXS_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define VXS_OK 0
#define VXS_ERR_CUDA (-1)
#define VXS_ERR_ARG (-2)
#define VXS_ERR_TOO_FEW_VOXELS (-3) /* reference: "Too Less Voxel" exit(0), voxel_map.hpp:345-348 */
#define VXS_ERR_COMM (-4)
#define VXS_ERR_NOMEM (-5)
#define VXS_ERR_RANGE (-6)   /* voxel coordinate outside the packable range (see vxs_build_*) */
#define VXS_ERR_CALLBACK (-7)
#define VXS_WARN_SINGULAR 1  /* a zero pivot was met in the LDLT (Eigen would continue with zeros) */

typedef struct vxs_ctx vxs_ctx;
typedef struct vxs_factor vxs_factor;

/* ---------------------------------------------------------------- context */
int vxs_version(void);
int vxs_ctx_create(int device, vxs_ctx** out);
int vxs_ctx_destroy(vxs_ctx* ctx);
const char* vxs_ctx_last_error(const vxs_ctx* ctx);
/* pinned host memory for callers that want full-speed H2D/D2H (optional) */
int vxs_host_alloc(void** out, uint64_t bytes);
int vxs_host_free(void* p);
/* kernels launched by this ctx since creation (bench.py's gpu_launches) */
int64_t vxs_ctx_launch_count(const vxs_ctx* ctx);
/* per-stage CUDA-event timing on the ctx stream: enable, run calls, then read the accumulated stages.
 * names: up to cap stage names (static strings), ms_total / calls per stage.  Stage names are the kernel names. */
int vxs_ctx_timing_enable(vxs_ctx* ctx, int on);
int vxs_ctx_timing_read(vxs_ctx* ctx, int cap, const char** names, double* ms_total, int64_t* calls, int* n_out);
int vxs_ctx_timing_reset(vxs_ctx* ctx);
/* one CUDA-event stopwatch on the ctx stream (bench.py times its K steps with it): start records an event, stop records a
 * second one, synchronises and returns the elapsed device time in milliseconds */
int vxs_ctx_timer_start(vxs_ctx* ctx);
int vxs_ctx_timer_stop(vxs_ctx* ctx, double* ms);
/* diagnostics: measured fp64 FMA throughput of this device (TFLOP/s, 2 flop per FMA) — the roofline denominator of the
 * SYRK part of the Hessian, which MEASURED_PEAKS.json does not carry */
int vxs_diag_fp64_tflops(vxs_ctx* ctx, double* tflops);
/* same for the fp64 tensor-core path, in the MMA shape the SYRK issues (mma.sync.m16n8k4.f64, SASS DMMA.16x8x4) */
int vxs_diag_dmma_tflops(vxs_ctx* ctx, double* tflops);
/* measured throughput (TFLOP/s) of each fp64 mma.sync shape: tflops[0..3] = m8n8k4, m16n8k4, m16n8k8, m16n8k16 */
int vxs_diag_dmma_shapes(vxs_ctx* ctx, double tflops[4]);
/* damped solve of a synthetic n x n system: out[0] = ms per solve (events), out[1..4] = us per 32-column panel that CTA 0 spends in
 * {panel load, strip solve, Schur update, grid barrier}, out[5] = panels, out[6] = SM clock (kHz) used for the conversion,
 * out[7] = us per panel of the look-ahead diagonal factor, out[8] = residual |(H + u diag H) dx + g|_inf / |g|_inf of the solve
 * checked on the host, out[9..11] reserved (0).
 * VXS_LDLT_LOOKAHEAD_CTA=0 in the environment keeps the look-ahead on CTA 0 (A/B switch). */
int vxs_diag_ldlt_phases(vxs_ctx* ctx, int n, double out[12]);
/* the damped, gauge-fixed solve of the LM drivers on a caller-supplied n x n system (column-major hess, jact; host buffers):
 * rows / columns < gauge zeroed with an identity block, D = diag, dx = (H + u D)^-1 (-jact) by the pivoted LDL^T the solvers use
 * (voxel_map.hpp:397-403, 591-597, 800-811).  For parity tests of the solver at the headline sizes (n = 750, 753, ...). */
int vxs_diag_solve_damped(vxs_ctx* ctx, const double* hess, const double* jact, int n, int gauge, double u, double* dx, int* singular);

/* ---------------------------------------------------------------- multi-GPU (one process per GPU; NCCL over NVLink)
 * Voxel-sharded BA: every rank holds the factor voxels it owns and the replicated poses; [H_lidar, g, r] are
 * all-reduced once per Hessian build and the scalar residual once per residual evaluation (SURVEY.md §8e). */
int vxs_comm_unique_id(unsigned char id[128]);
int vxs_ctx_comm_init(vxs_ctx* ctx, const unsigned char id[128], int rank, int nranks);
int vxs_ctx_comm_destroy(vxs_ctx* ctx);

/* ---------------------------------------------------------------- LidarFactor  (voxel_map.hpp:109-290) */
int vxs_factor_create(vxs_ctx* ctx, int win_size, vxs_factor** out);          /* LidarFactor(int _w)      :120 */
int vxs_factor_destroy(vxs_factor* f);
int vxs_factor_clear(vxs_factor* f);                                            /* LidarFactor::clear       :281 */
int vxs_factor_set_win_size(vxs_factor* f, int win_size);                       /* voxhess.win_size = ...   voxelslam.cpp:1609 */
/* Batched LidarFactor::push_voxel (:122-130).  CSR over the frames that observe each voxel (N != 0), frames ascending
 * within a voxel.  fix10 may be NULL (all-zero fix clusters), coe may be NULL (all 1.0, voxel_map.hpp:1316). */
int vxs_factor_push_voxels(vxs_factor* f, int64_t n_vox, const int64_t* entry_ptr, const int32_t* entry_frame,
                           const double* entry_cluster10, const double* fix10, const double* coe, const double* eig12,
                           const double* sum10);
/* Asynchronous variant for an EMPTY factor (the per-solve upload of the shim): returns as soon as the copies are queued.  The bulk
 * (clusters, 80 B per entry) travels on a copy stream in chunks of whole voxel groups and the first Hessian build of the next
 * vxs_lidar_ba / vxs_li_ba runs chunk by chunk behind it, so the PCIe transfer overlaps the Jacobian and SYRK kernels.  The host
 * buffers must stay valid — and should be pinned (vxs_host_alloc) — until that solve (or vxs_factor_sync_uploads) has returned.
 * Falls back to the synchronous vxs_factor_push_voxels when the factor is not empty or the push is tiny. */
int vxs_factor_push_voxels_async(vxs_factor* f, int64_t n_vox, const int64_t* entry_ptr, const int32_t* entry_frame,
                                 const double* entry_cluster10, const double* fix10, const double* coe, const double* eig12,
                                 const double* sum10);
int vxs_factor_sync_uploads(vxs_factor* f);   /* host-side wait for everything queued by the async push */
/* Same, in the reference's dense layout vector<vector<PointCluster>>: clusters10 is [n_vox][win_size][10], N==0 = absent. */
int vxs_factor_push_voxels_dense(vxs_factor* f, int64_t n_vox, const double* clusters10, const double* fix10,
                                 const double* coe, const double* eig12, const double* sum10);
int vxs_factor_counts(const vxs_factor* f, int64_t* n_vox, int64_t* n_entries, int* win_size);
/* eig_values / eig_vectors / pcr_adds as left by the last residual evaluation (read by OctoTree::margi :1217-1222) */
int vxs_factor_read_back(vxs_factor* f, double* eig12, double* sum10);
/* Keep / restore a device-side copy of the cached eig / pcr_adds.  A solve overwrites the cache (voxel_map.hpp:271-273); callers
 * that re-run a solve from the same map state (bench.py's repeated steps, motion_init retries) restore it instead of re-pushing. */
int vxs_factor_cache_save(vxs_factor* f);
int vxs_factor_cache_restore(vxs_factor* f);
/* the stored structure (for tests and for callers that keep the factor device-resident) */
int vxs_factor_read_structure(vxs_factor* f, int64_t* entry_ptr, int32_t* entry_frame, double* entry_cluster10,
                              double* fix10, double* coe);

/* LidarFactor::evaluate_only_residual(xs, 0, size, residual)  :243-279 — overwrites the cached eig / sum */
int vxs_factor_evaluate_residual(vxs_ctx* ctx, vxs_factor* f, const double* poses12, double* residual);
/* LidarFactor::acc_evaluate2(xs, 0, size, Hess, JacT, residual)  :132-241 — uses the CACHED eig / sum.
 * hess: (6W x 6W) column-major, jact: 6W. */
int vxs_factor_evaluate_hessian(vxs_ctx* ctx, vxs_factor* f, const double* poses12, double* hess, double* jact,
                                double* residual);

/* ---------------------------------------------------------------- LM solvers */
typedef struct vxs_lm_trace { double r1, r2, u, v, q1; int32_t accepted; int32_t hess_built; } vxs_lm_trace;

/* Lidar_BA_Optimizer::damping_iter(x_stats, voxhess, hess, resis, max_iter)  voxel_map.hpp:367-442.
 * poses12 in/out (W x 12).  hess_out (6W x 6W col-major, may be NULL) = raw Hessian of the last build (:391).
 * resis[2] = {first residual1, last residual2} (:394-395,440).  thd_num only reproduces the reference's
 * "voxels < threads" error (VXS_ERR_TOO_FEW_VOXELS); pass Lidar_BA_Optimizer::thd_num (:296).
 * trace (may be NULL): up to trace_cap entries, *trace_len written. */
int vxs_lidar_ba(vxs_ctx* ctx, vxs_factor* f, double* poses12, int max_iter, int thd_num, double* hess_out,
                 double resis[2], int* is_converge, vxs_lm_trace* trace, int trace_cap, int* trace_len);

/* The IMU factor stays on the CPU (preintegration.hpp, out of scope); the LI solvers call back into it.
 *  eval     : sum over the W-1 factors of IMU_PRE::give_evaluate (:137) or give_evaluate_g (:214).  states: W x 24.
 *             if want_jac: blocks[(W-1)][bs*bs] column-major and gvec[(W-1)][bs], bs = 30 (33 with gravity);
 *             *cost = sum of r^T cov^-1 r (unscaled; the solver applies imu_coef, voxel_map.hpp:505-507).
 *  update   : IMU_PRE::update_state(dxi.block<15,1>(15 j)) for every factor j (:296; voxel_map.hpp:608-609)
 *  rollback : dbg = dbg_buf, dba = dba_buf (voxel_map.hpp:639-643)
 * Callbacks return 0 on success. */
typedef struct vxs_imu_hooks {
  void* user;
  int (*eval)(void* user, const double* states24, int W, int with_gravity, int want_jac, double* blocks, double* gvec, double* cost);
  int (*update)(void* user, const double* dxi, int W);
  int (*rollback)(void* user);
} vxs_imu_hooks;

/* LI_BA_Optimizer::damping_iter (voxel_map.hpp:562-653; with_gravity=0, n=15W; the reference hard-codes 3 iterations, :581 —
 * max_iter > 3 is clamped to 3, smaller values step fewer iterations)
 * and LI_BA_OptimizerGravity::damping_iter (:775-862; with_gravity=1, n=15W+3, max_iter default 2).
 * states24 in/out (W x 24); hess_out (n x n col-major, may be NULL); resis[2] as above; imu_coef = voxel_map.hpp:446. */
int vxs_li_ba(vxs_ctx* ctx, vxs_factor* f, double* states24, int with_gravity, int max_iter, double imu_coef,
              const vxs_imu_hooks* imu, double* hess_out, double resis[2], vxs_lm_trace* trace, int trace_cap,
              int* trace_len);

/* ---------------------------------------------------------------- voxel map (build-from-scratch semantics) */
typedef struct vxs_map_params {
  double voxel_size;        /* voxel_map.hpp:87 / gba_voxel_size loop_refine.hpp:271 */
  double min_eigen_value;   /* voxel_map.hpp:84 / loop_refine.hpp:270 */
  double plane_thre[4];     /* plane_eigen_value_thre, already inverted (voxelslam.cpp:825 / :2490) */
  double min_point[4];      /* voxel_map.hpp:83 min_point (voxelslam.cpp:812 sets 5,5,5,5); ignored by the GBA map (literal 10) */
  int32_t max_layer;        /* voxel_map.hpp:85 */
  int32_t reserved;
} vxs_map_params;

/* voxel quantisation + hash, bit-exact (voxel_map.hpp:1511-1518, tools.hpp:24-49): xyz[n][3], hash[n] */
int vxs_voxel_keys(vxs_ctx* ctx, const double* pw, int64_t n, double voxel_size, int64_t* xyz, uint64_t* hash);

/* Identity of a factor voxel for order-independent comparison: root cell + layer + octant path (sum leaf_l * 8^(depth-l)). */
typedef struct vxs_voxel_id { int64_t x, y, z; int32_t layer; int32_t path; } vxs_voxel_id;

/* cut_voxel for every scan of the window (voxel_map.hpp:1504-1540) then OctoTree::recut + tras_opt on every root
 * (voxel_map.hpp:1148-1194, 1308-1333) — the from-scratch sequence of voxelslam.cpp:600-628 / 1171-1180.
 * pts_body: all scans concatenated (fp64 xyz, body frame), scan_offsets[W+1]; poses12: W x 12.
 * fix_pts (may be NULL): already-world fixed map points (cut_voxel :1641-1671).  The factor `out` is cleared and refilled
 * (device-resident; nothing is copied back unless ids_out / vxs_factor_read_* are used).
 * ids_out (may be NULL, capacity ids_cap): identity of every factor voxel in factor order; *n_out = number of voxels. */
int vxs_build_window_factor(vxs_ctx* ctx, const vxs_map_params* mp, const double* pts_body, const int64_t* scan_offsets,
                            const double* poses12, int W, const double* fix_pts, int64_t n_fix, vxs_factor* out,
                            vxs_voxel_id* ids_out, int64_t ids_cap, int64_t* n_out);

/* OctreeGBA::cut_voxel for every keyframe + OctreeGBA_multi_recut (loop_refine.hpp:446-479, 483-537).
 * xyz: float points of all keyframes concatenated (x,y,z per point, stride_floats between points: 3 for packed xyz,
 * 12 for pcl::PointXYZINormal), kf_offsets[W+1] in points. */
int vxs_build_gba_factor(vxs_ctx* ctx, const vxs_map_params* mp, const float* xyz, int stride_floats,
                         const int64_t* kf_offsets, const double* poses12, int W, vxs_factor* out, vxs_voxel_id* ids_out,
                         int64_t ids_cap, int64_t* n_out);

/* The BA loop of HBA_add_edge (voxelslam.cpp:2360-2399): per outer iteration rebuild the GBA map at the current poses,
 * recut, Lidar_BA_Optimizer::damping_iter(up=4); coarse-to-fine switch to `fine` on convergence / last iteration.
 * poses12 in/out; hess_out (6W x 6W) = raw Hessian of the last build (consumed by the PGO edge extraction :2405-2427).
 * resis_log (may be NULL, 2 doubles per outer iteration); *outer_iters = iterations run. */
int vxs_hba_window(vxs_ctx* ctx, const vxs_map_params* coarse, const vxs_map_params* fine, const float* xyz,
                   int stride_floats, const int64_t* kf_offsets, double* poses12, int W, int max_iter, int thread_num,
                   double* hess_out, double* resis_log, int* outer_iters);

/* The BOTTOM level of the hierarchical global BA as one batch: thd_globalmapping (voxelslam.cpp:2484-2557) calls
 *     HBA_add_edge(xs, smp_local, gba_edges1, mps, max_iter = 1, thread_num = 2, plptr)
 * once per window of win_size = 10 keyframes (stride mgsize = 5): with max_iter = 1 that is ONE map build with the fine parameters
 * (:2362-2372), OctreeGBA_multi_recut, Lidar_BA_Optimizer::damping_iter(up = 4) and the PGO edges (:2405-2427) — hundreds of independent
 * 6*win_size-dof problems.  Here all windows of a chunk are built, solved (LM loop on the device, block-diagonal Hessian, one CTA per window
 * for the solve) and read back together.  Windows are independent, so a multi-GPU run simply gives every rank its share of `win_first`.
 *   xyz / kf_offsets / poses12: all K keyframes (clouds as in vxs_build_gba_factor, poses = the keyframes' x0); win_first[w] = first keyframe of window w.
 *   max_points_per_chunk (<= 0: default 96 Mi): bound on the points of the windows processed together (device memory).
 *   poses_out [nwin][win_size][12]: the windows' refined copies of the poses (the keyframes themselves are not moved, as in the reference);
 *   resis [nwin][2]; status [nwin]: 0, VXS_WARN_SINGULAR or VXS_ERR_TOO_FEW_VOXELS (the reference would exit(0), voxel_map.hpp:345-348 — such a
 *   window keeps its poses, reports is_converge = 0 and resis = {residual1 at its poses, 0}, as damping_iter leaves them at that exit); is_converge / lm_iters [nwin]; edges: for pair p = (i, j), i < j in lexicographic order, P = win_size (win_size - 1) / 2
 *   per window: edge_valid [nwin][P], edge_v6 [nwin][P][6], edge_rot [nwin][P][9], edge_tra [nwin][P][3]; hess_out (may be NULL)
 *   [nwin][(6 win_size)^2] column-major raw Hessians.  Every output but poses_out may be NULL.
 * The submap merge of the reference's post-step (:2428-2447) stays a per-window call (vxs_submap_merge). */
int vxs_hba_bottom_batch(vxs_ctx* ctx, const vxs_map_params* fine, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, int K,
                         const int32_t* win_first, int nwin, int win_size, int thread_num, int64_t max_points_per_chunk, double* poses_out, double* resis, int32_t* status,
                         int32_t* is_converge, int32_t* lm_iters, int32_t* edge_valid, double* edge_v6, double* edge_rot, double* edge_tra, double* hess_out);

/* One PASS of the hierarchical global BA (thd_globalmapping, voxelslam.cpp:2484-2557) over K keyframes, single- or multi-GPU (the ranks of vxs_ctx_comm_init):
 *   windows w = 0 .. nwin-1, nwin = (K - win_size) / win_stride + 1, first keyframe w * win_stride (the reference: win_size 10, stride 5, :2501-2502);
 *   rank r of n takes the contiguous share [nwin r / n, nwin (r + 1) / n) of the bottom level: vxs_hba_bottom_batch + vxs_submap_merge_batch on keyframe clouds that are
 *   uploaded once and on merged submaps that STAY on the device; the submaps are exchanged between the ranks' device buffers over NCCL; the top level
 *   (HBA_add_edge over all submaps, W = nwin, top_max_iter = GBA/total_max_iter, thread_num 5, :2538) runs voxel-sharded with the all-reduced Hessian.
 * Outputs (host): bottom_* for THIS rank's windows only (layouts of vxs_hba_bottom_batch; *my_first_window / *my_window_count say which), top_poses [nwin][12]
 * (identical on every rank), top_resis_log [2 top_max_iter], submap_sizes [nwin] (cells per merged submap), phase_ms [6] = device time of
 * {upload + bottom BA, merge, exchange, top}, then the plane voxels and (voxel, keyframe) clusters of this rank's bottom windows.  Every bottom_* / top_resis_log / submap_sizes / phase_ms pointer but bottom_poses may be NULL. */
int vxs_hba_pass(vxs_ctx* ctx, const vxs_map_params* coarse, const vxs_map_params* fine, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, int K,
                 int win_size, int win_stride, int bottom_thread_num, int top_thread_num, int top_max_iter, int64_t max_points_per_chunk, double* bottom_poses, double* bottom_resis,
                 int32_t* bottom_status, int32_t* bottom_edge_valid, double* bottom_edge_v6, double* bottom_edge_rot, double* bottom_edge_tra, int32_t* my_first_window,
                 int32_t* my_window_count, double* top_poses, double* top_resis_log, int* top_outer_iters, int64_t* submap_sizes, double* phase_ms);

/* PGO edge extraction of HBA_add_edge (voxelslam.cpp:2405-2427) from the raw Hessian of the LAST vxs_lidar_ba / vxs_hba_window
 * on this ctx, without downloading the Hessian: for every pair i<j whose six diagonal entries of block (i,j) are all >= 1e-6 in
 * magnitude, one edge with variance v6[k] = 1/|H(6i+k, 6j+k)|, rot = R_i^T R_j (row-major), tra = R_i^T (p_j - p_i).
 * edge_ij: [cap][2] int32, v6: [cap][6], rot: [cap][9], tra: [cap][3]; *n_edges = number found (may exceed cap: truncated).
 * Edges come out in the reference's lexicographic (i, j) order, the same on every run (and the first `cap` of them when truncated).
 * VXS_ERR_ARG when the Hessian resident on the ctx is not the lidar-only 6W system of a BA with this W. */
int vxs_hba_edges(vxs_ctx* ctx, int W, const double* poses12, int64_t cap, int32_t* edge_ij, double* v6, double* rot, double* tra,
                  int64_t* n_edges);

/* ---------------------------------------------------------------- voxel-grid down-sampling (SURVEY.md §8f rows 2 and 4)
 * down_sampling_voxel (tools.hpp:201-238; callers voxelslam.cpp:2440 submap merge, :1146 / :2118 scan pre-processing): one point per
 * occupied cell of size voxel_size, the running FLOAT mean of the cell's points taken in input order (bit-exact, order dependent).
 * down_sampling_close (tools.hpp:240-302): one INPUT point per cell, the one nearest to the cell's float centroid.
 * pts: n points, x,y,z float at the start of each point, stride_floats between points (3 packed, 12 for pcl::PointXYZINormal).
 * Outputs (each may be NULL, capacity cap): xyz_out[.][3]; count_out = points in the cell (the reference stores it in `curvature`);
 * index_out = input index of the cell's FIRST point (voxel: the point whose other fields the reference keeps) / of the PICKED point
 * (close).  Cells come out in ascending (x, y, z) cell order (the reference's unordered_map order is unspecified).
 * *n_out = number of cells, or -1 when voxel_size < 0.001 (the reference returns with the cloud untouched). */
int vxs_down_sampling_voxel(vxs_ctx* ctx, const float* pts, int stride_floats, int64_t n, double voxel_size, float* xyz_out, float* count_out,
                            int64_t* first_index_out, int64_t cap, int64_t* n_out);
int vxs_down_sampling_close(vxs_ctx* ctx, const float* pts, int stride_floats, int64_t n, double voxel_size, float* xyz_out, float* count_out,
                            int64_t* picked_index_out, int64_t cap, int64_t* n_out);

/* down_sampling_pvec (voxel_map.hpp:23-64, the scan pre-processing of the odometry): pointVar records (`stride_doubles` >= 12 apart: pnt at
 * [0..2], the symmetric 3x3 var at [3..11]); per cell the running fp64 mean of pnt and var in input order; out: float(pnt), float(diag(var))
 * (what the reference writes to x,y,z / normal_x,y,z), the cell's point count and the index of its first point; cells in ascending cell order. */
int vxs_down_sampling_pvec(vxs_ctx* ctx, const double* pv, int stride_doubles, int64_t n, double voxel_size, float* xyz_out, float* var_diag_out,
                           float* count_out, int64_t* first_index_out, int64_t cap, int64_t* n_out);

/* Submap merge of HBA_add_edge (voxelslam.cpp:2428-2447): the clouds of the W keyframes of a window are moved into the frame of
 * keyframe 0 (v' = dR v + dp in fp64, dR = R_0^T R_i, dp = R_0^T (p_i - p_0), stored as float) and passed through
 * down_sampling_voxel(voxel_size) — the caller passes the reference's voxel_size / 8.  Outputs as vxs_down_sampling_voxel;
 * first_index_out indexes the concatenated input, so the keyframe of a surviving point (the reference stores its map id in
 * `intensity`) follows from kf_offsets.  voxel_size < 0.001: the merged cloud is returned as it is (count 0). */
int vxs_submap_merge(vxs_ctx* ctx, const float* xyz, int stride_floats, const int64_t* kf_offsets, const double* poses12, int W,
                     double voxel_size, float* xyz_out, float* count_out, int64_t* first_index_out, int64_t cap, int64_t* n_out);

/* The same for MANY windows at once (the post-step of every bottom-level HBA_add_edge, after vxs_hba_bottom_batch): poses_win [nwin][win_size][12] are the
 * windows' refined poses, window w merges keyframes win_first[w] .. win_first[w] + win_size - 1 into the frame of its first keyframe and down-samples.
 * Outputs are the windows' clouds back to back, win_offsets[nwin + 1] delimits them (cells of a window in ascending cell order); first_index_out indexes the
 * window's own concatenated input.  *n_out = total cells (may exceed cap: truncated).  voxel_size >= 0.001 (the reference's voxel_size / 8). */
int vxs_submap_merge_batch(vxs_ctx* ctx, const float* xyz, int stride_floats, const int64_t* kf_offsets, int K, const double* poses_win, const int32_t* win_first, int nwin, int win_size,
                           double voxel_size, int64_t max_points_per_chunk, float* xyz_out, float* count_out, int64_t* first_index_out, int64_t cap, int64_t* win_offsets, int64_t* n_out);

/* ---------------------------------------------------------------- odometry association (SURVEY.md §8f rank 3)
 * The per-point loop of the EKF update (voxelslam.cpp:876-918): world point and its covariance, match() against the voxel map
 * (voxel_map.hpp:1674-1698, 1335-1392), HTH += R_inv jac jac^T, HTz -= R_inv jac resi, nnt += n n^T, match_num++.
 * vxs_odom_set_planes: the plane leaves of the current map, exported by the caller after every marginalisation (the octree stays on
 * the host until §8f rank 1 lands): cube centre (OctoTree::voxel_center) and layer, plane.center / normal / plane_var (6x6 row-major)
 * / radius as written by plane_update (voxel_map.hpp:1118-1146).  Leaves with plane.radius == 0 never match and may be left out.
 * vxs_odom_accumulate: pv12 = n pointVar records (pnt 3 | var 3x3 row-major), NULL = re-use the scan of the previous call;
 * pose12 = R row-major | p of x_curr; rot_var9 / tsl_var9 = x_curr.cov blocks (0,0) and (3,3).  flags (may be NULL): 1 where the point matched. */
int vxs_odom_set_planes(vxs_ctx* ctx, const vxs_map_params* mp, int64_t n, const double* voxel_center, const int32_t* layer, const double* center,
                        const double* normal, const double* plane_var36, const float* radius);
int vxs_odom_accumulate(vxs_ctx* ctx, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9,
                        double* HTH36, double* HTz6, double* nnt9, int64_t* match_num, int32_t* flags);
/* lio_state_estimation (voxelslam.cpp:856-958) in one call against the table of vxs_odom_set_planes; arguments, outputs and errors as
 * vxs_map_lio_update (below), which shares its driver and its step kernel. */
int vxs_odom_lio_update(vxs_ctx* ctx, const double* pv12, int64_t n, double* state24, double* cov225, int32_t* ok, int32_t* iters, int64_t* match_num,
                        double* trace12, int32_t* flags);

/* Point variances of a scan (voxelslam.hpp:187-214; call sites voxelslam.cpp:1246-1250, 1584-1594), the step between down-sampling and the EKF:
 *   vxs_var_init    = var_init: per point calcBodyVar (voxelslam.hpp:163-184: range / bearing noise, dept_err and beam_err narrow to float at the
 *                     call as in the reference; a point with z == 0 gets z = 0.0001) then the extrinsic, pnt = ext.R pnt + ext.p,
 *                     var = ext.R var ext.R^T.  pts: x, y, z float at the start of each point, stride_floats apart (12 for PointType).
 *                     pv12_out (host, may be NULL): n pointVar records (pnt 3 | var 3x3 row-major).  The records also STAY on the device as the
 *                     ctx's resident scan: vxs_odom_accumulate / vxs_map_odom_accumulate / vxs_pvec_update / vxs_map_push_scan take pv12 = NULL.
 *   vxs_pvec_update = pvec_update: var = R var R^T + hat(pnt) rot_var hat(pnt)^T + tsl_var in place (pnt stays in the body frame),
 *                     pwld = R pnt + p.  pv12 (host) may be NULL = the resident scan; pv12_out / pwld_out (host, n x 12 / n x 3) may be NULL. */
int vxs_var_init(vxs_ctx* ctx, const float* pts, int stride_floats, int64_t n, const double* ext_R9, const double* ext_p3, double dept_err, double beam_err, double* pv12_out);
int vxs_pvec_update(vxs_ctx* ctx, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, double* pv12_out, double* pwld_out);

/* ---------------------------------------------------------------- persistent local map of the sliding-window loop (SURVEY.md §8f rank 1)
 * The device-resident counterpart of `surf_map` / `surf_map_slide` (unordered_map<VOXEL_LOC, OctoTree*>, voxelslam.hpp) and of the per-scan
 * calls around the BA in thd_odometry_localmapping (voxelslam.cpp:1599-1712).  A scan is uploaded ONCE; the map, the slide windows
 * (SlideWindow, voxel_map.hpp:896-930), the raw points that are still re-cuttable and the marginalised points kept in point_fix stay in HBM.
 *   vxs_map_push_scan = cut_voxel_multi (voxel_map.hpp:1543-1639; single-thread form cut_voxel :1504-1540) of the NEW scan at window position
 *                       win_count-1 + multi_recut (voxelslam.cpp:1398-1453: OctoTree::recut :1148-1194 on every slide root, then tras_opt
 *                       :1308-1333) — `out` receives the LidarFactor of the window (cleared first; may be NULL).
 *                       pv12: n pointVar records (body-frame pnt 3 | var 3x3 row-major, as pvec_update left it, voxelslam.hpp:203-214); NULL = the ctx's
 *                       resident scan (vxs_var_init / vxs_pvec_update), copied device to device;
 *                       poses12: x_buf, win_count poses INCLUDING the new scan's (R row-major | p).
 *   vxs_map_margi     = multi_margi (voxelslam.cpp:1321-1395: OctoTree::margi voxel_map.hpp:1196-1305 with plane_update :1118-1146, erase of the
 *                       roots that ceased to exist + clear_slwd :1482-1500) with x_buf AFTER the BA and the factor the BA ran on (its cached
 *                       eig / pcr_adds are read in place, nothing is downloaded), then the slot-ring rotation mp[i] += mgsize
 *                       (voxelslam.cpp:1689-1693).  The caller shifts its own x_buf / pvec_buf / imu_pre_buf (:1695-1712).
 *                       multi_margi hard-codes mgsize 1 (:1360); 1..4 are accepted.
 * The reference's silent early-outs when there are fewer roots than threads (voxel_map.hpp:1597, voxelslam.cpp:1343, 1409) are not
 * reproduced: the work is always done.  One map belongs to one ctx (and its thread). */
typedef struct vxs_map vxs_map;
int vxs_map_create(vxs_ctx* ctx, const vxs_map_params* mp, int win_size, int max_points /* voxel_map.hpp:86, default 100 */, vxs_map** out);
int vxs_map_destroy(vxs_map* m);
int vxs_map_push_scan(vxs_map* m, const double* pv12, int64_t n, const double* poses12, int win_count, vxs_factor* out);
int vxs_map_margi(vxs_map* m, const double* poses12, int win_count, int mgsize, vxs_factor* f);
/* The per-point loop of the EKF update (voxelslam.cpp:876-918; match voxel_map.hpp:1674-1698, OctoTree::match :1335-1392) against the RESIDENT map:
 * root cell through the map's root hash, descent by centre comparison, 3-sigma gates on the plane row plane_update left in the leaf — nothing is
 * exported (vxs_odom_set_planes / vxs_odom_accumulate are the path for a caller that keeps the reference's host octree).  Arguments and outputs as
 * vxs_odom_accumulate; pv12 = NULL uses the ctx's resident scan (vxs_var_init). */
int vxs_map_odom_accumulate(vxs_map* m, const double* pv12, int64_t n, const double* pose12, const double* rot_var9, const double* tsl_var9, double* HTH36, double* HTz6,
                            double* nnt9, int64_t* match_num, int32_t* flags);
/* The whole odometry update, lio_state_estimation (voxelslam.cpp:856-958), in one call: cov_inv = cov^-1 once, then up to 4 EKF iterations,
 * each an association pass (as vxs_map_odom_accumulate, but with the 34 sums reduced in a fixed order, so the result is the same on every run)
 * followed by the 15x15 update on the device: K_1 = (H_T_H + cov_inv)^-1 (LU with partial pivoting), x_curr += solution (tools.hpp:154-173 Exp /
 * Log), the convergence test, rematch_num and the stop rule as written; at the stop cov = (I - G) cov and ok = smallest eigenvalue of that
 * pass's nnt >= 14.  No host round trip between iterations: one read-back and one synchronisation per call.
 *   pv12 = n pointVar records, NULL = the ctx's resident scan (vxs_var_init / vxs_pvec_update), which must have n records.
 *   state24 / cov225 (15x15 row-major) in/out: x_curr before and after; g (state24[21..23]) is not touched.
 *   ok = the reference's return value; iters = iterations executed (2..4); match_num = the last pass's count.
 *   trace12 (may be NULL): per executed iteration match count, |rot_add|, |tra_add|.  flags (may be NULL): the last pass's per-point match flags.
 * n == 0 or an empty map: K_1 = cov, G = 0, iters == 2, ok == 0, state and cov unchanged (as the reference).  A cov (or H_T_H + cov_inv) that
 * meets an exact zero pivot: VXS_ERR_ARG, state24 / cov225 unchanged.  The IMU propagation and the degeneracy counter stay with the caller. */
int vxs_map_lio_update(vxs_map* m, const double* pv12, int64_t n, double* state24, double* cov225, int32_t* ok, int32_t* iters, int64_t* match_num,
                       double* trace12, int32_t* flags);
/* bookkeeping: nodes in the table, points in the point_fix pool, resident scans, ring[win_size] = slot of every logical window position */
int vxs_map_counts(const vxs_map* m, int64_t* n_nodes, int64_t* n_fix_points, int* win_count, int32_t* ring);
/* Every leaf of the map, 32 + 10 * win_size doubles each (for tests and debugging): voxel_center 3 | cube half length | layer | is_plane |
 * isexist | has a slide window | root in the slide map | opt_state | last_num | points in point_fix | pcr_add 10 | pcr_fix 10 | the window
 * clusters pcrs_local[mp[i]], i < win_size.  *n_out = number of leaves (rows are written when cap suffices). */
int vxs_map_read_leaves(vxs_map* m, double* rows, int64_t cap, int64_t* n_out);
/* Plane leaves (is_plane, radius > 0) as plane_update left them, 52 doubles each: plane centre 3 | normal 3 | plane_var 6x6 row-major | radius |
 * N | voxel_center 3 | cube half length | trace(cov_add) | eig_value 3;  ids5 (may be NULL): root x, y, z, layer, octant path. */
int vxs_map_read_planes(vxs_map* m, double* rows52, int64_t* ids5, int64_t cap, int64_t* n_out);

#ifdef __cplusplus
}
#endif
#endif /* VXS_H */
