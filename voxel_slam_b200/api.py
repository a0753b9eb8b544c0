"""ctypes mirror of include/vxs.h (libvxs.so).

Names follow the reference's call surface: ``Factor`` = LidarFactor (voxel_map.hpp:109-290), ``Context.lidar_ba`` =
Lidar_BA_Optimizer::damping_iter (voxel_map.hpp:367), ``Context.li_ba`` = LI_BA_Optimizer(+Gravity)::damping_iter
(voxel_map.hpp:562, 775), ``Context.build_window_factor`` = cut_voxel + recut + tras_opt (voxel_map.hpp:1504, 1148, 1308).
"""
import ctypes as C
import os
import re

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvxs.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "vxs.h")

VXS_OK = 0
VXS_WARN_SINGULAR = 1
VXS_ERR_TOO_FEW_VOXELS = -3


class VxsError(RuntimeError):
    def __init__(self, code, what=""):
        super().__init__(f"libvxs error {code}: {what}")
        self.code = code


class MapParams(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("min_eigen_value", C.c_double), ("plane_thre", C.c_double * 4),
                ("min_point", C.c_double * 4), ("max_layer", C.c_int32), ("reserved", C.c_int32)]

    @staticmethod
    def make(voxel_size=1.0, min_eigen_value=0.0025, plane_thre=(0.25,) * 4, min_point=(5.0,) * 4, max_layer=2):
        p = MapParams()
        p.voxel_size, p.min_eigen_value, p.max_layer = voxel_size, min_eigen_value, max_layer
        for i in range(4):
            p.plane_thre[i] = plane_thre[i]
            p.min_point[i] = min_point[i]
        return p


class LmTrace(C.Structure):
    _fields_ = [("r1", C.c_double), ("r2", C.c_double), ("u", C.c_double), ("v", C.c_double), ("q1", C.c_double),
                ("accepted", C.c_int32), ("hess_built", C.c_int32)]


class VoxelId(C.Structure):
    _fields_ = [("x", C.c_int64), ("y", C.c_int64), ("z", C.c_int64), ("layer", C.c_int32), ("path", C.c_int32)]


VOXEL_ID_DTYPE = np.dtype([("x", "<i8"), ("y", "<i8"), ("z", "<i8"), ("layer", "<i4"), ("path", "<i4")])
LM_TRACE_DTYPE = np.dtype([("r1", "<f8"), ("r2", "<f8"), ("u", "<f8"), ("v", "<f8"), ("q1", "<f8"), ("accepted", "<i4"), ("hess_built", "<i4")])

IMU_EVAL = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_double), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double))
IMU_UPDATE = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_double), C.c_int)
IMU_ROLLBACK = C.CFUNCTYPE(C.c_int, C.c_void_p)


class ImuHooks(C.Structure):
    _fields_ = [("user", C.c_void_p), ("eval", IMU_EVAL), ("update", IMU_UPDATE), ("rollback", IMU_ROLLBACK)]


def declared_symbols(header=HEADER_PATH):
    """Every function name include/vxs.h declares (used by the ABI test)."""
    txt = open(header).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(vxs_[a-z0-9_]+)\s*\(", txt)))


_lib = None


def lib():
    """Load libvxs.so (fails loudly if the CUDA extension has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VxsError(-100, f"{LIB_PATH} is missing — run __graft_entry__.build(); there is no CPU fallback")
        _lib = C.CDLL(LIB_PATH)
        _lib.vxs_ctx_last_error.restype = C.c_char_p
        _lib.vxs_ctx_launch_count.restype = C.c_int64
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


# ---------------------------------------------------------------------------------------------- libvxs
class Context:
    def __init__(self, device=0):
        self._p = C.c_void_p()
        rc = lib().vxs_ctx_create(C.c_int(device), C.byref(self._p))
        if rc != 0:
            raise VxsError(rc, "vxs_ctx_create failed (no CUDA device? libvxs has no CPU fallback)")
        self.device = device

    def close(self):
        if self._p:
            lib().vxs_ctx_destroy(self._p)      # releases the device memory of any factor still alive on this ctx
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise VxsError(rc, (lib().vxs_ctx_last_error(self._p) or b"").decode())
        return rc

    @property
    def launches(self):
        return int(lib().vxs_ctx_launch_count(self._p))

    def timing(self, on=True):
        self._check(lib().vxs_ctx_timing_enable(self._p, C.c_int(int(on))))

    def timing_reset(self):
        self._check(lib().vxs_ctx_timing_reset(self._p))

    def timing_read(self):
        cap = 64
        names = (C.c_char_p * cap)()
        ms = (C.c_double * cap)()
        calls = (C.c_int64 * cap)()
        n = C.c_int(0)
        self._check(lib().vxs_ctx_timing_read(self._p, C.c_int(cap), names, ms, calls, C.byref(n)))
        return {names[i].decode(): (ms[i], calls[i]) for i in range(n.value)}

    def timer_start(self):
        self._check(lib().vxs_ctx_timer_start(self._p))

    def timer_stop(self):
        ms = C.c_double(0)
        self._check(lib().vxs_ctx_timer_stop(self._p, C.byref(ms)))
        return ms.value

    def fp64_tflops(self):
        t = C.c_double(0)
        self._check(lib().vxs_diag_fp64_tflops(self._p, C.byref(t)))
        return t.value

    def dmma_tflops(self):
        t = C.c_double(0)
        self._check(lib().vxs_diag_dmma_tflops(self._p, C.byref(t)))
        return t.value

    DMMA_SHAPES = ("m8n8k4", "m16n8k4", "m16n8k8", "m16n8k16")

    def dmma_shapes_tflops(self):
        """Measured TFLOP/s of each fp64 mma.sync shape, as {shape: rate} in DMMA_SHAPES order."""
        t = (C.c_double * 4)()
        self._check(lib().vxs_diag_dmma_shapes(self._p, t))
        return dict(zip(self.DMMA_SHAPES, list(t)))

    def ldlt_phases(self, n):
        out = (C.c_double * 12)()
        self._check(lib().vxs_diag_ldlt_phases(self._p, int(n), out))
        return list(out)

    # --- multi-GPU
    def solve_damped(self, hess, jact, gauge, u):
        """vxs_diag_solve_damped: the LM drivers' gauge-fixed damped LDL^T solve on a host system (n x n, any layout: symmetric)."""
        H = np.asfortranarray(hess, dtype=np.float64)
        g = _f64(jact)
        n = g.shape[0]
        dx = np.zeros(n)
        sing = C.c_int(0)
        self._check(lib().vxs_diag_solve_damped(self._p, H.ctypes.data_as(C.POINTER(C.c_double)), _dp(g), C.c_int(n), C.c_int(gauge), C.c_double(u), _dp(dx), C.byref(sing)))
        return dx, sing.value

    @staticmethod
    def comm_unique_id():
        buf = (C.c_ubyte * 128)()
        rc = lib().vxs_comm_unique_id(buf)
        if rc != 0:
            raise VxsError(rc, "vxs_comm_unique_id")
        return bytes(buf)

    def comm_init(self, uid, rank, nranks):
        buf = (C.c_ubyte * 128).from_buffer_copy(uid)
        self._check(lib().vxs_ctx_comm_init(self._p, buf, C.c_int(rank), C.c_int(nranks)))

    # --- evaluation
    def evaluate_residual(self, f, poses12):
        p = _f64(poses12)
        r = C.c_double(0)
        self._check(lib().vxs_factor_evaluate_residual(self._p, f._p, _dp(p), C.byref(r)))
        return r.value

    def evaluate_hessian(self, f, poses12):
        p = _f64(poses12)
        n = 6 * f.win_size
        H = np.zeros((n, n), order="F")
        J = np.zeros(n)
        r = C.c_double(0)
        self._check(lib().vxs_factor_evaluate_hessian(self._p, f._p, _dp(p), _dp(H), _dp(J), C.byref(r)))
        return H, J, r.value

    # --- solvers
    def lidar_ba(self, f, poses12, max_iter=3, thd_num=2, want_hess=True, trace_cap=64):
        p = _f64(poses12).copy()
        n = 6 * f.win_size
        H = np.zeros((n, n), order="F") if want_hess else None
        resis = np.zeros(2)
        conv = C.c_int(0)
        tr = np.zeros(trace_cap, dtype=LM_TRACE_DTYPE)
        tl = C.c_int(0)
        rc = self._check(lib().vxs_lidar_ba(self._p, f._p, _dp(p), C.c_int(max_iter), C.c_int(thd_num), _dp(H), _dp(resis), C.byref(conv),
                                            tr.ctypes.data_as(C.POINTER(LmTrace)), C.c_int(trace_cap), C.byref(tl)))
        return dict(poses=p, hess=H, resis=resis, is_converge=bool(conv.value), trace=tr[: tl.value], status=rc)

    def li_ba(self, f, states24, imu, with_gravity=False, max_iter=3, imu_coef=1e-4, want_hess=True, trace_cap=64):
        s = _f64(states24).copy()
        n = 15 * f.win_size + (3 if with_gravity else 0)
        H = np.zeros((n, n), order="F") if want_hess else None
        resis = np.zeros(2)
        tr = np.zeros(trace_cap, dtype=LM_TRACE_DTYPE)
        tl = C.c_int(0)
        rc = self._check(lib().vxs_li_ba(self._p, f._p, _dp(s), C.c_int(int(with_gravity)), C.c_int(max_iter), C.c_double(imu_coef), C.byref(imu.hooks), _dp(H), _dp(resis),
                                         tr.ctypes.data_as(C.POINTER(LmTrace)), C.c_int(trace_cap), C.byref(tl)))
        return dict(states=s, hess=H, resis=resis, trace=tr[: tl.value], status=rc)

    # --- voxel map
    def voxel_keys(self, pw, voxel_size):
        p = _f64(pw).reshape(-1, 3)
        n = p.shape[0]
        xyz = np.zeros((n, 3), dtype=np.int64)
        h = np.zeros(n, dtype=np.uint64)
        self._check(lib().vxs_voxel_keys(self._p, _dp(p), C.c_int64(n), C.c_double(voxel_size), xyz.ctypes.data_as(C.POINTER(C.c_int64)), h.ctypes.data_as(C.POINTER(C.c_uint64))))
        return xyz, h

    def build_window_factor(self, mp, pts_body, scan_offsets, poses12, out, fix_pts=None, want_ids=False, ids_cap=0):
        pts = _f64(pts_body).reshape(-1, 3)
        off = np.ascontiguousarray(scan_offsets, dtype=np.int64)
        W = off.shape[0] - 1
        p = _f64(poses12)
        fx = _f64(fix_pts).reshape(-1, 3) if fix_pts is not None else None
        ids = np.zeros(ids_cap, dtype=VOXEL_ID_DTYPE) if want_ids else None
        n_out = C.c_int64(0)
        self._check(lib().vxs_build_window_factor(self._p, C.byref(mp), _dp(pts), off.ctypes.data_as(C.POINTER(C.c_int64)), _dp(p), C.c_int(W), _dp(fx),
                                                  C.c_int64(0 if fx is None else fx.shape[0]), out._p,
                                                  ids.ctypes.data_as(C.POINTER(VoxelId)) if want_ids else None, C.c_int64(ids_cap), C.byref(n_out)))
        return (n_out.value, ids[: n_out.value]) if want_ids else n_out.value

    def build_gba_factor(self, mp, xyz_f32, kf_offsets, poses12, out, stride_floats=3, want_ids=False, ids_cap=0):
        x = np.ascontiguousarray(xyz_f32, dtype=np.float32)
        off = np.ascontiguousarray(kf_offsets, dtype=np.int64)
        W = off.shape[0] - 1
        p = _f64(poses12)
        ids = np.zeros(ids_cap, dtype=VOXEL_ID_DTYPE) if want_ids else None
        n_out = C.c_int64(0)
        self._check(lib().vxs_build_gba_factor(self._p, C.byref(mp), x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride_floats), off.ctypes.data_as(C.POINTER(C.c_int64)),
                                               _dp(p), C.c_int(W), out._p, ids.ctypes.data_as(C.POINTER(VoxelId)) if want_ids else None, C.c_int64(ids_cap), C.byref(n_out)))
        return (n_out.value, ids[: n_out.value]) if want_ids else n_out.value

    def hba_window(self, coarse, fine, xyz_f32, kf_offsets, poses12, max_iter, thread_num=2, stride_floats=3):
        x = np.ascontiguousarray(xyz_f32, dtype=np.float32)
        off = np.ascontiguousarray(kf_offsets, dtype=np.int64)
        W = off.shape[0] - 1
        p = _f64(poses12).copy()
        H = np.zeros((6 * W, 6 * W), order="F")
        log = np.zeros(2 * max(max_iter, 1))
        it = C.c_int(0)
        self._check(lib().vxs_hba_window(self._p, C.byref(coarse), C.byref(fine), x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride_floats),
                                         off.ctypes.data_as(C.POINTER(C.c_int64)), _dp(p), C.c_int(W), C.c_int(max_iter), C.c_int(thread_num), _dp(H), _dp(log), C.byref(it)))
        return dict(poses=p, hess=H, resis_log=log[: 2 * it.value], outer_iters=it.value)


def _hba_edges(self, W, poses12, cap=None):
    cap = cap if cap is not None else W * (W - 1) // 2
    p = _f64(poses12)
    eij = np.zeros((max(cap, 1), 2), dtype=np.int32); v6 = np.zeros((max(cap, 1), 6)); rot = np.zeros((max(cap, 1), 9)); tra = np.zeros((max(cap, 1), 3))
    n = C.c_int64(0)
    self._check(lib().vxs_hba_edges(self._p, C.c_int(W), _dp(p), C.c_int64(cap), eij.ctypes.data_as(C.POINTER(C.c_int32)), _dp(v6), _dp(rot), _dp(tra), C.byref(n)))
    m = min(n.value, cap)      # the library returns the edges in the reference's lexicographic (i, j) order
    return dict(n=n.value, ij=eij[:m], v6=v6[:m], rot=rot[:m], tra=tra[:m])


Context.hba_edges = _hba_edges


def _down_sampling(self, pts_f32, voxel_size, close=False, stride_floats=None):
    """down_sampling_voxel / down_sampling_close (tools.hpp:201-302) on the device.  Returns None when the reference would leave the
    cloud untouched, else dict(xyz, count, index) in ascending cell order."""
    x = np.ascontiguousarray(pts_f32, dtype=np.float32)
    stride = int(stride_floats) if stride_floats else (x.shape[1] if x.ndim == 2 else 3)
    n = x.size // stride
    xyz = np.zeros((max(n, 1), 3), dtype=np.float32); cnt = np.zeros(max(n, 1), dtype=np.float32); idx = np.zeros(max(n, 1), dtype=np.int64)
    m = C.c_int64(0)
    fn = lib().vxs_down_sampling_close if close else lib().vxs_down_sampling_voxel
    self._check(fn(self._p, x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride), C.c_int64(n), C.c_double(voxel_size), xyz.ctypes.data_as(C.POINTER(C.c_float)),
                   cnt.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(n), C.byref(m)))
    if m.value < 0:
        return None
    return dict(xyz=xyz[: m.value], count=cnt[: m.value], index=idx[: m.value])


Context.down_sampling = _down_sampling


def _down_sampling_pvec(self, pv_f64, voxel_size):
    """down_sampling_pvec (voxel_map.hpp:23-64): pv rows = pnt(3) | var(9)."""
    x = np.ascontiguousarray(pv_f64, dtype=np.float64)
    stride = x.shape[1]
    n = x.shape[0]
    xyz = np.zeros((max(n, 1), 3), dtype=np.float32); nrm = np.zeros((max(n, 1), 3), dtype=np.float32); cnt = np.zeros(max(n, 1), dtype=np.float32)
    idx = np.zeros(max(n, 1), dtype=np.int64)
    m = C.c_int64(0)
    self._check(lib().vxs_down_sampling_pvec(self._p, _dp(x), C.c_int(stride), C.c_int64(n), C.c_double(voxel_size), xyz.ctypes.data_as(C.POINTER(C.c_float)),
                                             nrm.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int64)),
                                             C.c_int64(n), C.byref(m)))
    return dict(xyz=xyz[: m.value], var_diag=nrm[: m.value], count=cnt[: m.value], index=idx[: m.value])


Context.down_sampling_pvec = _down_sampling_pvec


def _odom_set_planes(self, mp, voxel_center, layer, center, normal, plane_var, radius):
    vc, c, nr, pv = _f64(voxel_center).reshape(-1, 3), _f64(center).reshape(-1, 3), _f64(normal).reshape(-1, 3), _f64(plane_var).reshape(-1, 36)
    ly = np.ascontiguousarray(layer, dtype=np.int32)
    rd = np.ascontiguousarray(radius, dtype=np.float32)
    self._check(lib().vxs_odom_set_planes(self._p, C.byref(mp), C.c_int64(vc.shape[0]), _dp(vc), ly.ctypes.data_as(C.POINTER(C.c_int32)), _dp(c), _dp(nr), _dp(pv),
                                          rd.ctypes.data_as(C.POINTER(C.c_float))))


def _odom_accumulate(self, pv12, pose12, rot_var, tsl_var, n=None, want_flags=True):
    """One accumulation pass of the odometry EKF (voxelslam.cpp:876-918).  pv12=None re-uses the resident scan (pass n)."""
    pv = _f64(pv12).reshape(-1, 12) if pv12 is not None else None
    n = pv.shape[0] if pv is not None else int(n)
    HTH, HTz, nnt = np.zeros((6, 6)), np.zeros(6), np.zeros((3, 3))
    flags = np.zeros(max(n, 1), dtype=np.int32) if want_flags else None
    m = C.c_int64(0)
    self._check(lib().vxs_odom_accumulate(self._p, _dp(pv), C.c_int64(n), _dp(_f64(pose12)), _dp(_f64(rot_var)), _dp(_f64(tsl_var)), _dp(HTH), _dp(HTz), _dp(nnt), C.byref(m),
                                          flags.ctypes.data_as(C.POINTER(C.c_int32)) if want_flags else None))
    return dict(n=m.value, HTH=HTH, HTz=HTz, nnt=nnt, flags=flags[:n] if want_flags else None)


def _var_init(self, pts_f32, ext_R, ext_p, dept_err, beam_err, want_out=True, stride_floats=None):
    """var_init (voxelslam.hpp:187-203): pointVar records of a scan; they also stay on the device as the ctx's resident scan."""
    x = np.ascontiguousarray(pts_f32, dtype=np.float32)
    stride = int(stride_floats) if stride_floats else (x.shape[1] if x.ndim == 2 else 3)
    n = x.size // stride
    out = np.zeros((max(n, 1), 12)) if want_out else None
    self._check(lib().vxs_var_init(self._p, x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride), C.c_int64(n), _dp(_f64(ext_R)), _dp(_f64(ext_p)), C.c_double(dept_err), C.c_double(beam_err),
                                   _dp(out)))
    return out[:n] if want_out else n


def _pvec_update(self, pv12, pose12, rot_var, tsl_var, n=None, want_pv=True, want_pwld=True):
    """pvec_update (voxelslam.hpp:205-214); pv12=None works on the resident scan (pass n)."""
    pv = _f64(pv12).reshape(-1, 12) if pv12 is not None else None
    n = pv.shape[0] if pv is not None else int(n)
    out = np.zeros((max(n, 1), 12)) if want_pv else None
    pw = np.zeros((max(n, 1), 3)) if want_pwld else None
    self._check(lib().vxs_pvec_update(self._p, _dp(pv), C.c_int64(n), _dp(_f64(pose12)), _dp(_f64(rot_var)), _dp(_f64(tsl_var)), _dp(out), _dp(pw)))
    return dict(pv=out[:n] if want_pv else None, pwld=pw[:n] if want_pwld else None)


def _lio_update(ctx, fn, handle, pv12, state24, cov, n, want_flags):
    pv = _f64(pv12).reshape(-1, 12) if pv12 is not None else None
    n = pv.shape[0] if pv is not None else int(n)
    st, cv = _f64(state24).reshape(24).copy(), _f64(cov).reshape(15, 15).copy()
    ok, iters, m = C.c_int32(0), C.c_int32(0), C.c_int64(0)
    trace = np.zeros((4, 3))
    flags = np.zeros(max(n, 1), dtype=np.int32) if want_flags else None
    ctx._check(fn(handle, _dp(pv), C.c_int64(n), _dp(st), _dp(cv), C.byref(ok), C.byref(iters), C.byref(m), _dp(trace),
                  flags.ctypes.data_as(C.POINTER(C.c_int32)) if want_flags else None))
    return dict(ok=bool(ok.value), state=st, cov=cv, iters=iters.value, n=m.value, trace=trace[: iters.value], flags=flags[:n] if want_flags else None)


def _odom_lio_update(self, pv12, state24, cov, n=None, want_flags=False):
    """lio_state_estimation (voxelslam.cpp:856-958) in one call against the plane table of odom_set_planes: up to 4 EKF iterations on the device.
    pv12=None = the resident scan (pass n).  Returns ok, state (24), cov (15x15), iters, n (last pass's match count), trace (iters x [match count,
    |rot_add|, |tra_add|]) and flags (last pass, want_flags)."""
    return _lio_update(self, lib().vxs_odom_lio_update, self._p, pv12, state24, cov, n, want_flags)


Context.var_init = _var_init
Context.pvec_update = _pvec_update
Context.odom_set_planes = _odom_set_planes
Context.odom_lio_update = _odom_lio_update
Context.odom_accumulate = _odom_accumulate


def _hba_bottom_batch(self, fine, xyz_f32, kf_offsets, poses12, win_first, win_size=10, thread_num=2, stride_floats=None, max_points_per_chunk=0, want_hess=False):
    """vxs_hba_bottom_batch: the bottom level of the hierarchical global BA (one HBA_add_edge(max_iter=1) per window) for all windows at once."""
    x = np.ascontiguousarray(xyz_f32, dtype=np.float32)
    stride = int(stride_floats) if stride_floats else (x.shape[1] if x.ndim == 2 else 3)
    off = np.ascontiguousarray(kf_offsets, dtype=np.int64)
    p = _f64(poses12).reshape(-1, 12)
    K = p.shape[0]
    wf = np.ascontiguousarray(win_first, dtype=np.int32)
    nw, P, n = wf.shape[0], win_size * (win_size - 1) // 2, 6 * win_size
    out = dict(poses=np.zeros((nw, win_size, 12)), resis=np.zeros((nw, 2)), status=np.zeros(nw, dtype=np.int32), is_converge=np.zeros(nw, dtype=np.int32),
               lm_iters=np.zeros(nw, dtype=np.int32), edge_valid=np.zeros((nw, P), dtype=np.int32), edge_v6=np.zeros((nw, P, 6)), edge_rot=np.zeros((nw, P, 9)),
               edge_tra=np.zeros((nw, P, 3)), hess=np.zeros((nw, n * n)) if want_hess else None)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
    rc = self._check(lib().vxs_hba_bottom_batch(self._p, C.byref(fine), x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride), off.ctypes.data_as(C.POINTER(C.c_int64)), _dp(p), C.c_int(K),
                                                ip(wf), C.c_int(nw), C.c_int(win_size), C.c_int(thread_num), C.c_int64(max_points_per_chunk), _dp(out["poses"]), _dp(out["resis"]),
                                                ip(out["status"]), ip(out["is_converge"]), ip(out["lm_iters"]), ip(out["edge_valid"]), _dp(out["edge_v6"]), _dp(out["edge_rot"]),
                                                _dp(out["edge_tra"]), _dp(out["hess"])))
    out["rc"] = rc
    if want_hess:
        out["hess"] = out["hess"].reshape(nw, n, n).transpose(0, 2, 1)      # column-major -> [w][row][col]
    return out


def _submap_merge_batch(self, xyz_f32, kf_offsets, poses_win, win_first, voxel_size, stride_floats=None, max_points_per_chunk=0, cap=None):
    """vxs_submap_merge_batch: the submap merge + down-sampling of every window (voxelslam.cpp:2428-2447) in one pass."""
    x = np.ascontiguousarray(xyz_f32, dtype=np.float32)
    stride = int(stride_floats) if stride_floats else (x.shape[1] if x.ndim == 2 else 3)
    off = np.ascontiguousarray(kf_offsets, dtype=np.int64)
    pw = _f64(poses_win)
    wf = np.ascontiguousarray(win_first, dtype=np.int32)
    nw, ws = pw.shape[0], pw.shape[1]
    if cap is None:
        cap = int(sum(off[k + ws] - off[k] for k in wf))
    xyz = np.zeros((max(cap, 1), 3), dtype=np.float32); cnt = np.zeros(max(cap, 1), dtype=np.float32); idx = np.zeros(max(cap, 1), dtype=np.int64)
    woff = np.zeros(nw + 1, dtype=np.int64)
    n = C.c_int64(0)
    self._check(lib().vxs_submap_merge_batch(self._p, x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride), off.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int(off.shape[0] - 1), _dp(pw),
                                             wf.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int(nw), C.c_int(ws), C.c_double(voxel_size), C.c_int64(max_points_per_chunk),
                                             xyz.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(cap),
                                             woff.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(n)))
    m = min(n.value, cap)
    return dict(xyz=xyz[:m], count=cnt[:m], index=idx[:m], win_offsets=woff, n=n.value)


def _hba_pass(self, coarse, fine, xyz_f32, kf_offsets, poses12, win_size=10, win_stride=5, top_max_iter=1, stride_floats=None, max_points_per_chunk=0, nranks=1, rank=0):
    """vxs_hba_pass: bottom windows (this rank's share) + submap merge + exchange + top level, clouds and submaps device-resident."""
    x = xyz_f32 if (isinstance(xyz_f32, np.ndarray) and xyz_f32.dtype == np.float32 and xyz_f32.flags["C_CONTIGUOUS"]) else np.ascontiguousarray(xyz_f32, dtype=np.float32)
    stride = int(stride_floats) if stride_floats else (x.shape[1] if x.ndim == 2 else 3)
    off = np.ascontiguousarray(kf_offsets, dtype=np.int64)
    p = _f64(poses12).reshape(-1, 12)
    K = p.shape[0]
    nwin = (K - win_size) // win_stride + 1
    lo, hi = nwin * rank // nranks, nwin * (rank + 1) // nranks
    nm, P = max(hi - lo, 1), win_size * (win_size - 1) // 2
    out = dict(bottom_poses=np.zeros((nm, win_size, 12)), bottom_resis=np.zeros((nm, 2)), bottom_status=np.zeros(nm, dtype=np.int32), edge_valid=np.zeros((nm, P), dtype=np.int32),
               edge_v6=np.zeros((nm, P, 6)), edge_rot=np.zeros((nm, P, 9)), edge_tra=np.zeros((nm, P, 3)), top_poses=np.zeros((nwin, 12)), top_resis=np.zeros(2 * max(top_max_iter, 1)),
               submap_sizes=np.zeros(nwin, dtype=np.int64), phase_ms=np.zeros(6))
    first, cnt, outer = C.c_int32(0), C.c_int32(0), C.c_int(0)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
    self._check(lib().vxs_hba_pass(self._p, C.byref(coarse), C.byref(fine), x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride), off.ctypes.data_as(C.POINTER(C.c_int64)), _dp(p), C.c_int(K),
                                   C.c_int(win_size), C.c_int(win_stride), C.c_int(2), C.c_int(5), C.c_int(top_max_iter), C.c_int64(max_points_per_chunk), _dp(out["bottom_poses"]),
                                   _dp(out["bottom_resis"]), ip(out["bottom_status"]), ip(out["edge_valid"]), _dp(out["edge_v6"]), _dp(out["edge_rot"]), _dp(out["edge_tra"]), C.byref(first),
                                   C.byref(cnt), _dp(out["top_poses"]), _dp(out["top_resis"]), C.byref(outer), out["submap_sizes"].ctypes.data_as(C.POINTER(C.c_int64)), _dp(out["phase_ms"])))
    assert first.value == lo and cnt.value == hi - lo, (first.value, cnt.value, lo, hi)
    out.update(first_window=lo, window_count=hi - lo, top_outer_iters=outer.value, nwin=nwin)
    return out


Context.hba_pass = _hba_pass
Context.hba_bottom_batch = _hba_bottom_batch
Context.submap_merge_batch = _submap_merge_batch


def _submap_merge(self, xyz_f32, kf_offsets, poses12, voxel_size, stride_floats=None):
    """Submap merge of HBA_add_edge (voxelslam.cpp:2428-2447): clouds into the frame of keyframe 0 + down_sampling_voxel."""
    x = np.ascontiguousarray(xyz_f32, dtype=np.float32)
    stride = int(stride_floats) if stride_floats else (x.shape[1] if x.ndim == 2 else 3)
    off = np.ascontiguousarray(kf_offsets, dtype=np.int64)
    W = off.shape[0] - 1
    n = int(off[-1])
    p = _f64(poses12)
    xyz = np.zeros((max(n, 1), 3), dtype=np.float32); cnt = np.zeros(max(n, 1), dtype=np.float32); idx = np.zeros(max(n, 1), dtype=np.int64)
    m = C.c_int64(0)
    self._check(lib().vxs_submap_merge(self._p, x.ctypes.data_as(C.POINTER(C.c_float)), C.c_int(stride), off.ctypes.data_as(C.POINTER(C.c_int64)), _dp(p), C.c_int(W),
                                       C.c_double(voxel_size), xyz.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_float)),
                                       idx.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(n), C.byref(m)))
    return dict(xyz=xyz[: m.value], count=cnt[: m.value], index=idx[: m.value])


Context.submap_merge = _submap_merge


class Factor:
    """Device-resident LidarFactor."""

    def __init__(self, ctx, win_size):
        self.ctx = ctx
        self._p = C.c_void_p()
        ctx._check(lib().vxs_factor_create(ctx._p, C.c_int(win_size), C.byref(self._p)))

    def close(self):
        if self._p:
            lib().vxs_factor_destroy(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def clear(self):
        self.ctx._check(lib().vxs_factor_clear(self._p))

    def counts(self):
        v, e, w = C.c_int64(0), C.c_int64(0), C.c_int(0)
        self.ctx._check(lib().vxs_factor_counts(self._p, C.byref(v), C.byref(e), C.byref(w)))
        return v.value, e.value, w.value

    @property
    def win_size(self):
        return self.counts()[2]

    def push_voxels(self, entry_ptr, entry_frame, entry_cluster10, eig12, sum10, fix10=None, coe=None):
        ptr = np.ascontiguousarray(entry_ptr, dtype=np.int64)
        fr = np.ascontiguousarray(entry_frame, dtype=np.int32)
        cl, e, s = _f64(entry_cluster10), _f64(eig12), _f64(sum10)
        fx = _f64(fix10) if fix10 is not None else None
        co = _f64(coe) if coe is not None else None
        self.ctx._check(lib().vxs_factor_push_voxels(self._p, C.c_int64(ptr.shape[0] - 1), ptr.ctypes.data_as(C.POINTER(C.c_int64)), fr.ctypes.data_as(C.POINTER(C.c_int32)),
                                                     _dp(cl), _dp(fx), _dp(co), _dp(e), _dp(s)))

    def push_voxels_async(self, entry_ptr, entry_frame, entry_cluster10, eig12, sum10, fix10=None, coe=None):
        """vxs_factor_push_voxels_async: returns with the copies queued; the arrays are kept alive on this object until the next push /
        sync (pass pinned arrays from api.pinned_array for a real overlap)."""
        ptr = np.ascontiguousarray(entry_ptr, dtype=np.int64)
        fr = np.ascontiguousarray(entry_frame, dtype=np.int32)
        cl, e, s = _f64(entry_cluster10), _f64(eig12), _f64(sum10)
        fx = _f64(fix10) if fix10 is not None else None
        co = _f64(coe) if coe is not None else None
        self._async_keep = (ptr, fr, cl, e, s, fx, co)
        self.ctx._check(lib().vxs_factor_push_voxels_async(self._p, C.c_int64(ptr.shape[0] - 1), ptr.ctypes.data_as(C.POINTER(C.c_int64)),
                                                           fr.ctypes.data_as(C.POINTER(C.c_int32)), _dp(cl), _dp(fx), _dp(co), _dp(e), _dp(s)))

    def sync_uploads(self):
        self.ctx._check(lib().vxs_factor_sync_uploads(self._p))
        self._async_keep = None

    def push_voxels_raw(self, n_vox, ptr_p, frame_p, cl_p, fix_p, coe_p, eig_p, sum_p):
        """Raw-pointer variant (pinned buffers from vxs_host_alloc) used by bench.py's end-to-end leg."""
        self.ctx._check(lib().vxs_factor_push_voxels(self._p, C.c_int64(n_vox), ptr_p, frame_p, cl_p, fix_p, coe_p, eig_p, sum_p))

    def push_voxels_dense(self, clusters10, eig12, sum10, fix10=None, coe=None):
        cl, e, s = _f64(clusters10), _f64(eig12), _f64(sum10)
        n = e.reshape(-1, 12).shape[0]
        fx = _f64(fix10) if fix10 is not None else None
        co = _f64(coe) if coe is not None else None
        self.ctx._check(lib().vxs_factor_push_voxels_dense(self._p, C.c_int64(n), _dp(cl), _dp(fx), _dp(co), _dp(e), _dp(s)))

    def cache_save(self):
        self.ctx._check(lib().vxs_factor_cache_save(self._p))

    def cache_restore(self):
        self.ctx._check(lib().vxs_factor_cache_restore(self._p))

    def read_back(self):
        v = self.counts()[0]
        eig, s = np.zeros((v, 12)), np.zeros((v, 10))
        self.ctx._check(lib().vxs_factor_read_back(self._p, _dp(eig), _dp(s)))
        return eig, s

    def read_structure(self):
        v, e, _ = self.counts()
        ptr = np.zeros(v + 1, dtype=np.int64)
        fr = np.zeros(e, dtype=np.int32)
        cl, fx, co = np.zeros((e, 10)), np.zeros((v, 10)), np.zeros(v)
        self.ctx._check(lib().vxs_factor_read_structure(self._p, ptr.ctypes.data_as(C.POINTER(C.c_int64)), fr.ctypes.data_as(C.POINTER(C.c_int32)), _dp(cl), _dp(fx), _dp(co)))
        return ptr, fr, cl, fx, co


class LocalMap:
    """vxs_map: the device-resident `surf_map` / `surf_map_slide` of the sliding-window loop (voxelslam.cpp:1599-1712)."""

    def __init__(self, ctx, mp, win_size, max_points=100):
        self.ctx, self.W = ctx, win_size
        self._p = C.c_void_p()
        ctx._check(lib().vxs_map_create(ctx._p, C.byref(mp), C.c_int(win_size), C.c_int(max_points), C.byref(self._p)))

    def close(self):
        if self._p:
            lib().vxs_map_destroy(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push_scan(self, pv12, poses12, factor=None, n=None):
        """cut_voxel_multi + multi_recut + tras_opt of one new scan; pv12 rows = body pnt (3) | var (9); poses12 = x_buf incl. the new scan."""
        pv = _f64(pv12).reshape(-1, 12) if pv12 is not None else None      # None: the ctx's resident scan (var_init / pvec_update), pass n
        p = _f64(poses12).reshape(-1, 12)
        nn = pv.shape[0] if pv is not None else int(n)
        self.ctx._check(lib().vxs_map_push_scan(self._p, _dp(pv), C.c_int64(nn), _dp(p), C.c_int(p.shape[0]), factor._p if factor is not None else None))

    def odom_accumulate(self, pv12, pose12, rot_var, tsl_var, n=None, want_flags=True):
        """vxs_map_odom_accumulate: the EKF accumulation pass (voxelslam.cpp:876-918) against the resident map; pv12=None = resident scan (pass n)."""
        pv = _f64(pv12).reshape(-1, 12) if pv12 is not None else None
        n = pv.shape[0] if pv is not None else int(n)
        HTH, HTz, nnt = np.zeros((6, 6)), np.zeros(6), np.zeros((3, 3))
        flags = np.zeros(max(n, 1), dtype=np.int32) if want_flags else None
        m = C.c_int64(0)
        self.ctx._check(lib().vxs_map_odom_accumulate(self._p, _dp(pv), C.c_int64(n), _dp(_f64(pose12)), _dp(_f64(rot_var)), _dp(_f64(tsl_var)), _dp(HTH), _dp(HTz), _dp(nnt), C.byref(m),
                                                      flags.ctypes.data_as(C.POINTER(C.c_int32)) if want_flags else None))
        return dict(n=m.value, HTH=HTH, HTz=HTz, nnt=nnt, flags=flags[:n] if want_flags else None)

    def lio_update(self, pv12, state24, cov, n=None, want_flags=False):
        """vxs_map_lio_update: lio_state_estimation (voxelslam.cpp:856-958) against the resident map in one call; outputs as Context.odom_lio_update."""
        return _lio_update(self.ctx, lib().vxs_map_lio_update, self._p, pv12, state24, cov, n, want_flags)

    def margi(self, poses12, factor, mgsize=1):
        p = _f64(poses12).reshape(-1, 12)
        self.ctx._check(lib().vxs_map_margi(self._p, _dp(p), C.c_int(p.shape[0]), C.c_int(mgsize), factor._p))

    def counts(self):
        nn, nf, wc = C.c_int64(0), C.c_int64(0), C.c_int(0)
        ring = np.zeros(self.W, dtype=np.int32)
        self.ctx._check(lib().vxs_map_counts(self._p, C.byref(nn), C.byref(nf), C.byref(wc), ring.ctypes.data_as(C.POINTER(C.c_int32))))
        return dict(nodes=nn.value, fix_points=nf.value, win_count=wc.value, ring=ring)

    def leaves(self):
        """every leaf, same fields as the oracle's SlidingSim.state()"""
        W = self.W
        n = C.c_int64(0)
        self.ctx._check(lib().vxs_map_read_leaves(self._p, None, C.c_int64(0), C.byref(n)))
        rows = np.zeros((max(n.value, 1), 32 + 10 * W))
        self.ctx._check(lib().vxs_map_read_leaves(self._p, _dp(rows), C.c_int64(n.value), C.byref(n)))
        r = rows[: n.value]
        c = self.counts()
        return dict(win_count=c["win_count"], ring=c["ring"], voxel_center=r[:, 0:3], half=r[:, 3], layer=r[:, 4].astype(int), is_plane=r[:, 5] > 0, isexist=r[:, 6] > 0,
                    has_sw=r[:, 7] > 0, in_slide=r[:, 8] > 0, opt_state=r[:, 9].astype(int), last_num=r[:, 10].astype(int), n_point_fix=r[:, 11].astype(int),
                    pcr_add=r[:, 12:22], pcr_fix=r[:, 22:32], slots=r[:, 32:].reshape(n.value, W, 10))

    def planes(self):
        n = C.c_int64(0)
        self.ctx._check(lib().vxs_map_read_planes(self._p, None, None, C.c_int64(0), C.byref(n)))
        rows = np.zeros((max(n.value, 1), 52)); ids = np.zeros((max(n.value, 1), 5), dtype=np.int64)
        self.ctx._check(lib().vxs_map_read_planes(self._p, _dp(rows), ids.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(n.value), C.byref(n)))
        r = rows[: n.value]
        return dict(center=r[:, 0:3], normal=r[:, 3:6], plane_var=r[:, 6:42].reshape(-1, 6, 6), radius=r[:, 42], N=r[:, 43], voxel_center=r[:, 44:47], half=r[:, 47],
                    cov_trace=r[:, 48], eig=r[:, 49:52], ids=ids[: n.value])


def host_alloc(nbytes):
    p = C.c_void_p()
    rc = lib().vxs_host_alloc(C.byref(p), C.c_uint64(nbytes))
    if rc != 0:
        raise VxsError(rc, "vxs_host_alloc")
    return p


def host_free(p):
    lib().vxs_host_free(p)


_PINNED = []


def pinned_array(shape, dtype):
    """numpy view over pinned (page-locked) host memory."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape))
    p = host_alloc(max(n * dtype.itemsize, 16))
    buf = (C.c_char * (n * dtype.itemsize)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)
    _PINNED.append(p)  # freed at interpreter exit
    return arr
