"""The odometry's iterated EKF update, lio_state_estimation (voxelslam.cpp:856-958), as one device call (vxs_odom_lio_update against the
exported plane table, vxs_map_lio_update against the resident map), against the numpy restatement _ekf_update_numpy that
tests/test_ref_pin.py pins to the reference's own member function, and against the reference's golden vectors.

The host loop (_ekf_update_numpy fed by a path's own odom_accumulate, fp64 atomics) and the device update (fixed-order partial rows) sum the
same contributions in different orders, so state and cov agree to rounding only; every test scene is checked for convergence tests that lie
within 1e-6 relative of their thresholds, so that no branch of either run is decided by that rounding."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import golden_cases as gc
import oracle_api as oa
import scenes
import synth
import voxel_slam_b200 as vx
from parity_checks import compare_leaves, pv_records

HERE = os.path.dirname(os.path.abspath(__file__))
L = 6.0
WN = 4
COV0 = np.diag([1e-4] * 3 + [1e-3] * 3 + [1e-2] * 3 + [1e-6] * 6)
# start errors (rotation, translation sigma, seed) of the EKF scenes: between them they give runs of 3 and 4 iterations on both paths;
# 2 iterations come from feeding a converged result back in
STARTS = [(1e-3, 5e-3, 77), (2e-2, 8e-2, 79), (5e-3, 3e-2, 81)]


def ekf_numpy(accum, pv, st, cov):
    """_ekf_update_numpy (test_ref_pin) with `accum`; also returns the number of passes and the last pass's flags"""
    from test_ref_pin import _ekf_update_numpy
    passes = []

    def acc(p_, x_, rv, tv):
        o = accum(p_, x_, rv, tv)
        passes.append(o)
        return o
    ok, x, c, nm = _ekf_update_numpy(acc, pv, st, cov)
    return dict(ok=ok, state=x, cov=c, n=nm, iters=len(passes), flags=passes[-1]["flags"])


def start_state(truth, rs, ps, seed):
    st = np.zeros(24)
    st[:12] = synth.perturb_pose(truth, seed, rs, ps)
    st[12:15] = (0.3, -0.1, 0.05); st[21:24] = (0, 0, -9.8)
    return st


def relinf(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def margins_ok(trace):
    """no convergence test of the run lies within 1e-6 relative of its threshold (voxelslam.cpp:931)"""
    return bool(np.all(np.abs(trace[:, 1] * 57.3 - 0.01) > 1e-6 * 0.01) and np.all(np.abs(trace[:, 2] * 100 - 0.015) > 1e-6 * 0.015))


# ---------------------------------------------------------------- the two maps, built as test_gpu_odom_edges.py builds them
class TableScene:
    """oa.LocalMap over a 4-scan window; the device holds its planes through vxs_odom_set_planes"""
    path = "table"

    def __init__(self, pts=None, off=None, tr=None):
        self.mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
        if pts is None:
            tr, _ = scenes.poses_true_est(WN, L, 5)
            pts, off = scenes.make_points(WN, 6000, L, 5, tr)
        self.tr = tr
        self.lm = oa.LocalMap(self.mp, pts, off, tr, 1e-4, mgsize=1)
        self.P = self.lm.planes()
        self.truth = tr[WN - 1]

    def oracle(self, pv, pose, rv, tv):
        return self.lm.odom_accumulate(pv, pose, rv, tv, passes=1)

    def scan(self, sigma):
        s = synth.gen_scan(L, WN - 1, 4000, self.truth, seed=0x5EED0000 + 5, sigma=sigma)
        pv = np.zeros((s.shape[0], 12)); pv[:, :3] = s; pv[:, [3, 7, 11]] = 1e-4
        return pv


class ResidentScene:
    """oa.SlidingSim fed scan by scan (cut + recut, margi once the window is full); the device replays it through vx.LocalMap"""
    path = "resident"

    def __init__(self, scans=None):
        self.mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
        self.sim = oa.SlidingSim(self.mp, WN, 1, max_points=100)
        if scans is None:
            scans = []
            for i in range(WN + 4):
                pose = synth.true_pose(L, i)
                est = synth.perturb_pose(pose, 700 + i, 1e-3, 5e-3) if i else pose.copy()
                scans.append((pv_records(synth.gen_scan(L, i, 4000, pose, seed=0x5EED0000 + 61), 500 + i, True), est))
        self.scans = scans
        for pv, est in scans:
            self.sim.add_scan_pv(pv, est)
        self.truth = synth.true_pose(L, WN + 4)

    def oracle(self, pv, pose, rv, tv):
        return self.sim.odom_accumulate(pv, pose, rv, tv)

    def scan(self, sigma):
        return pv_records(synth.gen_scan(L, WN + 4, 4000, self.truth, seed=0x5EED0000 + 62, sigma=sigma), 900, True)


class Device:
    def __init__(self, ctx, sc):
        self.ctx, self.sc = ctx, sc
        if sc.path == "table":
            self.load()
        else:
            self.dm = vx.LocalMap(ctx, sc.mp, WN, max_points=100)
            f = vx.Factor(ctx, WN)
            x = []
            for pv, est in sc.scans:
                x.append(est)
                self.dm.push_scan(pv, np.stack(x), f)
                if len(x) >= WN:
                    self.dm.margi(np.stack(x), f, mgsize=1)
                    x = x[1:]
            f.close()
            compare_leaves(self.dm.leaves(), sc.sim.state(), "lio")

    def load(self):
        if self.sc.path == "table":
            P = self.sc.P
            layer = np.rint(np.log2(self.sc.mp.voxel_size / (2.0 * P["half"]))).astype(np.int32)
            self.ctx.odom_set_planes(self.sc.mp, P["voxel_center"], layer, P["center"], P["normal"], P["plane_var"], P["radius"])

    def accumulate(self, pv, pose, rv, tv):
        if self.sc.path == "table":
            return self.ctx.odom_accumulate(pv, pose, rv, tv)
        return self.dm.odom_accumulate(pv, pose, rv, tv)

    def lio(self, pv, st, cov, n=None, want_flags=True):
        if self.sc.path == "table":
            return self.ctx.odom_lio_update(pv, st, cov, n=n, want_flags=want_flags)
        return self.dm.lio_update(pv, st, cov, n=n, want_flags=want_flags)

    def close(self):
        if self.sc.path == "resident":
            self.dm.close()


def planar_scans(n_scans, n_pts, seed):
    """scans of one plane (z = 0.4, a few mm of noise) seen from slightly different poses: every leaf has the same normal"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_scans):
        pose = np.concatenate([np.eye(3).ravel(), [0.05 * i, -0.03 * i, 0.0]])
        w = np.stack([rng.uniform(-3.5, 3.5, n_pts), rng.uniform(-3.5, 3.5, n_pts), 0.4 + rng.normal(0, 0.003, n_pts)], axis=1)
        out.append((pv_records(w - pose[9:], 40 + i, True), pose))
    return out


# ---------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    yield c
    c.close()


_SCENES = {}


def scene(path):
    if path not in _SCENES:
        _SCENES[path] = TableScene() if path == "table" else ResidentScene()
    return _SCENES[path]


@pytest.fixture(scope="module")
def device(ctx):
    made = {}

    def get(path):
        if path not in made:
            made[path] = Device(ctx, scene(path))
        made[path].load()               # the ctx holds one plane table at a time
        return made[path]
    yield get
    for d in made.values():
        d.close()


PATHS = ("table", "resident")


# ---------------------------------------------------------------- 1. golden vectors
@pytest.mark.gpu
def test_golden_vectors(ctx):
    m = gc.lio_case()
    lm = oa.LocalMap(m["mp"], m["pts"], m["off"], m["tr"], 1e-4, mgsize=1)
    P = lm.planes()
    layer = np.rint(np.log2(m["mp"].voxel_size / (2.0 * P["half"]))).astype(np.int32)
    ctx.odom_set_planes(m["mp"], P["voxel_center"], layer, P["center"], P["normal"], P["plane_var"], P["radius"])
    r = ctx.odom_lio_update(m["pv"], m["state"], m["cov"])
    ge = json.load(open(os.path.join(HERE, "golden", "reference_outputs.json")))["cases"]["lio_state_estimation"]
    s_ref = np.array([float.fromhex(v) for v in ge["state"]])
    c_ref = np.array([float.fromhex(v) for v in ge["cov"]]).reshape(15, 15)
    assert r["ok"] == bool(ge["ok"]) and 500 < r["n"] <= len(m["pv"])
    assert np.max(np.abs(r["state"][:21] - s_ref[:21])) < 1e-11 and relinf(r["cov"], c_ref) < 1e-11
    assert np.array_equal(r["state"][21:], m["state"][21:])                 # g is not touched
    assert np.max(np.abs(s_ref[:12] - m["state"][:12])) > 3e-3


# ---------------------------------------------------------------- 2 + 3. the same update as the host loop, both paths
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_same_update_as_the_host_loop(device, path):
    d = device(path)
    seen = set()
    for sigma in (0.01, 0.12):
        pv = d.sc.scan(sigma)
        runs = []
        for rs, ps, seed in STARTS:
            runs.append(start_state(d.sc.truth, rs, ps, seed))
        for st in runs:
            g = d.lio(pv, st, COV0)
            h = ekf_numpy(d.accumulate, pv, st, COV0)
            assert g["iters"] == h["iters"] and g["n"] == h["n"] and g["ok"] == h["ok"], (sigma, k, g["iters"], h["iters"], g["n"], h["n"])
            assert np.array_equal(g["flags"], h["flags"])
            assert np.max(np.abs(g["state"] - h["state"])) < 1e-12 and relinf(g["cov"], h["cov"]) < 1e-12
            assert margins_ok(g["trace"]), g["trace"]
            assert g["trace"].shape == (g["iters"], 3) and g["trace"][-1, 0] == g["n"]
            assert g["ok"]                                                    # 4. a well-constrained scene passes the eigenvalue check
            if sigma < 0.05:
                assert g["n"] > 3000
            else:
                assert 0.5 * len(pv) < g["n"] < 0.85 * len(pv)               # ~30 % of the noisy scan fails the 3-sigma gates
            seen.add(g["iters"])
            # the converged state fed back in (with the prior's covariance, so that the gates stay as wide): 2 or 3 iterations
            g2 = d.lio(pv, g["state"], COV0)
            h2 = ekf_numpy(d.accumulate, pv, g["state"], COV0)
            assert g2["iters"] == h2["iters"] and g2["n"] == h2["n"] and g2["ok"] == h2["ok"]
            assert np.array_equal(g2["flags"], h2["flags"]) and margins_ok(g2["trace"])
            assert np.max(np.abs(g2["state"] - h2["state"])) < 1e-12 and relinf(g2["cov"], h2["cov"]) < 1e-12
            seen.add(g2["iters"])
    assert seen == {2, 3, 4}, seen


@pytest.mark.gpu
def test_against_the_oracle_accumulation(device):
    d = device("table")
    for sigma in (0.01, 0.12):
        pv = d.sc.scan(sigma)
        for rs, ps, seed in STARTS:
            st = start_state(d.sc.truth, rs, ps, seed)
            g = d.lio(pv, st, COV0)
            o = ekf_numpy(d.sc.oracle, pv, st, COV0)
            assert g["ok"] == o["ok"] and g["n"] == o["n"] and g["iters"] == o["iters"]
            assert np.max(np.abs(g["state"] - o["state"])) < 1e-11 and relinf(g["cov"], o["cov"]) < 1e-11


# ---------------------------------------------------------------- 4. degeneracy
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_one_plane_is_degenerate(ctx, path):
    scans = planar_scans(WN + 2, 3000, 3)
    if path == "table":
        pts = np.concatenate([s[0][:, :3] for s in scans[:WN]])
        off = np.arange(WN + 1) * 3000
        sc = TableScene(pts, off, np.stack([s[1] for s in scans[:WN]]))
    else:
        sc = ResidentScene(scans)
    d = Device(ctx, sc)
    try:
        pv = planar_scans(1, 3000, 99)[0][0]
        st = start_state(np.concatenate([np.eye(3).ravel(), np.zeros(3)]), 1e-3, 5e-3, 5)
        g = d.lio(pv, st, COV0)
        h = ekf_numpy(d.accumulate, pv, st, COV0)
        assert g["n"] > 1000 and g["n"] == h["n"] and g["iters"] == h["iters"]
        assert not g["ok"] and not h["ok"]
        assert np.max(np.abs(g["state"] - h["state"])) < 1e-12 and relinf(g["cov"], h["cov"]) < 1e-12
    finally:
        d.close()


# ---------------------------------------------------------------- 5. no match
def _unchanged(r, st, cov):
    assert r["iters"] == 2 and r["n"] == 0 and not r["ok"]
    assert np.array_equal(r["state"], st) and np.array_equal(r["cov"], cov)
    assert np.array_equal(r["trace"][:, 0], [0, 0]) and np.all(r["trace"][:, 1:] == 0)


@pytest.mark.gpu
def test_no_match(ctx, device):
    rng = np.random.default_rng(8)
    A = rng.standard_normal((15, 15)) * 0.01
    covs = [COV0, A @ A.T + np.eye(15) * 1e-6]
    for path in PATHS:
        d = device(path)
        st = start_state(d.sc.truth, 1e-3, 5e-3, 77)
        far = d.sc.scan(0.01); far[:, :3] += 1000.0                      # every point outside the map
        for cov in covs:
            _unchanged(d.lio(np.zeros((0, 12)), st, cov), st, cov)       # n == 0
            r = d.lio(far, st, cov)
            _unchanged(r, st, cov)
            assert not r["flags"].any()
    m = vx.LocalMap(ctx, vx.MapParams.make(voxel_size=1.0, max_layer=2), WN)       # an empty map
    try:
        pv = scene("table").scan(0.01)
        for cov in covs:
            _unchanged(m.lio_update(pv, st, cov, want_flags=True), st, cov)
    finally:
        m.close()


# ---------------------------------------------------------------- 6. deterministic
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_deterministic(device, path):
    d = device(path)
    pv = d.sc.scan(0.12)
    st = start_state(d.sc.truth, 2e-2, 8e-2, 79)
    a, b = d.lio(pv, st, COV0), d.lio(pv, st, COV0)
    for k in ("state", "cov", "flags", "trace"):
        assert np.array_equal(a[k], b[k]), k
    assert (a["ok"], a["iters"], a["n"]) == (b["ok"], b["iters"], b["n"])


# ---------------------------------------------------------------- 7. the resident hand-over var_init -> lio_update -> pvec_update -> push_scan
@pytest.mark.gpu
def test_resident_scan_through_the_update_into_the_map(ctx):
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    maps = [vx.LocalMap(ctx, mp, WN), vx.LocalMap(ctx, mp, WN)]
    fs = [vx.Factor(ctx, WN), vx.Factor(ctx, WN)]
    ident, zero = np.eye(3), np.zeros(3)
    xs = [[], []]
    iters = []
    try:
        for i in range(WN + 3):
            pose = synth.true_pose(L, i)
            cloud = synth.gen_scan(L, i, 4000, pose, seed=0x5EED0000 + 41, dtype=np.float32)
            st = start_state(pose, 1e-3, 5e-3, 300 + i) if i else start_state(pose, 0, 0, 1)
            pv_host = ctx.var_init(cloud, ident, zero, 0.02, 0.05)
            a = maps[0].lio_update(pv_host, st, COV0)
            upd = ctx.pvec_update(pv_host, a["state"][:12], a["cov"][:3, :3], a["cov"][3:6, 3:6])
            xs[0].append(a["state"][:12])
            maps[0].push_scan(upd["pv"], np.stack(xs[0]), fs[0])
            n = ctx.var_init(cloud, ident, zero, 0.02, 0.05, want_out=False)
            b = maps[1].lio_update(None, st, COV0, n=n)
            ctx.pvec_update(None, b["state"][:12], b["cov"][:3, :3], b["cov"][3:6, 3:6], n=n, want_pv=False, want_pwld=False)
            xs[1].append(b["state"][:12])
            maps[1].push_scan(None, np.stack(xs[1]), fs[1], n=n)
            assert np.array_equal(a["state"], b["state"]) and np.array_equal(a["cov"], b["cov"]) and a["iters"] == b["iters"]
            iters.append(b["iters"])
            for j in range(2):
                if len(xs[j]) >= WN:
                    maps[j].margi(np.stack(xs[j]), fs[j], mgsize=1)
                    xs[j] = xs[j][1:]
        assert max(iters) > 2                                                # the update did work once the map had planes
        la, lb = maps[0].leaves(), maps[1].leaves()
        assert len(la["layer"]) == len(lb["layer"]) > 50
        ka = np.lexsort(np.concatenate([np.round(la["voxel_center"], 9), la["layer"][:, None]], axis=1).T)
        kb = np.lexsort(np.concatenate([np.round(lb["voxel_center"], 9), lb["layer"][:, None]], axis=1).T)
        for k in ("voxel_center", "layer", "is_plane", "pcr_add", "slots"):
            assert np.array_equal(la[k][ka], lb[k][kb]), k
        assert fs[0].counts() == fs[1].counts() and fs[0].counts()[0] > 20
    finally:
        for m in maps: m.close()
        for f in fs: f.close()


# ---------------------------------------------------------------- 8. one call, bounded work
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_launches_per_call(device, path):
    d = device(path)
    pv = d.sc.scan(0.01)
    st = start_state(d.sc.truth, 2e-2, 8e-2, 79)
    d.lio(pv, st, COV0)
    l0 = d.ctx.launches
    r = d.lio(pv, st, COV0)
    assert d.ctx.launches - l0 <= 9 and r["iters"] >= 2


# ---------------------------------------------------------------- 9. errors leave the caller's buffers alone
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_errors(device, path):
    d = device(path)
    pv = d.sc.scan(0.01)
    st0 = start_state(d.sc.truth, 1e-3, 5e-3, 77)
    d.lio(pv, st0, COV0)                                                     # pv is now the resident scan
    sing = COV0.copy(); sing[14, 14] = 0.0
    fn, h = (vx.lib().vxs_odom_lio_update, d.ctx._p) if path == "table" else (vx.lib().vxs_map_lio_update, d.dm._p)
    for n, cov in ((len(pv) + 1, COV0), (len(pv), sing)):
        st, cv = st0.copy(), cov.copy()
        ok, it, m = C.c_int32(7), C.c_int32(7), C.c_int64(7)
        tr = np.full(12, 3.0)
        rc = fn(h, None, C.c_int64(n), vx.api._dp(st), vx.api._dp(cv), C.byref(ok), C.byref(it), C.byref(m), vx.api._dp(tr), None)
        assert rc == -2
        assert np.array_equal(st, st0) and np.array_equal(cv, cov) and (ok.value, it.value, m.value) == (7, 7, 7) and np.all(tr == 3.0)
        with pytest.raises(vx.VxsError) as ei:
            d.lio(None, st0, cov, n=n)
        assert ei.value.code == -2
    assert d.lio(None, st0, COV0, n=len(pv))["iters"] >= 2                  # the resident scan is still there


# ---------------------------------------------------------------- 10. the shim's call, as voxelslam.cpp:1583-1594 writes it (CPU)
SHIM_LIO = r'''
#define VXS_SHIM_WITH_REFERENCE_TYPES
#include "voxel_slam_b200/csrc/shim/voxel_ba_shim.hpp"
void scan(vxs_shim::SurfMap& surf_map, IMUST& extrin_para, IMUST& x_curr, pcl::PointCloud<PointType>& pl_down, double dept_err, double beam_err, int& degrade_cnt, PLV(3)& pwld) {
  vxs_shim::Context& c = vxs_shim::default_context();
  PVecPtr pptr(new PVec);
  vxs_shim::var_init(c, extrin_para, pl_down, pptr, dept_err, beam_err);      // voxelslam.cpp:1584
  if (vxs_shim::lio_state_estimation(surf_map, pptr, x_curr, false))          // :1586, the scan var_init left on the device
  {
    if (degrade_cnt > 0) degrade_cnt--;
  }
  else
    degrade_cnt++;
  bool again = vxs_shim::lio_state_estimation(surf_map, pptr, x_curr);        // uploading pptr
  (void)again;
  pwld.clear();
  vxs_shim::pvec_update(c, pptr, x_curr, pwld);                               // :1594
}
int main() { return 0; }
'''


def _compile(prefix, flags):
    import subprocess
    import tempfile
    root = os.path.dirname(HERE)
    with tempfile.NamedTemporaryFile("w", suffix=".cpp", delete=False) as f:
        f.write(prefix + SHIM_LIO)
    try:
        return subprocess.run(["g++", "-fsyntax-only"] + flags(root) + [f.name], capture_output=True, text=True)
    finally:
        os.unlink(f.name)


def test_shim_lio_state_estimation_type_checks_against_the_stubs():
    r = _compile('#include "tests/shim_stubs/reference_stubs.hpp"\n', lambda root: ["-std=c++14", "-I", root])
    assert r.returncode == 0, r.stderr


def test_shim_lio_state_estimation_compiles_against_the_reference_headers():
    ref = os.environ.get("VXS_REFERENCE_SRC", "/root/reference/VoxelSLAM/src")      # same default as oracle/Makefile
    if not os.path.exists(os.path.join(ref, "voxel_map.hpp")):
        pytest.skip("reference sources (VXS_REFERENCE_SRC) not present")
    r = _compile('#include "voxel_map.hpp"\n', lambda root: ["-std=c++17", "-w", "-I", os.path.join(root, "oracle", "ref_standin"), "-I", ref, "-I", root])
    assert r.returncode == 0, r.stderr[-4000:]
