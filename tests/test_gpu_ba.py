"""GPU parity tests (run on an H100): CUDA path through the C-ABI vs the CPU oracle on the same seeded inputs.
Tolerances: BASELINE.json asks for 1e-5 relative on residuals / H / g / pose increments; the kernels are fp64 and are held
to far tighter bounds here (stated per assert)."""
import threading

import numpy as np
import pytest

import oracle_api as oa
import scenes
import synth
import voxel_slam_b200 as vx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    yield c
    c.close()


def relinf(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def gpu_factor(ctx, sc, W=None):
    f = vx.Factor(ctx, W or sc["W"])
    f.push_voxels_dense(sc["clusters10"], sc["eig12"], sc["sum10"], fix10=sc["fix10"])
    return f


def check_eig(e_gpu, e_ref, tol):
    assert relinf(e_gpu[:, :3], e_ref[:, :3]) < tol
    Ug, Ur = e_gpu[:, 3:].reshape(-1, 3, 3), e_ref[:, 3:].reshape(-1, 3, 3)
    # eigenvectors compared up to sign, only where the eigenvalue gap makes them well defined
    lam = e_ref[:, :3]
    for k in range(3):
        gap = np.min(np.abs(lam - lam[:, [k]]) + np.eye(3)[k] * 1e300, axis=1) / np.max(np.abs(lam), axis=1)
        ok = gap > 1e-3
        d = np.abs(np.abs(np.sum(Ug[ok, :, k] * Ur[ok, :, k], axis=1)) - 1.0)
        assert d.size == 0 or d.max() < 1e-8


@pytest.mark.parametrize("W,pts,L", [(5, 4000, 6.0), (10, 20000, 12.0), (20, 6000, 8.0)])
def test_residual_and_cache_parity(ctx, W, pts, L):
    sc = scenes.make_window(W=W, pts_per_scan=pts, L=L, seed=3)
    f = gpu_factor(ctx, sc)
    of = sc["oracle_factor"]
    v, e, w = f.counts()
    assert v == of.size() and w == W
    r_gpu = ctx.evaluate_residual(f, sc["poses_true"])
    r_ref = of.residual(sc["poses_true"])
    assert abs(r_gpu - r_ref) / abs(r_ref) < 1e-10
    eig, s = f.read_back()
    ex = of.export()
    assert relinf(s, ex["sum10"]) < 1e-12
    check_eig(eig, ex["eig12"], 1e-7)   # lambda0 carries the cancellation of cov = P/N - c c^T (cond ~1e8): 1e-7 of lambda_max


@pytest.mark.parametrize("W,pts,L", [(5, 4000, 6.0), (10, 20000, 12.0), (20, 6000, 8.0), (37, 3000, 6.0), (50, 2500, 6.0), (70, 2000, 5.0), (130, 1200, 4.0)])
def test_hessian_parity(ctx, W, pts, L):
    sc = scenes.make_window(W=W, pts_per_scan=pts, L=L, seed=5)
    f = gpu_factor(ctx, sc)
    of = sc["oracle_factor"]
    H, J, r = ctx.evaluate_hessian(f, sc["poses_est"])
    Hr, Jr, rr = of.hessian(sc["poses_est"])
    assert abs(r - rr) / abs(rr) < 1e-12
    assert relinf(J, Jr) < 1e-9
    assert relinf(H, Hr) < 1e-9
    # blockwise: every 6x6 block that is non-zero in the oracle agrees to 1e-7 of its own scale
    n = 6 * W
    Hb, Hrb = H.reshape(W, 6, W, 6), Hr.reshape(W, 6, W, 6)
    scale = np.max(np.abs(Hrb), axis=(1, 3))
    err = np.max(np.abs(Hb - Hrb), axis=(1, 3))
    nz = scale > 0
    assert np.all(err[nz] / scale[nz] < 1e-7)
    assert np.all(err[~nz] == 0)


def test_sparse_window_path(ctx):
    """k << W: frames remapped into a wide window so that the pair-scatter kernel (k_pairs) is used."""
    sc = scenes.make_window(W=6, pts_per_scan=5000, L=6.0, seed=9)
    W2, stride = 60, 10
    n = sc["eig12"].shape[0]
    cl = np.zeros((n, W2, 10))
    cl[:, ::stride, :] = sc["clusters10"]
    poses = np.stack([synth.true_pose(6.0, 0)] * W2)
    poses[::stride] = sc["poses_est"]
    f = vx.Factor(ctx, W2)
    f.push_voxels_dense(cl, sc["eig12"], sc["sum10"], fix10=sc["fix10"])
    of = oa.OracleFactor.from_dense(W2, cl, sc["fix10"], None, sc["eig12"], sc["sum10"])
    H, J, r = ctx.evaluate_hessian(f, poses)
    Hr, Jr, rr = of.hessian(poses)
    assert relinf(H, Hr) < 1e-9 and relinf(J, Jr) < 1e-9 and abs(r - rr) / abs(rr) < 1e-12
    assert abs(ctx.evaluate_residual(f, poses) - of.residual(poses)) / abs(rr) < 1e-10


def test_csr_push_roundtrip_and_append(ctx):
    sc = scenes.make_window(W=5, pts_per_scan=3000, L=6.0, seed=2)
    cl = sc["clusters10"]
    n, W = cl.shape[0], cl.shape[1]
    ptr, fr, ent = [0], [], []
    for v in range(n):
        for i in range(W):
            if cl[v, i, 9] != 0:
                fr.append(i); ent.append(cl[v, i])
        ptr.append(len(fr))
    ptr, fr, ent = np.array(ptr), np.array(fr, dtype=np.int32), np.array(ent)
    f = vx.Factor(ctx, W)
    h = n // 2
    f.push_voxels(ptr[: h + 1], fr[: ptr[h]], ent[: ptr[h]], sc["eig12"][:h], sc["sum10"][:h], fix10=sc["fix10"][:h])
    f.push_voxels(ptr[h:] - ptr[h], fr[ptr[h]:], ent[ptr[h]:], sc["eig12"][h:], sc["sum10"][h:], fix10=sc["fix10"][h:])   # append => storage grows
    p2, f2, c2, fx2, co2 = f.read_structure()
    assert np.array_equal(p2, ptr) and np.array_equal(f2, fr) and np.array_equal(c2, ent) and np.array_equal(fx2, sc["fix10"]) and np.all(co2 == 1.0)
    e2, s2 = f.read_back()
    assert np.array_equal(e2, sc["eig12"]) and np.array_equal(s2, sc["sum10"])
    r = ctx.evaluate_residual(f, sc["poses_est"])
    assert abs(r - sc["oracle_factor"].residual(sc["poses_est"])) / r < 1e-10
    f.clear()
    assert f.counts()[0] == 0


@pytest.mark.parametrize("W,pts,L,iters", [(5, 4000, 6.0, 4), (10, 20000, 12.0, 4), (20, 6000, 8.0, 3)])
def test_lidar_ba_parity(ctx, W, pts, L, iters):
    sc = scenes.make_window(W=W, pts_per_scan=pts, L=L, seed=7)
    f = gpu_factor(ctx, sc)
    of = sc["oracle_factor"]
    g = ctx.lidar_ba(f, sc["poses_est"], max_iter=iters)
    r = of.lidar_ba(sc["poses_est"], max_iter=iters)
    assert g["status"] == 0 and len(g["trace"]) == len(r["trace"])
    for a, b in zip(g["trace"], r["trace"]):   # LM trace equality (SURVEY §8c pin 6)
        assert a["accepted"] == b["accepted"]
        assert abs(a["r1"] - b["r1"]) / b["r1"] < 1e-9 and abs(a["r2"] - b["r2"]) / b["r2"] < 1e-9
        assert abs(a["u"] - b["u"]) / b["u"] < 1e-5 and a["v"] == b["v"]
        assert abs(a["q1"] - b["q1"]) <= 1e-6 * abs(b["q1"]) + 1e-12 * b["r1"]
    dpose_ref = np.max(np.abs(r["poses"] - sc["poses_est"]))
    assert np.max(np.abs(g["poses"] - r["poses"])) < 1e-6 * dpose_ref          # solved pose increments within 1e-5 rel (held to 1e-6)
    assert relinf(g["hess"], r["hess"]) < 1e-8
    assert g["is_converge"] == r["is_converge"] and relinf(g["resis"], r["resis"]) < 1e-9
    # factor side effects read by OctoTree::margi (voxel_map.hpp:1217-1222)
    eig, s = f.read_back()
    ex = of.export()
    assert relinf(s, ex["sum10"]) < 1e-10


@pytest.mark.parametrize("gravity,iters", [(False, 3), (True, 3), (True, 5)])
def test_li_ba_parity(ctx, gravity, iters):
    W = 8
    sc = scenes.make_window(W=W, pts_per_scan=6000, L=8.0, seed=13)
    f = gpu_factor(ctx, sc)
    of = sc["oracle_factor"]
    st = scenes.states_from_poses(sc["poses_est"])
    st[:, 12:15] += 0.02 * np.random.default_rng(0).standard_normal((W, 3))
    imu_g = synth.ImuWindow(sc["poses_true"])
    imu_r = synth.ImuWindow(sc["poses_true"])
    g = ctx.li_ba(f, st, imu_g, with_gravity=gravity, max_iter=iters)
    r = of.li_ba(st, imu_r, with_gravity=gravity, max_iter=iters)
    assert len(g["trace"]) == len(r["trace"]) >= 1
    for a, b in zip(g["trace"], r["trace"]):
        assert a["accepted"] == b["accepted"]
        assert abs(a["r1"] - b["r1"]) / b["r1"] < 1e-8 and abs(a["r2"] - b["r2"]) / b["r2"] < 1e-8
    dref = np.max(np.abs(r["states"] - st))
    assert np.max(np.abs(g["states"] - r["states"])) < 1e-5 * dref
    assert relinf(g["hess"], r["hess"]) < 1e-8
    assert relinf(g["resis"], r["resis"]) < 1e-8


def test_too_few_voxels_is_an_error_not_an_exit(ctx):
    sc = scenes.make_window(W=5, pts_per_scan=3000, L=6.0, seed=2)
    f = vx.Factor(ctx, 5)
    f.push_voxels_dense(sc["clusters10"][:1], sc["eig12"][:1], sc["sum10"][:1])
    with pytest.raises(vx.VxsError) as ei:
        ctx.lidar_ba(f, sc["poses_est"], max_iter=2, thd_num=2)
    assert ei.value.code == -3


def test_two_concurrent_callers(ctx):
    """Local BA and global BA run on two threads in the reference (voxelslam.cpp:2617-2619): one ctx per thread."""
    sc = scenes.make_window(W=6, pts_per_scan=5000, L=6.0, seed=4)
    ref = sc["oracle_factor"].lidar_ba(sc["poses_est"], max_iter=3)
    outs = [None, None]

    def work(i):
        c = vx.Context(0)
        for _ in range(3):
            f = gpu_factor(c, sc)     # a solve overwrites the factor's cached eig/sums (voxel_map.hpp:271-273), so start fresh
            outs[i] = c.lidar_ba(f, sc["poses_est"], max_iter=3)
            f.close()
        c.close()

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    [t.start() for t in th]
    [t.join() for t in th]
    for o in outs:
        assert np.max(np.abs(o["poses"] - ref["poses"])) < 1e-8


def test_async_push_matches_sync_push(ctx):
    """vxs_factor_push_voxels_async: the chunked first Hessian build behind the upload events gives the same solve as the synchronous
    push (accumulation order differs: RED of four voxel chunks instead of one launch)."""
    W = 12
    sc = scenes.make_window(W=W, pts_per_scan=40000, L=14.0, seed=23)
    fs = gpu_factor(ctx, sc)
    ptr, fr, cl, fix, coe = fs.read_structure()
    eig, s = fs.read_back()
    assert ptr.shape[0] - 1 >= 256          # large enough for the chunked path
    ref = ctx.lidar_ba(fs, sc["poses_est"], max_iter=3, thd_num=2)
    hp = dict(ptr=vx.api.pinned_array(ptr.shape, np.int64), fr=vx.api.pinned_array(fr.shape, np.int32), cl=vx.api.pinned_array(cl.shape, np.float64),
              eig=vx.api.pinned_array(eig.shape, np.float64), s=vx.api.pinned_array(s.shape, np.float64), fix=vx.api.pinned_array(fix.shape, np.float64))
    hp["ptr"][:] = ptr; hp["fr"][:] = fr; hp["cl"][:] = cl; hp["eig"][:] = eig; hp["s"][:] = s; hp["fix"][:] = fix
    fa = vx.Factor(ctx, W)
    for rep in range(2):                     # second round: clear() while nothing is pending, then reuse of the staging buffers
        fa.clear()
        fa.push_voxels_async(hp["ptr"], hp["fr"], hp["cl"], hp["eig"], hp["s"], fix10=hp["fix"])
        got = ctx.lidar_ba(fa, sc["poses_est"], max_iter=3, thd_num=2)
        assert len(got["trace"]) == len(ref["trace"])
        for a, b in zip(got["trace"], ref["trace"]):
            assert a["accepted"] == b["accepted"] and abs(a["r1"] - b["r1"]) / b["r1"] < 1e-10 and abs(a["r2"] - b["r2"]) / b["r2"] < 1e-10
        assert got["trace"][0]["r1"] == ref["trace"][0]["r1"]      # same cached eigenvalues, same deterministic reduction
        assert np.max(np.abs(got["poses"] - ref["poses"])) < 1e-9 * np.max(np.abs(ref["poses"] - sc["poses_est"]))
        assert relinf(got["hess"], ref["hess"]) < 1e-12
    # consumers other than the Hessian build wait for the upload too
    fa.clear()
    fa.push_voxels_async(hp["ptr"], hp["fr"], hp["cl"], hp["eig"], hp["s"], fix10=hp["fix"])
    p2, f2, c2, _, _ = fa.read_structure()
    assert np.array_equal(p2, ptr) and np.array_equal(f2, fr) and np.array_equal(c2, cl)
    fa.clear()
    fa.push_voxels_async(hp["ptr"], hp["fr"], hp["cl"], hp["eig"], hp["s"], fix10=hp["fix"])
    assert abs(ctx.evaluate_residual(fa, sc["poses_est"]) - ctx.evaluate_residual(fs, sc["poses_est"])) <= 1e-12 * abs(ctx.evaluate_residual(fs, sc["poses_est"]))
    fa.sync_uploads()
