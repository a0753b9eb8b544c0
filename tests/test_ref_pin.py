"""PINS THE ORACLE AGAINST THE REFERENCE'S OWN SOURCE (CPU).

oracle/_ref/libvxref.so is the reference's hot-path code itself — VoxelSLAM/src/{tools,preintegration,voxel_map,loop_refine}.hpp
compiled unmodified (oracle/Makefile, `ref` target) against stand-ins for the absent third-party headers (oracle/ref_standin/: an eager
mini-Eigen restating Eigen 3.3.7's published kernels, PCL / ROS / GTSAM declarations).  Every check below runs the SAME seeded inputs through
that library (ref_api) and through the hand-written restatement (oracle_api) that the GPU parity tests compare against, so the restatement's
control flow, constants and formulas are anchored in the reference's real code; the tolerance left over is Eigen-internal summation order.
Also pins the harness's IMU stand-in (tests/harness/synth.hpp) against the real IMU_PRE.

The reference's side is replayed from what that library returned for these same calls (tests/ref_replay.py, tapes under tests/golden/ref_pin/,
re-recorded with VXS_RECORD_REFERENCE=1 where the reference build exists), so the comparison runs in every checkout, with or without the reference
sources."""
import json
import os

import numpy as np
import pytest

import oracle_api as oa
import ref_replay
import scenes
import synth
import voxel_slam_b200 as vx

ra = ref_replay.reference()
HERE = os.path.dirname(os.path.abspath(__file__))
ORDER = ["x", "y", "z", "layer", "path"]


@pytest.fixture(autouse=True)
def _reference_tape(request):
    ref_replay.tape.begin(request.node.name.replace("[", "__").replace("]", "").replace("/", "_"))
    yield
    ref_replay.tape.end()


def relinf(a, b):
    return float(np.max(np.abs(np.ma.asarray(a) - np.ma.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def same(a, b):
    """np.array_equal over the rows a recorded reference array kept (all rows of an array that is not a sample)"""
    if not (np.ma.isMaskedArray(a) or np.ma.isMaskedArray(b)):
        return np.array_equal(a, b)
    return np.shape(a) == np.shape(b) and bool(np.all((np.ma.asarray(a) == np.ma.asarray(b)).filled(True)))


def same_rows(a, b):
    """a and b hold the same rows in any order (bit for bit: pass integer views); for a recorded sample, its rows are rows of b"""
    if not np.ma.isMaskedArray(a):
        return len(a) == len(b) and np.array_equal(a[np.lexsort(a.T)], b[np.lexsort(b.T)])
    rows = {r.tobytes() for r in np.ascontiguousarray(b)}
    kept = np.ascontiguousarray(a.data[~np.ma.getmaskarray(a).any(axis=1)])
    return len(a) == len(b) and all(r.tobytes() in rows for r in kept)


def test_keys_and_hash_bit_exact():
    cases = json.load(open(os.path.join(HERE, "golden", "voxel_keys.json")))
    for vs in sorted({c["voxel_size"] for c in cases}):
        sub = [c for c in cases if c["voxel_size"] == vs]
        p = np.array([[float.fromhex(h) for h in c["p"]] for c in sub])
        xyz, h = ra.voxel_keys(p, vs)                      # the reference's cut_voxel + std::hash<VOXEL_LOC>
        assert xyz.tolist() == [c["key"] for c in sub]
        assert [int(v) for v in h] == [int(c["hash"]) for c in sub]
    rng = np.random.default_rng(7)
    p = np.concatenate([rng.uniform(-500, 500, (20000, 3)), np.round(rng.uniform(-50, 50, (2000, 3))), rng.uniform(-1e-6, 1e-6, (500, 3)), rng.uniform(-3e7, 3e7, (500, 3))])
    for vs in (0.3, 1.0, 2.0, 15.0):
        a, ha = ra.voxel_keys(p, vs)
        b, hb = oa.voxel_keys(p, vs)
        assert same(a, b) and same(ha, hb)


def test_eigensolver_qr_vs_jacobi():
    """Eigen's tridiagonal-QR (stand-in restatement of SelfAdjointEigenSolver::compute) vs the oracle's cyclic Jacobi vs LAPACK."""
    rng = np.random.default_rng(3)
    worst = 0.0
    for t in range(400):
        if t % 2 == 0:                                     # thin plane far from the origin: cov = P/N - c c^T with heavy cancellation
            n = rng.standard_normal(3); n /= np.linalg.norm(n)
            pts = rng.uniform(-0.5, 0.5, (50, 3)); pts -= np.outer(pts @ n, n) * (1 - 0.01)
            pts += rng.uniform(-100, 100, 3)
            A = np.cov(pts.T, bias=True)
        else:
            B = rng.standard_normal((3, 3)); A = B @ B.T * 10 ** rng.uniform(-6, 3)
        wr, Ur = ra.eig3(A)
        wo, Uo = oa.eig3(A)
        wn = np.linalg.eigvalsh(A)
        s = max(abs(wn).max(), 1e-300)
        assert np.max(np.abs(wr - wn)) < 1e-13 * s and np.max(np.abs(wo - wn)) < 1e-13 * s
        worst = max(worst, np.max(np.abs(wr - wo)) / s)
        assert np.allclose(Ur @ Ur.T, np.eye(3), atol=1e-13)
        for k in range(3):
            gap = min(abs(wn[k] - wn[j]) for j in range(3) if j != k) / s
            if gap > 1e-4:
                assert abs(abs(Ur[:, k] @ Uo[:, k]) - 1) < 1e-9 / gap * 1e-4 + 1e-12
    assert worst < 1e-14


def test_point_cluster_and_exp():
    rng = np.random.default_rng(5)
    pts = rng.uniform(-30, 30, (500, 3))
    assert same(ra.cluster_from_points(pts), oa.cluster_from_points(pts))            # same operations in the same order: bit-exact
    c = oa.cluster_from_points(pts)
    for i in range(20):
        pose = synth.perturb_pose(synth.true_pose(20.0, i), 99 + i, 0.3, 5.0)
        a, b = ra.cluster_transform(c, pose), oa.cluster_transform(c, pose)
        assert np.max(np.abs(a - b) / (np.abs(b) + 1e-9)) < 1e-14
    for w in ([0, 0, 0], [1e-12, 0, 0], [1e-11, 2e-11, 0], [0.3, -0.2, 0.9], [3.0, 0.1, -0.2]):
        assert np.max(np.abs(ra.so3_exp(w) - oa.so3_exp(w))) < 1e-16 + 1e-15


@pytest.mark.parametrize("W,pts,L", [(5, 4000, 6.0), (10, 8000, 10.0)])
def test_factor_residual_hessian_and_lidar_ba(W, pts, L):
    sc = scenes.make_window(W=W, pts_per_scan=pts, L=L, seed=3)
    of = sc["oracle_factor"]
    rf = ra.OracleFactor.from_dense(W, sc["clusters10"], sc["fix10"], None, sc["eig12"], sc["sum10"])
    assert rf.size() == of.size()
    # acc_evaluate2 with the map-time cache
    Hr, Jr, rr = rf.hessian(sc["poses_est"])
    Ho, Jo, ro = of.hessian(sc["poses_est"])
    assert abs(rr - ro) <= 1e-15 * abs(ro) and relinf(Jr, Jo) < 1e-12 and relinf(Hr, Ho) < 1e-12
    Hb = Hr.reshape(W, 6, W, 6)
    assert all(same(Hb[i, :, j, :], Hb[j, :, i, :].T) for i in range(W) for j in range(i))   # lower block triangle mirrored (voxel_map.hpp:237-239)
    # evaluate_only_residual + the cache it leaves behind
    # sum of lambda_0: every lambda_0 (~1e-4) carries the eigensolvers' 1e-16 * lambda_max (QR here, Jacobi in the restatement)
    assert abs(rf.residual(sc["poses_true"]) - of.residual(sc["poses_true"])) < 1e-11 * abs(ro)
    er, eo = rf.export(), of.export()
    assert relinf(er["sum10"], eo["sum10"]) < 1e-14
    assert np.max(np.abs(er["eig12"][:, :3] - eo["eig12"][:, :3]) / np.max(np.abs(eo["eig12"][:, :3]), axis=1, keepdims=True)) < 1e-9
    # Lidar_BA_Optimizer::damping_iter, thread split included
    for iters, thd in ((4, 2), (3, 1)):
        a = ra.OracleFactor.from_dense(W, sc["clusters10"], sc["fix10"], None, sc["eig12"], sc["sum10"]).lidar_ba(sc["poses_est"], max_iter=iters, thd_num=thd)
        b = oa.OracleFactor.from_dense(W, sc["clusters10"], sc["fix10"], None, sc["eig12"], sc["sum10"]).lidar_ba(sc["poses_est"], max_iter=iters, thd_num=thd)
        inc = np.max(np.abs(b["poses"] - sc["poses_est"]))
        assert np.max(np.abs(a["poses"] - b["poses"])) < 1e-8 * inc
        assert relinf(a["hess"], b["hess"]) < 1e-10 and relinf(a["resis"], b["resis"]) < 1e-11 and a["is_converge"] == b["is_converge"]


def test_too_few_voxels_is_the_reference_exit_path():
    sc = scenes.make_window(W=5, pts_per_scan=3000, L=6.0, seed=2)
    rf = ra.OracleFactor.from_dense(5, sc["clusters10"][:1], sc["fix10"][:1], None, sc["eig12"][:1], sc["sum10"][:1])
    assert rf.lidar_ba(sc["poses_est"], max_iter=2, thd_num=2)["status"] == -3


def test_imu_standin_matches_real_imu_pre():
    """tests/harness/synth.hpp ImuPre (what bench.py and the GPU tests hand to vxs_li_ba) vs the reference's IMU_PRE on the same samples."""
    W = 8
    tr = np.stack([synth.true_pose(8.0, i) for i in range(W)])
    st = scenes.states_from_poses(np.stack([synth.perturb_pose(tr[i], 50 + i, 2e-3, 1e-2) for i in range(W)]))
    st[:, 12:15] += 0.02 * np.random.default_rng(0).standard_normal((W, 3))
    st[:, 15:21] += 1e-3 * np.random.default_rng(1).standard_normal((W, 6))
    a, b = ra.RefImuWindow(tr), synth.ImuWindow(tr)
    for g in (False, True):
        ca, Ba, ga = a.eval(st, with_gravity=g)
        cb, Bb, gb = b.eval(st, with_gravity=g)
        assert abs(ca - cb) < 1e-9 * abs(cb) and relinf(Ba, Bb) < 1e-9 and relinf(ga, gb) < 1e-9


@pytest.mark.parametrize("gravity,iters", [(False, 3), (True, 3), (True, 5)])
def test_li_ba_against_the_reference_optimizers(gravity, iters):
    W = 8
    sc = scenes.make_window(W=W, pts_per_scan=6000, L=8.0, seed=13)
    st = scenes.states_from_poses(sc["poses_est"])
    st[:, 12:15] += 0.02 * np.random.default_rng(0).standard_normal((W, 3))
    rf = ra.OracleFactor.from_dense(W, sc["clusters10"], sc["fix10"], None, sc["eig12"], sc["sum10"])
    of = oa.OracleFactor.from_dense(W, sc["clusters10"], sc["fix10"], None, sc["eig12"], sc["sum10"])
    a = rf.li_ba(st, ra.RefImuWindow(sc["poses_true"]), with_gravity=gravity, max_iter=iters)      # LI_BA_Optimizer(+Gravity)::damping_iter + IMU_PRE
    b = of.li_ba(st, synth.ImuWindow(sc["poses_true"]), with_gravity=gravity, max_iter=iters)      # restatement + harness IMU stand-in
    inc = np.max(np.abs(b["states"] - st))
    assert np.max(np.abs(a["states"] - b["states"])) < 1e-6 * inc
    assert relinf(a["hess"], b["hess"]) < 1e-8
    if gravity:
        assert relinf(a["resis"], b["resis"]) < 1e-9
    ea, eb = rf.export(), of.export()                                                              # cache left for OctoTree::margi
    assert relinf(ea["sum10"], eb["sum10"]) < 1e-9


def compare_factor_sets(ea, eb, W, tol=1e-12):
    assert len(ea["ids"]) == len(eb["ids"])
    pa, pb = np.argsort(ea["ids"], order=ORDER), np.argsort(eb["ids"], order=ORDER)
    assert same(ea["ids"][pa], eb["ids"][pb])
    ca, cb = ea["clusters10"][pa], eb["clusters10"][pb]
    assert same(ca[:, :, 9], cb[:, :, 9])                                                 # bit-exact point-to-(voxel, frame) assignment
    assert np.max(np.abs(ca - cb) / (np.abs(cb) + 1e-6)) < tol
    for k in ("sum10", "fix10"):
        assert np.max(np.abs(ea[k][pa] - eb[k][pb]) / (np.abs(eb[k][pb]) + 1e-6)) < tol
    la, lb = ea["eig12"][pa][:, :3], eb["eig12"][pb][:, :3]
    assert np.max(np.abs(la - lb) / np.max(np.abs(lb), axis=1, keepdims=True)) < 1e-12


@pytest.mark.parametrize("W,pts,L,ml", [(5, 6000, 6.0, 2), (4, 20000, 14.0, 2), (3, 5000, 6.0, 0), (6, 3000, 5.0, 3)])
def test_window_map_build(W, pts, L, ml):
    """cut_voxel + OctoTree::recut + tras_opt (the reference's motion_init sequence) vs the restatement: identical voxel set and assignment."""
    tr, est = scenes.poses_true_est(W, L, 11)
    p, off = scenes.make_points(W, pts, L, 11, tr)
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=ml)
    a, b = ra.build_window_factor(mp, p, off, est), oa.build_window_factor(mp, p, off, est)
    assert a.size() == b.size() > 20
    compare_factor_sets(a.export(), b.export(), W)
    # fixed map points + a shifted scene (negative coordinates, a plane on a cell face)
    sh = np.array([-7.37, -3.37, -0.37])
    est2 = est.copy(); est2[:, 9:] += sh
    fix = (p[: pts // 2] @ tr[0, :9].reshape(3, 3).T + tr[0, 9:]) + sh
    a, b = ra.build_window_factor(mp, p, off, est2, fix_pts=fix), oa.build_window_factor(mp, p, off, est2, fix_pts=fix)
    assert a.size() == b.size() > 20
    compare_factor_sets(a.export(), b.export(), W)


@pytest.mark.parametrize("vs,me,thre,minp,ml", [(0.5, 0.0025, (0.25, 0.25, 0.25, 0.25), (5, 5, 5, 5), 2), (2.0, 0.01, (0.1, 0.15, 0.2, 0.3), (20, 12, 8, 5), 3),
                                                (1.0, 0.001, (1 / 16.0, 1 / 9.0, 1 / 4.0, 1.0), (30, 20, 10, 5), 2), (1.5, 0.05, (0.5, 0.5, 0.5, 0.5), (5, 5, 5, 5), 1)])
def test_window_map_build_nondefault_parameters(vs, me, thre, minp, ml):
    """The same sequence under parameter sets away from the launch-file defaults: voxel size, min_eigen_value, per-layer plane thresholds
    (plane_eigen_value_thre, already inverted as voxelslam.cpp:825 leaves them) and per-layer min_point — every branch of plane_judge / recut keyed on them."""
    W, pts, L = 5, 8000, 9.0
    tr, est = scenes.poses_true_est(W, L, 23)
    p, off = scenes.make_points(W, pts, L, 23, tr)
    mp = vx.MapParams.make(voxel_size=vs, min_eigen_value=me, plane_thre=thre, min_point=tuple(float(x) for x in minp), max_layer=ml)
    a, b = ra.build_window_factor(mp, p, off, est), oa.build_window_factor(mp, p, off, est)
    assert a.size() == b.size() > 5
    compare_factor_sets(a.export(), b.export(), W)
    ga, gb = ra.build_gba_factor(mp, p.astype(np.float32), off, est, threads=2).export(), oa.build_gba_factor(mp, p.astype(np.float32), off, est, threads=2).export()
    assert len(ga["sum10"]) == len(gb["sum10"]) > 5
    ka = np.lexsort(np.round(ga["sum10"][:, [8, 7, 6, 9]], 6).T); kb = np.lexsort(np.round(gb["sum10"][:, [8, 7, 6, 9]], 6).T)
    assert same(ga["clusters10"][ka][:, :, 9], gb["clusters10"][kb][:, :, 9])
    assert np.max(np.abs(ga["sum10"][ka] - gb["sum10"][kb]) / (np.abs(gb["sum10"][kb]) + 1e-6)) < 1e-12


def test_ragged_and_empty_scans():
    """Edge cases of the map builds and the down-sampling: scans of very different sizes, an EMPTY scan and a one-point scan inside the window; empty and
    one-point clouds through down_sampling_voxel."""
    W, L = 6, 7.0
    tr, est = scenes.poses_true_est(W, L, 31)
    sizes = [5000, 0, 1, 7000, 37, 2500]
    scans = [synth.gen_scan(L, i, max(n, 1), tr[i], seed=0x5EED0000 + 31)[:n] for i, n in enumerate(sizes)]
    p = np.concatenate(scans); off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    a, b = ra.build_window_factor(mp, p, off, est), oa.build_window_factor(mp, p, off, est)
    assert a.size() == b.size() > 50
    ea, eb = a.export(), b.export()
    compare_factor_sets(ea, eb, W)
    assert np.all(eb["clusters10"][:, 1, 9] == 0) and np.sum(eb["clusters10"][:, 2, 9]) <= 1            # the empty scan observes nothing, the one-point scan at most one voxel
    ga, gb = ra.build_gba_factor(mp, p.astype(np.float32), off, est, threads=2).export(), oa.build_gba_factor(mp, p.astype(np.float32), off, est, threads=2).export()
    assert len(ga["sum10"]) == len(gb["sum10"]) > 50
    ka = np.lexsort(np.round(ga["sum10"][:, [8, 7, 6, 9]], 6).T); kb = np.lexsort(np.round(gb["sum10"][:, [8, 7, 6, 9]], 6).T)
    assert same(ga["clusters10"][ka][:, :, 9], gb["clusters10"][kb][:, :, 9])
    for cloud in (np.zeros((0, 3), dtype=np.float32), np.array([[1.25, -2.5, 0.75]], dtype=np.float32)):
        da, db = ra.down_sampling(cloud, 0.5), oa.down_sampling(cloud, 0.5)
        assert len(da["xyz"]) == len(db["xyz"]) == len(cloud) and same(da["xyz"], db["xyz"]) and same(da["count"], db["count"])


def test_gba_map_build():
    W = 6
    tr, est = scenes.poses_true_est(W, 8.0, 41, rot_sigma=3e-3, pos_sigma=2e-2)
    xyz, off = scenes.make_points(W, 3000, 8.0, 41, tr, dtype=np.float32)
    for vs, me in ((2.0, 0.1), (1.0, 0.0025)):
        mp = vx.MapParams.make(voxel_size=vs, min_eigen_value=me, max_layer=2)
        for thd in (1, 2):
            ea, eb = ra.build_gba_factor(mp, xyz, off, est, threads=thd).export(), oa.build_gba_factor(mp, xyz, off, est, threads=thd).export()
            assert len(ea["sum10"]) == len(eb["sum10"]) > 10
            # OctreeGBA keeps no identity: voxels are matched by their (exactly equal) point counts and centroids
            ka = np.lexsort(np.round(ea["sum10"][:, [8, 7, 6, 9]], 6).T); kb = np.lexsort(np.round(eb["sum10"][:, [8, 7, 6, 9]], 6).T)
            assert same(ea["clusters10"][ka][:, :, 9], eb["clusters10"][kb][:, :, 9])
            assert np.max(np.abs(ea["clusters10"][ka] - eb["clusters10"][kb]) / (np.abs(eb["clusters10"][kb]) + 1e-6)) < 1e-12
            assert np.max(np.abs(ea["sum10"][ka] - eb["sum10"][kb]) / (np.abs(eb["sum10"][kb]) + 1e-6)) < 1e-12


def test_down_sampling():
    rng = np.random.default_rng(8)
    pts = np.concatenate([rng.uniform(-20, 20, (30000, 3)), np.round(rng.uniform(-5, 5, (500, 3)))]).astype(np.float32)
    for vs in (0.25, 1.0):
        for close in (False, True):
            a, b = ra.down_sampling(pts, vs, close=close), oa.down_sampling(pts, vs, close=close)
            # same cells (identified by their first / picked point), float running means bit-exact, same counts
            cells = lambda d, m: m.column_stack([d["index"].astype(np.int64), d["xyz"].view(np.uint32).astype(np.int64)] + ([] if close else [d["count"].astype(np.int64)]))
            assert same_rows(cells(a, np.ma), cells(b, np))
    assert ra.down_sampling(pts, 0.0005) is None
    pv = np.concatenate([rng.uniform(-20, 20, (20000, 3)), rng.uniform(0, 1e-3, (20000, 9))], axis=1)
    a, b = ra.down_sampling_pvec(pv, 0.5), oa.down_sampling_pvec(pv, 0.5)
    assert same_rows(np.ma.concatenate([a["xyz"], a["var_diag"]], axis=1).view(np.uint32), np.concatenate([b["xyz"], b["var_diag"]], axis=1).view(np.uint32))


def test_margi_plane_update_and_match():
    """OctoTree::margi + plane_update (incl. the cov_add by-product of push) + match + the EKF accumulation loop."""
    W, L = 4, 6.0
    tr, est = scenes.poses_true_est(W, L, 5)
    pts, off = scenes.make_points(W, 6000, L, 5, tr)
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    a, b = ra.LocalMap(mp, pts, off, tr, 1e-4, mgsize=1), oa.LocalMap(mp, pts, off, tr, 1e-4, mgsize=1)
    pa, pb = a.planes(), b.planes()
    assert len(pa["N"]) == len(pb["N"]) > 20
    ka, kb = np.lexsort(np.round(pa["voxel_center"], 9).T), np.lexsort(np.round(pb["voxel_center"], 9).T)
    assert same(pa["voxel_center"][ka], pb["voxel_center"][kb]) and same(pa["half"][ka], pb["half"][kb]) and same(pa["N"][ka], pb["N"][kb])
    assert np.max(np.abs(pa["center"][ka] - pb["center"][kb])) < 1e-13
    assert np.max(np.abs(np.abs(np.sum(pa["normal"][ka] * pb["normal"][kb], axis=1)) - 1)) < 1e-9          # normals up to sign
    Va, Vb = pa["plane_var"][ka], pb["plane_var"][kb]
    sgn = np.sign(np.sum(pa["normal"][ka] * pb["normal"][kb], axis=1))
    Vb = Vb.copy(); Vb[:, :3, 3:] *= sgn[:, None, None]; Vb[:, 3:, :3] *= sgn[:, None, None]              # cov(n, c) flips with the sign of n
    assert np.max(np.abs(Va - Vb) / (np.max(np.abs(Vb), axis=(1, 2), keepdims=True))) < 1e-6
    assert same(pa["radius"][ka], pb["radius"][kb]) or np.max(np.abs(pa["radius"][ka] - pb["radius"][kb]) / pb["radius"][kb]) < 1e-6
    # odometry association of a new scan: match flags bit-exact, sums 1e-9
    pose = synth.perturb_pose(tr[W - 1], 77, 1e-3, 5e-3)
    scan = synth.gen_scan(L, W - 1, 4000, tr[W - 1], seed=0x5EED0000 + 5)
    pv = np.zeros((scan.shape[0], 12)); pv[:, :3] = scan; pv[:, [3, 7, 11]] = 1e-4
    rv, tv = np.eye(3) * 1e-6, np.eye(3) * 1e-5
    for passes in (1, 2):
        oa_, ob_ = a.odom_accumulate(pv, pose, rv, tv, passes=passes), b.odom_accumulate(pv, pose, rv, tv, passes=passes)
        assert oa_["n"] == ob_["n"] > 500 and same(oa_["flags"], ob_["flags"])
        assert relinf(oa_["HTH"], ob_["HTH"]) < 1e-9 and relinf(oa_["HTz"], ob_["HTz"]) < 1e-9 and relinf(oa_["nnt"], ob_["nnt"]) < 1e-9


def test_sliding_window_map_sequence():
    """voxelslam.cpp:1599-1712 map side over 14 scans with a 5-scan window: after EVERY scan the two implementations hold the same leaves with the
    same slot clusters, fix clusters, plane flags, opt_state and ring."""
    Wn, L, nscan = 5, 6.0, 14
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    a, b = ra.SlidingSim(mp, Wn, 1, max_points=100), oa.SlidingSim(mp, Wn, 1, max_points=100)
    for i in range(nscan):
        pose = synth.true_pose(L, i)
        est = synth.perturb_pose(pose, 700 + i, 1e-3, 5e-3) if i else pose
        scan = synth.gen_scan(L, i, 3000, pose, seed=0x5EED0000 + 21)
        a.add_scan(scan, est); b.add_scan(scan, est)
        sa, sb = a.state(), b.state()
        assert sa["win_count"] == sb["win_count"] and sa["win_base"] == sb["win_base"] and same(sa["ring"], sb["ring"])
        assert same(sa["poses"], sb["poses"])
        key = lambda s: np.lexsort(np.concatenate([np.round(s["voxel_center"], 9), s["layer"][:, None]], axis=1).T)
        ka, kb = key(sa), key(sb)
        assert len(ka) == len(kb)
        for f in ("voxel_center", "half", "layer", "is_plane", "isexist", "has_sw", "in_slide", "last_num", "n_point_fix"):
            assert same(sa[f][ka], sb[f][kb]), (i, f)
        assert same(sa["opt_state"][ka] >= 0, sb["opt_state"][kb] >= 0)
        for f in ("pcr_add", "pcr_fix", "slots"):
            x, y = sa[f][ka], sb[f][kb]
            assert same(x[..., 9], y[..., 9]), (i, f)
            assert np.max(np.abs(x - y) / (np.abs(y) + 1e-6)) < 1e-11, (i, f)
    assert sa["win_base"] == nscan - Wn + 1 and int(np.sum(sa["pcr_fix"][:, 9] > 0)) > 10       # scans were marginalised into pcr_fix


def _pv_records(scan, seed):
    """pointVar records with a full (symmetric positive) per-point variance, as pvec_update leaves them"""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((scan.shape[0], 3, 3)) * 0.01
    var = A @ np.transpose(A, (0, 2, 1)) + np.eye(3) * 1e-5
    return np.concatenate([scan, var.reshape(-1, 9)], axis=1)


def test_sliding_window_with_ba_between_recut_and_margi():
    """The loop as the reference runs it: per scan cut + recut + tras_opt, then (window full) a BA that moves x_buf and overwrites the factor cache,
    then margi reads pcr_add / eig back from the factor (opt_state path) — reference build vs restatement, plus the plane table and one odometry pass."""
    Wn, L, nscan = 6, 6.0, 16
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    a, b = ra.SlidingSim(mp, Wn, 1, max_points=60), oa.SlidingSim(mp, Wn, 1, max_points=60)
    for i in range(nscan):
        pose = synth.true_pose(L, i)
        est = synth.perturb_pose(pose, 900 + i, 2e-3, 1e-2) if i else pose
        pv = _pv_records(synth.gen_scan(L, i, 2500, pose, seed=0x5EED0000 + 33), i)
        a.add_scan_pv(pv, est, ba_iters=2); b.add_scan_pv(pv, est, ba_iters=2)
        sa, sb = a.state(), b.state()
        assert sa["win_count"] == sb["win_count"] and same(sa["ring"], sb["ring"])
        assert np.max(np.abs(sa["poses"] - sb["poses"])) < 1e-9                                   # x_buf after the BA
        key = lambda s: np.lexsort(np.concatenate([np.round(s["voxel_center"], 9), s["layer"][:, None]], axis=1).T)
        ka, kb = key(sa), key(sb)
        for f in ("voxel_center", "layer", "is_plane", "isexist", "has_sw", "in_slide", "last_num", "n_point_fix"):
            assert same(sa[f][ka], sb[f][kb]), (i, f)
        for f in ("pcr_add", "pcr_fix", "slots"):
            x, y = sa[f][ka], sb[f][kb]
            assert same(x[..., 9], y[..., 9]), (i, f)
            assert np.max(np.abs(x - y) / (np.abs(y) + 1e-6)) < 1e-8, (i, f)
    fa, fb = a.factor().export(), b.factor().export()
    assert len(fa["sum10"]) == len(fb["sum10"]) > 20
    pa, pb = a.planes(), b.planes()
    assert len(pa["N"]) == len(pb["N"]) > 20
    ka, kb = np.lexsort(np.round(pa["voxel_center"], 9).T), np.lexsort(np.round(pb["voxel_center"], 9).T)
    assert same(pa["N"][ka], pb["N"][kb]) and np.max(np.abs(pa["center"][ka] - pb["center"][kb])) < 1e-9
    assert np.max(np.abs(pa["cov_trace"][ka] - pb["cov_trace"][kb]) / pb["cov_trace"][kb]) < 1e-10      # the Bf_var accumulation with full variances
    sgn = np.sign(np.sum(pa["normal"][ka] * pb["normal"][kb], axis=1))
    Vb = pb["plane_var"][kb].copy(); Vb[:, :3, 3:] *= sgn[:, None, None]; Vb[:, 3:, :3] *= sgn[:, None, None]
    assert np.max(np.abs(pa["plane_var"][ka] - Vb) / np.max(np.abs(Vb), axis=(1, 2), keepdims=True)) < 1e-5
    pose = synth.perturb_pose(synth.true_pose(L, nscan), 78, 1e-3, 5e-3)
    pv = _pv_records(synth.gen_scan(L, nscan, 3000, synth.true_pose(L, nscan), seed=0x5EED0000 + 33), 99)
    oa_, ob_ = a.odom_accumulate(pv, pose, np.eye(3) * 1e-6, np.eye(3) * 1e-5), b.odom_accumulate(pv, pose, np.eye(3) * 1e-6, np.eye(3) * 1e-5)
    assert oa_["n"] == ob_["n"] > 300 and same(oa_["flags"], ob_["flags"])
    assert relinf(oa_["HTH"], ob_["HTH"]) < 1e-8 and relinf(oa_["HTz"], ob_["HTz"]) < 1e-8


def test_var_init_and_pvec_update_against_the_reference_functions():
    """calcBodyVar / var_init / pvec_update (voxelslam.hpp:163-214, cut out of voxelslam.hpp at build time): the restatement vs the reference's code,
    incl. a point with z == 0 (the reference moves it to z = 1e-4) and points on the axes' neighbourhood."""
    rng = np.random.default_rng(5)
    n = 4000
    pts = np.zeros((n, 12), dtype=np.float32)                       # PointType stride (12 floats)
    pts[:, :3] = rng.uniform(-40, 40, (n, 3)).astype(np.float32)
    pts[0, :3] = (3.0, -2.0, 0.0)                                  # z == 0 trap (voxelslam.hpp:165)
    pts[1, :3] = (0.01, 0.02, 35.0)
    pts[2, :3] = (25.0, -25.0, 1e-3)
    ext_R = oa.so3_exp(np.array([0.02, -0.01, 0.03])); ext_p = np.array([0.05, -0.02, 0.1])
    a = oa.var_init(pts, ext_R, ext_p, 0.02, 0.05)
    b = ra.var_init(pts, ext_R, ext_p, 0.02, 0.05)
    assert same(a[:, :3], b[:, :3])
    assert np.max(np.abs(a[:, 3:] - b[:, 3:]) / (np.max(np.abs(b[:, 3:]), axis=1, keepdims=True))) < 1e-12
    assert abs(a[0, 2] - (ext_R @ np.array([3.0, -2.0, 1e-4]) + ext_p)[2]) < 1e-15
    pose = np.concatenate([oa.so3_exp(np.array([0.3, 0.1, -0.2])).ravel(), [5.0, -3.0, 1.0]])
    A = rng.standard_normal((3, 3)) * 1e-3; rot_var = A @ A.T
    B = rng.standard_normal((3, 3)) * 1e-2; tsl_var = B @ B.T
    pa, wa = oa.pvec_update(a, pose, rot_var, tsl_var)
    pb, wb = ra.pvec_update(a, pose, rot_var, tsl_var)
    assert same(pa[:, :3], a[:, :3])                      # pnt stays in the body frame
    assert np.max(np.abs(wa - wb)) < 1e-12
    assert np.max(np.abs(pa[:, 3:] - pb[:, 3:]) / np.max(np.abs(pb[:, 3:]), axis=1, keepdims=True)) < 1e-12


@pytest.mark.parametrize("max_iter", [1, 4])
def test_hba_add_edge_against_the_reference_member_function(max_iter):
    """The reference's own HBA_add_edge (voxelslam.cpp:2319-2482, cut out of the ROS node class at build time): coarse -> fine outer loop over OctreeGBA map
    builds and Lidar_BA_Optimizer solves, the PGO edges of the final Hessian and the merged + down-sampled submap — against the oracle's hba_window /
    hba_edges / submap_merge chain that the GPU tests (vxs_hba_window, vxs_hba_edges, vxs_submap_merge, vxs_hba_bottom_batch, vxs_hba_pass) compare with.
    The reference optimises a private copy of the poses, so they are pinned through the edges' relative poses and the merged cloud."""
    W = 8
    tr, est = scenes.poses_true_est(W, 8.0, 43, rot_sigma=3e-3, pos_sigma=2e-2)
    xyz, off = scenes.make_points(W, 4000, 8.0, 43, tr, dtype=np.float32)
    coarse = vx.MapParams.make(voxel_size=2.0, min_eigen_value=0.1, max_layer=2)
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    a = ra.hba_add_edge(coarse, fine, xyz, off, est, max_iter, thread_num=2)
    w = oa.hba_window(coarse, fine, xyz, off, est, max_iter, thread_num=2)
    assert w["status"] == 0 and w["outer_iters"] == max_iter
    e = oa.hba_edges(w["hess"], W, w["poses"])
    assert a["n"] == e["n"] == W * (W - 1) // 2 and same(a["ij"], e["ij"])      # lexicographic (i, j), voxelslam.cpp:2405-2406
    assert np.max(np.abs(a["v6"] - e["v6"]) / np.abs(e["v6"])) < 1e-10
    assert np.max(np.abs(a["rot"] - e["rot"])) < 1e-12 and np.max(np.abs(a["tra"] - e["tra"])) < 1e-12
    assert np.max(np.abs(w["poses"] - est)) > 1e-4                                       # the solve moved the poses: the edges above are not the input's
    m = oa.submap_merge(xyz, off, w["poses"], fine.voxel_size / 8)
    assert len(a["submap"]) == len(m["xyz"]) > 1000
    assert same_rows(a["submap"].view(np.uint32), m["xyz"].view(np.uint32))          # float running means of the same cells, bit-exact


def _hat(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def _so3_log(R):                      # tools.hpp:86-91
    tr_ = np.trace(R)
    th = 0.0 if tr_ > 3.0 - 1e-6 else np.arccos(0.5 * (tr_ - 1))
    K = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return 0.5 * K if abs(th) < 0.001 else 0.5 * th / np.sin(th) * K


def _ekf_update_numpy(accum, pv, st, cov, num_max_iter=4):
    """lio_state_estimation (voxelslam.cpp:856-954) with its association + accumulation loop (:876-918) replaced by `accum`: a FULL match of every point in
    every iteration — what vxs_odom_accumulate / vxs_map_odom_accumulate do — instead of the reference's per-point leaf cache (octos[i])."""
    x_prop, x, cov = st.copy(), st.copy(), cov.copy()
    G, H15, I15 = np.zeros((15, 15)), np.zeros((15, 15)), np.eye(15)
    rematch = 0
    cov_inv = np.linalg.inv(cov)
    for it in range(num_max_iter):
        o = accum(pv, x[:12], cov[:3, :3], cov[3:6, 3:6])
        H15[:6, :6] = o["HTH"]
        K1 = np.linalg.inv(H15 + cov_inv)
        G[:, :6] = K1[:, :6] @ o["HTH"]
        vec = np.zeros(15)                                                          # x_prop - x_curr, IMUST::operator- (tools.hpp:164-173)
        vec[:3] = _so3_log(x[:9].reshape(3, 3).T @ x_prop[:9].reshape(3, 3)); vec[3:] = x_prop[9:21] - x[9:21]
        sol = K1[:, :6] @ o["HTz"] + vec - G[:, :6] @ vec[:6]
        x = x.copy(); x[:9] = (x[:9].reshape(3, 3) @ oa.so3_exp(sol[:3])).ravel(); x[9:21] += sol[3:]   # IMUST::operator+= (tools.hpp:154-162)
        conv = np.linalg.norm(sol[:3]) * 57.3 < 0.01 and np.linalg.norm(sol[3:6]) * 100 < 0.015
        if conv or (rematch == 0 and it == num_max_iter - 2):
            rematch += 1
        if rematch >= 2 or it == num_max_iter - 1:
            cov = (I15 - G) @ cov
            break
    return bool(np.linalg.eigvalsh(o["nnt"])[0] >= 14), x, cov, o["n"]


@pytest.mark.parametrize("sigma", [0.01, 0.12])
def test_lio_state_estimation_against_the_reference_member_function(sigma):
    """The reference's whole odometry update (lio_state_estimation, voxelslam.cpp:856-954, cut out of the node class at build time: up to 4 EKF iterations, each
    re-associating the scan through its per-point leaf cache) against the oracle's accumulation with a full match per iteration + the 15x15 EKF algebra in numpy.
    Equal to rounding -> the leaf cache is a pure shortcut and the CUDA path (no cache, full match per call) reproduces the reference's update; sigma = 0.12
    leaves ~30 % of the points unmatched (3-sigma gates), which is where a cached leaf and a fresh descent could disagree."""
    W, L = 4, 6.0
    tr, est = scenes.poses_true_est(W, L, 5)
    pts, off = scenes.make_points(W, 6000, L, 5, tr)
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    a, b = ra.LocalMap(mp, pts, off, tr, 1e-4, mgsize=1), oa.LocalMap(mp, pts, off, tr, 1e-4, mgsize=1)
    scan = synth.gen_scan(L, W - 1, 4000, tr[W - 1], seed=0x5EED0000 + 5, sigma=sigma)
    pv = np.zeros((scan.shape[0], 12)); pv[:, :3] = scan; pv[:, [3, 7, 11]] = 1e-4
    for seed, rs, ps in ((77, 1e-3, 5e-3), (79, 2e-2, 8e-2)):
        st = np.zeros(24); st[:12] = synth.perturb_pose(tr[W - 1], seed, rs, ps); st[12:15] = (0.3, -0.1, 0.05); st[21:24] = (0, 0, -9.8)
        cov = np.diag([1e-4] * 3 + [1e-3] * 3 + [1e-2] * 3 + [1e-6] * 6)
        ok_r, st_r, cov_r = a.lio_state_estimation(pv, st, cov)
        ok_o, st_o, cov_o, nm = _ekf_update_numpy(lambda p_, x_, rv, tv: b.odom_accumulate(p_, x_, rv, tv, passes=1), pv, st, cov)
        assert ok_r == ok_o and (nm == 4000 if sigma < 0.05 else 2000 < nm < 3500)
        assert np.max(np.abs(st_r[:21] - st_o[:21])) < 1e-12 and np.max(np.abs(cov_r - cov_o)) / np.max(np.abs(cov_o)) < 1e-12
        assert np.max(np.abs(st_r[:12] - st[:12])) > 3e-3                                   # the update moved the state ...
        if sigma < 0.05 or ps > 0.05:                                                          # (a 5 mm start error is below what a 12 cm noise scan resolves)
            assert np.max(np.abs(st_r[9:12] - tr[W - 1][9:12])) < np.max(np.abs(st[9:12] - tr[W - 1][9:12]))   # ... towards the truth
