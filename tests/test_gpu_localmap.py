"""GPU parity of the persistent device map (vxs_map_*: cut_voxel_multi + multi_recut + tras_opt per scan, multi_margi + plane_update after the
BA; SURVEY.md §8f rank 1) against the oracle's sliding-window simulator, which tests/test_ref_pin.py pins against the reference's own
OctoTree code.  After EVERY scan of a sequence the two maps must hold the same leaves (bit-exact cell / layer / flags / point counts, sums to
1e-10), the extracted factors must agree, and at the end the plane table and one odometry association pass are compared."""
import numpy as np
import pytest

import oracle_api as oa
import synth
import voxel_slam_b200 as vx
from parity_checks import compare_factor, compare_leaves, pv_records

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    yield c
    c.close()


def run_sequence(ctx, Wn, L, nscan, pts, max_layer, max_points, ba_iters, full_var, seed):
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=max_layer)
    sim = oa.SlidingSim(mp, Wn, 1, max_points=max_points)
    dm = vx.LocalMap(ctx, mp, Wn, max_points=max_points)
    f = vx.Factor(ctx, Wn)
    x_buf = []
    for i in range(nscan):
        pose = synth.true_pose(L, i)
        est = synth.perturb_pose(pose, seed * 100 + i, 2e-3, 1e-2) if i else pose
        pv = pv_records(synth.gen_scan(L, i, pts, pose, seed=0x5EED0000 + seed), seed + i, full_var)
        x_buf.append(est)
        dm.push_scan(pv, np.stack(x_buf), f)                       # cut_voxel_multi + multi_recut + tras_opt on the device
        if len(x_buf) >= Wn:
            if ba_iters > 0 and f.counts()[0] >= 2:
                o = ctx.lidar_ba(f, np.stack(x_buf), max_iter=ba_iters, thd_num=2, want_hess=False)
                x_buf = [p for p in o["poses"]]
            dm.margi(np.stack(x_buf), f, mgsize=1)                 # multi_margi + ring rotation
            x_buf = x_buf[1:]
        sim.add_scan_pv(pv, est, ba_iters=ba_iters)
        so = sim.state()
        if ba_iters > 0 and len(so["poses"]):
            assert np.max(np.abs(np.stack(x_buf) - so["poses"])) < 1e-8, i
        compare_leaves(dm.leaves(), so, i, tol=1e-10 if ba_iters == 0 else 1e-8)
    return dm, sim, f, mp


@pytest.mark.parametrize("Wn,pts,max_layer,max_points,ba_iters,full_var", [(5, 3000, 2, 100, 0, False), (6, 2500, 2, 60, 2, True), (4, 4000, 1, 100, 0, True), (5, 3000, 3, 40, 1, True)])
def test_sliding_window_map_sequence(ctx, Wn, pts, max_layer, max_points, ba_iters, full_var):
    nscan = Wn + 10
    dm, sim, f, mp = run_sequence(ctx, Wn, 6.0, nscan, pts, max_layer, max_points, ba_iters, full_var, seed=21 + Wn)
    c = dm.counts()
    assert c["win_count"] == Wn - 1 and c["fix_points"] > 0
    # the plane table plane_update left behind
    pg, po = dm.planes(), sim.planes()
    assert len(pg["N"]) == len(po["N"]) > 20
    kg, ko = np.lexsort(np.round(pg["voxel_center"], 9).T), np.lexsort(np.round(po["voxel_center"], 9).T)
    assert np.array_equal(pg["voxel_center"][kg], po["voxel_center"][ko]) and np.array_equal(pg["N"][kg], po["N"][ko])
    assert np.max(np.abs(pg["center"][kg] - po["center"][ko])) < 1e-9
    assert np.max(np.abs(pg["cov_trace"][kg] - po["cov_trace"][ko]) / po["cov_trace"][ko]) < 1e-9
    sgn = np.sign(np.sum(pg["normal"][kg] * po["normal"][ko], axis=1))
    assert np.max(np.abs(np.abs(np.sum(pg["normal"][kg] * po["normal"][ko], axis=1)) - 1)) < 1e-8
    Vo = po["plane_var"][ko].copy(); Vo[:, :3, 3:] *= sgn[:, None, None]; Vo[:, 3:, :3] *= sgn[:, None, None]
    assert np.max(np.abs(pg["plane_var"][kg] - Vo) / np.max(np.abs(Vo), axis=(1, 2), keepdims=True)) < 1e-5
    assert np.array_equal(pg["radius"][kg].astype(np.float32), po["radius"][ko].astype(np.float32)) or np.max(np.abs(pg["radius"][kg] - po["radius"][ko]) / po["radius"][ko]) < 1e-6
    # one association pass of the odometry EKF (voxelslam.cpp:876-918) against the RESIDENT map: no plane table is exported
    pose = synth.perturb_pose(synth.true_pose(6.0, nscan), 991, 1e-3, 5e-3)
    scan = pv_records(synth.gen_scan(6.0, nscan, 6000, synth.true_pose(6.0, nscan), seed=0x5EED0000 + 5), 77, True)
    rng = np.random.default_rng(3)
    A = rng.standard_normal((3, 3)) * 1e-3; B = rng.standard_normal((3, 3)) * 1e-2
    rot_var, tsl_var = A @ A.T, B @ B.T
    og, oo = dm.odom_accumulate(scan, pose, rot_var, tsl_var), sim.odom_accumulate(scan, pose, rot_var, tsl_var)
    assert oo["n"] > 500 and og["n"] == oo["n"] and np.array_equal(og["flags"], oo["flags"])
    for k in ("HTH", "HTz", "nnt"):
        assert np.max(np.abs(og[k] - oo[k])) / np.max(np.abs(oo[k])) < 1e-9, k
    og2 = dm.odom_accumulate(None, pose, rot_var, tsl_var, n=scan.shape[0])      # the scan stayed resident
    assert og2["n"] == og["n"] and np.array_equal(og2["HTH"] != 0, og["HTH"] != 0) and np.max(np.abs(og2["HTH"] - og["HTH"])) / np.max(np.abs(og["HTH"])) < 1e-12
    dm.close(); f.close()


def test_factor_of_every_scan_and_larger_scene(ctx):
    """W=10, 20 k pts/scan, L=12: the factor tras_opt extracts on the device after every scan vs the oracle's, through two window lengths of slides"""
    Wn, L, pts = 10, 12.0, 20000
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    sim = oa.SlidingSim(mp, Wn, 1, max_points=100)
    dm = vx.LocalMap(ctx, mp, Wn, max_points=100)
    f = vx.Factor(ctx, Wn)
    x_buf = []
    for i in range(2 * Wn + 3):
        pose = synth.true_pose(L, i)
        est = synth.perturb_pose(pose, 5000 + i, 1e-3, 5e-3) if i else pose
        pv = pv_records(synth.gen_scan(L, i, pts, pose, seed=0x5EED0000 + 77), 300 + i, True)
        x_buf.append(est)
        dm.push_scan(pv, np.stack(x_buf), f)
        # the oracle simulator extracts its factor inside add_scan (before its margi): compare before the device margi as well
        sim_f = None
        if len(x_buf) < Wn:
            sim.add_scan_pv(pv, est)
            compare_factor(f, sim.factor(), Wn)
        else:
            # window full: the simulator marginalises inside add_scan; its factor copy is the one tras_opt produced (margi only reads it)
            sim.add_scan_pv(pv, est)
            compare_factor(f, sim.factor(), Wn)
            dm.margi(np.stack(x_buf), f, mgsize=1)
            x_buf = x_buf[1:]
        compare_leaves(dm.leaves(), sim.state(), i)
    assert f.counts()[0] > 300
    dm.close(); f.close()


def test_push_scan_argument_checks(ctx):
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    dm = vx.LocalMap(ctx, mp, 3)
    f = vx.Factor(ctx, 3)
    pose = synth.true_pose(6.0, 0)
    pv = pv_records(synth.gen_scan(6.0, 0, 500, pose), 1)
    with pytest.raises(vx.VxsError):
        dm.push_scan(pv, np.stack([pose, pose]), f)                # win_count must be resident scans + 1
    dm.push_scan(pv, pose[None, :], f)
    dm.push_scan(pv[:0], np.stack([pose, pose]), f)                # an empty scan is legal
    assert dm.counts()["win_count"] == 2
    dm.close(); f.close()
