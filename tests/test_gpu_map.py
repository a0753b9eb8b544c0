"""GPU parity tests for the voxel-map construction (cut_voxel + recut + tras_opt; OctreeGBA) through the C-ABI.
Bit-exact: voxel keys, hash values, point-to-voxel assignment (per-(voxel, frame) point counts and the voxel identity set).
Floating point: cluster sums 1e-12 relative (summation order differs), eigenvalues 1e-7 of lambda_max."""
import json
import os

import numpy as np
import pytest

import oracle_api as oa
import scenes
import synth
import voxel_slam_b200 as vx
from parity_checks import compare_factors

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    yield c
    c.close()


def test_voxel_keys_golden_and_oracle(ctx):
    cases = json.load(open(os.path.join(HERE, "golden", "voxel_keys.json")))
    for vs in sorted({c["voxel_size"] for c in cases}):
        sub = [c for c in cases if c["voxel_size"] == vs]
        p = np.array([[float.fromhex(h) for h in c["p"]] for c in sub])
        xyz, h = ctx.voxel_keys(p, vs)
        assert xyz.tolist() == [c["key"] for c in sub]
        assert [int(v) for v in h] == [int(c["hash"]) for c in sub]
    rng = np.random.default_rng(7)
    p = np.concatenate([rng.uniform(-500, 500, (200000, 3)), np.round(rng.uniform(-50, 50, (5000, 3))), rng.uniform(-1e-6, 1e-6, (1000, 3))])
    for vs in (0.3, 1.0, 2.0):
        a, ha = ctx.voxel_keys(p, vs)
        b, hb = oa.voxel_keys(p, vs)
        assert np.array_equal(a, b) and np.array_equal(ha, hb)


@pytest.mark.parametrize("W,pts,L,max_layer,vs", [(4, 6000, 5.0, 2, 1.0), (10, 20000, 12.0, 2, 1.0), (6, 8000, 6.0, 0, 1.0), (5, 8000, 6.0, 3, 2.0), (7, 5000, 5.0, 1, 0.5)])
def test_window_factor_parity(ctx, W, pts, L, max_layer, vs):
    sc = scenes.make_window(W=W, pts_per_scan=pts, L=L, seed=17, max_layer=max_layer, voxel_size=vs)
    f = vx.Factor(ctx, W)
    n, ids = ctx.build_window_factor(sc["mp"], sc["pts"], sc["offsets"], sc["poses_est"], f, want_ids=True, ids_cap=sc["oracle_factor"].size() + 1000)
    assert n == f.counts()[0]
    compare_factors(f, ids, sc["oracle_factor"], W)
    # the device-resident factor is directly usable by the solver and gives the oracle's answer
    g = ctx.lidar_ba(f, sc["poses_est"], max_iter=3)
    r = sc["oracle_factor"].lidar_ba(sc["poses_est"], max_iter=3)
    assert np.max(np.abs(g["poses"] - r["poses"])) < 1e-6 * np.max(np.abs(r["poses"] - sc["poses_est"]))
    assert abs(g["resis"][1] - r["resis"][1]) / r["resis"][1] < 1e-8


def test_window_factor_negative_coordinates_and_plane_on_cell_boundary(ctx):
    """Adversarial placement (SURVEY trap B#1): the room is shifted so that cells have negative indices and one plane sits
    exactly on a cell boundary (x = 0)."""
    W, pts, L = 4, 8000, 5.0
    tr, est = scenes.poses_true_est(W, L, 23)
    p, off = scenes.make_points(W, pts, L, 23, tr)
    shift = np.array([-0.37 - 2.0, -7.37, -0.37])        # plane x=0.37 -> x=-2.0 (exact cell boundary), others negative
    tr2, est2 = tr.copy(), est.copy()
    tr2[:, 9:] += shift; est2[:, 9:] += shift
    mp = vx.MapParams.make()
    of = oa.build_window_factor(mp, p, off, est2)
    f = vx.Factor(ctx, W)
    n, ids = ctx.build_window_factor(mp, p, off, est2, f, want_ids=True, ids_cap=of.size() + 100)
    assert (ids["x"] < 0).any() and n > 20
    compare_factors(f, ids, of, W)


def test_window_factor_with_fixed_map_points(ctx):
    W, pts, L = 4, 6000, 5.0
    sc = scenes.make_window(W=W, pts_per_scan=pts, L=L, seed=29)
    fixp = synth.gen_scan(L, 77, 9000, synth.true_pose(L, 0), seed=99)            # body frame of pose 0 ...
    R0, t0 = sc["poses_true"][0, :9].reshape(3, 3), sc["poses_true"][0, 9:]
    fixw = fixp @ R0.T + t0                                                  # ... moved to the world: the "fixed map"
    of = oa.build_window_factor(sc["mp"], sc["pts"], sc["offsets"], sc["poses_est"], fix_pts=fixw)
    f = vx.Factor(ctx, W)
    n, ids = ctx.build_window_factor(sc["mp"], sc["pts"], sc["offsets"], sc["poses_est"], f, fix_pts=fixw, want_ids=True, ids_cap=of.size() + 100)
    assert np.abs(of.export()["fix10"]).max() > 0
    compare_factors(f, ids, of, W)
    r_g, r_o = ctx.evaluate_residual(f, sc["poses_true"]), of.residual(sc["poses_true"])
    assert abs(r_g - r_o) / r_o < 1e-9


def make_gba(W, pts, L, seed):
    tr, est = scenes.poses_true_est(W, L, seed, rot_sigma=3e-3, pos_sigma=2e-2)
    xyz, off = scenes.make_points(W, pts, L, seed, tr, dtype=np.float32)
    return tr, est, xyz, off


@pytest.mark.parametrize("stride", [3, 12])
def test_gba_factor_parity(ctx, stride):
    W = 8
    tr, est, xyz, off = make_gba(W, 5000, 8.0, 51)
    if stride != 3:   # pcl::PointXYZINormal layout: 48-byte points
        wide = np.zeros((xyz.shape[0], stride), dtype=np.float32); wide[:, :3] = xyz; xyz = wide
    mp = vx.MapParams.make(voxel_size=2.0, min_eigen_value=0.1, max_layer=2)
    of = oa.build_gba_factor(mp, xyz, off, est, threads=2, stride_floats=stride)
    f = vx.Factor(ctx, W)
    n, ids = ctx.build_gba_factor(mp, xyz, off, est, f, stride_floats=stride, want_ids=True, ids_cap=of.size() + 100)
    assert n > 10
    compare_factors(f, ids, of, W)


def test_hba_window_parity(ctx):
    W = 10
    tr, est, xyz, off = make_gba(W, 4000, 8.0, 53)
    coarse = vx.MapParams.make(voxel_size=2.0, min_eigen_value=0.1, max_layer=2)
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    g = ctx.hba_window(coarse, fine, xyz, off, est, max_iter=4, thread_num=2)
    r = oa.hba_window(coarse, fine, xyz, off, est, max_iter=4, thread_num=2)
    assert g["outer_iters"] == r["outer_iters"]
    assert np.max(np.abs(g["resis_log"] - r["resis_log"]) / r["resis_log"]) < 1e-6
    inc = np.max(np.abs(r["poses"] - est))
    assert np.max(np.abs(g["poses"] - r["poses"])) < 1e-5 * inc
    assert np.max(np.abs(g["hess"] - r["hess"])) < 1e-6 * np.max(np.abs(r["hess"]))
    assert np.abs(g["poses"] - tr).max() < 0.5 * np.abs(est - tr).max()


def test_hba_edges_on_device(ctx):
    """PGO edge extraction (voxelslam.cpp:2405-2427) from the device-resident raw Hessian vs the oracle on the oracle's Hessian."""
    W = 10
    tr, est, xyz, off = make_gba(W, 4000, 8.0, 57)
    coarse = vx.MapParams.make(voxel_size=2.0, min_eigen_value=0.1, max_layer=2)
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    g = ctx.hba_window(coarse, fine, xyz, off, est, max_iter=3, thread_num=2)
    e = ctx.hba_edges(W, g["poses"])
    r = oa.hba_window(coarse, fine, xyz, off, est, max_iter=3, thread_num=2)
    eo = oa.hba_edges(r["hess"], W, r["poses"])
    assert e["n"] == eo["n"] > 0 and np.array_equal(e["ij"], eo["ij"])         # same edges in the reference's lexicographic (i, j) order, unsorted
    assert np.max(np.abs(e["v6"] - eo["v6"]) / eo["v6"]) < 1e-6
    cap = e["n"] // 2                                                          # truncation keeps the FIRST cap edges, deterministically
    e2 = ctx.hba_edges(W, g["poses"], cap=cap)
    assert e2["n"] == e["n"] and np.array_equal(e2["ij"], e["ij"][:cap]) and np.array_equal(e2["v6"], e["v6"][:cap])
    # a different system on the ctx (n = 15 W) must be refused instead of being read with the wrong stride (ADVICE r1)
    sc = scenes.make_window(W=W, pts_per_scan=3000, L=6.0, seed=2)
    f = vx.Factor(ctx, W)
    f.push_voxels_dense(sc["clusters10"], sc["eig12"], sc["sum10"], fix10=sc["fix10"])
    ctx.li_ba(f, scenes.states_from_poses(sc["poses_est"]), synth.ImuWindow(sc["poses_true"]), max_iter=1)
    with pytest.raises(vx.VxsError):
        ctx.hba_edges(W, g["poses"])
    f.close()
    assert np.max(np.abs(e["rot"] - eo["rot"])) < 1e-9 and np.max(np.abs(e["tra"] - eo["tra"])) < 1e-8


def test_factor_cache_save_restore(ctx):
    sc = scenes.make_window(W=5, pts_per_scan=3000, L=6.0, seed=2)
    f = vx.Factor(ctx, 5)
    f.push_voxels_dense(sc["clusters10"], sc["eig12"], sc["sum10"], fix10=sc["fix10"])
    f.cache_save()
    a = ctx.lidar_ba(f, sc["poses_est"], max_iter=2)
    e1, _ = f.read_back()
    assert not np.array_equal(e1, sc["eig12"])              # the solve overwrote the cache
    f.cache_restore()
    e2, s2 = f.read_back()
    assert np.array_equal(e2, sc["eig12"]) and np.array_equal(s2, sc["sum10"])
    b = ctx.lidar_ba(f, sc["poses_est"], max_iter=2)
    assert np.max(np.abs(a["poses"] - b["poses"])) < 1e-12    # same re-run from the restored map state (fp64 RED order is the only difference)


def test_radix_sort_and_scan_at_scale(ctx):
    """1.5 M points, multiple sort tiles and scan blocks: per-voxel counts must still match the oracle exactly."""
    W, pts, L = 3, 500000, 30.0
    sc = scenes.make_window(W=W, pts_per_scan=pts, L=L, seed=61, threads=8)
    f = vx.Factor(ctx, W)
    n, ids = ctx.build_window_factor(sc["mp"], sc["pts"], sc["offsets"], sc["poses_est"], f, want_ids=True, ids_cap=sc["oracle_factor"].size() + 1000)
    compare_factors(f, ids, sc["oracle_factor"], W)


def _ds_cloud(n, seed, stride=3, span=40.0):
    rng = np.random.default_rng(seed)
    pts = np.zeros((n, stride), dtype=np.float32)
    pts[:, :3] = rng.uniform(-span, span, size=(n, 3)).astype(np.float32)
    pts[: n // 10, :3] = np.round(pts[: n // 10, :3] * 2) / 2      # on cell faces, incl. 0 and negatives (the loc < 0 branch)
    pts[n // 10: n // 5, :3] = pts[: n // 5 - n // 10, :3]           # exact duplicates
    if stride > 3:
        pts[:, 3:] = rng.uniform(size=(n, stride - 3)).astype(np.float32)
    return pts


@pytest.mark.parametrize("close", [False, True])
@pytest.mark.parametrize("stride,vs,span", [(3, 0.5, 40.0), (12, 0.125, 6.0), (3, 2.0, 6.0)])
def test_down_sampling_parity(ctx, close, stride, vs, span):
    """tools.hpp:201-302 — bit-exact against the oracle: same cells, same float means / picked points, same counts."""
    pts = _ds_cloud(200000, 5 + stride, stride, span)
    g = ctx.down_sampling(pts, vs, close=close, stride_floats=stride)
    o = oa.down_sampling(pts, vs, close=close, stride_floats=stride)
    assert len(g["index"]) == len(o["index"])
    go, oo = np.argsort(g["index"]), np.argsort(o["index"])
    assert np.array_equal(g["index"][go], o["index"][oo])
    assert np.array_equal(g["xyz"][go].view(np.uint32), o["xyz"][oo].view(np.uint32))
    assert np.array_equal(g["count"][go], o["count"][oo])
    assert int(g["count"].sum()) == pts.shape[0]
    # cells come out in ascending cell order
    k = oa.voxel_keys(pts[g["index"], :3].astype(np.float64), vs)[0]
    lin = (k[:, 0] - k[:, 0].min()) * (1 << 40) + (k[:, 1] - k[:, 1].min()) * (1 << 20) + (k[:, 2] - k[:, 2].min())
    assert np.all(np.diff(lin) > 0)


def test_down_sampling_edges_and_scale(ctx):
    pts = _ds_cloud(1000, 3)
    assert ctx.down_sampling(pts, 0.0005) is None and ctx.down_sampling(pts, 0.0005, close=True) is None
    assert len(ctx.down_sampling(pts[:0], 0.5)["index"]) == 0
    one = ctx.down_sampling(pts[:1], 0.5)
    assert one["index"].tolist() == [0] and np.array_equal(one["xyz"][0], pts[0, :3]) and one["count"][0] == 1
    # 5 M points: every point lands in exactly one cell, the first-point indices are unique, a second pass at the same size keeps
    # the number of cells or merges means that crossed a face (never grows)
    big = _ds_cloud(5_000_000, 9, 3, 120.0)
    g = ctx.down_sampling(big, 0.25)
    assert int(g["count"].sum()) == big.shape[0] and len(np.unique(g["index"])) == len(g["index"])
    g2 = ctx.down_sampling(g["xyz"], 0.25)
    assert len(g2["index"]) <= len(g["index"])
    c = ctx.down_sampling(big, 0.25, close=True)
    assert len(c["index"]) == len(g["index"]) and np.array_equal(c["xyz"], big[c["index"], :3])


@pytest.mark.parametrize("stride", [3, 12])
def test_submap_merge_parity(ctx, stride):
    """voxelslam.cpp:2428-2447 — merged cloud and its down-sampling bit-exact against the oracle."""
    rng = np.random.default_rng(31 + stride)
    W, per = 10, 30000
    poses = np.stack([synth.true_pose(20.0, i) for i in range(W)])
    pts = np.zeros((W * per, stride), dtype=np.float32)
    pts[:, :3] = rng.uniform(-25, 25, (W * per, 3)).astype(np.float32)
    off = np.arange(W + 1, dtype=np.int64) * per
    off[3] -= 1000                                           # ragged keyframes
    for vs in (0.0, 0.125, 1.0):
        g = ctx.submap_merge(pts, off, poses, vs, stride_floats=stride)
        o = oa.submap_merge(pts, off, poses, vs, stride_floats=stride)
        assert len(g["index"]) == len(o["index"])
        go, oo = np.argsort(g["index"]), np.argsort(o["index"])
        assert np.array_equal(g["index"][go], o["index"][oo])
        assert np.array_equal(g["xyz"][go].view(np.uint32), o["xyz"][oo].view(np.uint32))
        assert np.array_equal(g["count"][go], o["count"][oo])
    # empty window and empty keyframes
    e = ctx.submap_merge(pts[:0], np.zeros(W + 1, dtype=np.int64), poses, 0.125, stride_floats=stride)
    assert len(e["index"]) == 0


def test_down_sampling_pvec_parity(ctx):
    """voxel_map.hpp:23-64 — bit-exact against the oracle (fp64 running means in input order, float outputs)."""
    rng = np.random.default_rng(41)
    n = 150000
    pv = np.zeros((n, 12))
    pv[:, :3] = rng.uniform(-30.0, 30.0, (n, 3))
    pv[: n // 8, :3] = np.round(pv[: n // 8, :3] * 4) / 4
    pv[n // 8: n // 4, :3] = pv[: n // 4 - n // 8, :3]
    a = rng.uniform(-1e-2, 1e-2, (n, 3, 3))
    pv[:, 3:] = (a @ a.transpose(0, 2, 1)).reshape(n, 9)
    for vs in (0.5, 0.1):
        g = ctx.down_sampling_pvec(pv, vs)
        o = oa.down_sampling_pvec(pv, vs)
        assert len(g["index"]) == len(o["index"])
        go, oo = np.argsort(g["index"]), np.argsort(o["index"])
        assert np.array_equal(g["index"][go], o["index"][oo])
        assert np.array_equal(g["xyz"][go].view(np.uint32), o["xyz"][oo].view(np.uint32))
        assert np.array_equal(g["var_diag"][go].view(np.uint32), o["var_diag"][oo].view(np.uint32))
        assert np.array_equal(g["count"][go], o["count"][oo]) and int(g["count"].sum()) == n
    assert len(ctx.down_sampling_pvec(pv[:0], 0.5)["index"]) == 0


def test_odom_accumulate_parity(ctx):
    """voxelslam.cpp:876-918 + voxel_map.hpp:1335-1392, 1674-1698 — point -> plane-leaf association bit-exact against the oracle's octree
    descent (flags equal), accumulated HTH / HTz / nnt to 1e-9 (warp-tree + RED summation order)."""
    W, L, sigma = 4, 6.0, 0.01
    tr, _ = scenes.poses_true_est(W, L, 5)
    pts, off = scenes.make_points(W, 6000, L, 5, tr)
    mp = vx.MapParams.make(voxel_size=1.0, max_layer=2)
    lm = oa.LocalMap(mp, pts, off, tr, sigma ** 2, mgsize=1)
    P = lm.planes()
    layer = np.rint(np.log2(1.0 / (2.0 * P["half"]))).astype(np.int32)
    assert layer.min() >= 0 and layer.max() <= 2 and len(layer) > 50
    ctx.odom_set_planes(mp, P["voxel_center"], layer, P["center"], P["normal"], P["plane_var"], P["radius"])
    rng = np.random.default_rng(3)
    pose_true = synth.true_pose(L, W)
    body = synth.gen_scan(L, W, 20000, pose_true, seed=0x5EED0000 + 77)
    var = np.tile((sigma ** 2 * np.eye(3)).reshape(1, 9), (body.shape[0], 1)) * rng.uniform(0.5, 2.0, (body.shape[0], 1))
    pv = np.concatenate([body, var], axis=1)
    rot_var, tsl_var = 1e-6 * np.eye(3), 1e-4 * np.eye(3)
    for k, (rs, ps) in enumerate([(2e-3, 1e-2), (0.0, 0.0), (2e-2, 5e-2)]):
        pose = synth.perturb_pose(pose_true, 99 + k, rs, ps) if rs > 0 else pose_true
        g = ctx.odom_accumulate(pv if k == 0 else None, pose, rot_var, tsl_var, n=pv.shape[0])      # later passes re-use the resident scan
        o = lm.odom_accumulate(pv, pose, rot_var, tsl_var)
        assert g["n"] == o["n"] and (k == 2 or o["n"] > 3000)
        assert np.array_equal(g["flags"], o["flags"])
        for a, b in ((g["HTH"], o["HTH"]), (g["HTz"], o["HTz"]), (g["nnt"], o["nnt"])):
            assert np.max(np.abs(a - b)) <= 1e-9 * max(np.max(np.abs(b)), 1e-300)
    # empty plane table: nothing matches
    ctx.odom_set_planes(mp, P["voxel_center"][:0], layer[:0], P["center"][:0], P["normal"][:0], P["plane_var"][:0], P["radius"][:0])
    e = ctx.odom_accumulate(pv, pose_true, rot_var, tsl_var)
    assert e["n"] == 0 and not e["flags"].any() and not e["HTH"].any()


def test_down_sampling_golden_vectors(ctx):
    """The CUDA down-sampling kernels against the committed golden vectors (tests/golden/downsample.json), bit-exact."""
    scenes.check_downsample_against_golden(lambda p, vs: ctx.down_sampling(p, vs), lambda p, vs: ctx.down_sampling(p, vs, close=True), lambda pv, vs: ctx.down_sampling_pvec(pv, vs))
