"""GPU parity of vxs_hba_bottom_batch — the bottom level of the hierarchical global BA for all windows at once (SURVEY.md §8a12, §8e(1)) —
against the oracle's HBA_add_edge restatement (voxelslam.cpp:2360-2427, pinned against the reference's OctreeGBA / Lidar_BA_Optimizer code by
tests/test_ref_pin.py) run window by window with max_iter = 1, and against the single-window device path."""
import numpy as np
import pytest

import oracle_api as oa
import scenes
import voxel_slam_b200 as vx
from parity_checks import compare_bottom_window

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = vx.Context(0)
    yield c
    c.close()


def trajectory(K, pts, L, seed, stride=3):
    tr, est = scenes.poses_true_est(K, L, seed, rot_sigma=3e-3, pos_sigma=2e-2)
    xyz, off = scenes.make_points(K, pts, L, seed, tr, dtype=np.float32)
    if stride != 3:
        wide = np.zeros((xyz.shape[0], stride), dtype=np.float32); wide[:, :3] = xyz; xyz = wide
    return tr, est, xyz, off


def oracle_window(fine, xyz, off, est, k0, ws):
    lo, hi = off[k0], off[k0 + ws]
    r = oa.hba_window(fine, fine, xyz[lo:hi], off[k0:k0 + ws + 1] - lo, est[k0:k0 + ws], max_iter=1, thread_num=2, stride_floats=xyz.shape[1])
    e = oa.hba_edges(r["hess"], ws, r["poses"])
    return r, e


@pytest.mark.parametrize("K,ws,step,pts,stride,chunk", [(25, 10, 5, 3000, 3, 0), (16, 6, 2, 2500, 12, 40000), (12, 10, 1, 2000, 3, 0)])
def test_bottom_batch_vs_per_window_oracle(ctx, K, ws, step, pts, stride, chunk):
    tr, est, xyz, off = trajectory(K, pts, 8.0, 60 + K, stride)
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    win_first = np.arange(0, K - ws + 1, step, dtype=np.int32)
    g = ctx.hba_bottom_batch(fine, xyz, off, est, win_first, win_size=ws, thread_num=2, max_points_per_chunk=chunk, want_hess=True)
    assert np.all(g["status"] == 0)
    for w, k0 in enumerate(win_first):
        r, e = oracle_window(fine, xyz, off, est, int(k0), ws)
        assert r["outer_iters"] == 1
        compare_bottom_window(g, w, r, e, est[k0:k0 + ws])     # poses, resis, raw Hessian, and the same edges in the same order
    # the windows move towards the truth
    w = 0
    assert np.abs(g["poses"][w][1:, 9:] - tr[win_first[w] + 1:win_first[w] + ws, 9:]).max() < np.abs(est[1:ws, 9:] - tr[1:ws, 9:]).max()


def test_bottom_batch_residual_with_poses_from_global_memory(ctx):
    """32 overlapping windows of 8 (W = 256 frames in one chunk), each owning its copy of a 24 m room's cells: enough voxels that the
    residual kernel's pose table does not fit in shared memory next to its batch accumulators"""
    from test_gpu_kernel_paths import resid_plan
    K, ws, nwin = 39, 8, 32
    tr, est, xyz, off = trajectory(K, 4000, 24.0, 71)
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    win_first = np.arange(nwin, dtype=np.int32)
    V = sum(oa.build_gba_factor(fine, xyz[off[k]:off[k + ws]], off[k:k + ws + 1] - off[k], est[k:k + ws], threads=2).size() for k in win_first)
    assert not resid_plan(V, nwin * ws)[1], V
    g = ctx.hba_bottom_batch(fine, xyz, off, est, win_first, win_size=ws, thread_num=2, want_hess=True)
    assert np.all(g["status"] == 0)
    for w, k0 in enumerate(win_first):
        r, e = oracle_window(fine, xyz, off, est, int(k0), ws)
        assert r["outer_iters"] == 1
        compare_bottom_window(g, w, r, e, est[k0:k0 + ws])


def test_bottom_batch_matches_the_single_window_device_path(ctx):
    K, ws = 15, 10
    tr, est, xyz, off = trajectory(K, 3000, 8.0, 91)
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    win_first = np.array([0, 5], dtype=np.int32)
    g = ctx.hba_bottom_batch(fine, xyz, off, est, win_first, win_size=ws)
    for w, k0 in enumerate(win_first):
        lo, hi = off[k0], off[k0 + ws]
        s = ctx.hba_window(fine, fine, xyz[lo:hi], off[k0:k0 + ws + 1] - lo, est[k0:k0 + ws], max_iter=1, thread_num=2)
        inc = np.max(np.abs(s["poses"] - est[k0:k0 + ws]))
        assert np.max(np.abs(g["poses"][w] - s["poses"])) < 1e-6 * inc


def test_bottom_batch_too_few_voxels_is_a_status_not_an_exit(ctx):
    """a window whose clouds give fewer plane voxels than thread_num: the reference exit(0)s (voxel_map.hpp:345-348); here its status says so and its poses stay"""
    K, ws = 12, 6
    tr, est, xyz, off = trajectory(K, 2500, 8.0, 93)
    xyz = xyz.copy()
    xyz[off[6]:off[12]] = np.random.default_rng(1).uniform(-50, 50, (off[12] - off[6], 3)).astype(np.float32)      # no planes in the second window
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    g = ctx.hba_bottom_batch(fine, xyz, off, est, np.array([0, 6], dtype=np.int32), win_size=ws)
    assert g["status"][0] == 0 and g["status"][1] == -3
    assert np.array_equal(g["poses"][1], est[6:12])


def test_submap_merge_batch_vs_per_window_oracle(ctx):
    """merge + down_sampling_voxel(voxel_size / 8) of every window in one pass: bit-exact float means, cells grouped by window in cell order"""
    K, ws = 20, 10
    tr, est, xyz, off = trajectory(K, 3000, 8.0, 97, stride=12)
    win_first = np.array([0, 5, 10], dtype=np.int32)
    poses_win = np.stack([est[k:k + ws] for k in win_first])
    for chunk in (0, 35000):
        g = ctx.submap_merge_batch(xyz, off, poses_win, win_first, 0.125, max_points_per_chunk=chunk)
        assert g["win_offsets"][0] == 0 and g["win_offsets"][-1] == g["n"] == len(g["xyz"])
        for w, k0 in enumerate(win_first):
            lo, hi = off[k0], off[k0 + ws]
            o = oa.submap_merge(xyz[lo:hi], off[k0:k0 + ws + 1] - lo, est[k0:k0 + ws], 0.125, stride_floats=12)
            a, b = g["win_offsets"][w], g["win_offsets"][w + 1]
            assert b - a == len(o["xyz"]) > 1000
            # the oracle reports cells in its hash-map order: match them through the index of the cell's first point
            ko, kg = np.argsort(o["index"]), np.argsort(g["index"][a:b])
            assert np.array_equal(o["index"][ko], g["index"][a:b][kg])
            assert np.array_equal(o["xyz"][ko].view(np.uint32), g["xyz"][a:b][kg].view(np.uint32)) and np.array_equal(o["count"][ko], g["count"][a:b][kg])


def test_hba_pass_equals_the_separate_calls(ctx):
    """vxs_hba_pass (device-resident clouds and submaps) == vxs_hba_bottom_batch + vxs_submap_merge_batch + vxs_hba_window through host buffers"""
    K, ws, st = 30, 10, 5
    tr, est, xyz, off = trajectory(K, 3000, 8.0, 99)
    fine = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    p = ctx.hba_pass(fine, fine, xyz, off, est, win_size=ws, win_stride=st)
    wf = np.arange(0, K - ws + 1, st, dtype=np.int32)
    b = ctx.hba_bottom_batch(fine, xyz, off, est, wf, win_size=ws)
    m = ctx.submap_merge_batch(xyz, off, b["poses"], wf, 0.125)
    top = ctx.hba_window(fine, fine, m["xyz"], m["win_offsets"], est[wf], max_iter=1, thread_num=5)
    # (the Hessian / gradient accumulators are fp64 REDs: two runs agree to rounding, not bit for bit)
    assert p["nwin"] == len(wf) and np.max(np.abs(p["bottom_poses"] - b["poses"])) < 1e-10 and np.array_equal(p["edge_valid"], b["edge_valid"])
    assert np.array_equal(p["submap_sizes"], np.diff(m["win_offsets"]))
    inc = np.max(np.abs(top["poses"] - est[wf]))
    assert inc > 0 and np.max(np.abs(p["top_poses"] - top["poses"])) < 1e-9 * max(inc, 1e-6) + 1e-13
    assert np.max(np.abs(p["top_resis"][:2] - top["resis_log"][:2]) / top["resis_log"][:2]) < 1e-10
    assert np.all(p["phase_ms"][[0, 1, 3, 4, 5]] > 0)
