"""Host-side legs of bench.py that need no GPU: the in-run cpu_baseline (oracle port + the reference's own sources when oracle/_ref was built) on a small
oracle-built factor.  A broken leg here would cost the bench line its cpu_baseline on the GPU box, where it cannot be debugged."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _small_csr():
    import bench
    import oracle_api as oa
    import voxel_slam_b200 as vx
    W = 10
    tr, est, p, off = bench.scene_points(vx, W, 20000, 12.0, seed=1)
    mp = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    ex = oa.build_window_factor(mp, p, off, est, threads=2).export()
    cl = ex["clusters10"]
    mask = cl[:, :, 9] > 0
    ptr = np.concatenate([[0], np.cumsum(mask.sum(1))]).astype(np.int64)
    vv, fr = np.nonzero(mask)
    return bench, vx, W, tr, est, ptr, fr.astype(np.int32), cl[vv, fr], ex["eig12"], ex["sum10"]


def test_cpu_baseline_from_structure_runs_on_host():
    bench, vx, W, tr, est, ptr, fr, cl, eig, s = _small_csr()
    out = bench.cpu_baseline_from_structure(vx, W, ptr, fr, cl, eig, s, bench.states_from(est), tr, reps=1)
    assert out["kind"] == "port" and out["cores"] == 5 and out["value"] > 0 and out["unit"] == bench.UNIT
    assert "error" not in out["all_cores_variant"], out["all_cores_variant"]
    assert out["first_iteration"]["r1"] > 0
    import ref_api as ra
    rs = out["reference_sources"]
    if ra.available():          # oracle/_ref is built where the reference sources exist (VXS_REFERENCE_SRC); on a box without it the leg must say so, not crash
        assert "error" not in rs, rs
        assert rs["kind"] == "reference" and rs["value"] > 0 and 1 <= rs["iterations_per_call"] <= 3


def test_csr_round_trip_matches_dense_oracle_factor():
    """oracle_factor_from_csr (the CSR the CUDA side exports -> the dense layout the oracle takes) must rebuild the same factor: same residual."""
    bench, vx, W, tr, est, ptr, fr, cl, eig, s = _small_csr()
    import oracle_api as oa
    of = bench.oracle_factor_from_csr(W, ptr, fr, cl, eig, s)
    dense = np.zeros((ptr.shape[0] - 1, W, 10))
    dense[np.repeat(np.arange(ptr.shape[0] - 1), np.diff(ptr)), fr] = cl
    od = oa.OracleFactor.from_dense(W, dense, None, None, eig, s)
    assert of.size() == od.size() == ptr.shape[0] - 1
    assert of.residual(est) == od.residual(est)
