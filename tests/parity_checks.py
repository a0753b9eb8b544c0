"""Comparators shared by the GPU map-build and bottom-level batch tests: a device factor against the oracle's factor, and one window of
vxs_hba_bottom_batch against the oracle's HBA_add_edge restatement run on that window alone.

Every comparator takes an optional note(family, ratio) callback that receives the worst error / tolerance of each comparison family."""
import numpy as np

ORDER = ["x", "y", "z", "layer", "path"]


def _noop(family, ratio):
    pass


def compare_factors(f_gpu, ids_gpu, of, W, note=_noop):
    """Voxel identity set and per-(voxel, frame) point counts bit-exact, cluster / point / fix sums to 1e-12 relative (summation order
    differs), eigenvalues to 1e-7 of lambda_max.  Returns the permutations that put the device and the oracle voxels in one order."""
    ex = of.export()
    assert len(ids_gpu) == of.size(), (len(ids_gpu), of.size())
    pg, po = np.argsort(ids_gpu, order=ORDER), np.argsort(ex["ids"], order=ORDER)
    assert np.array_equal(ids_gpu[pg], ex["ids"][po])                       # identical voxel set (root cell, layer, octant path)
    ptr, fr, cl, fx, co = f_gpu.read_structure()
    eig, s = f_gpu.read_back()
    dense = np.zeros((len(ids_gpu), W, 10))
    vox = np.repeat(np.arange(len(ids_gpu)), np.diff(ptr))
    dense[vox, fr] = cl
    assert np.all(np.diff(fr)[np.diff(vox) == 0] > 0)                        # frames ascending within a voxel
    dg, do = dense[pg], ex["clusters10"][po]
    assert np.array_equal(dg[:, :, 9], do[:, :, 9])                          # bit-exact per-(voxel, frame) point counts
    assert np.array_equal(s[pg][:, 9], ex["sum10"][po][:, 9])
    if len(ids_gpu) == 0:
        return pg, po
    sums = max(np.max(np.abs(dg - do) / (np.abs(do) + 1e-6)), np.max(np.abs(s[pg] - ex["sum10"][po]) / (np.abs(ex["sum10"][po]) + 1e-6)),
               np.max(np.abs(fx[pg] - ex["fix10"][po]) / (np.abs(ex["fix10"][po]) + 1e-6)))
    note("map sums", sums / 1e-12)
    assert sums < 1e-12
    assert np.all(co == 1.0)
    lam_g, lam_o = eig[pg][:, :3], ex["eig12"][po][:, :3]
    lam = np.max(np.abs(lam_g - lam_o) / np.max(np.abs(lam_o), axis=1, keepdims=True))
    note("map eigenvalues", lam / 1e-7)
    assert lam < 1e-7
    return pg, po


def compare_bottom_window(g, w, r, e, est_win, note=_noop):
    """Window w of a vxs_hba_bottom_batch result against the oracle's hba_window(max_iter = 1) result r and its PGO edges e: poses to 1e-5 of
    the increment, resis 1e-7, raw Hessian 1e-6 of its maximum (when the batch returned it), the same edges in the same order, variances 1e-5,
    relative rotations 1e-8 and translations 1e-7."""
    ws = est_win.shape[0]
    inc = np.max(np.abs(r["poses"] - est_win))
    dp = np.max(np.abs(g["poses"][w] - r["poses"]))
    note("bottom poses", dp / (1e-5 * inc))
    assert dp < 1e-5 * inc, (w, dp, inc)
    dr = np.max(np.abs(g["resis"][w] - r["resis_log"][:2]) / r["resis_log"][:2])
    note("bottom resis", dr / 1e-7)
    assert dr < 1e-7, (w, dr)
    if g.get("hess") is not None:
        dh = np.max(np.abs(g["hess"][w] - r["hess"])) / np.max(np.abs(r["hess"]))
        note("bottom hessian", dh / 1e-6)
        assert dh < 1e-6, (w, dh)
    pairs = [(i, j) for i in range(ws) for j in range(i + 1, ws)]
    valid = g["edge_valid"][w].astype(bool)
    ij = np.array([pairs[p] for p in range(len(pairs)) if valid[p]], dtype=np.int32).reshape(-1, 2)
    assert e["n"] == len(ij) and np.array_equal(ij, e["ij"]), w
    if e["n"]:
        dv = np.max(np.abs(g["edge_v6"][w][valid] - e["v6"]) / e["v6"])
        note("bottom edges", max(dv / 1e-5, np.max(np.abs(g["edge_rot"][w][valid] - e["rot"])) / 1e-8, np.max(np.abs(g["edge_tra"][w][valid] - e["tra"])) / 1e-7))
        assert dv < 1e-5, (w, dv)
        assert np.max(np.abs(g["edge_rot"][w][valid] - e["rot"])) < 1e-8 and np.max(np.abs(g["edge_tra"][w][valid] - e["tra"])) < 1e-7, w
