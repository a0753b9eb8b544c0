"""Comparators shared by the GPU map-build, bottom-level batch and resident local map tests: a device factor against the oracle's factor, one
window of vxs_hba_bottom_batch against the oracle's HBA_add_edge restatement run on that window alone, and the leaves / factor of the resident
map (vxs_map_*) against the oracle's sliding-window simulator.

compare_factors and compare_bottom_window take an optional note(family, ratio) callback that receives the worst error / tolerance of each
comparison family."""
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


def pv_records(scan, seed, full=True):
    rng = np.random.default_rng(seed)
    if full:
        A = rng.standard_normal((scan.shape[0], 3, 3)) * 0.01
        var = A @ np.transpose(A, (0, 2, 1)) + np.eye(3) * 1e-5
    else:
        var = np.broadcast_to(np.eye(3) * 1e-4, (scan.shape[0], 3, 3))
    return np.concatenate([scan, var.reshape(-1, 9)], axis=1)


def leaf_key(s):
    return np.lexsort(np.concatenate([np.round(s["voxel_center"], 9), s["layer"][:, None]], axis=1).T)


def compare_leaves(sg, so, tag, tol=1e-10):
    assert sg["win_count"] == so["win_count"] and np.array_equal(sg["ring"], so["ring"]), tag
    kg, ko = leaf_key(sg), leaf_key(so)
    assert len(kg) == len(ko), (tag, len(kg), len(ko))
    for f in ("voxel_center", "half", "layer", "is_plane", "isexist", "has_sw", "in_slide", "last_num", "n_point_fix"):
        assert np.array_equal(sg[f][kg], so[f][ko]), (tag, f, int(np.sum(sg[f][kg] != so[f][ko])))
    assert np.array_equal(sg["opt_state"][kg] >= 0, so["opt_state"][ko] >= 0), tag
    for f in ("pcr_add", "pcr_fix", "slots"):
        x, y = sg[f][kg], so[f][ko]
        assert np.array_equal(x[..., 9], y[..., 9]), (tag, f)                                      # bit-exact point-to-leaf assignment
        assert np.max(np.abs(x - y) / (np.abs(y) + 1e-6)) < tol, (tag, f)


def compare_factor(f_gpu, of, W, tol=1e-10):
    ex = of.export()
    ptr, fr, cl, fx, co = f_gpu.read_structure()
    eig, s = f_gpu.read_back()
    assert len(s) == of.size()
    if len(s) == 0:
        return
    kg, ko = np.lexsort(np.round(s[:, [8, 7, 6, 9]], 7).T), np.lexsort(np.round(ex["sum10"][:, [8, 7, 6, 9]], 7).T)     # matched by point count + centroid
    dense = np.zeros((len(s), W, 10))
    vox = np.repeat(np.arange(len(s)), np.diff(ptr))
    dense[vox, fr] = cl
    assert np.array_equal(dense[kg][:, :, 9], ex["clusters10"][ko][:, :, 9])
    assert np.max(np.abs(dense[kg] - ex["clusters10"][ko]) / (np.abs(ex["clusters10"][ko]) + 1e-6)) < tol
    assert np.max(np.abs(s[kg] - ex["sum10"][ko]) / (np.abs(ex["sum10"][ko]) + 1e-6)) < tol
    assert np.max(np.abs(fx[kg] - ex["fix10"][ko]) / (np.abs(ex["fix10"][ko]) + 1e-6)) < tol
    lg, lo = eig[kg][:, :3], ex["eig12"][ko][:, :3]
    assert np.max(np.abs(lg - lo) / np.max(np.abs(lo), axis=1, keepdims=True)) < 1e-7
