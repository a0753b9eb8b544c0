"""The oracle against GOLDEN VECTORS PRODUCED BY THE REFERENCE'S OWN CODE (tests/golden/reference_outputs.json, written by
tests/golden/make_reference_golden.py from oracle/_ref/libvxref.so in the build container).  Unlike tests/test_ref_pin.py this needs neither
the reference sources nor the reference build: the inputs are re-created from the seeded harness generators (tests/golden_cases.py), so the pin holds on the
GPU box and in any checkout.  Tolerances are those of test_ref_pin.py (what is left is Eigen-internal summation order)."""
import json
import os

import numpy as np

import golden_cases as gc
import oracle_api as oa
import synth

HERE = os.path.dirname(os.path.abspath(__file__))
G = json.load(open(os.path.join(HERE, "golden", "reference_outputs.json")))["cases"]


def fh(lst, shape=None):
    a = np.array([float.fromhex(v) for v in lst])
    return a.reshape(shape) if shape is not None else a


def relinf(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / max(np.max(np.abs(b)), 1e-300))


def test_window_build_matches_the_reference_vectors():
    w, g = gc.window_case(), G["window_build"]
    ex = oa.build_window_factor(w["mp"], w["pts"], w["off"], w["est"]).export()
    order = np.lexsort([ex["ids"][k] for k in ("path", "layer", "z", "y", "x")])
    V = len(g["ids"])
    assert V > 30 and [[int(ex["ids"][k][i]) for k in ("x", "y", "z", "layer", "path")] for i in order] == g["ids"]       # voxel set: root cell, layer, octant path
    assert ex["clusters10"][order][:, :, 9].astype(int).tolist() == g["counts"]                                       # point-to-(voxel, frame) assignment, bit-exact
    s_ref = fh(g["sum10"], (V, 10))
    assert np.max(np.abs(ex["sum10"][order] - s_ref) / (np.abs(s_ref) + 1e-6)) < 1e-12
    l_ref = fh(g["lambda"], (V, 3))
    assert np.max(np.abs(ex["eig12"][order][:, :3] - l_ref) / np.max(np.abs(l_ref), axis=1, keepdims=True)) < 1e-12


def test_factor_evaluation_and_lidar_ba_match_the_reference_vectors():
    w, g = gc.window_case(), G["factor_eval"]
    f = oa.build_window_factor(w["mp"], w["pts"], w["off"], w["est"])
    H, J, r = f.hessian(w["est"])
    n = 6 * w["W"]
    r_ref = float.fromhex(g["residual_at_est_cached"])
    assert abs(r - r_ref) <= 1e-12 * abs(r_ref) and relinf(J, fh(g["jact"])) < 1e-11 and relinf(H, fh(g["hess"], (n, n))) < 1e-11
    rt = float.fromhex(g["residual_at_true"])
    assert abs(f.residual(w["tr"]) - rt) < 1e-10 * abs(r_ref)
    o = oa.build_window_factor(w["mp"], w["pts"], w["off"], w["est"]).lidar_ba(w["est"], max_iter=4, thd_num=2)
    gl = G["lidar_ba"]
    p_ref = fh(gl["poses"], (w["W"], 12))
    inc = np.max(np.abs(p_ref - w["est"]))
    assert inc > 1e-3 and np.max(np.abs(o["poses"] - p_ref)) < 1e-7 * inc
    assert relinf(o["resis"], fh(gl["resis"])) < 1e-10 and int(o["is_converge"]) == gl["is_converge"] and int(o["status"]) == gl["status"]


def test_li_ba_matches_the_reference_vectors():
    """LI_BA_Optimizer::damping_iter with the reference's real IMU_PRE (golden) vs the restatement with the harness IMU stand-in."""
    w, g = gc.window_case(), G["li_ba"]
    imu = synth.ImuWindow(w["tr"]); imu.reset()
    st0 = gc.states(w["est"])
    o = oa.build_window_factor(w["mp"], w["pts"], w["off"], w["est"]).li_ba(st0, imu, with_gravity=False, max_iter=3)
    s_ref = fh(g["states"], (w["W"], 24))
    inc = np.max(np.abs(s_ref - st0))
    assert inc > 1e-3 and np.max(np.abs(o["states"] - s_ref)) < 1e-6 * inc
    assert relinf(np.diag(o["hess"]), fh(g["hess_diag"])) < 1e-8 and int(o["status"]) == g["status"] and len(o["trace"]) == 3


def test_hba_add_edge_matches_the_reference_vectors():
    h, g = gc.hba_case(), G["hba_add_edge"]
    w = oa.hba_window(h["coarse"], h["fine"], h["xyz"], h["off"], h["est"], 4, thread_num=2)
    e = oa.hba_edges(w["hess"], h["W"], w["poses"])
    m = len(g["ij"])
    assert m == h["W"] * (h["W"] - 1) // 2 and e["ij"].tolist() == g["ij"]
    v_ref = fh(g["v6"], (m, 6))
    assert np.max(np.abs(e["v6"] - v_ref) / np.abs(v_ref)) < 1e-9
    assert np.max(np.abs(e["rot"] - fh(g["rot"], (m, 9)))) < 1e-11 and np.max(np.abs(e["tra"] - fh(g["tra"], (m, 3)))) < 1e-11
    sm = oa.submap_merge(h["xyz"], h["off"], w["poses"], h["fine"].voxel_size / 8)["xyz"]
    assert len(sm) == g["submap_n"]
    ks = np.lexsort(sm.T)
    assert np.array_equal(sm[ks][:64].ravel().astype(np.float64), fh(g["submap_head"]))                          # first cells (by position), bit-exact floats
    assert np.max(np.abs(sm.astype(np.float64).sum(axis=0) - fh(g["submap_sum"]))) < 1e-6


def test_local_map_and_ekf_update_match_the_reference_vectors():
    from test_ref_pin import _ekf_update_numpy
    m = gc.lio_case()
    lm = oa.LocalMap(m["mp"], m["pts"], m["off"], m["tr"], 1e-4, mgsize=1)
    pl, g = lm.planes(), G["local_map_planes"]
    kp = np.lexsort(np.round(pl["voxel_center"], 9).T)
    n = g["n"]
    assert len(kp) == n > 20 and np.array_equal(pl["voxel_center"][kp], fh(g["voxel_center"], (n, 3))) and pl["N"][kp].astype(int).tolist() == g["N"]
    assert np.max(np.abs(pl["center"][kp] - fh(g["center"], (n, 3)))) < 1e-12
    r_ref = fh(g["radius"])
    assert np.max(np.abs(pl["radius"][kp] - r_ref) / r_ref) < 1e-6
    ok, st, cov, nm = _ekf_update_numpy(lambda p_, x_, rv, tv: lm.odom_accumulate(p_, x_, rv, tv, passes=1), m["pv"], m["state"], m["cov"])
    ge = G["lio_state_estimation"]
    assert ok == ge["ok"] and 500 < nm <= len(m["pv"])
    s_ref, c_ref = fh(ge["state"]), fh(ge["cov"], (15, 15))
    assert np.max(np.abs(st[:21] - s_ref[:21])) < 1e-11 and np.max(np.abs(cov - c_ref)) / np.max(np.abs(c_ref)) < 1e-11
    assert np.max(np.abs(s_ref[:12] - m["state"][:12])) > 3e-3


def test_var_init_and_pvec_update_match_the_reference_vectors():
    v, g = gc.pointvar_case(), G["pointvar"]
    pv = oa.var_init(v["pts"], v["ext_R"], v["ext_p"], 0.02, 0.05)
    n = pv.shape[0]
    p_ref = fh(g["var_init"], (n, 12))
    assert np.array_equal(pv[:, :3], p_ref[:, :3])
    assert np.max(np.abs(pv[:, 3:] - p_ref[:, 3:]) / np.max(np.abs(p_ref[:, 3:]), axis=1, keepdims=True)) < 1e-12
    pu, pw = oa.pvec_update(p_ref, v["pose"], v["rot_var"], v["tsl_var"])
    u_ref = fh(g["pvec_update_var"], (n, 9))
    assert np.max(np.abs(pw - fh(g["pwld"], (n, 3)))) < 1e-12
    assert np.max(np.abs(pu[:, 3:] - u_ref) / np.max(np.abs(u_ref), axis=1, keepdims=True)) < 1e-12
