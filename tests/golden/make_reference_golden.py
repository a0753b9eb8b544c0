#!/usr/bin/env python
"""Golden vectors FROM THE REFERENCE'S OWN CODE.  Runs oracle/_ref/libvxref.so (the reference's hot-path sources compiled where they lie under
VXS_REFERENCE_SRC, see oracle/Makefile) on small seeded inputs and writes its outputs to tests/golden/reference_outputs.json.  The inputs are not
stored: they come from the seeded generators of tests/synth.py / tests/scenes.py, which travel with the repo, so tests/test_oracle_reference_golden.py
can re-create them anywhere (any checkout without the reference sources included) and hold the hand-written oracle against these vectors.

    python tests/golden/make_reference_golden.py        (needs oracle/_ref/libvxref.so)

Floats are written as C99 hex strings (exact)."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import golden_cases as gc          # noqa: E402  (tests/golden_cases.py: the shared input recipes)
import ref_api as ra               # noqa: E402


def hx(a):
    a = np.asarray(a, dtype=np.float64)
    return [float(v).hex() for v in a.ravel()]


def main():
    if not ra.available():
        sys.exit("oracle/_ref/libvxref.so is not built: run `make -C oracle ref` (VXS_REFERENCE_SRC = the reference's VoxelSLAM/src)")
    out = {"generator": "tests/golden/make_reference_golden.py", "source": "oracle/_ref/libvxref.so = Voxel-SLAM/VoxelSLAM/src/{tools,preintegration,voxel_map,loop_refine}.hpp + "
           "cut-outs of voxelslam.hpp / voxelslam.cpp, compiled unmodified against oracle/ref_standin", "cases": {}}
    c = out["cases"]
    # ---- a: a small window, from-scratch map build (cut_voxel + recut + tras_opt)
    w = gc.window_case()
    f = ra.build_window_factor(w["mp"], w["pts"], w["off"], w["est"])
    ex = f.export()
    order = np.lexsort([ex["ids"][k] for k in ("path", "layer", "z", "y", "x")])
    c["window_build"] = {"ids": [[int(ex["ids"][k][i]) for k in ("x", "y", "z", "layer", "path")] for i in order], "counts": ex["clusters10"][order][:, :, 9].astype(int).tolist(),
                         "sum10": hx(ex["sum10"][order]), "lambda": hx(ex["eig12"][order][:, :3])}
    # ---- b: acc_evaluate2 / evaluate_only_residual / Lidar_BA_Optimizer on that factor
    H, J, r = f.hessian(w["est"])
    c["factor_eval"] = {"residual_at_est_cached": float(r).hex(), "jact": hx(J), "hess": hx(H), "residual_at_true": float(f.residual(w["tr"])).hex()}
    f2 = ra.build_window_factor(w["mp"], w["pts"], w["off"], w["est"])
    o = f2.lidar_ba(w["est"], max_iter=4, thd_num=2)
    c["lidar_ba"] = {"poses": hx(o["poses"]), "resis": hx(o["resis"]), "is_converge": int(o["is_converge"]), "status": int(o["status"])}
    # ---- c: LI_BA_Optimizer (3 iterations, real IMU_PRE objects)
    f3 = ra.build_window_factor(w["mp"], w["pts"], w["off"], w["est"])
    imu = ra.RefImuWindow(w["tr"]); imu.reset()
    o = f3.li_ba(gc.states(w["est"]), imu, with_gravity=False, max_iter=3)
    c["li_ba"] = {"states": hx(o["states"]), "hess_diag": hx(np.diag(o["hess"])), "status": int(o["status"])}    # the reference's optimizer exposes no per-iteration trace
    # ---- d: HBA_add_edge (coarse -> fine loop, edges, merged submap)
    h = gc.hba_case()
    e = ra.hba_add_edge(h["coarse"], h["fine"], h["xyz"], h["off"], h["est"], 4, thread_num=2)
    ks = np.lexsort(e["submap"].T)
    c["hba_add_edge"] = {"ij": e["ij"].tolist(), "v6": hx(e["v6"]), "rot": hx(e["rot"]), "tra": hx(e["tra"]), "submap_n": int(len(e["submap"])),
                         "submap_head": [float(v).hex() for v in e["submap"][ks][:64].ravel()], "submap_sum": hx(e["submap"].astype(np.float64).sum(axis=0))}
    # ---- e: lio_state_estimation on a local map
    m = gc.lio_case()
    lm = ra.LocalMap(m["mp"], m["pts"], m["off"], m["tr"], 1e-4, mgsize=1)
    ok, st, cov = lm.lio_state_estimation(m["pv"], m["state"], m["cov"])
    c["lio_state_estimation"] = {"ok": bool(ok), "state": hx(st), "cov": hx(cov)}
    pl = lm.planes()
    kp = np.lexsort(np.round(pl["voxel_center"], 9).T)
    c["local_map_planes"] = {"n": int(len(kp)), "voxel_center": hx(pl["voxel_center"][kp]), "center": hx(pl["center"][kp]), "N": pl["N"][kp].astype(int).tolist(), "radius": hx(pl["radius"][kp])}
    # ---- f: var_init / pvec_update
    v = gc.pointvar_case()
    pv = ra.var_init(v["pts"], v["ext_R"], v["ext_p"], 0.02, 0.05)
    pu, pw = ra.pvec_update(pv, v["pose"], v["rot_var"], v["tsl_var"])
    c["pointvar"] = {"var_init": hx(pv), "pvec_update_var": hx(pu[:, 3:]), "pwld": hx(pw)}
    path = os.path.join(HERE, "reference_outputs.json")
    json.dump(out, open(path, "w"), indent=0)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
