#!/usr/bin/env python
"""Per-scan cost of the odometry's iterated EKF update (lio_state_estimation, voxelslam.cpp:856-958) against the resident local map, two ways:

  (a) the host loop a caller writes without vxs_map_lio_update: up to 4 vxs_map_odom_accumulate passes (each ends in a synchronisation and
      brings the 34 sums back), the 15x15 EKF algebra in numpy between them, stopping where the reference stops;
  (b) one vxs_map_lio_update call (all iterations enqueued on the device, one read-back).

The scene is bench.py's local-mapping scene (W = 50 scans in the window, L = 130 m): the window is filled and warmed first, then every measured scan
is var_init'ed (resident, untimed), updated by (a) and by (b) in alternating order, and pushed into the map (push_scan + margi) as the loop would.
Host wall clock around calls that end in a synchronisation.  Prints one JSON line; the card's name and power limit are read in the same run.
    python tools/lio_probe.py [--points 20000 1000000] [--scans 50]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import synth  # noqa: E402
import voxel_slam_b200 as vx  # noqa: E402

COV = np.diag([1e-4] * 3 + [1e-3] * 3 + [1e-2] * 3 + [1e-6] * 6)


def so3_exp(w):                                       # tools.hpp:51-66
    n = np.linalg.norm(w)
    if n < 1e-11:
        return np.eye(3)
    a = w / n
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(n) * K + (1.0 - np.cos(n)) * K @ K


def so3_log(R):                                       # tools.hpp:86-91
    tr = np.trace(R)
    th = 0.0 if tr > 3.0 - 1e-6 else np.arccos(0.5 * (tr - 1))
    K = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return 0.5 * K if abs(th) < 0.001 else 0.5 * th / np.sin(th) * K


def host_loop(dm, n, st, cov):
    """(a): the EKF loop of voxelslam.cpp:870-956 on the host around vxs_map_odom_accumulate passes over the resident scan"""
    x_prop, x, cov = st.copy(), st.copy(), cov.copy()
    G, H15 = np.zeros((15, 15)), np.zeros((15, 15))
    cov_inv = np.linalg.inv(cov)
    rematch = 0
    for it in range(4):
        o = dm.odom_accumulate(None, x[:12], cov[:3, :3], cov[3:6, 3:6], n=n, want_flags=False)
        H15[:6, :6] = o["HTH"]
        K1 = np.linalg.inv(H15 + cov_inv)
        G[:, :6] = K1[:, :6] @ o["HTH"]
        vec = np.zeros(15)
        vec[:3] = so3_log(x[:9].reshape(3, 3).T @ x_prop[:9].reshape(3, 3)); vec[3:] = x_prop[9:21] - x[9:21]
        sol = K1[:, :6] @ o["HTz"] + vec - G[:, :6] @ vec[:6]
        x = x.copy(); x[:9] = (x[:9].reshape(3, 3) @ so3_exp(sol[:3])).ravel(); x[9:21] += sol[3:]
        if (np.linalg.norm(sol[:3]) * 57.3 < 0.01 and np.linalg.norm(sol[3:6]) * 100 < 0.015) or (rematch == 0 and it == 2):
            rematch += 1
        if rematch >= 2 or it == 3:
            cov = (np.eye(15) - G) @ cov
            break
    return dict(ok=bool(np.linalg.eigvalsh(o["nnt"])[0] >= 14), state=x, cov=cov, iters=it + 1, n=o["n"])


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        name, pl, clk = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=pl, max_sm_clock=clk)
    except Exception as e:          # noqa: BLE001
        import torch
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unknown ({e!r})")


def run(ctx, pts, W, L, scans, warm):
    mp = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    dm, f = vx.LocalMap(ctx, mp, W, max_points=100), vx.Factor(ctx, W)
    pv = np.zeros((pts, 12)); pv[:, [3, 7, 11]] = 1e-4
    xyz = np.empty((pts, 3))
    x_buf = []
    ta, tb, its, nm, dstate, dcov, agree = [], [], [], [], [], [], 0
    nscan = W + warm + scans
    for i in range(nscan):
        tr = synth.true_pose(L, i)
        synth.gen_scan(L, i, pts, tr, seed=0x5EED0000 + 9, out=xyz)
        pv[:, :3] = xyz
        est = tr
        if i >= W + warm:                                 # window full and warm: time the update of this scan
            st = np.zeros(24); st[:12] = synth.perturb_pose(tr, 91000 + i, 1e-3, 5e-3); st[12:15] = (0.3, -0.1, 0.05); st[21:24] = (0, 0, -9.8)
            ctx.var_init(xyz.astype(np.float32), np.eye(3), np.zeros(3), 0.02, 0.05, want_out=False)
            res = {}
            for which in (("a", "b") if i % 2 == 0 else ("b", "a")):
                t0 = time.perf_counter()
                res[which] = host_loop(dm, pts, st, COV) if which == "a" else dm.lio_update(None, st, COV, n=pts)
                (ta if which == "a" else tb).append((time.perf_counter() - t0) * 1e3)
            a, b = res["a"], res["b"]
            agree += int(a["iters"] == b["iters"] and a["n"] == b["n"] and a["ok"] == b["ok"])
            dstate.append(float(np.max(np.abs(a["state"] - b["state"])))); dcov.append(float(np.max(np.abs(a["cov"] - b["cov"])) / np.max(np.abs(b["cov"]))))
            its.append(b["iters"]); nm.append(b["n"] / pts)
            est = b["state"][:12]
        x_buf.append(est)
        dm.push_scan(pv, np.stack(x_buf), f)
        if len(x_buf) >= W:
            dm.margi(np.stack(x_buf), f, mgsize=1)
            x_buf = x_buf[1:]
    dm.close(); f.close()
    a, b = np.array(ta), np.array(tb)
    return {"points": pts, "scans": len(a), "ms_host_loop_mean": float(a.mean()), "ms_host_loop_median": float(np.median(a)),
            "ms_lio_update_mean": float(b.mean()), "ms_lio_update_median": float(np.median(b)), "speedup_median": float(np.median(a) / np.median(b)),
            "iters_hist": {str(k): int(np.sum(np.array(its) == k)) for k in (2, 3, 4)}, "matched_fraction": float(np.mean(nm)),
            "same_iters_n_ok": agree, "max_state_diff": max(dstate), "max_cov_rel_diff": max(dcov)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[20000, 1000000])
    ap.add_argument("--scans", type=int, default=50)
    ap.add_argument("--warm", type=int, default=4)
    ap.add_argument("--win", type=int, default=50)
    ap.add_argument("--L", type=float, default=130.0)
    args = ap.parse_args()
    ctx = vx.Context(0)
    out = {"probe": "lio_update", "what": "per scan, host wall clock: (a) host EKF loop around vxs_map_odom_accumulate passes, (b) one vxs_map_lio_update; "
                                          f"resident map of bench.py's local-mapping scene (W={args.win}, L={args.L}), window full and warm, (a) and (b) alternating",
           **card(), "results": [run(ctx, p, args.win, args.L, args.scans, args.warm) for p in args.points]}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
