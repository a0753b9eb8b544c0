#!/usr/bin/env python
"""fp64 tensor-core rates of the four mma.sync shapes and k_syrk at the bench's metric shape, from one process, beside the card they
were measured on.  The SYRK is timed for every VXS_SYRK_WAVES value the default was chosen from (one context per value, since a context
reads the VXS_* switches when it is created).  Needs an H100:
    python tools/dmma_shapes.py [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (scene_points / ClockSampler: the bench's own metric-shape scene and clock sampling)
import voxel_slam_b200 as vx  # noqa: E402

WAVES = (4, 8, 12, 16, 24)
W, PTS, L, REPS = 50, 1000000, 130.0, 10


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power, clk = [x.strip() for x in r.stdout.strip().split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clk}


def syrk_ms(ctx, mp, p, off, est):
    """k_syrk milliseconds per Hessian build at the metric shape (CUDA events around every launch), and the factor's V, E."""
    f = vx.Factor(ctx, W)
    ctx.build_window_factor(mp, p, off, est, f)
    for _ in range(3):
        ctx.evaluate_hessian(f, est)
    ctx.timing(True); ctx.timing_reset()
    for _ in range(REPS):
        ctx.evaluate_hessian(f, est)
    st = ctx.timing_read(); ctx.timing(False)
    V, E, _ = f.counts()
    ms, calls = st["k_syrk"]
    return ms / REPS, calls / REPS, V, E


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", help="also write the result there")
    args = ap.parse_args()
    for k in [k for k in os.environ if k.startswith("VXS_SYRK_")]:
        del os.environ[k]
    out = card()
    sampler = bench.ClockSampler(0); sampler.start()
    ctx = vx.Context(0)
    out["dmma_tflops"] = ctx.dmma_shapes_tflops()
    out["clocks_during_shape_probe"] = sampler.stop()
    _, est, p, off = bench.scene_points(vx, W, PTS, L, seed=1)
    mp = vx.MapParams.make(voxel_size=1.0, min_eigen_value=0.0025, max_layer=2)
    rows = {}
    sampler = bench.ClockSampler(0); sampler.start()
    for w in WAVES:
        os.environ["VXS_SYRK_WAVES"] = str(w)
        c = vx.Context(0)
        ms, launches, V, E = syrk_ms(c, mp, p, off, est)
        c.close()
        kv = E / V
        flops = V * 108.0 * kv * kv / launches        # as bench.py's roofline counts them: 3 rank-1 rows x (6k)^2 / 2 MACs per voxel
        rows[w] = {"us_per_build": ms * 1e3, "launches": launches, "tflops": flops / (ms / launches * 1e-3) / 1e12}
        print(f"waves {w:3d}: k_syrk {ms * 1e3:8.1f} us per build, {rows[w]['tflops']:.1f} TFLOP/s", file=sys.stderr, flush=True)
    del os.environ["VXS_SYRK_WAVES"]
    out["clocks_during_syrk"] = sampler.stop()
    out["syrk_metric_shape"] = {"W": W, "V": V, "E": E, "by_waves": rows}
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)
    ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
