"""Time of the drift per region (me_drift*) on C3 (10 M est vs 10 M gt) at region sizes 3.0 m and 0.5 m, beside one
point-to-point ICP iteration of the whole cloud on the same clouds, with the card's name and power limit read in the same
run.  One JSON line.

Per configuration, after one warm-up loop: the median time of one iteration (me_drift_step / me_icp_step, host clock
around work that ends in a device synchronise), the whole loop's iteration count, and the median of the begin call.  Then,
in a separate run of the same loop whose steps (not its begin call) run under torch.profiler, the device time per iteration
of its parts, from the kernel records: the transform (drift_transform_kernel), the est re-layout (the lattice build
kernels), the sweep (the nn_ kernels) and the fold (record positions, fold, merge).  Every profiled step but the last moves,
sweeps and folds once, so the totals are divided by that count.  `host_ms` is the median iteration time minus those device
parts (the host update, the block read-back, the transform upload and the gaps between launches).

    python tools/region_drift_time.py [--scale 1.0] [--R 1.0]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cloud_map_evaluation_b200 import _abi as A  # noqa: E402
from cloud_map_evaluation_b200 import api, synth  # noqa: E402

FOLD = ("record_pos_kernel", "drift_fold_kernel", "drift_merge_kernel")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (x.strip() for x in out.stdout.splitlines()[0].split(","))
    return name, power


def drift_loop(ctx, s, R, around_steps=contextlib.nullcontext):
    """(begin ms, the iterations' ms, regions, rows); around_steps() is entered after the begin call, around the steps"""
    t0 = time.perf_counter()
    n = ctx.drift_begin(s, R)
    ctx.synchronize()
    begin = (time.perf_counter() - t0) * 1e3
    with around_steps():
        its = _steps(ctx)
    rows = ctx.drift_end(n)
    return begin, its, n, rows


def _steps(ctx):
    its = []
    done = False
    while not done:
        t0 = time.perf_counter()
        done = ctx.drift_step()
        ctx.synchronize()
        if not done:
            its.append((time.perf_counter() - t0) * 1e3)
    return its


def icp_loop(ctx, R):
    T0 = np.eye(4)
    T0[:3, 3] = (0.05, -0.03, 0.02)        # an initial offset, so that the loop makes more than one update
    ctx.icp_begin(R, T0, method=A.ME_ICP_POINT_TO_POINT)
    ctx.icp_block()
    ctx.synchronize()
    its = []
    done = False
    while not done:
        t0 = time.perf_counter()
        done = ctx.icp_step()
        ctx.synchronize()
        if not done:
            its.append((time.perf_counter() - t0) * 1e3)
    ctx.icp_end()
    return its


def classify(name):
    if name.startswith("drift_transform_kernel") or "drift_transform_kernel" in name:
        return "transform_ms"
    if any(k in name for k in FOLD):
        return "fold_ms"
    if "nn_" in name:
        return "sweep_ms"
    return "relayout_ms"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--R", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    name, power = card()
    est, gt, cfg = synth.make_pair("C3", scale=args.scale)
    out = {"config": "C3", "scale": args.scale, "n_est": len(est), "n_gt": len(gt), "R": args.R, "gpu": name, "power_limit": power}
    with api.MapEvalB200(device=0, vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        icp_loop(ctx, args.R)                                   # warm-up
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        its = icp_loop(ctx, args.R)
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        out["icp_p2p_iteration_ms"] = float(np.median(its))
        out["icp_iterations"] = len(its)
        for s in (3.0, 0.5):
            drift_loop(ctx, s, args.R)                          # warm-up
            begin, its, n, rows = drift_loop(ctx, s, args.R)
            r = {"regions": n, "iterations": len(its), "begin_ms": begin, "iteration_ms": float(np.median(its)),
                 "converged": int((rows["status"] == A.ME_DRIFT_CONVERGED).sum()),
                 "ratio_to_icp": float(np.median(its)) / out["icp_p2p_iteration_ms"]}
            prof = profile(activities=[ProfilerActivity.CUDA])
            _, its_p, _, _ = drift_loop(ctx, s, args.R, lambda: prof)
            parts = {"transform_ms": 0.0, "relayout_ms": 0.0, "sweep_ms": 0.0, "fold_ms": 0.0}
            for e in prof.key_averages():
                if e.device_type.name != "CUDA" or "Memcpy" in e.key or "Memset" in e.key:
                    continue
                parts[classify(e.key)] += e.device_time_total / 1e3
            k = max(len(its_p), 1)      # the profiled steps that moved, swept and folded
            for key in parts:
                r[key] = parts[key] / k
            r["host_ms"] = r["iteration_ms"] - sum(r[key] for key in parts)
            out[f"s={s}"] = r
        torch.cuda.synchronize()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
