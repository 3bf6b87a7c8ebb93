"""Time of the point-to-plane metrics (me_nn_surface) after a C3 pass (10 M est vs 10 M gt, path A pairing, want_full_cd = 1):
the whole call (host clock around work that ends in a device synchronise), median of --calls calls after one warm-up call,
(b) with knn = 20 working normals on both clouds and (a) with given normals (estimated beforehand, knn = 0).  Then, in a
separate profiled run, the device time per call of the fold (surface_fold_kernel + surface_merge_kernel) beside the curve
call at K = 5 (nn_curve_kernel + nn_curve_merge_kernel) from the kernel records of torch.profiler.  The fold's byte model
is 100 B per query and direction (the records, and caller-order gathers of two points and two normals), reported against
a device-to-device copy of that many bytes (CUDA events, median of --calls copies).  With the card's name and power limit.
One JSON line.

    python tools/surface_metrics_time.py [--calls 20] [--scale 1.0]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cloud_map_evaluation_b200 import _abi as A  # noqa: E402
from cloud_map_evaluation_b200 import api, synth  # noqa: E402

FOLD = ("surface_fold_kernel", "surface_merge_kernel")
CURVE = ("nn_curve_kernel", "nn_curve_merge_kernel")
BYTES_PER_QUERY = 100


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (x.strip() for x in out.stdout.splitlines()[0].split(","))
    return name, power


def timed(fn, sync, calls):
    fn()
    sync()
    ms = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        sync()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms))


def copy_ms(nbytes, calls):
    """median of device-to-device copies of nbytes (CUDA events)"""
    import torch
    a = torch.empty(nbytes // 8, dtype=torch.float64, device="cuda:0")
    b = torch.empty_like(a)
    b.copy_(a)
    ms = []
    for _ in range(calls):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        b.copy_(a)
        e.record()
        e.synchronize()
        ms.append(s.elapsed_time(e))
    return float(np.median(ms))


def device_parts(ctx, calls, tau5):
    """device ms per call of the fold and of the curve at K = 5 (kernel records of torch.profiler)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ctx.surface_metrics()
            ctx.curve_accum_device(tau5)
            ctx.synchronize()
    fold = curve = 0.0
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total      # us over all calls
        if any(k in e.key for k in FOLD):
            fold += t
        elif any(k in e.key for k in CURVE):
            curve += t
    return round(fold / calls / 1e3, 4), round(curve / calls / 1e3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    name, power = card()
    est, gt, cfg = synth.make_pair("C3", scale=args.scale)
    p = A.make_nn_params(cfg["tau"], 1.0, want_full_cd=True)
    out = dict(gpu=name, power_limit=power, n_est=len(est), n_gt=len(gt), calls=args.calls)
    with api.MapEvalB200(device=0, vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        ctx.calculateMetricsWithInitialMatrix(p)
        out["working_knn20_ms_median"] = timed(lambda: ctx.surface_metrics(knn=20), ctx.synchronize, args.calls)
        ctx.estimate_normals(A.ME_CLOUD_EST, 20)
        ctx.estimate_normals(A.ME_CLOUD_GT, 20)
        out["given_ms_median"] = timed(lambda: ctx.surface_metrics(), ctx.synchronize, args.calls)
        out["fold_ms_device"], out["curve_K5_ms_device"] = device_parts(ctx, args.calls, sorted(cfg["tau"]))
    nbytes = BYTES_PER_QUERY * (len(est) + len(gt))
    out["model_bytes"] = nbytes
    out["copy_ms"] = round(copy_ms(nbytes, args.calls), 4)
    out["fold_GBps_model"] = round(nbytes / out["fold_ms_device"] / 1e6, 1) if out["fold_ms_device"] else None
    out["copy_GBps"] = round(nbytes / out["copy_ms"] / 1e6, 1)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
