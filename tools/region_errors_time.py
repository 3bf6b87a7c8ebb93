"""Time of the per-region table (me_nn_regions) after a C3 pass (10 M est vs 10 M gt, path A pairing) at region sizes 3.0 m
and 0.5 m: the whole call (host clock around work that ends in a device synchronise), median of --calls calls after one
warm-up call, and of its device half alone (me_nn_region_begin up to a synchronise: the rest of the call is the host's
finalize and the conversion to numpy); then, in a separate profiled run of the same calls, the device time of its two
parts from the kernel records of torch.profiler: the key / occupied-list part (keys, radix sort, heads, scan, list, counts)
and the record-fold part (record positions, fold, merge).  Beside it, in the same run: the curve call at K = 100 (me_nn_curve_accum_device), and the
card's name and power limit.  One JSON line.

    python tools/region_errors_time.py [--calls 20] [--scale 1.0]
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

FOLD_KERNELS = ("record_pos_kernel", "region_fold_kernel", "region_merge_kernel")


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


def parts(ctx, s, calls):
    """median per call of the device time of the list part and of the fold part (kernel records of torch.profiler)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ctx.region_errors(s)
            ctx.synchronize()
    fold = lst = 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total      # us over all calls
        if e.device_type != torch.autograd.DeviceType.CUDA or "Memcpy" in e.key or "Memset" in e.key:
            continue
        if any(k in e.key for k in FOLD_KERNELS):
            fold += t
        else:
            lst += t
    return round(lst / calls / 1e3, 4), round(fold / calls / 1e3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    name, power = card()
    est, gt, cfg = synth.make_pair("C3", scale=args.scale)
    p = A.make_nn_params(cfg["tau"], 1.0)
    out = dict(gpu=name, power_limit=power, n_est=len(est), n_gt=len(gt), calls=args.calls)
    with api.MapEvalB200(device=0, vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        ctx.calculateMetricsWithInitialMatrix(p)
        out["curve_K100_ms_median"] = timed(lambda: ctx.curve_accum_device(np.linspace(0.0, 0.5, 101)[1:]), ctx.synchronize, args.calls)
        for s in (3.0, 0.5):
            key = f"s{s:g}"
            out[f"{key}_ms_median"] = timed(lambda: ctx.region_errors(s), ctx.synchronize, args.calls)
            out[f"{key}_begin_ms_median"] = timed(lambda: ctx.region_begin(s), ctx.synchronize, args.calls)
            out[f"{key}_regions"] = int(len(ctx.region_errors(s)["n_est"]))
        for s in (3.0, 0.5):
            out[f"s{s:g}_list_ms_device"], out[f"s{s:g}_fold_ms_device"] = parts(ctx, s, args.calls)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
