"""Time of the accuracy curve (me_nn_curve_accum_device) after a C3 pass (10 M est vs 10 M gt, path A pairing), at K = 5,
100 and 1024 levels: CUDA events around the call on the context's stream, median of --calls calls after one warm-up call.
Beside it, in the same run: the five-level statistics pass it parallels (nn_stats_kernel and pair_as_written_kernel of one
me_eval_nn, from torch.profiler), a device-to-device copy of the bytes the curve reads (20 B per query and direction:
nn_idx, nn_d2, nn_sq), and the card's name and power limit.  One JSON line.

    python tools/accuracy_curve_time.py [--calls 20] [--scale 1.0]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cloud_map_evaluation_b200 import _abi as A  # noqa: E402
from cloud_map_evaluation_b200 import api, synth  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (x.strip() for x in out.stdout.splitlines()[0].split(","))
    return name, power


def timed(stream, fn, calls):
    import torch
    fn()
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    name, power = card()
    est, gt, cfg = synth.make_pair("C3", scale=args.scale)
    stream = torch.cuda.Stream()
    p = A.make_nn_params(cfg["tau"], 1.0)
    out = dict(gpu=name, power_limit=power, n_est=len(est), n_gt=len(gt), calls=args.calls)
    with api.MapEvalB200(device=0, stream=stream.cuda_stream, vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        ctx.calculateMetricsWithInitialMatrix(p)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                ctx.calculateMetricsWithInitialMatrix(p)
            torch.cuda.synchronize()
        for kern in ("nn_stats_kernel", "pair_as_written_kernel"):
            us = [e.device_time for e in prof.events() if kern in e.name and e.device_time > 0]
            out[kern + "_ms_median"] = float(np.median(us)) / 1000.0 if us else None
        for K in (5, 100, 1024):
            tau = np.linspace(0.0, 0.5, K + 1)[1:]
            out[f"curve_K{K}_ms_median"] = timed(stream, lambda: ctx.curve_accum_device(tau), args.calls)
    nbytes = 20 * (len(est) + len(gt))
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    dst = torch.empty_like(src)
    with torch.cuda.stream(stream):
        copy_ms = timed(stream, lambda: dst.copy_(src), args.calls)
    out.update(bytes_read=nbytes, d2d_copy_ms_median=copy_ms, d2d_copy_gbps=2 * nbytes / copy_ms / 1e6)
    for K in (5, 100, 1024):
        out[f"curve_K{K}_gbps_read"] = nbytes / out[f"curve_K{K}_ms_median"] / 1e6
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
