"""Time of the exact distance quantiles (me_nn_quantile_*) after a C3 pass (10 M est vs 10 M gt, path A pairing), for K = 4 and
K = 64 probabilities under both populations: the whole call (MapEvalB200.distance_quantiles: 8 selection passes with a host
round trip each), median of --calls calls after one warm-up call, host clock around work that ends in a device synchronise.
Per pass: begin (pass 0: the keys and the top digit) and each step (the reduced counts read back, the next pass), each up to
a synchronise, medians over the same calls.  Beside it, in the same run: the curve call at K = 100
(me_nn_curve_accum_device), and the card's name and power limit.  One JSON line.

    python tools/distance_quantiles_time.py [--calls 20] [--scale 1.0]
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


def per_pass(ctx, probs, pop, calls):
    """median ms of begin and of each step, each up to a synchronise"""
    rows = []
    for _ in range(calls + 1):
        t = []
        t0 = time.perf_counter()
        ctx.quantile_begin(probs, pop)
        ctx.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
        done = False
        while not done:
            t0 = time.perf_counter()
            done = ctx.quantile_step()
            ctx.synchronize()
            t.append((time.perf_counter() - t0) * 1e3)
        ctx.quantile_end()
        rows.append(t)
    return [round(float(x), 4) for x in np.median(np.array(rows[1:]), axis=0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    name, power = card()
    est, gt, cfg = synth.make_pair("C3", scale=args.scale)
    p = A.make_nn_params(cfg["tau"], 1.0)
    out = dict(gpu=name, power_limit=power, n_est=len(est), n_gt=len(gt), calls=args.calls)
    rng = np.random.default_rng(0)
    probs = {4: np.array([0.5, 0.9, 0.95, 0.99]), 64: np.sort(rng.random(64))}
    with api.MapEvalB200(device=0, vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        ctx.set_cloud(A.ME_CLOUD_EST, est)
        ctx.set_cloud(A.ME_CLOUD_GT, gt)
        ctx.calculateMetricsWithInitialMatrix(p)
        out["curve_K100_ms_median"] = timed(lambda: ctx.curve_accum_device(np.linspace(0.0, 0.5, 101)[1:]), ctx.synchronize, args.calls)
        for pop, pname in ((A.ME_DIST_KEPT, "kept"), (A.ME_DIST_NN, "nn")):
            for K, pr in probs.items():
                out[f"{pname}_K{K}_ms_median"] = timed(lambda: ctx.distance_quantiles(pr, pop), ctx.synchronize, args.calls)
                out[f"{pname}_K{K}_pass_ms_median"] = per_pass(ctx, pr, pop, args.calls)
        r = ctx.distance_quantiles(probs[4], A.ME_DIST_NN)
        out["hausdorff"] = r["hausdorff"]
        out["n_nn"] = [r["est_to_gt"]["n"], r["gt_to_est"]["n"]]
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
