#!/usr/bin/env python
"""Time of the registration stage (generalized ICP, registration_methods: 2) on one GPU, and the per-rank share of a
sharded registration.

    python tools/icp_breakdown.py [--pairs C3:1.0,C5:0.05] [--max-dist 1.0] [--reps 7] [--out DIR]

Per pair (a BASELINE config at a scale; C5 at 0.05 is a 10 M vs 10 M grid of rooms):
1. me_icp(GENERALIZED) and the same registration through the split API at world = 1 (me_icp_begin .. me_icp_end),
   alternated --reps times in one process (medians and the min / max of the totals are printed): total time, the k-NN
   normals of both clouds, iterations, time per iteration
   ((total - normals) / (iterations + 1): every iteration and the initial pass lay the moved cloud out and sweep it).
   Host clocks around calls that end in a device synchronise.
2. One rank at a time on the same device at world 2 and 8: its slice of the normals of both clouds, and one iteration of
   its sweep (me_icp_step on its own block; the gathered normals are filled in from the world = 1 estimate, so that the
   sweep reads real normals).  The slowest rank bounds a sharded iteration; the collectives are not included.
Wall time of a multi-GPU registration is not measured here.  Prints the card name and power limit with the numbers;
--out DIR also writes them to DIR/icp_breakdown.json.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from cloud_map_evaluation_b200 import _abi as A, api, synth_torch  # noqa: E402
from cloud_map_evaluation_b200 import dist as mdist  # noqa: E402

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
GICP = A.ME_ICP_GENERALIZED


def card():
    name = torch.cuda.get_device_name(0)
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:      # noqa: BLE001
        plim = f"unavailable ({e})"
    return name, plim


def _ctx(est, gt, rank=0, world=1):
    c = api.MapEvalB200(rank=rank, world=world)
    c.set_cloud(EST, est)
    c.set_cloud(GT, gt)
    c.synchronize()
    return c


def time_me_icp(est, gt, R):
    with _ctx(est, gt) as c:
        t0 = time.perf_counter()
        for w in (EST, GT):              # the estimate me_icp makes (lattices included), timed on its own; no read-back
            c._check(c._L.me_estimate_normals(c._ctx, w, 20))
        c.synchronize()
        t_n = time.perf_counter() - t0
    with _ctx(est, gt) as c:
        t0 = time.perf_counter()
        T, reg = c.performICPRegistration(R, method=GICP)
        t = time.perf_counter() - t0
    return dict(total_ms=1e3 * t, normals_ms=1e3 * t_n, iterations=reg.iterations, n_corr=reg.n_corr,
                per_iteration_ms=1e3 * (t - t_n) / (reg.iterations + 1)), T


def time_split(est, gt, R):
    with _ctx(est, gt) as c:
        t0 = time.perf_counter()
        c.icp_begin(R, method=GICP)
        c.icp_normals_slice(EST)
        c.icp_normals_slice(GT)
        c.synchronize()
        t_n = time.perf_counter() - t0
        c.icp_block()
        while not c.icp_step():
            pass
        T, reg = c.icp_end()
        t = time.perf_counter() - t0
    return dict(total_ms=1e3 * t, normals_ms=1e3 * t_n, iterations=reg.iterations, n_corr=reg.n_corr,
                per_iteration_ms=1e3 * (t - t_n) / (reg.iterations + 1)), T


def rank_share(est, gt, R, world, normals_w1, steps=3):
    """per rank: its normal slices of both clouds, and the mean time of `steps` iterations of its own sweep"""
    out = []
    for r in range(world):
        with _ctx(est, gt, r, world) as c:
            c.icp_begin(R, method=GICP)
            t0 = time.perf_counter()
            sl = [c.icp_normals_slice(w) for w in (EST, GT)]
            c.synchronize()
            t_n = time.perf_counter() - t0
            for (ptr, s, _), w in zip(sl, (EST, GT)):
                n = len(normals_w1[w])
                buf = torch.as_tensor(mdist._DeviceBlock(ptr, world * s * 3), device="cuda:0")
                mine = buf[3 * r * s:3 * min((r + 1) * s, n)].cpu().numpy()
                assert mine.tobytes() == normals_w1[w][r * s:(r + 1) * s].tobytes(), "slice differs from world = 1"
                buf[:3 * n].copy_(torch.from_numpy(normals_w1[w].reshape(-1)))
            torch.cuda.synchronize()
            c.icp_block()
            c.synchronize()
            t0 = time.perf_counter()
            k = 0
            for k in range(steps):
                if c.icp_step():
                    break
            c.synchronize()
            t_it = (time.perf_counter() - t0) / (k + 1)
            c.icp_end()
        out.append(dict(rank=r, normals_ms=1e3 * t_n, iteration_ms=1e3 * t_it))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="C3:1.0,C5:0.05")
    ap.add_argument("--max-dist", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--worlds", default="2,8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("icp_breakdown: no CUDA device")
    name, plim = card()
    res = {"device": name, "power_limit,max_sm_clock": plim, "max_dist": a.max_dist, "pairs": {}}
    print(f"# {name}  power.limit, clocks.max.sm = {plim}", flush=True)
    for spec in a.pairs.split(","):
        cfg, scale = spec.split(":")
        est_t, gt_t, _ = synth_torch.make_pair(cfg, float(scale), device="cuda")
        est, gt = est_t.cpu().numpy(), gt_t.cpu().numpy()
        del est_t, gt_t
        torch.cuda.empty_cache()
        key = f"{cfg}@{scale} ({len(est)} vs {len(gt)})"
        time_me_icp(est, gt, a.max_dist)                      # warm-up: module load, allocations
        runs = {"me_icp": [], "split_world1": []}
        Ts = {}
        for _ in range(a.reps):
            r1, Ts["me_icp"] = time_me_icp(est, gt, a.max_dist)
            r2, Ts["split"] = time_split(est, gt, a.max_dist)
            runs["me_icp"].append(r1)
            runs["split_world1"].append(r2)
            print(key, "me_icp", json.dumps(r1), flush=True)
            print(key, "split ", json.dumps(r2), flush=True)
        med = {k: {f: float(np.median([r[f] for r in v])) for f in ("total_ms", "normals_ms", "per_iteration_ms")}
               for k, v in runs.items()}
        spread = {k: [float(min(r["total_ms"] for r in v)), float(max(r["total_ms"] for r in v))] for k, v in runs.items()}
        print(key, "median", json.dumps(med), "total_ms min/max", json.dumps(spread), flush=True)
        entry = dict(runs=runs, median=med, total_ms_min_max=spread, T_max_abs_diff=float(np.abs(Ts["me_icp"] - Ts["split"]).max()))
        with _ctx(est, gt) as c:
            normals_w1 = {EST: c.estimate_normals(EST, 20), GT: c.estimate_normals(GT, 20)}
        for w in [int(x) for x in a.worlds.split(",")]:
            entry[f"world{w}"] = rank_share(est, gt, a.max_dist, w, normals_w1)
            for r in entry[f"world{w}"]:
                print(key, f"world {w}", json.dumps(r), flush=True)
        entry["multi_gpu_wall_time"] = "not measured (one GPU)"
        res["pairs"][key] = entry
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "icp_breakdown.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
