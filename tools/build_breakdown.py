#!/usr/bin/env python
"""Per-kernel breakdown of the two dense lattice builds of one pass, against the copy ceiling of the card.

    python tools/build_breakdown.py [--config C3] [--passes 5] [--out DIR]

1. Full passes as bench.py's device-resident arm runs them (MME of the estimated map, NN both ways, voxel stage), with
   both clouds resident in HBM: the stage timers give `grid_est` / `grid_gt`.
2. In a run of its own under torch.profiler (CUDA activities): `--passes` times, both clouds handed over again and both
   lattices built (estimated map first, as in a pass).  Every kernel, memset and copy of those builds, summed over the two
   builds of one pass: time, the bytes the step has to move (a model computed from the point and cell counts, below) and
   the achieved GB/s.  The estimated map's bounding box is part of its build here; in a pass it runs ahead of the timer.
3. A 320 MB device-to-device cudaMemcpyAsync timed with CUDA events: what a plain stream of reads and writes achieves on
   this card at its power limit (its GB/s counts the bytes read plus the bytes written).

Prints the card name and its power limit with the numbers; `--out DIR` also writes them as DIR/build_breakdown.json.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from cloud_map_evaluation_b200 import _abi as A, _lib, api, synth  # noqa: E402

# HBM bytes one step moves per cloud of n points on a dense table of `cells` cells (4 B each).  A per-point u32 (the
# cell id, or the in-cell rank) is written by the histogram and read by the scatter.  Random 32-byte record writes are
# counted once; the random reads of the count table, and partly written sectors, are left out.
BYTES = {
    "bbox_kernel": lambda n, cells: 24 * n,
    "cell_count_kernel": lambda n, cells: 24 * n + 4 * n,
    "occupancy_kernel": lambda n, cells: 4 * cells,
    "scan_tile_sum_kernel": lambda n, cells: 4 * cells,
    "scan_apply_kernel": lambda n, cells: 8 * cells,
    "scan_kernel": lambda n, cells: 8 * cells,
    "scatter_kernel": lambda n, cells: 4 * n + 24 * n + 32 * n,
    "rel_kernel": lambda n, cells: 32 * n + 16 * n,
    "Memset": lambda n, cells: 4 * cells,                          # the count table; the other memsets are a few bytes
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:      # noqa: BLE001
        plim = f"unavailable ({e})"
    return name, plim


def copy_ceiling(stream, mb=320, reps=20):
    src = torch.empty(mb * 1000 * 1000, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    src.fill_(1)
    with torch.cuda.stream(stream):
        for _ in range(3):
            dst.copy_(src)
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            dst.copy_(src)
            e1.record(stream)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
    t = float(np.median(ms))
    return {"bytes_copied": src.numel(), "ms_median": t, "ms_min": float(min(ms)), "reps": reps,
            "gbs_read_plus_write": 2 * src.numel() / (t * 1e-3) / 1e9}


def lattice_cells(d, cfg, n, other, n_other):
    """The dense table the planning step gives the pair (me_plan_lattice on the measured bounding boxes)."""
    L = _lib.load()
    dp = C.POINTER(C.c_double)
    lo, hi = d.min(0).values.tolist(), d.max(0).values.tolist()
    olo, ohi = other.min(0).values.tolist(), other.max(0).values.tolist()
    arr = lambda v: C.cast((C.c_double * 3)(*v), dp)      # noqa: E731
    out = A.me_lattice_plan()
    rc = L.me_plan_lattice(arr(lo), arr(hi), n, arr(olo), arr(ohi), n_other, cfg["vmd_voxel_size"] if cfg["awd"] else 0.0,
                           0.0, 0, 1, C.byref(out))
    if rc != 0 or out.sparse:
        raise SystemExit("build_breakdown: the config does not get a dense cell table")
    return int(out.ncells), list(out.dims)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=sorted(synth.CONFIGS))
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("build_breakdown.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    est, gt, cfg = synth.make_pair(args.config)
    d_est, d_gt = torch.from_numpy(est).to(dev), torch.from_numpy(gt).to(dev)
    n_est, n_gt = len(est), len(gt)
    p = A.make_nn_params(cfg["tau"], 1.0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    torch.cuda.synchronize()
    ctx = api.MapEvalB200(device=0, stream=stream.cuda_stream, vmd_voxel_size=cfg["vmd_voxel_size"] if cfg["awd"] else 0.0)

    def hand_over():
        ctx.set_cloud_device(A.ME_CLOUD_EST, d_est.data_ptr(), n_est, keepalive=d_est)
        ctx.set_cloud_device(A.ME_CLOUD_GT, d_gt.data_ptr(), n_gt, keepalive=d_gt)

    def full_pass():
        hand_over()
        ctx.accum_reset()
        if cfg["mme"]:
            ctx.eval_mme_accum_device(A.ME_CLOUD_EST, cfg["nn_radius"], 10)
            if cfg["gt_mme"]:
                ctx.eval_mme_accum_device(A.ME_CLOUD_GT, cfg["nn_radius"], 5)
        ctx.eval_nn_accum_device(p)
        if cfg["awd"]:
            ctx.calculateVMD(cfg["vmd_voxel_size"], 100, 5)

    # 1. stage times of full passes (profiler off)
    for _ in range(3):
        full_pass()
    stage = {}
    for _ in range(args.passes):
        full_pass()
        for k, v in ctx.stage_times_ms().items():
            stage[k] = stage.get(k, 0.0) + v / args.passes
    torch.cuda.synchronize()

    # 2. the builds alone, traced
    def builds():
        hand_over()
        ctx.build_grid(A.ME_CLOUD_EST)
        ctx.build_grid(A.ME_CLOUD_GT)

    for _ in range(2):
        builds()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.passes):
            builds()
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name.split("(")[0].split("<")[0].replace("me::", "").replace("void ", "").strip()
        r = rows.setdefault(name, {"us": 0.0, "calls": 0, "first": ev.time_range.start})
        r["us"] += ev.time_range.elapsed_us() / args.passes
        r["calls"] += 1
        r["first"] = min(r["first"], ev.time_range.start)
    cells_est, dims = lattice_cells(d_est, cfg, n_est, d_gt, n_gt)
    cells_gt, _ = lattice_cells(d_gt, cfg, n_gt, d_est, n_est)
    ceiling = copy_ceiling(stream)
    gpu, plim = card()

    out_rows = []
    total_us = total_bytes = 0.0
    for name, r in sorted(rows.items(), key=lambda kv: kv[1]["first"]):
        key = "Memset" if name.startswith("Memset") else name
        nb = None
        if key in BYTES:
            nb = BYTES[key](n_est, cells_est) + BYTES[key](n_gt, cells_gt)
        gbs = nb / (r["us"] * 1e-6) / 1e9 if nb and r["us"] > 0 else None
        total_us += r["us"]
        total_bytes += nb or 0
        out_rows.append({"step": name, "calls_per_pass": r["calls"] / args.passes, "us": r["us"], "bytes": nb, "gbs": gbs,
                         "of_ceiling": gbs / ceiling["gbs_read_plus_write"] if gbs else None})

    print(f"card: {gpu}; power limit, max SM clock: {plim}")
    print(f"{args.config}: {n_est} est + {n_gt} gt points, dense table {dims[0]} x {dims[1]} x {dims[2]} = {cells_est} cells "
          f"(est), {cells_gt} (gt); {args.passes} traced passes")
    print(f"stage timers of full passes (profiler off): grid_est {stage['grid_est']:.3f} ms, grid_gt {stage['grid_gt']:.3f} ms")
    print(f"copy ceiling: {ceiling['bytes_copied'] / 1e6:.0f} MB device-to-device in {ceiling['ms_median']:.3f} ms "
          f"= {ceiling['gbs_read_plus_write']:.0f} GB/s (read + write)")
    print(f"{'step (both builds of a pass)':34s} {'calls':>6s} {'us':>9s} {'MB':>9s} {'GB/s':>7s} {'of copy':>8s}")
    for r in out_rows:
        mb = f"{r['bytes'] / 1e6:9.0f}" if r["bytes"] else f"{'-':>9s}"
        gbs = f"{r['gbs']:7.0f}" if r["gbs"] else f"{'-':>7s}"
        frac = f"{100 * r['of_ceiling']:7.0f}%" if r["of_ceiling"] else f"{'-':>8s}"
        print(f"{r['step'][:34]:34s} {r['calls_per_pass']:6.1f} {r['us']:9.1f} {mb} {gbs} {frac}")
    print(f"{'sum of device time':34s} {'':6s} {total_us:9.1f} {total_bytes / 1e6:9.0f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "build_breakdown.json"), "w") as f:
            json.dump({"gpu": gpu, "power_limit_max_sm_clock": plim, "config": args.config, "n_est": n_est, "n_gt": n_gt,
                       "cells": [cells_est, cells_gt], "dims": dims, "passes": args.passes, "stage_ms": stage,
                       "copy_ceiling": ceiling, "rows": out_rows, "sum_us": total_us, "sum_bytes": total_bytes}, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
