#!/usr/bin/env python
"""Device timeline of one full metric pass: per-kernel device time and the idle gaps between device activities.

    python tools/pass_timeline.py [--config C3] [--passes 3] [--warmup 3] [--out DIR]

Runs bench.py's device-resident pass (both clouds resident in HBM; MME of the estimated map, and of the ground truth when the
config says so, NN both ways with the default pairing and full CD, the voxel stage, one fetch of the accumulators) after
`--warmup` passes, `--passes` times under torch.profiler (CUDA activities).  Every kernel, memset and copy of the traced
passes is listed in stream order; a gap is the time from the end of one device activity to the start of the next, i.e. the
device idles while the host works (planning, launches) or waits on a synchronise.  Summed per pass:
  - per kernel name: calls, device time
  - the span of a pass (first device start to last device end), the busy time and the idle time
  - the largest gaps, with the activities on both sides
The host-side stage timers (profiler off) are printed beside them.  Prints the card name and its power limit; `--out DIR`
also writes everything as DIR/pass_timeline.json.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from cloud_map_evaluation_b200 import _abi as A, api, synth  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:      # noqa: BLE001
        plim = f"unavailable ({e})"
    return name, plim


def short(name):
    return name.split("(")[0].replace("void ", "").replace("me::", "").strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=sorted(synth.CONFIGS))
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--gaps", type=int, default=15, help="how many of the largest gaps to list")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pass_timeline.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    est, gt, cfg = synth.make_pair(args.config)
    d_est, d_gt = torch.from_numpy(est).to(dev), torch.from_numpy(gt).to(dev)
    n_est, n_gt = len(est), len(gt)
    p = A.make_nn_params(cfg["tau"], 1.0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    torch.cuda.synchronize()
    ctx = api.MapEvalB200(device=0, stream=stream.cuda_stream, vmd_voxel_size=cfg["vmd_voxel_size"] if cfg["awd"] else 0.0)

    def one_pass():     # bench.py's device-resident pass at one GPU
        ctx.set_cloud_device(A.ME_CLOUD_EST, d_est.data_ptr(), n_est, keepalive=d_est)
        ctx.set_cloud_device(A.ME_CLOUD_GT, d_gt.data_ptr(), n_gt, keepalive=d_gt)
        ctx.accum_reset()
        if cfg["mme"]:
            ctx.eval_mme_accum_device(A.ME_CLOUD_EST, cfg["nn_radius"], 10)
            if cfg["gt_mme"]:
                ctx.eval_mme_accum_device(A.ME_CLOUD_GT, cfg["nn_radius"], 5)
        ctx.eval_nn_accum_device(p)
        if cfg["awd"]:
            ctx.calculateVMD(cfg["vmd_voxel_size"], 100, 5)
        nn_e, nn_g, mmes = ctx.accum_fetch(want_mme=(bool(cfg["mme"]), bool(cfg["mme"] and cfg["gt_mme"])))
        ctx.nn_finalize(p, nn_e, nn_g)

    for _ in range(args.warmup):
        one_pass()
    # stage timers and the pass time with the profiler off
    stage = {}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record(stream)
    for _ in range(args.passes):
        one_pass()
        for k, v in ctx.stage_times_ms().items():
            stage[k] = stage.get(k, 0.0) + v / args.passes
    ev1.record(stream)
    torch.cuda.synchronize()
    pass_ms = ev0.elapsed_time(ev1) / args.passes
    launches0 = ctx.launch_count()
    one_pass()
    launches = ctx.launch_count() - launches0

    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.passes):
            one_pass()
            torch.cuda.synchronize()      # the passes do not overlap: every gap belongs to one pass
    acts = sorted(((ev.time_range.start, ev.time_range.end, short(ev.name)) for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA), key=lambda a: a[0])
    # split the trace into passes at the largest gaps (the host synchronises between traced passes)
    gaps = [(acts[i + 1][0] - acts[i][1], i) for i in range(len(acts) - 1)]
    cuts = sorted(i for _, i in sorted(gaps, reverse=True)[:args.passes - 1])
    passes, lo = [], 0
    for c in cuts + [len(acts) - 1]:
        passes.append(acts[lo:c + 1])
        lo = c + 1
    per_kernel, top = {}, []
    span = busy = 0.0
    for ps in passes:
        span += (ps[-1][1] - ps[0][0]) / args.passes
        end = ps[0][0]
        for j, (s, e, name) in enumerate(ps):
            r = per_kernel.setdefault(name, {"calls": 0.0, "us": 0.0})
            r["calls"] += 1.0 / args.passes
            r["us"] += (e - s) / args.passes
            busy += max(0.0, e - max(s, end)) / args.passes
            if j > 0 and s > end:
                top.append({"gap_us": s - end, "after": ps[j - 1][2], "before": name})
            end = max(end, e)
    # the largest gaps, averaged over the passes by (after, before) pair
    by_pair = {}
    for g in top:
        k = (g["after"], g["before"])
        r = by_pair.setdefault(k, {"after": k[0], "before": k[1], "count": 0.0, "us": 0.0})
        r["count"] += 1.0 / args.passes
        r["us"] += g["gap_us"] / args.passes
    gap_rows = sorted(by_pair.values(), key=lambda r: -r["us"])[:args.gaps]
    kern_rows = sorted(({"kernel": k, **v} for k, v in per_kernel.items()), key=lambda r: -r["us"])
    gpu, plim = card()

    print(f"card: {gpu}; power limit, max SM clock: {plim}")
    print(f"{args.config}: {n_est} est + {n_gt} gt points; {args.passes} passes after {args.warmup} warm-up passes")
    print(f"pass (CUDA events, profiler off): {pass_ms:.3f} ms, {launches} launches")
    print("stage timers (profiler off): " + ", ".join(f"{k} {v:.3f}" for k, v in stage.items()) +
          f"; sum {sum(stage.values()):.3f} ms")
    print(f"traced pass: span {span / 1e3:.3f} ms, device busy {busy / 1e3:.3f} ms, idle {(span - busy) / 1e3:.3f} ms")
    print(f"{'kernel / copy (per pass)':44s} {'calls':>6s} {'us':>9s}")
    for r in kern_rows:
        print(f"{r['kernel'][:44]:44s} {r['calls']:6.1f} {r['us']:9.1f}")
    print(f"largest idle gaps per pass (summed by neighbours):")
    print(f"{'after':36s} {'before':36s} {'count':>6s} {'us':>8s}")
    for r in gap_rows:
        print(f"{r['after'][:36]:36s} {r['before'][:36]:36s} {r['count']:6.1f} {r['us']:8.1f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pass_timeline.json"), "w") as f:
            json.dump({"gpu": gpu, "power_limit_max_sm_clock": plim, "config": args.config, "n_est": n_est, "n_gt": n_gt,
                       "passes": args.passes, "pass_ms": pass_ms, "launches": launches, "stage_ms": stage,
                       "span_us": span, "busy_us": busy, "idle_us": span - busy, "kernels": kern_rows, "gaps": gap_rows},
                      f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
