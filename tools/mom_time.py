"""Time the mutually orthogonal metric (me_mom) on one GPU beside the local consistency call, and split its device time.

For each scene: the whole Python call (median of --reps after a warm-up; host clock up to a synchronise), the consistency
call on the same cloud (the same walk without the histogram, the families and the selection), then in a separate
torch.profiler run the device time of the MOM call by kernel group (sweep, histogram to block, fold and keys, selection) and
the host's share.  Prints one JSON line per scene, with the card's name and power limit read in the same run.

  python tools/mom_time.py [--scenes c3,indoor,outdoor] [--reps 20]
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

EST = A.ME_CLOUD_EST


def _card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode()
    return out.strip().splitlines()[0]


def _scene(name, n):
    if name == "c3":
        est, _, cfg = synth.make_pair("C3")
        return est, cfg["nn_radius"]
    if name == "indoor":
        return synth.indoor_scene(n, 1, 0.002).astype(np.float64), 0.1
    return synth.outdoor_scene(n, 2, 0.02).astype(np.float64), 1.0


def _median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def _group(name):
    if "mom_sweep" in name or "mom_init" in name:
        return "sweep"
    if "mom_to_block" in name:
        return "histogram"
    if "mom_fold" in name or "mom_merge" in name or "mom_keys" in name:
        return "families"
    if "nn_quantile_hist" in name:
        return "selection"
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="c3,indoor,outdoor")
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    card = _card()
    for name in args.scenes.split(","):
        pts, r = _scene(name, args.n)
        row = {"scene": name, "n": len(pts), "radius": r, "card": card}
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(EST, pts)

            def mom():
                ctx.mom(EST, r, 10)
                ctx.synchronize()

            def cons():
                ctx.local_consistency(EST, r, 10)
                ctx.synchronize()

            row["consistency_ms"] = _median_ms(cons, args.reps)
            row["mom_ms"] = _median_ms(mom, args.reps)
            res = ctx.mom(EST, r, 10)
            row.update(status=res["status"], mom=res["mom"], n_planar=res["n_planar"], n_family=[int(x) for x in res["n"]],
                       rings=res["rings"], solo=res["solo"])
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                mom()
                torch.cuda.synchronize()
            split = {"sweep": 0.0, "histogram": 0.0, "families": 0.0, "selection": 0.0, "other": 0.0}
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
                if t > 0 and ev.key.startswith(("me::", "void me::")):
                    split[_group(ev.key)] += t / 1e3
            row["device_ms"] = split
            row["host_ms"] = row["mom_ms"] - sum(split.values())
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
