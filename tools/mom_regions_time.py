"""Time the mutually orthogonal metric per region (me_mom_regions) on one GPU beside the MOM call it follows, and split its
device time.

For each scene and region size: the MOM call and the region call (median of --reps after a warm-up; host clock up to a
synchronise), the region count and how many rows are OK, then in a separate torch.profiler run the region call's device time
by kernel group (list: the occupied list and the region ids; fill; keys; sorts; selection: the medians and the chunk fold)
and the host's share.  Prints one JSON line per scene and size, with the card's name and power limit read in the same run.

  python tools/mom_regions_time.py [--scenes c3,indoor,outdoor] [--sizes 1,3] [--reps 20]
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
    if "region_key" in name or "region_head" in name or "region_list" in name or "region_count" in name or "region_rid" in name \
            or "bbox" in name:
        return "list"
    if "mom_region_fill" in name:
        return "fill"
    if "mom_region_keys" in name or "mom_region_segkey" in name:
        return "keys"
    if "rs_hist" in name or "rs_scatter" in name:
        return "sorts"
    if "mom_region_select" in name or "mom_region_fold" in name or "mom_region_merge" in name:
        return "selection"
    if "scan" in name:
        return "scans"
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="c3,indoor,outdoor")
    ap.add_argument("--sizes", default="1,3")
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    card = _card()
    for name in args.scenes.split(","):
        pts, r = _scene(name, args.n)
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(EST, pts)

            def mom():
                ctx.mom(EST, r, 10)
                ctx.synchronize()

            mom_ms = _median_ms(mom, args.reps)
            res = ctx.mom(EST, r, 10)
            for s in (float(x) for x in args.sizes.split(",")):
                row = {"scene": name, "n": len(pts), "radius": r, "region_size": s, "card": card, "mom_ms": mom_ms,
                       "status": res["status"], "n_family": [int(x) for x in res["n"]]}

                def regions():
                    out = ctx.mom_regions(s)
                    ctx.synchronize()
                    return out

                row["regions_ms"] = _median_ms(regions, args.reps)
                rows = regions()
                row.update(n_regions=len(rows["index"]), n_ok=int((rows["status"] == "OK").sum()))
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    regions()
                    torch.cuda.synchronize()
                split = {"list": 0.0, "fill": 0.0, "keys": 0.0, "sorts": 0.0, "scans": 0.0, "selection": 0.0, "other": 0.0}
                for ev in prof.key_averages():
                    t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
                    if t > 0:
                        split[_group(ev.key)] += t / 1e3
                row["device_ms"] = split
                row["host_ms"] = row["regions_ms"] - sum(split.values())
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
