"""Time the local consistency call (me_consistency) on one GPU, and split its device time.

For each scene: the whole Python call (median of --reps after a warm-up; host clock up to a synchronise) at region_size 0
and at --region-size, the C calls alone at
--region-size (begin / block / end, without the rows' conversion to numpy) and the region count, me_eval_mme's default sweep
and its ME_MME_WALK=1 sweep on the same cloud, then in separate torch.profiler runs the device time of the call by kernel
group (sweep, list, fold) and the host's share (the call's time less its device time).  Prints one JSON line per scene, with the card's name
and power limit read in the same run.

  python tools/consistency_time.py [--scenes c3,indoor,outdoor] [--reps 20]
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
    if name.startswith("me::consistency_walk") or "consistency_init" in name:
        return "sweep"
    if "consistency_fold" in name or "consistency_merge" in name:
        return "fold"
    return "list"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="c3,indoor,outdoor")
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--region-size", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    card = _card()
    for name in args.scenes.split(","):
        pts, r = _scene(name, args.n)
        row = {"scene": name, "n": len(pts), "radius": r, "card": card}
        with api.MapEvalB200() as ctx:
            ctx.set_cloud(EST, pts)

            def call(s):
                ctx.local_consistency(EST, r, 10, region_size=s)
                ctx.synchronize()

            def mme():
                ctx.computeMME(EST, r, 10)
                ctx.synchronize()

            row["mme_default_ms"] = _median_ms(mme, args.reps)
            os.environ["ME_MME_WALK"] = "1"
            row["mme_walk_ms"] = _median_ms(mme, args.reps)
            del os.environ["ME_MME_WALK"]
            row["call_ms"] = _median_ms(lambda: call(0.0), args.reps)
            row["call_regions_ms"] = _median_ms(lambda: call(args.region_size), args.reps)

            # the host's share at s > 0: the C call alone (begin, block, end), then the rows' conversion to numpy
            def c_call():
                n = ctx.consistency_begin(EST, r, 10, args.region_size)
                ctx.consistency_block()
                ctx.synchronize()
                return ctx.consistency_end(n)
            row["c_call_regions_ms"] = _median_ms(c_call, args.reps)
            row["n_regions"] = int(len(c_call()["index"]))
            w = ctx.local_consistency(EST, r, 10)["whole"]
            row.update(kernel=A.CONSISTENCY_KERNEL_NAMES[w["kernel"]], rings=w["rings"], solo=w["solo"], mme=w["mme"], mpv=w["mpv"])
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(args.region_size)
                torch.cuda.synchronize()
            split = {"sweep": 0.0, "list": 0.0, "fold": 0.0}
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
                if t > 0 and ev.key.startswith(("me::", "void me::")):
                    split[_group(ev.key.replace("void ", ""))] += t / 1e3
            row["device_ms_regions"] = split
            row["host_ms_regions"] = row["call_regions_ms"] - sum(split.values())
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(0.0)
                torch.cuda.synchronize()
            split0 = {"sweep": 0.0, "list": 0.0, "fold": 0.0}
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
                if t > 0 and ev.key.startswith(("me::", "void me::")):
                    split0[_group(ev.key.replace("void ", ""))] += t / 1e3
            row["device_ms"] = split0
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
