"""Time the Gaussian 2-Wasserstein stage (me_eval_w2) against the AWD stage (me_eval_awd) on C3 and C4, and measure how
both follow surface noise.

Timing: each call on a context whose stream is a torch stream, between CUDA events on that stream (both calls end with a
synchronise of the stream, so the events hold the whole call), median of --reps after a warm-up call.  Both stages run on
lattices already aligned with the voxel size.  Noise curve: a wavy surface with no thickness as the ground truth, and an
independent sample of the same surface with isotropic Gaussian noise sigma as the estimate; AWD (calculateVMD) beside AW2,
the mean offset and the mean shape term at v = 1 m.  Prints one JSON line per measurement, with the card's name and power
limit read in the same run.

  python tools/w2_time.py [--scenes C3,C4] [--reps 20] [--sigmas 0,0.005,0.01,0.02,0.05]
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


def _card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode()
    return out.strip().splitlines()[0]


def _timed(stream, fn, reps):
    import torch
    fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def _surface(n, extent, seed, sigma):
    rng = np.random.RandomState(seed)
    xy = rng.uniform(0, extent, (n, 2))
    z = 0.5 * np.sin(xy[:, 0] * 0.21) * np.cos(xy[:, 1] * 0.17)
    return np.ascontiguousarray(np.column_stack([xy, z]) + rng.normal(0, sigma, (n, 3)))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="C3,C4")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sigmas", default="0,0.005,0.01,0.02,0.05")
    args = ap.parse_args()
    card = _card()
    stream = torch.cuda.Stream()
    for name in args.scenes.split(","):
        est, gt, cfg = synth.make_pair(name)
        v = cfg["vmd_voxel_size"]
        with api.MapEvalB200(vmd_voxel_size=v) as ctx:
            ctx.set_stream(stream.cuda_stream)
            ctx.set_cloud(A.ME_CLOUD_EST, est)
            ctx.set_cloud(A.ME_CLOUD_GT, gt)
            awd = _timed(stream, lambda: ctx.calculateVMD(v, 100, 5), args.reps)
            w2 = _timed(stream, lambda: ctx.voxel_w2(v, 100, 5), args.reps)
            a, w = ctx.calculateVMD(v, 100, 5), ctx.voxel_w2(v, 100, 5)
            ctx.set_stream(None)
        print(json.dumps(dict(scene=name, card=card, voxel_size=v, n_est=len(est), n_gt=len(gt), n_pairs=w.n_pairs,
                              awd_ms=dict(zip(("median", "min", "max"), awd)), w2_ms=dict(zip(("median", "min", "max"), w2)),
                              awd=a.awd, aw2=w.aw2, mean_offset=w.mean_offset, mean_shape=w.mean_shape)), flush=True)
    v, n = 1.0, 2_000_000
    gt = _surface(n, 60.0, 1, 0.0)
    for s in (float(x) for x in args.sigmas.split(",")):
        est = _surface(n, 60.0, 2, s)
        with api.MapEvalB200(vmd_voxel_size=v) as ctx:
            ctx.set_cloud(A.ME_CLOUD_EST, est)
            ctx.set_cloud(A.ME_CLOUD_GT, gt)
            a = ctx.calculateVMD(v, 100, 5)
            w = ctx.voxel_w2(v, 100, 5)
        print(json.dumps(dict(curve="surface", card=card, voxel_size=v, sigma=s, n_pairs=w.n_pairs, awd=a.awd, aw2=w.aw2,
                              mean_offset=w.mean_offset, mean_shape=w.mean_shape, scs_w2=w.scs, scs_awd=a.scs)), flush=True)


if __name__ == "__main__":
    main()
