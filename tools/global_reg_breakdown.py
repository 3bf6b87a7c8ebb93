"""Stage times of me_global_registration on the H100, from the CUDA events the call records (me_global_reg_result.stage_ms):
copy + down-sample, normals (lattice, k-NN normals, orientation), FPFH, matching, RANSAC, refinement — each summed over both
clouds where it runs per cloud.  Indoor and outdoor generators at 10 M points per cloud (the estimate turned by 60° and
moved), feature voxels of 0.25 and 0.5 m; the median of --calls timed calls after one warm-up call.  The card's name and
power limit are read in the same run.  One JSON line per case.

    python tools/global_reg_breakdown.py [--points 10000000] [--calls 10] [--hypotheses 100000]
"""
import argparse
import json
import math
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--hypotheses", type=int, default=100_000)
    args = ap.parse_args()
    name, power = card()
    yaw = math.radians(60.0)
    M = np.array([[math.cos(yaw), -math.sin(yaw), 0, 40.0], [math.sin(yaw), math.cos(yaw), 0, -25.0], [0, 0, 1, 1.5], [0, 0, 0, 1]])
    gens = {"indoor": lambda n, s, z: synth.indoor_scene(n, s, z), "outdoor": lambda n, s, z: synth.outdoor_scene(n, s, z)}
    for scene, gen in gens.items():
        gt = gen(args.points, synth.GT_SEED, 0.002)
        est = gen(args.points, synth.EST_SEED, 0.01) @ M[:3, :3].T + M[:3, 3]
        for vox in (0.25, 0.5):
            with api.MapEvalB200(device=0) as ctx:
                ctx.set_cloud(A.ME_CLOUD_EST, est)
                ctx.set_cloud(A.ME_CLOUD_GT, gt)
                ctx.global_registration(vox, seed=1, n_hypotheses=args.hypotheses)          # warm-up
                runs = [ctx.global_registration(vox, seed=1, n_hypotheses=args.hypotheses) for _ in range(args.calls)]
            med = {k: float(np.median([r["stage_ms"][k] for r in runs])) for k in A.GLOBAL_REG_STAGES}
            r = runs[-1]
            print(json.dumps(dict(scene=scene, points=args.points, feature_voxel=vox, calls=args.calls, gpu=name, power_limit=power,
                                  stage_ms_median=med, total_ms_median=sum(med.values()), n_est_features=r["n_est_features"],
                                  n_gt_features=r["n_gt_features"], n_correspondences=r["n_correspondences"],
                                  n_inliers=r["n_inliers"])), flush=True)


if __name__ == "__main__":
    main()
