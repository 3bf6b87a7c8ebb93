#!/usr/bin/env python
"""The simulation operators of `evaluate_noised_gt` on one GPU: their time against a copy of the same bytes, and the
metric curves of the paper's two simulation figures (Noise Sensitivity, Outlier Robustness).

    python tools/degradation_sweep.py [--reps 10] [--skip-c5] [--skip-curves] [--out DIR]

1. Timing.  Each operator on a fresh library-owned copy of (a) C3's 10 M-point ground truth and (b) a 200 M-point C5
   indoor cloud generated on the device (synth_torch), timed with CUDA events after a warm-up (median of --reps), set
   against a timed device-to-device copy of the cloud's 24 N bytes.  Modelled HBM bytes per point:
     noise        48                                       (read and write xyz)
     deformation  24 + 24 x share inside the radius
     density      24 (flag) + 8 (scan) + 24 x keep share   (no normals here; with normals + 48 x keep share)
     outliers     48 (the copy into a grown buffer) + 48 per outlier
2. Metric curves on C2 (1 M points, full pass: NN both ways with the strict cut-off and geometric pairing of
   calculateMetrics, full Chamfer distance, MME of both clouds, AWD / SCS): the estimate is the ground truth with
   Gaussian noise sigma in {0, 0.005, 0.01, 0.02, 0.05, 0.1} m, then with sparse outliers (range 0.5 m) at ratio in
   {0, 0.01, 0.05, 0.1, 0.2}.  One JSON line per level.

Prints the card name and its power limit with both parts; `--out DIR` also writes DIR/degradation_sweep.json.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from cloud_map_evaluation_b200 import _abi as A, api, synth, synth_torch  # noqa: E402

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
SEED = synth.EST_SEED


def card():
    name = torch.cuda.get_device_name(0)
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:      # noqa: BLE001
        plim = f"unavailable ({e})"
    return name, plim


def timed(stream, fn, reps, prepare=None):
    """median / min ms of fn() on `stream` (prepare() runs before each rep, outside the timed span)"""
    ms = []
    for r in range(reps + 2):
        if prepare:
            prepare()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        if r >= 2:                      # two warm-up reps
            ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), float(min(ms))


def time_operators(name, d_gt, centre, radius, reps, stream):
    n = d_gt.shape[0]
    ctx = api.MapEvalB200(device=0, stream=stream.cuda_stream)
    ctx.set_cloud_device(GT, d_gt.data_ptr(), n, keepalive=d_gt)

    def fresh():
        # borrowing first releases the estimate's buffer, so the copy gets one of exactly N points (as in map_eval)
        ctx.set_cloud_device(EST, d_gt.data_ptr(), n, keepalive=d_gt)
        ctx.copy_cloud(GT, EST)

    fresh()
    ctx.add_non_uniform_density(EST, 0.3, 0.8, 1.0, SEED)
    keep = ctx.n[EST] / n
    d = torch.linalg.vector_norm(d_gt - torch.tensor(centre, dtype=torch.float64, device=d_gt.device), dim=1)
    inside = float((d < radius).double().mean())
    del d
    m = int(n * 0.05)
    copy_bytes = 24 * n
    dst = torch.empty_like(d_gt)
    cm, cmin = timed(stream, lambda: dst.copy_(d_gt), reps)
    del dst
    copy_gbs = 2 * copy_bytes / (cm * 1e-3) / 1e9
    ops = {
        "noise": (lambda: ctx.add_gaussian_noise(EST, 0.01, SEED), 48 * n),
        "deformation": (lambda: ctx.add_local_deformation(EST, radius, 0.1, centre), (24 + 24 * inside) * n),
        "density": (lambda: ctx.add_non_uniform_density(EST, 0.3, 0.8, 1.0, SEED), (24 + 8 + 24 * keep) * n),
        "outliers": (lambda: ctx.add_sparse_outliers(EST, 0.05, 0.5, SEED), 48 * n + 48 * m),
    }
    rows = []
    for op, (fn, nbytes) in ops.items():
        med, mn = timed(stream, fn, reps, prepare=fresh)
        gbs = nbytes / (med * 1e-3) / 1e9
        rows.append({"cloud": name, "n": n, "op": op, "ms_median": med, "ms_min": mn, "bytes": nbytes, "gbs": gbs,
                     "of_copy": gbs / copy_gbs})
    ctx.close()
    return {"cloud": name, "n": n, "share_inside": inside, "keep_share": keep, "outliers": m,
            "copy": {"bytes": copy_bytes, "ms_median": cm, "ms_min": cmin, "gbs_read_plus_write": copy_gbs}, "rows": rows}


def curves(stream):
    est, gt, cfg = synth.make_pair("C2")
    d_gt = torch.from_numpy(gt).cuda()
    p = A.make_nn_params(cfg["tau"], 1.0, cutoff_mode=A.ME_CUTOFF_DIST_LT_R, pairing=A.ME_PAIRING_GEOMETRIC)
    out = []
    with api.MapEvalB200(device=0, stream=stream.cuda_stream, vmd_voxel_size=cfg["vmd_voxel_size"]) as ctx:
        ctx.set_cloud_device(GT, d_gt.data_ptr(), len(gt), keepalive=d_gt)
        levels = [("noise_std_dev", s) for s in (0.0, 0.005, 0.01, 0.02, 0.05, 0.1)] + \
                 [("outlier_ratio", r) for r in (0.0, 0.01, 0.05, 0.1, 0.2)]
        for kind, level in levels:
            ctx.copy_cloud(GT, EST)
            if kind == "noise_std_dev":
                ctx.add_gaussian_noise(EST, level, SEED)
            else:
                ctx.add_sparse_outliers(EST, level, 0.5, SEED)
            nn = ctx.calculateMetricsWithInitialMatrix(p)
            mme = ctx.computeMME(EST, cfg["nn_radius"], 10)
            mme_gt = ctx.computeMME(GT, cfg["nn_radius"], 5)
            awd = ctx.calculateVMD(cfg["vmd_voxel_size"], 100, 5)
            row = {"sweep": kind, "level": level, "n_est": ctx.n[EST], "tau": list(cfg["tau"]),
                   "ac_rmse": list(nn.est_to_gt.rmse), "com_fitness": list(nn.est_to_gt.fitness), "cd": list(nn.cd),
                   "full_cd": nn.full_cd, "mme": mme.mme, "mme_gt": mme_gt.mme, "awd": awd.awd, "scs": awd.scs}
            print(json.dumps(row), flush=True)
            out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-c5", action="store_true")
    ap.add_argument("--skip-curves", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("degradation_sweep.py needs a CUDA device")
    stream = torch.cuda.Stream(device=0)
    torch.cuda.set_stream(stream)
    gpu, plim = card()
    result = {"gpu": gpu, "power_limit_max_sm_clock": plim, "timing": [], "curves": []}

    print(f"card: {gpu}; power limit, max SM clock: {plim}")
    _, d_gt, cfg = synth_torch.make_pair("C3", device="cuda")
    side = cfg["side"]
    clouds = [("C3 gt (10 M)", d_gt, [side / 2] * 3, side / 3)]
    if not args.skip_c5:
        clouds.append(("C5 indoor (200 M)", None, [40.0, 40.0, 1.5], 10.0))
    for name, d, centre, radius in clouds:
        if d is None:
            d_gt = None
            torch.cuda.empty_cache()
            d = synth_torch.indoor_scene(200_000_000, synth.GT_SEED, synth.GT_SURFACE_NOISE_SIGMA, device="cuda")
        t = time_operators(name, d, centre, radius, args.reps, stream)
        result["timing"].append(t)
        c = t["copy"]
        print(f"{name}: share inside the radius {t['share_inside']:.3f}, density keep share {t['keep_share']:.3f}, "
              f"{t['outliers']} outliers; copy of {c['bytes'] / 1e6:.0f} MB: {c['ms_median']:.3f} ms = "
              f"{c['gbs_read_plus_write']:.0f} GB/s (read + write)")
        print(f"  {'operator':12s} {'ms':>9s} {'MB':>8s} {'GB/s':>7s} {'of copy':>8s}")
        for r in t["rows"]:
            print(f"  {r['op']:12s} {r['ms_median']:9.3f} {r['bytes'] / 1e6:8.0f} {r['gbs']:7.0f} {100 * r['of_copy']:7.0f}%")
        del d
        torch.cuda.empty_cache()
    if not args.skip_curves:
        print(f"card: {gpu}; power limit, max SM clock: {plim}")
        result["curves"] = curves(stream)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "degradation_sweep.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
