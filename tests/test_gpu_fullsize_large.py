"""C4 (50 M vs 20 M outdoor, MME r = 1.0 m), C5 (200 M vs 200 M indoor) and S1 (100 M vs 100 M site-scale terrain, sparse
cell table) at the sizes the README quotes, against exact arithmetic (tests/exact_ref.py through tests/fullsize_ref.py).
The CPU oracle would need hours here, so the exact references are applied to every record where that is cheap and to
stratified samples where it is not.

One pass per config with bench.py's settings (path A as written, d2 <= R with R = 1.0, full CD; MME of est at nn_radius
with min_neighbors 10; calculateVMD(v, 100, 5)), clouds generated on the device (synth_torch) and handed over with
set_cloud_device.  Then:
  1. every NN record of both directions: index in range, d2 == d2_kd(q, ref[idx]) bit for bit (on the device);
  2. stratified samples (uniform, first / last 2^16 caller indices, bounding-box faces and corners, lowest / highest
     lattice rows and z-layers, the 1 000 largest d2, on S1 the sparsest tiles): index and d2 equal the exact NN;
  3. n_query, n_corr, n_inlier, n_ub exact, and mean, rmse, sigma, fitness, cd, f1, iou, full CD within exact_ref's
     bounds, from all records;
  4. MME: validity exact and entropy within B64 (+ B32(E) of the sweep's fp32 offsets) on a sample; n_valid and
     sum_entropy against the per-point array.  get_entropies writes 0.0 for a rejected point; an accepted point's
     entropy is 0.5 ln(2 pi e det), exactly 0.0 only if 2 pi e det rounds to 1, which no sampled point comes near (the
     check would report it as a validity mismatch with its exact entropy);
  5. voxels: the voxel and pair counts exact, every row's point counts exact, sampled voxels' Gaussians and W within the
     bounds, AWD, SCS and n_scs recomputed from the device's W table;
  6. accuracy_curve at the config's five levels: counts equal to eval_nn's bit for bit, values within the exact bounds
     of step 3 (its sums run in another order); distance_quantiles(ME_DIST_KEPT) equals np.quantile of the kept
     distances bit for bit;
  7. the kernel paths the trace records.
A config skips only when the device's free memory is below its measured peak (PEAK_GB, DESIGN.md §5)."""
import os
import resource
import sys
import time

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import exact_ref as X  # noqa: E402
import fullsize_ref as F  # noqa: E402
from test_exact_ref import check_nn  # noqa: E402

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
R = 1.0
PROBS = [0.0, 0.5, 0.9, 0.99, 1.0]
# device memory the run needs beyond what is in use when it starts (GB, one H100 80GB HBM3), as measured (DESIGN.md §5)
PEAK_GB = {"C4": 14.7, "C5": 53.0, "S1": 30.5}
# per config: NN sample size per direction (besides first / last 2^16), MME sample, smallest NN window edge, sparse tile
# edge, sparse tile, random voxels (C5's 2 m voxels hold ~60 000 points each, summed exactly in Python)
SETUP = {"C4": dict(n_nn=20000, n_mme=300, m_min=1 / 32, sparse=None, n_vox=40),
         "C5": dict(n_nn=20000, n_mme=2000, m_min=1 / 32, sparse=None, n_vox=20),
         "S1": dict(n_nn=20000, n_mme=2000, m_min=1 / 8, sparse=10.0, n_vox=60)}


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _nn_direction(name, torch, query, ref, idx_h, d2_h, n_uniform, m_min, h_rows, seed, sparse):
    """checks 1 and 2 for one direction; returns what was covered"""
    dev = query.device
    idx = torch.from_numpy(idx_h).to(dev)
    d2 = torch.from_numpy(d2_h).to(dev)
    F.check_records(query, ref, idx, d2)
    st = F.strata(query, d2, n_uniform, seed, h_rows, sparse_tile=sparse)
    del idx, d2
    qi = np.unique(np.concatenate(list(st.values())))
    ex_i, ex_d, n_brute = F.exact_nn_sample(query, ref, qi, d2_h[qi], m_min)
    F.check_sample(name, qi, idx_h, d2_h, ex_i, ex_d)
    beyond = int((ex_d > R).sum())          # no neighbour within the cut-off: the record is still the exact NN, not kept
    return dict(sample=len(qi), strata={k: len(v) for k, v in st.items()}, brute=n_brute, beyond_cutoff=beyond)


@pytest.mark.parametrize("name", ["C4", "C5", "S1"])
def test_full_size_against_exact(api, name):
    import torch
    from cloud_map_evaluation_b200 import synth_torch
    dev = torch.device("cuda", 0)
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0] / 2 ** 30
    if free < PEAK_GB[name]:
        pytest.skip(f"{name} needs {PEAK_GB[name]:.0f} GB of device memory; {free:.1f} GB free")
    meter = F.Meter()
    setup = SETUP[name]
    est, gt, cfg = synth_torch.make_pair(name, device=dev)
    n_est, n_gt = len(est), len(gt)
    assert (n_est, n_gt) == (synth_torch.synth.CONFIGS[name]["n_est"], synth_torch.synth.CONFIGS[name]["n_gt"])
    r, v, tau = cfg["nn_radius"], cfg["vmd_voxel_size"], cfg["tau"]
    p = A.make_nn_params(tau, R)
    torch.cuda.synchronize()
    meter.sample()

    # ---- one pass, bench.py's order: MME, NN, voxels ----------------------------------------------------------------
    with api.MapEvalB200(vmd_voxel_size=v) as ctx:
        ctx.set_cloud_device(EST, est.data_ptr(), n_est, keepalive=est)
        ctx.set_cloud_device(GT, gt.data_ptr(), n_gt, keepalive=gt)
        macc = ctx.eval_mme_accum(EST, r, 10)
        ent = ctx.get_entropies(EST)
        meter.sample()
        e_acc, g_acc = ctx.eval_nn_accum(p)
        nn = ctx.nn_finalize(p, e_acc, g_acc)
        ie, de = ctx.get_nn(EST)
        ig, dg = ctx.get_nn(GT)
        order = np.argsort(tau, kind="stable")     # the curve takes its levels ascending, the configs list them descending
        curve = ctx.accuracy_curve(np.asarray(tau)[order])
        quant = ctx.distance_quantiles(PROBS, A.ME_DIST_KEPT)
        meter.sample()
        awd, rows = ctx.calculateVMD(v, 100, 5, want_rows=True)
        meter.sample()
        trace, _ = ctx.kernel_trace(events=True)
    t_pass = time.time() - meter.t0
    covered = {"trace": sorted(trace)}

    # ---- 7. the paths that ran --------------------------------------------------------------------------------------
    # all three take the sparse cell table for the 1-NN sweeps (the plan refines the edge below the dense budget), reach
    # the far kernel, and sweep MME on a lattice of its own (r spans more than 3 shared cells) with two rings; only S1's
    # solo lattice is sparse.  The trace is a function of the seeded clouds.
    expect = {"ME_KBIT_NN_ROWS_SPARSE", "ME_KBIT_NN_FAR", "ME_KBIT_MME_SOLO", "ME_KBIT_SCS_R5",
              "ME_KBIT_MME_FLAT2_SPARSE" if name == "S1" else "ME_KBIT_MME_FLAT2_DENSE"}
    assert trace == expect, sorted(trace)

    # ---- 1 + 2. every record, and the stratified samples ------------------------------------------------------------
    covered["est_to_gt"] = _nn_direction(f"{name} est->gt", torch, est, gt, ie, de, setup["n_nn"], setup["m_min"], r, 1,
                                         setup["sparse"])
    meter.sample()
    covered["gt_to_est"] = _nn_direction(f"{name} gt->est", torch, gt, est, ig, dg, setup["n_nn"], setup["m_min"], r, 2,
                                         setup["sparse"])
    meter.sample()

    # ---- 3. whole-map statistics from all records -------------------------------------------------------------------
    de_t, dg_t = torch.from_numpy(de).to(dev), torch.from_numpy(dg).to(dev)
    ie_t, ig_t = torch.from_numpy(ie).to(dev), torch.from_numpy(ig).to(dev)
    sq_e, d_e, ub_e = F.kept_pairs_t(est, gt, ie_t, de_t, R, A.ME_CUTOFF_SQDIST_LE_R)
    ex_e = F.dir_stats_t(sq_e, d_e, n_est, tau)
    del sq_e
    kept_e = d_e.cpu().numpy()
    del d_e
    sq_g, d_g, ub_g = F.kept_pairs_t(gt, est, ig_t, dg_t, R, A.ME_CUTOFF_SQDIST_LE_R, as_written=True)
    ex_g = F.dir_stats_t(sq_g, d_g, n_gt, tau)
    del sq_g
    kept_g = d_g.cpu().numpy()
    del d_g, ie_t, ig_t
    meter.sample()
    F.check_accum("est_to_gt", e_acc, ex_e, n_est, ub_e)
    F.check_accum("gt_to_est", g_acc, ex_g, n_gt, ub_g)
    res = X.nn_result(ex_e, ex_g, n_est, n_gt)
    res["full_cd"] = float(F.exact_sum_t(F.sqrt_rn(de_t)) / n_est + F.exact_sum_t(F.sqrt_rn(dg_t)) / n_gt)
    del de_t, dg_t
    check_nn(nn, ex_e, ex_g, res)
    covered["n_ub_gt_to_est"] = ub_g

    # ---- 6. consumers of the same records ---------------------------------------------------------------------------
    # the curve sums its levels as prefix sums over bins (DESIGN.md §3.10), in another order than eval_nn: its counts are
    # eval_nn's bit for bit, its values are held to the same exact statistics and bounds as eval_nn's
    for d, ex in (("est_to_gt", ex_e), ("gt_to_est", ex_g)):
        got, want = curve[d], getattr(nn, d)
        assert list(got["n_inlier"]) == list(np.array(want.n_inlier)[order]), d
        mean_all = float(ex["mean_all"])
        for j, k in enumerate(order):
            for f in ("mean", "rmse", "fitness"):
                assert abs(got[f][j] - ex[f][k]) <= X.rel_bound(ex[f][k]), (d, f, k, got[f][j], ex[f][k])
            assert abs(got["sigma"][j] - ex["sigma"][k]) <= X.sigma_bound(ex["sigma"][k], mean_all), (d, k)
    for f in ("cd", "f1", "iou"):
        for j, k in enumerate(order):
            assert abs(curve[f][j] - res[f][k]) <= X.rel_bound(res[f][k]), (f, k, curve[f][j], res[f][k])
    for d, kept in (("est_to_gt", kept_e), ("gt_to_est", kept_g)):
        assert quant[d]["n"] == len(kept), d
        want = np.quantile(kept, PROBS, method="linear")
        np.testing.assert_array_equal(quant[d]["value"].view(np.int64), want.view(np.int64), err_msg=d)
    del kept_e, kept_g

    # ---- 4. MME -----------------------------------------------------------------------------------------------------
    assert macc.n_query == n_est
    ent_t = torch.from_numpy(ent).to(dev)
    assert macc.n_valid == int((ent_t != 0).sum())
    s_ex = F.exact_sum_t(ent_t)
    s_abs = float(F.exact_sum_t(ent_t.abs()))
    del ent_t
    assert abs(macc.sum_entropy - float(s_ex)) <= n_est * X.U * s_abs, (macc.sum_entropy, float(s_ex))
    rs = np.random.RandomState(3)
    mst = F.strata(est, None, setup["n_mme"], 4, r, per=16)
    mq = np.unique(np.concatenate([mst["uniform"]] + [rs.choice(mst[k], min(32, len(mst[k])), replace=False)
                                                      for k in ("faces", "corners", "rows", "first", "last")]))
    qh, nbs = F.ball_neighbours(est, mq, r)
    exs = F.mme_sample_exact(qh, nbs, 10)
    maxabs = float(est.abs().max())
    E = F.sweep_offsets(trace, r, maxabs)
    if E == "unknown":          # a shared-lattice sweep whose cell edge the trace does not bound: B64 + 2 tau
        for ex in exs:
            ex["b64"] += 2 * X.TAU_FP64
        E = None
    checked, worst_mme, und = F.check_mme_sample(mq, ent, exs, E)
    assert checked > 0.9 * len(mq), (checked, len(mq), und)
    ks = [ex["k"] for ex in exs]
    covered["mme"] = dict(sample=len(mq), undetermined=und, worst=worst_mme, k_median=float(np.median(ks)),
                          k_max=int(max(ks)), E=E)
    del ent
    meter.sample()

    # ---- 5. voxels --------------------------------------------------------------------------------------------------
    packing, ue, ce, ug, cg, pairs = F.voxel_counts(est, gt, v, 100)
    assert (awd.n_voxels_est, awd.n_voxels_gt, awd.n_pairs) == (len(ue), len(ug), len(pairs))
    lo, dims = packing
    rk = torch.from_numpy(F.row_keys(rows, v)).to(dev)
    pk = F.pack_keys(rk, lo, dims)
    assert torch.equal(torch.sort(pk).values, torch.sort(pairs).values)
    n_e_rows = ce[torch.searchsorted(ue, pk)].cpu().numpy()
    n_g_rows = cg[torch.searchsorted(ug, pk)].cpu().numpy()
    np.testing.assert_array_equal(rows[:, 11].astype(np.int64), n_e_rows)
    np.testing.assert_array_equal(rows[:, 10].astype(np.int64), n_g_rows)
    meter.sample()
    del ue, ce, ug, cg, pairs
    rk_h = F.row_keys(rows, v)
    pick = set(rs.choice(len(rows), min(len(rows), setup["n_vox"]), replace=False).tolist())
    pick |= set(np.argsort(-(n_e_rows + n_g_rows))[:5].tolist())
    for a in range(3):
        pick |= {int(np.argmin(rk_h[:, a])), int(np.argmax(rk_h[:, a]))}
    pick = sorted(pick)
    keys_t = pk[torch.tensor(pick, device=dev)]
    pe, pg = F.voxel_points(est, v, packing, keys_t), F.voxel_points(gt, v, packing, keys_t)
    worst_w = max(F.check_voxel_row(rows[i], tuple(rk_h[i]), pe[tuple(rk_h[i])], pg[tuple(rk_h[i])], v) for i in pick)
    del pe, pg
    # AWD: the mean of the device's W; the device's sum of n positive values in any order is within (n - 1) u of it
    w = rows[:, 9]
    awd_ex = float(X.exact_sum(w) / len(w))
    assert abs(awd.awd - awd_ex) <= (len(w) + 1) * X.U * awd_ex, (awd.awd, awd_ex)
    # SCS of the device's W table: shifted sums on the key grid, checked against mpmath on a sample of keys
    term, cnt = F.scs_grid(rk_h, w, 5, device=dev)
    has = cnt > 0
    assert awd.n_scs == int(has.sum())
    scs = float(X.exact_sum(term[has]) / int(has.sum()))
    assert abs(awd.scs - scs) <= 1e-10 * abs(scs), (awd.scs, scs)
    table = {tuple(int(c) for c in k): x for k, x in zip(rk_h, w)}
    for i in rs.choice(np.nonzero(has)[0], min(50, int(has.sum())), replace=False):
        t_ex = F.scs_key_exact(table, tuple(int(c) for c in rk_h[i]), 5)
        assert abs(term[i] - float(t_ex)) <= 1e-12 * abs(float(t_ex)), (i, term[i], float(t_ex))
    covered["voxels"] = dict(rows=len(rows), sampled=len(pick), worst_w=worst_w, n_voxels_est=awd.n_voxels_est,
                             n_voxels_gt=awd.n_voxels_gt)
    meter.sample()
    del est, gt
    torch.cuda.empty_cache()
    wall = time.time() - meter.t0
    host_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    print(f"\n{name}: {n_est} est vs {n_gt} gt; wall {wall:.0f} s (pass + records {t_pass:.0f} s); device peak "
          f"{meter.peak / 2 ** 30:.1f} GB beyond the start; host max RSS {host_gb:.1f} GB; covered {covered}")
