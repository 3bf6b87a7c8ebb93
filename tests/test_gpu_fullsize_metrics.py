"""The per-map metrics of C4 (50 M vs 20 M), C5 (200 M vs 200 M) and S1 (100 M vs 100 M) at full size against exact
arithmetic (tests/exact_ref.py, tests/consistency_ref.py through tests/fullsize_ref.py): the region table
(me_nn_regions, DESIGN §3.12), the point-to-plane metrics and normal consistency (me_nn_surface, §3.14), local consistency
(me_consistency, §3.15) and the GT-side MME.  A module of its own beside test_gpu_fullsize_large.py: it leaves normals on
both clouds and lets consistency lay the clouds out again, its memory peak differs, and a failure names the feature.

One pass per config, clouds generated on the device, bench.py's NN settings (path A as written, d2 <= R with R = 1.0, full
CD), every consumer reading fresh records:
  1. eval_mme_accum(EST, r, 10), 2. eval_mme_accum(GT, r, 5), 3. eval_nn_accum, 4. region_errors at vmd_voxel_size (and
  on S1 at 0.875 m: 1.8 M regions, close to ME_REGION_MAX_REGIONS = 2^21), 5. surface_metrics(knn=20), estimate_normals of
  both clouds, surface_metrics(0) on them, 6. the normals handed back scaled by 2^k per point and by non-dyadic factors
  with zeroed and NaN normals, 7. local_consistency of est (r, 10) and gt (r, 5) at s = 0 and s = vmd_voxel_size.
Checks:
  * regions: the region of each query is IEEE floor(x / s) (torch's fp64 division is checked to round correctly); the
    occupied list, n_est, n_gt, n_query, n_corr, n_inlier, max_d and max_nn of every region and direction exact; Sd, Sd^2
    and sum_nn within (n_r - 1) u sum|x| of exact segmented sums; ~2 000 uniform regions, the 20 most populated, the
    extreme keys and the regions of the 1 000 largest d^2 against exact_ref's values and bounds; the rows' counts sum to
    the whole-map accumulators;
  * surface: e and c per pair with one torch operation per kernel operation, so the kernel's bits: counts and maxima
    exact, the statistics within exact_ref's bounds; every kept pair whose e lies within 2 beta of a level decided exactly
    in rationals (beta: fullsize_ref.plane_beta, e's rounding from d, three products, two sums, a square root and a
    division: <= 8 u sum|d_i n_i| / ||n||), and e and c on 10 000 pairs against mpmath within beta;
  * k-NN normals: ~2 600 stratified points per cloud (uniform, faces, corners, first / last caller indices, extreme rows,
    S1's sparsest tiles) against exact_reg.check_normal with their exact 20 nearest neighbours (fullsize_ref.window_knn:
    the 20th neighbour proven inside the window's boundary, else a larger window, else brute force);
  * scaled normals: the clouds' own normals, and those scaled by 2^k per point (k in -3..3), give the working normals'
    result bit for bit (every field compared by its bits); factors in [0.5, 3] with 10 000
    zeroed and 1 000 NaN normals give results within the bounds and n_no_normal exact;
  * consistency: n_query, n_valid, n_pv and max_pv exact, Se, Sv and S sqrt(v) of the map and of every region within the
    order bound; the region list equal to the region table's; on a sample (as MME's), validity exact, e within B64 and v
    within consistency_ref.fp64_bound of the mpmath lambda3; n_valid equal to MME's or each differing point undecidable;
  * GT-side MME (m = 5): validity and entropy on a sample, as test_gpu_fullsize_large.py step 4;
  * teeth: a pair filed under its reference point's region, e / ||n||^2, v as the largest eigenvalue and the covariance
    divided by k (on every valid sampled query) each break their check at full size; the key as x (1 / s) is counted
    (the points it would file elsewhere), not asserted: on these float32-quantised clouds it can move none at s = 2, 3
    and 0.875 m, so no check here would notice a kernel that formed the key with a reciprocal;
  * the kernel paths the trace records after the MME and NN passes, and no bit after the surface and consistency steps
    (local_consistency reports its sweep in its result: the walk, solo lattice, two rings).
A config skips only when the device's free memory is below its measured peak (PEAK_GB, DESIGN.md §5)."""
import math
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

pytestmark = pytest.mark.gpu

EST, GT = A.ME_CLOUD_EST, A.ME_CLOUD_GT
R = 1.0
# device memory the run needs beyond what is in use when it starts (GB, one H100 80GB HBM3), as measured (DESIGN.md §5)
PEAK_GB = {"C4": 20.1, "C5": 75.6, "S1": 41.5}
# per config: MME / consistency sample, extra region sizes (S1: between 2^20 and 2^21 occupied regions), the first window
# edge of the exact 20-NN search, sparse tile edge of the normal sample
SETUP = {"C4": dict(n_mme=300, extra=[], m_knn=1 / 8, sparse=None),
         "C5": dict(n_mme=2000, extra=[], m_knn=1 / 32, sparse=None),
         "S1": dict(n_mme=2000, extra=[0.875], m_knn=1 / 8, sparse=10.0)}


@pytest.fixture(scope="module")
def api():
    from cloud_map_evaluation_b200 import api as _api
    return _api


def _mme_sample(torch, cloud, r, m, setup, seed):
    """the MME sample of test_gpu_fullsize_large.py step 4: (indices, query coordinates, neighbours, exact points)"""
    rs = np.random.RandomState(seed)
    mst = F.strata(cloud, None, setup["n_mme"], seed + 1, r, per=16)
    mq = np.unique(np.concatenate([mst["uniform"]] + [rs.choice(mst[k], min(32, len(mst[k])), replace=False)
                                                      for k in ("faces", "corners", "rows", "first", "last")]))
    qh, nbs = F.ball_neighbours(cloud, mq, r)
    return mq, qh, nbs, F.mme_sample_exact(qh, nbs, m)


def _assert_same_bits(a, b, what, path=""):
    """two surface_dict results equal bit for bit: every float by its bits (NaN included), every count by value"""
    if isinstance(a, dict):
        assert a.keys() == b.keys(), (what, path)
        for k in a:
            _assert_same_bits(a[k], b[k], what, f"{path}.{k}")
        return
    x, y = np.asarray(a), np.asarray(b)
    assert x.dtype == y.dtype and x.shape == y.shape, (what, path)
    if x.dtype.kind == "f":
        assert np.array_equal(x.view(np.int64), y.view(np.int64)), (what, path, x, y)
    else:
        assert np.array_equal(x, y), (what, path, x, y)


def _normal_sample(cloud, r, setup, seed):
    """>= 2 000 points per cloud: 2 000 uniform, and up to 128 of each of the faces, corners, first / last caller indices,
    lowest / highest lattice rows and (S1) the sparsest 10 m tiles"""
    rs = np.random.RandomState(seed)
    st = F.strata(cloud, None, 2000, seed + 1, r, per=64, sparse_tile=setup["sparse"])
    parts = [st["uniform"]] + [rs.choice(st[k], min(128, len(st[k])), replace=False)
                               for k in ("faces", "corners", "first", "last", "rows", "sparse") if k in st]
    return np.unique(np.concatenate(parts))


def _mme_check(ent, mq, exs, E):
    if E == "unknown":
        for ex in exs:
            ex["b64"] += 2 * X.TAU_FP64
        E = None
    checked, worst, und = F.check_mme_sample(mq, ent, exs, E)
    assert checked > 0.9 * len(mq), (checked, len(mq), und)
    return dict(sample=len(mq), undetermined=und, worst=worst, k_median=float(np.median([ex["k"] for ex in exs])))


# ---------------------------------------------------------------------------------------------------------------
# the region table
# ---------------------------------------------------------------------------------------------------------------
def _check_regions(torch, name, est, gt, rows, s, recs, tau, e_acc, g_acc, rs):
    L = F.region_list_t(est, gt, s)
    n = L["keys"].numel()
    assert len(rows["n_est"]) == n, (name, s, len(rows["n_est"]), n)
    np.testing.assert_array_equal(rows["index"], L["index"].cpu().numpy())
    np.testing.assert_array_equal(rows["n_est"], L["n_est"].cpu().numpy())
    np.testing.assert_array_equal(rows["n_gt"], L["n_gt"].cpu().numpy())
    # the sampled rows: ~2 000 uniform regions, the 20 most populated, the extreme keys, the regions of the 1 000 largest d2
    pick = set(rs.choice(n, min(n, 2000), replace=False).tolist())
    pick |= set(np.argsort(-(rows["n_est"] + rows["n_gt"]))[:20].tolist())
    for a in range(3):
        pick |= {int(np.argmin(rows["index"][:, a])), int(np.argmax(rows["index"][:, a]))}
    for seg, (_, _, idx, d2, _) in ((L["seg_est"], recs[0]), (L["seg_gt"], recs[1])):
        pick |= set(seg[torch.topk(d2.nan_to_num(nan=-1.0), 1000).indices].cpu().tolist())
    pick = sorted(pick)
    pick_t = torch.tensor(pick, dtype=torch.int64, device=est.device)
    D = {}
    worst = 0.0
    for d, seg, other, (query, ref, idx, d2, aw), acc in (("est_to_gt", L["seg_est"], L["seg_gt"], recs[0], e_acc),
                                                          ("gt_to_est", L["seg_gt"], L["seg_est"], recs[1], g_acc)):
        qi, sq, dist = F.region_pairs_t(query, ref, idx, d2, R, aw)
        row = rows[d]
        T = F.region_direction_t(seg, n, idx, d2, qi, sq, dist, tau, row=row, pick=pick_t)
        worst = max(worst, T["worst"])
        for f in ("n_query", "n_corr"):
            np.testing.assert_array_equal(row[f], T[f].cpu().numpy(), err_msg=f"{name} s={s} {d} {f}")
        np.testing.assert_array_equal(row["n_inlier"], torch.stack(T["n_inlier"], 1).cpu().numpy(),
                                      err_msg=f"{name} s={s} {d} n_inlier")
        for f in ("max_d", "max_nn"):
            np.testing.assert_array_equal(row[f].view(np.int64), T[f].cpu().numpy().view(np.int64),
                                          err_msg=f"{name} s={s} {d} {f}")
        # the rows' counts add up to the whole-map accumulators
        assert (int(row["n_query"].sum()), int(row["n_corr"].sum())) == (acc.n_query, acc.n_corr), (name, d)
        assert list(row["n_inlier"].sum(0)) == list(acc.n_inlier), (name, d)
        # tooth: a pair filed under its reference point's region (the as-written pair's point is a swapped index)
        if not aw:
            wrong = torch.bincount(other[idx[qi].to(torch.int64)], minlength=n).cpu().numpy()
            assert not np.array_equal(wrong, row["n_corr"]), (name, s, d, "filed under the reference region passes")
        D[d] = T
        del qi, sq, dist
    for pos, i in enumerate(pick):
        F.check_region_row(rows, i, D["est_to_gt"], D["gt_to_est"], tau, pos)
    del D
    # the key as x (1 / s): how many points it files elsewhere (none can move at s = 2, and on float32 coordinates none
    # moved at 3 m or 0.875 m either: a multiple k s of such an edge gives k (1 + delta) with |delta| <= 2^-54, which rounds
    # back to k; test_fullsize_reference.py shows the variant on fp64 faces)
    W = F.region_list_t(est, gt, s, recip=True)
    moved = int((W["keys"][W["seg_est"]] != L["keys"][L["seg_est"]]).sum() +
                (W["keys"][W["seg_gt"]] != L["keys"][L["seg_gt"]]).sum())
    del W, L
    return dict(regions=n, sampled=len(pick), worst_sum=worst, recip_moved=moved)


# ---------------------------------------------------------------------------------------------------------------
# point-to-plane
# ---------------------------------------------------------------------------------------------------------------
def _surface_expected(torch, est, gt, ne, ng, recs, tau, n_est, n_gt, wrong_norm=False):
    P = []
    ex = []
    for (query, ref, idx, d2, _), qn, rn, n_src in ((recs[0], ne, ng, n_est), (recs[1], ng, ne, n_gt)):
        p = F.surface_pairs_t(query, ref, qn, rn, idx, d2, R, wrong_norm=wrong_norm)
        ex.append(F.surface_direction_t(p, n_src, tau))
        P.append(p)
    return P, ex


def _check_surface(name, got, ex, tau, n_est, n_gt):
    nc = [F.check_surface_dir(f"{name} {d}", got[d], e, tau) for d, e in (("est_to_gt", ex[0]), ("gt_to_est", ex[1]))]
    res = X.nn_result(ex[0], ex[1], n_est, n_gt)
    for f in ("cd", "f1", "iou"):
        for k in range(5):
            assert F._close(float(got[f][k]), res[f][k], X.rel_bound(res[f][k])), (name, f, k, got[f][k], res[f][k])
    full = float(ex[0]["sum_nn"] / n_est + ex[1]["sum_nn"] / n_gt)
    assert abs(got["full_cd"] - full) <= X.rel_bound(full), (name, got["full_cd"], full)
    want = (nc[0] + nc[1]) / 2
    assert F._close(got["normal_consistency"], want, X.rel_bound(want) + 2 * X.U * abs(want)), name


def _plane_definition(torch, recs, ne, ng, P, tau, rs):
    """pairs within 2 beta of a level decided exactly; e and c on 10 000 pairs against mpmath"""
    undecided, checked, worst = 0, 0, 0.0
    for (query, ref, idx, d2, _), qn, rn, p in ((recs[0], ne, ng, P[0]), (recs[1], ng, ne, P[1])):
        sel = torch.nonzero(p["kept"] & p["ok_n"]).reshape(-1)
        j = idx[sel].to(torch.int64)
        dd = query[sel] - ref[j]
        nv = rn[j]
        beta = 8.0 * X.U * (dd.abs() * nv.abs()).sum(1) / F.sqrt_rn(F.sqnorm_eigen_t(nv)) * (1 + 1e-10)
        e = p["e"][sel]
        for t in tau:
            near = torch.nonzero((e - t).abs() <= 2 * beta).reshape(-1)
            for a in near.cpu().tolist():
                undecided += 1
                qa, ja = int(sel[a]), int(j[a])
                exact = F.exact_inlier(query[qa].tolist(), ref[ja].tolist(), rn[ja].tolist(), t)
                if exact != bool(e[a] <= t):
                    assert abs(float(e[a]) - t) <= float(beta[a]), (qa, float(e[a]), t, float(beta[a]))
        pick = torch.from_numpy(rs.choice(sel.numel(), min(5000, sel.numel()), replace=False)).to(sel.device)
        for a in pick.cpu().tolist():
            qa, ja = int(sel[a]), int(j[a])
            m = qn[qa].tolist() if bool(p["ok_m"][qa]) else None
            e_ex, c_ex = F.exact_plane(query[qa].tolist(), ref[ja].tolist(), rn[ja].tolist(), m)
            b = float(beta[a])
            err = abs(float(e[a]) - e_ex)
            assert err <= b, (qa, float(e[a]), e_ex, b)
            worst = max(worst, err / b if b > 0 else 0.0)
            if m is not None:
                mv, nn = np.array(m), np.array(rn[ja].tolist())
                bc = 8.0 * X.U * float((np.abs(mv) * np.abs(nn)).sum() / (math.sqrt(X.sqnorm_eigen(mv[None])[0]) *
                                                                           math.sqrt(X.sqnorm_eigen(nn[None])[0])))
                assert abs(float(p["c"][qa]) - c_ex) <= bc * (1 + 1e-10), (qa, float(p["c"][qa]), c_ex, bc)
            checked += 1
        del sel, j, dd, nv, beta, e
    return dict(near_level=undecided, mpmath_pairs=checked, worst_e=worst)


def _dyadic_normals(torch, nrm, seed):
    """each normal scaled by 2^k, k uniform in -3..3 (seeded)"""
    gen = torch.Generator(device=nrm.device).manual_seed(seed)
    k = torch.randint(-3, 4, (len(nrm), 1), generator=gen, device=nrm.device).to(torch.float64)
    return nrm * torch.exp2(k)


def _odd_normals(torch, nrm, seed):
    """each normal scaled by a factor in [0.5, 3] that is not a power of two, 10 000 of them zeroed and 1 000 set to NaN
    (seeded: the same normals on every call on one device)"""
    gen = torch.Generator(device=nrm.device).manual_seed(seed)
    f = torch.rand((len(nrm), 1), generator=gen, device=nrm.device, dtype=torch.float64) * 2.5 + 0.5
    f = torch.where(torch.frexp(f)[0] == 0.5, f * 1.25, f)
    o = nrm * f
    cut = torch.randperm(len(nrm), generator=gen, device=nrm.device)[:11000]
    o[cut[:10000]] = 0.0
    o[cut[10000:]] = float("nan")
    return o


@pytest.mark.parametrize("name", ["C4", "C5", "S1"])
def test_full_size_metrics_against_exact(api, name):
    import torch
    from cloud_map_evaluation_b200 import synth_torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0] / 2 ** 30
    if free < PEAK_GB[name]:
        pytest.skip(f"{name} needs {PEAK_GB[name]:.0f} GB of device memory; {free:.1f} GB free")
    meter = F.Meter()
    setup = SETUP[name]
    est, gt, cfg = synth_torch.make_pair(name, device=dev)
    n_est, n_gt = len(est), len(gt)
    r, v, tau = cfg["nn_radius"], cfg["vmd_voxel_size"], list(cfg["tau"])
    sizes = [v] + setup["extra"]
    p = A.make_nn_params(tau, R)
    rs = np.random.RandomState(11)
    covered = {}
    meter.sample()

    # ---- the pass: every library call, then the context is closed so that the checks have the device to themselves -----
    with api.MapEvalB200(vmd_voxel_size=v) as ctx:
        ctx.set_cloud_device(EST, est.data_ptr(), n_est, keepalive=est)
        ctx.set_cloud_device(GT, gt.data_ptr(), n_gt, keepalive=gt)
        # 1-3. MME of both clouds, then the NN pass
        macc_e = ctx.eval_mme_accum(EST, r, 10)
        ent_e = ctx.get_entropies(EST)
        macc_g = ctx.eval_mme_accum(GT, r, 5)
        ent_g = ctx.get_entropies(GT)
        meter.sample()
        e_acc, g_acc = ctx.eval_nn_accum(p)
        ie, de = ctx.get_nn(EST)
        ig, dg = ctx.get_nn(GT)
        trace_nn, _ = ctx.kernel_trace(events=True)
        # 4. the region table
        region_rows = {s: ctx.region_errors(s) for s in sizes}
        meter.sample()
        # 5. point-to-plane with working normals, then the same normals held by the clouds
        surf = ctx.surface_metrics(knn=20)
        ne_h = ctx.estimate_normals(EST, 20)
        ng_h = ctx.estimate_normals(GT, 20)
        again = ctx.surface_metrics(knn=0)
        meter.sample()
        # 6. scaled normals: 2^k per point, then non-dyadic factors with zeroed and NaN normals
        # (formed on the host: the context holds most of the device here)
        for which, nrm in ((EST, ne_h), (GT, ng_h)):
            ctx.set_normals(which, _dyadic_normals(torch, torch.from_numpy(nrm), 7 + which).numpy())
        dyadic = ctx.surface_metrics(knn=0)
        for which, nrm in ((EST, ne_h), (GT, ng_h)):
            ctx.set_normals(which, _odd_normals(torch, torch.from_numpy(nrm), 9 + which).numpy())
        surf_odd = ctx.surface_metrics(knn=0)
        meter.sample()
        trace_pass, _ = ctx.kernel_trace(events=True)
        # 7. local consistency (may lay the clouds out again: after every consumer of the records)
        cons = {}
        for which, m in ((EST, 10), (GT, 5)):
            for s in (0.0, v):
                res = ctx.local_consistency(which, r, m, s)
                cons[(which, s)] = (res,) + ctx.get_consistency_points(which)
            meter.sample()
        trace_cons, _ = ctx.kernel_trace(events=True)
    t_pass = time.time() - meter.t0
    meter.sample()

    recs = ((est, gt, torch.from_numpy(ie).to(dev), torch.from_numpy(de).to(dev), False),
            (gt, est, torch.from_numpy(ig).to(dev), torch.from_numpy(dg).to(dev), True))
    del ie, de, ig, dg
    # ---- 4. the region table ------------------------------------------------------------------------------------------
    covered["division_checked"] = sum(F.division_is_rounded(c, s, 20000, 5 + j) for s in sizes for j, c in enumerate((est, gt)))
    covered["regions"] = {}
    region_lists = {}
    for s in sizes:
        rows = region_rows.pop(s)
        region_lists[s] = (rows["index"], rows["n_est"], rows["n_gt"])
        covered["regions"][s] = _check_regions(torch, name, est, gt, rows, s, recs, tau, e_acc, g_acc, rs)
        del rows
        meter.sample()
    if name == "S1":
        assert (1 << 20) <= covered["regions"][0.875]["regions"] <= A.ME_REGION_MAX_REGIONS, covered["regions"]

    # ---- 5. point-to-plane ----------------------------------------------------------------------------------------------
    _assert_same_bits(again, surf, f"{name}: the clouds' normals against the working normals")
    _assert_same_bits(dyadic, surf, f"{name}: normals scaled by 2^k against unit normals")
    # the k-NN normals themselves on a stratified sample: exact 20 nearest neighbours, exact_reg.check_normal's bounds
    covered["normals"] = {}
    for side, cloud, nrm, seed in (("est", est, ne_h, 31), ("gt", gt, ng_h, 32)):
        qn = _normal_sample(cloud, r, setup, seed)
        nbs, n_brute = F.exact_knn_sample(cloud, qn, 20, setup["m_knn"], 8.0)
        checked, signed, worst = F.check_normals_sample(cloud, qn, nbs, nrm[qn])
        covered["normals"][side] = dict(sample=checked, sign_checked=signed, worst_sin=worst, brute=n_brute)
        meter.sample()
    ne, ng = torch.from_numpy(ne_h).to(dev), torch.from_numpy(ng_h).to(dev)
    P, ex = _surface_expected(torch, est, gt, ne, ng, recs, tau, n_est, n_gt)
    _check_surface(f"{name} unit", surf, ex, tau, n_est, n_gt)
    covered["surface"] = _plane_definition(torch, recs, ne, ng, P, tau, rs)
    covered["surface"]["n_corr"] = (ex[0]["n_corr"], ex[1]["n_corr"])
    del P, ex
    meter.sample()
    # ---- 6. the non-dyadic normals: within the bounds, n_no_normal exact; e / ||n||^2 breaks the check ---------------
    del ne, ng
    odd = [_odd_normals(torch, torch.from_numpy(ne_h), 9 + EST).to(dev), _odd_normals(torch, torch.from_numpy(ng_h), 9 + GT).to(dev)]
    del ne_h, ng_h
    P, ex = _surface_expected(torch, est, gt, odd[0], odd[1], recs, tau, n_est, n_gt)
    _check_surface(f"{name} non-dyadic", surf_odd, ex, tau, n_est, n_gt)
    assert ex[0]["n_no_normal"] > 0 and ex[1]["n_no_normal"] > 0
    covered["surface"]["no_normal"] = (ex[0]["n_no_normal"], ex[1]["n_no_normal"])
    del P, ex
    Pw, exw = _surface_expected(torch, est, gt, odd[0], odd[1], recs, tau, n_est, n_gt, wrong_norm=True)
    with pytest.raises(AssertionError):
        _check_surface(f"{name} e / |n|^2", surf_odd, exw, tau, n_est, n_gt)
    del Pw, exw, odd, recs
    meter.sample()
    cons = {k: (c[0], torch.from_numpy(c[1]).to(dev), torch.from_numpy(c[2]).to(dev)) for k, c in cons.items()}

    # ---- consistency: every point, every region -------------------------------------------------------------------------
    covered["consistency"] = {}
    for which, cloud, m, macc, ent in ((EST, est, 10, macc_e, ent_e), (GT, gt, 5, macc_g, ent_g)):
        side = "est" if which == EST else "gt"
        cv = {}
        for s in (0.0, v):
            res, e_p, v_p = cons[(which, s)]
            if s == 0:
                seg, nseg = torch.zeros(len(cloud), dtype=torch.int64, device=dev), 1
            else:
                L = F.region_list_t(est, gt, s)
                seg, nseg = (L["seg_est"] if which == EST else L["seg_gt"]), L["keys"].numel()
                idx_t, ne_t, ng_t = region_lists[s]
                np.testing.assert_array_equal(res["index"], idx_t, err_msg=f"{name} {side} consistency regions")
                np.testing.assert_array_equal(res["n_points"], ne_t if which == EST else ng_t)
                del L
            T = F.consistency_regions_t(e_p, v_p, seg, nseg)
            W = res["whole"]
            assert (W["n_query"], W["n_valid"], W["n_pv"]) == (len(cloud), int(T["n_valid"].sum()), int(T["n_pv"].sum()))
            assert W["max_pv"] == float(T["max_pv"].max()), (W["max_pv"], float(T["max_pv"].max()))
            worst = 0.0
            valid, pv = e_p != 0, torch.isfinite(v_p)
            for f, x in (("sum_entropy", e_p[valid]), ("sum_pv", v_p[pv]), ("sum_sqrt_pv", F.sqrt_rn(v_p[pv]))):
                # the whole map (the rows' sums added in list order, or one region): within n u sum|x| of the exact sum
                s_ex, s_abs = F.exact_sum_t(x), float(F.exact_sum_t(x.abs()))
                assert abs(W[f] - float(s_ex)) <= x.numel() * X.U * s_abs, (name, side, s, f, W[f], float(s_ex))
                if s > 0:
                    cnt = T["n_valid"] if f == "sum_entropy" else T["n_pv"]
                    got = torch.from_numpy(np.ascontiguousarray(res[f])).to(dev)
                    worst = max(worst, F.check_seg_sum(f"{side} {f}", got, T[f], cnt))
                del x
            if s > 0:
                for f in ("n_query", "n_valid", "n_pv"):
                    np.testing.assert_array_equal(res[f], T[f].cpu().numpy(), err_msg=f"{name} {side} {f}")
                has = res["n_pv"] > 0
                np.testing.assert_array_equal(res["max_pv"][has].view(np.int64),
                                              T["max_pv"].cpu().numpy()[has].view(np.int64))
            cv[s] = dict(regions=nseg, worst_sum=worst)
            del T, seg
        # n_valid against MME on the same cloud
        res0, e_p, v_p = cons[(which, 0.0)]
        ent_t = torch.from_numpy(ent).to(dev)
        diff = torch.nonzero((ent_t != 0) != (e_p != 0)).reshape(-1).cpu().numpy()
        assert macc.n_valid == int((ent_t != 0).sum())
        # each point whose validity differs from MME's: its exact determinant is one B64 + B32(E) of MME's fp32-offset
        # sweep cannot decide (B32 infinite: the certificate does not hold)
        assert len(diff) <= 2000, (name, side, len(diff), "points whose validity differs from MME's")
        if len(diff):
            qd, nbd = F.ball_neighbours(cloud, diff, r)
            exd = F.mme_sample_exact(qd, nbd, m)
            E = F.sweep_offsets(trace_nn, r, float(cloud.abs().max()))
            for i, exi in zip(diff, exd):
                assert exi["cov"] is not None, (name, side, int(i), exi["k"])
                b32 = 0.0 if E is None else math.inf if E == "unknown" else \
                    X.mme_fp32_certificate(exi["cov"], exi["k"], E)
                assert not exi["determined"] or b32 == math.inf, (name, side, int(i), exi["k"], b32)
        # the sample: validity, e within B64, v within fp64_bound of lambda3; the teeth
        mq, qh, nbs, exs = _mme_sample(torch, cloud, r, m, SETUP[name], 20 + which)
        e_h, v_h = e_p.cpu().numpy(), v_p.cpu().numpy()
        cs = _mme_check(e_h, mq, exs, None)
        lam = F.consistency_sample_exact(qh, nbs, exs, m)
        worst_v, bite_k, bite_max, n_v = 0.0, 0, 0, 0
        lam_k = F.consistency_sample_exact(qh, nbs, exs, m, divisor_k=True)
        lam_max = F.consistency_sample_exact(qh, nbs, exs, m, largest=True)
        for t, i in enumerate(mq):
            (l3, b), got = lam[t], float(v_h[i])
            if math.isnan(l3):
                assert math.isnan(got), (name, side, int(i), got)
                continue
            assert abs(got - l3) <= b, (name, side, int(i), got, l3, b)
            worst_v = max(worst_v, abs(got - l3) / b if b > 0 else 0.0)
            n_v += 1
            bite_k += abs(got - lam_k[t][0]) > lam_k[t][1]
            bite_max += abs(got - lam_max[t][0]) > lam_max[t][1]
        # both wrong variants break the bound on every valid sampled query
        assert n_v > 0 and bite_k == n_v and bite_max == n_v, (name, side, n_v, bite_k, bite_max)
        cv["sample"] = dict(cs, worst_v=worst_v, n_valid_vs_mme=len(diff), teeth_k=bite_k, teeth_max=bite_max)
        # GT-side MME (m = 5) on its own sample, as test_gpu_fullsize_large.py step 4
        if which == GT:
            assert macc.n_query == n_gt and macc.n_valid == int((ent_t != 0).sum())
            s_ex = F.exact_sum_t(ent_t)
            s_abs = float(F.exact_sum_t(ent_t.abs()))
            assert abs(macc.sum_entropy - float(s_ex)) <= n_gt * X.U * s_abs, (macc.sum_entropy, float(s_ex))
            E = F.sweep_offsets(trace_nn, r, float(gt.abs().max()))
            mq2, _, _, exs2 = _mme_sample(torch, gt, r, 5, SETUP[name], 40)
            covered["gt_mme"] = _mme_check(ent, mq2, exs2, E)
        covered["consistency"][side] = cv
        del ent_t, e_p, v_p
        meter.sample()
    cons_sweeps = {k: (c[0]["kernel"], c[0]["whole"]["rings"], c[0]["whole"]["solo"]) for k, c in cons.items()}
    del cons

    # ---- the paths that ran -----------------------------------------------------------------------------------------
    expect = {"ME_KBIT_NN_ROWS_SPARSE", "ME_KBIT_NN_FAR", "ME_KBIT_MME_SOLO",
              "ME_KBIT_MME_FLAT2_SPARSE" if name == "S1" else "ME_KBIT_MME_FLAT2_DENSE"}
    covered["trace"] = dict(nn=sorted(trace_nn), surface=sorted(trace_pass), consistency=sorted(trace_cons))
    del est, gt
    torch.cuda.empty_cache()
    wall = time.time() - meter.t0
    host_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    print(f"\n{name}: {n_est} est vs {n_gt} gt; wall {wall:.0f} s (pass {t_pass:.0f} s); device peak "
          f"{meter.peak / 2 ** 30:.1f} GB beyond the start; host max RSS {host_gb:.1f} GB; covered {covered}")
    # the MME sweeps of both clouds and the NN pass (the trace is reset when read).  The normals' exact k-NN walk sets no
    # sweep bit, and on these clouds no query leaves its fine rings (no ME_TEV_KNN_COARSE).  local_consistency sets no bit
    # by design (§3.15): its result names the sweep, which is MME's choice, the walk on a solo lattice with two rings.
    assert set(trace_nn) == expect, sorted(trace_nn)
    assert set(trace_pass) == set(), sorted(trace_pass)
    assert set(trace_cons) == set(), sorted(trace_cons)
    for (which, s), res in cons_sweeps.items():
        assert res == ("WALK", 2, 1), (name, which, s, res)
