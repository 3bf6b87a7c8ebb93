"""CPU-side checks of the drop-in boundary: the shared library loads, exports exactly the symbols the header
declares, the ctypes mirrors match the C struct sizes, and the host-only finalisers agree with the oracle's
restatement of the reference formulas (no GPU compute is called here)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from cloud_map_evaluation_b200 import _abi as A
from cloud_map_evaluation_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return _lib.load()


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "mapeval_b200.h")).read()
    return sorted(set(re.findall(r"^ME_API\s+[\w\s\*]+?\b(me_[a-z_0-9]+)\s*\(", text, flags=re.M)))


def test_header_and_library_export_the_same_symbols(L):
    declared = _header_symbols()
    assert declared == sorted(_lib.SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = sorted(s for s in re.findall(r" T (me_[a-z_0-9]+)", out))
    assert exported == declared
    for s in declared:
        assert hasattr(L, s)


def test_struct_sizes_match_the_header(tmp_path):
    src = tmp_path / "sz.c"
    names = ["me_options", "me_nn_params", "me_nn_accum", "me_dir_result", "me_nn_result", "me_mme_accum",
             "me_mme_result", "me_awd_result"]
    src.write_text('#include <stdio.h>\n#include "mapeval_b200.h"\nint main(){' +
                   "".join(f'printf("%zu\\n", sizeof({n}));' for n in names) + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert sizes == [C.sizeof(getattr(A, n)) for n in names]
    assert C.sizeof(A.me_nn_accum) == 8 * (A.ME_NN_ACCUM_I64 + A.ME_NN_ACCUM_F64)


def test_kernel_bit_enum_mirror_matches_the_header():
    """enum me_kernel_bit of the header and its ctypes mirror: the same names with the same values, one bit each, dense
    from 0 to ME_KBIT_COUNT - 1 (the kernel-path tests generate their cases from the mirror)."""
    text = open(os.path.join(ROOT, "include", "mapeval_b200.h")).read()
    body = re.search(r"enum\s+me_kernel_bit\s*\{(.*?)\};", text, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    declared = {k: int(v) for k, v in re.findall(r"\b(ME_KBIT_\w+)\s*=\s*(\d+)", body)}
    assert len(declared) == body.count("=")      # every entry carries an explicit value
    count = declared.pop("ME_KBIT_COUNT")
    assert declared == A.KERNEL_BITS
    assert sorted(declared.values()) == list(range(count)) and count == A.ME_KBIT_COUNT
    assert A.kernel_bit_names((1 << A.ME_KBIT_NN_TILE) | (1 << A.ME_KBIT_SCS_R5)) == {"ME_KBIT_NN_TILE", "ME_KBIT_SCS_R5"}


def test_trace_event_enum_mirror_matches_the_header():
    """enum me_trace_event of the header and its ctypes mirror: the same names with the same values, above the sweep bits
    and inside the 32-bit device word; kernel_bit_names leaves them out."""
    text = open(os.path.join(ROOT, "include", "mapeval_b200.h")).read()
    body = re.search(r"enum\s+me_trace_event\s*\{(.*?)\};", text, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    declared = {k: int(v) for k, v in re.findall(r"\b(ME_TEV_\w+)\s*=\s*(\d+)", body)}
    assert declared and len(declared) == body.count("=")
    assert declared == A.TRACE_EVENTS
    assert all(A.ME_KBIT_COUNT <= v < 32 for v in declared.values())
    mask = (1 << A.ME_KBIT_MME_SOLO) | (1 << A.ME_TEV_MME_FP64_FINISH)
    assert A.kernel_bit_names(mask) == {"ME_KBIT_MME_SOLO"}
    assert A.trace_event_names(mask) == {"ME_TEV_MME_FP64_FINISH"}


def test_no_cpu_fallback_without_a_device(L):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    opt = A.me_options()
    opt.abi_version, opt.world = A.ME_ABI_VERSION, 1
    ctx = C.c_void_p()
    assert L.me_create(C.byref(opt), C.byref(ctx)) == A.ME_ERR_NO_DEVICE
    assert b"no CPU path" in L.me_last_error(None)
    opt.abi_version = 99
    assert L.me_create(C.byref(opt), C.byref(ctx)) == A.ME_ERR_INVALID


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "cloud_map_evaluation_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in text.lower().replace("no cpu", ""), f"{f} mentions the oracle"


def test_finalizers_match_the_reference_formulas(L):
    """me_nn_finalize / me_mme_finalize (host only) against accumulators computed with numpy."""
    from oracle import oracle as O
    from cloud_map_evaluation_b200 import synth
    est, gt, cfg = synth.make_pair("C1", scale=0.05)
    tau = cfg["tau"]
    p = A.make_nn_params(tau, 1.0, pairing=A.ME_PAIRING_GEOMETRIC)
    exp = O.eval_nn(est, gt, p)
    accs = []
    for q, r in ((est, gt), (gt, est)):
        idx, d2 = O.knn1(q, r)
        keep = d2 <= 1.0
        d = q[keep] - r[idx[keep]]
        sq = d[:, 0] ** 2 + (d[:, 1] ** 2 + d[:, 2] ** 2)
        nd = np.sqrt(sq)
        a = A.me_nn_accum()
        a.n_query, a.n_corr = len(q), int(keep.sum())
        for k, t in enumerate(tau):
            m = nd <= t
            a.n_inlier[k], a.sum_d[k], a.sum_d2[k] = int(m.sum()), nd[m].sum(), sq[m].sum()
        a.sum_d_all, a.sum_d2_all, a.sum_nn_dist = nd.sum(), sq.sum(), np.sqrt(d2).sum()
        accs.append(a)
    out = A.me_nn_result()
    assert L.me_nn_finalize(C.byref(p), C.byref(accs[0]), C.byref(accs[1]), len(est), len(gt), C.byref(out)) == 0
    for d in ("est_to_gt", "gt_to_est"):
        g, e = getattr(out, d), getattr(exp, d)
        assert list(g.n_inlier) == list(e.n_inlier) and g.n_corr == e.n_corr
        for k in ("mean", "rmse", "fitness", "sigma"):
            np.testing.assert_allclose(list(getattr(g, k)), list(getattr(e, k)), rtol=1e-9, err_msg=k)
    for k in ("cd", "f1", "iou"):
        np.testing.assert_allclose(list(getattr(out, k)), list(getattr(exp, k)), rtol=1e-9)
    np.testing.assert_allclose(out.full_cd, exp.full_cd, rtol=1e-12)

    m = A.me_mme_accum()
    m.n_query, m.n_valid, m.sum_entropy, m.min_entropy, m.max_entropy = 10, 4, -32.0, -9.5, -6.25
    r = A.me_mme_result()
    assert L.me_mme_finalize(C.byref(m), 10, C.byref(r)) == 0
    assert (r.mme, r.n_valid, r.n_total, r.min_abs_entropy, r.max_abs_entropy) == (-8.0, 4, 10, 6.25, 9.5)
    m.n_valid, m.sum_entropy, m.min_entropy, m.max_entropy = 0, 0.0, np.inf, -np.inf
    assert L.me_mme_finalize(C.byref(m), 10, C.byref(r)) == 0
    assert r.mme == 0.0 and np.isnan(r.min_abs_entropy)


def test_finalizer_merges_the_rank_moments(L):
    """me_nn_finalize on per-rank (n, mean, M2) slots: sigma from the merged moments, to the exact two-pass value, where the
    closed form on sum(d) and sum(d^2) of the same distances loses it to cancellation (a cluster 1e-9 m wide around
    2.6 cm, split over three ranks)"""
    from fractions import Fraction
    rng = np.random.RandomState(4)
    nd = 0.026 + 1e-9 * rng.rand(3000)
    tau = [1.0, 0.026 + 5e-10, 0.02, 1.0, 1.0]
    a = A.me_nn_accum()
    a.n_query = a.n_corr = len(nd)
    for k, t in enumerate(tau):
        m = nd <= t
        a.n_inlier[k], a.sum_d[k], a.sum_d2[k] = int(m.sum()), nd[m].sum(), (nd[m] ** 2).sum()
    a.sum_d_all, a.sum_d2_all = nd.sum(), (nd ** 2).sum()
    for r, part in enumerate(np.array_split(nd, 3)):
        a.rank_n[5 * r], a.rank_mean[5 * r] = len(part), part.mean()
        a.rank_m2[5 * r] = ((part - part.mean()) ** 2).sum()
    p = A.make_nn_params(tau, 1.0, pairing=A.ME_PAIRING_GEOMETRIC, directions=1)
    out = A.me_nn_result()
    assert L.me_nn_finalize(C.byref(p), C.byref(a), None, len(nd), 1, C.byref(out)) == 0
    F = [Fraction(x) for x in nd]
    for k in range(5):
        mean = Fraction(out.est_to_gt.mean[k])
        exact = float(sum((f - mean) ** 2 for f in F) / len(F)) ** 0.5
        assert abs(out.est_to_gt.sigma[k] - exact) <= 1e-10 * exact + 1e3 * 2.0 ** -53 * 0.026, k
    # the same accumulator without its moments falls back to the closed form, which is far off here
    for r in range(3):
        a.rank_n[5 * r] = a.rank_mean[5 * r] = a.rank_m2[5 * r] = 0.0
    assert L.me_nn_finalize(C.byref(p), C.byref(a), None, len(nd), 1, C.byref(out)) == 0
    assert abs(out.est_to_gt.sigma[0] - exact) > 1e3 * 2.0 ** -53 * 0.026
