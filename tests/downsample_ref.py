"""numpy statement of VoxelDownSample (me_voxel_downsample), with and without normals, and the scenes that check it
(not collected as a test module):

* origin   org = min − s·0.5 per axis, in IEEE fp64 (the min over the whole cloud);
* keys     floor((p − org) / s) per axis, IEEE fp64 subtraction and division;
* order    voxels in increasing (ix, iy, iz), the library's order;
* sums     per voxel, the points (and the normals without a NaN component) summed sequentially in INPUT order from +0.0,
           then divided by the count of all the voxel's points.

Every sum is one sequential fp64 chain, so the statement is bit-exact: never np.sum / np.add.reduceat / np.add.at on a
run (they may sum pairwise).  The members of the voxels up to LONG_RUN points are added rank by rank (the r-th member of
every voxel in one vector step); a longer voxel is summed by np.cumsum over its run, which is sequential by definition.
tests/test_downsample_reference.py checks the statement against a plain Python loop and the oracle, and that the scenes
below can tell a right kernel from a wrong one; tests/test_gpu_downsample.py checks the device against it.
"""
from fractions import Fraction

import numpy as np

AXIS_BITS = 21          # downsample.cu: voxel indices per axis below 2^21
LONG_RUN = 1024         # voxels with more members are summed by np.cumsum over their run


def voxel_keys(xyz, s):
    """(N, 3) int64 voxel indices and the origin org = min − s·0.5"""
    xyz = np.asarray(xyz, dtype=np.float64)
    org = xyz.min(0) - s * 0.5
    return np.floor((xyz - org) / s).astype(np.int64), org


def key_bits(xyz, s):
    """bits per axis of the library's packed key (downsample.cu, voxel_downsample): floor((max − org) / s) + 3 voxels
    (two of slack), the smallest b with 2^b >= that; None where the library refuses the cloud (2^21 voxels or more)"""
    xyz = np.asarray(xyz, dtype=np.float64)
    mn, mx = xyz.min(0), xyz.max(0)
    bits = []
    for a in range(3):
        org = float(mn[a]) - s * 0.5
        nv = np.floor((float(mx[a]) - org) / s) + 3.0
        if not nv < float(1 << AXIS_BITS):
            return None
        b = 1
        while (1 << b) < int(nv):
            b += 1
        bits.append(b)
    return bits


def radix_passes(bits):
    """8-bit digits the LSD radix sort runs over a key of sum(bits) bits"""
    return -(-sum(bits) // 8)


def _sequential_sums(src, start, cnt):
    """(V, 3): for each voxel v the sequential sum from +0.0 of src[start[v] : start[v] + cnt[v]]"""
    out = np.zeros((len(start), 3))
    short = np.flatnonzero(cnt <= LONG_RUN)
    byc = short[np.argsort(-cnt[short], kind="stable")]      # largest first: voxels with more than r members are a prefix
    neg = -cnt[byc]
    for r in range(int(cnt[byc[0]]) if len(byc) else 0):
        v = byc[:np.searchsorted(neg, -r, side="left")]
        out[v] += src[start[v] + r]
    for v in np.flatnonzero(cnt > LONG_RUN):
        # cumsum starts from the first member, not from +0.0: 0.0 + (...) makes an all −0.0 run +0.0 as the chain from
        # +0.0 gives (any other run has the same value either way)
        out[v] = 0.0 + np.cumsum(src[start[v]:start[v] + cnt[v]], axis=0)[-1]
    return out


def voxel_downsample(xyz, s, normals=None):
    """(points, normals or None, counts) of VoxelDownSample(s), voxels in increasing (ix, iy, iz)"""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64)
    n = len(xyz)
    k, _ = voxel_keys(xyz, s)
    assert k.min() >= 0 and k.max() < (1 << AXIS_BITS)
    order = np.argsort((k[:, 0] << (2 * AXIS_BITS)) | (k[:, 1] << AXIS_BITS) | k[:, 2], kind="stable")
    ks = k[order]
    start = np.flatnonzero(np.r_[True, (ks[1:] != ks[:-1]).any(1)])
    cnt = np.diff(np.r_[start, n])
    c = cnt.astype(np.float64)[:, None]
    pts = _sequential_sums(xyz[order], start, cnt) / c
    if normals is None:
        return pts, None, cnt
    nrm = np.asarray(normals, dtype=np.float64)[order]
    # a normal with a NaN component is skipped; adding +0.0 instead leaves a chain that starts at +0.0 unchanged
    nrm = np.where(np.isnan(nrm).any(1, keepdims=True), 0.0, nrm)
    return pts, _sequential_sums(nrm, start, cnt) / c, cnt


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
def rounds_up(x, org, s):
    """x − org < k·s in exact arithmetic, but floor((x − org) / s) = k in IEEE fp64"""
    k = int(np.floor((x - org) / s))
    return Fraction(float(x)) - Fraction(float(org)) < k * Fraction(s)


def face_values(base, s, near=200, keep=2000):
    """values along one axis whose minimum is `base`: the first `near` faces org + k·s (fp64) and one ulp either side of
    them; among the faces up to 400 m out (40 000 at most) and their neighbours, up to `keep` whose quotient rounds up to
    k and up to `keep` that a multiplication by 1/s puts in another voxel than the division; at the origin also −0.0 next
    to +0.0.  Returns (values, the round-up values)."""
    org = base - s * 0.5
    on = org + np.arange(1, int(min(400.0 / s, 40_000)) + 1) * s
    cand = np.concatenate([on, np.nextafter(on, -np.inf), np.nextafter(on, np.inf)])
    q = (cand - org) / s
    up = np.array([x for x in cand[q == np.floor(q)] if rounds_up(x, org, s)])      # a round-up lands on k exactly
    recip = cand[np.floor((cand - org) * (1.0 / s)) != np.floor(q)]
    first = on[:near]
    extra = [-0.0, 0.0] if base == 0.0 else [base]
    return np.concatenate([extra, first, np.nextafter(first, -np.inf), np.nextafter(first, np.inf),
                           up[::max(1, len(up) // keep)], recip[::max(1, len(recip) // keep)]]), up


def face_scene(base, s, n=20_000, seed=0):
    """points whose coordinates are drawn from face_values on every axis (the min point included, so org is known)"""
    rng = np.random.RandomState(seed)
    vals, _ = face_values(base, s)
    pts = np.stack([rng.choice(vals, n) for _ in range(3)], 1)
    pts[0] = base
    return pts


def order_scene(n_vox=6000, seed=0, base=(1500.0, -1500.0, 1500.0), s=0.01, layout="spread"):
    """n_vox voxels of 3–50 members with random low bits 1.5 km out, where the rounding of a voxel's sum depends on the
    order of its members, and single-point voxels that fill the gaps.  layout: "spread" puts member j of voxel v at
    j·n_vox + v (the members of a voxel are n_vox places apart: different sort tiles, warps and 32-key chunks),
    "shuffled" permutes that cloud, "contiguous" keeps each voxel's members together.  The first point is the min.
    Returns (points, normals)."""
    rng = np.random.RandomState(seed)
    base = np.asarray(base, dtype=np.float64)
    cnt = rng.randint(3, 51, n_vox)
    n_fill = 50 * n_vox - cnt.sum()
    side = int(np.ceil((n_vox + n_fill) ** (1 / 3))) + 1
    cell = rng.permutation(side ** 3)[:n_vox + n_fill]
    ijk = np.stack([cell // (side * side), (cell // side) % side, cell % side], 1) + 1
    # voxel k spans [org + k s, org + (k + 1) s) with org = base − s/2: its centre is base + k s
    vox = np.concatenate([np.repeat(np.arange(n_vox), cnt), n_vox + np.arange(n_fill)])
    pts = base + ijk[vox] * s + rng.uniform(-0.45 * s, 0.45 * s, (len(vox), 3))
    nrm = rng.randn(len(vox), 3)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    if layout != "contiguous":
        rank = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        slot = np.ones((50, n_vox), bool)
        slot[rank, vox[:cnt.sum()]] = False                 # slot (j, v) of a member; the free slots take the fillers
        where = np.empty(len(vox), np.int64)
        where[:cnt.sum()] = rank * n_vox + vox[:cnt.sum()]
        where[cnt.sum():] = np.flatnonzero(slot.reshape(-1))
        p = np.argsort(where)
        if layout == "shuffled":
            p = p[rng.permutation(len(p))]
        pts, nrm = pts[p], nrm[p]
    return np.concatenate([base[None], pts]), np.concatenate([[[0.0, 0.0, 1.0]], nrm])
