"""Independent numpy restatement of the pose-hypothesis contract (include/pfgpu.h pfgpu_pf_hypotheses, DESIGN §3.10): bins from
single IEEE operations, components from scipy.sparse.csgraph.connected_components over explicitly listed neighbour pairs, and
two-pass f64 moments.  Also a plain-Python BFS of the components, the cross-check of the first.  Test infrastructure only."""
import collections
import math

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

TWO_PI = 6.283185307179586
I32_MAX, I32_MIN = 2 ** 31 - 1, -2 ** 31

Hyp = collections.namedtuple("Hyp", ["mass", "count", "bins", "label", "mean", "cov"])


def sat_i32(v):
    """Rust's `as i32` of an f64 array: saturating, NaN -> 0"""
    v = np.asarray(v, dtype=np.float64)
    out = np.where(np.isnan(v), 0.0, np.clip(v, I32_MIN, I32_MAX))
    return np.trunc(out).astype(np.int64)


def members(aos5):
    p = np.asarray(aos5, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        return np.isfinite(p[:, :4]).all(axis=1) & (p[:, 4] > 0.0) & (p[:, 4] < np.inf)


def bin_keys(aos5, xy_res, yaw_bins):
    """(n, 3) int64 keys (kx, ky, kt); rows of non-members are meaningless"""
    p = np.asarray(aos5, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        kx = sat_i32(np.floor(p[:, 0] / xy_res))
        ky = sat_i32(np.floor(p[:, 1] / xy_res))
        m = TWO_PI * np.floor(p[:, 2] / TWO_PI)
        theta = p[:, 2] - m
        q = np.floor(theta / (TWO_PI / yaw_bins))
        kt = np.where(~(q >= 0.0), 0.0, np.where(q > yaw_bins - 1, yaw_bins - 1, q)).astype(np.int64)
    return np.stack([kx, ky, kt], axis=1)


def offsets():
    return [(dx, dy, dt) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dt in (-1, 0, 1) if (dx, dy, dt) != (0, 0, 0)]


def bin_components(keys, yaw_bins):
    """keys (B, 3) of the distinct occupied bins -> component id of each bin (connected_components over listed pairs)"""
    B = keys.shape[0]
    ux, uy = np.unique(keys[:, 0]), np.unique(keys[:, 1])
    ix, iy = np.searchsorted(ux, keys[:, 0]), np.searchsorted(uy, keys[:, 1])
    code = (ix * len(uy) + iy) * yaw_bins + keys[:, 2]
    order = np.argsort(code)
    scode = code[order]
    rows, cols = [np.arange(B)], [np.arange(B)]
    for dx, dy, dt in offsets():
        nx, ny = keys[:, 0] + dx, keys[:, 1] + dy
        nt = (keys[:, 2] + dt) % yaw_bins
        ok = (nx >= I32_MIN) & (nx <= I32_MAX) & (ny >= I32_MIN) & (ny <= I32_MAX)
        jx, jy = np.searchsorted(ux, nx), np.searchsorted(uy, ny)
        ok &= (jx < len(ux)) & (jy < len(uy))
        ok &= np.where(ok, ux[np.minimum(jx, len(ux) - 1)] == nx, False) & np.where(ok, uy[np.minimum(jy, len(uy) - 1)] == ny, False)
        nc = (jx * len(uy) + jy) * yaw_bins + nt
        pos = np.searchsorted(scode, nc)
        ok &= pos < B
        ok &= np.where(ok, scode[np.minimum(pos, B - 1)] == nc, False)
        rows.append(np.flatnonzero(ok))
        cols.append(order[pos[ok]])
    r, c = np.concatenate(rows), np.concatenate(cols)
    g = coo_matrix((np.ones(r.size, dtype=np.int8), (r, c)), shape=(B, B)).tocsr()
    return connected_components(g, directed=False)[1]


def wrap(a):
    """into [-pi, pi): a - T floor((a + pi) / T)"""
    return a - TWO_PI * np.floor((a + math.pi) / TWO_PI)


def hypotheses(aos5, xy_res=0.5, yaw_bins=24):
    """([Hyp] in contract order, rank per particle (-1: not a member))"""
    p = np.asarray(aos5, dtype=np.float64).reshape(-1, 5)
    n = p.shape[0]
    mem = members(p)
    rank = np.full(n, -1, dtype=np.int64)
    idx = np.flatnonzero(mem)
    if idx.size == 0:
        return [], rank
    keys = bin_keys(p[idx], xy_res, yaw_bins)
    ubins, binof = np.unique(keys, axis=0, return_inverse=True)
    binof = binof.reshape(-1)
    comp = bin_components(ubins, yaw_bins)[binof]
    ncomp = comp.max() + 1
    label = np.full(ncomp, n, dtype=np.int64)
    np.minimum.at(label, comp, idx)
    o = np.argsort(comp, kind="stable")                      # members grouped by component, in slot order
    cs, q = comp[o], p[idx[o]]
    starts = np.flatnonzero(np.r_[True, cs[1:] != cs[:-1]])
    w = q[:, 4]

    def seg(a):
        return np.add.reduceat(a, starts)

    M = seg(w)
    ss, sc = seg(w * np.sin(q[:, 2])), seg(w * np.cos(q[:, 2]))
    mean = np.stack([seg(w * q[:, 0]) / M, seg(w * q[:, 1]) / M, np.where((ss == 0.0) & (sc == 0.0), 0.0, np.arctan2(ss, sc)),
                     seg(w * q[:, 3]) / M], axis=1)
    mc = mean[cs]
    d = np.stack([q[:, 0] - mc[:, 0], q[:, 1] - mc[:, 1], wrap(q[:, 2] - mc[:, 2]), q[:, 3] - mc[:, 3]], axis=1)
    cov = np.empty((ncomp, 4, 4))
    for a in range(4):
        for b in range(a, 4):
            cov[:, a, b] = cov[:, b, a] = seg(w * d[:, a] * d[:, b]) / M
    count = np.diff(np.r_[starts, cs.size])
    pairs = np.unique(np.stack([comp, binof], axis=1), axis=0)
    bins = np.bincount(pairs[:, 0], minlength=ncomp)
    order = np.lexsort((label, -M))
    rk = np.empty(ncomp, dtype=np.int64)
    rk[order] = np.arange(ncomp)
    rank[idx] = rk[comp]
    return [Hyp(float(M[c]), int(count[c]), int(bins[c]), int(label[c]), mean[c], cov[c]) for c in order], rank


def bfs_components(aos5, xy_res=0.5, yaw_bins=24):
    """plain-Python BFS over the occupied bins: {label: sorted member slots}"""
    p = np.asarray(aos5, dtype=np.float64).reshape(-1, 5)
    mem = members(p)
    keys = bin_keys(p, xy_res, yaw_bins)
    bins = collections.defaultdict(list)
    for t in np.flatnonzero(mem):
        bins[tuple(int(v) for v in keys[t])].append(int(t))
    seen, out = set(), {}
    for b in bins:
        if b in seen:
            continue
        seen.add(b)
        queue, comp = [b], []
        while queue:
            x, y, k = queue.pop()
            comp += bins[(x, y, k)]
            for dx, dy, dt in offsets():
                nb = (x + dx, y + dy, (k + dt) % yaw_bins)
                if nb in bins and nb not in seen:
                    seen.add(nb)
                    queue.append(nb)
        out[min(comp)] = sorted(comp)
    return out
