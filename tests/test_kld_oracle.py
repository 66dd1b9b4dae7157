"""The glibc oracle's resample_adaptive (oracle/pf_oracle.c) against the independent pure-Python restatement of
tests/golden/make_golden.py on every adversarial KLD case (tests/_kld_cases.py), bit for bit: the stopping length, the
ancestor of every draw and every particle.  make_golden's mcl_resample_adaptive runs itself on every case with finite poses
and a small cloud; a line-for-line copy that accepts NaN and +-inf poses and a faster search covers the rest, and it is held
to make_golden's bits wherever both run.  The GPU test (tests/test_gpu_kld.py) takes the oracle as its reference on the same
clouds, so this is what makes that reference trustworthy there.  Both sides draw r_t = U53(seed, PF_RESAMPLE, 0, t)."""
import bisect
import math
import os
import sys

import numpy as np
import pytest

import _kld_cases as K
from _oracle import OraclePF

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden as MG  # noqa: E402


def lower_bound(cum, r):
    """first i < len - 1 with r <= c_i, else len - 1: the linear scan's answer when cum[:-1] does not go down"""
    return bisect.bisect_left(cum, r, 0, len(cum) - 1)


def linear_scan(cum, r):
    """mcl.rs:387-392 as written: the first i with r <= c_i, else len - 1"""
    for i, cw in enumerate(cum):
        if r <= cw:
            return i
    return len(cum) - 1


def floor_as_i32(v):
    """`v.floor() as i32`: make_golden's saturating cast after a floor that leaves NaN and +-inf as they are"""
    return MG.sat_i32(math.floor(v) if math.isfinite(v) else v)


def resample_adaptive(ps, nmin, nmax, eps, z, rs, search):
    """make_golden.mcl_resample_adaptive with two changes it cannot take as written: a pose may be NaN or +-inf (its
    math.floor raises there), and a large cloud needs a faster search than the linear scan.  Every other line is the same,
    kld_required and sat_i32 are make_golden's own, and on every case make_golden can run, both give the same bits."""
    cum = []
    c = 0.0
    for p in ps:
        c += p.w
        cum.append(c)
    cum[-1] = 1.0
    bins = set()
    new, idxs = [], []
    required = nmin
    while len(new) < nmax:
        idx = search(cum, rs[len(new)])
        s = ps[idx]
        bins.add((floor_as_i32(s.x / 0.5), floor_as_i32(s.y / 0.5), floor_as_i32(s.yaw / (15.0 * MG.PI / 180.0))))
        required = max(required, MG.kld_required(len(bins), nmin, nmax, eps, z))
        new.append(s.clone())
        idxs.append(idx)
        if len(new) >= nmin and len(new) >= required:
            break
    uw = 1.0 / float(len(new))
    for p in new:
        p.w = uw
    return new, idxs


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def oracle_for(L, c, fast):
    o = OraclePF(L, c.n_min, seed=c.seed, mode=1, max_particles=c.n_max, kld_epsilon=c.eps, kld_z=c.z)
    o.L.orc_pf_set_fast_search(o.h, int(fast))
    return o


def as_arrays(new, idxs):
    return np.array([p.row() for p in new]), np.array(idxs, dtype=np.uint32)


def restated(c, cloud, r):
    """make_golden.mcl_resample_adaptive itself where it can run (finite poses, small clouds); resample_adaptive elsewhere"""
    ps = lambda: [MG.P(*row) for row in cloud.tolist()]    # noqa: E731
    if c.big:
        cum = np.add.accumulate(cloud[:, 4])
        assert c.monotone and np.all(np.diff(cum[:-1]) >= 0.0)
        return as_arrays(*resample_adaptive(ps(), c.n_min, c.n_max, c.eps, c.z, r, lower_bound))
    mine = as_arrays(*resample_adaptive(ps(), c.n_min, c.n_max, c.eps, c.z, r, linear_scan))
    if np.all(np.isfinite(cloud[:, :3])):
        want = as_arrays(*MG.mcl_resample_adaptive(ps(), c.n_min, c.n_max, c.eps, c.z, r))
        assert np.array_equal(bits(mine[0]), bits(want[0])) and np.array_equal(mine[1], want[1]), c.name
    return mine


@pytest.mark.parametrize("name", [c.name for c in K.CASES])
def test_oracle_resample_adaptive_matches_restatement(oracle_libm, name):
    c = K.BY_NAME[name]
    cloud = c.cloud(oracle_libm)
    o = oracle_for(oracle_libm, c, fast=c.big)
    o.set_particles(cloud)
    o.resample()
    want, want_idx = restated(c, cloud, K.draws(oracle_libm, c.seed, c.n_max))
    n = o.count()
    if c.expect is not None:
        assert n == c.expect, f"{name}: the oracle stops at {n}, the case was built for {c.expect}"
    assert n == want.shape[0], f"{name}: count {n} vs restatement {want.shape[0]}"
    assert np.array_equal(o.last_indices(), want_idx), name
    assert np.array_equal(bits(o.particles()), bits(want)), name
    assert np.all(o.particles()[:, 4] == 1.0 / n)


@pytest.mark.parametrize("name", [c.name for c in K.CASES if c.monotone and not c.big])
def test_oracle_lower_bound_equals_linear_scan(oracle, name):
    """the GPU tests run the contract-math oracle with its lower-bound search on clouds with a non-decreasing CDF: on every such
    case it gives the linear scan's count, ancestors and particles"""
    c = K.BY_NAME[name]
    cloud = c.cloud(oracle)
    out = []
    for fast in (0, 1):
        o = oracle_for(oracle, c, fast)
        o.set_particles(cloud)
        o.resample()
        out.append((o.count(), o.last_indices(), bits(o.particles())))
    assert out[0][0] == out[1][0]
    assert np.array_equal(out[0][1], out[1][1]) and np.array_equal(out[0][2], out[1][2])


def test_cases_hit_their_structure(oracle):
    """the cases are what their names say: distinct keys, colliding slots at the handle's table size, chunk-boundary targets"""
    h = K.BY_NAME["hash_collisions"]
    a = h.cloud()
    keys = [K.key(*row[:3]) for row in a]
    assert len(set(keys)) == h.n_min
    tcap = K.table_size(h.n_max)
    assert tcap == 4096
    slots = K.bin_hash(*np.array(keys).T) & np.uint32(tcap - 1)
    assert np.sum(slots == tcap - 1) >= 128 and np.sum(slots == 5) >= 64
    same_ab = [k for k, s in zip(keys, slots) if s == tcap - 1 and k[:2] == (1234, -77)]
    assert len(same_ab) >= 64
    q = K.BY_NAME["quantiser_edges"].cloud()
    qk = [K.key(*row[:3]) for row in q]
    assert (2147483647, 0, 0) in qk and (-2147483648, 0, 0) in qk and (0, 0, 0) in qk
    assert K.key(2.0 ** 30 - 0.5, 0.0, 0.0)[0] == 2147483647 and K.key(-2.0 ** 30, 0.0, 0.0)[0] == -2147483648
    assert K.key(float("nan"), 0.0, 0.0) == K.key(0.25, 0.0, 0.0) == K.key(-0.0, 0.0, 0.0)
    assert K.key(0.0, 0.0, 1e300)[2] == 2147483647 and K.key(0.0, 0.0, -1e3)[2] == -3820
    for c in K.CASES:                                    # the stop_* parameters still hit their targets under the plain rule
        if c.name.startswith("stop_"):
            ks = K.bins_after_each_draw(c.cloud(), K.draws(oracle, c.seed, c.n_max))
            assert K.stop_length(ks, c.n_min, c.n_max, c.eps, c.z) == c.expect, c.name
