"""Worker of tests/test_gpu_hypotheses.py::test_hypotheses_multi_process: one process per GPU (torchrun).  A sharded
MonteCarloLocalizer with augmented MCL steps through scans from a region start; after every step each rank queries the pose
hypotheses.  Every rank must return the same bytes, and a single-GPU handle loaded with the gathered global set must return them too,
with this rank's slice of the per-slot ranks."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import api, dist as rdist, scenarios  # noqa: E402

CAP = 64


def query(g, n_local):
    """(the raw hypothesis records, total, per-slot ranks) of one call"""
    out, tot, rk = (api._Hyp * CAP)(), C.c_size_t(), np.empty(n_local, dtype=np.uint32)
    rc = g.L.pfgpu_pf_hypotheses(g.h, 0.5, 24, out, CAP, C.byref(tot), rk.ctypes.data_as(api.c_u32p))
    assert rc == 0, rc
    return bytes(out)[:min(CAP, tot.value) * C.sizeof(api._Hyp)], tot.value, rk


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.ScanScenario(steps=steps)
    cfg = rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1)
    g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, cfg, seed=5, device=local, shard=(uid, rank, world))
    g.set_likelihood_field(sc.obstacles, sc.RES)
    g.enable_recovery(0.1, 0.6, sc.REGION)
    single = rr.MonteCarloLocalizer(cfg, seed=5, device=local)
    lo, hi = rdist.shard_bounds(n, rank, world)
    allgather = lambda b: grp._exchange(b, lambda parts: b"".join(parts))       # noqa: E731
    for t in range(steps):
        g.try_step_scan(sc.controls[t], *sc.scan_args(t))
        recs, total, rk = query(g, hi - lo)
        assert query(g, hi - lo)[0] == recs, f"rank {rank} step {t}: two calls differ"
        everyone = allgather(recs)
        assert everyone == recs * world, f"rank {rank} step {t}: ranks differ"
        glob = np.frombuffer(allgather(g.get_particles().tobytes()), dtype=np.float64).reshape(n, 5)
        single.set_particles(glob)
        srecs, stotal, srk = query(single, n)
        assert (srecs, stotal) == (recs, total), f"rank {rank} step {t}: single-GPU handle differs"
        assert np.array_equal(srk[lo:hi], rk), f"rank {rank} step {t}: per-slot ranks"
        grp.barrier()
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK hypotheses world={world} n={n}")
    grp.close()


if __name__ == "__main__":
    main()
