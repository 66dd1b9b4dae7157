"""Worker of tests/test_gpu_pf_moments.py::test_sharded_multi_process: one process per GPU (torchrun).  A sharded
ParticleFilterLocalizer at UTM coordinates: every rank gathers every shard's moments and merges them in rank order, so every
rank must return the same bits, within the bar of the exact reference over the concatenated cloud."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
import _pf_moments_cases as pm  # noqa: E402


def gather(grp, arr):
    """every rank's array, concatenated in rank order, on every rank"""
    blob = grp._exchange(arr.tobytes(), lambda parts: b"".join(parts))
    return np.frombuffer(blob, dtype=np.float64).reshape(-1, *arr.shape[1:]).copy()


def agree(grp, g, a, what, rank):
    est, cov = g.estimate(), g.calc_covariance()
    bad = pm.violations(est, cov, a)
    assert not bad, f"rank {rank} {what}: {bad}"
    bits = gather(grp, np.concatenate([est, cov.ravel()])[None, :])
    assert all(np.array_equal(bits[0], b) for b in bits), f"rank {rank} {what}: ranks return different bits"


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    n = 1 << 14
    lo, hi = rdist.shard_bounds(n, rank, world)
    g = rr.ParticleFilterLocalizer(rr.ParticleFilterConfig(n, 0.6, 0.25), seed=5, device=local, shard=(uid, rank, world))
    far = pm.cloud(n, (-pm.UTM[0], -pm.UTM[1]), 1.0, "uniform", seed=1)
    g.set_particles(far[lo:hi])
    agree(grp, g, far, "far cloud", rank)
    for name, a in [("utm 1mm", pm.cloud(n, pm.UTM, 1e-3, "random", seed=2)), ("utm zero spread", pm.cloud(n, pm.UTM, 0.0, "uniform")),
                    ("injected 10 km", pm.injected(n, 1e4, seed=3)), ("ones", pm.cloud(n, (1e4, 1e4), 1e-2, "ones", seed=4))]:
        g.set_particles(a[lo:hi])
        agree(grp, g, a, name, rank)
    sc = scenarios.PfScenario("c1", steps=20)
    init = [sc.init[0] + pm.UTM[0], sc.init[1] + pm.UTM[1], sc.init[2], sc.init[3]]
    assert g.L.pfgpu_pf_init_state(g.h, rr.api._dp(np.asarray(init, dtype=np.float64))) == 0
    agree(grp, g, gather(grp, g.get_particles()), "init_state", rank)
    for t in range(20):
        obs = np.column_stack([sc.obs[t][:, 0], sc.obs[t][:, 1] + pm.UTM[0], sc.obs[t][:, 2] + pm.UTM[1]])
        g.try_step(sc.controls[t], obs)
        agree(grp, g, gather(grp, g.get_particles()), f"step {t}", rank)
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK world={world} n={n}")
    grp.close()


if __name__ == "__main__":
    main()
