"""Worker of tests/test_gpu_recovery.py::test_recovery_multi_process: one process per GPU (torchrun).  Every rank steps its shard of
a sharded MonteCarloLocalizer with augmented MCL through a kidnap; every step is compared bit for bit with the full-size CPU oracle:
this rank's particles, resample indices, and (w_slow, w_fast, p), which every rank computes from the global S."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
from _recovery_oracle import OracleRecovery  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.KidnapScenario(before=6, after=steps - 6, pitch_deg=12.0)
    g = rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(*sc.config(n)), seed=5, device=local,
                                                      shard=(uid, rank, world))
    o = OracleRecovery(n, range_noise=0.25, velocity_noise=0.05, yaw_rate_noise=0.02, seed=5, mode=1, max_particles=n, threads=4)
    g.enable_recovery(0.1, 0.6, sc.REGION)
    o.enable(0.1, 0.6, sc.REGION)
    o.init_state(sc.init)
    lo, hi = rdist.shard_bounds(n, rank, world)
    total = 0
    for t in range(steps):
        g.try_step(sc.controls[t], sc.obs[t])
        o.step(sc.controls[t], sc.obs[t])
        grp.barrier()
        assert np.array_equal(g.last_indices(), o.last_indices()[lo:hi]), f"rank {rank} step {t}: indices"
        assert np.array_equal(g.get_particles(), o.particles()[lo:hi]), f"rank {rank} step {t}: particles"
        ws, wf, p, inj = g.recovery_state()
        w, oinj = o.state()
        assert np.array_equal([ws, wf, p], w) and inj <= oinj, f"rank {rank} step {t}: recovery state"
        total += oinj
        grp.barrier()
    assert total > 0, "no step injected"
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK recovery world={world} n={n} injected={total}")
    grp.close()


if __name__ == "__main__":
    main()
