"""Worker of tests/test_gpu_beam.py::test_beam_multi_process: one process per GPU (torchrun).  Every rank loads the same beam map into its
shard of a sharded MonteCarloLocalizer with augmented MCL and steps it with beam scans; every step is compared bit for bit with the
full-size CPU oracle: this rank's particles, resample indices, and (w_slow, w_fast, p)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
from _beam_oracle import OracleBeam  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.ScanScenario(steps=steps)
    init = [sc.truth[0][0], sc.truth[0][1], sc.truth[0][2], 1.0]
    g = rr.MonteCarloLocalizer.try_with_initial_state(init, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1), seed=5,
                                                      device=local, shard=(uid, rank, world))
    o = OracleBeam(n, range_noise=0.25, velocity_noise=0.2, yaw_rate_noise=0.1, seed=5, mode=1, max_particles=n, threads=4)
    o.init_state(init)
    g.set_beam_model(sc.obstacles, sc.RES)
    assert o.set_beam_map(sc.obstacles, sc.RES) == 0
    g.enable_recovery(0.1, 0.6, sc.REGION)
    o.enable(0.1, 0.6, sc.REGION)
    lo, hi = rdist.shard_bounds(n, rank, world)
    for t in range(steps):
        g.try_step_beam_scan(sc.controls[t], *sc.scan_args(t))
        o.step_beam(sc.controls[t], *sc.scan_args(t))
        grp.barrier()
        assert np.array_equal(g.last_indices(), o.last_indices()[lo:hi]), f"rank {rank} step {t}: indices"
        assert np.array_equal(g.get_particles(), o.particles()[lo:hi]), f"rank {rank} step {t}: particles"
        ws, wf, p, _ = g.recovery_state()
        w, _ = o.state()
        assert np.array_equal([ws, wf, p], w), f"rank {rank} step {t}: recovery state"
        grp.barrier()
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK beam world={world} n={n}")
    grp.close()


if __name__ == "__main__":
    main()
