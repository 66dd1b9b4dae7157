"""Worker of tests/test_gpu_odom.py::test_odom_multi_process: one process per GPU (torchrun).  Every rank steps its shard of a sharded
MonteCarloLocalizer with augmented MCL by odometry pairs (OdomScenario), with likelihood-field and beam steps and one velocity step;
every step is compared bit for bit with the full-size CPU oracle: this rank's particles, resample indices, and (w_slow, w_fast, p)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
from _odom_oracle import OracleOdom  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n = int(sys.argv[1])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.OdomScenario(legs=((3, 1.0, 0.05), (2, 0.0, 0.0), (2, 0.0, 1.0), (2, -0.5, 0.0)))
    init = [sc.start[0], sc.start[1], sc.start[2], 0.0]
    g = rr.MonteCarloLocalizer.try_with_initial_state(init, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1), seed=5,
                                                      device=local, shard=(uid, rank, world))
    o = OracleOdom(n, range_noise=0.25, velocity_noise=0.2, yaw_rate_noise=0.1, seed=5, mode=1, max_particles=n, threads=4)
    o.init_state(init)
    g.set_likelihood_field(sc.obstacles, sc.RES)
    assert o.set_map(sc.obstacles, sc.RES) == 0
    g.set_beam_model(sc.obstacles, sc.RES)
    assert o.set_beam_map(sc.obstacles, sc.RES) == 0
    g.set_odometry_noise(0.1, 0.05, 0.1, 0.05)
    assert o.set_odom_noise((0.1, 0.05, 0.1, 0.05)) == 0
    g.enable_recovery(0.1, 0.6, sc.REGION)
    o.enable(0.1, 0.6, sc.REGION)
    lo, hi = rdist.shard_bounds(n, rank, world)
    for t in range(sc.steps):
        a, b = sc.odom_pair(t)
        if t == 4:
            g.try_step_scan(sc.controls[t], *sc.scan_args(t))
            o.step_scan(sc.controls[t], *sc.scan_args(t))
        elif t % 2:
            g.try_step_beam_scan_odometry(a, b, *sc.scan_args(t))
            o.step_beam_odom(a, b, *sc.scan_args(t))
        else:
            g.try_step_scan_odometry(a, b, *sc.scan_args(t))
            o.step_scan_odom(a, b, *sc.scan_args(t))
        grp.barrier()
        assert np.array_equal(g.last_indices(), o.last_indices()[lo:hi]), f"rank {rank} step {t}: indices"
        assert np.array_equal(g.get_particles(), o.particles()[lo:hi]), f"rank {rank} step {t}: particles"
        ws, wf, p, _ = g.recovery_state()
        w, _ = o.state()
        assert np.array_equal([ws, wf, p], w), f"rank {rank} step {t}: recovery state"
        grp.barrier()
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK odom world={world} n={n}")
    grp.close()


if __name__ == "__main__":
    main()
