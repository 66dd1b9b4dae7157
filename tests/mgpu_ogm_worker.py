"""Worker of tests/test_gpu_ogm.py::test_ogm_multi_process: one process per GPU (torchrun).  Every rank maps ScanScenario's trajectory
into an OccupancyGridMap on its own device and hands it to its shard of a sharded MonteCarloLocalizer with set_beam_model_from_grid;
the grid must equal the contract-math oracle's, and every beam step is compared bit for bit with the full-size CPU oracle loaded with
the oracle's obstacle mask: this rank's particles and resample indices."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
from _beam_oracle import OracleBeam  # noqa: E402
import _ogm_oracle as OO  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.ScanScenario()
    W, H = sc.obstacles.shape
    gm = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H), device=local)
    om = OO.OracleOgm(resolution=sc.RES, width=W, height=H)
    gm.update_with_scans(sc.truth, np.stack(sc.scans), sc.ANGLE_MIN, sc.ANGLE_INC)
    om.update_with_scans(sc.truth, np.stack(sc.scans), sc.ANGLE_MIN, sc.ANGLE_INC)
    assert np.array_equal(gm.grid.view(np.uint64), om.grid.view(np.uint64)), f"rank {rank}: grid"
    init = [sc.truth[0][0], sc.truth[0][1], sc.truth[0][2], 1.0]
    g = rr.MonteCarloLocalizer.try_with_initial_state(init, rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1), seed=5,
                                                      device=local, shard=(uid, rank, world))
    o = OracleBeam(n, range_noise=0.25, velocity_noise=0.2, yaw_rate_noise=0.1, seed=5, mode=1, max_particles=n, threads=4)
    o.init_state(init)
    g.set_beam_model_from_grid(gm, 0.5)
    assert o.set_beam_map(om.obstacles(0.5), sc.RES) == 0
    lo, hi = rdist.shard_bounds(n, rank, world)
    for t in range(steps):
        g.try_step_beam_scan(sc.controls[t], *sc.scan_args(t))
        o.step_beam(sc.controls[t], *sc.scan_args(t))
        grp.barrier()
        assert np.array_equal(g.last_indices(), o.last_indices()[lo:hi]), f"rank {rank} step {t}: indices"
        assert np.array_equal(g.get_particles(), o.particles()[lo:hi]), f"rank {rank} step {t}: particles"
        grp.barrier()
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK ogm world={world} n={n}")
    grp.close()


if __name__ == "__main__":
    main()
