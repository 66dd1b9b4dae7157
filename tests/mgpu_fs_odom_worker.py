"""Worker of tests/test_gpu_fs_odom.py::test_fs_odom_multi_process: one process per GPU (torchrun).  Every rank steps its shard of
the sharded FastSLAM 2.0 engine by odometry pairs (a drive, a stop, a turn in place, a reverse): known-id steps with observations
(fs2_propose_odom_kernel, reading ancestors' landmarks through the peer mapping), steps without observations (fs3_odom_predict_kernel),
one velocity step, then unknown-association steps (fs3_assoc_odom_kernel).  Every step is compared bit for bit with the full-size
CPU oracle: gate, indices, this rank's poses, weights and landmarks."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
from _fs_odom_oracle import OracleFsOdom  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.FsOdomScenario(side=4, start=(15.0, 15.0, 0.0), legs=((4, 1.0, 0.05), (2, 0.0, 0.0), (2, 0.0, 1.0), (2, -0.5, 0.0),
                                                                        (steps, 1.0, -0.05)), max_range=40.0)
    g = rr.FastSlam2(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=9, device=local, shard=(uid, rank, world))
    o = OracleFsOdom(n, sc.m, seed=9, variant=2, nth=n / 1.5)
    o.L.orc_fs_set_threads(o.h, 4)
    g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    g.set_odometry_noise(0.1, 0.05, 0.1, 0.05)
    o.set_odom_noise((0.1, 0.05, 0.1, 0.05))
    nl = n // world
    grp.barrier()
    crossed = 0
    for t in range(steps):
        a, b = sc.odom_pair(t)
        z = sc.obs[t] if t % 4 != 1 else []
        if t == 5:
            did = g.fastslam2_update(sc.controls[t], z)
            odid = o.step(sc.controls[t], z)
        elif t >= steps // 2:
            zu = [(d, ang) for d, ang, _ in z]
            did = g.fastslam2_update_unknown_odometry(a, b, zu)
            odid = o.step_unknown_odom(a, b, zu)
        else:
            did = g.fastslam2_update_odometry(a, b, z)
            odid = o.step_odom(a, b, z)
        assert did == bool(odid), f"rank {rank} step {t}: gate"
        grp.barrier()                                                          # every rank's step is over before anyone reads
        if did:
            idx = o.last_indices()
            assert np.array_equal(g.last_indices(), idx[rank * nl:(rank + 1) * nl]), f"rank {rank} step {t}: indices"
            crossed += int((idx[rank * nl:(rank + 1) * nl] // nl != rank).any())
        gp, gl = g.state()
        op, ol = o.state()
        assert np.array_equal(gp, op[rank * nl:(rank + 1) * nl]) and np.array_equal(gl, ol[rank * nl:(rank + 1) * nl]), f"rank {rank} step {t}: state"
        grp.barrier()                                                          # nobody steps on while a peer still reads
    crossed = grp.max(crossed)
    assert world == 1 or crossed > 0, crossed
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK fs_odom world={world} n={n} crossed={int(crossed)}")
    grp.close()


if __name__ == "__main__":
    main()
