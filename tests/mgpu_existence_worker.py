"""Worker of tests/test_gpu_existence.py::test_existence_multi_process: one process per GPU (torchrun).  Every rank steps its
shard of the sharded FastSLAM 2.0 engine with unknown data association and existence counters (the counters' cudaIpc handles are
exchanged once, at enable, so counters of ancestors on other ranks are read through the peer mapping).  Every step is compared
bit for bit with the full-size CPU oracle: gate, indices, this rank's poses, landmarks and counters."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
from _exist_oracle import OracleFS2Exist  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.FastSlamScenario(6, (25.0, 5.0, 0.0), (1.0, 0.05), steps, seed=7)
    m = 24
    g = rr.FastSlam2(n, m, rr.FsConfig(nth=n / 1.5), seed=9, device=local, shard=(uid, rank, world))
    o = OracleFS2Exist(n, m, seed=9, nth=n / 1.5)
    pw = np.tile([1.0 / n, *sc.start], (n, 1))
    lm = np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1))
    rng = np.random.default_rng(n)                                             # slots 0..7: landmarks nothing observes, to be removed
    lm[:, :8, 0] = sc.start[0] + rng.uniform(-6.0, 6.0, (n, 8))
    lm[:, :8, 1] = sc.start[1] + rng.uniform(-6.0, 6.0, (n, 8))
    lm[:, :8, 2:] = [0.5, 0.0, 0.0, 0.5]
    nl = n // world
    g.set_state(pw[rank * nl:(rank + 1) * nl], lm[rank * nl:(rank + 1) * nl])
    o.set_state(pw, lm)
    g.enable_existence(8.0)
    o.enable_existence(8.0)
    grp.barrier()
    removed = crossed = 0
    for t in range(steps):
        z = [(d, a) for d, a, _ in sc.obs[t]]
        did = g.fastslam2_update_unknown(sc.control, z)                       # (synchronises this rank)
        assert did == o.step_unknown(sc.control, z), f"rank {rank} step {t}: gate"
        grp.barrier()                                                          # every rank's step is over before anyone reads
        if did:
            idx = o.last_indices()
            assert np.array_equal(g.last_indices(), idx[rank * nl:(rank + 1) * nl]), f"rank {rank} step {t}: indices"
            crossed += int((idx[rank * nl:(rank + 1) * nl] // nl != rank).any())
        gp, gl = g.state()
        op, ol = o.state()
        assert np.array_equal(gp, op[rank * nl:(rank + 1) * nl]) and np.array_equal(gl, ol[rank * nl:(rank + 1) * nl]), f"rank {rank} step {t}: state"
        assert np.array_equal(g.existence_counts(), o.existence_counts()[rank * nl:(rank + 1) * nl]), f"rank {rank} step {t}: counters"
        removed += o.removed
        grp.barrier()                                                          # nobody steps on while a peer still reads
    crossed = grp.max(crossed)
    assert removed > 0 and (world == 1 or crossed > 0), (removed, crossed)
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK existence world={world} n={n} removed={removed} crossed={int(crossed)}")
    grp.close()


if __name__ == "__main__":
    main()
