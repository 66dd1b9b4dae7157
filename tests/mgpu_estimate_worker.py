"""Worker of tests/test_gpu_estimate.py::test_estimate_multi_process: one process per GPU (torchrun).  Every rank steps its shard
of the sharded FastSLAM engine, takes its estimate moments (pfgpu_fs_moments) between barriers, the moments of all ranks travel
over the control connection, and every rank merges them (pfgpu_fs_estimate_merge) and compares the estimate with numpy over the
full-size oracle's state."""
import ctypes as C
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
import _oracle  # noqa: E402
from test_gpu_estimate import check, ref_estimate  # noqa: E402


def gather_moments(grp, pose, lm, m):
    """every rank's (pose moments, landmark moments), in rank order, on every rank"""
    ps = C.sizeof(pose)
    blob = grp._exchange(bytes(pose) + lm.tobytes(), lambda parts: b"".join(parts))
    per = ps + m * 7 * 8
    out = []
    for r in range(grp.world):
        chunk = blob[r * per:(r + 1) * per]
        out.append((rr.api._FsPoseMoments.from_buffer_copy(chunk[:ps]), np.frombuffer(chunk[ps:], dtype=np.float64).reshape(m, 7).copy()))
    return out


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.c3_scenario(steps=steps)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=9, device=local, shard=(uid, rank, world))
    o = _oracle.OracleFS(_oracle.load(libm=False), n, sc.m, seed=9, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    nl = n // world
    remote = checked = 0
    for t in range(steps):
        did = g.fastslam_update(sc.control, sc.obs[t])                      # (synchronises this rank)
        assert did == bool(o.step(sc.control, sc.obs[t])), f"rank {rank} step {t}: gate"
        if did:
            remote += int(((g.last_indices() // nl) != rank).sum())
        if t % 4 == 3:
            for cm in (100.0, math.inf):
                grp.barrier()                       # every rank has finished step t
                pose, lm = g.moments(cm)
                grp.barrier()                       # nobody steps on while a peer still reads through remote references
                est = rr.FastSlam1.merge_moments(gather_moments(grp, pose, lm, sc.m))
                op, ol = o.state()
                check(est, ref_estimate(op, ol, op[-1, 1:4], cm), f"rank {rank} step {t} cov00_max {cm}")
                checked += 1
    remote = grp.max(remote)
    assert checked > 0 and (world == 1 or remote > 0), f"checked {checked}, remote ancestors {remote}"
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK estimate world={world} n={n} checked={checked} remote_ancestors={int(remote)}")
    grp.close()


if __name__ == "__main__":
    main()
