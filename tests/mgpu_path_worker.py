"""Worker of tests/test_gpu_path.py::test_path_multi_process: one process per GPU (torchrun).  Every rank steps its shard of the
sharded FastSLAM engine with path history enabled (the rings' cudaIpc handles are exchanged once, at enable), then, between
barriers, reads the paths of sampled global slots (parents on other ranks are read through the peer mapping) and its path
moments.  Paths are compared bit for bit with the genealogy of the full-size CPU oracle; the moments of all ranks travel over the
control connection and every rank merges them step by step and compares with numpy."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import dist as rdist, scenarios  # noqa: E402
import _oracle  # noqa: E402
from _path_oracle import Genealogy, ref_path_estimate  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    n, steps = int(sys.argv[1]), int(sys.argv[2])
    grp = rdist.TcpGroup()
    uid = rdist.broadcast_unique_id(grp, rdist.nccl_unique_id)
    sc = scenarios.FastSlamScenario(4, (15.0, 15.0, 0.0), (1.0, 0.025), steps)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=9, device=local, shard=(uid, rank, world))
    o = _oracle.OracleFS(_oracle.load(libm=False), n, sc.m, seed=9, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    g.enable_history(steps + 1)
    gen = Genealogy(steps + 1)
    gen.root(0, o.state()[0])
    for t in range(steps):
        did = g.fastslam_update(sc.control, sc.obs[t])                      # (synchronises this rank)
        assert did == bool(o.step(sc.control, sc.obs[t])), f"rank {rank} step {t}: gate"
        gen.record(t + 1, o.state()[0], o.last_indices())
    grp.barrier()                                   # every rank has recorded its last entry
    slots = sorted({o.best(), 0, n - 1, *np.random.default_rng(3).integers(0, n, 16).tolist()})
    crossed = 0
    for s in slots:
        got, want = g.path(s), gen.path(s)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), f"rank {rank} slot {s}"
        crossed += int(len(set((want[1] // (n // world)).tolist())) > 1)
    steps_, mom = g.path_moments()
    grp.barrier()                                   # nobody steps on while a peer still reads this rank's ring
    ps = C.sizeof(rr.api._FsPoseMoments)
    blob = grp._exchange(b"".join(bytes(m) for m in mom), lambda parts: b"".join(parts))
    per = ps * len(mom)
    ranks = [(steps_, [rr.api._FsPoseMoments.from_buffer_copy(blob[r * per + j * ps:r * per + (j + 1) * ps]) for j in range(len(mom))])
             for r in range(world)]
    est = rr.FastSlam1.merge_path_moments(ranks)
    wsteps, mean, cov = ref_path_estimate(gen, o.state()[0][:, 0])
    assert np.array_equal(est.steps, wsteps)
    assert np.allclose(est.pose, mean, rtol=1e-9, atol=1e-9) and np.allclose(est.pose_cov, cov, rtol=1e-7, atol=1e-12), f"rank {rank}: moments"
    crossed = grp.max(crossed)
    assert world == 1 or crossed > 0, "no lineage crossed ranks"
    grp.barrier()
    if rank == 0:
        print(f"MGPU_OK path world={world} n={n} slots={len(slots)} crossed={int(crossed)}")
    grp.close()


if __name__ == "__main__":
    main()
