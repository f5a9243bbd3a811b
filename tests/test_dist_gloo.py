"""N > 1 path on CPU: world_size-2 gloo.  The ensemble shards across ranks with no data-path collective;
the one exchange is the all-reduce of [grad_theta; loss].  Each rank evaluates its shard with the CPU
oracle (standing in for the GPU kernels, which need an H100) and the reduced result must equal the
single-process full-ensemble result."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, N, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import oracle as O
    from helpers import glorot_theta, synthetic_ensemble
    from universal_differential_equations_b200.dist import allreduce_loss_grad, shard_range
    theta = glorot_theta((2, 32, 32, 2), seed=1).astype(np.float64)
    u0, y = synthetic_ensemble(N)
    lo, hi = shard_range(N, rank, world)
    m = O.lv_model()
    l, g, _ = O.ensemble_loss_grad(m, theta, u0[:, lo:hi].copy(), y[:, :, lo:hi].copy(), np.ones(2), 0.1, 30, n_threads=1)
    buf = torch.from_numpy(np.concatenate([g, [l]]))
    allreduce_loss_grad(buf)
    if rank == 0:
        ret["buf"] = buf.numpy().copy()
        ret["ranges"] = [shard_range(N, r, world) for r in range(world)]
    dist.destroy_process_group()


def test_shard_range_covers_ensemble():
    from universal_differential_equations_b200.dist import shard_range
    for n, w in ((65536, 8), (10, 3), (7, 8), (1, 2)):
        r = [shard_range(n, k, w) for k in range(w)]
        assert r[0][0] == 0 and r[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(r[:-1], r[1:]))
        assert max(b - a for a, b in r) - min(b - a for a, b in r) <= 1


def test_world2_allreduce_equals_full_batch(O):
    N, world = 37, 2
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_worker, args=(world, port, N, ret), nprocs=world, join=True)
        buf = np.array(ret["buf"])
    from helpers import glorot_theta, synthetic_ensemble
    theta = glorot_theta((2, 32, 32, 2), seed=1).astype(np.float64)
    u0, y = synthetic_ensemble(N)
    l, g, _ = O.ensemble_loss_grad(O.lv_model(), theta, u0, y, np.ones(2), 0.1, 30, n_threads=1)
    assert abs(buf[-1] - l) <= 1e-12 * abs(l)
    assert np.linalg.norm(buf[:-1] - g) <= 1e-12 * np.linalg.norm(g)
