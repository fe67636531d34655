"""world_size-2 gloo test of the N>1 host logic (spicedb-kubeapi-proxy_b200/dist.py):
slicing, all-gather back to caller order, max-over-ranks timing. The evaluator is the
CPU oracle here (there is no GPU); on the GPU box the same class wraps engine.check_bulk.
A world_size-3 test runs the sharded store's TorchDeviceTransport on CPU tensors."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist

    import zgpu  # noqa: F401  (registers spicedb_kubeapi_proxy_b200)
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import dist as zdist, workloads

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        w = workloads.cfg4(scale=0.0005)
        o = Oracle(w.schema)
        w.load_into(o)
        items = w.check_items(o, zgpu.CHECK_DTYPE)[:5003]  # not divisible by the world size
        calls = []

        def evaluate(part):
            calls.append(part.size)
            return o.check_bulk(part, nthreads=1)

        sc = zdist.ShardedChecker(evaluate)
        got = sc.check_bulk(items)
        want = o.check_bulk(items, nthreads=1)
        lo, hi = zdist.shard_bounds(items.size, rank, world)
        ok = bool(np.array_equal(got, want)) and calls == [hi - lo]
        empty_ok = sc.check_bulk(items[:1]).size == 1  # one rank gets an empty slice
        mx = zdist.max_over_ranks(float(rank + 1))
        q.put((rank, ok, empty_ok, mx, hi - lo))
    finally:
        dist.destroy_process_group()


def test_sharded_checker_world2():
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in procs)
    [p.join(timeout=60) for p in procs]
    assert [r[1] for r in res] == [True, True], res
    assert [r[2] for r in res] == [True, True]
    assert [r[3] for r in res] == [2.0, 2.0]
    assert sum(r[4] for r in res) == 5003 and abs(res[0][4] - res[1][4]) <= 1


def test_shard_bounds_cover_exactly():
    sys.path.insert(0, ROOT)
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200.dist import shard_bounds

    for n in (0, 1, 7, 8, 1000003):
        for world in (1, 2, 3, 8):
            b = [shard_bounds(n, r, world) for r in range(world)]
            assert b[0][0] == 0 and b[-1][1] == n
            assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
            assert max(hi - lo for lo, hi in b) - min(hi - lo for lo, hi in b) <= 1


def _a2a_part(src, dst):
    """The items rank src sends rank dst: (src + dst) % 3 * 5 of them (ragged, some empty), 3 bytes each."""
    n = (src + dst) % 3 * 5
    return np.stack([np.full(n, 10 * src + dst), np.arange(n), np.full(n, 7)], axis=1).astype(np.uint8)


def _a2a_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist

    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200 import dist as zdist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        t = zdist.TorchDeviceTransport(device=torch.device("cpu"))
        send_counts = [_a2a_part(rank, d).shape[0] for d in range(world)]
        recv_counts = t.exchange_counts(send_counts)
        send = torch.from_numpy(np.concatenate([_a2a_part(rank, d).ravel() for d in range(world)]))
        got = t.alltoall(send, send_counts, recv_counts, 3)
        want = np.concatenate([_a2a_part(s, rank).ravel() for s in range(world)])
        ok = recv_counts == [_a2a_part(s, rank).shape[0] for s in range(world)] and np.array_equal(got.numpy(), want)
        q.put((rank, ok, t.allreduce_sum(rank + 1)))
    finally:
        dist.destroy_process_group()


def test_torch_device_transport_ragged_alltoall_world3():
    """The transport of the device-resident sharded store (nccl in bench.py), here on CPU tensors over gloo."""
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_a2a_worker, args=(r, 3, port, q)) for r in range(3)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in procs)
    [p.join(timeout=60) for p in procs]
    assert [r[1] for r in res] == [True, True, True], res
    assert [r[2] for r in res] == [6, 6, 6]
