"""CPU test of parallel.sync_bn_group with the gloo backend, world size 2: one cached communicator per rank list
(the default group and an explicit WORLD share it), collectives on it sum across the ranks, and a group that does not
span every rank is refused instead of hanging in torch.distributed.new_group."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    from yolov3_tensorflow_b200 import parallel
    parallel.init_from_env("gloo")
    g = parallel.sync_bn_group()
    assert parallel.sync_bn_group(None) is g and parallel.sync_bn_group(dist.group.WORLD) is g
    assert g is not dist.group.WORLD and dist.get_process_group_ranks(g) == [0, 1]
    t = torch.full((8,), float(rank + 1))
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=g)
    assert torch.equal(t, torch.full((8,), 3.0))
    sub = dist.new_group([0])                          # collective over the default group: both ranks create it
    if rank == 0:
        with pytest.raises(ValueError):
            parallel.sync_bn_group(sub)
    dist.barrier()
    dist.destroy_process_group()
    out.put((rank, True))


def test_sync_bn_group_gloo_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, True), (1, True)]
