"""Data-parallel host logic (SURVEY.md §8e): one process per GPU, batch sharded across ranks, ONE
all-reduce of the flat gradient buffer per training step (NCCL over NVLink on GPUs; the same code
runs over gloo on CPU tensors for the tests).  The reference has no multi-GPU support
(README.md:140,210) — this is new functionality whose contract is "same math as one big batch":
every loss term is a mean over the local batch (model.py:276-302), so averaging the per-rank
gradients equals the single-device gradient of the concatenated batch when BN is frozen.

In BN training mode the statistics stay per rank by default, as in standard DP: each shard is normalised with its
own batch statistics and each rank keeps its own moving statistics.  train_step(sync_bn=True) synchronises them
(the reference lists "multi-GPUs with sync batch norm" as a TODO): every BN layer's per-channel sums Σz / Σz² in
the forward and Σdact·ẑ / Σdact in the backward are all-reduced between the kernel that produces them and the
kernel that consumes them, on a communicator of their own (sync_bn_group).  The step then equals the single-device
step on the concatenated batch up to fp32 summation order, and every rank holds the same moving statistics."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Initialise torch.distributed from the torchrun environment (RANK / WORLD_SIZE / LOCAL_RANK /
    MASTER_*).  Returns (rank, world, local_rank).  No-op for single-process runs."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl":
            torch.cuda.set_device(local)
            kw["device_id"] = torch.device(f"cuda:{local}")
        dist.init_process_group(backend, **kw)
    return rank, world, local


def shard_batch(n_global, rank, world):
    """Contiguous image range [lo, hi) of this rank (equal shards; n_global must divide)."""
    if n_global % world:
        raise ValueError(f"global batch {n_global} is not divisible by world size {world}")
    per = n_global // world
    return rank * per, (rank + 1) * per


def allreduce_gradients(flat_grad, group=None):
    """Sum the flat gradient over the ranks in place and return the factor that turns the sum into
    the mean (applied inside the fused optimizer kernel, not as a separate pass)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world > 1:
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    return 1.0 / world


def gradient_buckets(layer_floats, bucket_floats):
    """Split the layers (creation order, `layer_floats[i]` = floats layer i owns in the flat gradient) into contiguous
    buckets of roughly `bucket_floats`, listed in BACKWARD order (detection heads first): [(first_layer, last_layer), ...].
    The backward pass finishes a bucket's gradients from its last layer down to its first; its all-reduce can start then."""
    out, hi, acc = [], len(layer_floats) - 1, 0
    for i in range(len(layer_floats) - 1, -1, -1):
        acc += int(layer_floats[i])
        if acc >= bucket_floats or i == 0:
            out.append((i, hi))
            hi, acc = i - 1, 0
    return out


_SYNC_BN_GROUPS = {}


def sync_bn_group(group=None):
    """A second process group over the ranks of `group` (None: the default group) for the synchronised-BN exchanges,
    created on first use and cached by its rank list.  Those all-reduces are small (<= 8 KB, 2 x 72 per step) and each
    one blocks the next layer, so they get their own NCCL communicator and stream instead of queueing behind the 32 MB
    gradient buckets on `group`.  NCCL requires every rank to issue the collectives of both groups in the same
    program order: train_step_sync_bn's fixed sequence of yields guarantees it.
    torch.distributed.new_group is collective over the default group, so only a group spanning every rank is
    supported: with a proper subgroup the ranks outside it would never make the call."""
    base = group if group is not None else dist.group.WORLD
    ranks = tuple(dist.get_process_group_ranks(base))
    if len(ranks) != dist.get_world_size():
        raise ValueError(f"sync_bn needs a process group over all {dist.get_world_size()} ranks, got ranks {list(ranks)}")
    g = _SYNC_BN_GROUPS.get(ranks)
    if g is None:
        g = _SYNC_BN_GROUPS[ranks] = dist.new_group(list(ranks))
    return g


class BucketedAllReduce:
    """Overlap of the gradient all-reduce with the backward pass (SURVEY.md 8e; VERDICT r01 #3): every finished bucket is
    handed to NCCL with async_op=True — torch's NCCL stream waits for the work enqueued so far on the compute stream and
    runs the collective while the compute stream carries on with the next bucket's backward; wait() joins them before
    the optimizer update.  Over gloo (CPU tensors, tests) the same calls run synchronously."""

    def __init__(self, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.pending = []

    def reduce(self, flat_slice):
        if self.world > 1:
            self.pending.append(dist.all_reduce(flat_slice, op=dist.ReduceOp.SUM, group=self.group, async_op=True))

    def wait(self):
        """Returns the factor that turns the summed gradient into the mean (folded into the optimizer kernel)."""
        for w in self.pending:
            w.wait()
        self.pending = []
        return 1.0 / self.world


def max_over_ranks(value, device):
    """Device-side max of a per-rank scalar (multi-GPU timings are reported as the max over ranks)."""
    t = torch.tensor([float(value)], device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)
