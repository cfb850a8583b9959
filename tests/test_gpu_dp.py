"""2-GPU NCCL test of the data-parallel training step (needs >= 2 devices; skipped on a single-GPU machine).

DP-equivalence (SURVEY.md §4(3)): every loss term is a mean over the local batch (model.py:276-302), so the
N-rank step — local backward, NCCL all-reduce (sum) of the flat gradient, 1/world folded into the optimizer kernel —
must equal the 1-rank step on the concatenated batch.  BN is frozen (train_step(freeze_bn=True): the graph of
forward(is_training=False)) so that an image's activations do not depend on which other images share its rank.
Checked on the ENGINE: the parameter update of the 2-rank run against a 1-rank run of all 4 images, on layers at
the bottom, middle and top of the network, plus bit-identical parameters on both ranks."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYERS = (0, 1, 30, 57, 58, 66, 73, 74)


def _flat(m, keys=("w", "gamma", "beta", "b")):
    plan = m._last_plan
    out = []
    for i in LAYERS:
        ps = plan.conv_params(i)
        out += [ps[k].reshape(-1).clone() for k in keys if k in ps]
    return out


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    import yolov3_tensorflow_b200 as pkg
    from yolov3_tensorflow_b200 import parallel
    from oracle import yolov3_oracle as O
    from tests.test_gpu_path import _train_case
    parallel.init_from_env("nccl")
    params, x, y_true = _train_case(n=4)
    lo, hi = parallel.shard_batch(4, rank, world)
    xs = torch.from_numpy(x[lo:hi]).cuda()
    ys = [torch.from_numpy(y[lo:hi]).cuda() for y in y_true]
    lr = 1e-2

    def fresh():
        m = pkg.yolov3(80, O.COCO_ANCHORS, use_label_smooth=True, use_focal_loss=True, dtype="bf16")
        m.set_params(params, "HWIO")
        return m

    # ---- 2-rank data-parallel step through the public API (NCCL all-reduce inside train_step)
    m_dp = fresh()
    m_dp.train_step(xs, ys, lr, freeze_bn=True)
    dp = _flat(m_dp)
    gathered = []
    for t in dp:
        ws = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(ws, t)
        gathered.append(ws)
    same = all(torch.equal(ws[0], ws[1]) for ws in gathered)
    # ---- the same step with ONE blocking all-reduce after the whole backward: the bucketed, backward-overlapped
    # ---- reduction must give the same update (two runs differ only by the order of the fp32 atomics inside wgrad)
    m_blk = fresh()
    m_blk.train_step(xs, ys, lr, freeze_bn=True, bucket_mb=0)
    blk = _flat(m_blk)
    nb = len(m_dp._last_plan._buckets)
    bucket_err = max(float((a - b).double().norm() / b.double().norm().clamp(min=1e-30)) for a, b in zip(dp, blk))
    # ---- 1-rank step on the concatenated batch (no collective), same engine, same parameters
    m_1 = fresh()
    m_1.train_step(torch.from_numpy(x).cuda(), [torch.from_numpy(y).cuda() for y in y_true], lr, freeze_bn=True,
                   data_parallel=False)
    one = _flat(m_1)
    m_0 = fresh()
    m_0.forward(xs)                                   # uploads the parameters: the "before" values in arena layout
    before = _flat(m_0)
    errs = []
    for a, b, w0 in zip(dp, one, before):
        da, db = (a - w0).double(), (b - w0).double()
        errs.append(float((da - db).norm() / db.norm().clamp(min=1e-30)))
    moved = all(float((b - w0).abs().max()) > 0 for b, w0 in zip(one, before))
    dist.barrier()
    dist.destroy_process_group()
    q.put((rank, max(errs), same, moved, nb, bucket_err))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_dp_train_step_equals_single_rank_on_concatenated_batch():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=900)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = sorted(q.get(timeout=5) for _ in range(2))
    for rank, err, same, moved, nb, bucket_err in res:
        print(f"rank {rank}: {nb} gradient buckets; bucketed vs blocking all-reduce, max relative L2 difference of the parameters: {bucket_err:.3g}")
        assert nb >= 4 and bucket_err < 1e-6
        print(f"rank {rank}: max relative L2 error of the parameter update, 2-rank DP vs 1-rank on 4 images: {err:.3g}")
        assert moved, "the 1-rank reference step did not move the parameters"
        # fp32 atomic-accumulation order in wgrad / BN reductions is the only difference (1/N is a power of two)
        assert err < 1e-3, f"rank {rank}: DP update differs from the single-rank update on the concatenated batch ({err})"
        assert same, "ranks hold different parameters after the data-parallel update"
