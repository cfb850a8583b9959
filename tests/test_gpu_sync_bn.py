"""Synchronised batch norm for data-parallel training (train_step(sync_bn=True) / train_step_sync_bn).

BN runs in training mode throughout.  In training mode the fused step is itself not reproducible bit for bit: the
conv epilogues accumulate the batch sums with fp32 atomics, and at this random-BN initialisation the BN backward is a
near-cancellation, so two runs of the same fused step on the same inputs differ in the update of the backbone
weights by O(1) relative (measured on an H100: 0.8 in bf16, 0.35 in fp16).  The bars below therefore check the
quantities that this noise leaves measurable, each at about 2x the worst value measured on an H100 SXM (80 GB,
400 W power limit), which is also the fused step's own run-to-run spread:
  - layer 0's moving statistics (the stem's sums are reproducible);
  - the worst relative error of the moving-statistics change over all 72 BN layers;
  - the losses;
  - the update of the last detection head (layer 74), the weights least affected by the cancellation.
None of these depends on the BN backward; a per-layer check against autograd on the engine's own tensors covers it.
The layered step is driven through the train_step_sync_bn generator, whose exchange points the tests serve
themselves: two models on one GPU stand in for two ranks, and their BN slabs and gradients are summed in lockstep.
That makes the sync-BN equivalence checkable on a single card:
  0. per BN layer, each rank's dz and the summed backward sums equal autograd over the concatenated rows with global
     statistics, and the check fails without the BN exchange or with only the forward one;
  1. one rank with an identity exchange computes what the fused train_step computes (within its run-to-run spread);
  2. two ranks with summed BN slabs equal one rank on the concatenated batch (update, moving statistics, loss),
     and end with bit-identical moving statistics and parameters equal to rounding;
  3. the same run without the BN exchange (per-rank statistics, plain DP) misses the moving statistics by far more;
  4. the host rejects layer calls out of the plan's order;
  5. over NCCL with 2 GPUs (skipped on one card) train_step(sync_bn=True) equals the 1-rank step on 4 images."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests.test_gpu_path import _train_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYERS = (0, 1, 30, 57, 58, 66, 73, 74)
LR = 1e-2
# {dtype: bar}, from two H100 runs.  The worst moving-statistics error is a maximum over 144 vectors and varies
# most from run to run, so its bar is about 2x the larger of the two runs.
# Layered world-1 step against the fused step (measured: moving bf16 0.026-0.068 / fp16 0.0043-0.0093, losses
# 0.020-0.15 / 0.010-0.012, layer 74 update 0.0094-0.010 / 0.0015; fused against fused: 0.026 / 0.0039, 0.095 /
# 0.0033, 0.0085 / 0.0015).
W1_MOVING = {"bf16": 0.15, "fp16": 0.02}
W1_LOSS = {"bf16": 0.3, "fp16": 0.03}
W1_UPDATE74 = {"bf16": 0.02, "fp16": 0.003}
# 2 virtual ranks x 2 images against 1 rank x 4 images (measured: layer-0 moving 2.2e-7-3.5e-6 / 7.7e-6-7.8e-6,
# moving 0.018-0.046 / 0.0027-0.0065, mean loss 0.053-0.055 / 0.0030-0.0033, layer 74 update 0.0066-0.0067 /
# 0.0010; fused 4-image step against itself: 3.5e-6 / 7.1e-6, 0.018 / 0.0028, 0.040 / 0.0086, 0.0066 / 0.0011).
# Without the BN exchange: layer-0 moving 1.1e-3, moving 0.47, layer 74 update 0.027 (bf16).
R2_MOVING0 = 2e-5
R2_MOVING = {"bf16": 0.1, "fp16": 0.015}
R2_LOSS = {"bf16": 0.1, "fp16": 0.02}
R2_UPDATE74 = {"bf16": 0.015, "fp16": 0.003}


def _pkg():
    import yolov3_tensorflow_b200 as pkg
    return pkg


def _model(params, dt):
    m = _pkg().yolov3(80, O.COCO_ANCHORS, use_label_smooth=True, use_focal_loss=True, dtype=dt)
    m.set_params(params, "HWIO")
    return m


def _cuda(x, ys, lo=None, hi=None):
    s = slice(lo, hi)
    return torch.from_numpy(x[s]).cuda(), [torch.from_numpy(y[s]).cuda() for y in ys]


def _lockstep(gens, factor, exchange_bn=True, exchange_bwd=True):
    """Serve the exchange points of several train_step_sync_bn generators, one virtual rank each: every BN slab
    (unless exchange_bn is False; the backward ones unless exchange_bwd is False) and every gradient bucket is
    replaced by the sum over the ranks, and `factor` is the mean factor of the gradient.  Returns each generator's
    result."""
    n_bn = sum(t[4] for t in _pkg().yolov3.conv_table(80))   # the first n_bn BN slabs are the forward ones
    replies, outs, seen_bn = [None] * len(gens), [None] * len(gens), 0
    while True:
        items = []
        for k, g in enumerate(gens):
            try:
                items.append(g.send(replies[k]))
            except StopIteration as done:
                outs[k] = done.value
                items.append(None)
        if all(it is None for it in items):
            return outs
        assert all(it is not None for it in items), "the ranks left the step at different points"
        kinds = {it[0] for it in items}
        assert len(kinds) == 1, kinds
        kind = items[0][0]
        replies = [factor if kind == "grad_scale" else None] * len(gens)
        if kind == "bn":
            seen_bn += 1
        if kind == "grad_scale" or len(gens) == 1 or (kind == "bn" and not exchange_bn):
            continue
        if kind == "bn" and seen_bn > n_bn and not exchange_bwd:
            continue
        total = items[0][1].clone()
        for it in items[1:]:
            total += it[1]
        for it in items:
            it[1].copy_(total)


def _params(m):
    """{layer: {name: fp32 numpy}} of the arena's master parameters and BN moving statistics."""
    plan = m._last_plan
    return {i: {k: v.detach().cpu().numpy().copy() for k, v in plan.conv_params(i).items()} for i in range(plan.num_layers)}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _initial(params):
    """The initial parameters in the arena layout (w OHWI) for update deltas."""
    out = {}
    for i, p in enumerate(params):
        q = {k: np.asarray(v, np.float32) for k, v in p.items()}
        q["w"] = np.transpose(q["w"], (3, 0, 1, 2))
        out[i] = q
    return out


def _update_err(got, ref, init, layers=LAYERS):
    return max(_rel(got[i][k] - init[i][k], ref[i][k] - init[i][k])
               for i in layers for k in ("w", "gamma", "beta", "b") if k in ref[i])


def _moving_err(got, ref, init, layers=None):
    """Worst relative error of the moving mean / variance change over the BN layers."""
    return max(_rel(got[i][k] - init[i][k], ref[i][k] - init[i][k])
               for i in (ref if layers is None else layers) for k in ("mean", "var") if k in ref[i])


def _losses(ls):
    return np.array([float(v) for v in ls], np.float64)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_layered_world1_equals_fused_step(dt):
    params, x, ys = _train_case()
    xs, yts = _cuda(x, ys)
    init = _initial(params)
    m_f = _model(params, dt)
    l_f = _losses(m_f.train_step(xs, yts, LR))
    m_l = _model(params, dt)
    (l_l,) = _lockstep([m_l.train_step_sync_bn(xs, yts, LR, bn_replicas=1)], factor=1.0)
    l_l = _losses(l_l)
    m_s = _model(params, dt)                       # sync_bn=True without torch.distributed: the fused step
    l_s = _losses(m_s.train_step(xs, yts, LR, sync_bn=True))
    pf, pl, ps = _params(m_f), _params(m_l), _params(m_s)
    for tag, p, l in (("layered", pl, l_l), ("sync_bn=True, one rank", ps, l_s)):
        upd = _update_err(p, pf, init, layers=(74,))
        mov = _moving_err(p, pf, init)
        loss = float(np.max(np.abs(l - l_f) / np.abs(l_f)))
        print(f"{dt}: {tag} vs fused: layer 74 update {upd:.3g}, moving statistics {mov:.3g}, losses {loss:.3g}")
        assert _moving_err(p, pf, init, layers=(0,)) < R2_MOVING0, "layer 0 moving statistics differ"
        assert upd < W1_UPDATE74[dt] and mov < W1_MOVING[dt] and loss < W1_LOSS[dt]


def _bn_backward_errors(models, slabs_summed=True):
    """Every BN layer's backward on the engine's own tensors against autograd over the CONCATENATED rows of all
    ranks (global batch statistics): each rank's dz, the backward exchange slab [Σdact·ẑ | Σdact] and the dgamma /
    dbeta of the flat gradient (which the lockstep sums over the ranks like the data-parallel all-reduce).  Run after a
    step at lr 0, so the parameters are those the step used.  -> [(layer, dz err, slab err, flat-gradient err)]."""
    rows = []
    plans = [m._last_plan for m in models]
    for i in range(plans[0].num_layers):
        info = plans[0].layer_info(i)
        if not info.has_bn:
            continue
        zs, dAs, dzs = [], [], []
        for plan in plans:
            zs.append(plan.train_buffer(i, "z").double())
            dA = plan.train_buffer(i, "dA").double()
            if info.upsample2x:
                dA = dA[:, 0::2, 0::2] + dA[:, 1::2, 0::2] + dA[:, 0::2, 1::2] + dA[:, 1::2, 1::2]
            dAs.append(dA)
            dz = plan.train_buffer(i, "dz").double()
            dzs.append(dz[:, ::2, ::2] if dz.shape[1] != info.out_h else dz)   # zero-inserted dz (YB_DGRAD_S2=dilated)
        p = plans[0].conv_params(i)
        ga = p["gamma"].double().requires_grad_(True)
        be = p["beta"].double().requires_grad_(True)
        z = torch.cat(zs).requires_grad_(True)
        mu, var = z.mean(dim=(0, 1, 2)), z.var(dim=(0, 1, 2), unbiased=False)
        y = (z - mu) / torch.sqrt(var + 1e-5) * ga + be
        torch.where(y > 0, y, 0.1 * y).backward(torch.cat(dAs))
        e_dz = max(_rel(dz.cpu(), ref.cpu()) for dz, ref in zip(dzs, torch.split(z.grad, [t.shape[0] for t in zs])))
        ref = torch.cat([ga.grad, be.grad]).cpu()
        c, cp = info.cout, plans[0].bn_exchange_buffer(i, backward=True).numel() // 2
        e_slab = max(_rel(torch.cat([s_[:c], s_[cp:cp + c]]).double().cpu(), ref)
                     for s_ in (plan.bn_exchange_buffer(i, backward=True) for plan in plans))
        g = plans[0].layer_grads(i)
        e_flat = _rel(torch.cat([g["gamma"], g["beta"]]).double().cpu(), ref)
        rows.append((i, e_dz, e_slab, e_flat))
    return rows


# Relative-L2 bars of the per-layer check, the 5e-2 of test_gpu_path.py::test_train_backward_self_consistency.  dz is
# stored 16-bit; the engine normalises with statistics its conv epilogue summed from the fp32 accumulators, the
# reference with those of the stored 16-bit z, and Σdact·ẑ nearly cancels at this initialisation.  Measured on an
# H100 over two runs (1 and 2 ranks, bf16 and fp16): dz <= 0.033, slab and flat dgamma/dbeta <= 0.034.  Without the BN exchange,
# or with only the forward slabs exchanged: worst dz 0.29 / 0.40, worst slab 0.91 / 0.90.
DZ_BAR = SUM_BAR = 5e-2


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("ranks", [1, 2])
def test_sync_bn_backward_matches_autograd_on_concatenated_rows(dt, ranks):
    """The backward half of sync BN layer by layer, free of the step's run-to-run noise: bn_bwd_reduce's summed
    slab and bn_bwd_apply's dz with M = replicas x rows, against autograd over all ranks' rows."""
    params, x, ys = _train_case(n=2 * ranks)
    models = [_model(params, dt) for _ in range(ranks)]
    gens = [m.train_step_sync_bn(*_cuda(x, ys, 2 * r, 2 * r + 2), 0.0, bn_replicas=ranks) for r, m in enumerate(models)]
    _lockstep(gens, factor=1.0 / ranks)
    rows = _bn_backward_errors(models)
    print(f"{dt}, {ranks} rank(s): worst BN-backward error vs autograd on the concatenated rows: dz "
          f"{max(r[1] for r in rows):.3g}, slab {max(r[2] for r in rows):.3g}, flat dgamma/dbeta {max(r[3] for r in rows):.3g}")
    bad = [r for r in rows if r[1] > DZ_BAR or r[2] > SUM_BAR or r[3] > SUM_BAR]
    assert not bad, bad[:8]


@pytest.mark.parametrize("exchange", ["none", "forward_only"])
def test_sync_bn_backward_check_sees_a_missing_exchange(exchange):
    """Control of the check above: with no BN exchange (per-rank statistics) or with the forward slabs summed but the
    backward slabs left local, the engine's dz no longer matches the global BN backward."""
    params, x, ys = _train_case(n=4)
    models = [_model(params, "bf16") for _ in range(2)]
    reps = 1 if exchange == "none" else 2
    gens = [m.train_step_sync_bn(*_cuda(x, ys, 2 * r, 2 * r + 2), 0.0, bn_replicas=reps) for r, m in enumerate(models)]
    _lockstep(gens, factor=0.5, exchange_bn=exchange != "none", exchange_bwd=False)
    rows = _bn_backward_errors(models)
    failing = [r for r in rows if r[2] > SUM_BAR]
    print(f"{exchange}: slab fails on {len(failing)} of {len(rows)} BN layers, worst dz {max(r[1] for r in rows):.3g}, "
          f"median dz {float(np.median([r[1] for r in rows])):.3g}, worst slab {max(r[2] for r in rows):.3g}")
    assert len(failing) > len(rows) // 2 and max(r[1] for r in rows) > 2 * DZ_BAR


def _two_rank_case(dt, exchange_bn=True):
    params, x, ys = _train_case(n=4)
    init = _initial(params)
    m_a, m_b = _model(params, dt), _model(params, dt)
    xa, ya = _cuda(x, ys, 0, 2)
    xb, yb = _cuda(x, ys, 2, 4)
    ga = m_a.train_step_sync_bn(xa, ya, LR, bn_replicas=2 if exchange_bn else 1)
    gb = m_b.train_step_sync_bn(xb, yb, LR, bn_replicas=2 if exchange_bn else 1)
    la, lb = _lockstep([ga, gb], factor=0.5, exchange_bn=exchange_bn)
    m_c = _model(params, dt)
    xc, yc = _cuda(x, ys)
    lc = m_c.train_step(xc, yc, LR)
    return init, _params(m_a), _params(m_b), _params(m_c), _losses(la), _losses(lb), _losses(lc)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_two_virtual_ranks_equal_concatenated_batch(dt):
    init, pa, pb, pc, la, lb, lc = _two_rank_case(dt)
    upd = _update_err(pa, pc, init, layers=(74,))
    mov0, mov = _moving_err(pa, pc, init, layers=(0,)), _moving_err(pa, pc, init)
    loss = float(np.max(np.abs((la + lb) / 2 - lc) / np.abs(lc)))
    print(f"{dt}: 2 ranks x 2 vs 1 rank x 4: layer 74 update {upd:.3g}, layer 0 moving {mov0:.3g}, moving statistics "
          f"{mov:.3g}, mean loss {loss:.3g}")
    assert upd < R2_UPDATE74[dt] and mov0 < R2_MOVING0 and mov < R2_MOVING[dt] and loss < R2_LOSS[dt]
    # both ranks normalise with the same summed statistics: identical moving statistics.  The parameters see the same
    # summed gradient, but the optimizer's per-tensor clip norms are fp32 atomic sums, so they agree to rounding.
    assert all(np.array_equal(pa[i][k], pb[i][k]) for i in pa for k in ("mean", "var") if k in pa[i]), "moving statistics differ"
    spread = _update_err(pa, pb, init, layers=range(75))
    print(f"{dt}: parameter update, rank a vs rank b: {spread:.3g} (bit-identical: {spread == 0})")
    assert spread < 1e-5, "the ranks diverged"


@pytest.mark.parametrize("dt", ["bf16"])
def test_without_bn_exchange_misses_concatenated_batch(dt):
    init, pa, pb, pc, la, lb, lc = _two_rank_case(dt, exchange_bn=False)
    mov0, mov = _moving_err(pa, pc, init, layers=(0,)), _moving_err(pa, pc, init)
    print(f"{dt}: per-rank BN statistics (no exchange) vs 1 rank x 4: layer 0 moving {mov0:.3g}, moving statistics "
          f"{mov:.3g}, layer 74 update {_update_err(pa, pc, init, layers=(74,)):.3g}")
    assert mov0 > 10 * R2_MOVING0 and mov > R2_MOVING[dt]
    assert not all(np.array_equal(pa[i]["mean"], pb[i]["mean"]) for i in pa if "mean" in pa[i])


def test_phase_order_is_enforced():
    pkg = _pkg()
    lib, _lib = pkg._lib.lib, pkg._lib
    params, x, ys = _train_case()
    xs, yts = _cuda(x, ys)
    m = _model(params, "bf16")
    with pytest.raises(ValueError):
        m.train_step(xs, yts, LR, sync_bn=True, freeze_bn=True)
    _, _, plan, _, _ = m._train_setup(xs, yts, LR, 0.9, 100.0, "momentum", 0.9, 0.9, 0.999, None, False)
    h, st, px = plan.handle, _lib.stream_handle(), _lib.ptr(xs)
    LOC, GLO = _lib.YB_PHASE_LOCAL, _lib.YB_PHASE_GLOBAL

    def fwd(i, ph, rep=1):
        return lib.yb_net_train_forward_layer(h, px, i, ph, rep, 0.99, None, None, None, 0, st)

    def bad(rc, what=b"out of order"):
        assert rc == -1 and what in lib.yb_last_error_string(), lib.yb_last_error_string()

    bad(fwd(0, GLO))                                   # GLOBAL before its LOCAL
    assert fwd(0, LOC) == 0
    bad(fwd(1, LOC))                                   # layer 0 GLOBAL skipped
    assert fwd(0, GLO) == 0
    bad(fwd(2, LOC))                                   # layer 1 skipped
    bad(fwd(1, LOC, rep=2), b"bn_replicas")            # replicas changed inside a step
    bad(lib.yb_net_train_backward_layer(h, px, 74, LOC, 1, 0, st))
    bad(lib.yb_net_train_loss(h, _lib.ptr(yts[0]), _lib.ptr(yts[1]), _lib.ptr(yts[2]),
                              _lib.fptr(m.anchors.reshape(-1)), 1, 1, 1.0, _lib.ptr(plan.loss4), st))
    p, n = C.c_void_p(), C.c_size_t()
    bad(lib.yb_net_bn_exchange_buffer(h, 58, 0, C.byref(p), C.byref(n)), b"no batch norm")
    assert lib.yb_net_bn_exchange_buffer(h, 57, 1, C.byref(p), C.byref(n)) == 0 and n.value == 2 * 1024
    # the plan still runs a correct step, starting again at layer 0
    init = _initial(params)
    (l_l,) = _lockstep([m.train_step_sync_bn(xs, yts, LR, bn_replicas=1)], factor=1.0)
    m_f = _model(params, "bf16")
    l_f = m_f.train_step(xs, yts, LR)
    upd = _update_err(_params(m), _params(m_f), init, layers=(74,))
    loss = float(np.max(np.abs(_losses(l_l) - _losses(l_f)) / np.abs(_losses(l_f))))
    assert upd < W1_UPDATE74["bf16"] and loss < W1_LOSS["bf16"], (upd, loss)


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from yolov3_tensorflow_b200 import parallel
    parallel.init_from_env("nccl")
    params, x, ys = _train_case(n=4)
    init = _initial(params)
    lo, hi = parallel.shard_batch(4, rank, world)
    xs, yts = _cuda(x, ys, lo, hi)
    m_dp = _model(params, "bf16")
    m_dp.train_step(xs, yts, LR, sync_bn=True)
    dp = _params(m_dp)
    same = True
    for i in sorted(dp):                              # moving statistics: bit-identical on both ranks
        for k in ("mean", "var") if "mean" in dp[i] else ():
            t = torch.from_numpy(dp[i][k]).cuda()
            ws = [torch.empty_like(t) for _ in range(world)]
            dist.all_gather(ws, t)
            same = same and all(torch.equal(ws[0], w) for w in ws)
    spread = 0.0                                      # parameters: equal up to the optimizer's atomic clip norms
    for i in sorted(dp):
        for k in ("w", "gamma", "beta", "b"):
            if k in dp[i]:
                t = torch.from_numpy(dp[i][k] - init[i][k]).cuda()
                ws = [torch.empty_like(t) for _ in range(world)]
                dist.all_gather(ws, t)
                spread = max(spread, _rel(ws[1].cpu(), ws[0].cpu()))
    m_blk = _model(params, "bf16")
    m_blk.train_step(xs, yts, LR, sync_bn=True, bucket_mb=0)
    bucket_err = _update_err(_params(m_blk), dp, init, layers=(74,))
    m_1 = _model(params, "bf16")
    xc, yc = _cuda(x, ys)
    m_1.train_step(xc, yc, LR, data_parallel=False)
    one = _params(m_1)
    err, mov0, mov = _update_err(dp, one, init, layers=(74,)), _moving_err(dp, one, init, (0,)), _moving_err(dp, one, init)
    dist.barrier()
    dist.destroy_process_group()
    q.put((rank, err, mov0, mov, same, bucket_err, spread))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_nccl_sync_bn_equals_single_rank_on_concatenated_batch():
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
    for rank, err, mov0, mov, same, bucket_err, spread in sorted(q.get(timeout=5) for _ in range(2)):
        print(f"rank {rank}: layer 74 update {err:.3g}, layer 0 moving {mov0:.3g}, moving statistics {mov:.3g}, "
              f"bucketed vs blocking layer 74 update {bucket_err:.3g}")
        # not measured on 2 GPUs: the bars of the 2-virtual-rank test (the atomics make bucketed and blocking differ
        # as much as two runs of one step)
        assert err < R2_UPDATE74["bf16"] and mov0 < R2_MOVING0 and mov < R2_MOVING["bf16"] and bucket_err < R2_UPDATE74["bf16"]
        assert same, "ranks hold different moving statistics after the sync-BN step"
        assert spread < 1e-5, f"ranks hold different parameters after the sync-BN step ({spread:.3g})"
