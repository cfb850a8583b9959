"""The loss and optimizer launches of a training step against float64 (tests/train_tail_ref.py).

a. yb_loss_layer on its own, in the plan's storage forms: the benchmark's shapes (batch 32 at 416² and 608², 80
   classes, bf16 dfm with ld 256), fp16 with loss scale 1024, the fp32 dfm, 20 and 1 classes, every (label_smooth,
   focal) pair, 288 x 480 and batch 1.  Logits are normal plus edge values (conf / class at +-20, t_wh <= -105 where
   expf underflows, t_wh >= 21 past the 1e9 clamp); ground truth has 0, 1, 31, 32, 33 and 64+ boxes per image at one
   scale, boxes in the last row and column, mixup weights in [0.5, 1], and m == 0 boxes engineered to an IoU of 0.5
   plus or minus a few bounds with a ground-truth box.  dfm, its pad columns and guard rows after it start as NaN.
   Every gradient column is within its bound, the pad columns are +0, the guard rows keep their bits, loss4 is within
   its bound and a second launch adds to it.
b. The plan's own loss launch (yb_net_train_loss) on the plan's fp32 head maps: each head's dz, its pad column, and
   plan.loss4.  This checks train_loss's wiring (dfm offsets, anchor groups, dfm_ld) as well as the kernel.
c. The optimizer on the plan's gradient from (b): three updates of each kind from yb_net_train_reset_state, with
   grad_scale = 0.5 / loss_scale, clip_norm at the median tensor norm (then 0) and lr large enough that the median
   step is >= 2^12 ulps of w.  Every element of the 222 tensors: w, both slots, the norms (yb_net_opt_norms), w16
   bit for bit, the dgrad weights bit for bit, and ctrl.  Frozen tensors keep every bit even with a NaN gradient, which
   does not skip the step; a NaN or +inf in a trainable element skips it with every bit kept, and the next Adam update
   uses t = applied + 1.  A second plan of another shape on the same arena continues from the state the first left.

"TAIL" lines report the worst err / bound per check and the number of ambiguous ignore-mask boxes."""
import ctypes as C
import math
import time
import zlib

import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests import train_tail_ref as R
from tests.synth import gen_fms
from tests.test_gpu_path import _train_case

pytestmark = pytest.mark.gpu
GUARD = 64                       # guard rows after dfm
GROUP = {0: O.COCO_ANCHORS[6:9], 1: O.COCO_ANCHORS[3:6], 2: O.COCO_ANCHORS[0:3]}


@pytest.fixture(scope="module")
def L():
    from yolov3_tensorflow_b200 import _lib
    return _lib


def _sms(L):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    return s.value


def _report(what, frac):
    print(f"TAIL {what}: worst err/bound {frac:.3f}")


# ------------------------------------------------------------------------------------------------- a. standalone loss
COUNTS = (0, 1, 31, 32, 33, 64, 70)


def _gt(rng, n, h, w, C, scale):
    """y_true of 3 scales: image i has COUNTS[i % 7] boxes at `scale` (anchor 3(2 - scale)'s size, distinct cells, the
    last row and column included) plus a few random boxes; mixup weights in [0.5, 1]."""
    s = (32, 16, 8)[scale]
    gh, gw = h // s, w // s
    aw, ah = GROUP[scale][0]
    ys = [[], [], []]
    for i in range(n):
        k = min(COUNTS[(i + 5) % len(COUNTS)], gh * gw)
        cells = rng.choice(gh * gw, size=k, replace=False)
        if k:
            cells[0] = gh * gw - 1                           # last row and column
        cy, cx = (cells // gw + rng.uniform(0.2, 0.8, k)) * s, (cells % gw + rng.uniform(0.2, 0.8, k)) * s
        bw, bh = aw * rng.uniform(0.9, 1.1, k), ah * rng.uniform(0.9, 1.1, k)
        boxes = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2, rng.uniform(0.5, 1.0, k)], 1)
        labels = rng.integers(0, C, k)
        if i % 3 == 1:
            b2, l2 = O.synth_gt(rng, w, h, C, 6)
            b2[:, 4] = rng.uniform(0.5, 1.0, len(b2))
            boxes, labels = np.concatenate([b2, boxes]), np.concatenate([l2, labels])
        y = O.process_box(boxes.astype(np.float32), labels, [w, h], C, O.COCO_ANCHORS)
        for j in range(3):
            ys[j].append(y[j])
    return [np.stack(y) for y in ys]


def _logits(rng, fm, y, C, scale, img_hw):
    """Edge values, and m == 0 boxes engineered to an IoU of 0.5 (1 + delta) with a concentric ground-truth box."""
    E = 5 + C
    n, gh, gw = fm.shape[:3]
    f = fm.reshape(n, gh, gw, 3, E)
    pos = y[..., 4] != 0
    flat = f.reshape(-1, E)
    pidx, nidx = np.flatnonzero(pos.reshape(-1)), np.flatnonzero(~pos.reshape(-1))
    flat[nidx[::13], 4] = 20.0
    flat[nidx[5::13], 4] = -20.0
    flat[pidx[::3], 5:] = np.where(rng.random((len(pidx[::3]), C)) < 0.5, 20.0, -20.0)
    flat[pidx[1::3], 4] = rng.choice([-20.0, 20.0], len(pidx[1::3]))
    for j, v in enumerate((-105.0, -120.0, 21.0, 25.0, 40.0)):
        flat[nidx[j::29], 2 + (j & 1)] = v
        flat[pidx[j + 2::17], 2 + (j & 1)] = v
    # threshold boxes: at a ground-truth cell, another anchor slot (m == 0)
    ratio_h, ratio_w = img_hw[0] / gh, img_hw[1] / gw
    anchors = np.asarray(GROUP[scale], np.float32)
    deltas = (-3e-4, -1e-4, -3e-5, -3e-6, 3e-6, 3e-5, 1e-4, 3e-4)   # the IoU bound is about 1e-5 of it
    made = 0
    for b, yy, xx, a in zip(*np.nonzero(pos)):
        k = (a + 1) % 3
        if pos[b, yy, xx, k]:
            continue
        gx, gy, gwid, ghei = y[b, yy, xx, a, :4]
        d = deltas[made % len(deltas)]
        sx, sy = (min(max(v, 1e-3), 1 - 1e-3) for v in (gx / ratio_w - xx, gy / ratio_h - yy))
        f[b, yy, xx, k, 0] = math.log(sx / (1 - sx))
        f[b, yy, xx, k, 1] = math.log(sy / (1 - sy))
        f[b, yy, xx, k, 2] = math.log(0.5 * (1 + d) * gwid / anchors[k, 0])
        f[b, yy, xx, k, 3] = math.log(ghei / anchors[k, 1])
        f[b, yy, xx, k, 4] = 0.0
        made += 1
    return made


def _launch(L, fm, yt, anchors, img_hw, cn, ls, fo, loss_scale, code, ld, loss4=None):
    n, gh, gw = fm.shape[:3]
    E = 5 + cn
    need = C.c_size_t()
    L.check(L.lib.yb_loss_workspace_bytes(n, gh, gw, C.byref(need)), "loss_workspace_bytes")
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    rows = n * gh * gw
    if code == L.YB_F32:
        dfm = torch.full(((rows * 3 + GUARD) * E,), math.nan, dtype=torch.float32, device="cuda")
    else:
        dt = torch.float16 if code == L.YB_F16 else torch.bfloat16
        dfm = torch.full((rows + GUARD, ld), math.nan, dtype=dt, device="cuda")
    if loss4 is None:
        loss4 = torch.zeros(4, dtype=torch.float64, device="cuda")
    an = np.asarray(anchors, np.float32).reshape(-1)
    L.check(L.lib.yb_loss_layer(L.ptr(fm), L.ptr(yt), n, gh, gw, img_hw[0], img_hw[1], cn, L.fptr(an), int(ls), int(fo),
                                R.f32(1.0 / n), float(loss_scale), L.ptr(ws), ws.numel(), L.ptr(loss4), L.ptr(dfm), code,
                                ld, L.stream_handle()), "yb_loss_layer")
    return dfm, loss4


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _check_scale(L, cid, res, dfm, code, ld, shape, C, sms):
    n, gh, gw = shape
    E = 5 + C
    rows = n * gh * gw
    dt = {L.YB_F32: torch.float32, L.YB_F16: torch.float16, L.YB_BF16: torch.bfloat16}[code]
    val, bnd, alt, alt_b = R.grad_dense(res, C, dt)
    if dt != torch.float32:
        assert float(val.abs().max()) < 0.99 * float(torch.finfo(dt).max), f"{cid}: the gradient overflows {dt}"
    if code == L.YB_F32:
        got = dfm[:rows * 3 * E].view(n, gh, gw, 3, E)
        guard = dfm[rows * 3 * E:]
    else:
        got = dfm[:rows, :3 * E].reshape(n, gh, gw, 3, E)
        pad = dfm[:rows, 3 * E:]
        assert bool((_bits(pad) == 0).all()), f"{cid}: pad columns are not +0"
        guard = dfm[rows:]
    assert bool(torch.isnan(guard).all()) and bool((_bits(guard) == _bits(torch.full_like(guard, math.nan))).all()), \
        f"{cid}: guard rows after dfm were written"
    return R.check_grad(got, val, bnd, alt, alt_b, f"{cid} gradient")


LOSS_CONFIGS = [   # (id, n, (H, W), classes, label_smooth, focal, dfm dtype, loss_scale)
    ("b32-416-bf16", 32, (416, 416), 80, True, True, "bf16", 1.0),
    ("b32-608-bf16", 32, (608, 608), 80, True, True, "bf16", 1.0),
    ("b32-416-fp16", 32, (416, 416), 80, True, True, "fp16", 1024.0),
    ("b32-416-fp32", 32, (416, 416), 80, True, True, "fp32", 1.0),
    ("c20-bf16", 8, (416, 416), 20, True, True, "bf16", 1.0),
    ("c1-fp16", 8, (416, 416), 1, True, True, "fp16", 1024.0),
    ("flags00-fp32", 8, (416, 416), 80, False, False, "fp32", 1.0),
    ("flags10-fp32", 8, (416, 416), 80, True, False, "fp32", 1.0),
    ("flags01-fp32", 8, (416, 416), 80, False, True, "fp32", 1.0),
    ("288x480-bf16", 8, (288, 480), 80, True, True, "bf16", 1.0),
    ("b1-fp16", 1, (416, 416), 80, True, True, "fp16", 1024.0),
]


@pytest.mark.parametrize("cid,n,hw,C_,ls,fo,dt,lscale", LOSS_CONFIGS, ids=[c[0] for c in LOSS_CONFIGS])
def test_loss_layer_against_float64(L, cid, n, hw, C_, ls, fo, dt, lscale):
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    sms = _sms(L)
    rng = np.random.default_rng(zlib.crc32(cid.encode()))
    code = {"bf16": L.YB_BF16, "fp16": L.YB_F16, "fp32": L.YB_F32}[dt]
    E = 5 + C_
    ld = 0 if code == L.YB_F32 else -(-3 * E // 32) * 32
    eng_scale = 2
    ys = _gt(rng, n, hw[0], hw[1], C_, eng_scale)
    fms = gen_fms(int(rng.integers(1 << 30)), n, hw[0], hw[1], C_, scale=1.5)
    worst, worst_l, namb, made, decided = 0.0, 0.0, 0, 0, 0
    for s in range(3):
        k = _logits(rng, fms[s], ys[s], C_, s, hw)
        fm, yt = torch.from_numpy(fms[s]).cuda(), torch.from_numpy(ys[s]).cuda()
        gm = R.f32(R.f32(1.0 / n) * lscale)
        res = R.loss_eval(R.F64, fm, yt, GROUP[s], hw, C_, ls, fo, gm)
        dfm, loss4 = _launch(L, fm, yt, GROUP[s], hw, C_, ls, fo, lscale, code, ld)
        shape = fm.shape[:3]
        worst = max(worst, _check_scale(L, f"{cid} scale {s}", res, dfm, code, ld, shape, C_, sms))
        v4, b4 = R.loss4_ref(res, fm.shape[0] * fm.shape[1] * fm.shape[2] * 3, C_, R.f32(1.0 / n), sms)
        got = loss4.cpu().numpy()
        assert np.all(np.abs(got - v4) <= b4), f"{cid} scale {s}: loss4 {got} ref {v4} bound {b4}"
        worst_l = max(worst_l, float(np.max(np.abs(got - v4) / b4)))
        _launch(L, fm, yt, GROUP[s], hw, C_, ls, fo, lscale, code, ld, loss4)       # accumulates
        got2 = loss4.cpu().numpy()
        assert np.all(np.abs(got2 - 2 * v4) <= 2 * b4), f"{cid} scale {s}: second launch {got2} ref {2 * v4}"
        namb += int(res["amb"].sum())
        if s == eng_scale:
            # the engineered threshold boxes: most are decided, on both sides of 0.5
            f = fm.view(*res["amb"].shape, E)
            eng = (f[..., 4] == 0) & ~res["pos"]
            decided = int((eng & ~res["amb"]).sum())
            sides = set(res["ign"][eng & ~res["amb"]].tolist())
            assert sides == {0.0, 1.0}, f"{cid}: the decided threshold boxes fall on one side of 0.5 only: {sides}"
            namb -= int((eng & res["amb"]).sum())
            made = k
        del res
    nbox = sum(f.size // E for f in fms)
    assert namb <= max(4, nbox // 20000), f"{cid}: {namb} ambiguous ignore-mask boxes"
    assert made >= 30 and decided >= made // 2, (made, decided)
    _report(f"{cid} loss gradient ({dt})", worst)
    _report(f"{cid} loss4", worst_l)
    print(f"TAIL {cid}: {namb} ambiguous ignore-mask boxes of {nbox} besides the threshold boxes, {made - decided} of "
          f"{made} threshold boxes ambiguous, "
          f"{time.time() - t0:.1f} s, peak CUDA memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------------------- b. the plan's loss launch
PLAN_CONFIGS = [   # (id, dtype, n, (H, W), classes)
    ("plan-fp16", "fp16", 8, (416, 416), 80),
    ("plan-bf16", "bf16", 8, (416, 416), 80),
    ("plan-bf16-c20", "bf16", 2, (288, 480), 20),
]


class Run:
    def __init__(self, L, dt, n, hw, C_):
        import yolov3_tensorflow_b200 as pkg
        self.L, self.n, self.hw, self.C = L, n, hw, C_
        params, x, ys = _train_case(seed=43, n=n, h=hw[0], w=hw[1], cn=C_)
        self.m = pkg.yolov3(C_, O.COCO_ANCHORS, use_label_smooth=True, use_focal_loss=True, batch_norm_decay=0.99,
                            dtype=dt)
        self.m.set_params(params, "HWIO")
        self.x = torch.from_numpy(x).cuda()
        self.ys = [torch.from_numpy(y).cuda() for y in ys]
        self.m._train_setup(self.x, self.ys, 0.0, 0.9, 100.0, "momentum", 0.9, 0.9, 0.999, None, False)
        self.plan = self.m._plan(n, hw[0], hw[1], training=True)
        self.heads = [i for i in range(self.plan.num_layers) if not self.plan.layer_info(i).has_bn]

    def dz_full(self, i):
        dz = self.plan.train_buffer(i, "dz")
        n, h, w, _ = dz.shape
        return dz.as_strided((n, h, w, dz.stride(2)), dz.stride(), dz.storage_offset())

    def forward_loss(self):
        L, m, plan = self.L, self.m, self.plan
        h, st, px = plan.handle, L.stream_handle(), L.ptr(self.x)
        for i in range(plan.num_layers):
            for ph in (L.YB_PHASE_LOCAL, L.YB_PHASE_GLOBAL):
                L.check(L.lib.yb_net_train_forward_layer(h, px, i, ph, 1, 0.99, None, None, None, 0, st), "forward")
        for i in self.heads:
            self.dz_full(i).fill_(math.nan)
        L.check(L.lib.yb_net_train_loss(h, L.ptr(self.ys[0]), L.ptr(self.ys[1]), L.ptr(self.ys[2]),
                                        L.fptr(m.anchors.reshape(-1)), 1, 1, float(m.loss_scale), L.ptr(plan.loss4), st),
                "train_loss")
        torch.cuda.synchronize()

    def backward(self):
        L, plan = self.L, self.plan
        h, st, px = plan.handle, L.stream_handle(), L.ptr(self.x)
        for i in range(plan.num_layers - 1, -1, -1):
            for ph in (L.YB_PHASE_LOCAL, L.YB_PHASE_GLOBAL):
                L.check(L.lib.yb_net_train_backward_layer(h, px, i, ph, 1, 0, st), "backward")
        L.check(L.lib.yb_net_train_join(h, st), "train_join")
        torch.cuda.synchronize()

    def check_loss(self, cid):
        plan, C_ = self.plan, self.C
        E = 5 + C_
        tot_v, tot_b, worst, namb = np.zeros(4), np.zeros(4), 0.0, 0
        sms = _sms(self.L)
        gm = R.f32(R.f32(1.0 / self.n) * float(self.m.loss_scale))
        for s, i in enumerate(self.heads):
            fm = plan.layer_output(i).contiguous()
            res = R.loss_eval(R.F64, fm, self.ys[s], GROUP[s], self.hw, C_, True, True, gm)
            dt = plan.act_dtype
            val, bnd, alt, alt_b = R.grad_dense(res, C_, dt)
            full = self.dz_full(i)
            assert full.shape[3] == -(-3 * E // 32) * 32, f"{cid} layer {i}: dz ld {full.shape[3]}"
            assert bool((_bits(full[..., 3 * E:]) == 0).all()), f"{cid} layer {i}: dz pad columns are not +0"
            got = full[..., :3 * E].reshape(val.shape)
            worst = max(worst, R.check_grad(got, val, bnd, alt, alt_b, f"{cid} layer {i} dz"))
            v4, b4 = R.loss4_ref(res, val[..., 0].numel(), C_, R.f32(1.0 / self.n), sms)
            tot_v += v4
            tot_b += b4
            namb += int(res["amb"].sum())
            del res, val, bnd
        got = plan.loss4.cpu().numpy()
        assert np.all(np.abs(got - tot_v) <= tot_b), f"{cid}: plan.loss4 {got} ref {tot_v} bound {tot_b}"
        _report(f"{cid} head dz ({plan.act_dtype})", worst)
        _report(f"{cid} loss4", float(np.max(np.abs(got - tot_v) / tot_b)))
        print(f"TAIL {cid}: {namb} ambiguous ignore-mask boxes")


# ------------------------------------------------------------------------------------------- c. the optimizer
class State:
    """Flat views of the 222 tensors of a plan in the optimizer's order (yb_net_opt_norms)."""

    def __init__(self, run):
        plan = run.plan
        self.run = run
        gflat = plan.grad_flat()
        base = gflat.data_ptr()
        idx, seg, l2, self.layer_of = [], [], [], []
        for i in range(plan.num_layers):
            for k, g in plan.layer_grads(i).items():
                off = (g.data_ptr() - base) // 4
                seg.append(torch.full((g.numel(),), len(l2), dtype=torch.long, device="cuda"))
                idx.append(torch.arange(off, off + g.numel(), device="cuda"))
                l2.append(k == "w")
                self.layer_of.append((i, k))
        self.idx, self.seg = torch.cat(idx), torch.cat(seg)
        self.l2 = torch.tensor(l2, device="cuda")
        self.T = len(l2)
        sizes = torch.zeros(self.T, dtype=torch.long, device="cuda").index_add_(0, self.seg, torch.ones_like(self.seg))
        self.sizes = sizes
        self.chunks = (sizes + 65535) // 65536

    def w(self):
        plan = self.run.plan
        return torch.cat([plan.conv_params(i)[k].reshape(-1) for i, k in self.layer_of])

    def snap(self):
        slots, ctrl = self.run.m.optimizer_state()
        g = self.run.plan.grad_flat()
        return dict(w=self.w(), v1=slots[0][self.idx].clone(), v2=slots[1][self.idx].clone(), g=g[self.idx].clone(),
                    ctrl=ctrl.clone().cpu().tolist(), w16=self.w16(), wd=self.wdgrad())

    def w16(self):
        plan = self.run.plan
        return [plan.train_buffer(i, "w16").clone() for i in range(1, plan.num_layers)]

    def wdgrad(self):
        plan = self.run.plan
        return [plan.dgrad_weights(i).clone() for i in range(1, plan.num_layers)]


def _opt(L, kind, lr, gs, clip):
    return L.Optimizer(kind=R.KINDS[kind], lr=lr, grad_scale=gs, momentum=0.9, decay=0.9, beta1=0.9, beta2=0.999,
                       epsilon=1e-10 if kind == "rmsprop" else 1e-8, weight_decay=5e-4, clip_norm=clip)


def _o(opt):
    return {k: float(getattr(opt, k)) for k in ("lr", "grad_scale", "momentum", "decay", "beta1", "beta2", "epsilon",
                                                "weight_decay", "clip_norm")}


def _update(L, plan, opt):
    L.check(L.lib.yb_net_train_update(plan.handle, C.byref(opt), L.stream_handle()), "train_update")
    torch.cuda.synchronize()


def _check_update(L, S, plan, kind, opt, before, trainable, worst, cid):
    """After an update through `plan`: every element against the reference from `before`."""
    slots, ctrl = S.run.m.optimizer_state()
    applied = before["ctrl"][1]
    assert ctrl.cpu().tolist() == [0, applied + 1, before["ctrl"][2]], f"{cid}: ctrl {ctrl.cpu().tolist()}"
    tr = trainable[S.seg]
    sel = tr.nonzero().squeeze(1)
    tsel = trainable.nonzero().squeeze(1)
    # the reference over the trainable tensors, renumbered densely
    remap = torch.cumsum(trainable.long(), 0) - 1
    sq, nw, n1, n2 = R.opt_eval(R.F64, kind, before["w"][sel], before["g"][sel], before["v1"][sel], before["v2"][sel],
                                remap[S.seg[sel]], S.l2[tsel], S.chunks[tsel], _o(opt), applied)
    norms = plan.opt_norms()
    assert norms.numel() == S.T
    worst["sqnorm"] = max(worst.get("sqnorm", 0), R.check_ev(norms[tsel], sq, f"{cid} {kind} sqnorm"))
    assert bool((norms[~trainable] == 0).all()), f"{cid}: a frozen tensor has a norm"
    w = S.w()
    worst["w"] = max(worst.get("w", 0), R.check_ev(w[sel], nw, f"{cid} {kind} w"))
    if kind != "sgd":
        worst["slot 1"] = max(worst.get("slot 1", 0), R.check_ev(slots[0][S.idx][sel], n1, f"{cid} {kind} slot 1"))
    if kind in ("rmsprop", "adam"):
        worst["slot 2"] = max(worst.get("slot 2", 0), R.check_ev(slots[1][S.idx][sel], n2, f"{cid} {kind} slot 2"))
    fro = (~tr).nonzero().squeeze(1)
    for name, now in (("w", w), ("slot 1", slots[0][S.idx]), ("slot 2", slots[1][S.idx])):
        key = {"w": "w", "slot 1": "v1", "slot 2": "v2"}[name]
        if kind == "sgd" and name != "w" or kind == "momentum" and name == "slot 2":
            fro_sel = torch.arange(now.numel(), device="cuda")      # untouched slots: every element
        else:
            fro_sel = fro
        assert bool((_bits(now[fro_sel]) == _bits(before[key][fro_sel])).all()), f"{cid} {kind}: {name} of a frozen tensor or an unused slot changed"
    # 16-bit copies: RN16 of the new masters, bit for bit; frozen layers keep theirs
    plan_ = S.run.plan
    dt = plan_.act_dtype
    for li in range(1, plan_.num_layers):
        info = plan_.layer_info(li)
        w16 = plan_.train_buffer(li, "w16")
        want = torch.zeros_like(w16)
        want[:info.cout] = plan_.conv_params(li)["w"].reshape(info.cout, -1).to(dt)
        bad = int((_bits(w16) != _bits(want)).sum())
        assert bad == 0, f"{cid} {kind}: layer {li}: {bad} elements of w16 differ from RN16(w)"
        if info.stride == 1:
            k, kco = info.ksize, -(-info.cout // 32) * 32
            cin_pad = L.lib.yb_conv_cout_pad(info.cin)
            wd = torch.zeros((cin_pad, k, k, kco), dtype=dt, device="cuda")
            wd[:info.cin, :, :, :info.cout] = plan_.conv_params(li)["w"].to(dt).flip(1, 2).permute(3, 1, 2, 0)
            bad = int((_bits(plan_.dgrad_weights(li)) != _bits(wd.reshape(-1))).sum())
            assert bad == 0, f"{cid} {kind}: layer {li}: {bad} dgrad weights differ from flip + transpose of RN16(w)"


def _unchanged(S, before, cid):
    after = S.snap()
    for k in ("w", "v1", "v2"):
        assert bool((_bits(after[k]) == _bits(before[k])).all()), f"{cid}: {k} changed on a skipped step"
    for a, b in zip(after["w16"] + after["wd"], before["w16"] + before["wd"]):
        assert bool((_bits(a) == _bits(b)).all()), f"{cid}: a 16-bit weight copy changed on a skipped step"
    return after


def _lr_for(S, kind, before, opt, trainable):
    """lr that makes the median step >= 2^12 ulps of w (the update is linear in lr from these slots)."""
    o = _o(opt)
    o["lr"] = 1.0
    sel = trainable[S.seg].nonzero().squeeze(1)
    remap = torch.cumsum(trainable.long(), 0) - 1
    tsel = trainable.nonzero().squeeze(1)
    _, nw, n1, _ = R.opt_eval(R.F64, kind, before["w"][sel], before["g"][sel], before["v1"][sel], before["v2"][sel],
                              remap[S.seg[sel]], S.l2[tsel], S.chunks[tsel], o, before["ctrl"][1])
    step1 = (n1.v if kind == "rmsprop" else before["w"][sel].double() - nw.v).abs()
    w = before["w"][sel].double().abs()
    ulpw = torch.exp2(torch.floor(torch.log2(w.clamp(min=2.0 ** -126))) - 23)
    ratio = (ulpw / step1)[step1 > 0]
    return 2.0 ** round(math.log2(float(ratio.median()) * 2 ** 13))


@pytest.mark.parametrize("cid,dt,n,hw,C_", PLAN_CONFIGS, ids=[c[0] for c in PLAN_CONFIGS])
def test_plan_loss_and_optimizer_against_float64(L, cid, dt, n, hw, C_):
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    run = Run(L, dt, n, hw, C_)
    run.forward_loss()
    run.check_loss(cid)
    if C_ != 80:
        return
    run.backward()
    S = State(run)
    assert S.T == 222
    grad = run.plan.grad_flat().clone()
    assert bool(torch.isfinite(grad).all())
    gs = R.f32(0.5 / float(run.m.loss_scale))
    plan = run.plan
    worst = {}
    allt = torch.ones(S.T, dtype=torch.bool, device="cuda")
    for kind in ("momentum", "sgd", "rmsprop", "adam"):
        L.check(L.lib.yb_net_train_reset_state(plan.handle, R.KINDS[kind], L.stream_handle()), "reset_state")
        run.m._opt_kind = R.KINDS[kind]
        plan.grad_flat().copy_(grad)                          # reset_state zeroes the gradient buffer
        lr, clip = None, None
        for step in range(3):
            before = S.snap()
            if clip is None:
                g = before["g"].double() * gs + torch.where(S.l2[S.seg], R.f32(5e-4), 0.0) * before["w"].double()
                nrm = torch.zeros(S.T, dtype=torch.float64, device="cuda").index_add_(0, S.seg, g * g).sqrt()
                srt = nrm.sort().values
                clip = R.f32(math.sqrt(float(srt[S.T // 2 - 1] * srt[S.T // 2])))
                lr = _lr_for(S, kind, before, _opt(L, kind, 1.0, gs, clip), allt)
            opt = _opt(L, kind, lr, gs, clip if step < 2 else 0.0)
            _update(L, plan, opt)
            _check_update(L, S, plan, kind, opt, before, allt, worst, f"{cid} step {step}")
    # adam continues: frozen tensors, with a NaN gradient in one of them
    frozen = [5, 66]
    run.m.set_trainable(frozen, False)
    tr = torch.tensor([li not in frozen for li, _ in S.layer_of], device="cuda")
    gflat = plan.grad_flat()
    fidx = int(S.idx[(S.seg == [t for t, (li, k) in enumerate(S.layer_of) if li == 5][0]).nonzero()[0, 0]])
    keep = gflat[fidx].clone()
    gflat[fidx] = math.nan
    before = S.snap()
    opt = _opt(L, "adam", lr, gs, clip)
    _update(L, plan, opt)
    _check_update(L, S, plan, "adam", opt, before, tr, worst, f"{cid} frozen")
    gflat[fidx] = keep
    run.m.set_trainable(frozen, True)
    # skipped steps: NaN, then +inf, in the first chunk of a multi-chunk tensor and in the last element of the last tensor
    big = int((S.chunks > 1).nonzero()[0, 0])
    for at in (int(S.idx[(S.seg == big).nonzero()[5, 0]]), int(S.idx[-1])):
        for bad in (math.nan, math.inf):
            keep = gflat[at].clone()
            gflat[at] = bad
            before = S.snap()
            _update(L, plan, _opt(L, "adam", lr, gs, clip))
            _unchanged(S, before, f"{cid} skipped ({bad} at {at})")
            c = run.m.optimizer_state()[1].cpu().tolist()
            assert c == [0, before["ctrl"][1], before["ctrl"][2] + 1], f"{cid}: ctrl {c} after a skipped step"
            gflat[at] = keep
    before = S.snap()
    opt = _opt(L, "adam", lr, gs, clip)
    _update(L, plan, opt)
    _check_update(L, S, plan, "adam", opt, before, allt, worst, f"{cid} after skips")
    # a second plan of another shape on the same arena continues from this state
    plan2 = run.m._plan(1, 288, 480, training=True)
    assert plan2.par.data_ptr() == plan.par.data_ptr()
    before = S.snap()
    opt = _opt(L, "adam", lr, gs, clip)
    _update(L, plan2, opt)
    _check_update(L, S, plan2, "adam", opt, before, allt, worst, f"{cid} second plan")
    for k, v in worst.items():
        _report(f"{cid} optimizer {k}", v)
    print(f"TAIL {cid}: {time.time() - t0:.1f} s, peak CUDA memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
