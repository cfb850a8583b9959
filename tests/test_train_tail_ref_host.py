"""CPU tests of tests/train_tail_ref.py, the float64 reference of the loss kernel and the optimizer.

  - its loss values and hand-written gradient agree with the oracle's autograd (TF autodiff restated) in float64, over
    the four (label_smooth, focal) combinations, mixup weights below 1, an image without boxes, and logits that take
    the pw_zero branch, both clamps and the saturated sigmoid;
  - its update agrees with oracle.train_step's rules for momentum, sgd, rmsprop and adam from non-zero slots, with
    clip_by_norm engaged on some tensors;
  - a plain float32 evaluation of the same formulas stays inside the bounds, and mutations of the kind a kernel bug
    would make fall outside them."""
import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests import train_tail_ref as R
from tests.synth import gen_fms

H, W = 96, 128
GROUPS = [O.COCO_ANCHORS[6:9], O.COCO_ANCHORS[3:6], O.COCO_ANCHORS[0:3]]


def _case(C=80, n=3, seed=5):
    """Logits with edge values and ground truth with mixup weights in [0.5, 1]; image n - 1 has no boxes."""
    rng = np.random.default_rng(seed)
    fms = gen_fms(seed, n, H, W, C, scale=1.5)
    ys = [[], [], []]
    for i in range(n):
        if i == n - 1:
            boxes, labels = np.zeros((0, 5), np.float32), np.zeros(0, np.int64)
        else:
            boxes, labels = O.synth_gt(rng, W, H, C, 12)
            boxes[:, 4] = rng.uniform(0.5, 1.0, len(boxes))
        y = O.process_box(boxes, labels, [W, H], C, O.COCO_ANCHORS)
        for j in range(3):
            ys[j].append(y[j])
    ys = [np.stack(y) for y in ys]
    E = 5 + C
    for s in range(3):
        f = fms[s].reshape(*fms[s].shape[:3], 3, E)
        pos = ys[s][..., 4] != 0
        flat = np.flatnonzero(pos.reshape(-1))
        neg = np.flatnonzero(~pos.reshape(-1))
        ff = f.reshape(-1, E)
        # positives: pw_zero (exp underflows in float32 and float64 alike), lower and upper clamp
        for k, idx in enumerate(flat[:6]):
            ff[idx, 2 + (k & 1)] = (-800.0, -30.0, 22.0)[k // 2]
        # saturated conf / class logits, and pw_zero on negatives
        ff[neg[::7], 4] = 20.0
        ff[neg[3::7], 4] = -20.0
        ff[flat[::2], 5:] = np.where(rng.random((len(flat[::2]), C)) < 0.5, 20.0, -20.0)
        ff[neg[5::11], 2] = -800.0
    return fms, ys


def _ours(be, fms, ys, C, ls, fo, n):
    inv_n = R.f32(1.0 / n)
    return [R.loss_eval(be, torch.from_numpy(fms[s]), torch.from_numpy(ys[s]), GROUPS[s], (H, W), C, ls, fo, inv_n)
            for s in range(3)]


def _dense32(res, C):
    g = res["g"]
    shape = g[0].shape
    out = torch.zeros(shape + (5 + C,), dtype=torch.float64)
    for j in range(5):
        out[..., j] = g[j].double()
    cv = out[..., 5:]
    cv[res["pos"]] = res["cls_g"].double()
    return out


@pytest.mark.parametrize("ls,fo", [(False, False), (True, False), (False, True), (True, True)])
def test_loss_reference_matches_oracle_autograd(ls, fo):
    C, n = 80, 3
    fms, ys = _case(C, n)
    ref = _ours(R.F64, fms, ys, C, ls, fo, n)
    losses, grads = O.loss_and_grad(fms, ys, O.COCO_ANCHORS, (H, W), C, ls, fo, dtype=torch.float64)
    tot = np.zeros(4)
    bnd = np.zeros(4)
    namb = 0
    for s in range(3):
        val, b, alt, alt_b = R.grad_dense(ref[s], C)
        og = torch.from_numpy(grads[s]).reshape(val.shape)
        R.check_grad(og, val, b, alt, alt_b, f"scale {s} oracle autograd vs reference")
        v4, b4 = R.loss4_ref(ref[s], val[..., 0].numel(), C, R.f32(1.0 / n))
        tot += v4
        bnd += b4
        namb += int(ref[s]["amb"].sum())
    assert namb == 0
    assert np.all(np.abs(np.array(losses[1:]) - tot) <= bnd), (losses[1:], tot, bnd)
    # the edge branches were taken
    y0 = ys[0]
    assert bool((torch.from_numpy(fms[0]).reshape(*y0.shape[:4], -1)[..., 2] == -800).any())


def test_loss_float32_evaluation_inside_bounds_and_mutations_outside():
    C, n = 80, 3
    fms, ys = _case(C, n, seed=9)
    worst = 0.0
    for ls, fo in ((True, True), (False, False)):
        ref = _ours(R.F64, fms, ys, C, ls, fo, n)
        f32 = _ours(R.F32, fms, ys, C, ls, fo, n)
        for s in range(3):
            val, b, alt, alt_b = R.grad_dense(ref[s], C)
            worst = max(worst, R.check_grad(_dense32(f32[s], C), val, b, alt, alt_b, f"scale {s} float32"))
            for k in range(4):
                t64, t32 = ref[s]["loss"][k], f32[s]["loss"][k]
                keep = ~ref[s]["amb"] if k == 2 else torch.ones_like(t32, dtype=torch.bool)
                assert bool(((t32.double() - t64.v).abs() <= t64.e.expand_as(t64.v))[keep].all()), (s, k)
            for dt in (torch.float16, torch.bfloat16):
                val16, b16, alt, alt_b = R.grad_dense(ref[s], C, dt)
                got16 = _dense32(f32[s], C).to(dt)
                R.check_grad(got16, val16, b16, alt, alt_b, f"scale {s} {dt}")
    assert 0 < worst <= 1.0
    # mutations a kernel bug would make are outside the fp32 bounds
    ref = _ours(R.F64, fms, ys, C, True, True, n)
    plain = _ours(R.F64, fms, ys, C, False, True, n)
    nofocal = _ours(R.F64, fms, ys, C, True, False, n)
    s = 2
    val, b, alt, alt_b = R.grad_dense(ref[s], C)
    pos = ref[s]["pos"]
    mix = torch.from_numpy(ys[s][..., -1]).double()
    f = torch.sigmoid(torch.from_numpy(fms[s]).reshape(val.shape)[..., 4:5].double())
    focal = (torch.from_numpy(ys[s][..., 4:5]).double() - f) ** 2
    mutants = {
        "class gradient without mix": torch.where(pos[..., None] & (mix[..., None] < 1), val / mix[..., None], val),
        "label smoothing missing from the class gradient": torch.cat([val[..., :5], R.grad_dense(plain[s], C)[0][..., 5:]], -1),
        "focal term 2 f s (1 - s) bce dropped": torch.cat([val[..., :4], R.grad_dense(nofocal[s], C)[0][..., 4:5] * focal,
                                                           val[..., 5:]], -1),
    }
    for name, mv in mutants.items():
        with pytest.raises(AssertionError):
            R.check_grad(mv, val, b, alt, alt_b, name)


# ----------------------------------------------------------------------------------------------------------- optimizer
def _oracle_case(seed=3):
    params = O.make_params(80, seed=seed, random_bn=True)
    rng = np.random.default_rng(seed)
    x = rng.random((1, 32, 32, 3), dtype=np.float32)
    boxes, labels = O.synth_gt(rng, 32, 32, 80, 3)
    ys = [y[None] for y in O.process_box(boxes, labels, [32, 32], 80, O.COCO_ANCHORS)]
    return params, x, ys


@pytest.fixture(scope="module")
def oracle_grads():
    params, x, ys = _oracle_case()
    vel = [{k: np.zeros_like(v) for k, v in p.items() if k in ("w", "gamma", "beta", "b")} for p in params]
    _, grads, _, _ = O.train_step(x, ys, params, vel, 0.0, O.COCO_ANCHORS, 80, dtype=torch.float64)
    return params, x, ys, grads


def _flat(params, grads, wd):
    """Flat w, data gradient (the L2 term removed), segment ids and L2 flags in the optimizer's tensor order."""
    ws, gs, seg, l2, keys = [], [], [], [], []
    for li, (p, g) in enumerate(zip(params, grads)):
        for k in ("w", "gamma", "beta", "b"):
            if k not in g:
                continue
            w = torch.from_numpy(np.asarray(p[k], np.float32)).reshape(-1)
            gr = torch.from_numpy(g[k]).reshape(-1)
            if k == "w":
                gr = gr - wd * w.double()
            seg.append(torch.full((w.numel(),), len(keys), dtype=torch.long))
            ws.append(w)
            gs.append(gr.float())
            l2.append(k == "w")
            keys.append((li, k))
    return torch.cat(ws), torch.cat(gs), torch.cat(seg), torch.tensor(l2), keys


@pytest.mark.parametrize("kind", ["momentum", "sgd", "rmsprop", "adam"])
def test_update_reference_matches_oracle_rules(oracle_grads, kind):
    params, x, ys, grads = oracle_grads
    wd = R.f32(5e-4)
    w, g, seg, l2, keys = _flat(params, grads, wd)
    assert len(keys) == 222
    T = len(keys)
    nrm = torch.zeros(T, dtype=torch.float64).index_add_(0, seg, (g.double() + torch.where(l2[seg], wd, 0.0) * w.double()) ** 2).sqrt()
    clip = R.f32(float(nrm.median()) * 1.01)
    assert 50 < int((nrm > clip).sum()) < 170
    rng = np.random.default_rng(11)
    v1 = torch.from_numpy(rng.standard_normal(w.numel()).astype(np.float32) * 1e-3)
    v2 = torch.from_numpy(rng.uniform(0.5, 1.5, w.numel()).astype(np.float32) * (1e-4 if kind == "adam" else 1.0))
    o = dict(lr=2.0 ** -10, grad_scale=1.0, momentum=R.f32(0.9), decay=R.f32(0.9), beta1=R.f32(0.9), beta2=R.f32(0.999),
             epsilon=R.f32(1e-10 if kind == "rmsprop" else 1e-8), weight_decay=wd, clip_norm=clip)
    chunks = torch.zeros(T, dtype=torch.long).index_add_(0, seg, torch.ones_like(seg))
    chunks = (chunks + 65535) // 65536
    _, nw, n1, n2 = R.opt_eval(R.F64, kind, w, g, v1, v2, seg, l2, chunks, o, applied=2)

    def unflat(t):
        out, at = [], 0
        for li, p in enumerate(params):
            d = {}
            for k in ("w", "gamma", "beta", "b"):
                if k in p:
                    d[k] = t[at: at + p[k].size].reshape(p[k].shape).numpy()
                    at += p[k].size
            out.append(d)
        return out
    s2 = unflat(v2) if kind in ("rmsprop", "adam") else None
    _, _, new_p, new_v = O.train_step(x, ys, params, unflat(v1), o["lr"], O.COCO_ANCHORS, 80, dtype=torch.float64,
                                      optimizer=kind, clip=clip, weight_decay=wd, momentum=o["momentum"],
                                      decay=o["decay"], beta1=o["beta1"], beta2=o["beta2"], epsilon=o["epsilon"],
                                      slot2=s2, step=2)
    ow = torch.cat([torch.from_numpy(np.asarray(new_p[li][k])).reshape(-1) for li, k in keys])
    frac = R.check_ev(ow, nw, f"{kind}: oracle w vs reference")
    if kind != "sgd":
        ov = new_v[0] if kind in ("rmsprop", "adam") else new_v
        R.check_ev(torch.cat([torch.from_numpy(np.asarray(ov[li][k])).reshape(-1) for li, k in keys]), n1, f"{kind} slot 1")
    if kind in ("rmsprop", "adam"):
        R.check_ev(torch.cat([torch.from_numpy(np.asarray(new_v[1][li][k])).reshape(-1) for li, k in keys]), n2, f"{kind} slot 2")
    assert frac <= 1.0
    # float32 evaluation inside the bounds; the step is resolvable: a 1 % error of it leaves them
    sq32, nw32, n132, n232 = R.opt_eval(R.F32, kind, w, g, v1, v2, seg, l2, chunks, o, applied=2)
    sq64 = R.opt_eval(R.F64, kind, w, g, v1, v2, seg, l2, chunks, o, applied=2)[0]
    R.check_ev(sq32, sq64, f"{kind} float32 sqnorm")
    R.check_ev(nw32, nw, f"{kind} float32 w")
    R.check_ev(n132, n1, f"{kind} float32 slot 1")
    R.check_ev(n232, n2, f"{kind} float32 slot 2")
    step = nw.v - w.double()
    with pytest.raises(AssertionError):
        R.check_ev(w.double() + 1.01 * step, nw, "1 % step error")
