"""Float64 references and derived per-element bounds for the two ends of a training step: the loss kernel
(csrc/loss.cu: loss_kernel and loss_pad_kernel, run once per scale by net_train.cu's train_loss) and the multi-tensor
optimizer (csrc/optim.cu: opt_norm_kernel, opt_update_kernel and opt_finish_kernel over the chunk table train_bind
builds).  tests/test_train_tail_ref_host.py ties the formulas to the oracle; tests/test_gpu_train_tail.py holds the
kernels to the bounds.

Error model.  Every quantity is an `Ev`: its value, evaluated in float64 on the kernel's own float32 inputs, and a bound
e on |(the kernel's float32 result) - value|.  Each fp32 operation of the kernel is one Ev operation, in the kernel's
order.  It adds the error it propagates (first order in the input bounds, plus e_a e_b for a product) to the rounding
it commits (u = 2^-24, TINY = 2^-149 the fp32 subnormal spacing, r the result):
  - +, -, *, / and sqrtf are correctly rounded (build.sh passes no --use_fast_math): u (|r| + e) + TINY / 2;
  - the default -fmad=true lets the compiler contract any a * b + c into one fma.  Uncontracted, the pair rounds twice;
    contracted, once.  Charging both operations covers either;
  - library functions err by n ulp of the result, n = 2 for expf and rsqrtf, 1 for logf and log1pf, 4 for powf (the
    CUDA C Programming Guide's maximum ulp errors); one ulp is at most 2^-23 |r| + TINY;
  - propagated error: exp: e^v (e^{e_a} - 1); log: -log(1 - e_a / v); log1p: e_a / (1 + v - e_a); sqrt:
    sqrt(v) - sqrt(v - e_a); rsqrt: 1 / sqrt(v - e_a) - 1 / sqrt(v); a / b: (e_a + |a / b| e_b) / (|b| - e_b).  fmaxf,
    fminf, fabsf and negation are exact and 1-Lipschitz: they pass the larger bound on, or, where the two operands'
    intervals are apart, the chosen operand's own (a clamp that surely engages yields the constant exactly).
A 16-bit store adds half an ulp of the stored type at |value| + e (conv_ref.ulp, subnormals included).

The `F32` backend evaluates the same formulas in plain float32 torch, one rounded op each; the host test checks that
this stays inside the bounds, so they are not vacuous.

Discrete predicates are decided as TensorFlow's float32 graph decides them, not in float64:
  - exp(t_wh) underflowing to 0 (pw_zero: ptw := 1, so its log is 0 and its gradient 0), the 1e-9 / 1e9 clamp and
    the gradient mask w_in = (1e-9 < ptw < 1e9): from a float32 evaluation of the decode.  exp(t) underflows below
    t = -103.3 and ptw crosses 1e9 near t = 20.7; the tests keep t_wh away from both edges, so every float32
    evaluation decides alike;
  - the ignore mask `best < 0.5`: the float32 best IoU lies in [max_j (v_j - e_j), max_j (v_j + e_j)] over the
    image's ground-truth boxes j.  A box whose interval holds 0.5 is ambiguous: its conf loss and conf gradient are
    accepted under either ignore value (`g4_alt`, `l2_alt`), and the loss sum's bound takes the spread.  The tests
    count such boxes and assert that they are rare.

Loss sums (loss4).  Lane 0 adds its warp's per-box terms in float: at most D = ceil(nbox / 8 G) boxes per warp, with
G = min(ceil(nbox / 8), 16 SMs) blocks of 8 warps.  A box's class term first sums ceil(C / 32) values per lane, then 5
shuffle levels.  A float sum of k terms errs by at most k u sum |terms| (first order), so
    |loss4[k] - ref| <= inv_n (sum_boxes e_box + (D + d_k) u sum |term|) + (G + 10) 2^-53 inv_n sum |term|
with d_3 = ceil(C / 32) + 5 for the class term and 0 otherwise.  The last term covers the double sums: 8 warp partials
per block, G atomics and the product by inv_n.

Optimizer.  sqnorm[t] = fp32 sum over tensor t of g'^2, g' = grad * grad_scale + wd * w.  Each element's square passes
through at most 256 per-thread adds (65,536-element chunks, 256 threads), 5 shuffle levels, 8 warp partials and one
atomic per chunk of its tensor:
    |sqnorm - ref| <= sum e(g'^2) + (269 + chunks) u sum g'^2.
nrm = sqrtf(sqnorm), cs = clip / fmaxf(nrm, clip) (or 1 when clip <= 0) carry that bound on, and every element of w,
slot 1 and slot 2 follows its rule as Ev operations.  Adam's lr_t = lr sqrtf(1 - powf(b2, t)) / (1 - powf(b1, t)) with
t = updates applied + 1.  The 16-bit copy must be RN16 of the new w bit for bit.
"""
import math

import numpy as np
import torch

from tests.conv_ref import ulp

U = 2.0 ** -24                 # fp32 unit roundoff
ULP = 2.0 ** -23               # one fp32 ulp of r is at most ULP |r| + TINY
TINY = 2.0 ** -149             # fp32 subnormal spacing
U64 = 2.0 ** -53
SMS = 132


def f32(x):
    return float(np.float32(x))


class Ev:
    """float64 value v and a bound e on |float32 result - v| (module docstring)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def _o(self, o):
        if isinstance(o, Ev):
            return o
        assert f32(o) == o, f"constant {o} is not a float32 value"
        return Ev(torch.tensor(float(o), dtype=torch.float64, device=self.v.device), torch.zeros((), dtype=torch.float64, device=self.v.device))

    def __getitem__(self, i):
        return Ev(self.v[i], self.e[i])

    def __neg__(self):
        return Ev(-self.v, self.e)

    def __add__(self, o):
        o = self._o(o)
        v = self.v + o.v
        return Ev(v, _rnd(v, self.e + o.e))

    def __sub__(self, o):
        o = self._o(o)
        v = self.v - o.v
        return Ev(v, _rnd(v, self.e + o.e))

    def __mul__(self, o):
        o = self._o(o)
        v = self.v * o.v
        return Ev(v, _rnd(v, _m(self.v.abs(), o.e) + _m(o.v.abs(), self.e) + _m(self.e, o.e)))

    def __truediv__(self, o):
        o = self._o(o)
        v = self.v / o.v
        den = o.v.abs() - o.e
        prop = torch.where(den > 0, (self.e + v.abs() * o.e) / den.clamp(min=1e-300), math.inf)
        return Ev(v, _rnd(v, prop))

    __radd__ = __add__
    __rmul__ = __mul__

    def __rsub__(self, o):
        return self._o(o) - self

    def __rtruediv__(self, o):
        return self._o(o) / self


def _m(x, y):
    """x * y with 0 * inf = 0: an exact zero factor makes an exact product."""
    return torch.where((x == 0) | (y == 0), 0.0, x * y)


def _rnd(v, e):
    """e plus one correctly rounded fp32 operation with result v."""
    return e + U * (v.abs() + e) + TINY / 2


def _ulps(v, e, n):
    return e + n * (ULP * (v.abs() + e) + TINY)


def exp(a):
    if not isinstance(a, Ev):
        return torch.exp(a)
    v = torch.exp(a.v)
    return Ev(v, _ulps(v, v * torch.expm1(a.e), 2))


def log(a):
    if not isinstance(a, Ev):
        return torch.log(a)
    v = torch.log(a.v)
    prop = torch.where(a.e < a.v, -torch.log1p(-(a.e / a.v).clamp(max=1 - 1e-16)), math.inf)
    return Ev(v, _ulps(v, prop, 1))


def log1p(a):
    if not isinstance(a, Ev):
        return torch.log1p(a)
    v = torch.log1p(a.v)
    return Ev(v, _ulps(v, a.e / (1 + a.v - a.e), 1))


def sqrt(a):
    if not isinstance(a, Ev):
        return torch.sqrt(a)
    v = torch.sqrt(a.v)
    return Ev(v, _rnd(v, v - torch.sqrt((a.v - a.e).clamp(min=0))))


def rsqrt(a):
    if not isinstance(a, Ev):
        return torch.rsqrt(a)
    v = torch.rsqrt(a.v)
    lo = a.v - a.e
    prop = torch.where(lo > 0, torch.rsqrt(lo.clamp(min=1e-300)) - v, math.inf)
    return Ev(v, _ulps(v, prop, 2))


def _pair(a, b):
    if isinstance(a, Ev):
        return a, a._o(b)
    if isinstance(b, Ev):
        return b._o(a), b
    return None


def fmax(a, b):
    p = _pair(a, b)
    if p is None:
        return torch.maximum(a, b) if isinstance(b, torch.Tensor) else torch.clamp(a, min=b)
    a, b = p
    return _select(a, b, a.v - a.e >= b.v + b.e, a.v + a.e <= b.v - b.e, torch.maximum(a.v, b.v))


def fmin(a, b):
    p = _pair(a, b)
    if p is None:
        return torch.minimum(a, b) if isinstance(b, torch.Tensor) else torch.clamp(a, max=b)
    a, b = p
    return _select(a, b, a.v + a.e <= b.v - b.e, a.v - a.e >= b.v + b.e, torch.minimum(a.v, b.v))


def _select(a, b, take_a, take_b, v):
    """Where the two intervals are apart the float32 result is one operand with its own bound (a clamped value is the
    constant itself); where they overlap, the larger bound."""
    e = torch.where(take_a, a.e, torch.where(take_b, b.e, torch.maximum(a.e, b.e)))
    return Ev(torch.where(take_a, a.v, torch.where(take_b, b.v, v)), e)


def fabs(a):
    return Ev(a.v.abs(), a.e) if isinstance(a, Ev) else a.abs()


def where(p, a, b):
    q = _pair(a, b)
    if q is None:
        return torch.where(p, a, b)
    a, b = q
    return Ev(torch.where(p, a.v, b.v), torch.where(p, a.e, b.e))


def sigmoid(x):                                  # sigmoid_f: 1.0f / (1.0f + expf(-x))
    return 1.0 / (1.0 + exp(-x))


def bce(z, y):                                   # bce_logits: fmaxf(z, 0) - z * y + log1pf(expf(-fabsf(z)))
    return fmax(z, 0.0) - z * y + log1p(exp(-fabs(z)))


class F64:
    """Float64 values with bounds."""
    @staticmethod
    def lift(t):
        return Ev(t.double())

    @staticmethod
    def const(c, device):
        return Ev(torch.tensor(f32(c), dtype=torch.float64, device=device))

    @staticmethod
    def val(x):
        return x.v


class F32:
    """Plain float32, one rounding per op (the host test's evaluation of the kernel's formulas)."""
    @staticmethod
    def lift(t):
        return t.float()

    @staticmethod
    def const(c, device):
        return torch.tensor(f32(c), dtype=torch.float32, device=device)

    @staticmethod
    def val(x):
        return x.double()


# ---------------------------------------------------------------------------------------------------------------- loss
def _decode32(f, aw, ah, rw, rh):
    """ptw, pth of the float32 decode (the predicates' inputs)."""
    pw = torch.exp(f[..., 2]) * (aw / rw) * rw
    ph = torch.exp(f[..., 3]) * (ah / rh) * rh
    return pw / aw, ph / ah


def loss_eval(be, fm, y_true, anchors, img_hw, C, label_smooth, focal, grad_mul):
    """loss_kernel's formulas on one scale.  fm [n, gh, gw, 3E] float32, y_true [n, gh, gw, 3, E + 1] float32, anchors
    [3, 2] (w, h) pixels of this scale, img_hw (H, W).  -> dict:
      g: the five box / conf gradient lanes [n, gh, gw, 3];  g4_alt: lane 4 under the other ignore value;
      amb: ambiguous ignore mask [n, gh, gw, 3];  ign: the ignore value (where not ambiguous);  pos: m != 0 [n, gh, gw, 3] (bool);  cls_g: class gradient [P, C] of the
      positive boxes in pos.nonzero() order;  loss: [xy, wh, conf] per box and class per positive box;  l2_alt."""
    n, gh, gw = fm.shape[:3]
    E = 5 + C
    dev = fm.device
    f = fm.reshape(n, gh, gw, 3, E).float()
    y = y_true.float()
    img_h, img_w = img_hw
    rh, rw = f32(img_h / gh), f32(img_w / gw)          # ratio_h, ratio_w as the host passes them
    an = torch.as_tensor(np.asarray(anchors, np.float32).reshape(3, 2), device=dev)
    aw32, ah32 = an[:, 0], an[:, 1]
    L = be.lift
    aw, ah = L(aw32), L(ah32)
    offx = L(torch.arange(gw, device=dev, dtype=torch.float32).view(1, 1, gw, 1))
    offy = L(torch.arange(gh, device=dev, dtype=torch.float32).view(1, gh, 1, 1))
    tx, ty, tw, th, tc = (L(f[..., j]) for j in range(5))
    gx, gy, gwt, ght, m = (L(y[..., j]) for j in range(5))
    mix = L(y[..., E])
    # decode
    sx, sy = sigmoid(tx), sigmoid(ty)
    pcx, pcy = (sx + offx) * rw, (sy + offy) * rh
    pw = exp(tw) * (aw / rw) * rw
    ph = exp(th) * (ah / rh) * rh
    # predicates, in float32
    ptw32, pth32 = _decode32(f, aw32, ah32, rw, rh)
    pw_zero, ph_zero = ptw32 == 0, pth32 == 0
    ptw32, pth32 = torch.where(pw_zero, 1.0, ptw32), torch.where(ph_zero, 1.0, pth32)
    w_in = (ptw32 > f32(1e-9)) & (ptw32 < f32(1e9))
    h_in = (pth32 > f32(1e-9)) & (pth32 < f32(1e9))
    ign, amb = _ignore(be, pcx, pcy, pw, ph, y)
    # box terms
    scale = 2.0 - (gwt / float(img_w)) * (ght / float(img_h))
    cbox = m * scale * mix
    true_x, true_y = gx / rw - offx, gy / rh - offy
    pred_x, pred_y = pcx / rw - offx, pcy / rh - offy
    one = be.const(1.0, dev)
    ttw = where(y[..., 2] == 0, one, gwt / aw)
    tth = where(y[..., 3] == 0, one, ght / ah)
    ptw = where(pw_zero, one, pw / aw)
    pth = where(ph_zero, one, ph / ah)

    def clog(t):
        return log(fmin(fmax(t, f32(1e-9)), f32(1e9)))
    dx, dy = true_x - pred_x, true_y - pred_y
    dw, dh = clog(ttw) - clog(ptw), clog(tth) - clog(pth)
    # conf
    sc = sigmoid(tc)
    bce_c = bce(tc, m)
    fm_ = m - sc

    def conf(ig):
        wconf = m + (1.0 - m) * ig
        l2 = (wconf * bce_c * (fm_ * fm_) if focal else wconf * bce_c) * mix
        gc = wconf * mix * grad_mul
        g4 = gc * (fm_ * fm_ * (sc - m) - 2.0 * fm_ * sc * (1.0 - sc) * bce_c) if focal else gc * (sc - m)
        return l2, g4
    l2, g4 = conf(ign)
    l2_alt, g4_alt = conf(1.0 - ign)
    zero = be.const(0.0, dev)
    cg = cbox * f32(grad_mul)
    g = [-2.0 * dx * sx * (1.0 - sx) * cg, -2.0 * dy * sy * (1.0 - sy) * cg,
         where(w_in & ~pw_zero, -2.0 * dw * cg, zero), where(h_in & ~ph_zero, -2.0 * dh * cg, zero), g4]
    l0 = (dx * dx + dy * dy) * cbox
    l1 = (dw * dw + dh * dh) * cbox
    # class terms of the positive boxes
    pos = y[..., 4] != 0
    z = L(f[..., 5:][pos])
    t = L(y[..., 5:E][pos])
    if label_smooth:
        t = f32(1.0 - f32(0.01)) * t + be.const(0.01, dev) / float(C)
    terms = bce(z, t)
    if isinstance(terms, Ev):
        depth = -(-C // 32) + 5
        cls = Ev(terms.v.sum(-1), terms.e.sum(-1) + depth * U * terms.v.abs().sum(-1))
    else:
        cls = terms.sum(-1)
    mp, mixp = m[pos], mix[pos]
    cls_g = mp[:, None] * mixp[:, None] * (sigmoid(z) - t) * f32(grad_mul)
    l3 = mp * cls * mixp
    return dict(g=g, g4_alt=g4_alt, amb=amb, ign=be.val(ign), pos=pos, cls_g=cls_g, loss=[l0, l1, l2, l3], l2_alt=l2_alt)


def _ignore(be, pcx, pcy, pw, ph, y):
    """(ignore, ambiguous) per box: best IoU with the image's ground-truth boxes of this scale against 0.5."""
    n = y.shape[0]
    shape = y.shape[:4]
    dev = y.device
    ign = torch.ones(shape, dtype=torch.float64 if be is F64 else torch.float32, device=dev)
    amb = torch.zeros(shape, dtype=torch.bool, device=dev)
    h = 1.0 / 2.0
    for i in range(n):
        gt = y[i][..., 0:4][y[i][..., 4] != 0]               # [V, 4] cx, cy, w, h
        if gt.shape[0] == 0:
            continue                                          # reduce_max over nothing: -FLT_MAX < 0.5
        G = be.lift(gt)
        gxv, gyv, gzv, gwv = (G[:, j][None, :] for j in range(4))
        P = [a[i].reshape(-1)[:, None] if not isinstance(a, Ev) else Ev(a.v[i].reshape(-1)[:, None], a.e[i].expand_as(a.v[i]).reshape(-1)[:, None])
             for a in (pcx, pcy, pw, ph)]
        cx, cy, w, hh = P
        px0, px1 = cx - w / 2.0, cx + w / 2.0
        py0, py1 = cy - hh / 2.0, cy + hh / 2.0
        parea = w * hh
        ix = fmax(fmin(px1, gxv + gzv / 2.0) - fmax(px0, gxv - gzv / 2.0), 0.0)
        iy = fmax(fmin(py1, gyv + gwv / 2.0) - fmax(py0, gyv - gwv / 2.0), 0.0)
        inter = ix * iy
        iou = inter / (parea + gzv * gwv - inter + f32(1e-10))
        if isinstance(iou, Ev):
            lo = (iou.v - iou.e).max(-1).values
            hi = (iou.v + iou.e).max(-1).values
            ign[i] = (hi < h).double().view(shape[1:])
            amb[i] = ((hi >= h) & (lo < h)).view(shape[1:])
        else:
            ign[i] = (iou.max(-1).values < h).float().view(shape[1:])
    return (Ev(ign) if be is F64 else ign), amb


def grad_dense(res, C, dtype=None):
    """-> (value, bound, alt) float64 [n, gh, gw, 3, E]: the gradient columns, bounds with the 16-bit store's half ulp
    when dtype is fp16 / bf16, and lane 4's value under the other ignore value (NaN where not ambiguous)."""
    g = res["g"]
    shape = g[0].v.shape
    E = 5 + C
    val = torch.zeros(shape + (E,), dtype=torch.float64, device=g[0].v.device)
    bnd = torch.zeros_like(val)
    for j in range(5):
        val[..., j] = g[j].v
        bnd[..., j] = g[j].e.expand(shape)
    pos = res["pos"]
    cv, ce = val[..., 5:], bnd[..., 5:]          # views: the assignments below write val and bnd
    cv[pos] = res["cls_g"].v
    ce[pos] = res["cls_g"].e.expand_as(res["cls_g"].v)
    alt = torch.where(res["amb"], res["g4_alt"].v, math.nan)
    if dtype is not None and dtype != torch.float32:
        bnd = bnd + 0.5 * ulp(val.abs() + bnd, dtype)
        ab = res["g4_alt"].e.expand(shape)
        alt_b = ab + 0.5 * ulp(res["g4_alt"].v.abs() + ab, dtype)
    else:
        alt_b = res["g4_alt"].e.expand(shape)
    return val, bnd, alt, alt_b


def check_grad(got, val, bnd, alt, alt_b, what):
    """|got - ref| <= bound per element (lane 4 of an ambiguous box: against either value) -> worst err / bound."""
    err = (got.double() - val).abs()
    frac = torch.where(err == 0, 0.0, err / bnd)
    a = ~torch.isnan(alt)
    if bool(a.any()):
        ea = (got[..., 4].double() - alt).abs()
        fa = torch.where(ea == 0, 0.0, ea / alt_b)
        frac[..., 4] = torch.where(a, torch.minimum(frac[..., 4], fa), frac[..., 4])
    bad = ~(frac <= 1.0)
    if bool(bad.any()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} gradient elements out of bound; first at {idx}: "
                             f"got {float(got[idx]):.7g} ref {float(val[idx]):.7g} bound {float(bnd[idx]):.3g}")
    return float(frac.max())


def loss4_ref(res, nbox, C, inv_n, sms=SMS):
    """(value [4], bound [4]) float64 of what one launch adds to loss4 (module docstring)."""
    G = min(-(-nbox // 8), sms * 16)
    D = -(-nbox // (8 * G))
    val, bnd = [], []
    for k, t in enumerate(res["loss"]):
        s_abs = float(t.v.abs().sum())
        e = float(t.e.expand_as(t.v).sum())
        v = float(t.v.sum())
        d = D + (-(-C // 32) + 5 if k == 3 else 0)
        b = e + d * U * s_abs
        if k == 2:                                          # ambiguous boxes: either ignore value
            amb = res["amb"]
            alt = res["l2_alt"]
            spread = (alt.v - t.v)[amb]
            v += 0.5 * float(spread.sum())
            b += 0.5 * float(spread.abs().sum()) + float(alt.e.expand_as(alt.v)[amb].sum())
            s_abs += float(alt.v.abs()[amb].sum())
        b += (G + 10) * U64 * s_abs
        val.append(v * inv_n)
        bnd.append(b * inv_n)
    return np.array(val), np.array(bnd)


# ----------------------------------------------------------------------------------------------------------- optimizer
KINDS = {"sgd": 0, "momentum": 1, "rmsprop": 2, "adam": 3}


def opt_eval(be, kind, w, g, v1, v2, seg, l2, chunks, o, applied):
    """One opt_update_kernel pass over the flat trainable elements.  w, g, v1, v2 float32 [N]; seg [N] tensor index
    (0..T-1, dense); l2 [T] bool; chunks [T] 65,536-element chunks per tensor; o: dict of the yb_optimizer fields;
    applied: ctrl[1] before the step.  -> (sqnorm [T], w, v1, v2) as Ev (F64) or float32 (F32)."""
    dev = w.device
    K = lambda c: be.const(c, dev)
    L = be.lift
    T = l2.numel()
    wd = L(torch.where(l2, f32(o["weight_decay"]), 0.0).float()[seg])
    w_, g_, s1, s2 = L(w), L(g), L(v1), L(v2)
    gp = g_ * K(o["grad_scale"]) + wd * w_
    sq = gp * gp
    if be is F64:
        sv = torch.zeros(T, dtype=torch.float64, device=dev).index_add_(0, seg, sq.v)
        se = torch.zeros(T, dtype=torch.float64, device=dev).index_add_(0, seg, sq.e)
        sqn = Ev(sv, se + (269 + chunks.double()) * U * sv)
    else:                                        # per chunk a float32 (cascade) sum, then the chunks in order
        sqn = torch.zeros(T, dtype=torch.float32, device=dev)
        bounds = torch.searchsorted(seg, torch.arange(T + 1, device=dev))
        for t in range(T):
            for c0 in range(int(bounds[t]), int(bounds[t + 1]), 65536):
                sqn[t] += sq[c0: min(c0 + 65536, int(bounds[t + 1]))].sum()
    clip = f32(o["clip_norm"])
    if clip > 0:
        cs = K(clip) / fmax(sqrt(sqn), K(clip))
        cs = cs[seg]
    else:
        cs = K(1.0)
    gg = gp * cs
    lr = K(o["lr"])
    if kind == "sgd":
        nw, n1, n2 = w_ - lr * gg, s1, s2
    elif kind == "momentum":
        n1 = K(o["momentum"]) * s1 + gg
        nw, n2 = w_ - lr * n1, s2
    elif kind == "rmsprop":
        d = K(o["decay"])
        n2 = d * s2 + (1.0 - d) * gg * gg
        n1 = K(o["momentum"]) * s1 + lr * gg * rsqrt(n2 + K(o["epsilon"]))
        nw = w_ - n1
    elif kind == "adam":
        t = float(applied + 1)
        b1, b2 = K(o["beta1"]), K(o["beta2"])
        lr_t = lr * sqrt(1.0 - _powf(be, f32(o["beta2"]), t, dev)) / (1.0 - _powf(be, f32(o["beta1"]), t, dev))
        n1 = b1 * s1 + (1.0 - b1) * gg
        n2 = b2 * s2 + (1.0 - b2) * gg * gg
        nw = w_ - lr_t * n1 / (sqrt(n2) + K(o["epsilon"]))
    else:
        raise ValueError(kind)
    return sqn, nw, n1, n2


def _powf(be, b, t, dev):
    if be is F64:
        v = torch.tensor(b, dtype=torch.float64, device=dev) ** t
        return Ev(v, _ulps(v, torch.zeros_like(v), 4))
    return torch.tensor(b, dtype=torch.float32, device=dev) ** torch.tensor(t, dtype=torch.float32, device=dev)


def check_ev(got, ref, what):
    """|got - ref.v| <= ref.e per element -> worst err / bound."""
    err = (got.double() - ref.v).abs()
    frac = torch.where(err == 0, 0.0, err / ref.e.expand_as(err))
    bad = ~(frac <= 1.0)
    if bool(bad.any()):
        idx = int(bad.nonzero()[0, 0])
        e = ref.e.expand_as(err)
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements out of bound; first at {idx}: got "
                             f"{float(got[idx]):.9g} ref {float(ref.v[idx]):.9g} bound {float(e[idx]):.3g}")
    return float(frac.max()) if frac.numel() else 0.0
