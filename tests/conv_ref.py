"""Float64 reference and per-element error bounds for the implicit-GEMM conv (csrc/conv_igemm.cu).

The kernel multiplies 16-bit operands on the tensor cores and accumulates in fp32 registers, then applies the epilogue in
fp32 and stores once.  The reference repeats that on the same 16-bit-rounded operands in float64, so every difference
is the kernel's own rounding, and the bound below says how much rounding is allowed:

    |got - ref| <= 1/2 ulp_T(|ref| + e32) + e32
    e32 = |scale| * c_acc * S  +  3 u (|scale| S + |shift| + |res|),    S = sum |x * w|,   u = 2^-24
    c_acc = 4 * 2^-23 * n16,                                            n16 = K / 16 k16 steps

- Accumulation (c_acc): a product of two fp16 (11-bit) or two bf16 (8-bit) significands is exact in fp32.  Each k16
  step of a wgmma adds 16 products to the accumulator; allowing the tensor core to round or truncate the partial sum up
  to four times per step (it adds the products in groups), and each such step to lose at most one fp32 ulp of a partial
  sum, which is at most S, gives 4 * 2^-23 * S per step.
- Epilogue (3 u terms): fmaf(acc, scale, shift), the 0.1f leaky product and the residual add round once each.
- Store: round-to-nearest into the output type T (fp16 / bf16) adds half an ulp of the stored value, subnormal spacing
  included; fp32 outputs have no such term.

S comes from a second float64 conv of |x| and |w|.  The leaky slope is the kernel's float32 0.1f, not 0.1.

Batch statistics: the kernel sums the fp32 accumulators of each column, 16 rows per thread, then into per-warpgroup
shared-memory sums (one add per 16-row group, 64-row half and unit), then one atomic add per warpgroup flush into the
global sums.  A value passes through at most `depth` = 16 + 8 U + 2 G additions (U units per warpgroup, G CTAs), each of
which rounds once, so
    |ssum - sum raw| <= sum e_acc + depth u sum(|raw| + e_acc)
    |ssq - sum raw^2| <= sum (2 |raw| e_acc + e_acc^2) + depth u sum (|raw| + e_acc)^2
with e_acc = c_acc S per element.
"""
import numpy as np
import torch

SLOPE = float(np.float32(0.1))     # the kernel's 0.1f
U32 = 2.0 ** -24                   # fp32 unit roundoff
C_STEP = 4 * 2.0 ** -23            # accumulator error per k16 step, relative to sum |x * w|

_FMT = {torch.float16: (10, -14), torch.bfloat16: (7, -126)}   # significand bits after the point, smallest normal exponent


def ulp(a, dtype):
    """Spacing of `dtype` at magnitude |a| (float64 tensor), subnormal spacing included."""
    mant, emin = _FMT[dtype]
    _, e = torch.frexp(a.abs())                 # |a| = m 2^e, m in [0.5, 1): floor(log2 |a|) = e - 1
    e = torch.where(a == 0, emin, torch.clamp(e.to(torch.float64) - 1, min=emin))
    return torch.exp2(e - mant)


def im2col(x, k, stride, pad):
    """NHWC float64 [n, h, w, c] -> [n * P * Q, k * k * c] in the (r, s, c) order of the packed OHWI weights."""
    n, h, w, c = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, pad, pad, pad, pad))
    P, Q = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    cols = xp.unfold(1, k, stride).unfold(2, k, stride)          # [n, P, Q, c, k, k]
    return cols[:, :P, :Q].permute(0, 1, 2, 4, 5, 3).reshape(n * P * Q, k * k * c)


def conv_raw(x, w_ohwi, stride, pad):
    """Raw conv and the conv of magnitudes, float64 [M, cout] each (x NHWC, w OHWI, both already 16-bit-rounded)."""
    k = w_ohwi.shape[1]
    cols = im2col(x.double(), k, stride, pad)
    wm = w_ohwi.double().reshape(w_ohwi.shape[0], -1).t()
    return cols @ wm, cols.abs() @ wm.abs()


def epilogue(raw, scale=None, shift=None, leaky=False, res=None):
    """Float64 scale / shift, leaky (slope 0.1f), residual; raw [..., cout], scale / shift [cout]."""
    v = raw if scale is None else raw * scale.double() + shift.double()
    if leaky:
        v = torch.where(v > 0, v, SLOPE * v)
    if res is not None:
        v = v + res.double()
    return v


def out_bound(ref, S, n16, dtype, scale=None, shift=None, res=None):
    """Per-element bound of |got - ref| (see the module docstring); dtype = the stored type (torch.float32: no rounding)."""
    sc = 1.0 if scale is None else scale.double().abs()
    sh = 0.0 if shift is None else shift.double().abs()
    r = 0.0 if res is None else res.double().abs()
    e32 = sc * (C_STEP * n16) * S + 3 * U32 * (sc * S + sh + r)
    if dtype == torch.float32:
        return e32
    return e32 + 0.5 * ulp(ref.abs() + e32, dtype)


def check_out(got, ref, bound, what=""):
    """Assert |got - ref| <= bound elementwise; returns the worst |got - ref| / bound."""
    err = (got.double() - ref).abs()
    frac = torch.where(err == 0, 0.0, err / bound)     # exact where the bound is 0 (all-zero operands): fine
    bad = ~(frac <= 1.0)                               # NaN counts as bad
    if bool(bad.any()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements out of bound; first at {idx}: got "
                             f"{float(got[idx]):.7g} ref {float(ref[idx]):.7g} bound {float(bound[idx]):.3g}; "
                             f"worst err / bound {float(frac[~torch.isnan(frac)].max()) if (~torch.isnan(frac)).any() else float('nan'):.3g}")
    return float(frac.max()) if frac.numel() else 0.0


def stats_bound(raw, S, n16, depth):
    """Bounds of the column sums and sums of squares of the raw conv (see the module docstring); raw, S [M, cout]."""
    ea = (C_STEP * n16) * S
    a = raw.abs() + ea
    b_sum = ea.sum(0) + depth * U32 * a.sum(0)
    b_sq = (2 * raw.abs() * ea + ea * ea).sum(0) + depth * U32 * (a * a).sum(0)
    return b_sum, b_sq


def stats_depth(units_per_wg, grid):
    return 16 + 8 * units_per_wg + 2 * grid


def old_criterion_ok(got, ref, dtype):
    """The earlier test bar: |err| <= 2^-9 max(1, |ref|) (fp16), 2^-6 (bf16), 1e-4 (fp32)."""
    eps = {torch.float16: 2.0 ** -9, torch.bfloat16: 2.0 ** -6, torch.float32: 1e-4}[dtype]
    return bool(((got.double() - ref).abs() <= eps * ref.abs().clamp(min=1.0)).all())


def units_per_warpgroup(info):
    """Fewest work units any consumer warpgroup runs under a yb_conv_schedule result (ping-pong: the two warpgroups of
    CTA b take units b + w G + 2 G j of the G clusters' units; cooperative: both take every unit of their CTA)."""
    units, G = info.units, info.grid // info.cluster
    if info.pingpong:
        return max(0, -(-(units - (2 * G - 1)) // (2 * G)))
    return max(0, -(-(units - (G - 1)) // G))


def last_unit_warpgroup(info):
    """Consumer warpgroup that runs the last work unit (ping-pong; 0 under the cooperative schedule)."""
    units, G = info.units, info.grid // info.cluster
    return ((units - 1) // G) % 2 if info.pingpong else 0
