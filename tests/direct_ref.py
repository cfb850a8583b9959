"""Float64 references and per-element error bounds for the direct (non-implicit-GEMM) forward conv kernels: the
halo-tile conv and the fused stem + Conv_1 (csrc/conv_halo.cu), the mma.sync thin kernel and stems (csrc/conv_thin.cu)
and the CUDA-core stem (csrc/layers.cu).  The float64 conv, epilogue and store model are tests/conv_ref.py's.

Halo-tile conv.  Per 16 x 8-pixel tile the two consumer warpgroups issue, for each of the 9 taps, cin / 16 wgmma k16
steps on 16-bit operands into one fp32 accumulator chain: conv_ref.out_bound with n16 = 9 cin / 16 (halo_n16).  Both
epilogues round exactly three times in fp32 before the store: the TMA-store epilogue (epi_box_to_slab, csrc/wgmma.cuh)
computes fmaf(acc, scale, shift), fmaxf(v, slope v) (the product rounds once; slope = 1 without leaky, exact) and
adds the residual from the stage's box, then packs to 16 bits for stmatrix; the staging epilogue (the e4m3 output and
YB_CONV_RES=ldg) stores the accumulators to shared memory as fp32 (exact) and does the same three operations.

Thin kernel and plain mma.sync stem.  mma.sync m16n8k16 on 16-bit operands accumulates in fp32 like a wgmma k16 step
(DESIGN.md §2: these kernels fit the C_STEP model): out_bound with n16 = 18 (9 taps x 32 channels; THIN_N16) and 2 for
the stem (K = 27 padded to 32; STEM_N16), on RN16 operands (the stem rounds its float32 image and weights).  Epilogue:
fmaf, leaky01, residual add, store.

Split-precision stem (ThinCfg<..., SPLIT>, the training forward).  Every image value and weight is split into
hi = T(v), lo = T(v - hi) (v - hi is exact in fp32) and the kernel multiplies K = 96 = [x_hi | x_lo | x_hi] .
[w_hi ; w_hi ; w_lo].  The reference is the float64 conv of the UNROUNDED float32 image and weights.  With
r_v = v - hi - lo, |r_v| <= u_T^2 |v| + eta_T and |lo| <= (u_T + u_T^2)|v| + 2 eta_T (u_T, eta_T: wgrad_ref._U16,
_ETA; eta_T is half the fp16 subnormal spacing, the floor of both roundings), each product's split error is

    x w - (x_hi w_hi + x_lo w_hi + x_hi w_lo) = x_lo w_lo + r_x w + (x - r_x) r_w,

summed over the 27 taps:  e_split = c2 S + c1 (A_w + A_x) + 27 c0,   S = sum |x w|,  A_w = sum |w|,  A_x = sum |x|
with c2 = (u + u^2)^2 + 2 u^2 + u^4, c1 = eta (1 + u^2 + 2 (u + u^2)), c0 = 5 eta^2 (split_bound).  The tensor cores
add |hi| |w_hi| + |lo| |w_hi| + |hi| |w_lo| <= (|hi| + |lo|)(|w_hi| + |w_lo|), and |hi| + |lo| <= (1 + u)^2 |v| + 3 eta,
so the magnitude sum of the 6 k16 steps is at most S' = sum ((1 + u)^2 |x| + 3 eta)((1 + u)^2 |w| + 3 eta).  Then
out_bound's accumulation (C_STEP per step on S'), three fp32 epilogue roundings and the store.

Split stem batch sums.  Thread (warp q, lane c) of a persistent CTA adds the stored 16-bit value (exact in fp32) of
channel c of 32 pixels of every tile the CTA runs, st += v and st2 = fmaf(v, v, st2), one rounding each; then each
of the 4 warps of each of the `grid` CTAs adds its lane's total to the global sum with one atomic.  Every add rounds
once relative to a partial sum of magnitudes, at most sum |z| + |s0| (s0 the initial sum: the kernel accumulates), so

    |ssum - (s0 + sum z)| <= depth u (|s0| + sum |z|),   depth = 32 T + 4 G + 1,

T the tiles of the busiest CTA and G the grid, and the same with z^2.  The grid, min(tiles, SMs x per_sm) with
per_sm <= 8, is not exported: sums_depth bounds T by ceil(tiles / min(tiles, SMs)) and G by min(tiles, 8 SMs).

CUDA-core stem (stem_conv_kernel).  Per output one float32 fmaf chain over the 27 (r, s, ci) taps from 0 on the
unrounded operands: |acc - raw| <= gamma_27 S, gamma_n = n u / (1 - n u); then fmaf(acc, scale, shift) and the leaky
product round once each, then the store (cuda_stem_bound).

Fused stem + Conv_1 (interval method).  The fused kernel's stem value v0 (mma.sync, K = 32, on RN16 operands) is never
stored; it is within e0 = out_bound(v0, S, 2, fp32) of the float64 value, so the 16-bit value Conv_1 reads lies in
[RN16(v0 - e0), RN16(v0 + e0)].  Conv_1 is checked on x* = RN16(v0) with |scale_1| conv(d, |w_1|) added to its bound,
d the width of that interval on the wider side, and S taken over |x*| + d (stem_interval, conv1_on_interval).
"""
import torch

from tests import conv_ref as R
from tests.wgrad_ref import _ETA, _U16

U32 = R.U32
STEM_N16 = 2                       # mma.sync stem: K = 27 padded to 32
SPLIT_N16 = 6                      # split stem: K = 96
THIN_N16 = 18                      # thin kernel: 9 taps x 32 channels


def halo_n16(cin):
    return 9 * cin // 16


def rn16(v, dtype):
    """Round-to-nearest-even of float64 v into fp16 / bf16, as float64 (exact: scaled by the spacing at |v|)."""
    q = R.ulp(v, dtype)
    return torch.round(v / q) * q


def gamma(n):
    return n * U32 / (1 - n * U32)


# ---------------------------------------------------------------------------------------------------------- split stem
def split16(v, dtype):
    """The kernel's split of float32 v: (hi, lo) as float32 tensors (lo = T(v - hi), v - hi exact in fp32)."""
    v = v.float()
    hi = v.to(dtype).float()
    return hi, (v - hi).to(dtype).float()


def split_bound(S, Ax, Aw, dtype):
    """Bound of |conv(x, w) - conv_split(x, w)| (module docstring): S [M, cout], Ax [M, 1] = sum |x| over the 27 patch
    values, Aw [cout] = sum |w| over the 27 taps."""
    u, eta = _U16[dtype], _ETA[dtype]
    c2 = (u + u * u) ** 2 + 2 * u * u + u ** 4
    c1 = eta * (1 + u * u + 2 * (u + u * u))
    return c2 * S + c1 * (Aw + Ax) + 27 * 5 * eta * eta


def split_mag(S, Ax, Aw, dtype):
    """S' of the module docstring: the magnitude sum of what the tensor cores add."""
    u, eta = _U16[dtype], _ETA[dtype]
    a = (1 + u) ** 2
    return a * a * S + 3 * eta * a * (Aw + Ax) + 27 * 9 * eta * eta


def stem_split_bound(ref, S, Ax, Aw, dtype, scale=None, shift=None):
    """Per-element bound of the split stem's stored output against the float64 conv of the unrounded operands."""
    sc = 1.0 if scale is None else scale.double().abs()
    sh = 0.0 if shift is None else shift.double().abs()
    s1 = split_mag(S, Ax, Aw, dtype)
    e32 = sc * (split_bound(S, Ax, Aw, dtype) + R.C_STEP * SPLIT_N16 * s1) + 3 * U32 * (sc * s1 + sh)
    return e32 + 0.5 * R.ulp(ref.abs() + e32, dtype)


def stem_patch_abs(x):
    """sum |x| over each output pixel's 27 patch values (SAME padding), float64 [M, 1]; x [n, h, w, 3]."""
    return R.im2col(x.double().abs(), 3, 1, 1).sum(1, keepdim=True)


def sums_depth(tiles, sms):
    """Depth of the split stem's statistics chain (module docstring), conservative in the unexported grid."""
    g_min = min(tiles, sms)
    return 32 * -(-tiles // g_min) + 4 * min(tiles, 8 * sms) + 1


def sums_bound(z, s0, q0, depth):
    """Bounds of |ssum - (s0 + sum z)| and |ssq - (q0 + sum z^2)|; z [M, C] the stored values, s0 / q0 [C]."""
    za = z.double().abs()
    return (depth * U32 * (s0.double().abs() + za.sum(0)),
            depth * U32 * (q0.double().abs() + (za * za).sum(0)))


# -------------------------------------------------------------------------------------------------- CUDA-core stem
def cuda_stem_bound(ref, S, dtype, scale=None, shift=None):
    """Per-element bound of stem_conv_kernel's stored output against the float64 epilogue of the unrounded conv."""
    sc = 1.0 if scale is None else scale.double().abs()
    sh = 0.0 if shift is None else shift.double().abs()
    g = gamma(27)
    e32 = sc * g * S + 2 * U32 * (sc * (1 + g) * S + sh)
    return e32 + 0.5 * R.ulp(ref.abs() + e32, dtype)


# ------------------------------------------------------------------------------------------- fused stem + Conv_1
def stem_interval(v0, S, dtype, scale, shift):
    """(x*, d): the stem's 16-bit value Conv_1 reads lies in [x* - d, x* + d] (module docstring); v0, S [..., 32]."""
    e0 = R.out_bound(v0, S, STEM_N16, torch.float32, scale=scale, shift=shift)
    xs = rn16(v0, dtype)
    d = torch.maximum(rn16(v0 + e0, dtype) - xs, xs - rn16(v0 - e0, dtype))
    return xs, d


def conv1_on_interval(xs, d, w1, stride, scale1):
    """Conv_1 of the interval: (raw on x*, S over |x*| + d, the extra bound term |scale_1| conv(d, |w_1|))."""
    raw, _ = R.conv_raw(xs, w1, stride, 1)
    _, S = R.conv_raw(xs.abs() + d, w1, stride, 1)
    extra = scale1.double().abs() * R.conv_raw(d, w1, stride, 1)[1]
    return raw, S, extra
