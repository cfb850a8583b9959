"""Float64 / exact-float32 references and per-element bounds for the batch-norm training kernels (csrc/bn.cu).

Rows are [rows, c] (compact; tests gather them out of their strided buffers first).  u = 2^-24, u_T the unit
roundoff of the stored 16-bit type T (2^-11 fp16, 2^-8 bf16), ulp_T its spacing (conv_ref.ulp).

Coefficients (bn_batch_coeffs, bn_moving_update).  Every operation is an explicitly rounded fp32 op, so the same
sequence of float32 ops here gives mean, var, scale, shift and the moving statistics bit for bit, once the kernel's
invstd is taken as given.  invstd = rsqrtf(fl32(var + eps)) is not correctly rounded: the CUDA C Programming Guide
bounds rsqrtf by 2 ulp, so |invstd - 1 / sqrt(fl32(var + eps))| <= 2 ulp_32(invstd) against float64.  Frozen BN (no
batch sums) forms shift = beta - mean * scale without explicit rounding, so the compiler may fuse it: within 1 ulp_32.

Apply (bn_act_apply_kernel).  y = fmaf(z, sc, sh): z * sc is exact in float64 (at most 11 + 24 significand bits), and
so is the float64 sum with sh unless its exponents are far apart.  TwoSum finds the elements whose float64 sum was
inexact; there rounding float64 -> float32 is a double rounding and may land one fp32 ulp off, which can move the
16-bit result by one ulp_T.  Everywhere else y is the correctly rounded fmaf.  The leaky product 0.1f * y and the
residual add are single fp32 ops (the kernel does not fuse them; its SASS holds FMUL by 0.1 then FADD), done here in
float32, and the store rounds to nearest even.  So the kernel must match bit for bit except on the TwoSum elements,
which may differ by one ulp_T.

Reduce (bn_bwd_reduce_kernel), exact operands.  dact = (leaky and y <= 0) ? fl32(0.1f * dA) : dA.  The sign of y is the
sign of the exact z * sc + sh (rounding keeps signs, and a float64 sum is zero only when exact), so it is decided
here without rounding.  With z, dA, save_mean integers and save_invstd a power of two, every per-thread, per-block,
per-slot and final partial of sum(dact) and invstd * (sum(dact * z) - mean * sum(dact)) is an integer times invstd of
magnitude at most G + |mean| A (G = sum |dact z|, A = sum |dact|) times invstd.  Below 2^24 fp32 holds each exactly,
so every block, slot and atomic order gives the float64 result bit for bit.  The premise needs dact integral: 0.1f * 10k
rounds to exactly k for |k| <= 16, which covers dA in 10 * {-4..4} and the sum of 4 such upsampled copies;
the tests assert it, and G + |mean| A < 2^24, on every exact case.

Reduce, float operands.  A value passes through at most rows_per_block / lanes fmaf steps of its thread's chain, lanes
shared-memory adds, one centring fma and the invstd product, `grid` atomic adds (per slot, or into dgamma directly) and
BN_SLOTS final adds, each rounding once to at most the magnitude sum:
    |dbeta - ref| <= n_ops u A,   |dgamma - ref| <= n_ops u invstd (G + |mean| A),
    n_ops = rows_per_block / lanes + lanes + grid + BN_SLOTS + 4.
The atomic adds are the one place subnormals do not survive: float atomicAdd (PTX atom / red .add.f32) flushes
subnormal inputs and results to sign-preserving zero, so each of the `grid` atomic adds a value passes through may
also drop less than 2^-126 twice, its input and its result.  Both bounds carry the absolute term 2 grid 2^-126 for it
(it matters only for a channel whose sums are themselves near the subnormal range).

bwd apply (bn_bwd_apply_kernel).  k1 = ga is, k2 = -k1 is dg inv_m, k3 = -k1 db inv_m - k2 mu with inv_m = fl32(1 / M),
dz = fmaf(k1, dact, fmaf(k2, z, k3)).  Relative errors: inv_m 1 u, k1 1 u, k2 5 u, k1 db inv_m 4 u, k2 mu 6 u, k3's
difference 1 u of its operands' magnitude sum, the two fmaf 1 u each of theirs.  With
    S = |k1 dact| + |k2 z| + |k1 db / M| + |k2 mu|     (float64, exact coefficients)
every term is at most 9 u S; with the second-order terms
    |dz - ref| <= 10 u S + 1/2 ulp_T(|ref| + 10 u S).
dact itself is emulated exactly (float32), so the leaky slope adds no error.
"""
import torch

from tests.conv_ref import SLOPE, U32, ulp

RSQRT_ULP = 2          # rsqrtf, CUDA C Programming Guide (single-precision mathematical functions)
EXACT_LIMIT = 2.0 ** 24
BN_SLOTS = 16          # csrc/bn.cu
FTZ32 = 2.0 ** -126    # smallest normal float32: what one flushing atomic add may drop, per input and per result
_F32 = torch.float32


def f32(x):
    return torch.as_tensor(x, dtype=_F32)


def ulp32(x):
    """Spacing of float32 at |x| (normal range)."""
    _, e = torch.frexp(x.double().abs())
    return torch.exp2(e.double() - 24)


def batch_coeffs(su, sq, count, ga, be, eps, invstd):
    """bn_batch_coeffs in float32 ops, given the kernel's invstd -> (mean, var, scale, shift), each float32 [c]."""
    cnt, eps = f32(count), f32(eps)
    mean = su / cnt
    var = torch.clamp_min(sq / cnt - mean * mean, 0.0)
    sc = ga * invstd
    sh = be - mean * sc
    return mean, var, sc, sh


def invstd_error(var, eps, invstd):
    """|invstd - 1 / sqrt(fl32(var + eps))| in units of the float32 ulp of invstd (must be <= RSQRT_ULP)."""
    ref = 1.0 / torch.sqrt((var + f32(eps)).double())
    return ((invstd.double() - ref).abs() / ulp32(invstd)).max().item()


def moving_update(mm, mv, mean, var, count, decay):
    """bn_moving_update in float32 ops -> (moving_mean, moving_var)."""
    cnt, decay = f32(count), f32(decay)
    unb = var * cnt / (cnt - 1) if count > 1 else var
    keep = f32(1.0) - decay
    return mm * decay + keep * mean, mv * decay + keep * unb


def fma_f32(a, b, c):
    """fmaf(a, b, c) for float32 tensors with a * b exact in float64 -> (float32 result, inexact mask): where the
    float64 sum was inexact (TwoSum) the result may be one float32 ulp off the correctly rounded fmaf."""
    p = a.double() * b.double()
    cd = c.double()
    s = p + cd
    bb = s - p
    err = (p - (s - bb)) + (cd - bb)
    return s.float(), err != 0


def apply_ref(z, sc, sh, res, leaky, dtype):
    """bn_act_apply on compact rows: z, res [rows, c] 16-bit (res may be None), sc / sh float32 [c]
    -> (dtype result, mask of the elements allowed one ulp_T)."""
    y, inexact = fma_f32(z.float(), sc, sh)
    if leaky:
        y = torch.where(y > 0, y, y * SLOPE)          # float32 * float32: the kernel's 0.1f product
    if res is not None:
        y = y + res.float()
    return y.to(dtype), inexact


def check_apply(got, want, inexact, dtype, what):
    """Bit-exact except on `inexact` elements, which may be one ulp_T off -> number of such differing elements."""
    diff = got.view(torch.int16) != want.view(torch.int16)
    hard = diff & ~inexact
    if bool(hard.any()):
        idx = tuple(hard.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(hard.sum())}/{hard.numel()} elements differ from the exactly rounded result; "
                             f"first at {idx}: got {float(got[idx])} want {float(want[idx])}")
    soft = diff & inexact
    if bool(soft.any()):
        g, w = got[soft].double(), want[soft].double()
        step = ulp(torch.maximum(g.abs(), w.abs()), dtype)
        assert bool(((g - w).abs() <= step).all()), f"{what}: an inexact-sum element is more than one ulp off"
    return int(soft.sum())


def upsampled_rows(buf4):
    """[n, 2h, 2w, c] gradient of a 2x-upsampled store -> [n, h, w, c] float32, summed the kernel's way:
    v + ((t0 + t1) + t2) with v the top-left copy, t0 its right neighbour, t1 the one below, t2 the diagonal."""
    v, t0 = buf4[:, 0::2, 0::2].float(), buf4[:, 0::2, 1::2].float()
    t1, t2 = buf4[:, 1::2, 0::2].float(), buf4[:, 1::2, 1::2].float()
    return v + ((t0 + t1) + t2)


def dact(dv, z, sc, sh, leaky):
    """The kernel's float32 dact of compact rows (dv float32 [rows, c], z 16-bit)."""
    if not leaky:
        return dv
    neg = (z.double() * sc.double() + sh.double()) <= 0
    return torch.where(neg, dv * SLOPE, dv)


def reduce_sums(da, z, mu, invstd):
    """float64 (dgamma, dbeta, G, A) of one slab of rows: dgamma = invstd (sum da z - mu sum da), dbeta = sum da,
    G = sum |da z|, A = sum |da|.  Slabs add up linearly; `reduce_ref` finishes them."""
    dd, zd = da.double(), z.double()
    sdz, sd = (dd * zd).sum(0), dd.sum(0)
    return sdz, sd, (dd * zd).abs().sum(0), dd.abs().sum(0)


def reduce_ref(parts, mu, invstd):
    """Sum of reduce_sums slabs -> float64 (dgamma, dbeta, G, A)."""
    sdz, sd, G, A = (sum(p[i] for p in parts) for i in range(4))
    return invstd.double() * (sdz - mu.double() * sd), sd, G, A


def reduce_bound(G, A, mu, invstd, rows_per_block, lanes, grid):
    """Float-operand bounds of (dgamma, dbeta) (module docstring)."""
    n_ops = -(-rows_per_block // lanes) + lanes + grid + BN_SLOTS + 4
    ftz = 2 * grid * FTZ32
    return (n_ops * U32 * invstd.double().abs() * (G + mu.double().abs() * A) + ftz, n_ops * U32 * A + ftz)


def bwd_apply_ref(da, z, ga, invstd, mu, dg, db, count, dtype):
    """float64 dz of compact rows and its bound (module docstring)."""
    k1 = ga.double() * invstd.double()
    k2 = k1 * invstd.double() * dg.double() / count
    dd, zd = da.double(), z.double()
    ref = k1 * (dd - db.double() / count) - k2 * (zd - mu.double())
    S = (k1 * dd).abs() + (k2 * zd).abs() + (k1 * db.double() / count).abs() + (k2 * mu.double()).abs()
    e32 = 10 * U32 * S
    return ref, e32 + 0.5 * ulp(ref.abs() + e32, dtype)
