"""e4m3 rounding and the error bound of the e4m3 implicit-GEMM conv (csrc/conv_igemm.cu with 1-byte operands).

e4m3 here is the OCP "fn" format of torch.float8_e4m3fn: 4 exponent bits (bias 7), 3 significand bits, no infinities,
largest finite 448, smallest normal 2^-6, subnormal spacing 2^-9.  The engine stores RN-satfinite codes
(cvt.rn.satfinite.e4m3x2.f32), so the reference clamps to +-448 before it rounds.

Bound of the e4m3 conv: the products of two e4m3 codes are exact; the tensor core adds them in fp32-like accumulators
whose additions may keep fewer bits than fp32 (fp8 wgmma on Hopper is documented to accumulate with reduced
precision), so each k32 step is allowed C_STEP8 * S of error, S = sum |x * w| in code units.  The epilogue rounds
fmaf(acc, scale, shift), the leaky product, the residual fma and the 1/s_out product once each in fp32.  An output
equals RN(ref) wherever ref lies farther than the bound from a rounding midpoint; everywhere it is within one e4m3 ulp
of RN(ref), or, near zero where the subnormal spacing (2^-9) is finer than the bound, within one ulp plus the bound.
"""
import numpy as np
import torch

E4M3_MAX = 448.0
U32 = 2.0 ** -24
C_STEP8 = 2.0 ** -13               # accumulator error per k32 step, relative to sum |x * w| (about 14-bit accumulation)


def e4m3_round(x):
    """Round-to-nearest-even to e4m3 values after clamping to +-448; float64 tensor in, float64 tensor out."""
    x = x.double().clamp(-E4M3_MAX, E4M3_MAX)
    _, e = torch.frexp(x.abs())                          # |x| = m 2^e, m in [0.5, 1)
    q = torch.exp2(torch.clamp(e.double() - 1, min=-6) - 3)   # spacing: 2^(floor(log2|x|) - 3), subnormals 2^-9
    return torch.round(x / q) * q                         # torch.round: half to even; x / q is exact


def e4m3_ulp(a):
    """Spacing of e4m3 at magnitude |a| (float64)."""
    _, e = torch.frexp(a.abs())
    e = torch.where(a == 0, torch.full_like(a, -6.0), torch.clamp(e.double() - 1, min=-6))
    return torch.exp2(e - 3)


def to_codes(v):
    """float tensor of e4m3 values -> uint8 codes (via torch.float8_e4m3fn; exact for representable values)."""
    return v.float().to(torch.float8_e4m3fn).view(torch.uint8)


def from_codes(u):
    return u.view(torch.float8_e4m3fn).double()


def fp8_bound(S, n32, scale, shift, res=None, res_scale=1.0):
    """Per-element bound of the fp32 value before the e4m3 store (see the module docstring); S in code units."""
    sc = scale.double().abs()
    r = 0.0 if res is None else res.double().abs() * res_scale
    return sc * (C_STEP8 * n32) * S + 4 * U32 * (sc * S + shift.double().abs() + r)


def check_e4m3(got_codes, ref_scaled, bound_scaled, what=""):
    """got: e4m3 codes; ref: float64 value / s_out; bound: its bound / s_out.  Asserts the two criteria of the module
    docstring and returns (exact fraction checked, worst |got - RN(ref)| in ulps, outputs more than one ulp away)."""
    got = from_codes(got_codes)
    ref = ref_scaled.clamp(-E4M3_MAX, E4M3_MAX)
    rn = e4m3_round(ref)
    ulp = e4m3_ulp(rn)
    err_ulp = (got - rn).abs() / ulp
    # within one ulp of RN(ref); near zero, where the e4m3 spacing is finer than the accumulation bound, within one
    # ulp plus the bound
    far = (err_ulp > 1.0) & ((got - ref).abs() > ulp + bound_scaled)
    if bool(far.any()):
        i = far.nonzero()[0]
        i = tuple(i.tolist())
        raise AssertionError(f"{what}: {int(far.sum())} outputs more than one ulp (+ bound) from RN(ref); first at {i}: "
                             f"got {float(got[i])} RN(ref) {float(rn[i])} ref {float(ref[i]):.6g} bound {float(bound_scaled[i]):.3g}")
    # distance of ref to the nearest rounding midpoint: half an ulp minus its distance to RN(ref)
    a, r = ref.abs(), rn.abs()
    lo_ulp = torch.minimum(ulp, e4m3_ulp(r - ulp * 0.75))    # below a power of two the spacing halves
    mid = torch.where(a >= r, 0.5 * ulp, 0.5 * lo_ulp) - (a - r).abs()
    safe = mid.abs() > bound_scaled
    bad = safe & (got != rn)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} outputs differ from RN(ref) away from a midpoint"
    return float(safe.double().mean()), float(err_ulp.max()), int((err_ulp > 1.0).sum())
