"""Float64 reference and per-element error bounds for the weight-gradient kernels (csrc/conv_wgrad.cu, and the stem's
csrc/conv_thin.cu: stem_wgrad_tc_kernel).

Reference.  dw = dw0 + dz^T . im2col(x), with dz [P, cout] the gradient of the conv's raw output (a dilated dz is
compacted to its (2p, 2q) positions first) and im2col in the (r, s, c) order of the OHWI weights (conv_ref.im2col).
S = |dz|^T . |im2col(x)| is the sum of the magnitudes of the products.  Both are computed in float64, a band of output
rows of one image at a time, so that even the 1.38 M-pixel layer-1 gradient needs no full im2col.

Exact operands.  When x and dz hold small integers (x, dz in {-2, ..., 2}) and dw0 holds integers, every product and
every partial sum is an integer, and all of them are at most max(S) + max|dw0| in magnitude.  Below 2^24 fp32 holds
each of them exactly; the tensor cores' operand alignment and truncation only drop bits below the sum's least
significant bit, which are zero.  So in every split and atomic order the kernel must equal the reference bit for bit.
The stem's image values k / 8 scale the grid to 1/8: there the premise is 8 (max(S) + max|dw0|) < 2^24.

Float bound of conv_wgrad_kernel (16-bit x and dz, fp32 dw0):

    |got - ref| <= C_STEP * n16 * S  +  (splits + 1) u (S + |dw0|)  +  C_STEP * n16 * (splits + 1) u S
    n16 = 4 * kb_per_split,   u = 2^-24,   C_STEP = 4 * 2^-23 (tests/conv_ref.py)

- Accumulation: one CTA reduces kb_per_split 64-pixel blocks of its split in one wgmma accumulator chain, 4 k16 steps
  per block.  Products of two 16-bit significands are exact in fp32; each k16 step may lose up to C_STEP times the
  magnitude sum of its partial result (conv_ref.py), and the CTA's partial magnitude sum is at most S.
- Reduction: the `splits` CTA partials are added into dw0 with one fp32 atomic each, and every add rounds once to the
  magnitude of the running sum, at most S + |dw0| (plus the accumulation error: the second-order term).

Bound of stem_wgrad_tc_kernel (float32 image x, 16-bit dz [P, 32], dw [32, 27]):

    |got - ref| <= e_split + C_STEP * n16 * S' + (G + 4) u (S' + |dw0|) + C_STEP * n16 * (G + 4) u S'
    e_split = u_T^2 S + eta_T A,   S' = (1 + 2 u_T) S,   n16 = 2 parts x 2 k16 steps x tiles per CTA

- Split: each image value is stored as hi = T(x) and lo = T(x - hi) (x - hi is exact in fp32).  With unit roundoff
  u_T of the 16-bit type T (2^-11 fp16, 2^-8 bf16), |x - hi - lo| <= u_T^2 |x| + eta_T, where eta_T = 2^-25 is half
  the fp16 subnormal spacing (lo of a small value underflows; bf16 has fp32's range: eta = 0).  Summed over the
  products: u_T^2 S + eta_T A with A[co] = sum_p |dz[p, co]|.
- Accumulation: each warp keeps its accumulators over all tiles of its persistent CTA and reduces 32 pixels of every
  128-pixel tile in 2 mma k16 steps, once for hi and once for lo: 2 x 2 steps per tile.  |hi| + |lo| <= (1 + 2 u_T)|x|,
  so the magnitude sum of what the tensor cores add is at most S'.
- Reduction: four warp partials into a zeroed shared-memory sum, then one global atomic per CTA (grid G) into dw0.

The CUDA-core stem_wgrad_kernel (YB_STEM_WGRAD=cuda) multiplies the float32 image directly: every lane runs one fmaf
chain of `ppw` pixels per element, then 8 warps add in shared memory and `blocks` CTAs atomically:

    |got - ref| <= (ppw + 8 + blocks) u (S + |dw0|)
"""
import torch
import torch.nn.functional as F

from tests.conv_ref import C_STEP, U32, im2col

EXACT_LIMIT = 2.0 ** 24
_U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
_ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}


def wgrad_ref(x, dz, k, stride, chunk=1 << 24):
    """x [n, h, w, cin] (any float type, on any device), dz [n, ho, wo, cout] compact -> float64 (ref, S), each
    [cout, k * k * cin] in OHWI order.  `chunk` bounds the float64 elements of one im2col band."""
    n, h, w, c = x.shape
    _, ho, wo, cout = dz.shape
    pad = k // 2
    K = k * k * c
    ref = torch.zeros((cout, K), dtype=torch.float64, device=x.device)
    S = torch.zeros_like(ref)
    rows = max(1, chunk // (wo * K))
    for i in range(n):
        xp = F.pad(x[i:i + 1].double(), (0, 0, pad, pad, pad, pad))
        for r0 in range(0, ho, rows):
            r1 = min(ho, r0 + rows)
            cols = im2col(xp[:, r0 * stride:(r1 - 1) * stride + k], k, stride, 0)
            assert cols.shape[0] == (r1 - r0) * wo, "dz does not match the conv's output size"
            g = dz[i, r0:r1].reshape(-1, cout).double()
            ref += g.t() @ cols
            S += g.abs().t() @ cols.abs()
    return ref, S


def compact_dilated(dzu):
    """[n, 2 ho, 2 wo, c] zero-inserted (stride-2) layout -> the [n, ho, wo, c] gradient at its (2p, 2q) positions."""
    return dzu[:, ::2, ::2]


def wgrad_bound(S, dw0, kb_per_split, splits):
    """Per-element bound of |got - ref| for conv_wgrad_kernel (module docstring); dw0 float64 tensor or 0."""
    acc = C_STEP * 4 * kb_per_split * S
    red = (splits + 1) * U32 * (S + abs(dw0))
    return acc + red + acc * (splits + 1) * U32


def stem_tc_bound(S, dz_abs_sum, dw0, dtype, tiles_per_cta, grid):
    """Per-element bound for stem_wgrad_tc_kernel (module docstring); dz_abs_sum [32] = sum_p |dz[p, co]|."""
    u = _U16[dtype]
    split = u * u * S + _ETA[dtype] * dz_abs_sum.double()[:, None]
    s1 = (1 + 2 * u) * S
    acc = C_STEP * 2 * 2 * tiles_per_cta * s1
    red = (grid + 4) * U32 * (s1 + abs(dw0))
    return split + acc + red + acc * (grid + 4) * U32


def stem_cuda_bound(S, dw0, pixels_per_warp, blocks):
    """Per-element bound for the CUDA-core stem_wgrad_kernel (module docstring)."""
    return (pixels_per_warp + 8 + blocks) * U32 * (S + abs(dw0))
