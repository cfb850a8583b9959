"""CPU tests of the batch-norm reference (tests/bn_ref.py): its float64 backward against torch autograd, its float32
emulation of the coefficient arithmetic against float64, the TwoSum flag of the fma emulation, and its bounds against
a float32 emulation of the kernels' arithmetic."""
import numpy as np
import pytest
import torch

from tests import bn_ref as B
from tests.conv_ref import SLOPE, ulp

EPS = 1e-5


def _layer(seed, rows, c, dtype, res=True):
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn((rows, c), generator=g) * (torch.rand(c, generator=g) + 0.5) + torch.randn(c, generator=g) * 2)
    z = z.to(dtype)
    r = torch.randn((rows, c), generator=g).to(dtype) if res else None
    ga = torch.rand(c, generator=g) + 0.5
    be = torch.randn(c, generator=g) * 0.2
    dA = (torch.randn((rows, c), generator=g) * 0.1).to(dtype)
    return z, r, ga, be, dA


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows,c", [(30, 16), (7, 8), (200, 32)])
def test_reference_matches_autograd(rows, c, dtype):
    """Forward output, dgamma, dbeta and dz of the reference == float64 autograd of leaky(BN(z)) + res."""
    z, r, ga, be, dA = _layer(rows + c, rows, c, dtype)
    zd = z.double().requires_grad_(True)
    gd, bd = ga.double().requires_grad_(True), be.double().requires_grad_(True)
    mu = zd.mean(0)
    var = zd.var(0, unbiased=False)
    y = (zd - mu) / torch.sqrt(var + EPS) * gd + bd
    a = torch.where(y > 0, y, SLOPE * y) + r.double()
    a.backward(dA.double())
    mu64, inv64 = mu.detach(), 1 / torch.sqrt(var.detach() + EPS)
    sc64 = ga.double() * inv64
    sh64 = be.double() - mu64 * sc64

    out, _ = B.apply_ref(z, sc64.float(), sh64.float(), r, True, dtype)
    err = (out.double() - a.detach()).abs()
    # the coefficients' float32 rounding, the fp32 epilogue and the 16-bit store
    assert bool((err <= 0.5 * ulp(a.detach(), dtype) + 1e-5 * (1 + a.detach().abs())).all()), float(err.max())

    da = B.dact(dA.float(), z, sc64, sh64, True)
    dg, db, G, A = B.reduce_ref([B.reduce_sums(da, z, mu64, inv64)], mu64, inv64)
    # the reference takes the kernel's float32 dact = fl32(0.1f * dA): one float32 rounding per term
    assert bool(((dg - gd.grad).abs() <= 2.0 ** -23 * inv64 * (G + mu64.abs() * A)).all())
    assert bool(((db - bd.grad).abs() <= 2.0 ** -23 * A).all())
    dz, bound = B.bwd_apply_ref(da, z, ga.double(), inv64, mu64, dg, db, rows, dtype)
    assert bool(((dz - zd.grad).abs() <= bound).all())


def test_coefficient_emulation_against_float64():
    """batch_coeffs / moving_update in float32 ops: within a few float32 ulps of the float64 formulas."""
    g = torch.Generator().manual_seed(1)
    c, count = 64, 1352
    z = torch.randn((count, c), generator=g, dtype=torch.float64) * 1.5 + 0.7
    su, sq = z.sum(0).float(), (z * z).sum(0).float()
    ga, be = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g)
    var32 = su / count
    var32 = torch.clamp_min(sq / count - var32 * var32, 0)
    inv = (1 / torch.sqrt((var32 + B.f32(EPS)).double())).float()
    assert B.invstd_error(var32, EPS, inv) <= 0.5
    mean, var, sc, sh = B.batch_coeffs(su, sq, count, ga, be, EPS, inv)
    m64 = su.double() / count
    v64 = sq.double() / count - m64 * m64
    assert bool(((mean.double() - m64).abs() <= B.ulp32(mean)).all())
    assert bool(((var.double() - v64).abs() <= 4 * B.ulp32(sq) / count).all())
    assert torch.equal(sc, ga * inv) and torch.equal(sh, be - mean * sc)
    mm, mv = B.moving_update(torch.zeros(c), torch.ones(c), mean, var, count, 0.99)
    d = float(np.float32(0.99))
    assert bool(((mm.double() - (1 - d) * mean.double()).abs() <= 2 * B.ulp32(mm)).all())
    want = d + (1 - d) * var.double() * count / (count - 1)
    assert bool(((mv.double() - want).abs() <= 3 * B.ulp32(mv)).all())


def test_fma_emulation_flags_inexact_sums():
    """fma_f32 is the correctly rounded fmaf where it does not flag the element; it flags a float64 sum that dropped
    bits (product ~2^-40 with 25 significant bits added to 1)."""
    a = torch.tensor([1.5, 1.5, 3.0, -2.0], dtype=torch.float32)
    b = torch.tensor([(1 + 2 ** -23) * 2 ** -40, 0.75, 1 + 2 ** -20, 0.5], dtype=torch.float32)
    c = torch.tensor([1.0, 0.25, -3.0, 1.0], dtype=torch.float32)
    y, inexact = B.fma_f32(a, b, c)
    assert inexact.tolist() == [True, False, False, False]
    assert y[1] == 1.375 and y[2] == 3.0 * 2 ** -20 and y[3] == 0.0


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_bwd_apply_bound_covers_float32_arithmetic(dtype):
    """bn_bwd_apply_kernel's arithmetic in float32 (k1, k2, k3 in the kernel's order, the two fmaf, the store) stays
    within bwd_apply_ref's bound, with a large mean offset so that k2 z and k3 nearly cancel."""
    rng = np.random.default_rng(2)
    rows, c, M = 4096, 64, 4096
    f = np.float32
    z = torch.from_numpy((rng.standard_normal((rows, c)) * 0.3 + 4.0).astype(f)).to(dtype)
    da = (rng.standard_normal((rows, c)) * 0.1).astype(f)
    ga = (rng.random(c) + 0.5).astype(f)
    inv = (rng.random(c) * 3 + 0.5).astype(f)
    mu = (4.0 + rng.standard_normal(c) * 0.01).astype(f)
    dg = (rng.standard_normal(c) * 20).astype(f)
    db = (rng.standard_normal(c) * 20).astype(f)
    inv_m = f(1) / f(M)
    k1 = ga * inv
    k2 = -k1 * inv * dg * inv_m
    k3 = -k1 * db * inv_m - k2 * mu
    zf = z.float().numpy()
    inner = (k2.astype(np.float64) * zf + k3).astype(f)
    out = (k1.astype(np.float64) * da + inner).astype(f)
    got = torch.from_numpy(out).to(dtype)
    t = lambda x: torch.from_numpy(np.asarray(x))
    ref, bound = B.bwd_apply_ref(t(da), z, t(ga), t(inv), t(mu), t(dg), t(db), M, dtype)
    frac = ((got.double() - ref).abs() / bound).max().item()
    assert frac <= 1.0, frac


def test_reduce_bound_covers_a_sequential_float32_sum():
    """One fp32 chain over all rows (lanes = grid = 1) stays within reduce_bound."""
    rng = np.random.default_rng(3)
    rows = 20000
    da = (rng.standard_normal((rows, 4)) * 0.1 + 0.05).astype(np.float32)
    z = torch.from_numpy((rng.standard_normal((rows, 4)) + 3).astype(np.float32)).to(torch.bfloat16)
    zf = z.float().numpy()
    ag = np.zeros(4, np.float32)
    ab = np.zeros(4, np.float32)
    for i in range(rows):
        ab = ab + da[i]
        ag = (da[i].astype(np.float64) * zf[i] + ag).astype(np.float32)     # fmaf: product exact in float64
    mu, inv = torch.full((4,), 3.0), torch.full((4,), 0.5)
    dg = ((ag - np.float32(3.0) * ab) * np.float32(0.5)).astype(np.float32)
    rg, rb, G, A = B.reduce_ref([B.reduce_sums(torch.from_numpy(da), z, mu, inv)], mu, inv)
    bg, bb = B.reduce_bound(G, A, mu, inv, rows, 1, 1)
    assert bool(((torch.from_numpy(dg).double() - rg).abs() <= bg).all())
    assert bool(((torch.from_numpy(ab).double() - rb).abs() <= bb).all())
