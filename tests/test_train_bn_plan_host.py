"""CPU tests of the machinery of tests/test_gpu_train_bn_plan.py (no GPU needed).

- On unbound training plans, through yb_bn_schedule at 132 SMs: every configuration's BN launches run the R-row loop
  past its first group, end in a short last block and put >= 16 blocks on every workspace slot; cpt4 runs CPT 4.
- The two-ranks configuration doubles the forward sums and the count: batch_coeffs gives the same bits.
- With the float32 emulations of tests/bn_ref.py on synthetic tensors, each fault the GPU test exists to catch breaks
  bit-equality or exceeds its bound, while the fault-free emulation passes: the count without the replicas, one
  upsampled copy of dA dropped, decay swapped with 1 - decay, the residual of the neighbouring layer, the shift of the
  neighbouring channel, dgamma and dbeta swapped.
- The column-sum bound covers a subnormal that yb_col_sum's atomic add flushes to zero.
- yb_net_bn_batch_stats rejects an unbound plan, an inference plan and a detection head."""
import ctypes as C

import pytest
import torch

from tests import bn_ref as B
from tests import conv_ref as R
from tests import train_bn_plan_ref as BP
from tests import train_plan_ref as T

DTYPES = [torch.float16, torch.bfloat16]


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    BP.set_options(_lib, {})
    yield _lib
    BP.set_options(_lib, {})


def _infos(L, n, H, W, code, training=1):
    net = C.c_void_p()
    L.check(L.lib.yb_net_create(C.byref(net), T.CLASSES, n, H, W, code, training), "net_create")
    try:
        out = []
        for i in range(L.lib.yb_net_num_layers(net)):
            info = L.LayerInfo()
            L.check(L.lib.yb_net_layer_info(net, i, C.byref(info)), "layer_info")
            out.append(info)
        return out
    finally:
        L.lib.yb_net_destroy(net)


@pytest.mark.parametrize("cid,opts,mode,dt,n,hw", BP.CONFIGS, ids=[c[0] for c in BP.CONFIGS])
def test_configuration_premise(L, cid, opts, mode, dt, n, hw):
    BP.set_options(L, opts)
    infos = _infos(L, n, hw[0], hw[1], L.YB_F16 if dt == "fp16" else L.YB_BF16)
    scheds = BP.premise(L, cid, opts, infos, n)
    assert len(scheds) == 72
    if cid != "cpt4":
        assert all(s.cpt == 8 for s in scheds.values()), cid


def test_bn_batch_stats_rejects(L):
    heads = T.Topology().heads
    for training in (1, 0):
        net = C.c_void_p()
        L.check(L.lib.yb_net_create(C.byref(net), T.CLASSES, 2, 416, 416, L.YB_BF16, training), "net_create")
        try:
            p = [C.c_void_p() for _ in range(4)]
            args = [C.byref(q) for q in p]
            assert L.lib.yb_net_bn_batch_stats(net, 0, *args) == -1
            msg = L.lib.yb_last_error_string().decode()
            assert ("not a bound training plan" if training else "bad argument") in msg, msg
            if training:
                assert L.lib.yb_net_bn_batch_stats(net, heads[0], *args) == -1
                msg = L.lib.yb_last_error_string().decode()
                assert f"layer {heads[0]} has no batch norm" in msg, msg
                assert L.lib.yb_net_bn_batch_stats(net, 75, *args) == -1
        finally:
            L.lib.yb_net_destroy(net)


# ---------------------------------------------------------------------------------------- synthetic float32 layer
class Layer:
    """A BN layer of n x h x w rows, c channels, stored in dtype, with its float32 coefficients."""

    def __init__(self, dtype, seed, n=2, h=6, w=8, c=16):
        g = torch.Generator().manual_seed(seed)
        self.n, self.h, self.w, self.c, self.dtype = n, h, w, c, dtype
        self.rows = n * h * w
        off = torch.randn(c, generator=g) * 2
        self.z = (torch.randn((self.rows, c), generator=g) * (torch.rand(c, generator=g) + 0.5) + off).to(dtype)
        zd = self.z.double()
        self.su, self.sq = zd.sum(0).float(), (zd * zd).sum(0).float()
        self.ga = torch.rand(c, generator=g) + 0.5
        self.be = torch.randn(c, generator=g) * 0.2
        self.mm, self.mv = torch.randn(c, generator=g) * 0.1, torch.rand(c, generator=g) + 0.5
        self.res = torch.randn((self.rows, c), generator=g).to(dtype)
        self.res_other = torch.randn((self.rows, c), generator=g).to(dtype)
        self.dA4 = (torch.randn((n, 2 * h, 2 * w, c), generator=g) * 0.1).to(dtype)
        self.dA = (torch.randn((self.rows, c), generator=g) * 0.1).to(dtype)
        self.coeffs(self.su, self.sq, self.rows)

    def coeffs(self, su, sq, count):
        mean = su / B.f32(count)
        var = torch.clamp_min(sq / B.f32(count) - mean * mean, 0.0)
        self.inv = (1.0 / torch.sqrt((var + B.f32(BP.EPS)).double())).float()      # a correctly rounded rsqrtf
        self.mean, self.var, self.sc, self.sh = B.batch_coeffs(su, sq, count, self.ga, self.be, BP.EPS, self.inv)

    def dact(self, dv):
        return B.dact(dv, self.z, self.sc, self.sh, True)

    def reduce32(self, da):
        """bn_bwd_reduce in float32 (a different summation order than the kernel's; within the same bound)."""
        zf = self.z.float()
        sdz, sd = (da * zf).sum(0), da.sum(0)
        return (sdz - self.mean * sd) * self.inv, sd

    def bwd_apply32(self, da, dg, db, count):
        """bn_bwd_apply_kernel's float32 k1 / k2 / k3 and its two fmaf (as float64 then rounded)."""
        inv_m = B.f32(1.0) / B.f32(count)
        k1 = self.ga * self.inv
        k2 = -k1 * self.inv * dg * inv_m
        k3 = -k1 * db * inv_m - k2 * self.mean
        inner = (k2.double() * self.z.double() + k3.double()).float()
        return (k1.double() * da.double() + inner.double()).float().to(self.dtype)

    def check_reduce(self, dg, db, da_ref):
        from yolov3_tensorflow_b200 import _lib
        s = BP.bn_schedule(_lib, self.rows, self.c)
        dg_ref, db_ref, G, A = B.reduce_ref([B.reduce_sums(da_ref, self.z, self.mean, self.inv)], self.mean, self.inv)
        bg, bb = B.reduce_bound(G, A, self.mean, self.inv, s.rows_per_block, s.lanes, s.grid)
        R.check_out(dg, dg_ref, bg, "dgamma")
        R.check_out(db, db_ref, bb, "dbeta")


def _fails(fn):
    with pytest.raises(AssertionError):
        fn()


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_doubled_sums_and_count_give_the_same_coefficients(dtype):
    s = Layer(dtype, 1)
    one = B.batch_coeffs(s.su, s.sq, s.rows, s.ga, s.be, BP.EPS, s.inv)
    two = B.batch_coeffs(s.su * 2, s.sq * 2, 2 * s.rows, s.ga, s.be, BP.EPS, s.inv)
    for a, b in zip(one, two):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_count_without_replicas_fails(dtype):
    s = Layer(dtype, 2)
    su2, sq2 = s.su * 2, s.sq * 2                       # the sums of two identical ranks
    want = B.batch_coeffs(su2, sq2, 2 * s.rows, s.ga, s.be, BP.EPS, s.inv)
    bad = B.batch_coeffs(su2, sq2, s.rows, s.ga, s.be, BP.EPS, s.inv)
    assert not torch.equal(want[0], bad[0]) and not torch.equal(want[1], bad[1]) and not torch.equal(want[3], bad[3])
    # dz: the backward sums of two ranks over 2 x rows
    da = s.dact(s.dA.float())
    dg, db = s.reduce32(da)
    dg2, db2 = dg * 2, db * 2
    ref, bound = B.bwd_apply_ref(da, s.z, s.ga, s.inv, s.mean, dg2, db2, 2 * s.rows, dtype)
    R.check_out(s.bwd_apply32(da, dg2, db2, 2 * s.rows), ref, bound, "dz")
    _fails(lambda: R.check_out(s.bwd_apply32(da, dg2, db2, s.rows), ref, bound, "dz, count without replicas"))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_dropped_upsampled_copy_fails(dtype):
    s = Layer(dtype, 3)
    b = s.dA4
    good = B.upsampled_rows(b).reshape(-1, s.c)
    v, t0, t1 = b[:, 0::2, 0::2].float(), b[:, 0::2, 1::2].float(), b[:, 1::2, 0::2].float()
    dropped = (v + (t0 + t1)).reshape(-1, s.c)
    da, da_bad = s.dact(good), s.dact(dropped)
    s.check_reduce(*s.reduce32(da), da)
    _fails(lambda: s.check_reduce(*s.reduce32(da_bad), da))
    dg, db = s.reduce32(da)
    ref, bound = B.bwd_apply_ref(da, s.z, s.ga, s.inv, s.mean, dg, db, s.rows, dtype)
    R.check_out(s.bwd_apply32(da, dg, db, s.rows), ref, bound, "dz")
    _fails(lambda: R.check_out(s.bwd_apply32(da_bad, dg, db, s.rows), ref, bound, "dz, copy dropped"))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_swapped_decay_fails(dtype):
    s = Layer(dtype, 4)
    mm, mv = B.moving_update(s.mm, s.mv, s.mean, s.var, s.rows, 0.99)
    mm2, mv2 = B.moving_update(s.mm, s.mv, s.mean, s.var, s.rows, 1 - 0.99)
    assert not torch.equal(mm, mm2) and not torch.equal(mv, mv2)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_neighbouring_residual_and_shift_fail(dtype):
    s = Layer(dtype, 5)
    want, inexact = B.apply_ref(s.z, s.sc, s.sh, s.res, True, dtype)
    got, _ = B.apply_ref(s.z, s.sc, s.sh, s.res, True, dtype)
    B.check_apply(got, want, inexact, dtype, "activation")
    other, _ = B.apply_ref(s.z, s.sc, s.sh, s.res_other, True, dtype)
    _fails(lambda: B.check_apply(other, want, inexact, dtype, "activation, residual of another layer"))
    shifted, _ = B.apply_ref(s.z, s.sc, s.sh.roll(1), s.res, True, dtype)
    _fails(lambda: B.check_apply(shifted, want, inexact, dtype, "activation, neighbouring channel's shift"))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_swapped_dgamma_dbeta_fail(dtype):
    s = Layer(dtype, 6)
    da = s.dact(s.dA.float())
    dg, db = s.reduce32(da)
    s.check_reduce(dg, db, da)
    _fails(lambda: s.check_reduce(db, dg, da))
    ref, bound = B.bwd_apply_ref(da, s.z, s.ga, s.inv, s.mean, dg, db, s.rows, dtype)
    _fails(lambda: R.check_out(s.bwd_apply32(da, db, dg, s.rows), ref, bound, "dz, dgamma / dbeta swapped"))


def test_col_sum_bound_covers_flushed_atomics():
    """A head column whose only nonzero dz is a bf16 subnormal: yb_col_sum's atomic add flushes the slab total, so the
    device sums to 0.  col_stats_bound covers that through its flush term; its depth term alone would not."""
    rows, c = 2 * 13 * 13, 255
    v = torch.tensor([1.83671e-40], dtype=torch.bfloat16).double()
    assert 0 < float(v) < B.FTZ32
    assert float(v.abs()) <= float(BP.col_stats_bound(v.abs(), rows, c, BP.SMS))
    assert float(v.abs()) > float(BP.col_stats_bound(v.abs(), rows, c, BP.SMS) - 2 * -(-rows // 32) * B.FTZ32)
