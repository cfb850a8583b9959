"""GPU parity tests of the training-mode operators (wgrad / dgrad on the tensor cores, BN
forward/backward, bias gradient) through the C ABI, against PyTorch fp32 autograd on the
same 16-bit-rounded operands."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _L():
    from yolov3_tensorflow_b200 import _lib
    return _lib


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-6))


WGRAD_SHAPES = [
    (2, 16, 16, 64, 128, 3, 1, 0),        # BNW=64, two A blocks
    (3, 13, 13, 128, 64, 1, 1, 0),        # 1x1, cout=64 (single A block), BNW=128
    (2, 20, 12, 32, 64, 3, 1, 0),         # cin=32 -> 64B-swizzled B
    (2, 26, 26, 128, 256, 3, 1, 256),     # input is a channel slice; 2 co tiles
    (2, 13, 13, 256, 255, 1, 1, 0),       # detection head: cout=255, dz_ld=256
    (2, 52, 52, 64, 128, 3, 2, 0),        # stride 2 (plain dz)
    (2, 32, 32, 32, 64, 3, 2, 0),         # layer-1 shape: cin=32, stride 2, all 9 taps in one CTA
]


@pytest.mark.parametrize("n,h,w,cin,cout,k,s,in_extra", WGRAD_SHAPES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])    # the fp16 training path runs fp16 wgrad
def test_wgrad_matches_autograd(n, h, w, cin, cout, k, s, in_extra, dtype):
    _wgrad_vs_autograd(n, h, w, cin, cout, k, s, in_extra, dtype)


@pytest.mark.parametrize("n,h,w,cin,cout,k,s,in_extra", [sh for sh in WGRAD_SHAPES if sh[5] == 3])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_wgrad_one_tap_per_cta(n, h, w, cin, cout, k, s, in_extra, dtype):
    """YB_WGRAD_TP=1: the 3x3 wgrad with one filter tap per CTA instead of one kernel row (three taps)."""
    L = _L()
    L.set_option("YB_WGRAD_TP", "1")
    try:
        _wgrad_vs_autograd(n, h, w, cin, cout, k, s, in_extra, dtype)
    finally:
        L.set_option("YB_WGRAD_TP", None)


def _wgrad_vs_autograd(n, h, w, cin, cout, k, s, in_extra, dtype):
    L = _L()
    g = torch.Generator().manual_seed(1)
    in_ld = cin + in_extra
    off = in_extra // 2 // 8 * 8
    xfull = torch.randn((n, h, w, in_ld), generator=g).to(dtype).cuda()
    ho, wo = h // s, w // s
    dz_ld = (cout + 7) // 8 * 8
    dz = torch.zeros((n, ho, wo, dz_ld), dtype=dtype, device="cuda")
    dz[..., :cout] = (torch.randn((n, ho, wo, cout), generator=g) * 0.1).to(dtype).cuda()
    dw = torch.zeros((cout, k, k, cin), dtype=torch.float32, device="cuda")
    d = L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=k, stride=s, in_ld=in_ld, out_ld=dz_ld, res_ld=0,
                   dtype=L.YB_F16 if dtype == torch.float16 else L.YB_BF16, out_fp32=0, leaky=0, upsample2x=0)
    xp = C.c_void_p(xfull.data_ptr() + off * 2)
    for _ in range(2):   # accumulates: run twice, expect 2x
        L.check(L.lib.yb_conv2d_wgrad(C.byref(d), xp, L.ptr(dz), dz_ld, 0, L.ptr(dw), L.stream_handle()), "wgrad")
    torch.cuda.synchronize()
    x = xfull[..., off:off + cin].float().permute(0, 3, 1, 2)
    wt = torch.zeros((cout, cin, k, k), device="cuda", requires_grad=True)
    y = F.conv2d(x, wt, None, stride=s, padding=k // 2)
    y.backward(dz[..., :cout].float().permute(0, 3, 1, 2))
    ref = 2 * wt.grad.permute(0, 2, 3, 1)
    assert _rel(dw, ref) < 2e-3, _rel(dw, ref)


def test_wgrad_dilated_dz_stride2():
    L = _L()
    g = torch.Generator().manual_seed(2)
    n, h, w, cin, cout = 2, 32, 48, 64, 128
    x = torch.randn((n, h, w, cin), generator=g).to(torch.bfloat16).cuda()
    dzc = (torch.randn((n, h // 2, w // 2, cout), generator=g) * 0.1).to(torch.bfloat16).cuda()
    dzu = torch.zeros((n, h, w, cout), dtype=torch.bfloat16, device="cuda")
    dzu[:, ::2, ::2] = dzc
    dw = torch.zeros((cout, 3, 3, cin), dtype=torch.float32, device="cuda")
    d = L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=3, stride=2, in_ld=cin, out_ld=cout, res_ld=0,
                   dtype=L.YB_BF16, out_fp32=0, leaky=0, upsample2x=0)
    L.check(L.lib.yb_conv2d_wgrad(C.byref(d), L.ptr(x), L.ptr(dzu), cout, 1, L.ptr(dw), L.stream_handle()), "wgrad")
    wt = torch.zeros((cout, cin, 3, 3), device="cuda", requires_grad=True)
    F.conv2d(x.float().permute(0, 3, 1, 2), wt, None, stride=2, padding=1).backward(dzc.float().permute(0, 3, 1, 2))
    assert _rel(dw, wt.grad.permute(0, 2, 3, 1)) < 2e-3


@pytest.mark.parametrize("k,s,cin,cout", [(3, 1, 64, 128), (1, 1, 128, 64), (3, 2, 64, 128), (1, 1, 256, 255)])
def test_dgrad_via_forward_kernel(k, s, cin, cout):
    """dX = yb_conv2d_fwd(dz [zero-inserted for stride 2], flipped/transposed weights)."""
    L = _L()
    g = torch.Generator().manual_seed(3)
    n, h, w = 2, 24, 16
    ho, wo = h // s, w // s
    wt = (torch.randn((cout, k, k, cin), generator=g) * 0.05).cuda()          # OHWI master
    kco = (cout + 31) // 32 * 32
    cin_pad = L.lib.yb_conv_cout_pad(cin)
    wd = torch.empty((cin_pad, k, k, kco), dtype=torch.bfloat16, device="cuda")
    L.check(L.lib.yb_pack_dgrad_weights(L.ptr(wt), cout, cin, k, kco, cin_pad, L.YB_BF16, L.ptr(wd), L.stream_handle()), "packd")
    dzc = torch.zeros((n, ho, wo, kco), dtype=torch.bfloat16, device="cuda")
    dzc[..., :cout] = (torch.randn((n, ho, wo, cout), generator=g) * 0.1).to(torch.bfloat16).cuda()
    if s == 2:
        dzin = torch.zeros((n, h, w, kco), dtype=torch.bfloat16, device="cuda"); dzin[:, ::2, ::2] = dzc
    else:
        dzin = dzc
    prev = (torch.randn((n, h, w, cin), generator=g) * 0.1).to(torch.bfloat16).cuda()   # earlier contribution, added in place
    out = prev.clone()
    one = torch.ones(cin_pad, device="cuda"); zero = torch.zeros(cin_pad, device="cuda")
    d = L.ConvDesc(n=n, h=h, w=w, cin=kco, cout=cin, ksize=k, stride=1, in_ld=kco, out_ld=cin, res_ld=cin,
                   dtype=L.YB_BF16, out_fp32=0, leaky=0, upsample2x=0)
    L.check(L.lib.yb_conv2d_fwd(C.byref(d), L.ptr(dzin), L.ptr(wd), L.ptr(one), L.ptr(zero), L.ptr(out), L.ptr(out), None, None,
                                L.stream_handle()), "dgrad")
    x = torch.zeros((n, cin, h, w), device="cuda", requires_grad=True)
    wq = wd[:cin, :, :, :cout].float()     # undo flip/transpose on the rounded values
    w_oihw = wq.flip(1, 2).permute(3, 0, 1, 2).contiguous()
    F.conv2d(x, w_oihw, None, stride=s, padding=k // 2).backward(dzc[..., :cout].float().permute(0, 3, 1, 2))
    ref = x.grad.permute(0, 2, 3, 1) + prev.float()
    err = (out.float() - ref).abs()
    assert torch.all(err <= 2.0 ** -6 * torch.clamp(ref.abs(), min=0.05)), float(err.max())


@pytest.mark.parametrize("cin,cout,with_res", [(32, 64, True), (64, 128, False), (256, 512, True)])
def test_dgrad_stride2_parity_classes(cin, cout, with_res):
    """dX of a 3x3 stride-2 conv as four parity-class convs over the plain dz (no zero insertion)."""
    L = _L()
    g = torch.Generator().manual_seed(8)
    n, h, w = 2, 24, 20
    ho, wo = h // 2, w // 2
    wt = (torch.randn((cout, 3, 3, cin), generator=g) * 0.05).cuda()
    kco = (cout + 31) // 32 * 32
    cin_pad = L.lib.yb_conv_cout_pad(cin)
    wd = torch.empty(9 * cin_pad * kco, dtype=torch.bfloat16, device="cuda")
    L.check(L.lib.yb_pack_dgrad_weights_s2(L.ptr(wt), cout, cin, kco, cin_pad, L.YB_BF16, L.ptr(wd), L.stream_handle()), "packd_s2")
    dz = (torch.randn((n, ho, wo, kco), generator=g) * 0.1).to(torch.bfloat16).cuda()
    prev = (torch.randn((n, h, w, cin), generator=g) * 0.1).to(torch.bfloat16).cuda()
    out = prev.clone() if with_res else torch.full((n, h, w, cin), 7.0, dtype=torch.bfloat16, device="cuda")
    d = L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=3, stride=2, in_ld=cin, out_ld=cout, res_ld=0,
                   dtype=L.YB_BF16, out_fp32=0, leaky=0, upsample2x=0)
    L.check(L.lib.yb_conv2d_dgrad_s2(C.byref(d), L.ptr(dz), kco, kco, L.ptr(wd), L.ptr(out) if with_res else None, cin,
                                     L.ptr(out), cin, L.stream_handle()), "dgrad_s2")
    x = torch.zeros((n, cin, h, w), device="cuda", requires_grad=True)
    wq = wt.to(torch.bfloat16).float()                    # the packer rounds the master weights to 16 bits
    F.conv2d(x, wq.permute(0, 3, 1, 2).contiguous(), None, stride=2, padding=1).backward(
        dz[..., :cout].float().permute(0, 3, 1, 2))
    ref = x.grad.permute(0, 2, 3, 1) + (prev.float() if with_res else 0)
    err = (out.float() - ref).abs()
    assert torch.all(err <= 2.0 ** -6 * torch.clamp(ref.abs(), min=0.05)), float(err.max())


@pytest.fixture(params=["cpt4", "cpt8"])
def bn_shape(request):
    """Both builds of the BN streaming kernels (4 or 8 channels per thread; csrc/bn.cu)."""
    L = _L()
    L.set_option("YB_BN_CPT", "4" if request.param == "cpt4" else None)
    yield request.param
    L.set_option("YB_BN_CPT", None)


@pytest.mark.parametrize("upsample,res,c", [(False, True, 64), (True, False, 128), (False, False, 32), (False, True, 1024),
                                            (False, False, 2048), (False, False, 8)])
def test_bn_train_forward_backward(upsample, res, c, bn_shape):
    L = _L()
    lib, ptr, st = L.lib, L.ptr, L.stream_handle
    g = torch.Generator().manual_seed(4)
    n, h, w = 3, 10, 6
    dt = torch.bfloat16
    z = (torch.randn((n, h, w, c), generator=g) * 2 + 0.3).to(dt).cuda()
    gamma = (torch.rand(c, generator=g) + 0.5).cuda(); beta = (torch.randn(c, generator=g) * 0.2).cuda()
    mm = torch.zeros(c).cuda(); mv = torch.ones(c).cuda()
    zf = z.float()
    rows = n * h * w
    ssum = zf.sum(dim=(0, 1, 2)); ssq = (zf * zf).sum(dim=(0, 1, 2))
    scale = torch.empty(c).cuda(); shift = torch.empty(c).cuda(); smean = torch.empty(c).cuda(); sinv = torch.empty(c).cuda()
    L.check(lib.yb_bn_finalize(ptr(ssum), ptr(ssq), rows, c, ptr(gamma), ptr(beta), 1e-5, 0.99, ptr(mm), ptr(mv), ptr(scale), ptr(shift),
                               ptr(smean), ptr(sinv), st()), "finalize")
    mean = zf.mean(dim=(0, 1, 2)); var = zf.var(dim=(0, 1, 2), unbiased=False)
    torch.testing.assert_close(smean, mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(sinv, 1 / torch.sqrt(var + 1e-5), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(mm, 0.01 * mean, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(mv, 0.99 + 0.01 * var * rows / (rows - 1), rtol=1e-4, atol=1e-6)
    r = (torch.randn((n, h, w, c), generator=g)).to(dt).cuda() if res else None
    up = 2 if upsample else 1
    out = torch.empty((n, h * up, w * up, c), dtype=dt, device="cuda")
    L.check(lib.yb_bn_act_apply(ptr(z), c, ptr(scale), ptr(shift), ptr(r), c, ptr(out), c, n, h, w, c, L.YB_BF16, 1, int(upsample), st()), "apply")
    # the one-launch form (statistics -> scale/shift inside the apply kernel) is bit-identical to the two calls above
    mm2 = torch.zeros(c).cuda(); mv2 = torch.ones(c).cuda()
    sc2 = torch.empty(c).cuda(); sh2 = torch.empty(c).cuda(); sm2 = torch.empty(c).cuda(); si2 = torch.empty(c).cuda()
    out2 = torch.empty_like(out)
    L.check(lib.yb_bn_stats_act_apply(ptr(z), c, ptr(ssum), ptr(ssq), ptr(gamma), ptr(beta), 1e-5, 0.99, ptr(mm2), ptr(mv2), ptr(sc2),
                                      ptr(sh2), ptr(sm2), ptr(si2), ptr(r), c, ptr(out2), c, n, h, w, c, L.YB_BF16, 1, int(upsample),
                                      st()), "stats_act_apply")
    for a_, b_ in ((mm2, mm), (mv2, mv), (sc2, scale), (sh2, shift), (sm2, smean), (si2, sinv), (out2, out)):
        assert torch.equal(a_, b_)
    # reference through autograd
    zr = zf.clone().requires_grad_(True); gr = gamma.clone().requires_grad_(True); br = beta.clone().requires_grad_(True)
    y = (zr - mean) / torch.sqrt(var + 1e-5)
    m2 = zr.mean(dim=(0, 1, 2)); v2 = zr.var(dim=(0, 1, 2), unbiased=False)
    y = (zr - m2) / torch.sqrt(v2 + 1e-5) * gr + br
    a = torch.where(y > 0, y, 0.1 * y)
    if res:
        a = a + r.float()
    if upsample:
        a = a.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    err = (out.float() - a).abs()
    assert torch.all(err <= 2.0 ** -6 * torch.clamp(a.abs(), min=1.0)), float(err.max())
    dA = (torch.randn(a.shape, generator=g) * 0.1).to(dt).cuda()
    a.backward(dA.float())
    dgam = torch.empty(c).cuda(); dbet = torch.empty(c).cuda()
    need = C.c_size_t()
    L.check(lib.yb_bn_bwd_reduce_workspace_bytes(C.byref(need)), "ws")
    ws = torch.zeros(need.value, dtype=torch.uint8, device="cuda")
    for workspace in (None, ws, ws):          # atomic path, two-stage path (twice: the ticket must reset itself)
        dgam.fill_(-1); dbet.fill_(-1)
        L.check(lib.yb_bn_bwd_reduce(ptr(dA), c, ptr(z), c, ptr(scale), ptr(shift), ptr(smean), ptr(sinv), n, h, w, c, L.YB_BF16, 1,
                                     int(upsample), ptr(dgam), ptr(dbet), ptr(workspace), st()), "bwd_reduce")
        torch.testing.assert_close(dgam, gr.grad, rtol=2e-3, atol=2e-3)
        torch.testing.assert_close(dbet, br.grad, rtol=2e-3, atol=2e-3)
    for dil in (0, 1):
        dz = torch.zeros((n, h * (2 if dil else 1), w * (2 if dil else 1), c), dtype=dt, device="cuda")
        L.check(lib.yb_bn_bwd_apply(ptr(dA), c, ptr(z), c, ptr(gamma), ptr(scale), ptr(shift), ptr(smean), ptr(sinv), ptr(dgam), ptr(dbet),
                                    n, h, w, c, L.YB_BF16, 1, int(upsample), dil, ptr(dz), c, st()), "bwd_apply")
        got = dz[:, ::2, ::2] if dil else dz
        e = (got.float() - zr.grad).abs()
        assert float(e.max()) <= 2e-2 * float(zr.grad.abs().max()), float(e.max())
        if dil:
            assert float(dz[:, 1::2].abs().max()) == 0 and float(dz[:, :, 1::2].abs().max()) == 0


def test_col_sum_and_stem_wgrad():
    L = _L()
    g = torch.Generator().manual_seed(5)
    x = (torch.randn((1000, 256), generator=g) * 0.1).to(torch.bfloat16).cuda()
    out = torch.empty(255).cuda()
    L.check(L.lib.yb_col_sum(L.ptr(x), 256, 1000, 255, L.YB_BF16, L.ptr(out), L.stream_handle()), "colsum")
    torch.testing.assert_close(out, x.float().sum(0)[:255], rtol=1e-4, atol=1e-4)
    n, h, w = 2, 24, 40
    img = torch.rand((n, h, w, 3), generator=g).cuda()
    dz = (torch.randn((n, h, w, 32), generator=g) * 0.1).to(torch.bfloat16).cuda()
    dw = torch.zeros((32, 3, 3, 3), device="cuda")
    L.check(L.lib.yb_stem_conv_wgrad(L.ptr(img), L.ptr(dz), L.YB_BF16, n, h, w, L.ptr(dw), L.stream_handle()), "stem_wgrad")
    wt = torch.zeros((32, 3, 3, 3), device="cuda", requires_grad=True)
    F.conv2d(img.permute(0, 3, 1, 2), wt, None, padding=1).backward(dz.float().permute(0, 3, 1, 2))
    assert _rel(dw, wt.grad.permute(0, 2, 3, 1)) < 1e-4
    # tensor-path kernel explicitly, fp16 gradients, a size that is not a multiple of the 8x16 tile
    n, h, w = 3, 20, 28
    img = torch.rand((n, h, w, 3), generator=g).cuda()
    for dt, code in ((torch.float16, L.YB_F16), (torch.bfloat16, L.YB_BF16)):
        dz = (torch.randn((n, h, w, 32), generator=g) * 0.1).to(dt).cuda()
        dw = torch.zeros((32, 3, 3, 3), device="cuda")
        L.check(L.lib.yb_stem_conv_wgrad_tc(L.ptr(img), L.ptr(dz), code, n, h, w, L.ptr(dw), L.stream_handle()), "stem_wgrad_tc")
        wt = torch.zeros((32, 3, 3, 3), device="cuda", requires_grad=True)
        F.conv2d(img.permute(0, 3, 1, 2), wt, None, padding=1).backward(dz.float().permute(0, 3, 1, 2))
        assert _rel(dw, wt.grad.permute(0, 2, 3, 1)) < 1e-4
