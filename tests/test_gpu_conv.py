"""GPU parity tests of the wgmma implicit-GEMM conv through the C ABI (yb_conv2d_fwd); the direct conv kernels
(halo-tile, thin, stems) are tested against float64 in tests/test_gpu_conv_direct.py.
Reference: plain PyTorch fp32 conv2d on the same
fp16/bf16-rounded operands.  Tolerance: fp32-accumulation-order noise + one output
rounding: |err| <= 2^-9 * max(1, |ref|) for fp16 storage (2^-6 for bf16)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["1cta", "2cta", "mc", "1cta-reg", "2cta-reg", "1cta-eg1", "2cta-eg1", "1cta-eg2", "2cta-eg2",
                        "1cta-pp"], autouse=True)
def conv_mode(request):
    """Every conv test runs against the kernel variants: one CTA per tile ("1cta", the default: ping-pong for the
    windowed convs and the 64-column 1x1 convs, cooperative for the 128-column 1x1 convs), clusters of 2 CTAs sharing a
    TMA-multicast weight tile ("2cta") and clusters of 4 ("mc"); for the first two also against the register-store
    epilogue ("-reg", instead of the shared-memory staging tile) and with one consumer warpgroup ("-eg1", 64-row tiles).
    "-eg2" pins two consumer warpgroups (128-row tiles) sharing every tile: "1cta-eg2" is the cooperative schedule
    wherever the default would ping-pong (YB_CONV_PP=0), "2cta-eg2" the 2-CTA clusters with the grid capped at one
    cluster (YB_CONV_CTAS=2), so that it runs many units.  "1cta-pp" is ping-pong wherever the kernel allows it
    (YB_CONV_PP=1), the 128-column 1x1 convs included.  The library's option table (yb_set_option) selects the variant;
    it is restored after each test."""
    L = _lib()
    mode, _, epi = request.param.partition("-")
    L.set_option("YB_CONV_MODE", "2cta" if mode == "mc" else mode)
    L.set_option("YB_CONV_MC", "1" if mode == "mc" else "0")
    L.set_option("YB_CONV_EPI", "reg" if epi == "reg" else None)
    L.set_option("YB_CONV_EG", epi[2:] if epi.startswith("eg") else None)
    L.set_option("YB_CONV_PP", {"1cta-eg2": "0", "1cta-pp": "1"}.get(request.param))
    L.set_option("YB_CONV_CTAS", "2" if request.param == "2cta-eg2" else None)
    yield request.param
    for k in ("YB_CONV_MODE", "YB_CONV_MC", "YB_CONV_EPI", "YB_CONV_EG", "YB_CONV_PP", "YB_CONV_CTAS"):
        L.set_option(k, None)


def _lib():
    from yolov3_tensorflow_b200 import _lib
    return _lib


def _run_conv(n, h, w, cin, cout, k, s, dtype=torch.float16, in_extra=0, out_extra=0, residual=False, upsample=False,
              out_fp32=False, leaky=True, stats=False, seed=0):
    L = _lib()
    lib, check, ptr, st = L.lib, L.check, L.ptr, L.stream_handle
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(seed)
    in_ld = cin + in_extra
    xfull = (torch.randn((n, h, w, in_ld), generator=g) * 1.0).to(dtype).to(dev)
    in_off = in_extra // 2 // 8 * 8
    x = xfull[..., in_off:in_off + cin]
    wt = (torch.randn((cout, k, k, cin), generator=g) / (k * (cin ** 0.5))).to(dev)      # OHWI fp32
    scale = (torch.rand(cout, generator=g) + 0.5).to(dev)
    shift = (torch.randn(cout, generator=g) * 0.1).to(dev)
    cout_pad = lib.yb_conv_cout_pad(cout)
    wp = torch.zeros((cout_pad, k, k, cin), dtype=dtype, device=dev)
    code = L.YB_F16 if dtype == torch.float16 else L.YB_BF16
    check(lib.yb_pack_conv_weights(ptr(wt), L.YB_W_OHWI, cout, cin, k, cout_pad, code, ptr(wp), st()), "pack")
    sc = torch.ones(cout_pad, device=dev); sc[:cout] = scale
    sh = torch.zeros(cout_pad, device=dev); sh[:cout] = shift
    ho, wo = h // s, w // s
    up = 2 if upsample else 1
    out_ld = cout + out_extra
    out_off = out_extra // 2 // 8 * 8 if not out_fp32 else 0
    odt = torch.float32 if out_fp32 else dtype
    outfull = torch.full((n, ho * up, wo * up, out_ld), -7.0, dtype=odt, device=dev)
    res = None
    if residual:
        res = (torch.randn((n, ho, wo, cout), generator=g)).to(dtype).to(dev)
    d = L.ConvDesc(n=n, h=h, w=w, cin=cin, cout=cout, ksize=k, stride=s, in_ld=in_ld, out_ld=out_ld,
                   res_ld=cout, dtype=code, out_fp32=int(out_fp32), leaky=int(leaky), upsample2x=int(upsample))
    esz = 4 if out_fp32 else 2
    ssum = torch.zeros(cout_pad, device=dev) if stats else None
    ssq = torch.zeros(cout_pad, device=dev) if stats else None
    xp = C.c_void_p(xfull.data_ptr() + in_off * 2)
    op = C.c_void_p(outfull.data_ptr() + out_off * esz)
    check(lib.yb_conv2d_fwd(C.byref(d), xp, ptr(wp), ptr(sc), ptr(sh), ptr(res), op, ptr(ssum), ptr(ssq), st()), "conv")
    torch.cuda.synchronize()
    # ---- reference (fp32 math on the rounded operands) ----
    xr = x.float().permute(0, 3, 1, 2)
    wr = wp[:cout].float().permute(0, 3, 1, 2)
    raw = F.conv2d(xr, wr, None, stride=s, padding=k // 2)
    y = raw * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    if leaky:
        y = torch.where(y > 0, y, 0.1 * y)
    if residual:
        y = y + res.float().permute(0, 3, 1, 2)
    if upsample:
        y = y.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    ref = y.permute(0, 2, 3, 1).contiguous()
    got = outfull[..., out_off:out_off + cout].float()
    eps = 2.0 ** -9 if dtype == torch.float16 else 2.0 ** -6
    if out_fp32:
        eps = 1e-4
    err = (got - ref).abs()
    tol = eps * torch.clamp(ref.abs(), min=1.0)
    bad = err > tol
    if bad.any():
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(
            f"conv mismatch n={n} h={h} w={w} cin={cin} cout={cout} k={k} s={s}: {int(bad.sum())}/{bad.numel()} bad, "
            f"max err {float(err.max()):.4g}, first bad at {idx}: got {float(got[tuple(idx)]):.5g} ref {float(ref[tuple(idx)]):.5g}; "
            f"got[0,0,0,:4]={got[0,0,0,:4].tolist()} ref[0,0,0,:4]={ref[0,0,0,:4].tolist()}")
    # untouched padding channels of a wider output buffer
    if out_extra and not out_fp32:
        mask = torch.ones(out_ld, dtype=torch.bool, device=dev); mask[out_off:out_off + cout] = False
        assert torch.all(outfull[..., mask] == -7.0), "conv wrote outside its channel slice"
    if stats:
        s_ref = raw.sum(dim=(0, 2, 3)); q_ref = (raw * raw).sum(dim=(0, 2, 3))
        torch.testing.assert_close(ssum[:cout], s_ref, rtol=2e-3, atol=2e-2 * float(raw.abs().max()))
        torch.testing.assert_close(ssq[:cout], q_ref, rtol=2e-3, atol=1e-2)
    return float(err.max())


def test_conv1x1_gemm_basic():
    _run_conv(2, 16, 16, 64, 128, 1, 1)          # M = 512: 4 full tiles, BN=128, BK=64


def test_conv1x1_tail_rows_and_bn64():
    _run_conv(3, 13, 13, 128, 64, 1, 1)          # M = 507: tail tile, BN=64


def test_conv1x1_bk32():
    _run_conv(2, 13, 13, 32, 64, 1, 1)           # cin = 32 -> 64B swizzle path


def test_conv1x1_long_k_multi_ntile():
    _run_conv(2, 13, 13, 1024, 512, 1, 1)        # 16 k-blocks (> pipeline depth), 4 n-tiles


def test_conv1x1_slices_residual():
    _run_conv(2, 26, 26, 256, 128, 1, 1, in_extra=128, out_extra=64, residual=True)


def test_conv1x1_head_fp32_255():
    _run_conv(2, 13, 13, 256, 255, 1, 1, out_fp32=True, leaky=False)


def test_conv1x1_upsample_into_concat():
    _run_conv(2, 13, 13, 128, 64, 1, 1, upsample=True, out_extra=128)


def test_conv3x3_s1_im2col():
    _run_conv(2, 16, 16, 64, 128, 3, 1)


def test_conv3x3_s1_odd_size_crossing_images():
    _run_conv(3, 13, 13, 64, 128, 3, 1, residual=True)   # 169 px/img: tiles straddle rows and images


def test_conv3x3_s1_bk32():
    _run_conv(2, 20, 12, 32, 64, 3, 1)            # non-square, cin=32


def test_conv3x3_s2():
    _run_conv(2, 52, 52, 64, 128, 3, 2)           # darknet pad-1 + stride 2 -> 26x26


def test_conv3x3_s2_nonsquare_bk32():
    _run_conv(1, 64, 96, 32, 64, 3, 2)


def test_conv3x3_input_slice_of_concat():
    _run_conv(2, 26, 26, 128, 256, 3, 1, in_extra=256)


def test_conv3x3_bf16_and_stats():
    _run_conv(2, 26, 26, 128, 128, 3, 1, dtype=torch.bfloat16, stats=True)


def test_conv3x3_tiny_tensor_under_128k():
    _run_conv(1, 4, 4, 64, 64, 3, 1)              # exercises the small-tensor im2col descriptor workaround


def test_conv3x3_wide_odd_mtiles_residual():
    _run_conv(3, 16, 16, 128, 512, 3, 1, residual=True)      # M=768: 3 m-tiles (odd: a pair of the 2x2 cluster idles), 2 n-tiles


def test_conv3x3_s2_wide():
    _run_conv(2, 52, 52, 128, 256, 3, 2)                     # 1 n-tile -> 2x1 cluster (B multicast only)


def test_conv1x1_wide_1024_bf16_stats():
    _run_conv(4, 13, 13, 512, 1024, 1, 1, dtype=torch.bfloat16, stats=True)   # 4 n-tiles, statistics epilogue


def test_conv1x1_residual_tail_rows_many_chunks():
    _run_conv(3, 13, 13, 128, 256, 1, 1, residual=True, out_extra=64)   # 507 rows: tail tile; 8 chunks/tile + TMA residual


def test_conv3x3_many_tiles_per_cta_residual():
    _run_conv(8, 52, 52, 64, 128, 3, 1, residual=True)                  # 169 m-tiles on <= 132 CTAs: persistent CTAs take several tiles


def test_conv1x1_cout32_single_chunk():
    _run_conv(2, 26, 26, 64, 32, 1, 1, residual=True)                   # cout 32: one valid chunk of a 64-wide tile


def test_conv_rejects_bad_arguments():
    L = _lib()
    d = L.ConvDesc(n=1, h=8, w=8, cin=24, cout=64, ksize=3, stride=1, in_ld=24, out_ld=64, res_ld=0, dtype=0,
                   out_fp32=0, leaky=1, upsample2x=0)
    t = torch.zeros(1 << 16, device="cuda")
    rc = L.lib.yb_conv2d_fwd(C.byref(d), L.ptr(t), L.ptr(t), L.ptr(t), L.ptr(t), None, L.ptr(t), None, None, L.stream_handle())
    assert rc == -1 and b"cin" in L.lib.yb_last_error_string()
    with pytest.raises(ValueError):
        L.check(rc, "conv")


def test_pack_weights_layouts():
    L = _lib()
    g = torch.Generator().manual_seed(1)
    cout, cin, k = 48, 32, 3
    ohwi = torch.randn((cout, k, k, cin), generator=g).cuda()
    hwio = ohwi.permute(1, 2, 3, 0).contiguous()
    oihw = ohwi.permute(0, 3, 1, 2).contiguous()
    for src, lay in ((hwio, L.YB_W_HWIO), (oihw, L.YB_W_OIHW), (ohwi, L.YB_W_OHWI)):
        dst = torch.full((64, k, k, cin), 9.0, dtype=torch.float16, device="cuda")
        L.check(L.lib.yb_pack_conv_weights(L.ptr(src), lay, cout, cin, k, 64, L.YB_F16, L.ptr(dst), L.stream_handle()), "pack")
        assert torch.equal(dst[:cout], ohwi.half())
        assert torch.all(dst[cout:] == 0)
