"""Every conv launch of a training step, on the plan's own tensors, against float64 (tests/train_plan_ref.py).

The standalone conv tests build their own operands and call yb_conv2d_fwd / yb_conv2d_dgrad_s2 / yb_conv2d_wgrad.  This
file checks the launches train_bind prepares: their requests, tensor maps, pointers and leading dimensions, and the
residual bookkeeping that routes each layer's input gradient.  A model runs two training steps through the layered
entry points: step 1 updates the weights (momentum), step 2 is checked, so the per-step zeroing of the BN sums and the
flat gradient and the refresh of the 16-bit weights after an update are part of what is checked.

  - weights (after step 1's update): every layer's 16-bit forward weights are RN16 of the fp32 masters bit for bit,
    padding rows zero; the stride-1 dgrad weights are the flip + transpose of RN16(master) bit for bit;
  - forward: each BN layer's raw z and batch sums [Σz | Σz²] against conv_ref.conv_raw of its own input view (concat
    slices included) and RN16(master), within conv_ref.out_bound / stats_bound; the heads' fp32 maps as conv + bias;
    the split-precision stem's z against the float64 conv of the image and its float32 masters, and its sums against
    float64 sums of the stored z (tests/direct_ref.py);
  - input gradient, checked right after each layer's backward GLOBAL phase: dX = conv_transpose(dz, RN16(master)) + R
    within out_bound, where R is dA(out_b) for the layer before a residual layer b, the gradient already there for a
    second consumer, and 0 otherwise; every channel and row outside the layer's slice keeps its bits;
  - weight gradient: the flat dW of every layer against wgrad_ref within wgrad_bound (the stem: stem_tc_bound);
  - hygiene: the heads' dz pad column is zero; under YB_DGRAD_S2=dilated the gaps of the zero-inserted dz are zero.

Each configuration of train_plan_ref.CONFIGS gets a fresh model, with its options set before the plan is bound, and
asserts its premise through yb_conv_schedule.  One "PLAN" line per configuration and check prints the worst error as
a fraction of its bound and the layer where it occurs."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests import conv_ref as R
from tests import direct_ref as D
from tests import train_plan_ref as T
from tests import wgrad_ref as W
from tests.test_gpu_path import _train_case

pytestmark = pytest.mark.gpu
LR = 1e-2
STEM_TH, STEM_TW = 8, 16          # stem_wgrad_tc_kernel's output tile


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    T.set_options(_lib, {})
    yield _lib
    T.set_options(_lib, {})


def _sms(L):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    return s.value


def _bits(t):
    return t.contiguous().view(torch.int16)


class Worst:
    """Worst err / bound per check kind, with its layer."""

    def __init__(self, cid):
        self.cid, self.v = cid, {}

    def add(self, kind, layer, frac):
        if kind not in self.v or frac > self.v[kind][0]:
            self.v[kind] = (frac, layer)

    def report(self):
        for kind, (frac, layer) in self.v.items():
            print(f"PLAN {self.cid} {kind}: worst err/bound {frac:.3f} at layer {layer}")


def _conv64(x, w_ohwi, stride, pad):
    """conv_ref.conv_raw one image at a time (bounded float64 im2col) -> raw, S [M, cout]."""
    raws, Ss = [], []
    for i in range(x.shape[0]):
        r, s = R.conv_raw(x[i:i + 1], w_ohwi, stride, pad)
        raws.append(r)
        Ss.append(s)
    return torch.cat(raws), torch.cat(Ss)


def _dgrad64(dz, w16, stride, in_h, in_w):
    """float64 conv_transpose2d of the compact dz [n, ho, wo, cout] with w16 [cout, k, k, cin] (stride 2: padding 1,
    output_padding 1) -> raw, S [n * in_h * in_w, cin], as a stride-1 conv of the zero-inserted dz with the flipped,
    transposed weights."""
    n, ho, wo, cout = dz.shape
    k = w16.shape[1]
    if stride == 2:
        d = torch.zeros((n, in_h, in_w, cout), dtype=torch.float64, device=dz.device)
        d[:, ::2, ::2] = dz.double()
    else:
        d = dz.double()
    wf = w16.double().flip(1, 2).permute(3, 1, 2, 0).contiguous()     # [cin, k, k, cout]
    return _conv64(d, wf, 1, k // 2)


def _full_rows(plan, t, c_off):
    """The whole buffer rows [n, h, w, ld] around the strided view t whose first channel is c_off."""
    n, h, w, _ = t.shape
    ld = t.stride(2)
    return t.as_strided((n, h, w, ld), t.stride(), t.storage_offset() - c_off)


class PlanRun:
    def __init__(self, L, cid, opts, dt, n, hw):
        self.L, self.cid = L, cid
        self.topo = T.Topology()
        T.set_options(L, opts)
        import yolov3_tensorflow_b200 as pkg
        params, x, ys = _train_case(seed=41, n=n, h=hw[0], w=hw[1])
        self.m = pkg.yolov3(80, O.COCO_ANCHORS, use_label_smooth=True, use_focal_loss=True, batch_norm_decay=0.99,
                            dtype=dt)
        self.m.set_params(params, "HWIO")
        self.x = torch.from_numpy(x).cuda()
        self.ys = [torch.from_numpy(y).cuda() for y in ys]
        self.dtype = self.m._torch_dtype
        self.worst = Worst(cid)

    def setup(self, lr):
        return self.m._train_setup(self.x, self.ys, lr, 0.9, 100.0, "momentum", 0.9, 0.9, 0.999, None, False)

    def step(self, lr, check):
        """One layered training step; with check, the forward is checked before the loss and every dgrad's output right
        after its launch."""
        L, m = self.L, self.m
        x, ys, plan, opt, _ = self.setup(lr)
        self.plan, self.image = plan, x
        h, st, px = plan.handle, L.stream_handle(), L.ptr(x)
        nl = plan.num_layers
        for i in range(nl):
            for ph in (L.YB_PHASE_LOCAL, L.YB_PHASE_GLOBAL):
                L.check(L.lib.yb_net_train_forward_layer(h, px, i, ph, 1, float(m.batch_norm_decay), None, None, None, 0,
                                                         st), "train_forward_layer")
        if check:
            self.check_forward()
        L.check(L.lib.yb_net_train_loss(h, L.ptr(ys[0]), L.ptr(ys[1]), L.ptr(ys[2]), L.fptr(m.anchors.reshape(-1)),
                                        int(m.use_label_smooth), int(m.use_focal_loss), float(m.loss_scale),
                                        L.ptr(plan.loss4), st), "train_loss")
        for i in range(nl - 1, -1, -1):
            L.check(L.lib.yb_net_train_backward_layer(h, px, i, L.YB_PHASE_LOCAL, 1, 0, st), "backward LOCAL")
            snap = _full_rows(plan, plan.train_buffer(i, "dX"), self._dx_off(i)).clone() if check and i else None
            L.check(L.lib.yb_net_train_backward_layer(h, px, i, L.YB_PHASE_GLOBAL, 1, 0, st), "backward GLOBAL")
            if snap is not None:
                self.check_dgrad(i, snap)
        L.check(L.lib.yb_net_train_join(h, st), "train_join")
        if lr:
            m._finish_step(plan, opt, 1.0 / float(m.loss_scale), [None] * 3, False)
        torch.cuda.synchronize()

    def _dx_off(self, i):
        return self.topo.out_off[self.topo.producer(i)] if len(self.topo.inputs[i]) == 1 else 0

    # ------------------------------------------------------------------ routing table against the plan
    def check_wiring(self):
        plan, topo, L = self.plan, self.topo, self.L
        for i in range(1, plan.num_layers):
            info = plan.layer_info(i)
            s = L.LayerSchedule()
            L.check(L.lib.yb_net_layer_schedule(plan.handle, i, T.SMS, C.byref(s)), "layer_schedule")
            assert bool(s.residual) == (i in topo.residual), f"layer {i}: residual {s.residual}"
            assert bool(info.upsample2x) == (i in topo.upsample), f"layer {i}: upsample2x {info.upsample2x}"
            p = topo.producer(i)
            xin, dx = plan.train_buffer(i, "in"), plan.train_buffer(i, "dX")
            out, dA = plan.layer_output(p), plan.train_buffer(p, "dA")
            assert (xin.data_ptr(), xin.stride()) == (out.data_ptr(), out.stride()), f"layer {i}: input is not out_{p}"
            assert (dx.data_ptr(), dx.stride()) == (dA.data_ptr(), dA.stride()), f"layer {i}: dX is not dA(out_{p})"
            assert dx.shape[3] == info.cin

    # ------------------------------------------------------------------ weights
    def check_weights(self):
        plan = self.plan
        for i in range(1, plan.num_layers):
            info = plan.layer_info(i)
            w = plan.conv_params(i)["w"]
            q = w.to(self.dtype)
            w16 = plan.train_buffer(i, "w16")
            want = torch.zeros_like(w16)
            want[:info.cout] = q.reshape(info.cout, -1)
            bad = int((_bits(w16) != _bits(want)).sum())
            assert bad == 0, f"layer {i}: {bad} elements of the 16-bit forward weights differ from RN16(master)"
            if info.stride == 1 or self.dilated:
                k, kco = info.ksize, -(-info.cout // 32) * 32
                cin_pad = self.L.lib.yb_conv_cout_pad(info.cin)
                want = torch.zeros((cin_pad, k, k, kco), dtype=self.dtype, device="cuda")
                want[:info.cin, :, :, :info.cout] = q.flip(1, 2).permute(3, 1, 2, 0)
                got = plan.dgrad_weights(i)
                bad = int((_bits(got) != _bits(want.reshape(-1))).sum())
                assert bad == 0, f"layer {i}: {bad} elements of the dgrad weights differ from flip + transpose of RN16(master)"

    # ------------------------------------------------------------------ forward
    def check_stem_forward(self):
        """Layer 0, the split-precision stem: z against the float64 conv of the image and the float32 master weights
        within direct_ref.stem_split_bound, its [Σz | Σz²] against float64 sums of the stored z within sums_bound."""
        plan, dt = self.plan, self.dtype
        # the model of the split stem: YB_STEM_TRAIN=cuda runs the CUDA-core stem and yb_col_stats instead
        assert self.L.get_option("YB_STEM_TRAIN")[:1] != "c" and self.L.get_option("YB_STEM_SPLIT")[:1] != "0"
        info = plan.layer_info(0)
        wt = plan.conv_params(0)["w"]
        Aw = wt.double().abs().reshape(info.cout, -1).sum(1)
        z = plan.train_buffer(0, "z")
        zs = torch.zeros(info.cout, dtype=torch.float64, device="cuda")
        zq, za = torch.zeros_like(zs), torch.zeros_like(zs)
        worst = 0.0
        for j in range(plan.n):
            x = self.image[j:j + 1]
            raw, S = R.conv_raw(x, wt, 1, 1)
            zj = z[j].reshape(-1, info.cout)
            b = D.stem_split_bound(raw, S, D.stem_patch_abs(x), Aw, dt)
            worst = max(worst, R.check_out(zj, raw, b, f"{self.cid} layer 0 z image {j}"))
            zd = zj.double()
            zs += zd.sum(0); zq += (zd * zd).sum(0); za += zd.abs().sum(0)
            del raw, S, b
        self.worst.add("stem z", 0, worst)
        tiles = plan.n * -(-plan.h // STEM_TH) * -(-plan.w // STEM_TW)
        depth = D.sums_depth(tiles, _sms(self.L))
        slab = plan.bn_exchange_buffer(0, False)
        cp = slab.numel() // 2
        name = f"{self.cid} layer 0"
        fs = R.check_out(slab[:info.cout], zs, depth * D.U32 * za, name + " sum z")
        fq = R.check_out(slab[cp:cp + info.cout], zq, depth * D.U32 * zq, name + " sum z^2")
        self.worst.add("stem sum z", 0, fs)
        self.worst.add("stem sum z^2", 0, fq)
        print(f"PLAN {self.cid} layer 0: z worst err/bound {worst:.3f}, sum z {fs:.3f}, sum z^2 {fq:.3f} (depth {depth})")

    def check_forward(self):
        plan = self.plan
        self.check_stem_forward()
        for i in range(1, plan.num_layers):
            info = plan.layer_info(i)
            p = plan.conv_params(i)
            w16 = p["w"].to(self.dtype)
            xin = plan.train_buffer(i, "in")
            assert bool(torch.isfinite(xin).all()), f"layer {i}: its input, written by layer {self.topo.producer(i)}, is not finite"
            raw, S = _conv64(xin, w16, info.stride, info.ksize // 2)
            n16 = info.ksize * info.ksize * info.cin // 16
            if not info.has_bn:
                fm = plan.layer_output(i).reshape(-1, info.cout)
                ref = raw + p["b"].double()
                bound = R.out_bound(ref, S, n16, torch.float32, shift=p["b"])
                self.worst.add("head forward", i, R.check_out(fm, ref, bound, f"{self.cid} layer {i} head forward"))
                continue
            z = plan.train_buffer(i, "z").reshape(-1, info.cout)
            self.worst.add("z", i, R.check_out(z, raw, R.out_bound(raw, S, n16, self.dtype), f"{self.cid} layer {i} z"))
            (_, _, _, _, _, sinfo), = [r for r in self.scheds[i] if r[0] == "fwd"]
            depth = R.stats_depth(max(R.units_per_warpgroup(sinfo), 1) + 1, sinfo.grid)
            b_sum, b_sq = R.stats_bound(raw, S, n16, depth)
            slab = plan.bn_exchange_buffer(i, False)
            cp = slab.numel() // 2
            name = f"{self.cid} layer {i}"
            self.worst.add("sum z", i, R.check_out(slab[:info.cout], raw.sum(0), b_sum, name + " sum z"))
            self.worst.add("sum z^2", i, R.check_out(slab[cp:cp + info.cout], (raw * raw).sum(0), b_sq, name + " sum z^2"))
            del raw, S

    # ------------------------------------------------------------------ input gradient
    def _dz(self, i):
        info = self.plan.layer_info(i)
        dz = self.plan.train_buffer(i, "dz")
        if dz.shape[1] != info.out_h:
            dz = W.compact_dilated(dz)
        return dz

    def check_dgrad(self, i, snap):
        plan, topo = self.plan, self.topo
        info = plan.layer_info(i)
        name = f"{self.cid} layer {i} dX"
        kind, b = topo.route(i)
        kco = -(-info.cout // 32) * 32
        w16 = plan.conv_params(i)["w"].to(self.dtype)
        raw, S = _dgrad64(self._dz(i), w16, info.stride, info.in_h, info.in_w)
        off = self._dx_off(i)
        rows = info.in_h * info.in_w * plan.n
        res = None
        if kind == "pass":
            res = plan.train_buffer(b, "dA").reshape(rows, info.cin)
        elif kind == "inplace":
            res = snap[..., off:off + info.cin].reshape(rows, info.cin)
        ref = raw if res is None else raw + res.double()
        if info.stride == 2 and not self.dilated:
            a = (torch.arange(info.in_h, device="cuda") & 1).view(1, -1, 1, 1)
            c = (torch.arange(info.in_w, device="cuda") & 1).view(1, 1, -1, 1)
            n16 = ((1 + a) * (1 + c) * kco // 16).expand(plan.n, info.in_h, info.in_w, 1).reshape(-1, 1).double()
        else:
            n16 = info.ksize * info.ksize * kco // 16
        bound = R.out_bound(ref, S, n16, self.dtype, res=res)
        full = _full_rows(plan, plan.train_buffer(i, "dX"), off)
        got = full[..., off:off + info.cin].reshape(rows, info.cin)
        self.worst.add(f"dX {kind}", i, R.check_out(got, ref, bound, f"{name} ({kind})"))
        outside = torch.ones(full.shape[3], dtype=torch.bool, device="cuda")
        outside[off:off + info.cin] = False
        if bool(outside.any()):
            bad = int((_bits(full[..., outside]) != _bits(snap[..., outside])).sum())
            assert bad == 0, f"{name}: {bad} elements outside channels [{off}, {off + info.cin}) changed"

    # ------------------------------------------------------------------ weight gradient, hygiene
    def check_wgrad(self):
        plan, L = self.plan, self.L
        sms = _sms(L)
        code = L.YB_F16 if self.dtype == torch.float16 else L.YB_BF16
        for i in range(plan.num_layers):
            info = plan.layer_info(i)
            got = plan.layer_grads(i)["w"].reshape(info.cout, -1)
            dz = self._dz(i)[..., :info.cout]
            if i == 0:
                ref, S = W.wgrad_ref(self.x, dz, 3, 1)
                tiles = plan.n * -(-plan.h // STEM_TH) * -(-plan.w // STEM_TW)
                grid = min(tiles, 4 * sms)
                dz_abs = sum(dz[j].double().abs().sum((0, 1)) for j in range(plan.n))
                bound = W.stem_tc_bound(S, dz_abs, 0.0, self.dtype, -(-tiles // grid), grid)
            else:
                ref, S = W.wgrad_ref(plan.train_buffer(i, "in"), dz, info.ksize, info.stride)
                d = L.ConvDesc(n=plan.n, h=info.in_h, w=info.in_w, cin=info.cin, cout=info.cout, ksize=info.ksize,
                               stride=info.stride, in_ld=self.topo.in_ld(i), out_ld=info.cout, res_ld=0, dtype=code,
                               out_fp32=0, leaky=0, upsample2x=0)
                s = L.WgradSchedule()
                L.check(L.lib.yb_wgrad_schedule(C.byref(d), sms, C.byref(s)), "wgrad_schedule")
                bound = W.wgrad_bound(S, 0.0, s.kb_per_split, s.splits)
            self.worst.add("dW", i, R.check_out(got, ref, bound, f"{self.cid} layer {i} dW"))
            del ref, S

    def check_hygiene(self):
        plan = self.plan
        for i in self.topo.heads:
            dz = plan.train_buffer(i, "dz")
            pad = dz.as_strided(dz.shape[:3] + (dz.stride(2) - dz.shape[3],), dz.stride(),
                                dz.storage_offset() + dz.shape[3])
            assert bool((pad == 0).all()), f"layer {i}: the dz pad columns are not zero"
        if self.dilated:
            for i in range(1, plan.num_layers):
                info = plan.layer_info(i)
                if info.stride != 2:
                    continue
                dz = plan.train_buffer(i, "dz")
                assert dz.shape[1:3] == (info.in_h, info.in_w), f"layer {i}: dz is not at the input resolution"
                gap = torch.ones(dz.shape[1:3], dtype=torch.bool, device="cuda")
                gap[::2, ::2] = False
                assert bool((dz[:, gap] == 0).all()), f"layer {i}: nonzero values in the gaps of the dilated dz"


@pytest.mark.parametrize("cid,opts,dt,n,hw", T.CONFIGS, ids=[c[0] for c in T.CONFIGS])
def test_train_plan_launches_against_float64(L, cid, opts, dt, n, hw):
    torch.cuda.reset_peak_memory_stats()
    run = PlanRun(L, cid, opts, dt, n, hw)
    run.dilated = "YB_DGRAD_S2" in opts
    try:
        plan = run.m._plan(n, hw[0], hw[1], training=True)     # binds: a configuration without a kernel fails here
    except (ValueError, L.YoloB200Error) as e:
        if "no kernel" in str(e):
            pytest.skip(f"{cid}: rejected at bind: {e}")
        raise
    infos = [plan.layer_info(i) for i in range(plan.num_layers)]
    code = L.YB_F16 if run.dtype == torch.float16 else L.YB_BF16
    run.scheds = T.schedules(L, run.topo, infos, n, code, run.dilated, sms=_sms(L))
    T.premise(cid, T.schedules(L, run.topo, infos, n, code, run.dilated), run.topo)
    run.step(LR, check=False)          # step 1: momentum update, then the 16-bit weights are refreshed
    run.check_weights()
    run.check_wiring()
    run.step(0.0, check=True)          # step 2: checked (no update, so the masters are what it read)
    run.check_wgrad()
    run.check_hygiene()
    run.worst.report()
    print(f"PLAN {cid}: {run.dtype} n {n} {hw[0]} x {hw[1]}, peak CUDA memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    assert np.isfinite(float(plan.loss4.sum()))
