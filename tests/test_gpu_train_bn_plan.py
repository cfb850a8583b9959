"""Every batch-norm launch of a training step, on the plan's own tensors, against float64 and exactly emulated float32
(tests/bn_ref.py).

tests/test_gpu_bn_train.py runs the BN kernels on operands it builds; this file checks the launches train_fwd_layer and
train_bwd_layer make inside a bound plan (csrc/net_train.cu): which buffers they read and write, the row count the
statistics divide by, the decay, the residual source, the 2x-upsampled and concat-slice stores, and where dgamma /
dbeta go.  A model runs two training steps: step 1 updates the weights and the moving statistics (lr > 0), step 2
(lr 0) is checked, so a value left over from step 1 is a wrong value.  The topology (residual source out(b - 2),
concat slices, upsampling layers) comes from train_plan_ref.Topology, not from the plan.

For every BN layer, after step 2:
  - coefficients: from the forward sums [Σz | Σz²] and count = replicas * n * h * w, bn_ref.batch_coeffs gives the
    saved mean, scale and shift bit for bit, given the saved invstd, which must lie within RSQRT_ULP of
    1 / sqrt(fl32(var + eps)); the moving statistics equal bn_ref.moving_update of the ones before the step bit for bit.
    Frozen BN: mean is the moving mean, scale = fl(gamma * invstd), shift within 1 ulp_32, moving statistics unchanged;
  - activation store: the layer output against bn_ref.apply_ref(z, scale, shift, res) (bit for bit except one ulp_T
    where the fma emulation was inexact), res = out(b - 2) for a residual layer b; all four copies of an upsampled
    store bit-identical; route layers in their concat slice, whose ld and offset must be the topology's;
  - dgamma / dbeta: from the plan's dA (summed over the 4 copies for upsampling layers), z and the saved coefficients,
    within bn_ref.reduce_bound for the launch shape yb_bn_schedule reports; on the layered path the backward exchange
    slab equals the flat gradient bit for bit (x2 for two ranks);
  - dz: bn_ref.bwd_apply_ref with the sums the kernel read (the exchange slab on the layered path, the flat gradient on
    the fused one, zeros when frozen) and the same count, within its bound; dilated stride-2 dz has zero gaps.
Detection heads: the bias gradient against the float64 column sum of the head's dz within train_bn_plan_ref's
col_stats_bound (the summation depth of yb_col_sum, and the subnormals its atomic adds flush).

The fused path is checked after the step.  That relies on every layer's z, activation, dA and dz being its own buffer,
not rewritten later in the step; every layered step asserts it, by fingerprinting each buffer right after the phase
that writes it and again after the step.

Each configuration prints one "BNPLAN <config> <check>: worst err/bound ... at layer ..." line per check, its peak
CUDA memory and its wall time."""
import ctypes as C
import gc
import time

import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests import bn_ref as B
from tests import conv_ref as R
from tests import train_bn_plan_ref as BP
from tests import train_plan_ref as T
from tests import wgrad_ref as W
from tests.test_gpu_path import _train_case

pytestmark = pytest.mark.gpu
LR = 1e-2
DECAY = 0.99
CHUNK = 1 << 23                   # float64 reference elements per image group


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    BP.set_options(_lib, {})
    yield _lib
    BP.set_options(_lib, {})


def _sms(L):
    s = C.c_int()
    L.check(L.lib.yb_device_info(C.byref(s), None, None), "device_info")
    return s.value


def _bits32(t):
    return t.contiguous().view(torch.int32)


def _fingerprint(t):
    """Sum of the 16-bit patterns of a strided [n, h, w, c] view, one image at a time."""
    return sum(int(t[j].reshape(-1).view(torch.int16).sum(dtype=torch.int64)) for j in range(t.shape[0]))


def _chunks(n, per_image):
    k = max(1, CHUNK // per_image)
    for i0 in range(0, n, k):
        yield i0, min(n, i0 + k)


class Worst:
    def __init__(self, cid):
        self.cid, self.v = cid, {}

    def add(self, kind, layer, frac):
        if kind not in self.v or frac > self.v[kind][0]:
            self.v[kind] = (frac, layer)

    def report(self):
        for kind, (frac, layer) in self.v.items():
            print(f"BNPLAN {self.cid} {kind}: worst err/bound {frac:.3f} at layer {layer}")


class BnPlanRun:
    def __init__(self, L, cid, opts, mode, dt, n, hw):
        self.L, self.cid, self.mode, self.n = L, cid, mode, n
        self.topo = T.Topology()
        BP.set_options(L, opts)
        import yolov3_tensorflow_b200 as pkg
        params, x, ys = _train_case(seed=43, n=n, h=hw[0], w=hw[1])
        self.m = pkg.yolov3(80, O.COCO_ANCHORS, use_label_smooth=True, use_focal_loss=True, batch_norm_decay=DECAY,
                            dtype=dt)
        self.m.set_params(params, "HWIO")
        self.x = torch.from_numpy(x).cuda()
        self.ys = [torch.from_numpy(y).cuda() for y in ys]
        self.dtype = self.m._torch_dtype
        self.replicas = 2 if mode == "replicas" else 1
        self.flags = L.YB_TRAIN_BN_FROZEN if mode == "frozen" else 0
        self.worst = Worst(cid)

    # ------------------------------------------------------------------------------------------------ the steps
    def _buffers(self, i, backward):
        plan = self.plan
        if backward:
            return [plan.train_buffer(i, "dz")] + ([plan.train_buffer(i, "dA")] if plan.layer_info(i).has_bn else [])
        return [plan.train_buffer(i, "z"), plan.layer_output(i)] if plan.layer_info(i).has_bn else []

    def step(self, lr, fused=False, flags=0, replicas=1):
        L, m = self.L, self.m
        x, ys, plan, opt, _ = m._train_setup(self.x, self.ys, lr, 0.9, 100.0, "momentum", 0.9, 0.9, 0.999, None, False)
        self.plan = plan
        h, st, px = plan.handle, L.stream_handle(), L.ptr(x)
        nl = plan.num_layers
        has_bn = [bool(plan.layer_info(i).has_bn) for i in range(nl)]
        anchors = L.fptr(m.anchors.reshape(-1))
        if fused:
            L.check(L.lib.yb_net_train_fwd_bwd(h, px, L.ptr(ys[0]), L.ptr(ys[1]), L.ptr(ys[2]), anchors,
                                               int(m.use_label_smooth), int(m.use_focal_loss), float(m.batch_norm_decay),
                                               float(m.loss_scale), None, None, None, L.ptr(plan.loss4), flags, st),
                    "train_fwd_bwd")
        else:
            prints = {}
            for i in range(nl):
                L.check(L.lib.yb_net_train_forward_layer(h, px, i, L.YB_PHASE_LOCAL, replicas, float(m.batch_norm_decay),
                                                         None, None, None, flags, st), "forward LOCAL")
                if replicas > 1 and has_bn[i]:
                    plan.bn_exchange_buffer(i, False).mul_(replicas)     # the all-reduce of identical ranks
                L.check(L.lib.yb_net_train_forward_layer(h, px, i, L.YB_PHASE_GLOBAL, replicas, float(m.batch_norm_decay),
                                                         None, None, None, flags, st), "forward GLOBAL")
                prints[(i, 0)] = [_fingerprint(t) for t in self._buffers(i, False)]
            L.check(L.lib.yb_net_train_loss(h, L.ptr(ys[0]), L.ptr(ys[1]), L.ptr(ys[2]), anchors, int(m.use_label_smooth),
                                            int(m.use_focal_loss), float(m.loss_scale), L.ptr(plan.loss4), st),
                    "train_loss")
            for i in range(nl - 1, -1, -1):
                L.check(L.lib.yb_net_train_backward_layer(h, px, i, L.YB_PHASE_LOCAL, replicas, flags, st), "backward LOCAL")
                if replicas > 1 and has_bn[i]:
                    plan.bn_exchange_buffer(i, True).mul_(replicas)
                L.check(L.lib.yb_net_train_backward_layer(h, px, i, L.YB_PHASE_GLOBAL, replicas, flags, st),
                        "backward GLOBAL")
                prints[(i, 1)] = [_fingerprint(t) for t in self._buffers(i, True)]
            L.check(L.lib.yb_net_train_join(h, st), "train_join")
            # the premise of checking after the step: nothing a phase wrote is rewritten later in the step
            for (i, bwd), fp in prints.items():
                assert [_fingerprint(t) for t in self._buffers(i, bwd)] == fp, \
                    f"{self.cid}: layer {i}'s {'dz / dA' if bwd else 'z / activation'} changed later in the step"
        if lr:
            m._finish_step(plan, opt, 1.0 / float(m.loss_scale), [None] * 3, False)
        torch.cuda.synchronize()

    # ------------------------------------------------------------------------------------------------ premises
    def check_premise(self, scheds):
        plan, L, cid = self.plan, self.L, self.cid
        if cid.startswith("bench"):
            assert self.dtype == torch.bfloat16 and plan.n == 32
        if cid == "fp16":
            assert self.dtype == torch.float16 and float(self.m.loss_scale) == 1024.0
        if cid in ("fin0", "frozen+fin0"):
            assert L.get_option("YB_BN_FIN")[:1] == "0"
        if cid == "cpt4":
            assert all(s.cpt == 4 for s in scheds.values())
        if cid == "dilated":
            s2 = [i for i in range(plan.num_layers) if plan.layer_info(i).stride == 2]
            assert s2 and all(plan.train_buffer(i, "dz").shape[1] == plan.layer_info(i).in_h for i in s2)
        if cid == "stem-cuda":
            assert L.get_option("YB_STEM_TRAIN")[:1] == "c"
        if cid == "rect":
            assert plan.h != plan.w

    def check_wiring(self):
        """Route and upsampling layers store where the topology says: the concat buffer of the layer reading them, at
        channel offset out_off and row pitch out_ld; every BN layer's dA mirrors its output."""
        plan, topo = self.plan, self.topo
        for cat, (up, route) in topo.concat.items():
            xin = plan.train_buffer(cat, "in")
            for j in (up, route):
                o, dA = plan.layer_output(j), plan.train_buffer(j, "dA")
                assert o.stride(2) == dA.stride(2) == topo.out_ld[j], (j, o.stride(), topo.out_ld[j])
                assert o.data_ptr() - xin.data_ptr() == 2 * topo.out_off[j], f"layer {j}: not at its concat offset"
        for i in range(plan.num_layers):
            if plan.layer_info(i).has_bn:
                o, dA = plan.layer_output(i), plan.train_buffer(i, "dA")
                assert o.shape == dA.shape and o.stride() == dA.stride(), i

    # ------------------------------------------------------------------------------------------------ checks
    def check_bn_layer(self, i, mm0, mv0, sched):
        plan, topo, dt, n = self.plan, self.topo, self.dtype, self.n
        info = plan.layer_info(i)
        c, oh, ow = info.cout, info.out_h, info.out_w
        rows = n * oh * ow
        count = self.replicas * rows
        name = f"{self.cid} layer {i}"
        frozen = self.mode == "frozen"
        p = plan.conv_params(i)
        ga, be = p["gamma"].clone(), p["beta"].clone()
        sv = {k: v.clone() for k, v in plan.bn_batch_stats(i).items()}
        mu, inv, sc, sh = sv["mean"], sv["invstd"], sv["scale"], sv["shift"]
        # ---- coefficients
        cpu = lambda t: t.cpu()   # noqa: E731  (float32 emulation on the host, as tests/test_gpu_bn_train.py does)
        if frozen:
            assert torch.equal(_bits32(mu), _bits32(mm0)), f"{name}: frozen mean is not the moving mean"
            err = B.invstd_error(cpu(mv0), BP.EPS, cpu(inv))
            assert err <= B.RSQRT_ULP, f"{name}: frozen invstd {err} ulp"
            assert torch.equal(cpu(sc), cpu(ga) * cpu(inv)), f"{name}: frozen scale"
            d = (cpu(sh).double() - (cpu(be).double() - cpu(mm0).double() * cpu(sc).double())).abs()
            assert bool((d <= B.ulp32(cpu(sh))).all()), f"{name}: frozen shift beyond 1 ulp"
            assert torch.equal(_bits32(p["mean"]), _bits32(mm0)) and torch.equal(_bits32(p["var"]), _bits32(mv0)), \
                f"{name}: frozen BN moved the moving statistics"
            self.worst.add("invstd ulp", i, err / B.RSQRT_ULP)
        else:
            slab = plan.bn_exchange_buffer(i, False)
            cp = slab.numel() // 2
            su, sq = cpu(slab[:c]), cpu(slab[cp:cp + c])
            mean, var, esc, esh = B.batch_coeffs(su, sq, count, cpu(ga), cpu(be), BP.EPS, cpu(inv))
            err = B.invstd_error(var, BP.EPS, cpu(inv))
            assert err <= B.RSQRT_ULP, f"{name}: invstd {err} ulp from 1 / sqrt(var + eps)"
            self.worst.add("invstd ulp", i, err / B.RSQRT_ULP)
            for got, want, what in ((mu, mean, "mean"), (sc, esc, "scale"), (sh, esh, "shift")):
                bad = int((_bits32(cpu(got)) != _bits32(want)).sum())
                assert bad == 0, f"{name}: {bad}/{c} saved {what} differ from batch_coeffs of the forward sums"
            emm, emv = B.moving_update(cpu(mm0), cpu(mv0), mean, var, count, DECAY)
            for got, want, what in ((p["mean"], emm, "moving mean"), (p["var"], emv, "moving var")):
                bad = int((_bits32(cpu(got)) != _bits32(want)).sum())
                assert bad == 0, f"{name}: {bad}/{c} {what} differ from moving_update"
        # ---- the sums dz read
        g = plan.layer_grads(i)
        xs = plan.bn_exchange_buffer(i, True)
        cp = xs.numel() // 2
        xg, xb = xs[:c].clone(), xs[cp:cp + c].clone()
        if self.mode == "fused":
            used = (g["gamma"].clone(), g["beta"].clone())
            # premise: the slab still holds step 1's sums, so a dz that read it would fail
            assert not torch.equal(_bits32(xg), _bits32(g["gamma"])), f"{name}: the backward slab is not stale"
        else:
            for got, flat, what in ((xg, g["gamma"], "dgamma"), (xb, g["beta"], "dbeta")):
                assert torch.equal(_bits32(got), _bits32(flat * self.replicas)), \
                    f"{name}: the backward exchange slab's {what} differs from the flat gradient's"
            used = (xg, xb)
        if frozen:
            used = (torch.zeros_like(xg), torch.zeros_like(xb))
        # ---- per image group: activation store, reduce sums, dz
        z4 = plan.train_buffer(i, "z")
        out4 = plan.layer_output(i)
        dA4 = plan.train_buffer(i, "dA")
        dz4 = plan.train_buffer(i, "dz")
        dilated = dz4.shape[1] != oh
        res4 = plan.layer_output(i - 2) if i in topo.residual else None
        if res4 is not None:
            assert res4.shape == z4.shape, f"{name}: out({i - 2}) is not the shape of the residual"
        up = i in topo.upsample
        assert bool(info.upsample2x) == up
        soft, parts, wz = 0, [], 0.0
        for i0, i1 in _chunks(n, oh * ow * c):
            zr = z4[i0:i1].reshape(-1, c)
            rr = None if res4 is None else res4[i0:i1].reshape(-1, c)
            want, inexact = B.apply_ref(zr, sc, sh, rr, True, dt)
            o = out4[i0:i1]
            copies = [o[:, a::2, b::2] for a in (0, 1) for b in (0, 1)] if up else [o]
            soft += B.check_apply(copies[0].reshape(-1, c), want, inexact, dt, f"{name} activation")
            for k, cpy in enumerate(copies[1:], 1):
                assert torch.equal(cpy.contiguous().view(torch.int16), copies[0].contiguous().view(torch.int16)), \
                    f"{name}: upsampled copy {k} differs from copy 0"
            dv = B.upsampled_rows(dA4[i0:i1]) if up else dA4[i0:i1].float()
            da = B.dact(dv.reshape(-1, c), zr, sc, sh, True)
            parts.append(B.reduce_sums(da, zr, mu, inv))
            ref, bound = B.bwd_apply_ref(da, zr, ga, inv, mu, used[0], used[1], count, dt)
            d = dz4[i0:i1]
            if dilated:
                gap = torch.ones(d.shape[1:3], dtype=torch.bool, device="cuda")
                gap[::2, ::2] = False
                assert bool((d[:, gap] == 0).all()), f"{name}: nonzero values in the gaps of the dilated dz"
                d = W.compact_dilated(d)
            wz = max(wz, R.check_out(d.reshape(-1, c), ref, bound, f"{name} dz"))
            del want, inexact, dv, da, ref, bound
        self.soft += soft
        self.worst.add("dz", i, wz)
        dg_ref, db_ref, G, A = B.reduce_ref(parts, mu, inv)
        bg, bb = B.reduce_bound(G, A, mu, inv, sched.rows_per_block, sched.lanes, sched.grid)
        self.worst.add("dgamma", i, R.check_out(g["gamma"], dg_ref, bg, f"{name} dgamma"))
        self.worst.add("dbeta", i, R.check_out(g["beta"], db_ref, bb, f"{name} dbeta"))

    def check_head(self, i, sms):
        plan = self.plan
        info = plan.layer_info(i)
        c = info.cout
        dz = plan.train_buffer(i, "dz")
        assert dz.stride(2) == 256 and c == 255
        rows = self.n * info.out_h * info.out_w
        ref = torch.zeros(c, dtype=torch.float64, device="cuda")
        A = torch.zeros_like(ref)
        for i0, i1 in _chunks(self.n, info.out_h * info.out_w * c):
            d = dz[i0:i1].reshape(-1, c).double()
            ref += d.sum(0)
            A += d.abs().sum(0)
        bound = BP.col_stats_bound(A, rows, c, sms)
        self.worst.add("head bias grad", i, R.check_out(plan.layer_grads(i)["b"], ref, bound,
                                                        f"{self.cid} layer {i} bias gradient"))

    def check_stem_sums(self, sms):
        """YB_STEM_TRAIN=cuda: layer 0's [Σz | Σz²] are yb_col_stats of the stored z."""
        plan = self.plan
        c = plan.layer_info(0).cout
        z = plan.train_buffer(0, "z")
        s1 = torch.zeros(c, dtype=torch.float64, device="cuda")
        s2, a1 = torch.zeros_like(s1), torch.zeros_like(s1)
        for i0, i1 in _chunks(self.n, plan.h * plan.w * c):
            d = z[i0:i1].reshape(-1, c).double()
            s1 += d.sum(0); s2 += (d * d).sum(0); a1 += d.abs().sum(0)
        rows = self.n * plan.h * plan.w
        slab = plan.bn_exchange_buffer(0, False)
        cp = slab.numel() // 2
        self.worst.add("stem sum z", 0, R.check_out(slab[:c], s1, BP.col_stats_bound(a1, rows, c, sms),
                                                    f"{self.cid} layer 0 sum z"))
        self.worst.add("stem sum z^2", 0, R.check_out(slab[cp:cp + c], s2, BP.col_stats_bound(s2, rows, c, sms),
                                                      f"{self.cid} layer 0 sum z^2"))


@pytest.mark.parametrize("cid,opts,mode,dt,n,hw", BP.CONFIGS, ids=[c[0] for c in BP.CONFIGS])
def test_train_bn_launches_against_float64(L, cid, opts, mode, dt, n, hw):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    run = BnPlanRun(L, cid, opts, mode, dt, n, hw)
    plan = run.m._plan(n, hw[0], hw[1], training=True)
    sms = _sms(L)
    infos = [plan.layer_info(i) for i in range(plan.num_layers)]
    BP.premise(L, cid, opts, infos, n)                      # at 132 SMs, as tests/test_train_bn_plan_host.py
    scheds = BP.schedules(L, infos, n, sms)                 # the launch shapes on this device, for the bounds
    if sms != BP.SMS:
        print(f"BNPLAN {cid}: {sms} SMs: the launch shapes differ from the {BP.SMS}-SM ones the table was chosen for")
    run.step(LR)                                            # step 1: weights and moving statistics move
    bn = [i for i in range(plan.num_layers) if infos[i].has_bn]
    mm0 = {i: plan.conv_params(i)["mean"].clone() for i in bn}
    mv0 = {i: plan.conv_params(i)["var"].clone() for i in bn}
    run.step(0.0, fused=mode == "fused", flags=run.flags, replicas=run.replicas)   # step 2: checked
    run.check_premise(scheds)
    run.check_wiring()
    if mode == "frozen":
        # premise: the batch statistics differ from the moving ones, so normalising with the wrong pair fails
        slab = plan.bn_exchange_buffer(0, False)
        c0 = infos[0].cout
        assert not torch.equal(slab[:c0] / (n * hw[0] * hw[1]), mm0[0]), f"{cid}: batch mean equals the moving mean"
    run.soft = 0
    for i in bn:
        run.check_bn_layer(i, mm0[i], mv0[i], scheds[i])
    for i in run.topo.heads:
        run.check_head(i, sms)
    if opts.get("YB_STEM_TRAIN"):
        run.check_stem_sums(sms)
    run.worst.report()
    assert np.isfinite(float(plan.loss4.sum()))
    print(f"BNPLAN {cid}: {run.dtype} n {n} {hw[0]} x {hw[1]}, {run.soft} one-ulp stores at inexact fma, peak CUDA "
          f"memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB, {time.time() - t0:.1f} s")
    del run, plan
    gc.collect()
    torch.cuda.empty_cache()
