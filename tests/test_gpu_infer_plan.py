"""Every launch of the 16-bit inference plan, on the plan's own tensors, against float64 (tests/infer_plan_ref.py).

bench.py times this plan at batch 64, 416^2 through detect_raw.  Each configuration of infer_plan_ref.CONFIGS gets a
fresh model with its options set before the plan binds; the activation arena is filled with 0xFF bytes (NaN in fp16,
bf16 and fp32) and forward() runs once.  Then, on what that forward left in the arena:

  a. every layer's output against conv_ref.conv_raw of its own input view and RN16(master weights), then conv_ref.epilogue
     with the scale / shift yb_bn_fold makes from the plan's float32 masters, within conv_ref.out_bound (n16 = k k cin / 16).
     The input view comes from the topology (a concat consumer reads the whole [upsampled | route] buffer, a residual
     layer b adds out(b - 2)), so a wrong pointer or pitch fails here.  The fold itself is checked against float64;
  b. the stem: fused into Conv_1 (the default), its output is never stored.  Its value v0 is computed in float64 on
     RN16(image) and RN16(stem weights) (both kernels round their operands that way) with the error bound e0 of a K = 32
     mma.sync conv (2 k16 steps) and its epilogue.  The stored stem value lies in [RN16(v0 - e0), RN16(v0 + e0)]; Conv_1
     is checked on x* = RN16(v0) with |scale_1| conv(d, |w_1|) added to its bound, d the width of that interval.  With
     the stem as its own launch, layer 0's output is checked directly and Conv_1 reads it;
  c. the heads: the float32 maps forward() returns, as raw + bias within the float32 bound; the heads' arena buffers
     still hold the sentinel (forward writes through the caller's pointers);
  d. the four copies an upsampling conv stores are bit-identical, and no sentinel is left in any concat-buffer row;
  e. every arena byte outside the layer-output buffers (alignment gaps, the fused stem's buffer, the heads' buffers)
     still holds 0xFF;
  f. (bench, 608, rect) detect_raw on the same images: its boxes equal predict_scores(forward) bit for bit, its kept
     detections equal batched_nms_raw on those boxes and scores for every image (and O.gpu_nms for the first and last
     image), and it leaves the arena bit-identical to the forward's, also with YB_HEAD_STREAM=0.

One "PLAN" line per configuration and check kind prints the worst error as a fraction of its bound and where it occurs.
"""
import time

import numpy as np
import pytest
import torch

from oracle import yolov3_oracle as O
from tests import conv_ref as R
from tests import direct_ref as D
from tests import infer_plan_ref as P
from tests.synth import gen_inputs
from tests.test_gpu_path import _train_case

pytestmark = pytest.mark.gpu
CLASSES = 80
NMS = (200, 0.3, 0.45)             # max_boxes, score_thresh, nms_thresh: bench.py's
EPS32 = float(np.float32(1e-5))    # the plan's BN epsilon (1e-5f)
FOLD_ULPS = 3                      # yb_bn_fold: var + eps, sqrtf and the divide round once each (< 2.5 u relative)


@pytest.fixture
def L():
    from yolov3_tensorflow_b200 import _lib
    P.set_options(_lib, {})
    yield _lib
    P.set_options(_lib, {})


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _count(mask):
    """Number of True elements; the reduction to a count (int64) runs only when there is one."""
    return int(torch.count_nonzero(mask)) if bool(mask.any()) else 0


def ulp32(a):
    _, e = torch.frexp(a.abs())
    e = torch.where(a == 0, -126.0, torch.clamp(e.double() - 1, min=-126.0))
    return torch.exp2(e - 23)


def params_for(weights):
    if weights == "cfg1":
        return O.make_params(CLASSES, seed=7)
    return O.make_params(CLASSES, seed=7, random_bn=True, det_scale=8.0, conf_bias=-2.0)


class Worst:
    """Worst err / bound per check kind, with where it occurs."""

    def __init__(self, cid):
        self.cid, self.v = cid, {}

    def add(self, kind, where, frac):
        if kind not in self.v or frac > self.v[kind][0]:
            self.v[kind] = (frac, where)

    def report(self):
        for kind, (frac, where) in self.v.items():
            print(f"PLAN {self.cid} {kind}: worst err/bound {frac:.3f} at {where}")


class InferRun:
    """One checked forward of one plan of model m."""

    def __init__(self, L, m, cid, x, worst):
        self.L, self.m, self.cid, self.x, self.worst = L, m, cid, x, worst
        self.topo = P.Topology()
        self.dtype = m._torch_dtype
        n, h, w = x.shape[:3]
        self.plan = m._plan(n, h, w)           # the plan forward() runs: a training plan if the key has one
        self.n = n
        self.near_mid = 0.0
        self.scheds = P.layer_schedules(L, self.plan.handle)
        self.fused = self.scheds[0].kernel == L.YB_LAYER_FUSED_STEM

    # ------------------------------------------------------------------ arena layout
    def buffers(self):
        """[(start, end, written)] byte ranges of the layer-output buffers in the activation arena, sorted; written =
        False for the buffers forward() must leave alone (the fused stem's, the heads')."""
        plan, topo = self.plan, self.topo
        base = plan.act.data_ptr()
        out = {}
        for i in range(plan.num_layers):
            t = plan.layer_output(i)
            esz = t.element_size()
            start = t.data_ptr() - base - topo.out_off[i] * esz
            rows = t.shape[0] * t.shape[1] * t.shape[2]
            end = start + rows * t.stride(2) * esz
            written = not (i in topo.heads or (i == 0 and self.fused))
            prev = out.get(start)
            assert prev is None or prev[0] == end, f"layer {i}: buffer at {start} has two sizes"
            out[start] = (end, written or (prev is not None and prev[1]))
        return sorted((s, e, w) for s, (e, w) in out.items())

    def prefix_end(self):
        """End of the layer-output buffers (a training plan's scratch follows them)."""
        end = max(e for _, e, _ in self.buffers())
        return (end + 255) & ~255

    def forward(self):
        """Fill the layer-output part of the arena with 0xFF, run forward(), keep the returned maps."""
        end = self.prefix_end()
        if not self.plan.training:
            assert end == self.plan.act.numel(), (end, self.plan.act.numel())
        self.plan.act[:end].fill_(0xFF)
        torch.cuda.synchronize()
        self.fms = self.m.forward(self.x)
        torch.cuda.synchronize()

    # ------------------------------------------------------------------ BN fold
    def fold(self, i):
        """(scale, shift) float32 [cout] made by yb_bn_fold from layer i's masters; heads: (1, bias).  Checks the fold
        against float64 within FOLD_ULPS fp32 ulps (shift: of itself and of mean * scale)."""
        L, plan = self.L, self.plan
        p = plan.conv_params(i)
        c = p["w"].shape[0]
        if "b" in p:
            return torch.ones(c, dtype=torch.float32, device="cuda"), p["b"].clone()
        sc = torch.empty(c, dtype=torch.float32, device="cuda")
        sh = torch.empty_like(sc)
        L.check(L.lib.yb_bn_fold(L.ptr(p["gamma"]), L.ptr(p["beta"]), L.ptr(p["mean"]), L.ptr(p["var"]), c, EPS32,
                                 L.ptr(sc), L.ptr(sh), L.stream_handle()), "bn_fold")
        s64 = p["gamma"].double() / torch.sqrt(p["var"].double() + EPS32)
        t64 = p["beta"].double() - p["mean"].double() * s64
        self.worst.add("fold scale", f"layer {i}", R.check_out(sc, s64, FOLD_ULPS * ulp32(s64), f"{self.cid} layer {i} fold scale"))
        bsh = FOLD_ULPS * (ulp32(t64) + ulp32(p["mean"].double() * s64))
        self.worst.add("fold shift", f"layer {i}", R.check_out(sh, t64, bsh, f"{self.cid} layer {i} fold shift"))
        return sc, sh

    # ------------------------------------------------------------------ a-d: layer outputs
    def _input(self, i):
        """Layer i's input view [n, h, w, cin] from the topology: a concat consumer's whole [upsampled | route] buffer."""
        plan, topo = self.plan, self.topo
        srcs = topo.inputs[i]
        t = plan.layer_output(srcs[0])
        if len(srcs) > 1:
            assert topo.out_off[srcs[0]] == 0
            t = t.as_strided(t.shape[:3] + (t.stride(2),), t.stride(), t.storage_offset())
        return t

    def check_layers(self):
        plan, topo, dt = self.plan, self.topo, self.dtype
        nl = plan.num_layers
        infos = [plan.layer_info(i) for i in range(nl)]
        w16 = [plan.conv_params(i)["w"].to(dt) for i in range(nl)]
        folds = [self.fold(i) for i in range(nl)]
        outs = [plan.layer_output(i) for i in range(nl)]
        ins = [None] + [self._input(i) for i in range(1, nl)]
        for i in range(1, nl):
            assert ins[i].shape[3] == infos[i].cin, (i, ins[i].shape, infos[i].cin)
        heads = {h: k for k, h in enumerate(topo.heads)}
        for im in range(self.n):
            # ---- b. the stem
            x16 = self.x[im:im + 1].to(dt)
            raw, S = R.conv_raw(x16, w16[0], 1, 1)
            sc0, sh0 = folds[0]
            v0 = R.epilogue(raw, sc0, sh0, leaky=True)
            if self.fused:
                xs, d = D.stem_interval(v0, S, dt, sc0, sh0)
                shp = (1, infos[0].out_h, infos[0].out_w, infos[0].cout)
                stem_in = (xs.reshape(shp), d.reshape(shp))
                self.near_mid = max(self.near_mid, float((d > 0).double().mean()))
            else:
                got = outs[0][im].reshape(-1, infos[0].cout)
                b = R.out_bound(v0, S, D.STEM_N16, dt, scale=sc0, shift=sh0)
                self.worst.add("stem", f"layer 0 image {im}", R.check_out(got, v0, b, f"{self.cid} layer 0 image {im}"))
                stem_in = None
            del raw, S, v0
            # ---- a / c / d. layers 1 ..
            for i in range(1, nl):
                f = infos[i]
                name = f"{self.cid} layer {i} image {im}"
                pad = f.ksize // 2
                extra = 0.0
                if i == 1 and stem_in is not None:
                    raw, S, extra = D.conv1_on_interval(*stem_in, w16[1], f.stride, folds[1][0])
                else:
                    xin = ins[i][im:im + 1]
                    assert bool(torch.isfinite(xin).all()), f"{name}: its input holds the sentinel or a non-finite value"
                    raw, S = R.conv_raw(xin, w16[i], f.stride, pad)
                n16 = f.ksize * f.ksize * f.cin // 16
                if i in heads:
                    got = self.fms[heads[i]][im].reshape(-1, f.cout)
                    b = folds[i][1]
                    ref = raw + b.double()
                    bound = R.out_bound(ref, S, n16, torch.float32, shift=b)
                    self.worst.add("head map", f"layer {i} image {im}", R.check_out(got, ref, bound, name + " head map"))
                    continue
                sc, sh = folds[i]
                res = None
                if i in topo.residual:
                    res = outs[i - 2][im].reshape(-1, f.cout)
                ref = R.epilogue(raw, sc, sh, leaky=True, res=res)
                e32 = R.out_bound(ref, S, n16, torch.float32, scale=sc, shift=sh, res=res) + extra
                bound = e32 + 0.5 * R.ulp(ref.abs() + e32, dt)
                o = outs[i][im]
                if f.upsample2x:
                    c0 = _bits(o[0::2, 0::2])
                    for dy, dx in ((0, 1), (1, 0), (1, 1)):
                        bad = _count(_bits(o[dy::2, dx::2]) != c0)
                        assert bad == 0, f"{name}: {bad} elements of upsampled copy ({dy}, {dx}) differ from copy (0, 0)"
                    o = o[0::2, 0::2]
                got = o.reshape(-1, f.cout)
                kind = {1: "igemm", 2: "halo", 3: "fused stem + Conv_1", 4: "stem", 5: "thin"}[self.scheds[i].kernel]
                if i in topo.residual:
                    kind += " residual"
                self.worst.add(kind, f"layer {i} image {im}", R.check_out(got, ref, bound, f"{name} ({kind})"))
                del raw, S, ref, bound
        # d. both halves of every concat buffer written on every row
        for cat, (up, route) in topo.concat.items():
            full = self._input(cat)
            bad = _count(_bits(full) == -1)
            assert bad == 0, f"{self.cid}: {bad} sentinel elements left in the concat buffer layer {cat} reads"

    # ------------------------------------------------------------------ e. arena hygiene
    def check_hygiene(self):
        act = self.plan.act
        pos = 0
        for s, e, written in self.buffers():
            assert s >= pos, f"{self.cid}: layer-output buffers overlap at byte {s}"
            spans = [(pos, s)] + ([] if written else [(s, e)])
            for a, b in spans:
                bad = _count(act[a:b] != 0xFF)
                assert bad == 0, f"{self.cid}: {bad} bytes in [{a}, {b}) of the activation arena were written " \
                                 f"({'a gap between buffers' if b == s else 'a buffer forward() must not write'})"
            pos = e
        end = self.prefix_end()
        bad = _count(act[pos:end] != 0xFF)
        assert bad == 0, f"{self.cid}: {bad} bytes after the last layer-output buffer were written"

    # ------------------------------------------------------------------ f. detect
    def check_detect(self):
        from yolov3_tensorflow_b200.utils.nms_utils import batched_nms_raw
        L, m, x = self.L, self.m, self.x
        mb, thr, iou = NMS
        snap = self.plan.act.clone()
        boxes, scores = m.predict_scores(self.fms)
        ub = batched_nms_raw(boxes, scores, CLASSES, mb, thr, iou)
        runs = []
        for hs in (None, "0"):
            L.set_option("YB_HEAD_STREAM", hs)
            fb = [t.clone() for t in m.detect_raw(x, mb, thr, iou)]
            torch.cuda.synchronize()
            L.set_option("YB_HEAD_STREAM", None)
            tag = f"{self.cid} detect_raw" + ("" if hs is None else " YB_HEAD_STREAM=0")
            assert torch.equal(fb[0], boxes), f"{tag}: decoded boxes differ from predict_scores(forward())"
            cu, cf = ub[4].cpu().numpy(), fb[5].cpu().numpy()
            assert np.array_equal(cu, cf), f"{tag}: counts {cf} != batched_nms_raw {cu}"
            for im in range(self.n):
                k = int(cu[im])
                for what, a, b in zip(("boxes", "scores", "labels", "indices"), ub[:4], fb[1:5]):
                    assert torch.equal(a[im, :k], b[im, :k]), f"{tag}: image {im} kept {what} differ"
            neq = _count(self.plan.act != snap)
            assert neq == 0, f"{tag}: {neq} arena bytes differ from the forward() run"
            runs.append(fb)
        cf = runs[0][5].cpu().numpy()
        assert int(cf.sum()) > 0, f"{self.cid}: no detections"
        for im in sorted({0, self.n - 1}):
            ob, os_, ol, oi = O.gpu_nms(boxes[im:im + 1].cpu().numpy(), scores[im:im + 1].cpu().numpy(), CLASSES, mb, thr, iou)
            k = int(cf[im])
            assert k == len(oi), f"{self.cid}: image {im}: {k} kept, O.gpu_nms keeps {len(oi)}"
            assert np.array_equal(runs[0][4][im, :k].cpu().numpy(), oi) and np.array_equal(runs[0][3][im, :k].cpu().numpy(), ol)
        print(f"PLAN {self.cid} detect: {int(cf.sum())} detections over {self.n} images, bit-identical to the unfused "
              f"pipeline with and without the head side stream")

    # ------------------------------------------------------------------ weights of a training plan
    def check_w16(self):
        plan = self.plan
        for i in range(1, plan.num_layers):
            info = plan.layer_info(i)
            q = plan.conv_params(i)["w"].to(self.dtype)
            w16 = plan.train_buffer(i, "w16")
            want = torch.zeros_like(w16)
            want[:info.cout] = q.reshape(info.cout, -1)
            bad = _count(_bits(w16) != _bits(want))
            assert bad == 0, f"{self.cid} layer {i}: {bad} elements of the 16-bit weights differ from RN16(master)"

    def check(self):
        self.check_layers()
        self.check_hygiene()


def make_model(dt, weights):
    import yolov3_tensorflow_b200 as pkg
    m = pkg.yolov3(CLASSES, O.COCO_ANCHORS, dtype=dt)
    m.set_params(params_for(weights), "HWIO")
    return m


@pytest.mark.parametrize("cid,opts,dt,weights,n,hw", P.CONFIGS, ids=[c[0] for c in P.CONFIGS])
def test_infer_plan_launches_against_float64(L, cid, opts, dt, weights, n, hw):
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    P.set_options(L, opts)
    m = make_model(dt, weights)
    worst = Worst(cid)
    topo = P.Topology()
    runs = []
    if cid == "trained":
        tn, thw = P.TRAIN_KEY
        _, xt, ys = _train_case(seed=41, n=tn, h=thw[0], w=thw[1])
        xt = torch.from_numpy(xt).cuda()
        m.train_step(xt, [torch.from_numpy(y).cuda() for y in ys], 1e-2, momentum=0.9)
        torch.cuda.synchronize()
        r = InferRun(L, m, cid, xt, worst)
        assert r.plan.training
        r.check_w16()
        runs.append(r)
    x = torch.from_numpy(gen_inputs(3 + hw[0], n, hw[0], hw[1])).cuda()
    r = InferRun(L, m, cid, x, worst)
    assert not r.plan.training
    infos = [r.plan.layer_info(i) for i in range(r.plan.num_layers)]
    P.premise(cid, r.scheds, infos, topo)
    runs.append(r)
    for r in runs:
        r.forward()
        r.check()
        if r.fused:
            print(f"PLAN {cid} stem interval: at most {r.near_mid:.2e} of an image's stem values have two candidates")
    if cid in ("bench", "608", "rect"):
        runs[-1].check_detect()
    worst.report()
    print(f"PLAN {cid}: {dt} n {n} {hw[0]} x {hw[1]}, peak CUDA memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB, "
          f"{time.time() - t0:.1f} s")
