"""The training plan's conv launches, rebuilt from the model's structure (tests/test_train_plan_host.py,
tests/test_gpu_train_plan.py).

Routing of the input gradients.  The backward runs the layers last to first.  Layer i's dgrad writes dX = the gradient
of its input tensor T, which the other consumers of T also feed:
  - a conv consumer with a higher index ran earlier: layer i accumulates in place onto what is there ("inplace");
  - otherwise layer i writes fresh, and if T is also the shortcut of a residual layer b (T = out(b - 2) = in(b - 1)),
    its dgrad adds dA(out_b), which passes through the shortcut unchanged ("pass", b);
  - everything else writes fresh with no residual ("fresh").
The concat consumers (60, 68) read the whole concat buffer [upsampled | route]; the route slice is also read by the
stride-2 conv after it (43, 26).

Requests.  Every implicit-GEMM launch train_bind prepares, as the yb_conv_desc / window / statistics triple that
yb_conv_schedule takes: the statistics forward of the BN layers (raw z, out_ld = cout), the detection heads' forward,
and the dgrads (the stride-1 conv over dz with the flipped weights; a stride-2 layer's four parity-class windows over
the plain dz, or under YB_DGRAD_S2=dilated one 3x3 conv over the zero-inserted dz at the input resolution).
"""
import ctypes as C

from tests.conv_ref import units_per_warpgroup
from yolov3_tensorflow_b200.model import yolov3

CLASSES = 80
BODY = 52                          # darknet53_body: layers 0..51; yolov3_head: 52..74
# (id, options, dtype, n, (H, W)).  Options are read when a plan is created and bound.
CONFIGS = [
    ("default-fp16", {}, "fp16", 8, (416, 416)),
    ("default-bf16", {}, "bf16", 8, (416, 416)),
    ("coop", {"YB_CONV_PP": "0"}, "bf16", 2, (416, 416)),
    ("pp", {"YB_CONV_PP": "1"}, "bf16", 2, (416, 416)),
    ("mcast-2x2", {"YB_CONV_MCAST": "2x2"}, "bf16", 2, (416, 416)),
    ("mcast-1x2", {"YB_CONV_MCAST": "1x2"}, "bf16", 2, (416, 416)),
    ("mcast-2x1", {"YB_CONV_MCAST": "2x1"}, "bf16", 2, (416, 416)),
    ("reg+mcast", {"YB_CONV_EPI": "reg", "YB_CONV_MCAST": "2x2"}, "bf16", 2, (416, 416)),
    ("ldg", {"YB_CONV_RES": "ldg"}, "bf16", 2, (416, 416)),
    ("dilated", {"YB_DGRAD_S2": "dilated"}, "fp16", 2, (416, 416)),
    ("eg1", {"YB_CONV_EG": "1"}, "bf16", 2, (416, 416)),
    ("2cta", {"YB_CONV_MODE": "2cta", "YB_CONV_MC": "1"}, "bf16", 2, (416, 416)),
    ("capped", {"YB_CONV_CTAS": "3"}, "bf16", 2, (160, 224)),
    ("capped+mcast", {"YB_CONV_CTAS": "3", "YB_CONV_MCAST": "2x2"}, "bf16", 2, (160, 224)),
]
KEYS = ("YB_CONV_PP", "YB_CONV_MCAST", "YB_CONV_EPI", "YB_CONV_RES", "YB_DGRAD_S2", "YB_CONV_EG", "YB_CONV_MODE",
        "YB_CONV_MC", "YB_CONV_CTAS")
SMS = 132


def set_options(L, opts):
    for k in KEYS:
        L.set_option(k, opts.get(k))


class Topology:
    """The layer graph of model.py's 75 convs, from conv_table and the darknet / YOLOv3 block structure."""

    def __init__(self, classes=CLASSES):
        t = yolov3.conv_table(classes)
        self.table = t
        nl = len(t)
        # residual blocks (utils/layer_utils.py:25-32): a 1x1 conv, then a 3x3 stride-1 conv adding the block input
        self.residual = [b for b in range(2, BODY) if t[b][2] == 3 and t[b][3] == 1 and t[b - 1][2] == 1]
        # the two routes: the last block output before the 52^2 -> 26^2 and 26^2 -> 13^2 stride-2 convs
        s2 = [i for i in range(BODY) if t[i][3] == 2]
        self.route1, self.route2 = s2[-2] - 1, s2[-1] - 1
        heads = [i for i in range(nl) if not t[i][4]]
        # after heads 1 and 2: the 1x1 conv of the yolo block's route (3 layers back), stored 2x upsampled into the
        # concat buffer; the next yolo block reads [upsampled | route]
        self.upsample = [h + 1 for h in heads[:2]]
        self.concat = {self.upsample[0] + 1: (self.upsample[0], self.route2),
                       self.upsample[1] + 1: (self.upsample[1], self.route1)}
        self.heads = heads
        self.inputs = {}                          # layer -> the layer(s) whose output it reads
        for i in range(1, nl):
            if i in self.concat:
                self.inputs[i] = list(self.concat[i])
            elif i in self.upsample:
                self.inputs[i] = [i - 3]          # the yolo block's route (its 5th conv) feeds the upsampling conv
            else:
                self.inputs[i] = [i - 1]
        self.out_ld = {}
        for j in range(nl):
            self.out_ld[j] = t[j][1]
        for cat, (up, route) in self.concat.items():
            ld = t[up][1] + t[route][1]
            self.out_ld[up] = self.out_ld[route] = ld
        self.out_off = {j: 0 for j in range(nl)}
        for cat, (up, route) in self.concat.items():
            self.out_off[route] = t[up][1]

    def in_ld(self, i):
        return self.out_ld[self.inputs[i][0]]

    def producer(self, i):
        """The layer at channel 0 of layer i's input."""
        return self.inputs[i][0]

    def conv_consumers(self, j):
        """Layers whose conv reads out_j (directly or through a concat buffer)."""
        return [i for i in self.inputs if j in self.inputs[i]]

    def route(self, i):
        """('fresh' | 'inplace' | 'pass', b) of layer i's dgrad (module docstring)."""
        srcs = self.inputs[i]
        if len(srcs) > 1:                     # a concat consumer writes the whole concat gradient
            assert all(max(self.conv_consumers(j)) == i for j in srcs), i
            return "fresh", None
        j = srcs[0]
        if max(self.conv_consumers(j)) != i:
            return "inplace", None
        b = [b for b in self.residual if b - 1 == i]
        return ("pass", b[0]) if b else ("fresh", None)


def _desc(L, **kw):
    d = dict(res_ld=0, out_fp32=0, leaky=0, upsample2x=0)
    d.update(kw)
    return L.ConvDesc(**d)


def requests(L, topo, infos, n, dtype_code, dilated):
    """{layer: [(what, desc, kh, kw, with_stats)]} of the implicit-GEMM launches train_bind prepares (module
    docstring).  infos: yb_layer_info of every layer."""
    out = {}
    for i in range(1, len(infos)):
        f = infos[i]
        kco = -(-f.cout // 32) * 32
        in_ld = topo.in_ld(i)
        rs = []
        if f.has_bn:
            rs.append(("fwd", _desc(L, n=n, h=f.in_h, w=f.in_w, cin=f.cin, cout=f.cout, ksize=f.ksize, stride=f.stride,
                                    in_ld=in_ld, out_ld=f.cout, dtype=dtype_code), 0, 0, 1))
        else:
            rs.append(("fwd", _desc(L, n=n, h=f.in_h, w=f.in_w, cin=f.cin, cout=f.cout, ksize=f.ksize, stride=f.stride,
                                    in_ld=in_ld, out_ld=f.cout, dtype=dtype_code, out_fp32=1), 0, 0, 0))
        dz_ld = f.cout if f.has_bn else kco
        kind, b = topo.route(i)
        res_ld = {"fresh": 0, "inplace": in_ld, "pass": topo.out_ld[b] if b is not None else 0}[kind]
        if f.stride == 2 and not dilated:
            for c in range(4):
                rs.append((f"dgrad class {c}", _desc(L, n=n, h=f.in_h // 2, w=f.in_w // 2, cin=kco, cout=f.cin, ksize=1,
                                                     stride=1, in_ld=dz_ld, out_ld=in_ld, res_ld=res_ld,
                                                     dtype=dtype_code), 1 + (c >> 1), 1 + (c & 1), 0))
        else:
            rs.append(("dgrad", _desc(L, n=n, h=f.in_h, w=f.in_w, cin=kco, cout=f.cin, ksize=f.ksize, stride=1,
                                      in_ld=dz_ld, out_ld=in_ld, res_ld=res_ld, dtype=dtype_code), 0, 0, 0))
        out[i] = rs
    return out


def schedule(L, desc, kh, kw, stats, sms=SMS):
    """yb_conv_schedule -> (rc, info, message)."""
    info = L.ConvSchedule()
    rc = L.lib.yb_conv_schedule(C.byref(desc), kh, kw, int(stats), sms, C.byref(info))
    return rc, info, (L.lib.yb_last_error_string().decode() if rc else "")


def schedules(L, topo, infos, n, dtype_code, dilated, sms=SMS):
    """{layer: [(what, desc, kh, kw, stats, info)]}; raises AssertionError naming the first request without a kernel."""
    out = {}
    for i, rs in requests(L, topo, infos, n, dtype_code, dilated).items():
        out[i] = []
        for what, d, kh, kw, st in rs:
            rc, info, msg = schedule(L, d, kh, kw, st, sms)
            if rc:
                raise AssertionError(f"layer {i} {what}: no kernel: {msg}")
            out[i].append((what, d, kh, kw, st, info))
    return out


def premise(cid, scheds, topo):
    """Asserts what configuration `cid` exists for (tests/test_gpu_train_plan.py, the configuration table)."""
    flat = [(i, what, d, info) for i, rs in scheds.items() for what, d, kh, kw, st, info in rs]
    dg = [(i, what, d, info) for i, what, d, info in flat if what.startswith("dgrad")]
    fw = [(i, what, d, info) for i, what, d, info in flat if what == "fwd" and topo.table[i][4]]
    par = [(i, what, d, info) for i, what, d, info in dg if what.startswith("dgrad class")]
    if cid == "pp":
        for b in (topo.route1, topo.route2):
            (_, _, d, info), = [x for x in dg if x[0] == b - 1]
            assert info.pingpong and info.res_smem == 1 and d.res_ld != d.out_ld, (b - 1, d.res_ld, d.out_ld)
    if cid.startswith("mcast"):
        shape = cid.split("-")[1]
        cm, cn = int(shape[0]), int(shape[2])
        for group, name in ((par, "parity-class dgrad"), (fw, "statistics forward")):
            assert any(info.cluster_m == cm and info.cluster_n == cn for _, _, _, info in group), \
                f"{cid}: no {name} runs a {shape} cluster"
    if cid == "reg+mcast":
        assert not any(info.pingpong for _, _, _, info in dg), "reg+mcast: a dgrad runs ping-pong"
        assert all(info.cluster == 1 for _, _, _, info in dg), "reg+mcast: a dgrad runs clustered"
        assert any(info.pingpong and info.cluster_n == 2 for _, _, _, info in fw), \
            "reg+mcast: no statistics forward runs as a ping-pong 2x2 cluster"
    if cid.startswith("capped"):
        for group, name in ((dg, "dgrad"), (par, "parity-class dgrad"), (fw, "statistics forward")):
            assert any(units_per_warpgroup(info) >= 3 for _, _, _, info in group), \
                f"{cid}: no {name} gives a warpgroup 3 units"
        if cid == "capped+mcast":
            assert any(info.cluster > 1 and units_per_warpgroup(info) >= 3 for _, _, _, info in fw), \
                f"{cid}: no clustered statistics forward gives a warpgroup 3 units"
    if cid == "dilated":
        s2 = [i for i in scheds if topo.table[i][3] == 2]
        assert s2 and not par
        for i in s2:
            (what, d, kh, kw, st, info), = [r for r in scheds[i] if r[0] == "dgrad"]
            assert d.ksize == 3 and info.num_kb * info.block_k == 9 * d.cin, i
    return flat
