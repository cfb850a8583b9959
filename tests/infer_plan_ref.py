"""The 16-bit inference plan's launches, as the configurations of tests/test_gpu_infer_plan.py exercise them
(tests/test_infer_plan_host.py checks every premise on unbound plans).

The layer graph is train_plan_ref.Topology: inputs, residual and upsampling layers, concat buffers and the channel
offsets of the route convs inside them.  The inference plan runs the same graph with other launches: folded BN, leaky
and the shortcut in the epilogue, the stem fused into Conv_1's halo launch, the halo kernel on Conv_3 with its residual
box, plan-rule multicast clusters, and the fused-decode heads under detect_raw.  What each layer launches is reported by
yb_net_layer_schedule's `kernel` field (YB_LAYER_*).
"""
import ctypes as C

from tests.conv_ref import units_per_warpgroup
from tests.train_plan_ref import CLASSES, SMS, Topology  # noqa: F401  (the graph is the training plan's)

# (id, options, dtype, weights, n, (H, W)).  Options are read when a plan binds and at every forward.  Weights: "cfg1"
# is Glorot init with identity BN and zero detection biases; "cfg2" is the benchmark's kind: random BN statistics,
# detection-head weights x 8 and confidence bias -2.
CONFIGS = [
    ("bench", {}, "fp16", "cfg2", 64, (416, 416)),
    ("bf16", {}, "bf16", "cfg1", 8, (416, 416)),
    ("608", {}, "fp16", "cfg2", 4, (608, 608)),
    ("rect", {}, "fp16", "cfg2", 3, (288, 480)),
    ("mcast-off", {"YB_CONV_MCAST": "0"}, "fp16", "cfg2", 8, (416, 416)),
    ("ldg", {"YB_CONV_RES": "ldg"}, "fp16", "cfg2", 8, (416, 416)),
    ("coop", {"YB_CONV_PP": "0"}, "bf16", "cfg2", 4, (416, 416)),
    ("stem-unfused", {"YB_STEM_FUSE": "0"}, "fp16", "cfg2", 4, (416, 416)),
    ("halo-off", {"YB_HALO": "0"}, "fp16", "cfg2", 4, (416, 416)),
    ("halo-all", {"YB_HALO": "1"}, "fp16", "cfg2", 4, (416, 416)),
    ("thin", {"YB_THIN": "2"}, "fp16", "cfg2", 4, (416, 416)),
    ("capped+mcast", {"YB_CONV_CTAS": "3"}, "bf16", "cfg2", 2, (160, 224)),
    ("trained", {}, "bf16", "cfg2", 8, (416, 416)),
]
TRAIN_KEY = (2, (416, 416))        # "trained": the training step's batch and size; inference then runs on both keys
KEYS = ("YB_CONV_PP", "YB_CONV_MCAST", "YB_CONV_RES", "YB_CONV_CTAS", "YB_STEM_FUSE", "YB_HALO", "YB_THIN",
        "YB_HEAD_STREAM", "YB_CONV_EPI", "YB_CONV_EG", "YB_CONV_MODE", "YB_CONV_MC", "YB_DGRAD_S2")


def set_options(L, opts):
    for k in KEYS:
        L.set_option(k, opts.get(k))


def layer_schedules(L, handle, sms=SMS):
    """yb_net_layer_schedule of every layer of a plan (bound or not) -> [LayerSchedule]."""
    out = []
    for i in range(L.lib.yb_net_num_layers(handle)):
        s = L.LayerSchedule()
        L.check(L.lib.yb_net_layer_schedule(handle, i, sms, C.byref(s)), "layer_schedule")
        out.append(s)
    return out


def premise(cid, scheds, infos, topo):
    """Asserts what configuration `cid` exists for (the table in tests/test_gpu_infer_plan.py); scheds / infos: the
    plan's yb_net_layer_schedule / yb_net_layer_info of every layer."""
    K = [s.kernel for s in scheds]
    ig = [i for i, s in enumerate(scheds) if s.igemm]
    res_ig = [i for i in ig if scheds[i].residual]
    c3 = topo.residual[0]                                    # Conv_3, the first residual layer (Cin = 32)
    assert all(scheds[i].kernel == 1 for i in topo.heads), f"{cid}: a head does not run the implicit GEMM"
    fused = K[0] == K[1] == 3
    default_like = cid in ("bench", "bf16", "608", "rect", "mcast-off", "ldg", "coop", "capped+mcast", "trained")
    if default_like:
        assert fused, f"{cid}: the stem is not fused into Conv_1 ({K[0]}, {K[1]})"
        assert K[c3] == 2 and scheds[c3].residual, f"{cid}: Conv_3 does not run the halo kernel with its residual"
        assert all(K[i] == 1 for i in range(2, len(K)) if i != c3), f"{cid}: a layer after Conv_1 leaves the implicit GEMM"
    if cid in ("bench", "608", "rect", "trained"):
        shapes = {(scheds[i].cluster_m, scheds[i].cluster_n) for i in ig}
        assert {(2, 2), (2, 1)} <= shapes, f"{cid}: plan-rule cluster shapes {shapes}"
        assert any(scheds[i].res_smem for i in res_ig), f"{cid}: no residual conv prefetches its shortcut"
        assert scheds[c3].res_smem, f"{cid}: Conv_3's halo launch does not load its residual box"
    if cid == "bench":
        # batch 64: clustered launches whose last cluster holds a tail m-tile, and launches whose units exceed the grid
        assert any(scheds[i].cluster_m > 1 and scheds[i].num_m_tiles % scheds[i].cluster_m for i in ig), \
            "bench: no clustered launch has a partial last cluster"
        assert any(scheds[i].units > scheds[i].grid // (scheds[i].cluster_m * scheds[i].cluster_n) for i in ig)
    if cid == "608":
        grids = {(infos[h].out_h, infos[h].out_w) for h in topo.heads}
        assert grids == {(19, 19), (38, 38), (76, 76)}, grids
        assert any(infos[i].out_h * infos[i].out_w * 4 % scheds[i].block_m for i in ig), "608: no m-tile tail"
    if cid == "rect":
        assert (infos[topo.heads[0]].out_h, infos[topo.heads[0]].out_w) == (9, 15)
    if cid == "mcast-off":
        assert all(scheds[i].cluster_m * scheds[i].cluster_n == 1 for i in ig), "mcast-off: a launch is clustered"
    if cid == "ldg":
        assert res_ig and not any(scheds[i].res_smem for i in res_ig), "ldg: a residual conv prefetches"
        assert K[c3] == 2 and not scheds[c3].res_smem, "ldg: Conv_3's halo launch does not read its residual globally"
    if cid == "coop":
        assert ig and not any(scheds[i].pingpong for i in ig), "coop: a launch runs ping-pong"
    if cid == "stem-unfused":
        assert K[0] == 4 and K[1] == 2, f"stem-unfused: layers 0 and 1 run {K[0]}, {K[1]}"
    if cid == "halo-off":
        assert 2 not in K and 3 not in K and K[0] == 4, f"halo-off: kernels {sorted(set(K))}"
        assert scheds[1].igemm and scheds[c3].igemm
    if cid == "halo-all":
        wide = [i for i in range(1, len(K)) if infos[i].ksize == 3 and infos[i].cin == 64 and infos[i].cout == 128]
        assert wide and any(K[i] == 2 for i in wide), "halo-all: no 64 -> 128 3x3 runs the halo kernel"
        assert fused
    if cid == "thin":
        assert K[0] == 4 and K[1] == 5 and K[c3] == 5, f"thin: layers 0, 1, {c3} run {K[0]}, {K[1]}, {K[c3]}"
    if cid == "capped+mcast":
        cl = [i for i in ig if scheds[i].cluster_m * scheds[i].cluster_n > 1]
        assert any(units_per_warpgroup(_conv_like(scheds[i])) >= 3 for i in cl), \
            "capped+mcast: no clustered launch gives a warpgroup 3 units"
        assert any(scheds[i].res_smem and scheds[i].cluster_m * scheds[i].cluster_n > 1 and
                   units_per_warpgroup(_conv_like(scheds[i])) >= 3 for i in res_ig), \
            "capped+mcast: no clustered shortcut prefetch over 3 units per warpgroup"
    return K


class _conv_like:
    """A LayerSchedule read as the yb_conv_schedule fields units_per_warpgroup uses."""

    def __init__(self, s):
        self.units, self.grid, self.pingpong = s.units, s.grid, s.pingpong
        self.cluster = s.cluster_m * s.cluster_n
