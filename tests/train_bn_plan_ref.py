"""The training plan's batch-norm launches: the configuration table and its premises (tests/test_gpu_train_bn_plan.py,
tests/test_train_bn_plan_host.py).

Every BN layer of a training step runs three streaming launches over its rows (csrc/net_train.cu): the activation
store (bn_stats_act_apply, or bn_finalize + bn_act_apply under YB_BN_FIN=0), the gradient sums dgamma / dbeta
(bn_bwd_reduce) and dz (bn_bwd_apply).  Their launch shape is yb_bn_schedule's: one wave of SM count x blocks-per-SM
blocks of rows_per_block rows, walked R rows per lane at a time.  A configuration is worth running only if its layers
reach the parts of that shape where a kernel can go wrong: the R-row loop past its first group, a short last block,
and >= 16 blocks per workspace slot of the reduce (so every slot takes several atomic adds).
"""
import ctypes as C

from tests.bn_ref import BN_SLOTS, FTZ32
from tests.conv_ref import U32

SMS = 132
EPS = 1e-5                         # yb_net's bn_eps (model.py:37)
KEYS = ("YB_BN_FIN", "YB_BN_CPT", "YB_DGRAD_S2", "YB_STEM_TRAIN")
# (id, options, mode, dtype, n, (H, W)).  Options are set before the plan binds.  mode: "fused" runs the step through
# yb_net_train_fwd_bwd (dgamma / dbeta only in the flat gradient), "frozen" passes YB_TRAIN_BN_FROZEN, "replicas"
# runs with bn_replicas = 2 and doubles both exchange slabs between LOCAL and GLOBAL; the rest run the layered step.
# bench-608 runs the benchmark's batch 32 beside float64 references computed a few images at a time.
CONFIGS = [
    ("bench-416", {}, "layered", "bf16", 32, (416, 416)),
    ("bench-608", {}, "layered", "bf16", 32, (608, 608)),
    ("fp16", {}, "layered", "fp16", 8, (416, 416)),
    ("fused", {}, "fused", "bf16", 8, (416, 416)),
    ("fin0", {"YB_BN_FIN": "0"}, "layered", "bf16", 2, (416, 416)),
    ("cpt4", {"YB_BN_CPT": "4"}, "layered", "fp16", 2, (416, 416)),
    ("frozen", {}, "frozen", "bf16", 2, (416, 416)),
    ("frozen+fin0", {"YB_BN_FIN": "0"}, "frozen", "fp16", 2, (416, 416)),
    ("two-ranks", {}, "replicas", "bf16", 2, (416, 416)),
    ("dilated", {"YB_DGRAD_S2": "dilated"}, "layered", "fp16", 2, (416, 416)),
    ("stem-cuda", {"YB_STEM_TRAIN": "cuda"}, "layered", "bf16", 2, (416, 416)),
    ("rect", {}, "layered", "bf16", 4, (288, 480)),
]


def set_options(L, opts):
    for k in KEYS:
        L.set_option(k, opts.get(k))


def bn_schedule(L, rows, c, sms=SMS):
    s = L.BnSchedule()
    L.check(L.lib.yb_bn_schedule(rows, c, sms, C.byref(s)), "bn_schedule")
    return s


def launch_premises(s, rows):
    """What one BN launch of `rows` rows reaches (module docstring)."""
    last = rows - (s.grid - 1) * s.rows_per_block
    return {"groups": -(-s.rows_per_block // s.lanes) > s.r,
            "short last block": last < s.rows_per_block,
            ">= 16 blocks per slot": s.grid >= 16 * BN_SLOTS}


def schedules(L, infos, n, sms=SMS):
    """{layer: yb_bn_schedule result} of every BN layer of a plan (infos: yb_layer_info of every layer)."""
    return {f.index: bn_schedule(L, n * f.out_h * f.out_w, f.cout, sms) for f in infos if f.has_bn}


def premise(L, cid, opts, infos, n):
    """Asserts that the BN layers of a plan reach every launch premise at SMS SMs (an H100 SXM), and that cpt4 runs
    the CPT-4 build everywhere.  Returns the schedules."""
    scheds, seen = schedules(L, infos, n), {}
    for f in infos:
        if not f.has_bn:
            continue
        s = scheds[f.index]
        for k, v in launch_premises(s, n * f.out_h * f.out_w).items():
            seen[k] = seen.get(k, 0) + int(v)
        if cid == "cpt4":
            assert s.cpt == 4, (cid, f.index, s.cpt)
    assert all(seen.get(k, 0) >= 1 for k in ("groups", "short last block", ">= 16 blocks per slot")), (cid, seen)
    return scheds


def col_stats_bound(mag, rows, c, sms):
    """Bound of one column sum of yb_col_stats / yb_col_sum (csrc/bn.cu) whose terms have magnitude sum `mag`.
    Launch shape: gy = ceil(c / 32) column groups, sms * 8 / gy row slabs of rpb >= 32 rows.  A value passes through
    ceil(rpb / 8) adds of its thread (every 8th row of the slab), the 7 adds of row lane 0 over the other lanes'
    partials and grid_x atomic adds of the slab totals into the zeroed output, plus one for the rounded product of the
    sum of squares: depth u mag.  Each atomic add may also flush a subnormal input and result to zero (tests/bn_ref.py):
    2 grid_x 2^-126 more."""
    gy = -(-c // 32)
    slabs = max(1, sms * 8 // gy)
    rpb = max(32, -(-rows // slabs))
    grid_x = -(-rows // rpb)
    depth = -(-rpb // 8) + 7 + grid_x + 1
    return depth * U32 * mag + 2 * grid_x * FTZ32
