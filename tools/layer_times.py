#!/usr/bin/env python
"""Per-layer times of the bench forward (batch 64, 416x416, fp16, bench.py's seeded weights), CUDA-event timed.

  python tools/layer_times.py [--batch B] [--size S] [--reps R] [--json FILE]

Every layer is launched alone through yb_net_forward_layers(first = last = i) --reps times after a warm-up, between
two events.  The detection heads run unfused here (fp32 feature map out), not with the decode of yb_net_detect.
Layer 0 (the stem) runs inside layer 1's launch.  Per layer: shape, kernel, ms, algorithmic TFLOP/s.

The `res` column marks the layers that add a shortcut.  Each shortcut layer is then paired with its no-shortcut
twins, the layers of the same GEMM (cin, cout, k, output size; stride free) and kernel: Conv_6/8 with Conv_4 at 104^2,
and at 52^2, 26^2 and 13^2 the darknet 3x3s with the yolo-block 3x3s.  The summary prints the time each class loses to
its shortcut (sum over its shortcut layers of ms - mean twin ms).

Then the conv_igemm time of a layer is split into a per-k-block and a per-tile fixed cost from pairs of layers
with the same tile count and different K (52^2: layer 68 vs 70/72; 26^2: layer 60 vs 62/64):
    t = waves * (kblocks * c_kb + c_fix),   waves = ceil(tiles / SMs)
and the fixed cost summed over the conv_igemm layers is printed beside the conv total.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CLASS_NUM = 80


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        return out or "nvidia-smi: no output"
    except Exception as e:                     # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def kernel_of(lib, info, batch):
    """Which kernel forward_layers_impl (csrc/net.cu) launches for a layer when none of its switches is set: the halo
    kernel (the stem fused into layer 1) for the Cin = 32 3x3 BN layers it supports, conv_igemm for every other."""
    from yolov3_tensorflow_b200._lib import ConvDesc, YB_F16
    if info.index == 0:
        return "stem (in layer 1)"
    d = ConvDesc(n=batch, h=info.in_h, w=info.in_w, cin=info.cin, cout=info.cout, ksize=info.ksize, stride=info.stride,
                 in_ld=info.cin, out_ld=info.cout, res_ld=0, dtype=YB_F16, out_fp32=0, leaky=1,
                 upsample2x=info.upsample2x)
    if info.has_bn and info.cin == 32 and lib.yb_conv3x3_halo_supported(C.byref(d)):
        return "conv_halo"
    return "conv_igemm"


def igemm_tiles(info, n, sms):
    """(tiles, k-blocks per tile, waves) of a conv_igemm launch: 128-row tiles, BN / BK as conv_launch picks them."""
    cout_pad = (info.cout + 63) // 64 * 64
    bn = 128 if cout_pad % 128 == 0 else 64
    bk = 64 if info.cin % 64 == 0 else 32
    m = n * info.out_h * info.out_w
    tiles = math.ceil(m / 128) * (cout_pad // bn)
    return tiles, info.ksize * info.ksize * info.cin // bk, math.ceil(tiles / sms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=416)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--json", default=None, help="also write the per-layer rows to FILE")
    args = ap.parse_args()

    import torch
    import yolov3_tensorflow_b200 as pkg
    from yolov3_tensorflow_b200._lib import LayerSchedule, lib, check, ptr, stream_handle
    from bench import make_bench_params

    for key in ("YB_HALO", "YB_THIN", "YB_STEM_FUSE", "YB_HEAD_STREAM"):
        if (lib.yb_get_option(key.encode()) or b""):
            sys.exit(f"layer_times: {key} is set; the kernel labels assume the default dispatch")
    torch.cuda.set_device(0)
    anchors = pkg.parse_anchors(os.path.join(ROOT, "yolov3_tensorflow_b200", "data", "yolo_anchors.txt"))
    model = pkg.yolov3(CLASS_NUM, anchors, dtype="fp16")
    model.set_params(make_bench_params(specs=pkg.yolov3.conv_table(CLASS_NUM)), "HWIO")
    B, S = args.batch, args.size
    x = torch.from_numpy(np.random.default_rng(2).random((B, S, S, 3), dtype=np.float32)).cuda()
    fms = model.forward(x)                     # creates the plan and uploads the weights
    plan = model._last_plan
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def run(i):
        check(lib.yb_net_forward_layers(plan.handle, ptr(x), ptr(fms[0]), ptr(fms[1]), ptr(fms[2]), i, i, stream_handle()),
              "yb_net_forward_layers")

    rows = []
    for i in range(plan.num_layers):
        info = plan.layer_info(i)
        kern = kernel_of(lib, info, B)
        flop = 2.0 * B * info.out_h * info.out_w * info.ksize * info.ksize * info.cin * info.cout
        if i == 1:
            flop += 2.0 * B * S * S * 27 * plan.layer_info(0).cout          # the stem's FLOPs run in this launch
        row = dict(layer=i, cin=info.cin, cout=info.cout, k=info.ksize, s=info.stride, hw=info.out_h,
                   up=info.upsample2x, kernel=kern, gflop=flop / 1e9, ms=0.0, sched="", res="")
        if i > 0:
            sc = LayerSchedule()
            check(lib.yb_net_layer_schedule(plan.handle, i, 0, C.byref(sc)), "yb_net_layer_schedule")
            # shortcut: "ldg" read by the epilogue from global memory, "smem" prefetched into shared memory
            row["res"] = ("smem" if sc.res_smem else "ldg") if sc.residual else ""
            if kern == "conv_igemm":           # the plan's schedule: ping-pong / cooperative, multicast cluster shape,
                row["sched"] = (("pp " if sc.pingpong else "co ") + f"{sc.cluster_m}x{sc.cluster_n}" +   # TMA-store epilogue
                                (" tma" if sc.epi_tma else ""))
        if i > 0:
            for _ in range(3):
                run(i)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                run(i)
            b.record()
            torch.cuda.synchronize()
            row["ms"] = a.elapsed_time(b) / args.reps
        if kern == "conv_igemm":
            row["tiles"], row["kb"], row["waves"] = igemm_tiles(info, B, sms)
        rows.append(row)

    print(f"# card: {card()}   SMs: {sms}   batch {B}, {S}x{S}, fp16, {args.reps} reps per layer")
    print(f"{'L':>3} {'cin':>5} {'cout':>5} {'k':>2} {'s':>2} {'out':>4} {'kernel':<10} {'sched':<10} {'res':<4} {'tiles':>6} {'kb':>4}"
          f" {'waves':>5} {'ms':>8} {'TFLOP/s':>8}")
    for r in rows:
        if r["layer"] == 0:
            continue
        tf = r["gflop"] / r["ms"] if r["ms"] > 0 else 0.0
        print(f"{r['layer']:>3} {r['cin']:>5} {r['cout']:>5} {r['k']:>2} {r['s']:>2} {r['hw']:>4} {r['kernel']:<10}"
              f" {r['sched']:<10} {r['res']:<4} {r.get('tiles', ''):>6} {r.get('kb', ''):>4} {r.get('waves', ''):>5} {r['ms']:8.4f} {tf:8.1f}")
    conv_ms = sum(r["ms"] for r in rows)
    igemm = [r for r in rows if r["kernel"] == "conv_igemm"]
    igemm_ms = sum(r["ms"] for r in igemm)
    gflop = sum(r["gflop"] for r in rows)
    print(f"# sum of layers: {conv_ms:.3f} ms ({gflop / conv_ms:.1f} TFLOP/s); conv_igemm: {igemm_ms:.3f} ms over "
          f"{len(igemm)} layers; conv_halo: {conv_ms - igemm_ms:.3f} ms")

    # shortcut penalty per class: each shortcut layer against the mean of its no-shortcut twins
    def gemm(r):
        return (r["cin"], r["cout"], r["k"], r["hw"], r["kernel"])
    res_rows = [r for r in rows if r["res"]]
    penalty = {}
    for key in sorted({gemm(r) for r in res_rows}, key=lambda g: -g[3]):
        sr = [r for r in res_rows if gemm(r) == key]
        tw = [r for r in rows if not r["res"] and r["layer"] > 1 and gemm(r) == key]   # layer 1 runs the stem too
        s_ms = sum(r["ms"] for r in sr)
        if not tw:
            print(f"# shortcut {key[3]}^2 {key[0]}->{key[1]} k{key[2]} ({key[4]}): layers "
                  f"{[r['layer'] for r in sr]} {s_ms:.3f} ms, no twin")
            continue
        t_ms = sum(r["ms"] for r in tw) / len(tw)
        pen = s_ms - len(sr) * t_ms
        penalty[f"{key[3]}^2 {key[0]}->{key[1]} k{key[2]}"] = pen
        print(f"# shortcut {key[3]}^2 {key[0]}->{key[1]} k{key[2]} ({key[4]}): layers {[r['layer'] for r in sr]} "
              f"mean {s_ms / len(sr):.4f} ms vs twins {[r['layer'] for r in tw]} mean {t_ms:.4f} ms -> "
              f"penalty {pen:.3f} ms")
    print(f"# shortcut penalty summed over the classes with a twin: {sum(penalty.values()):.3f} ms")

    # per-k-block / per-tile split from the two same-tile-count pairs
    fits = {}
    for hw, hi, lo in ((52, 68, (70, 72)), (26, 60, (62, 64))):
        rh, rl = rows[hi], [rows[j] for j in lo]
        assert rh["hw"] == hw and all(r["hw"] == hw and r["tiles"] == rh["tiles"] for r in rl), "layer table changed"
        t_lo = sum(r["ms"] for r in rl) / len(rl)
        c_kb = (rh["ms"] - t_lo) / (rh["waves"] * (rh["kb"] - rl[0]["kb"]))
        c_fix = t_lo / rh["waves"] - rl[0]["kb"] * c_kb
        fits[hw] = (c_kb, c_fix)
        print(f"# {hw}^2 fit: per k-block {c_kb * 1e3:.2f} us, fixed per tile {c_fix * 1e3:.2f} us (per CTA, one wave)")
    fixed = 0.0
    fixed_by_hw = {}
    for r in igemm:
        c_kb, c_fix = fits[52] if r["hw"] >= 52 else fits[26]
        fixed += r["waves"] * c_fix
        fixed_by_hw[r["hw"]] = fixed_by_hw.get(r["hw"], 0.0) + r["waves"] * c_fix
    print("# fixed per-tile cost by resolution (ms): " +
          ", ".join(f"{hw}^2 {v:.3f}" + ("" if hw in fits else " (extrapolated)") for hw, v in sorted(fixed_by_hw.items())))
    print(f"# fixed per-tile cost summed over conv_igemm layers: {fixed:.3f} ms = {100 * fixed / conv_ms:.1f} % of the "
          f"sum of layers.  Only the 52^2 and 26^2 terms are fitted at their own resolution: the 52^2 fit is extrapolated "
          f"to 104^2 / 208^2 and the 26^2 fit to 13^2")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), sms=sms, batch=B, size=S, reps=args.reps, rows=rows,
                           fits={str(k): v for k, v in fits.items()}, fixed_ms=fixed, shortcut_penalty_ms=penalty),
                      f, indent=1)


if __name__ == "__main__":
    main()
