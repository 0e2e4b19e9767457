#!/usr/bin/env python
"""Per-layer-class table of the conv launch set of one bench step, timed with CUDA events (Engine.profile_ops):
    python tools/conv_layers.py [--batch 256] [--warmup 2] [--passes 5]
    python tools/conv_layers.py --dry-run        shapes, FLOP, bytes and floors only (no GPU needed)
    python tools/conv_layers.py --backbone resnet50   the ResNet-50 trunk's plan (transposed convs are a class of their
                                                      own, k shown as "4T", FLOP by live taps)

Conv launches are grouped by (cin, cout, k, s, H_in, residual).  Per class: launches, device ms (the median of every
launch over the profiled passes, summed), TFLOP/s, algorithmic GB/s (input + output (+ residual) (+ extra terms) once),
the compute floor (FLOP over SMs x 4096 dense bf16 FLOP/clk x the SM clock sampled during the passes), the HBM floor
(algorithmic bytes over --hbm-gbs) and measured time over the larger floor.  `weights KB` is the layer's bf16 weight
tensor (cout x cin x k x k): layers whose packed weights do not fit in shared memory next to the operand stages stream
them (conv_tc_prepare), the others keep them resident.
The card name, power limit and SM clock are read in the same run."""
import argparse
import collections
import os
import subprocess
import sys
import threading

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"))
import numpy as np  # noqa: E402

from acr_b200 import lib as L  # noqa: E402
from acr_b200.engine import Engine  # noqa: E402

FLOP_PER_CLK_SM = 4096   # dense bf16 wgmma, per SM and clock (H100)


def smi(query, index=0):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", str(index)],
                         capture_output=True, text=True, timeout=10).stdout
    return [c.strip() for c in out.strip().split(",")]


class ClockSampler(threading.Thread):
    """SM clock (MHz) sampled every 0.2 s while the profiled passes run."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.mhz, self.done = index, [], threading.Event()

    def run(self):
        while not self.done.is_set():
            try:
                self.mhz.append(float(smi("clocks.sm", self.index)[0]))
            except Exception:   # noqa: BLE001 -- a missed sample only shortens the list
                pass
            self.done.wait(0.2)

    def stop(self):
        self.done.set()
        self.join(timeout=5)
        return float(np.median(self.mhz)) if self.mhz else None


def conv_classes(recs, batch, blocks=(), bottlenecks=()):
    """[(key, [rec indices], GFLOP, algorithmic MB, weights KB, issued GFLOP)] of the conv launches, in plan order of first
    use.  `blocks`: first records of the BasicBlocks that run as one fused launch (csrc/conv_block.cuh), a class of their
    own (k "3+3"): FLOP of both convs, bytes in + out, and the issued FLOP of the fused kernel (conv1 runs two N = 120
    ranges of flat pixels per 16x8 tile, 240 / 128 of its pixels; the x-paired form issues its side taps at full width,
    4/3).
    `bottlenecks`: first records of the Bottlenecks that run as one fused launch (csrc/conv_bottleneck.cuh), a class of
    their own (k "1+3+1", cin = the block input's channels): FLOP of the three convs, bytes in + residual (when it is not
    the input) + out, and the issued FLOP (conv1 runs 4 M blocks of 64 flat rows per 16x8 tile, 2x its pixels)."""
    agg = collections.OrderedDict()
    blocks, bottlenecks = set(blocks), set(bottlenecks)
    for i, r in enumerate(recs):
        if r["kind"] != L.OP_CONV or i - 1 in blocks or i - 1 in bottlenecks or i - 2 in bottlenecks:
            continue
        x, y, at = r["ins"][0], r["out"], r["attrs"]
        if i in bottlenecks:
            r3 = recs[i + 2]
            mid, out, res = y.C, r3["out"], r3["ins"][1]
            key = (x.C, out.C, "1+3+1", 1, x.H, True)
            a = agg.setdefault(key, [[], 0.0, 0.0, 0.0, 0.0])
            a[0] += [i, i + 1, i + 2]
            px = out.H * out.W * batch
            f1, f2, f3 = (2.0 * px * c / 1e9 for c in (mid * x.C, mid * mid * 9, out.C * mid))
            a[1] += f1 + f2 + f3
            a[2] += px * (x.C + out.C + (res.C if res is not x else 0)) * 2 / 1e6
            a[3] = (mid * x.C + mid * mid * 9 + out.C * mid) * 2 / 1024
            a[4] += 2 * f1 + f2 + f3
            continue
        if i in blocks:
            key = (x.C, y.C, "3+3", 1, x.H, True)
            a = agg.setdefault(key, [[], 0.0, 0.0, 0.0, 0.0])
            a[0] += [i, i + 1]
            gflop = 2 * 2.0 * y.H * y.W * y.C * x.C * 9 * batch / 1e9
            a[1] += gflop
            a[2] += batch * (x.H * x.W * x.C + y.H * y.W * y.C) * 2 / 1e6
            a[3] = 2 * y.C * x.C * 9 * 2 / 1024
            a[4] += gflop * (240 / 128 + 1) / 2 * (4 / 3 if x.C == 32 else 1)   # conv1 240 / 128, conv2 exact
            continue
        cin = 109 if "fold_side" in at else (27 if "stem" in at else x.C)   # real input channels of the GEMM
        deconv = bool(at.get("deconv"))
        taps = 4 if deconv else at["k"] ** 2                                  # transposed conv: 2x2 live taps per pixel
        key = (cin, y.C, f"{at['k']}T" if deconv else at["k"], at["s"], x.H, bool(at["residual"]))
        a = agg.setdefault(key, [[], 0.0, 0.0, 0.0, 0.0])
        a[0].append(i)
        a[1] += 2.0 * y.H * y.W * y.C * cin * taps * batch / 1e9
        a[4] = a[1]
        nbytes = batch * (x.H * x.W * x.C * 2 + y.H * y.W * y.C * (4 if y.dtype == "f32" else 2) * (2 if at["residual"] else 1))
        if at.get("extra"):
            nbytes += sum(batch * t.H * t.W * t.C * 2 for t in r["ins"][1:])
        a[2] += nbytes / 1e6
        a[3] = y.C * cin * at["k"] ** 2 * 2 / 1024
    return [(k, *v) for k, v in agg.items()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=2, help="unrecorded profiled passes first")
    ap.add_argument("--passes", type=int, default=5, help="profiled passes; every launch's median is used")
    ap.add_argument("--hbm-gbs", type=float, default=3000.0, help="HBM bandwidth of the floor (GB/s)")
    ap.add_argument("--sm-mhz", type=float, default=None, help="SM clock of the compute floor (default: sampled; 1600 dry)")
    ap.add_argument("--sms", type=int, default=132)
    ap.add_argument("--dry-run", action="store_true", help="no GPU: shapes, FLOP, bytes and floors without times")
    ap.add_argument("--backbone", choices=["hrnet", "resnet50"], default="hrnet", help="trunk of the plan (HRNet-W32 default)")
    args = ap.parse_args()

    ms_op = None
    if args.dry_run:
        eng = Engine(None, args.batch, "cpu", dry_run=True, backbone=args.backbone)
        fuse = os.environ.get("ACR_B200_FUSE_BLOCKS", "1") != "0"
        blocks, bottlenecks = (eng.block_starts, eng.bottleneck_starts) if fuse else ([], [])
        mhz = args.sm_mhz or 1600.0
        print(f"dry run (no GPU): batch {args.batch}, floors at {args.sms} SMs x {mhz:.0f} MHz and {args.hbm_gbs:.0f} GB/s")
    else:
        import torch
        from acr_b200.synth import load_bn_calibration, synth_state_dict
        dev = torch.device("cuda", torch.cuda.current_device())
        name, plimit = smi("name,power.limit", dev.index)[:2]
        if args.backbone == "resnet50":
            from acr_b200.netspec import build_acr_spec
            sd = synth_state_dict(0, spec=build_acr_spec(512, backbone="resnet50"))
        else:
            sd = synth_state_dict(0, bn_stats=load_bn_calibration(0))
        eng = Engine(sd, args.batch, dev, torch.bfloat16, 512, backbone=args.backbone)
        frames = torch.randint(0, 256, (args.batch, 512, 512, 3), generator=torch.Generator().manual_seed(1000),
                               dtype=torch.uint8).to(dev)
        for _ in range(args.warmup):
            eng.profile_ops(frames)
        sampler = ClockSampler(dev.index)
        sampler.start()
        runs = np.stack([eng.profile_ops(frames) for _ in range(args.passes)])
        sampled = sampler.stop()
        ms_op = np.median(runs, axis=0)
        launch = eng.launch_of_rec()
        blocks = [i for i in eng.block_starts if launch[i] == launch[i + 1]]
        bottlenecks = [i for i in eng.bottleneck_starts if launch[i] == launch[i + 2]]
        mhz = args.sm_mhz or sampled or 1600.0
        print(f"{name}, power limit {plimit} W, SM clock {sampled if sampled else 'n/a'} MHz (median during the passes); "
              f"batch {args.batch}, median of {args.passes} passes after {args.warmup} warm-up; "
              f"floors at {args.sms} SMs x {mhz:.0f} MHz and {args.hbm_gbs:.0f} GB/s")

    peak_tflops = args.sms * FLOP_PER_CLK_SM * mhz * 1e6 / 1e12
    rows = []
    for key, idx, gflop, mb, wkb, issued in conv_classes(eng.recs, args.batch, blocks, bottlenecks):
        t_c, t_m = issued / peak_tflops, mb / args.hbm_gbs       # ms (compute floor: the FLOP the kernel issues)
        ms = float(ms_op[idx].sum()) if ms_op is not None else None
        rows.append((key, len(idx) // {"3+3": 2, "1+3+1": 3}.get(key[2], 1), wkb, gflop, mb, t_c, t_m, ms))   # launches
    rows.sort(key=lambda r: -(r[7] if r[7] is not None else max(r[5], r[6])))
    head = "| cin | cout | k | s | H_in | res | n | weights KB | GFLOP | MB | compute floor ms | HBM floor ms | bound |"
    if ms_op is not None:
        head += " ms | TFLOP/s | GB/s | x floor |"
    print(head + "\n" + "|" + "---:|" * 5 + "---|" + "---:|" * 6 + "---|" + ("---:|" * 4 if ms_op is not None else ""))
    for key, n, wkb, gflop, mb, t_c, t_m, ms in rows:
        line = (f"| {key[0]} | {key[1]} | {key[2]} | {key[3]} | {key[4]} | {'y' if key[5] else ''} | {n} | {wkb:.0f} | "
                f"{gflop:.1f} | {mb:.0f} | {t_c:.2f} | {t_m:.2f} | {'compute' if t_c >= t_m else 'HBM'} |")
        if ms is not None:
            line += f" {ms:.2f} | {gflop / ms:.0f} | {mb / ms:.0f} | {ms / max(t_c, t_m):.1f} |"
        print(line)
    tc, tm = sum(r[5] for r in rows), sum(r[6] for r in rows)
    tf = sum(max(r[5], r[6]) for r in rows)
    tail = (f"\n{sum(r[1] for r in rows)} conv launches ({len(blocks)} fused blocks, {len(bottlenecks)} fused Bottlenecks), {sum(r[3] for r in rows):.0f} GFLOP, {sum(r[4] for r in rows) / 1e3:.1f} GB; "
            f"floors: compute {tc:.1f} ms, HBM {tm:.1f} ms, sum of per-class max {tf:.1f} ms")
    if ms_op is not None:
        t = sum(r[7] for r in rows)
        tail += f"; measured {t:.2f} ms ({sum(r[3] for r in rows) / t:.0f} TFLOP/s, {t / tf:.1f}x the floor)"
    print(tail)


if __name__ == "__main__":
    main()
