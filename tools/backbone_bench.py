#!/usr/bin/env python
"""Throughput of the sync-free pipeline (acr.main.ACR.fused_forward: trunk -> heads -> parse -> MANO, no host sync) for
the ResNet-50 and HRNet-W32 trunks, alternating trunks in one process so both see the same card state:
    python tools/backbone_bench.py [--steps 10] [--warmup 3] [--repeats 3]
Runs batch 64 fp16 (BASELINE configs 1-2 shape) and batch 256 bf16.  Per (config, trunk): images/s and ms per step (the
median over the repeats of CUDA-event time over --steps steps), conv ms per step (one separate serialised,
event-bracketed pass: the sum of the conv launches), GFLOP per image (conv_flops_per_image).  The card name, power
limit and the median SM clock sampled during the timed steps are printed with every line.  Synthetic seeded weights
and MANO models; nothing is written."""
import argparse
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from conv_layers import ClockSampler, smi  # noqa: E402

CONFIGS = [(64, "fp16"), (256, "bf16")]
TRUNKS = [("resnet50", "resnet"), ("hrnet_w32", "hrnet")]


def make_app(backbone_flag):
    from acr.config import ConfigContext, parse_args
    from acr.main import ACR
    from acr_b200.netspec import build_acr_spec
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    ConfigContext(parse_args(["--backbone", backbone_flag]))
    if backbone_flag == "resnet":
        sd = synth_state_dict(0, spec=build_acr_spec(512, backbone="resnet50"))
    else:
        sd = synth_state_dict(0, bn_stats=load_bn_calibration(0))
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    return ACR(state_dict=sd, mano_assets=assets)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3, help="alternating rounds over the trunks; the median is printed")
    args = ap.parse_args()
    from acr.config import ConfigContext, parse_args
    from acr_b200 import lib as L
    dev = torch.device("cuda", torch.cuda.current_device())
    name, plimit = smi("name,power.limit", dev.index)[:2]
    apps = {t: make_app(flag) for t, flag in TRUNKS}
    flags = dict(TRUNKS)
    for batch, prec in CONFIGS:
        frames = torch.randint(0, 256, (batch, 512, 512, 3), generator=torch.Generator().manual_seed(1000),
                               dtype=torch.uint8).to(dev)
        offsets = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(batch, 1).to(dev)
        res = {t: [] for t in apps}
        clocks = {t: [] for t in apps}
        for _ in range(args.repeats):
            for t, app in apps.items():
                ConfigContext(parse_args(["--backbone", flags[t], "--model_precision", prec]))
                for _ in range(args.warmup):
                    app.fused_forward(frames, offsets)
                torch.cuda.synchronize(dev)
                sampler = ClockSampler(dev.index)
                sampler.start()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    app.fused_forward(frames, offsets)
                e1.record()
                torch.cuda.synchronize(dev)
                clocks[t].append(sampler.stop())
                res[t].append(e0.elapsed_time(e1) / args.steps)
        for t, app in apps.items():
            ConfigContext(parse_args(["--backbone", flags[t], "--model_precision", prec]))
            eng = app.model.engine(batch, dev)
            ms_op = eng.profile_ops(frames)
            conv_ms = float(sum(ms_op[i] for i, r in enumerate(eng.recs) if r["kind"] == L.OP_CONV))
            ms = float(np.median(res[t]))
            mhz = [c for c in clocks[t] if c]
            print(f"{t:9s} batch {batch:3d} {prec}: {batch / ms * 1e3:8.1f} images/s, {ms:7.2f} ms/step "
                  f"(repeats {', '.join(f'{x:.2f}' for x in res[t])}), conv {conv_ms:6.2f} ms, "
                  f"{eng.flops_per_image / 1e9:6.2f} GFLOP/img; {name}, power limit {plimit} W, "
                  f"SM clock {np.median(mhz) if mhz else 'n/a'} MHz", flush=True)
    ConfigContext(parse_args([]))


if __name__ == "__main__":
    main()
