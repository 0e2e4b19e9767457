#!/usr/bin/env python
"""MANO backward timing, CUDA events after warm-up, one side, centre joint 9, cotangents on verts / joints / centre:
  forward       acr_b200_mano_forward alone (ops.mano_forward)
  backward      acr_b200_mano_backward alone (both kernels, ops.mano_backward)
  layer f+b     ManoLayer forward + loss.backward() through autograd
  torch f+b     the same loop through an fp32 torch restatement of the reference layer (tests/mano_torch_ref.py) on
                the same GPU: the reference's own path, the baseline
ns/hand and GB/s against the backward's compulsory traffic of 10 064 B/hand (read dverts 9 336 + djoints 252 +
dcenter 12 + poses/betas 232, write dposes/dbetas 232).
    python tools/mano_grad_bench.py [--hands 512,8192,65536] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT):
    sys.path.insert(0, p)
import torch  # noqa: E402

from acr_b200 import ops  # noqa: E402
from acr_b200.synth import make_synthetic_mano  # noqa: E402
from mano.manolayer import ManoLayer  # noqa: E402
from tests.mano_torch_ref import TorchMano  # noqa: E402

BWD_BYTES = 9336 + 252 + 12 + 232 + 232


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3   # us per call


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().split(",")])) if r.returncode == 0 else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hands", default="512,8192,65536")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    asset = make_synthetic_mano("right")
    layer = ManoLayer(center_idx=9, flat_hand_mean=False, ncomps=45, side="right", use_pca=False, asset=asset).cuda()
    model = layer.packed_model()
    ref = TorchMano(asset, "right", use_pca=False, flat_hand_mean=False, center_idx=9, dtype=torch.float32, device="cuda")
    print(json.dumps({"gpu": gpu_info()}))
    for n in (int(v) for v in args.hands.split(",")):
        g = torch.Generator().manual_seed(0)
        pose = (torch.randn(n, 48, generator=g) * 0.5).cuda()
        betas = torch.randn(n, 10, generator=g).cuda()
        gv, gj, gc = (torch.randn(n, 778, 3, generator=g).cuda(), torch.randn(n, 21, 3, generator=g).cuda(),
                      torch.randn(n, 1, 3, generator=g).cuda())

        def layer_step(fn):
            p, b = pose.clone().requires_grad_(), betas.clone().requires_grad_()
            v, j, c = fn(p, b)
            ((gv * v).sum() + (gj * j).sum() + (gc * c).sum()).backward()

        row = {"hands": n}
        row["forward_us"] = timed(lambda: ops.mano_forward(None, model, pose, betas, None, 1, 9), args.iters)
        row["backward_us"] = timed(lambda: ops.mano_backward(model, 1, pose, betas, 9, gv, gj, gc), args.iters)
        row["layer_fb_us"] = timed(lambda: layer_step(lambda p, b: layer(p, th_betas=b)), args.iters)
        row["torch_fb_us"] = timed(lambda: layer_step(lambda p, b: ref(p, b)), max(3, args.iters // 4), warmup=2)
        for k in ("forward", "backward", "layer_fb", "torch_fb"):
            row[k + "_ns_per_hand"] = round(row[k + "_us"] * 1e3 / n, 2)
            row[k + "_us"] = round(row[k + "_us"], 1)
        row["backward_GBs"] = round(n * BWD_BYTES / (row["backward_us"] * 1e3), 1)
        row["layer_vs_torch_speedup"] = round(row["torch_fb_us"] / row["layer_fb_us"], 2)
        print(json.dumps(row))
        del gv, gj, gc
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
