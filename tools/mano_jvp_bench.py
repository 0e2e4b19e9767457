#!/usr/bin/env python
"""ManoLayer Jacobian timing, CUDA events after warm-up, one side (axis angles, centre joint 9), ms per Jacobian of
all hands.  The per-hand joint Jacobian (63 x 58: 21 joints x 3 by 48 pose values + 10 betas, ``vmap`` over hands)
at each --hands size, four ways:
  fused_jacfwd      torch.func.vmap(jacfwd(layer)): the fused JVP kernel, 58 tangents per hand in one launch
  fused_joints_jvp  ops.mano_layer_jvp with the 58 basis tangents and no vertex output: the kernel's joints-only form
  fused_jacrev      torch.func.vmap(jacrev(layer)): the fused backward kernels, 63 cotangent rows per hand
  torch_jacfwd      torch.func.vmap(jacfwd(...)) of the fp32 torch restatement (tests/mano_torch_ref.TorchMano)
and the full vertex Jacobian (2334 x 58 per hand) at --vert-hands, fused and torch.  The card's name, power limit and
SM clock are read in the same run.  A torch arm that runs out of memory is reported as "oom".
    python tools/mano_jvp_bench.py [--hands 512,8192] [--vert-hands 512] [--iters 10]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT):
    sys.path.insert(0, p)
import torch  # noqa: E402
from torch.func import jacfwd, jacrev, vmap  # noqa: E402

from acr_b200 import lib as L  # noqa: E402
from acr_b200 import ops  # noqa: E402
from acr_b200.synth import make_synthetic_mano  # noqa: E402
from mano.manolayer import ManoLayer  # noqa: E402
from tests.mano_torch_ref import TorchMano  # noqa: E402


def timed(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / iters, 3)   # ms per call


def timed_or_oom(fn, iters):
    try:
        return timed(fn, iters)
    except torch.OutOfMemoryError:
        torch.cuda.empty_cache()
        return "oom"


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().split(",")])) if r.returncode == 0 else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hands", default="512,8192")
    ap.add_argument("--vert-hands", default="512")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    asset = make_synthetic_mano("right")
    layer = ManoLayer(center_idx=9, use_pca=False, flat_hand_mean=False, side="right", asset=asset).cuda()
    ref = TorchMano(asset, "right", use_pca=False, flat_hand_mean=False, center_idx=9, dtype=torch.float32,
                    device="cuda")
    model = layer.packed_model()
    print(json.dumps({"gpu": gpu_info()}))

    def per_hand(fn, out):
        return lambda p, b: fn(p[None], b[None])[out][0]
    fused = lambda p, b: layer(p, th_betas=b)
    plain = lambda p, b: ref(p, b)

    def inputs(n):
        g = torch.Generator().manual_seed(0)
        return (torch.randn(n, 48, generator=g) * 0.5).cuda(), torch.randn(n, 10, generator=g).cuda()

    for n in (int(v) for v in args.hands.split(",")):
        pose, betas = inputs(n)
        eye = torch.eye(58, device="cuda")
        tp = eye[:, :48, None].expand(58, 48, n).permute(0, 2, 1).contiguous()     # (58, n, 48) basis tangents
        tb = eye[:, 48:, None].expand(58, 10, n).permute(0, 2, 1).contiguous()     # (58, n, 10)
        row = {"hands": n, "jacobian": "joints 63x58 per hand"}
        row["fused_jacfwd_ms"] = timed(lambda: vmap(jacfwd(per_hand(fused, 1), argnums=(0, 1)))(pose, betas), args.iters)
        row["fused_joints_jvp_ms"] = timed(lambda: ops.mano_layer_jvp(model, 1, pose, L.POSE_AXISANG, betas, 9, False,
                                                                      tp, tb, want_verts=False), args.iters)
        row["fused_jacrev_ms"] = timed_or_oom(lambda: vmap(jacrev(per_hand(fused, 1), argnums=(0, 1)))(pose, betas),
                                              args.iters)
        row["torch_jacfwd_ms"] = timed_or_oom(lambda: vmap(jacfwd(per_hand(plain, 1), argnums=(0, 1)))(pose, betas),
                                              max(2, args.iters // 2))
        # the same Jacobian, three ways
        with torch.no_grad():
            a = vmap(jacfwd(per_hand(fused, 1), argnums=(0, 1)))(pose, betas)
            _, tj, _ = ops.mano_layer_jvp(model, 1, pose, L.POSE_AXISANG, betas, 9, False, tp, tb, want_verts=False)
            b = torch.cat(a, -1).permute(3, 0, 1, 2)        # (58, n, 21, 3)
            row["joints_only_vs_jacfwd_max_abs"] = float((tj - b).abs().max())
        print(json.dumps(row))
        torch.cuda.empty_cache()
    for n in (int(v) for v in args.vert_hands.split(",")):
        pose, betas = inputs(n)
        row = {"hands": n, "jacobian": "vertices 2334x58 per hand"}
        row["fused_jacfwd_ms"] = timed(lambda: vmap(jacfwd(per_hand(fused, 0), argnums=(0, 1)))(pose, betas), args.iters)
        row["torch_jacfwd_ms"] = timed_or_oom(lambda: vmap(jacfwd(per_hand(plain, 0), argnums=(0, 1)))(pose, betas),
                                              max(2, args.iters // 2))
        print(json.dumps(row))
        torch.cuda.empty_cache()
    print(json.dumps({"gpu_after": gpu_info()}))


if __name__ == "__main__":
    main()
