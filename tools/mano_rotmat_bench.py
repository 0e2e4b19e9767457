#!/usr/bin/env python
"""ManoLayer rotation-matrix mode timing, CUDA events after warm-up, one side, centre joint 9, cotangents on verts /
joints / centre, ns/hand for
  fwd / bwd         acr_b200_mano_layer_forward / _backward alone (ops.mano_layer_*), rotation matrices and, for
                    comparison, axis angles (the latter are exactly acr_b200_mano_forward / _backward)
  torch fwd / f+b   the fp32 torch restatement (tests/mano_rotmat_ref.py) on the same GPU: batched torch.linalg.svd
                    for the projection, autograd for the backward (the closed-form projection VJP)
The card's name, power limit and SM clock are read in the same run.
    python tools/mano_rotmat_bench.py [--hands 512,8192,65536] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT):
    sys.path.insert(0, p)
import torch  # noqa: E402

from acr_b200 import lib as L  # noqa: E402
from acr_b200 import ops  # noqa: E402
from acr_b200.synth import make_synthetic_mano  # noqa: E402
from mano.manolayer import ManoLayer  # noqa: E402
from tests.mano_rotmat_ref import TorchManoRot  # noqa: E402
from tests.mano_torch_ref import rodrigues  # noqa: E402


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
    model = ManoLayer(use_pca=False, joint_rot_mode="rotmat", side="right", asset=asset).cuda().packed_model()
    ref = TorchManoRot(asset, "right", use_pca=False, center_idx=9, dtype=torch.float32, device="cuda")
    print(json.dumps({"gpu": gpu_info()}))
    for n in (int(v) for v in args.hands.split(",")):
        g = torch.Generator().manual_seed(0)
        aa = torch.randn(n, 48, generator=g) * 0.5
        mats = (rodrigues(aa.reshape(-1, 3)).view(n, 16, 3, 3) + 0.05 * torch.randn(n, 16, 3, 3, generator=g)).cuda()
        aa, betas = aa.cuda(), torch.randn(n, 10, generator=g).cuda()
        gv, gj, gc = (torch.randn(n, 778, 3, generator=g).cuda(), torch.randn(n, 21, 3, generator=g).cuda(),
                      torch.randn(n, 1, 3, generator=g).cuda())

        def torch_fb():
            p, b = mats.clone().requires_grad_(), betas.clone().requires_grad_()
            v, j, c = ref.from_rotmats(p, b)
            ((gv * v).sum() + (gj * j).sum() + (gc * c).sum()).backward()

        row = {"hands": n}
        for name, pose, mode in (("rotmat", mats, L.POSE_ROTMAT), ("axisang", aa, L.POSE_AXISANG)):
            row[name + "_fwd"] = timed(lambda: ops.mano_layer_forward(model, 1, pose, mode, betas, 9, False), args.iters)
            row[name + "_bwd"] = timed(lambda: ops.mano_layer_backward(model, 1, pose, mode, betas, 9, False, gv, gj, gc),
                                       args.iters)
        few = max(3, args.iters // 4)
        with torch.no_grad():
            row["torch_fwd"] = timed(lambda: ref.from_rotmats(mats, betas), few, warmup=2)
        row["torch_fb"] = timed(torch_fb, few, warmup=2)
        out = {"hands": n}
        for k, us in row.items():
            if k != "hands":
                out[k + "_ns_per_hand"] = round(us * 1e3 / n, 2)
        out["rotmat_fb_vs_torch_fb"] = round(row["torch_fb"] / (row["rotmat_fwd"] + row["rotmat_bwd"]), 1)
        print(json.dumps(out))
        del gv, gj, gc
        torch.cuda.empty_cache()
    print(json.dumps({"gpu_after": gpu_info()}))


if __name__ == "__main__":
    main()
