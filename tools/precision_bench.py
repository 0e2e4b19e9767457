"""Throughput of the sync-free pipeline (ACR.fused_forward: backbone + heads + parse + MANO) per model_precision.

    python tools/precision_bench.py [--batches 64,256] [--steps 20] [--warmup 5] [--rounds 3] [--fp32-steps 2]

bf16, fp16 and tf32 run alternating in the same process (``--rounds`` rounds, each precision timed ``--steps`` steps with
CUDA events after ``--warmup`` steps; the median round is reported), then the fp32 validation plan at the first batch
size for the ratio.  Prints the card name and power limit, img/s per precision and batch, and the TF32 plan's per-op
device time (Engine.profile_ops: one serialised pass) grouped as tensor-core convs, the CUDA-core stem, the CUDA-core
attention pooling and the rest.  Needs a GPU; the last line is JSON."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    line = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 and q.stdout.strip() else ""
    return line or torch.cuda.get_device_name()


def time_steps(app, frames, offsets, steps, warmup):
    for _ in range(warmup):
        app.fused_forward(frames, offsets)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        app.fused_forward(frames, offsets)
    e1.record()
    torch.cuda.synchronize()
    return steps * frames.shape[0] / (e0.elapsed_time(e1) / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,256")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--fp32-steps", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("precision_bench needs a CUDA device")
    os.environ.setdefault("ACR_B200_SYNTHETIC_MANO", "1")
    from acr.config import args
    from acr.main import ACR
    from acr_b200 import lib as L
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    sd = synth_state_dict(0, bn_stats=load_bn_calibration(0))
    app = ACR(state_dict=sd, mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
    app.model.max_engines = 8                      # every (precision, batch) plan stays built
    batches = [int(b) for b in a.batches.split(",")]
    g = torch.Generator().manual_seed(0)
    precs = ("bf16", "fp16", "tf32")
    name = card()
    print("card:", name)
    res = {}
    for B in batches:
        frames = torch.randint(0, 256, (B, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
        offsets = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1).cuda()
        runs = {p: [] for p in precs}
        for _ in range(a.rounds):
            for p in precs:
                args().model_precision = p
                runs[p].append(time_steps(app, frames, offsets, a.steps, a.warmup))
        for p in precs:
            res[f"{p}_b{B}"] = statistics.median(runs[p])
            print(f"batch {B:4d} {p}: {res[f'{p}_b{B}']:8.1f} img/s   (rounds: {', '.join(f'{v:.1f}' for v in runs[p])})")
        if B == batches[0]:
            args().model_precision = "fp32"
            res[f"fp32_b{B}"] = time_steps(app, frames, offsets, a.fp32_steps, 1)
            print(f"batch {B:4d} fp32 validation plan: {res[f'fp32_b{B}']:8.2f} img/s; tf32 / fp32 = "
                  f"{res[f'tf32_b{B}'] / res[f'fp32_b{B}']:.1f}x")
            args().model_precision = "tf32"
            eng = app.model.engine(B, frames.device)
            ms = eng.profile_ops(frames)
            groups = {"tensor-core convs": 0.0, "CUDA-core stem": 0.0, "CUDA-core pooling": 0.0, "rest": 0.0}
            for r, t in zip(eng.recs, ms):
                k = r["kind"]
                key = ("tensor-core convs" if k == L.OP_CONV else "CUDA-core stem" if k == L.OP_STEM
                       else "CUDA-core pooling" if k == L.OP_POOL else "rest")
                groups[key] += float(t)
            tot = sum(groups.values())
            print(f"tf32 plan, batch {B}, per-op device time (serialised pass, {tot:.1f} ms):")
            for k, v in groups.items():
                print(f"  {k:20s} {v:9.2f} ms  {100 * v / tot:5.1f} %")
            res["tf32_profile_ms"] = groups
        del frames
    args().model_precision = "bf16"
    print(json.dumps({"card": name, **res}))


if __name__ == "__main__":
    main()
