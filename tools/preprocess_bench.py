#!/usr/bin/env python
"""Ragged pre-processing timing (BGR -> RGB, white pad, bicubic 512 x 512), for a folder-like mix of frame sizes:
  ragged_kernel_us    RaggedFrames.launch on frames already packed on the device: acr_b200_cubic_tables +
                      acr_b200_preprocess_ragged, CUDA events
  ragged_cuda_us      preprocess_frames(list of CUDA frames): the torch.cat packing, descriptors H2D, both kernels
  bucket_loop_us      today's alternative: one preprocess_frames launch per distinct (H, W), on 4-D CUDA tensors
                      stacked beforehand (the stacking is not timed)
  ragged_host_us      preprocess_frames(list of numpy frames): pinned staging, one H2D copy, both kernels; host
                      clock to a device synchronise
  host_cv2_us         the reference's host path per frame, as oracle/preprocess_ref.img_preprocess pads it, with
                      cv2.resize(INTER_CUBIC); host clock, not measured without cv2
and the batch-1 latency of one raw camera frame (numpy, host) to meshes, host clock to a device synchronise:
  frames_graph_b1_us  one replay of ACR.capture_frames_graph(1, ...)
  graph_b1_eager_resize_us  H2D + the 4-D preprocess_frames + one replay of ACR.capture_graph(1)
The card's name, power limit and SM clock are read in the same run.
    python tools/preprocess_bench.py [--frames 48] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from acr_b200.preprocess import RaggedFrames, preprocess_frames  # noqa: E402

# phone photos (portrait / landscape), screenshots, webcam and video frames
SIZES = [(3024, 4032), (4032, 3024), (2532, 1170), (1170, 2532), (1080, 1920), (1920, 1080), (720, 1280),
         (1280, 720), (480, 640), (600, 800), (1080, 1080), (2160, 3840)]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().split(",")])) if r.returncode == 0 else {}


def events(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def wall(fn, iters, warmup=3):
    """Mean latency of fn() up to a device synchronise, us."""
    for _ in range(warmup):
        fn()
        torch.cuda.synchronize()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return float(np.mean(t)) * 1e6


def frames_mix(n, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, SIZES[i % len(SIZES)] + (3,), dtype=np.uint8) for i in range(n)]


def host_cv2(frames):
    import cv2
    from oracle import preprocess_ref
    t0 = time.perf_counter()
    for f in frames:
        rgb = f[:, :, ::-1]
        h, w = rgb.shape[:2]
        t, r, b, l = preprocess_ref.paddings_to_square(h, w)
        padded = np.full((h + t + b, w + l + r, 3), 255, np.uint8)
        padded[t:t + h, l:l + w] = rgb
        cv2.resize(padded, (512, 512), interpolation=cv2.INTER_CUBIC)
    return (time.perf_counter() - t0) * 1e6


def batch_rows(n, iters):
    host = frames_mix(n)
    dev = [torch.from_numpy(f).cuda() for f in host]
    total = sum(f.size for f in host)
    rf = RaggedFrames(n, total)
    rf.load(dev)
    buckets = {}
    for i, f in enumerate(dev):
        buckets.setdefault(tuple(f.shape), []).append(i)
    stacked = [torch.stack([dev[i] for i in v]) for v in buckets.values()]
    ragged, _ = preprocess_frames(dev)
    bucket_out = torch.cat([preprocess_frames(s)[0] for s in stacked])
    order = [i for v in buckets.values() for i in v]
    assert torch.equal(ragged[order], bucket_out), "ragged and bucketed outputs differ"
    row = {"frames": n, "distinct_sizes": len(buckets), "megapixels": round(total / 3e6, 1)}
    res = {k: [] for k in ("ragged_kernel_us", "ragged_cuda_us", "bucket_loop_us")}
    for _ in range(3):     # alternate the arms
        res["ragged_kernel_us"].append(events(rf.launch, iters))
        res["ragged_cuda_us"].append(events(lambda: preprocess_frames(dev), iters))
        res["bucket_loop_us"].append(events(lambda: [preprocess_frames(s) for s in stacked], iters))
    row |= {k: [round(v, 1) for v in vs] for k, vs in res.items()}
    row["ragged_host_us"] = round(wall(lambda: preprocess_frames(host), max(3, iters // 4)), 1)
    try:
        row["host_cv2_us"] = round(min(host_cv2(host) for _ in range(2)), 1)
    except ImportError:
        row["host_cv2_us"] = "not measured (no cv2)"
    return row


def graph_rows(iters):
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)),
              mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
    g_old = app.capture_graph(1)
    rows = []
    for hw in ((720, 1280), (1080, 1920)):
        frame = np.random.default_rng(hw[0]).integers(0, 256, hw + (3,), dtype=np.uint8)
        g_new = app.capture_frames_graph(1, frame.size)

        def old():
            img, offs = preprocess_frames(torch.from_numpy(frame)[None].cuda(non_blocking=True))
            return g_old(img, offs)

        res = {"frames_graph_b1_us": [], "graph_b1_eager_resize_us": []}
        for _ in range(3):
            res["frames_graph_b1_us"].append(wall(lambda: g_new([frame]), iters))
            res["graph_b1_eager_resize_us"].append(wall(old, iters))
        rows.append({"frame": list(hw)} | {k: [round(v, 1) for v in vs] for k, vs in res.items()})
        del g_new
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="12,48")
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"gpu": gpu_info()}))
    for n in (int(v) for v in a.frames.split(",")):
        print(json.dumps(batch_rows(n, a.iters)))
    for row in graph_rows(max(20, a.iters)):
        print(json.dumps(row))
    print(json.dumps({"gpu_after": gpu_info()}))


if __name__ == "__main__":
    main()
