#!/usr/bin/env python
"""Camera-translation timing: CUDA events after warm-up, us per call, for
  lstsq / pnp        acr_b200_cam_trans / acr_b200_cam_trans_pnp on (j3d, pj2d) of synthetic MANO hands (clean, and at
                     the middle size also half of them with 1-8 joints moved 30-150 px)
  graph_b1_*         one replay of ACR.capture_graph(1) (the whole batch-1 pipeline) with cam_trans_mode 'lstsq' / 'pnp',
                     the two graphs alternated
  cpu_cv2_loop       the reference's host loop (estimate_translation: one cv2.solvePnPRansac per hand) at the middle
                     size, the host clock, without the device-to-host copy it needs first
The card's name, power limit and SM clock are read in the same run.
    python tools/cam_trans_bench.py [--hands 2,512,8192] [--iters 50]"""
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

from acr_b200 import ops  # noqa: E402
from acr_b200.synth import make_synthetic_mano  # noqa: E402
from oracle import mano_ref  # noqa: E402


def timed(fn, iters, warmup=5):
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


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().split(",")])) if r.returncode == 0 else {}


def hands(n, outliers, seed=0):
    rng = np.random.default_rng(seed)
    assets = {s: make_synthetic_mano(s) for s in ("left", "right")}
    poses = (0.5 * rng.standard_normal((n, 48))).astype(np.float32)
    betas = rng.standard_normal((n, 10)).astype(np.float32)
    cam = np.stack([rng.uniform(0.3, 3.0, n), rng.uniform(-.6, .6, n), rng.uniform(-.6, .6, n)], 1).astype(np.float32)
    out = mano_ref.mano_wrapper_forward(assets, poses, betas, n // 2, n - n // 2, cam)
    j3d, pj2d = out["j3d"].astype(np.float32), out["pj2d"].astype(np.float32)
    if outliers:
        for i in range(1, n, 2):
            k = rng.integers(1, 9)
            idx = rng.choice(21, k, replace=False)
            pj2d[i, idx] += (rng.uniform(30, 150, (k, 2)) * rng.choice([-1, 1], (k, 2)) / 256).astype(np.float32)
    return j3d, pj2d


def cpu_cv2_loop(j3d, pj2d, focal=1265.0):
    import cv2
    K = np.eye(3)
    K[0, 0] = K[1, 1] = focal
    K[:2, 2] = 256
    j2d = ((pj2d + 1) * 256).astype(np.float32)
    t0 = time.perf_counter()
    for i in range(j3d.shape[0]):
        m = (j2d[i, :, 1] > -2.) & (j3d[i, :, 2] != -2.)
        cv2.solvePnPRansac(j3d[i][m], j2d[i][m], K, None, flags=cv2.SOLVEPNP_EPNP, reprojectionError=20,
                           iterationsCount=100)
    return (time.perf_counter() - t0) * 1e6


def graph_latency(iters):
    from acr.config import args
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    sd = synth_state_dict(0, bn_stats=load_bn_calibration(0))
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    frame = torch.randint(0, 256, (1, 512, 512, 3), generator=torch.Generator().manual_seed(77), dtype=torch.uint8).cuda()
    offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).cuda()
    old, apps, replays = args().cam_trans_mode, [], {}
    try:
        for mode in ("lstsq", "pnp"):
            args().cam_trans_mode = mode
            apps.append(ACR(state_dict=sd, mano_assets=assets))   # a graph replays into its app's buffers: keep it
            replays[mode] = apps[-1].capture_graph(1)
    finally:
        args().cam_trans_mode = old
    res = {m: [] for m in replays}
    for _ in range(5):   # alternate the two graphs
        for m, r in replays.items():
            res[m].append(timed(lambda: r(frame, offs), iters))
    bufs, _ = replays["pnp"](frame, offs)
    torch.cuda.synchronize()
    return {f"graph_b1_{m}_us": [round(v, 1) for v in vs] for m, vs in res.items()} | {"graph_b1_hands": int(bufs.counts[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hands", default="2,512,8192")
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"gpu": gpu_info()}))
    sizes = [int(v) for v in a.hands.split(",")]
    mid = sizes[len(sizes) // 2]
    for n in sizes:
        for outl in ((False, True) if n == mid else (False,)):
            j3d, pj2d = hands(n, outl)
            J, P = torch.from_numpy(j3d).cuda(), torch.from_numpy(pj2d).cuda()
            row = {"hands": n, "outliers": outl,
                   "lstsq_us": round(timed(lambda: ops.cam_trans(J, P), a.iters), 2),
                   "pnp_us": round(timed(lambda: ops.cam_trans_pnp(J, P), a.iters), 2)}
            if n == mid:
                try:
                    row["cpu_cv2_loop_us"] = round(cpu_cv2_loop(j3d, pj2d), 1)
                except ImportError:
                    row["cpu_cv2_loop_us"] = "not measured (no cv2)"
            print(json.dumps(row))
    print(json.dumps(graph_latency(max(10, a.iters // 2))))
    print(json.dumps({"gpu_after": gpu_info()}))


if __name__ == "__main__":
    main()
