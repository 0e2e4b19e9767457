"""Device JPEG decode (acr_b200.jpeg) against cv2.imdecode on N host threads, and end to end from JPEG bytes to meshes.

    python tools/jpeg_bench.py [--batch 64] [--threads 1,8] [--reps 5] [--e2e-batch 16] [--json out.json]

Part 1: img/s of one decode launch sequence over a batch of `batch` distinct seeded files (cv2.imencode of smooth
frames with noise, quality 90), per size (720p, 1080p), sampling (4:2:0, 4:2:2, 4:4:0, 4:4:4) and restart interval
(none, 4 MCUs).  The device time is CUDA events around `reps` launches of a loaded JpegBatch (the H2D copy of the
coded bytes is not included); cv2 is a thread pool over the same files.
Part 2: img/s of capture_jpeg_graph replays (the H2D copy of coded bytes included) against capture_frames_graph
replays fed by cv2 decoding on the host threads, 1080p 4:2:0.  Prints the GPU name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path[:0] = [os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT]

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from acr_b200 import jpeg  # noqa: E402

SIZES = {"720p": (720, 1280), "1080p": (1080, 1920)}
SAMPLINGS = ["420", "422", "440", "444"]


def files(h, w, sampling, rst, n, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w].astype(np.float32)
    out = []
    for i in range(n):
        base = np.stack([128 + 100 * np.sin(xx / w * (3 + i % 5) + yy / h), 128 + 90 * np.cos(yy / h * (4 + i % 3)),
                         (xx + yy) * 255 / (w + h)], 2)
        img = np.clip(base + rng.normal(0, 6, base.shape), 0, 255).astype(np.uint8)
        p = [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
             getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{sampling}")]
        if rst:
            p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
        out.append(cv2.imencode(".jpg", img, p)[1].tobytes())
    return out


def cv2_rate(bufs, threads, reps):
    dec = lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(dec, bufs))
        t = time.perf_counter()
        for _ in range(reps):
            list(ex.map(dec, bufs))
        return reps * len(bufs) / (time.perf_counter() - t)


def device_rate(bufs, reps):
    lay, _ = jpeg.plan(bufs)
    jb = jpeg.JpegBatch(len(bufs), lay.coded_bytes, lay.out_bytes, lay.chunks, lay.blocks)
    jb.load(bufs, lay)
    jb.launch()
    jb.raise_on_status()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        jb.launch()
    e1.record()
    torch.cuda.synchronize()
    return reps * len(bufs) / (e0.elapsed_time(e1) / 1e3)


def e2e(batch, threads, reps):
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)), mano_assets=assets)
    bufs = files(1080, 1920, "420", 0, batch, seed=1)
    coded = sum(jpeg.parse(b).scan_len for b in bufs)
    fb = batch * 1080 * 1920 * 3
    rj = app.capture_jpeg_graph(batch, coded, fb)
    rf = app.capture_frames_graph(batch, fb)
    dec = lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    res = {}
    with ThreadPoolExecutor(threads) as ex:
        for name, step in (("capture_jpeg_graph", lambda: rj(bufs)),
                           ("capture_frames_graph + cv2", lambda: rf(list(ex.map(dec, bufs))))):
            step()
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(reps):
                step()
            torch.cuda.synchronize()
            res[name] = reps * batch / (time.perf_counter() - t)
    rj.jpeg.raise_on_status()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--threads", default="1,8")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--e2e-batch", type=int, default=16)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("jpeg_bench needs a GPU")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"# {gpu}; host threads {os.cpu_count()}")
    threads = [int(t) for t in a.threads.split(",")]
    rows = []
    print("| size | sampling | RST | device img/s | " + " | ".join(f"cv2 x{t} img/s" for t in threads) + " |")
    for sname, (h, w) in SIZES.items():
        for s in SAMPLINGS:
            for rst in (0, 4):
                bufs = files(h, w, s, rst, a.batch)
                dev = device_rate(bufs, a.reps)
                host = [cv2_rate(bufs, t, max(1, a.reps // 2)) for t in threads]
                rows.append(dict(size=sname, sampling=s, rst=rst, device=dev, cv2={t: r for t, r in zip(threads, host)}))
                print(f"| {sname} | {s} | {rst or '-'} | {dev:.0f} | " + " | ".join(f"{r:.0f}" for r in host) + " |",
                      flush=True)
    e = e2e(a.e2e_batch, max(threads), a.reps)
    for k, v in e.items():
        print(f"end to end 1080p 4:2:0 batch {a.e2e_batch}: {k}: {v:.1f} img/s")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows, e2e=e), f, indent=1)


if __name__ == "__main__":
    main()
