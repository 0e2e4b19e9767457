"""Device decode of progressive JPEG files (acr_b200.jpeg, ``max_scans``) against cv2.imdecode on N host threads.

    python tools/jpeg_progressive_bench.py [--batch 32] [--threads 1,8] [--reps 5] [--graph-batch 16]

1. img/s of one decode launch sequence over `batch` distinct progressive files (cv2's default script, quality 90,
   smooth frames with noise as in tools/jpeg_bench.py), 720p and 1080p, 4:2:0 and 4:4:4, without and with RST every
   4 MCUs; the device figure is the range over three timed runs of `reps` launches each (CUDA events, the H2D copy
   not included); cv2 is a thread pool over the same files.
2. batch-1 latency of one 1080p 4:2:0 progressive file, and the share of it spent in jpeg_refine_kernel (the
   refinement scans: serial walk and parallel decode), from torch.profiler's kernel times.
3. a baseline-only batch (1080p 4:2:0) decoded by buffers without scan capacity and by buffers with max_scans = 64
   (the launches a graph captured for progressive files runs), alternating.
4. img/s of capture_jpeg_graph(max_scans=...) replays at batch `graph-batch` from progressive 1080p 4:2:0 files.
Prints the GPU name and power limit with the numbers."""
import argparse
import os
import re
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path[:0] = [os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT, os.path.join(ROOT, "tools")]

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from acr_b200 import jpeg  # noqa: E402
from jpeg_bench import cv2_rate, files  # noqa: E402

SIZES = {"720p": (720, 1280), "1080p": (1080, 1920)}
MAX_SCANS = 64


def progressive(bufs):
    """The same frames coded again by cv2 as progressive files (cv2's default script)."""
    out = []
    for b in bufs:
        img = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
        info = jpeg.parse(b)
        s = {(1, 1): "444", (2, 2): "420"}[(info.hmax, info.vmax)]
        p = [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, 1, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
             getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{s}")]
        if info.restart:
            p += [cv2.IMWRITE_JPEG_RST_INTERVAL, info.restart]
        out.append(cv2.imencode(".jpg", img, p)[1].tobytes())
    return out


def loaded(bufs, max_scans):
    lay, _ = jpeg.plan(bufs, max_scans=max(max_scans, MAX_SCANS))
    jb = jpeg.JpegBatch(len(bufs), lay.coded_bytes, lay.out_bytes, lay.chunks + max_scans, lay.blocks,
                        max_scans=max_scans)
    jb.load(bufs, lay)
    jb.launch()
    jb.raise_on_status()
    return jb


def timed(jb, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        jb.launch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps   # ms per launch sequence


def kernel_times(jb, reps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            jb.launch()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"(jpeg_\w+_kernel)", e.key)
        if m and e.device_time_total > 0:
            out[m.group(1)] = out.get(m.group(1), 0.0) + e.device_time_total / 1e3 / reps   # ms per launch sequence
    return out


def graph_rate(batch, reps):
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)), mano_assets=assets)
    bufs = progressive(files(1080, 1920, "420", 0, batch, seed=1))
    lay, _ = jpeg.plan(bufs, max_scans=batch * MAX_SCANS)
    replay = app.capture_jpeg_graph(batch, lay.coded_bytes, lay.out_bytes, max_scans=len(lay.scans))
    replay(bufs)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        replay(bufs)
    torch.cuda.synchronize()
    replay.jpeg.raise_on_status()
    return reps * batch / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--threads", default="1,8")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--graph-batch", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("jpeg_progressive_bench needs a GPU")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"# {gpu}; host threads {os.cpu_count()}")
    threads = [int(t) for t in a.threads.split(",")]
    print("| size | sampling | RST | device img/s (3 runs) | " + " | ".join(f"cv2 x{t} img/s" for t in threads) + " |")
    for sname, (h, w) in SIZES.items():
        for s in ("420", "444"):
            for rst in (0, 4):
                bufs = progressive(files(h, w, s, rst, a.batch))
                jb = loaded(bufs, len(jpeg.plan(bufs, max_scans=a.batch * MAX_SCANS)[0].scans))
                rates = sorted(a.batch / (timed(jb, a.reps) / 1e3) for _ in range(3))
                host = [cv2_rate(bufs, t, max(1, a.reps // 2)) for t in threads]
                print(f"| {sname} | {s} | {rst or '-'} | {rates[0]:.0f}-{rates[-1]:.0f} | "
                      + " | ".join(f"{r:.0f}" for r in host) + " |", flush=True)
                del jb
    one = progressive(files(1080, 1920, "420", 0, 1, seed=2))
    jb = loaded(one, MAX_SCANS)
    lat = sorted(timed(jb, 1) for _ in range(21))
    kt = kernel_times(jb, 10)
    total = sum(kt.values())
    print(f"batch-1 latency, 1080p 4:2:0 progressive: median {lat[10]:.3f} ms (min {lat[0]:.3f}, max {lat[-1]:.3f})")
    for k, v in sorted(kt.items(), key=lambda kv: -kv[1]):
        print(f"  {k}: {v:.3f} ms ({100 * v / total:.1f}% of the kernel time)")
    base = files(1080, 1920, "420", 0, a.batch, seed=3)
    jb0, jb1 = loaded(base, 0), loaded(base, MAX_SCANS)
    r0, r1 = [], []
    for _ in range(3):
        r0.append(a.batch / (timed(jb0, a.reps) / 1e3))
        r1.append(a.batch / (timed(jb1, a.reps) / 1e3))
    torch.cuda.synchronize()
    assert torch.equal(jb0.out, jb1.out)
    print(f"baseline 1080p 4:2:0 batch {a.batch}: max_scans 0 {min(r0):.0f}-{max(r0):.0f} img/s, "
          f"max_scans {MAX_SCANS} {min(r1):.0f}-{max(r1):.0f} img/s")
    del jb0, jb1, jb
    print(f"capture_jpeg_graph replay, 1080p 4:2:0 progressive, batch {a.graph_batch}: "
          f"{graph_rate(a.graph_batch, a.reps):.1f} img/s")


if __name__ == "__main__":
    main()
