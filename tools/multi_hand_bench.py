#!/usr/bin/env python
"""Cost of multi-hand parsing (``max_hands_per_side`` = K).

1. The parse kernels alone on seeded multi-peak centre maps: acr_b200_parse (K = 1) and acr_b200_parse_topk at
   K = 2, 4, 16, at batch 1 and 256.  CUDA events around back-to-back eager calls (bound by the host's launch rate)
   and around replays of a graph of 20 calls (the device time of the three kernels).
2. ``ACR.capture_graph(B)`` replays of the whole pipeline (network + parse + MANO + cam_trans) at batch 1, 64 and 256
   with K = 1 and K = 4, the two K alternating per round on the same frames.

    python tools/multi_hand_bench.py [--out result.json] [--rounds 3]

One JSON object on stdout (and in --out), with the GPU's name, power limit and SM clocks read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT):
    sys.path.insert(0, p)
os.environ.setdefault("ACR_B200_SYNTHETIC_MANO", "1")
import torch  # noqa: E402

from acr.config import ConfigContext, parse_args  # noqa: E402
from acr_b200 import lib as L  # noqa: E402
from acr_b200 import ops  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split("\n")[0].split(",")])) if r.returncode == 0 else {}


def events_ms(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def graphed_us(fn, reps=20, iters=100):
    """Device time per call: ``reps`` calls captured in one CUDA graph, the graph replayed ``iters`` times (the eager
    calls are bound by the host's launch rate)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    return events_ms(g.replay, iters) / reps * 1e3


def device_maps(B, seed):
    """Multi-peak centre maps (0-10 peaks per image and side on a 0.08-sigma floor) and random parameter / prior
    maps, NHWC fp32 on the device, in the layout the engine hands to the parser."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    maps = {}
    for s in "lr":
        cm = torch.randn(B, 64, 64, 1, generator=g, device="cuda") * 0.08
        n = torch.randint(0, 11, (B,), generator=g, device="cuda")
        for k in range(10):
            pos = torch.randint(0, 4096, (B,), generator=g, device="cuda")
            val = torch.rand(B, generator=g, device="cuda") * 0.64 + 0.36
            keep = k < n
            cm.view(B, -1)[torch.arange(B, device="cuda")[keep], pos[keep]] = val[keep]
        maps[f"{s}_center"] = (cm.contiguous(), 1)
        maps[f"{s}_params"] = (torch.randn(B, 64, 64, 109, generator=g, device="cuda"), 109)
        maps[f"{s}_prior"] = (torch.randn(B, 64, 64, 106, generator=g, device="cuda") * 0.1, 106)
    return maps


def bench_parse(iters):
    out = []
    for B in (1, 256):
        maps = device_maps(B, B)
        for K in (1, 2, 4, 16):
            bufs = ops.ParseBuffers(B, "cuda", K)
            call = lambda: ops.parse_maps(maps, B, bufs, None, None, 0.35, K)
            ms = events_ms(call, iters)
            us_graph = graphed_us(call)
            torch.cuda.synchronize()
            out.append({"batch": B, "K": K, "entry": "acr_b200_parse" if K == 1 else "acr_b200_parse_topk",
                        "us_per_eager_call": round(ms * 1e3, 2), "us_per_call_in_graph": round(us_graph, 2),
                        "rows": int(bufs.counts[2]),
                        "detections": int(bufs.counts[3])})
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
    return out


def bench_graphs(rounds, steps):
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    ConfigContext(parse_args(["--return_maps", "false"]))
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)),
              mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
    out = []
    for B in (1, 64, 256):
        g = torch.Generator().manual_seed(B)
        frames = torch.randint(0, 256, (B, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
        offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1).cuda()
        replays = {}
        for K in (1, 4):
            ConfigContext(parse_args(["--return_maps", "false", "--max_hands_per_side", str(K)]))
            replays[K] = app.capture_graph(B)
        times = {1: [], 4: []}
        rows = {}
        for _ in range(rounds):
            for K in (1, 4):
                ConfigContext(parse_args(["--return_maps", "false", "--max_hands_per_side", str(K)]))
                times[K].append(events_ms(lambda: replays[K](frames, offs), steps))
                rows[K] = int(replays[K](frames, offs)[0].counts[2])
        torch.cuda.synchronize()
        for K in (1, 4):
            out.append({"batch": B, "K": K, "ms_per_replay": [round(t, 3) for t in times[K]], "hands": rows[K],
                        "mano_rows": 2 * K * B})
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
        del replays
        torch.cuda.empty_cache()
    ConfigContext(parse_args([]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parse-iters", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--parse-only", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("multi_hand_bench.py needs a CUDA device")
    L.load()
    res = {"gpu": gpu_info(), "parse": bench_parse(a.parse_iters)}
    if not a.parse_only:
        res["graph"] = bench_graphs(a.rounds, a.steps)
    res["gpu_after"] = gpu_info()
    s = json.dumps(res)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
