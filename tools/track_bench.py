#!/usr/bin/env python
"""Cost of multi-hand tracking (acr_b200_track_hands, acr_b200.ops.HandTracker).

1. The tracker kernel alone, smoothing on, on seeded row tables in the parse's layout (1..K hands per image and side,
   cells on a random walk): batch 1 and 256, K = 1, 4 and 16.  CUDA events around replays of a graph of 20 calls
   (the state carries from call to call, as in a stream).
2. ``ACR.capture_graph(B)`` replays of the whole pipeline at batch 1 and 256, K = 4, with and without a tracker,
   the two alternating per round on the same frames.

    python tools/track_bench.py [--out result.json] [--rounds 3]

One JSON object on stdout (and in --out), with the GPU's name, power limit and SM clocks read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT, os.path.dirname(__file__)):
    sys.path.insert(0, p)
os.environ.setdefault("ACR_B200_SYNTHETIC_MANO", "1")
import numpy as np  # noqa: E402
import torch  # noqa: E402

from acr.config import ConfigContext, parse_args  # noqa: E402
from acr_b200 import lib as L  # noqa: E402
from acr_b200 import ops  # noqa: E402
from multi_hand_bench import events_ms, gpu_info, graphed_us  # noqa: E402


def row_table(B, K, seed):
    """Rows of B frames, side-major then image-major: per image and side 1..K hands on a random walk."""
    rng = np.random.default_rng(seed)
    rows = []
    for s in (0, 1):
        pos = rng.integers(0, 64, (K, 2))
        for b in range(B):
            pos = np.clip(pos + rng.integers(-2, 3, (K, 2)), 0, 63)
            for k in range(int(rng.integers(1, K + 1))):
                rows.append((b, s, int(pos[k, 0]) * 64 + int(pos[k, 1]), -1))
    return np.asarray(rows, np.int32).reshape(-1, 4)


def bench_kernel():
    out = []
    for B in (1, 256):
        for K in (1, 4, 16):
            rows = row_table(B, K, 7 * B + K)
            n = rows.shape[0]
            rs = torch.from_numpy(rows).cuda()
            flag = torch.ones(n, device="cuda")
            poses, betas = torch.randn(n, 48, device="cuda") * 0.4, torch.randn(n, 10, device="cuda")
            t = ops.HandTracker("cuda", K)
            us = graphed_us(lambda: ops.track_rows(t, B, rs, flag, poses, betas))
            torch.cuda.synchronize()
            out.append({"batch": B, "K": K, "rows": n, "us_per_call_in_graph": round(us, 2)})
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
    return out


def bench_graphs(rounds, steps):
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    K = 4
    ConfigContext(parse_args(["--return_maps", "false", "--max_hands_per_side", str(K)]))
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)),
              mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
    out = []
    for B in (1, 256):
        g = torch.Generator().manual_seed(B)
        frames = torch.randint(0, 256, (B, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
        offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1).cuda()
        tracker = ops.HandTracker("cuda", K)
        replays = {"without": app.capture_graph(B), "with": app.capture_graph(B, tracker=tracker)}
        times = {k: [] for k in replays}
        for _ in range(rounds):
            for k, r in replays.items():
                times[k].append(events_ms(lambda: r(frames, offs), steps))
        torch.cuda.synchronize()
        rows = int(replays["with"](frames, offs)[0].counts[2])
        for k in replays:
            out.append({"batch": B, "K": K, "tracker": k, "ms_per_replay": [round(v, 3) for v in times[k]],
                        "rows": rows})
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
        del replays
        torch.cuda.empty_cache()
    ConfigContext(parse_args([]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--kernel-only", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("track_bench.py needs a CUDA device")
    L.load()
    res = {"gpu": gpu_info(), "kernel": bench_kernel()}
    if not a.kernel_only:
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
