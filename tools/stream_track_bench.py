#!/usr/bin/env python
"""Cost of tracking several streams in one batch (acr_b200_track_streams, acr_b200.ops.HandTracker(streams=S)).

1. The tracker alone, smoothing on, at batch 256 and K = 1, 4 and 16, on seeded row tables in the parse's layout
   (1..K hands per image and side on a random walk): one stream through acr_b200_track_hands (S = 1, every frame
   consecutive), and 16 and 256 streams interleaved at random through acr_b200_track_streams.  CUDA events around
   replays of a graph of 20 calls (the state carries from call to call).
2. ``ACR.capture_graph(256)`` replays of the whole pipeline at K = 4 with a 256-stream tracker (one frame per stream)
   and without a tracker, the two alternating per round on the same frames.

    python tools/stream_track_bench.py [--out result.json] [--rounds 3]

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
from track_bench import row_table  # noqa: E402

B = 256


def bench_kernel():
    out = []
    for K in (1, 4, 16):
        rows = row_table(B, K, 7 * B + K)
        n = rows.shape[0]
        rs = torch.from_numpy(rows).cuda()
        flag = torch.ones(n, device="cuda")
        poses, betas = torch.randn(n, 48, device="cuda") * 0.4, torch.randn(n, 10, device="cuda")
        for S in (1, 16, 256):
            t = ops.HandTracker("cuda", K, streams=S)
            if S == 1:        # the single-stream call
                us = graphed_us(lambda: ops.track_rows(t, B, rs, flag, poses, betas))
            else:             # S streams, B / S frames each, interleaved at random
                order = np.random.default_rng(S + K).permutation(np.arange(B) % S).astype(np.int32)
                fs = torch.from_numpy(order).cuda()
                us = graphed_us(lambda: ops.track_rows(t, B, rs, flag, poses, betas, frame_stream=fs))
            torch.cuda.synchronize()
            out.append({"batch": B, "K": K, "streams": S, "rows": n, "us_per_call_in_graph": round(us, 2)})
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
    return out


def bench_graphs(rounds, steps):
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    K = 4
    ConfigContext(parse_args(["--return_maps", "false", "--max_hands_per_side", str(K)]))
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)),
              mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
    g = torch.Generator().manual_seed(B)
    frames = torch.randint(0, 256, (B, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
    offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1).cuda()
    sid = torch.from_numpy(np.random.default_rng(0).permutation(B).astype(np.int32)).cuda()
    tracker = ops.HandTracker("cuda", K, streams=B)
    replays = {"without": app.capture_graph(B), "with_256_streams": app.capture_graph(B, tracker=tracker)}
    calls = {"without": lambda: replays["without"](frames, offs),
             "with_256_streams": lambda: replays["with_256_streams"](frames, offs, sid)}
    times = {k: [] for k in replays}
    for _ in range(rounds):
        for k, c in calls.items():
            times[k].append(events_ms(c, steps))
    torch.cuda.synchronize()
    rows = int(calls["with_256_streams"]()[0].counts[2])
    out = []
    for k in replays:
        out.append({"batch": B, "K": K, "tracker": k, "ms_per_replay": [round(v, 3) for v in times[k]], "rows": rows})
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
        sys.exit("stream_track_bench.py needs a CUDA device")
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
