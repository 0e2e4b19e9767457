"""Part labels on the H100: acr_b200_part_labels alone, and its share of a capture_frames_graph replay.

    python tools/part_labels_bench.py [--out results.json] [--replay-batches 16 256]

1. The kernel alone at batch 256 of 720p, 1080p and 2160p frames, on two kinds of 256 x 256 bf16 logit maps: "fields"
   (33 smooth random fields: part boundaries everywhere, the most mixed quads) and "hands" (background everywhere but
   a few hand-sized blobs of parts, closer to real frames).  Time from CUDA events over many launches; HBM floor =
   (labels + the 16-bit 48-channel map) / 3.35 TB/s, the H100 SXM data-sheet bandwidth.
2. capture_frames_graph replays of 1080p frames (CUDA frames, so no host copy is timed) with and without part labels,
   alternated over three rounds, at each batch of --replay-batches.
The card's name, power limit and clocks are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM = 3.35e12
SIZES = {"720p": (720, 1280), "1080p": (1080, 1920), "2160p": (2160, 3840)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else "unknown"


def maps(n, kind, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "fields":
        low = torch.randn(n, 33, 16, 16, generator=g) * 4
    else:       # background wins by 8 everywhere but three 3 x 3 blobs of random parts per image
        low = torch.randn(n, 33, 16, 16, generator=g)
        low[:, 0] += 8
        for i in range(n):
            for _ in range(3):
                y, x = torch.randint(1, 14, (2,), generator=g).tolist()
                low[i, 1:, y - 1:y + 2, x - 1:x + 2] += torch.rand(32, 3, 3, generator=g) * 16
    up = torch.nn.functional.interpolate(low.cuda(), size=(256, 256), mode="bilinear", align_corners=False)
    m = torch.zeros(n, 256, 256, 48, device="cuda", dtype=torch.bfloat16)
    m[..., :33] = up.permute(0, 2, 3, 1)
    return m


def time_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_alone(batch=256):
    from acr_b200 import ops
    from acr_b200.preprocess import offsets_vector
    rows = []
    for kind in ("fields", "hands"):
        segms = maps(batch, kind)
        for name, (h, w) in SIZES.items():
            offs = torch.from_numpy(np.tile(offsets_vector(h, w), (batch, 1))).cuda()
            buf = ops.PartLabels(batch * h * w, batch)
            ms = time_ms(lambda: ops.part_labels(segms, offs, buf), 20)
            floor = batch * (h * w + 256 * 256 * 48 * 2) / HBM * 1e3
            rows.append(dict(maps=kind, frames=name, batch=batch, ms=round(ms, 4), hbm_floor_ms=round(floor, 4),
                             of_floor=round(floor / ms, 3)))
            print(json.dumps(rows[-1]), flush=True)
        del segms
    return rows


def replay_share(batch, rounds=3, iters=5):
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    h, w = SIZES["1080p"]
    app = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)),
              mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
    g = torch.Generator(device="cuda").manual_seed(1)
    frames = [torch.randint(0, 256, (h, w, 3), generator=g, device="cuda", dtype=torch.uint8) for _ in range(batch)]
    nbytes = batch * h * w * 3
    graphs = {"off": app.capture_frames_graph(batch, nbytes), "on": app.capture_frames_graph(batch, nbytes,
                                                                                              part_labels=True)}
    times = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, rep in graphs.items():
            times[k].append(time_ms(lambda: rep(frames), iters, warmup=2))
    off, on = np.median(times["off"]), np.median(times["on"])
    row = dict(batch=batch, frames="1080p", replay_ms_off=[round(t, 3) for t in times["off"]],
               replay_ms_on=[round(t, 3) for t in times["on"]], median_off=round(off, 3), median_on=round(on, 3),
               labels_share=round((on - off) / on, 4))
    print(json.dumps(row), flush=True)
    del graphs, app
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--replay-batches", type=int, nargs="*", default=[16, 256])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("part_labels_bench needs a GPU")
    os.environ.setdefault("ACR_B200_SYNTHETIC_MANO", "1")
    info = card()
    print("card:", info, flush=True)
    res = dict(card=info, kernel=kernel_alone(), replay=[replay_share(b) for b in a.replay_batches], card_after=card())
    print("card after:", res["card_after"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
