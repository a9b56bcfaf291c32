"""bench_order.py -- what EventEmulator(row_order=...) adds to generate_events_batch at 1280x720.

    python bench_order.py [--frames 80] [--rounds 3]

Two clips of device-resident uint8 frames through the pixel model with the CLI defaults (device RNG):
  headline  bench.py's source texture moving 1 px per frame at 300 frames/s (about 0.1 events per pixel and frame)
  dense     the same texture moving 10 px per frame at 30 frames/s, bench_text.py's clip (about 1 event per pixel
            and frame)
For each clip one emulator per setting (row_order None / "canonical" / "shuffled"); every emulator sees the same calls
in the same order: the clip loops seamlessly, so call after call continues it. One warm-up call each, then --rounds
rounds in which the three settings alternate; a call is timed with CUDA events around generate_events_batch(...,
return_device=True) and the median over the rounds is reported. Prints one JSON line:
  rows, events_per_px_per_frame          of one call (the same for the three settings)
  ms / rows_per_s                        per setting, median call
  added_us_per_frame                     (ordered - None) / frames
  order_bytes_per_row                    HBM bytes the ordering passes move per row (count 16, scatter 16 + 24,
                                         sort 24 + 16; the bucket counters are 4 B per ~32 rows on top)
  order_gbytes_per_s                     rows * order_bytes_per_row / added time
  gpu                                    name, power limit, maximum and current SM clock, memory clock (read-only query)
Nothing is written inside the repository.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ORDER_BYTES_PER_ROW = 16 + (16 + 24) + (24 + 16)
SETTINGS = [None, "canonical", "shuffled"]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.mem",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else None
    except Exception:
        return None


def run_clip(name, px_per_frame, fps, frames, rounds):
    import torch
    import bench
    from v2e_b200 import EventEmulator
    H, W = 720, 1280
    # frames + 1 source frames: the last equals the first, so the next call continues the motion
    src = torch.from_numpy(bench.source_clip(H, W, frames + 1, seed=11, px_per_frame=px_per_frame)).cuda()
    ems = {}
    calls = {s: 0 for s in SETTINGS}
    ms = {s: [] for s in SETTINGS}
    rows = {}

    def call(s, timed):
        k0 = calls[s] * frames
        first = calls[s] == 0
        clip = src[:frames + 1] if first else src[1:frames + 1]          # the very first frame only initialises
        ts = [(k0 + k) / fps for k in range(0 if first else 1, frames + 1)]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r, _ = ems[s].generate_events_batch(clip, ts, return_device=True)
        b.record()
        torch.cuda.synchronize()
        calls[s] += 1
        if timed:
            ms[s].append(a.elapsed_time(b))
            rows.setdefault(s, []).append(int(r.shape[0]))

    for s in SETTINGS:
        # seeding happens in the constructor and the per-pixel thresholds are drawn by the first call: keep them together
        ems[s] = EventEmulator(device="cuda:0", rng_mode="device", seed=11, row_order=s, max_frames_per_step=frames,
                               **bench.CLI_DEFAULTS)
        call(s, False)
    for _ in range(rounds):
        for s in SETTINGS:
            call(s, True)
    assert rows[None] == rows["canonical"] == rows["shuffled"], "the three settings must emit the same rows"
    n = int(np.median(rows[None]))
    med = {s: float(np.median(ms[s])) for s in SETTINGS}
    out = {"clip": name, "frames": frames, "rows": n, "events_per_px_per_frame": n / (frames * H * W)}
    for s in SETTINGS:
        key = s or "none"
        out[key + "_ms"] = med[s]
        out[key + "_ms_all"] = ms[s]
        out[key + "_rows_per_s"] = n / (med[s] * 1e-3)
        if s is not None:
            added = med[s] - med[None]
            out[key + "_added_us_per_frame"] = added * 1e3 / frames
            out[key + "_added_fraction"] = added / med[None]
            out[key + "_order_gbytes_per_s"] = n * ORDER_BYTES_PER_ROW / (added * 1e-3) / 1e9 if added > 0 else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_order.py needs a CUDA device")
    if args.rounds < 3:
        raise SystemExit("--rounds must be at least 3")
    line = {"workload": "row_order_1280x720", "gpu": gpu_info(), "order_bytes_per_row": ORDER_BYTES_PER_ROW,
            "clips": [run_clip("headline", 1, 300.0, args.frames, args.rounds),
                      run_clip("dense", 10, 30.0, args.frames, args.rounds)]}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
