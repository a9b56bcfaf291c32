#!/usr/bin/env python
"""V2EPipeline.run_segments against V2EPipeline.run at 1280x720, U = 10, batch 8, with bench.py's seeded SloMo weights,
source clip and pixel-model settings (CLI defaults, rng_mode="device").

1. A clip that fits in one run (--pairs source frame pairs, default 384: 3840 interpolated frames): run and run_segments
   at 16, 64 and 256 pairs per segment, alternating in rounds. Every call returns host rows (copy=False) and starts one
   frame interval after the previous one on the same emulator. Reported per arm: ms per interpolated frame (median,
   min and max over the rounds) and the device memory the arm's first call added on top of what was allocated before
   it (torch.cuda.max_memory_allocated - memory_allocated: its frames, rows and the emulator's buffers; the SloMo
   engine's buffers are allocated outside torch's allocator and are the same for every arm).
2. A long clip that one run could not hold: more pairs than the card's memory has room for at run's footprint (the
   interpolated frames plus the event rows at the rate the first clip produced), streamed with the default segment
   length from frames fetched on the host. Reported: frames, events, wall time, max_memory_allocated and the bytes run
   would have needed.
Prints one JSON line with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

H, W, U, BATCH, SRC_FPS = 720, 1280, 10, 8, 30.0
SEGMENTS = (16, 64, 256)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=384, help="source frame pairs of the clip that fits in one run")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-long", action="store_true", help="skip the clip that does not fit in one run")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream.py needs a CUDA device")
    from bench import CLI_DEFAULTS, slomo_weights, source_clip
    from v2e_b200 import EventEmulator, SuperSloMo, V2EPipeline
    from v2e_b200.pipeline import DEFAULT_SEGMENT_PAIRS
    dev = torch.device("cuda", 0)
    sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=U, batch_size=BATCH, state_dicts=slomo_weights())
    loop = source_clip(H, W, 257, seed=0)[:256]          # source_clip loops: frame 256 is frame 0
    n = a.pairs + 1
    src_dev = torch.from_numpy(loop[np.arange(n) % 256]).to(dev)
    clip_s = (n - 1) / SRC_FPS
    period = clip_s * n / (n - 1)

    arms = {"run": None}
    arms.update({"seg%d" % s: s for s in SEGMENTS})
    state = {k: dict(em=EventEmulator(device="cuda:0", rng_mode="device", seed=1, **CLI_DEFAULTS), calls=0, ms=[],
                     events=0) for k in arms}

    def call(name):
        st = state[name]
        pipe = V2EPipeline(sl, st["em"])
        t0 = st["calls"] * period
        st["calls"] += 1
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        if arms[name] is None:
            ev, offs, t, nf = pipe.run(src_dev, clip_s, t_offset=t0)
            rows = len(ev)
        else:
            nf = rows = 0
            for ev, offs, t, k in pipe.run_segments(lambda p, q: src_dev[p:q], n, clip_s, t_offset=t0,
                                                    segment_pairs=arms[name]):
                nf += k
                rows += len(ev)
        torch.cuda.synchronize()
        return (time.perf_counter() - w0) * 1e3, nf, rows

    res = {}
    for name in arms:                                    # warm-up call per arm; it also takes the arm's memory
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _, nf, rows = call(name)
        res[name] = dict(added_device_bytes=torch.cuda.max_memory_allocated() - before, frames=nf, rows=rows)
    for _ in range(a.rounds):
        for name in arms:
            ms, nf, rows = call(name)
            state[name]["ms"].append(ms / nf)
            state[name]["events"] = rows
    for name in arms:
        v = state[name]["ms"]
        res[name].update(ms_per_frame_median=round(float(np.median(v)), 4), ms_per_frame_min=round(min(v), 4),
                         ms_per_frame_max=round(max(v), 4), events_last_call=state[name]["events"])
    events_per_frame = res["run"]["rows"] / max(res["run"]["frames"], 1)
    del state
    out = dict(bench="stream", size="%dx%d" % (W, H), U=U, batch=BATCH, rounds=a.rounds,
               fit_clip=dict(pairs=a.pairs, interp_frames=a.pairs * U, arms=res))

    if not a.no_long:
        del src_dev
        torch.cuda.synchronize()
        total = torch.cuda.get_device_properties(0).total_memory
        per_pair = U * H * W + events_per_frame * U * 16           # run: interpolated frames + device event rows
        pairs = int(np.ceil(1.05 * total / per_pair / BATCH)) * BATCH
        em = EventEmulator(device="cuda:0", rng_mode="device", seed=1, **CLI_DEFAULTS)
        torch.cuda.reset_peak_memory_stats()
        nf = rows = segs = 0
        w0 = time.perf_counter()
        for ev, offs, t, k in V2EPipeline(sl, em).run_segments(lambda p, q: loop[np.arange(p, q) % 256], pairs + 1,
                                                               pairs / SRC_FPS):
            nf += k
            rows += len(ev)
            segs += 1
        torch.cuda.synchronize()
        wall = time.perf_counter() - w0
        out["long_clip"] = dict(pairs=pairs, segments=segs, segment_pairs=DEFAULT_SEGMENT_PAIRS, interp_frames=nf,
                                events=rows, wall_s=round(wall, 2), ms_per_frame=round(wall * 1e3 / nf, 4),
                                max_memory_allocated=torch.cuda.max_memory_allocated(),
                                run_would_need_bytes=int(nf * H * W + rows * 16), card_total_bytes=total)
    sl.cleanup()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    out["gpu"] = q[0] if q else "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
