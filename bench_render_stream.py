#!/usr/bin/env python
"""The DVS video from V2EPipeline.run_segments at 1280x720, U = 10, batch 8, with bench.py's seeded SloMo weights,
source clip and pixel-model settings (CLI defaults, rng_mode="device") and v2e's default DVS video (DURATION exposure
of 0.01 s, full scale 2, packets of batch_size = 8 interpolated frames).

Arms, alternating in rounds over one clip of --pairs source frame pairs in segments of --segment pairs, every call one
clip period after the previous one on the arm's own emulator and renderer:
  none     run_segments without a renderer (host rows, copy=False);
  discard  with an EventRenderer whose video writer discards its frames: the plan, the render and one device-to-host
           copy per chunk of frames, plus the BGR conversion and the frame-times file;
  xvid     with an EventRenderer whose video writer is cv2.VideoWriter with XVID (v2ecore.v2e_utils.video_writer's
           codec) into a temporary directory;
  loop     run_segments without a renderer, and v2e.py's stage-3 loop written by hand: the host rows appended frame by
           frame, and render_events_to_frames (discarding writer) once per packet.
Reported per arm: ms per interpolated frame (median, min, max over the rounds), the device memory its first call
added (torch.cuda.max_memory_allocated - memory_allocated before it) and the device memory the renderer holds after a
call (its plan, chunk and held-row buffers). Also the AREA_COUNT scan's time per row on the
first segment's rows (one thread walks them; no video). Prints one JSON line with the card's name and power limit, read
in the same run."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

H, W, U, BATCH, SRC_FPS = 720, 1280, 10, 8, 30.0
DVS_VID = "dvs-video.avi"


class Discard:
    def __init__(self, *a, **k):
        self.frames = 0

    def write(self, frame):
        self.frames += 1

    def release(self):
        pass


def writer_modules(kind):
    """A v2ecore.v2e_utils with the two functions EventRenderer takes from it: a discarding writer, or XVID."""
    import cv2

    def checkAddSuffix(path, suffix):
        return path if path.endswith(suffix) else os.path.splitext(path)[0] + suffix

    def video_writer(output_path, height, width, frame_rate=30, fourcc=None):
        if kind == "discard":
            return Discard()
        w = cv2.VideoWriter(output_path, cv2.VideoWriter_fourcc(*"XVID"), frame_rate, (width, height))
        if not w.isOpened():
            raise RuntimeError("cv2.VideoWriter cannot open XVID here")
        return w
    pkg = types.ModuleType("v2ecore")
    pkg.__path__ = []
    utils = types.ModuleType("v2ecore.v2e_utils")
    utils.checkAddSuffix, utils.video_writer = checkAddSuffix, video_writer
    pkg.v2e_utils = utils
    return {"v2ecore": pkg, "v2ecore.v2e_utils": utils}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64, help="source frame pairs of the clip")
    ap.add_argument("--segment", type=int, default=32, help="source frame pairs per segment")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render_stream.py needs a CUDA device")
    from bench import CLI_DEFAULTS, slomo_weights, source_clip
    from v2e_b200 import EventEmulator, SuperSloMo, V2EPipeline
    from v2e_b200.renderer import RENDER_CHUNK_FRAMES, EventRenderer, ExposureMode
    dev = torch.device("cuda", 0)
    sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=U, batch_size=BATCH, state_dicts=slomo_weights())
    loop = source_clip(H, W, 257, seed=0)[:256]
    n = a.pairs + 1
    src_dev = torch.from_numpy(loop[np.arange(n) % 256]).to(dev)
    clip_s = (n - 1) / SRC_FPS
    period = clip_s * n / (n - 1)
    tmp = tempfile.mkdtemp(prefix="bench_render_stream_")
    arms = ("none", "discard", "xvid", "loop")
    mods = {"discard": writer_modules("discard"), "xvid": writer_modules("xvid"), "loop": writer_modules("discard")}

    def renderer(name, k):
        sys.modules.update(mods[name])
        out = os.path.join(tmp, "%s%d" % (name, k))
        os.makedirs(out)
        return EventRenderer(full_scale_count=2, output_path=out, dvs_vid=DVS_VID,
                             exposure_mode=ExposureMode.DURATION, exposure_value=0.01)

    state = {k: dict(em=EventEmulator(device="cuda:0", rng_mode="device", seed=1, **CLI_DEFAULTS), calls=0, ms=[])
             for k in arms}

    def call(name):
        st = state[name]
        r = renderer(name, st["calls"]) if name in ("discard", "xvid", "loop") else None
        pipe = V2EPipeline(sl, st["em"], renderer=r if name in ("discard", "xvid") else None)
        t0 = st["calls"] * period
        st["calls"] += 1
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        nf = rows = 0
        events, i = np.zeros((0, 4), np.float32), 0
        for ev, offs, t, k in pipe.run_segments(lambda p, q: src_dev[p:q], n, clip_s, t_offset=t0,
                                                segment_pairs=a.segment):
            nf += k
            rows += len(ev)
            if name == "loop":                           # v2e.py:826-846
                for f in range(k):
                    new = ev[offs[f]:offs[f + 1]]
                    if new.shape[0] > 0:
                        events = np.append(events, new, axis=0)
                        if i % BATCH == 0:
                            r.render_events_to_frames(events, height=H, width=W)
                            events = np.zeros((0, 4), np.float32)
                    i += 1
        if name == "loop" and len(events) > 0:
            r.render_events_to_frames(events, height=H, width=W)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - w0) * 1e3
        written = r.numFramesWritten if r is not None else 0
        if r is not None:
            r.cleanup()
            held = [] if r._held is None else [r._held]
            st["render_bytes"] = sum(b.numel() * b.element_size() for b in list(r._bufs.values()) + held
                                     if b.is_cuda)
        return ms, nf, rows, written

    res = {}
    for name in arms:                                    # warm-up call per arm; it also takes the arm's memory
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _, nf, rows, written = call(name)
        res[name] = dict(added_device_bytes=torch.cuda.max_memory_allocated() - before, frames=nf, rows=rows,
                         dvs_frames=written)
    for _ in range(a.rounds):
        for name in arms:
            ms, nf, rows, written = call(name)
            state[name]["ms"].append(ms / nf)
    for name in arms:
        v = state[name]["ms"]
        res[name].update(ms_per_frame_median=round(float(np.median(v)), 4), ms_per_frame_min=round(min(v), 4),
                         ms_per_frame_max=round(max(v), 4))
    for name in ("discard", "xvid", "loop"):
        res[name]["added_ms_per_frame_vs_none"] = round(res[name]["ms_per_frame_median"]
                                                        - res["none"]["ms_per_frame_median"], 4)
        res[name]["renderer_device_bytes"] = state[name]["render_bytes"]

    # the AREA_COUNT scan on one segment's rows: one device thread walks them (v2e_render_area_scan)
    em = EventEmulator(device="cuda:0", rng_mode="device", seed=1, **CLI_DEFAULTS)
    ev, offs, _, _ = next(iter(V2EPipeline(sl, em).run_segments(lambda p, q: src_dev[p:q], n, clip_s,
                                                                  segment_pairs=a.segment, return_device=True)))
    ev = ev.clone()
    r = EventRenderer(full_scale_count=2, exposure_mode=ExposureMode.AREA_COUNT, exposure_value=1000,
                      area_dimension=64)
    r.render_frame_rows(ev[:1], offs[:1], 0, BATCH, height=H, width=W)
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    frames = r.render_frame_rows(ev, offs, 0, BATCH, end_of_clip=True, height=H, width=W)
    torch.cuda.synchronize()
    scan_s = time.perf_counter() - w0
    sl.cleanup()
    shutil.rmtree(tmp, ignore_errors=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    out = dict(bench="render_stream", size="%dx%d" % (W, H), U=U, batch=BATCH, pairs=a.pairs, segment_pairs=a.segment,
               rounds=a.rounds, exposure="duration 0.01 s, full scale 2", chunk_frames=RENDER_CHUNK_FRAMES, arms=res,
               area_count_scan=dict(rows=int(ev.shape[0]), frames=int(frames), ms=round(scan_s * 1e3, 3),
                                    ns_per_row=round(scan_s * 1e9 / max(int(ev.shape[0]), 1), 3)),
               gpu=q[0] if q else "unknown")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
