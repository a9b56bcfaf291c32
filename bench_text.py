"""bench_text.py -- throughput of the DVS text sink (v2e_b200.sinks.events_to_text) on the rows of an 80-frame
1280x720 clip, and of the reference writer's per-row loop (DVSTextOutput.appendEvents) on the host.

    python bench_text.py [--frames 80] [--reps 10] [--ref-rows 100000]

Prints one JSON line:
  device_rows_per_s / device_bytes_per_s   events_to_text (layout, one synchronisation to read the length, write)
                                           on device-resident rows, CUDA-event timed over --reps calls after a warm-up
  device_to_file_rows_per_s                events_to_text + the D2H copy of the body (what write_text costs before
                                           the file write), host clock
  reference_rows_per_s                     DVSTextOutput.appendEvents with np.float = float set for the run (the alias
                                           numpy 1.24 removed) on the first --ref-rows rows, written to a temporary
                                           file; null when the reference tree is not present
The GPU name and power limit are part of the line. Nothing is written inside the repository.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def clip_rows(frames):
    """Rows of the headline's source texture (1280x720) translating 10 px per frame through the pixel model with the
    CLI defaults (device RNG), as one device tensor."""
    import torch
    import bench
    from v2e_b200 import EventEmulator
    H, W = 720, 1280
    src = bench.source_clip(H, W, frames, seed=0, px_per_frame=10)
    em = EventEmulator(device="cuda:0", rng_mode="device", seed=11, **bench.CLI_DEFAULTS)
    ts = [k / 30.0 for k in range(frames)]
    rows, offs = em.generate_events_batch(torch.from_numpy(src).cuda(), ts, return_device=True)
    return rows.clone()


def reference_rate(rows, n):
    import ref_shim
    if not ref_shim.reference_available():
        return None
    ref_shim.load_reference()
    from v2ecore.output.ae_text_output import DVSTextOutput
    ev = np.ascontiguousarray(rows[:n])
    had = hasattr(np, "float")
    np.float = float
    try:
        with tempfile.TemporaryDirectory() as td:
            w = DVSTextOutput(os.path.join(td, "ev.txt"))
            t0 = time.perf_counter()
            w.appendEvents(ev)
            w.file.flush()
            dt = time.perf_counter() - t0
            w.close()
    finally:
        if not had:
            del np.float
    return len(ev) / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ref-rows", type=int, default=100000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_text.py needs a CUDA device")
    from v2e_b200 import sinks
    rows = clip_rows(args.frames)
    n = rows.shape[0]
    body = sinks.events_to_text(rows)                   # warm-up (module load) and the body size
    nbytes = body.numel()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.reps):
        body = sinks.events_to_text(rows)
    b.record()
    torch.cuda.synchronize()
    dev_s = a.elapsed_time(b) / 1e3 / args.reps
    t0 = time.perf_counter()
    for _ in range(max(1, args.reps // 2)):
        host = sinks.events_to_text(rows).cpu().numpy().tobytes()
    d2f_s = (time.perf_counter() - t0) / max(1, args.reps // 2)
    assert len(host) == nbytes
    ref = reference_rate(rows.cpu().numpy(), args.ref_rows)
    line = {"workload": "dvs_text_%dx1280x720" % args.frames, "gpu": gpu_info(), "rows": int(n),
            "bytes": int(nbytes), "bytes_per_row": nbytes / max(n, 1),
            "device_rows_per_s": n / dev_s, "device_bytes_per_s": nbytes / dev_s,
            "device_to_file_rows_per_s": n / d2f_s,
            "reference_rows": min(args.ref_rows, int(n)), "reference_rows_per_s": ref,
            "speedup_device_to_host_vs_reference": (n / d2f_s) / ref if ref else None}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
