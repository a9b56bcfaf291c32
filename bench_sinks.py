"""Event-file cost of the batched pixel-model path, and the device merge of a sharded clip's bands.

  python bench_sinks.py [--frames 32] [--reps 5]

Prints one JSON line per measurement:
  * generate_events_batch on 1280 x 720 frames (rng_mode='device', the v2e CLI's default DVS parameters, a moving
    texture) with no sink, with dvs_aedat2 and with dvs_text: seconds per call and per frame, host clock around calls
    that end in a synchronise. The files go to a temporary directory on local disk. The sinks are the reference's
    writers (oracle/_ref/, made by build()); without them the sink lines say so. The AEDAT-2.0 writer takes only the
    jAER cameras' sizes, so its rows are packed with the 346 x 260 layout (the cost per event does not depend on it).
  * generate_events once per frame, as v2e's frame loop calls it, on host uint8 frames of the same texture at 346 x 260
    and 1280 x 720, with no sink, with dvs_aedat2 and with dvs_text: ms per frame, host clock around --frames frames
    that end in a synchronise, after one such pass of warm-up.
  * parallel.merge_by_key_device against the host merge_by_key on 2 and 8 row bands of one clip: the canonical stream
    of the clip above cut into bands of rows (each band's rows keep their order, as a band's own run orders them), the
    keys those of row_order='canonical' ((p < 0) << 32 | pixel). The merged rows are checked to be the stream again.
The GPU's name, power limit and maximum SM clock are printed first (nvidia-smi, read only)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

CLI = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.01,
           shot_noise_rate_hz=0.001, refractory_period_s=0.0005)
H, W = 720, 1280


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
    except Exception as e:
        name, power, clock = torch.cuda.get_device_name(0), "unknown (%s)" % e, "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def clip(T, seed=0, h=H, w=W):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h // 8 + T + 4, w // 8 + 2 * T + 4)).astype(np.uint8)
    big = np.kron(base, np.ones((8, 8), np.uint8))
    return np.stack([np.ascontiguousarray(big[k:k + h, 2 * k:2 * k + w]) for k in range(T)])


def bench_batch(frames, ts, sink, reps, folder):
    from v2e_b200 import EventEmulator
    kw = {} if sink is None else {sink: "ev_%s" % sink, "output_folder": folder}
    em = EventEmulator(device="cuda:0", rng_mode="device", seed=1, row_order="canonical", output_width=346,
                       output_height=260, **kw, **CLI)
    if sink is not None and em._sinks is None:
        return {"bench": "generate_events_batch", "sink": sink, "result": "not available (the writers do not import)"}
    fr = torch.from_numpy(frames).cuda()
    span = ts[-1] + ts[1]
    em.generate_events_batch(fr, ts, return_device=True)             # warm-up: first frame, buffers, files
    times, n = [], 0
    for r in range(1, reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rows, _ = em.generate_events_batch(fr, [t + r * span for t in ts], return_device=True)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        n = rows.shape[0]
    em.cleanup()
    med = float(np.median(times))
    return {"bench": "generate_events_batch", "size": "%dx%d" % (W, H), "sink": sink or "none", "frames": len(ts),
            "rows_per_call": int(n), "s_per_call_median": med, "s_per_call_min": float(min(times)),
            "ms_per_frame": 1e3 * med / len(ts), "reps": reps}


def bench_frames(h, w, sink, n, reps, folder):
    from v2e_b200 import EventEmulator
    kw = {} if sink is None else {sink: "pf_%s_%dx%d" % (sink, w, h), "output_folder": folder}
    em = EventEmulator(device="cuda:0", rng_mode="device", seed=1, output_width=346, output_height=260, **kw, **CLI)
    if sink is not None and em._sinks is None:
        return {"bench": "generate_events", "sink": sink, "result": "not available (the writers do not import)"}
    frames = clip(n * (reps + 1), h=h, w=w)
    times, rows = [], 0
    for r in range(reps + 1):                                        # pass 0 warms up: first frame, buffers, files
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(r * n, (r + 1) * n):
            ev = em.generate_events(frames[k], k / 300.)
            rows += len(ev) if ev is not None and r > 0 else 0
        torch.cuda.synchronize()
        if r > 0:
            times.append(time.perf_counter() - t0)
    em.cleanup()
    return {"bench": "generate_events", "size": "%dx%d" % (w, h), "sink": sink or "none", "frames": n,
            "rows_per_frame": rows / (n * reps), "ms_per_frame_median": 1e3 * float(np.median(times)) / n,
            "ms_per_frame_min": 1e3 * min(times) / n, "reps": reps}


def bands_of(rows, offs, n_shot, world):
    """The clip's canonical stream cut into `world` row bands (parallel.row_band), with canonical keys."""
    from v2e_b200.parallel import row_band
    T = len(offs) - 1
    frame = np.repeat(np.arange(T), np.diff(offs))
    shot = np.arange(len(rows)) >= (offs[1:] - n_shot)[frame]
    keys = ((rows[:, 3] < 0).astype(np.uint64) << np.uint64(32)) | (rows[:, 2].astype(np.uint64) * W
                                                                    + rows[:, 1].astype(np.uint64))
    out = ([], [], [], [])
    for r in range(world):
        y0, y1 = row_band(H, r, world)
        m = (rows[:, 2] >= y0) & (rows[:, 2] < y1)
        f = frame[m]
        out[0].append(np.ascontiguousarray(rows[m]))
        out[1].append(keys[m])
        out[2].append(np.concatenate([[0], np.cumsum(np.bincount(f, minlength=T))]).astype(np.int64))
        out[3].append(np.bincount(f[shot[m]], minlength=T).astype(np.int64))
    return out


def bench_merge(rows, offs, n_shot, world, reps):
    from v2e_b200.parallel import merge_by_key, merge_by_key_device
    s, k, o, n = bands_of(rows, offs, n_shot, world)
    t0 = time.perf_counter()
    host, hoffs = merge_by_key(s, k, o, n)
    t_host = time.perf_counter() - t0
    sd = [torch.from_numpy(x).cuda() for x in s]
    kd = [torch.from_numpy(x.view(np.int64)).cuda() for x in k]
    dev, doffs = merge_by_key_device(sd, kd, o, n)                   # warm-up
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        a = time.perf_counter()
        dev, doffs = merge_by_key_device(sd, kd, o, n)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - a)
    same = dev.cpu().numpy().tobytes() == host.tobytes() == rows.tobytes() and np.array_equal(doffs.cpu().numpy(), hoffs)
    return {"bench": "merge_bands", "bands": world, "rows": int(len(rows)), "frames": len(offs) - 1,
            "host_merge_by_key_s": t_host, "device_merge_s_median": float(np.median(times)),
            "device_merge_s_min": float(min(times)), "speedup": t_host / float(np.median(times)),
            "equal_to_host_and_stream": bool(same), "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sinks.py needs a CUDA device")
    print(json.dumps(gpu_info()), flush=True)
    try:
        import ref_shim
        if ref_shim.reference_available():
            ref_shim.load_reference()
    except Exception as e:
        print(json.dumps({"note": "the reference's writers do not load: %s" % e}), flush=True)
    frames = clip(a.frames)
    ts = [k / 300. for k in range(a.frames)]
    with tempfile.TemporaryDirectory() as d:
        for sink in (None, "dvs_aedat2", "dvs_text"):
            print(json.dumps(bench_batch(frames, ts, sink, a.reps, d)), flush=True)
        for h, w in ((260, 346), (H, W)):
            for sink in (None, "dvs_aedat2", "dvs_text"):
                print(json.dumps(bench_frames(h, w, sink, a.frames, a.reps, d)), flush=True)
    from v2e_b200 import EventEmulator
    em = EventEmulator(device="cuda:0", rng_mode="device", seed=1, row_order="canonical", label_signal_noise=True,
                       **CLI)
    rows, offs, lab = em.generate_events_batch(frames, ts, return_labels=True)
    n_shot = np.array([int((~lab[offs[f]:offs[f + 1]]).sum()) for f in range(len(offs) - 1)], np.int64)
    for world in (2, 8):
        print(json.dumps(bench_merge(rows, offs, n_shot, world, a.reps)), flush=True)


if __name__ == "__main__":
    main()
