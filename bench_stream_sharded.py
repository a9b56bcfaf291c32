#!/usr/bin/env python
"""V2EPipeline.run_segments_sharded against V2EPipeline.run_clip_sharded: one clip over several ranks at 1280x720,
U = 10, batch 8, with bench.py's seeded SloMo weights, source clip and pixel-model settings (CLI defaults,
rng_mode="device", row_order="canonical", which write_sinks needs).

Arms: run_clip_sharded, and run_segments_sharded at 16, 64 and 256 source frame pairs per segment (of the group).
Reported per rank and arm: the device memory the arm's first call added on top of what was allocated before it
(torch.cuda.max_memory_allocated - memory_allocated: frames, bands, rows and the emulator's buffers; the SloMo engine's
buffers are allocated outside torch's allocator and are the same for every arm), without sinks and, for run_clip_sharded
and 16 pairs per segment, with write_sinks=True and a dvs_text file (the bands of every rank gathered and merged there; the merged stream is
the same for every sink, and the reference's AEDAT-2.0 writer takes only camera sizes up to 640x480).

With at least 2 GPUs the ranks are NCCL processes, one GPU each (--world, default every GPU up to 8), and the arms are
also timed in alternating rounds: ms per interpolated frame (median, min, max). With one GPU the ranks are gloo
processes sharing it: gloo stages every exchange through the host and the ranks compete for one GPU, so the memory is
reported and the time is "not measured". Prints one JSON line with the card's name and power limit, read in the same
run."""
import argparse
import json
import os
import shutil
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

H, W, U, BATCH, SRC_FPS = 720, 1280, 10, 8, 30.0
SEGMENTS = (16, 64, 256)


def _rank(rank, world, port, backend, pairs, rounds, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import ref_shim
        if ref_shim.reference_available():
            ref_shim.load_reference()          # the text writer's header; without it the sinks arm writes nothing
        from bench import CLI_DEFAULTS, slomo_weights, source_clip
        from v2e_b200 import EventEmulator, SuperSloMo, V2EPipeline
        sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=U, batch_size=BATCH,
                        device="cuda:%d" % dev, state_dicts=slomo_weights())
        loop = source_clip(H, W, 257, seed=0)[:256]       # source_clip loops: frame 256 is frame 0
        n = pairs + 1
        src = torch.from_numpy(loop[np.arange(n) % 256]).to(dev)
        clip_s = pairs / SRC_FPS
        arms = {"clip": None}
        arms.update({"seg%d" % s: s for s in SEGMENTS})
        tmp = tempfile.mkdtemp()

        def call(name, sinks=False):
            kw = dict(output_folder=tmp, dvs_text=name, output_width=W, output_height=H) if sinks and rank == 0 else {}
            em = EventEmulator(device="cuda:%d" % dev, rng_mode="device", seed=1, row_order="canonical",
                               shard=(rank, world, None), **CLI_DEFAULTS, **kw)
            pipe = V2EPipeline(sl, em)
            dist.barrier()
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            w0 = time.perf_counter()
            if arms[name] is None:
                rows, t, nf = pipe.run_clip_sharded(src, clip_s, write_sinks=sinks)
                nrows = len(rows)
            else:
                nf = nrows = 0
                for rows, t, k in pipe.run_segments_sharded(lambda a, b: src[a:b], n, clip_s,
                                                            segment_pairs=arms[name], write_sinks=sinks):
                    nf += k
                    nrows += len(rows)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - w0) * 1e3
            added = torch.cuda.max_memory_allocated() - before
            wrote = sinks and rank == 0 and em.dvs_text is not None
            em.cleanup()
            return ms / nf, added, nf, nrows, wrote

        call("seg64")                                   # the SloMo engine exists before any measurement
        res = {}
        for name in arms:
            _, added, nf, nrows, _ = call(name)
            res[name] = dict(added_device_bytes=added, frames=nf, rows=nrows)
        for name in ("clip", "seg16"):                 # the text of every event is written: the two extremes only
            _, added, _, _, wrote = call(name, sinks=True)
            res[name]["added_device_bytes_write_sinks"] = added
            res[name]["text_written"] = bool(wrote)
        for _ in range(rounds):
            for name in arms:
                res[name].setdefault("ms", []).append(call(name)[0])
        for name in arms:
            v = res[name].pop("ms", None)
            if v:
                res[name].update(ms_per_frame_median=round(float(np.median(v)), 4), ms_per_frame_min=round(min(v), 4),
                                 ms_per_frame_max=round(max(v), 4))
            else:
                res[name]["time"] = "not measured"
        sl.cleanup()
        shutil.rmtree(tmp, ignore_errors=True)
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=128, help="source frame pairs of the clip")
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds (NCCL, one GPU per rank, only)")
    ap.add_argument("--world", type=int, default=None, help="ranks (default: every GPU up to 8, or 2 on one GPU)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_sharded.py needs a CUDA device")
    n_gpu = torch.cuda.device_count()
    backend = "nccl" if n_gpu >= 2 else "gloo"
    world = a.world or (min(n_gpu, 8) if backend == "nccl" else 2)
    if backend == "nccl" and world > n_gpu:
        raise SystemExit("--world %d needs as many GPUs (%d present)" % (world, n_gpu))
    rounds = a.rounds if backend == "nccl" else 0
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, world, port, backend, a.pairs, rounds, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        per_rank = dict(q.get(timeout=3600) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    out = dict(bench="stream_sharded", size="%dx%d" % (W, H), U=U, batch=BATCH, pairs=a.pairs, interp_frames=a.pairs * U,
               backend=backend, world=world, gpus=n_gpu, rounds=rounds,
               time=None if rounds else "not measured (needs NCCL ranks on at least 2 GPUs)",
               ranks={str(r): per_rank[r] for r in sorted(per_rank)}, gpu=smi[0] if smi else "unknown")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
