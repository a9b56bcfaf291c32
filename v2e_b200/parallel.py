"""Multi-GPU plumbing for the two hot paths (SURVEY.md 8e). One process per GPU (torchrun), NCCL on
the GPU box, gloo in the CPU tests.

The paths shard without a data-path collective:
  * independent clips (BASELINE config 4): clips are dealt round-robin to ranks, every rank runs the
    whole SloMo + pixel-model path on its clips;
  * the only exchange is the merge of the packed event streams at the end (`gather_event_streams`).
One clip over several GPUs (BASELINE config 5): SloMo is sharded over frame PAIRS (every (pair, t) is
independent given the pair, slomo.py:404-433, so no halo), the pixel model over pixel ROWS (per-pixel state;
one all-reduce(MAX) of an int32 per frame, emulator.py:773-775); in between every rank needs its rows of
every frame: `exchange_frame_bands`, one all-to-all of uint8 row bands.
Nothing here touches model arithmetic.
"""
import numpy as np
import torch
import torch.distributed as dist


def shard_clips(n_clips, rank, world):
    """Indices of the clips rank `rank` owns: round-robin so that clips of similar cost spread evenly."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    return list(range(rank, n_clips, world))


def row_band(height, rank, world, align=1):
    """[y0, y1) of the pixel rows rank `rank` owns when ONE clip's pixel model is sharded over ranks
    (BASELINE config 5). Bands differ by at most `align` rows; empty bands are allowed."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    units = (height + align - 1) // align
    base, extra = divmod(units, world)
    u0 = rank * base + min(rank, extra)
    u1 = u0 + base + (1 if rank < extra else 0)
    return min(u0 * align, height), min(u1 * align, height)


def pair_range(n_pairs, rank, world):
    """[p0, p1) of the consecutive frame pairs rank `rank` interpolates when ONE clip's SloMo is sharded
    over ranks (contiguous, so that the rank's interpolated frames are a contiguous run of the clip)."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    base, extra = divmod(n_pairs, world)
    p0 = rank * base + min(rank, extra)
    return p0, p0 + base + (1 if rank < extra else 0)


def batch_pair_range(n_pairs, batch_size, rank, world):
    """[p0, p1) of the consecutive frame pairs rank `rank` interpolates when ONE clip's SloMo is sharded over ranks
    with a U chosen per batch (auto_upsample, slomo.py:366-385): the clip's batches of `batch_size` pairs, counted from
    its first pair, are dealt to the ranks whole and contiguous, so that every rank's batches -- and so its U's -- are
    those of a single-GPU run. Only the last rank gets the clip's short final batch. Raises ValueError when there are
    fewer batches than ranks."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    n_batches = -(-n_pairs // batch_size)
    if n_batches < world:
        raise ValueError("fewer batches of frame pairs than ranks")
    b0, b1 = pair_range(n_batches, rank, world)
    return b0 * batch_size, min(b1 * batch_size, n_pairs)


def band_with_halo(height, rank, world, halo=0):
    """row_band widened by `halo` rows either side, clipped to the frame (the centre-surround pixel model reads its
    neighbours' rows: emulator.py:1102-1124)."""
    y0, y1 = row_band(height, rank, world)
    return max(0, y0 - halo), min(height, y1 + halo)


def exchange_frame_bands(frames_local, height, group=None, halo=0):
    """frames_local: [M_r, H, W] uint8, the interpolated frames this rank synthesised (ranks hold consecutive
    runs of the clip, in rank order). Returns [sum_r M_r, y1-y0, W]: rows `band_with_halo(H, rank, world, halo)`
    of EVERY frame of the clip, in clip order. NCCL: one all-to-all of the row bands (rank r sends rank q the
    band q of its frames). Backends without all-to-all (gloo, in the tests): every rank's frames are
    all-gathered and cut locally."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if frames_local.dim() != 3 or frames_local.dtype != torch.uint8 or frames_local.shape[1] != height:
        raise ValueError("frames_local must be [M, H, W] uint8")
    W = frames_local.shape[2]
    dev = frames_local.device
    m = torch.tensor([frames_local.shape[0]], dtype=torch.int64, device=dev)
    ms = [torch.zeros_like(m) for _ in range(world)]
    dist.all_gather(ms, m, group=group)
    ms = [int(x.item()) for x in ms]
    y0, y1 = band_with_halo(height, rank, world, halo)
    if dist.get_backend(group) == "nccl":
        send = [frames_local[:, a:b, :].contiguous() for a, b in (band_with_halo(height, q, world, halo) for q in range(world))]
        recv = [torch.empty((ms[r], y1 - y0, W), dtype=torch.uint8, device=dev) for r in range(world)]
        dist.all_to_all(recv, send, group=group)
        return torch.cat(recv, 0)
    mx = max(ms)
    pad = torch.zeros((mx, height, W), dtype=torch.uint8, device=dev)
    pad[:frames_local.shape[0]] = frames_local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    return torch.cat([b[:c, y0:y1, :] for b, c in zip(bufs, ms)], 0).contiguous()


def gather_event_streams(rows, clip_ids=None, dst=0, group=None):
    """Gathers every rank's packed event rows ([N_r, 4] float32: t, x, y, p) on rank `dst`.

    Row counts differ per rank, so counts are all-gathered first and rows are padded to the largest
    count for the (fixed-size) gather. Returns on `dst` a list with one [N_r, 4] tensor per rank (in rank
    order, on the input's device), elsewhere None. Works with NCCL (CUDA tensors) and gloo (CPU)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if rows.dim() != 2 or rows.shape[1] != 4:
        raise ValueError("rows must be [N, 4]")
    n = torch.tensor([rows.shape[0]], dtype=torch.int64, device=rows.device)
    counts = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(counts, n, group=group)
    counts = [int(c.item()) for c in counts]
    mx = max(counts)
    pad = torch.zeros((mx, 4), dtype=rows.dtype, device=rows.device)
    pad[:rows.shape[0]] = rows
    if rank == dst:
        bufs = [torch.empty_like(pad) for _ in range(world)]
        dist.gather(pad, bufs, dst=dst, group=group)
        return [b[:c] for b, c in zip(bufs, counts)]
    dist.gather(pad, None, dst=dst, group=group)
    return None


def merge_by_time(streams):
    """Merges per-rank streams of ONE clip (pixel-sharded) into a single stream with non-decreasing
    timestamps (stable: ties keep rank order, like concatenating the bands of each timestamp group)."""
    if not streams:
        return torch.zeros((0, 4), dtype=torch.float32)
    allr = torch.cat(streams, 0)
    order = torch.argsort(allr[:, 0], stable=True)
    return allr[order]


def merge_by_key(streams, keys, offsets, n_shot):
    """Merges the row bands of ONE pixel-sharded clip, generated with EventEmulator(row_order=...), into the stream
    one GPU produces with the same row_order -- bit for bit, because every band sorted its rows by the whole frame's
    keys. Per rank r: streams[r] [N_r, 4] rows with global y, keys[r] [N_r] uint64 and offsets[r] [T + 1] as
    generate_events_band_batch(..., return_keys=True) returns them, n_shot[r] [T] the shot-noise rows that end each
    frame (EventEmulator.last_n_shot). Per frame: the signal rows of all bands by (timestamp, key) -- every band stamps
    an iteration with the same float32 time, the frame maximum being all-reduced; the iterations of a frame must have
    distinct float32 timestamps --, equal keys by (y, x, polarity); then the shot rows by key (ON before OFF, each by
    pixel). Host, numpy. Returns (rows [N, 4] float32, offsets [T + 1] int64)."""
    to_np = lambda a, dt: (a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)).astype(dt, copy=False)
    streams = [to_np(r, np.float32).reshape(-1, 4) for r in streams]
    keys = [to_np(k, np.int64).view(np.uint64) if isinstance(k, torch.Tensor) else np.asarray(k, np.uint64) for k in keys]
    offsets = [np.asarray(o, np.int64) for o in offsets]
    n_shot = [np.asarray(s, np.int64) for s in n_shot]
    if not (len(streams) == len(keys) == len(offsets) == len(n_shot)) or not streams:
        raise ValueError("one stream, key array, offset array and shot-count array per rank")
    T = len(offsets[0]) - 1
    frame, shot = [], []
    for r, k, o, s in zip(streams, keys, offsets, n_shot):
        if len(o) != T + 1 or len(s) != T or o[-1] != len(r) or len(k) != len(r):
            raise ValueError("streams, keys, offsets and n_shot do not fit together")
        f = np.repeat(np.arange(T), np.diff(o))
        frame.append(f)
        shot.append(np.arange(len(r)) >= (o[1:] - s)[f])
    rows, key = np.concatenate(streams, 0), np.concatenate(keys)
    frame, shot = np.concatenate(frame), np.concatenate(shot)
    t = np.where(shot, np.float32(0), rows[:, 0])
    order = np.lexsort((rows[:, 3] < 0, rows[:, 1], rows[:, 2], key, t, shot, frame))
    merged_offsets = np.concatenate([[0], np.cumsum(np.bincount(frame, minlength=T))]).astype(np.int64)
    return np.ascontiguousarray(rows[order]), merged_offsets
