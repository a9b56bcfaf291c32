"""CPU, world_size 2, gloo: the host-side logic of the N>1 path (clip sharding, event-stream gather
with ragged counts, time merge, frame band exchange). No GPU, no model arithmetic."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from v2e_b200 import parallel


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rng = np.random.default_rng(100 + rank)
        n = [5, 0, 9][rank % 3] if rank else 7          # ragged, includes an empty stream
        rows = torch.from_numpy(np.concatenate([np.sort(rng.uniform(0, 1, (n, 1)), 0),
                                                rng.integers(0, 64, (n, 2)), rng.choice([-1.0, 1.0], (n, 1))],
                                               1).astype(np.float32))
        out = parallel.gather_event_streams(rows, dst=0)
        if rank == 0:
            q.put(("gather", [o.numpy() for o in out]))
        else:
            assert out is None
            q.put(("rows", rank, rows.numpy()))
    finally:
        dist.destroy_process_group()


def test_gather_event_streams_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    gathered = [g for g in got if g[0] == "gather"][0]
    others = {g[1]: g[2] for g in got if g[0] == "rows"}
    assert len(gathered[1]) == world
    assert gathered[1][0].shape == (7, 4)
    for r, rows in others.items():
        assert np.array_equal(gathered[1][r], rows)


def test_shard_clips_and_row_bands():
    for world in (1, 2, 4, 8):
        owned = sorted(sum((parallel.shard_clips(11, r, world) for r in range(world)), []))
        assert owned == list(range(11))
        for H, align in ((720, 1), (260, 4), (7, 1), (720, 32)):
            bands = [parallel.row_band(H, r, world, align) for r in range(world)]
            assert bands[0][0] == 0 and bands[-1][1] == H
            assert all(bands[i][1] == bands[i + 1][0] for i in range(world - 1))
            sizes = [b - a for a, b in bands]
            assert max(sizes) - min(sizes) < 2 * align or H < world * align   # last band is clipped to H
    with pytest.raises(ValueError):
        parallel.shard_clips(4, 2, 2)


def test_merge_by_time_is_stable_and_sorted():
    a = torch.tensor([[0.1, 1, 1, 1], [0.2, 2, 2, -1]], dtype=torch.float32)
    b = torch.tensor([[0.1, 9, 9, 1], [0.15, 3, 3, 1], [0.2, 8, 8, 1]], dtype=torch.float32)
    m = parallel.merge_by_time([a, b])
    assert torch.all(m[1:, 0] >= m[:-1, 0])
    assert m[0, 1] == 1 and m[1, 1] == 9          # ties keep rank order
    assert m.shape == (5, 4)


def _exchange_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        H, W, n_pairs, U = 11, 7, 5, 3
        clip = np.arange(n_pairs * U * H * W, dtype=np.int64).reshape(n_pairs * U, H, W) % 251
        p0, p1 = parallel.pair_range(n_pairs, rank, world)
        local = torch.from_numpy(clip[p0 * U:p1 * U].astype(np.uint8))       # this rank's run of the clip
        bands = parallel.exchange_frame_bands(local, H)
        y0, y1 = parallel.row_band(H, rank, world)
        q.put((rank, bands.numpy(), clip[:, y0:y1].astype(np.uint8)))
    finally:
        dist.destroy_process_group()


def test_exchange_frame_bands_world2():
    """One clip over two ranks: ragged runs of frames in, every frame's row band out, in clip order."""
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_exchange_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, bands, want in got:
        assert bands.shape == want.shape and np.array_equal(bands, want), rank


def test_pair_range_covers_all_pairs_contiguously():
    for n, w in [(8, 8), (9, 4), (30, 8), (5, 2), (3, 3)]:
        edges = [parallel.pair_range(n, r, w) for r in range(w)]
        assert edges[0][0] == 0 and edges[-1][1] == n
        for (a0, a1), (b0, b1) in zip(edges, edges[1:]):
            assert a1 == b0 and a1 >= a0
        assert max(b - a for a, b in edges) - min(b - a for a, b in edges) <= 1


def _halo_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from v2e_b200 import parallel
        H, W = 23, 7
        p0, p1 = parallel.pair_range(5, rank, world)
        local = torch.stack([torch.full((H, W), 10 * k, dtype=torch.uint8) + torch.arange(H, dtype=torch.uint8)[:, None]
                             for k in range(p0, p1)])
        out = parallel.exchange_frame_bands(local, H, halo=3)
        q.put((rank, out.numpy(), parallel.band_with_halo(H, rank, world, 3)))
    finally:
        dist.destroy_process_group()


def test_frame_band_exchange_with_halo_rows():
    """Centre-surround sharding (BASELINE config 5): every rank gets its rows PLUS `halo` rows of each neighbour,
    clipped at the image border, of every frame of the clip in clip order."""
    import socket
    import torch.multiprocessing as mp
    world = 3
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_halo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=30)
        assert p.exitcode == 0
    bands = {r: b for r, _, b in res}
    assert bands[0][0] == 0 and bands[world - 1][1] == 23 and bands[1][0] < bands[0][1]     # overlap = the halo
    for r, out, (y0, y1) in res:
        assert out.shape == (5, y1 - y0, 7)
        for k in range(5):
            assert (out[k, :, 0] == (10 * k + np.arange(y0, y1)).astype(np.uint8)).all()
