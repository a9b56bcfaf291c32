"""GPU: EventEmulator(row_order="canonical" | "shuffled") against oracle/row_order.py, bit for bit and UNSORTED.

The oracle is fed the device's own Philox draws (as tests/test_emulator_device_rng.py does), returns its rows in the
reference's order before randperm, and oracle/row_order.py turns those into the shuffled order. The device must return
exactly those bytes whichever kernels, chunk sizes, replays and buffer growth produced the rows, and the row bands of a
sharded clip must merge (v2e_b200.parallel.merge_by_key) into the unsharded stream."""
import ctypes

import numpy as np
import pytest
import torch

import row_order
from helpers import DeviceDrawRNG, canonical
from test_emulator_device_rng import C3_PARAMS, CLI_DEFAULTS, _state, draws_from, texture_frames
from test_row_order import oracle_clip
from test_sharded_options import _init, _spawn

pytestmark = pytest.mark.gpu

SEED = 1234
MODES = ["canonical", "shuffled"]


def _emulator(order, **kw):
    from v2e_b200 import EventEmulator
    return EventEmulator(device="cuda", rng_mode="device", seed=SEED, row_order=order, **kw)


def _fused_counters(em):
    v = [ctypes.c_longlong(0) for _ in range(4)]
    em._lib.v2e_emu_fused_stats(em._h, ctypes.byref(v[0]), ctypes.byref(v[1]))
    em._lib.v2e_emu_fused_frames(em._h, ctypes.byref(v[2]), ctypes.byref(v[3]))
    return tuple(x.value for x in v)            # chunks, rejected, frames multi, frames single


def _order_stats(em):
    b, r = ctypes.c_uint64(0), ctypes.c_longlong(0)
    em._lib.v2e_emu_order_stats(em._h, ctypes.byref(b), ctypes.byref(r))
    return b.value, r.value


def _oracle(em, kw, frames, ts):
    """The oracle on the device's draws: (rows in the reference's pre-shuffle order, offsets, iteration counts, shot
    rows, oracle)."""
    from emu_oracle import OracleEmulator
    rng = DeviceDrawRNG(draws_from(em), photoreceptor_noise=kw.get("photoreceptor_noise", False))
    orc = OracleEmulator(seed=SEED, rng=rng, shuffle=False, **kw)
    return oracle_clip(orc, frames, ts, rng=rng) + (orc,)


def _want(mode, rows, offs, iters, n_shot, W):
    return rows if mode == "canonical" else row_order.order_rows(rows, offs, iters, n_shot, "shuffled", seed=SEED, W=W)


def _assert_rows(got, want, offs, ctx):
    assert got.shape == want.shape, (ctx, got.shape, want.shape)
    if got.tobytes() != want.tobytes():
        bad = int(np.flatnonzero(np.any(got != want, axis=1))[0])
        f = int(np.searchsorted(offs, bad, side="right") - 1)
        raise AssertionError("%s: row %d (frame %d) is %s, want %s" % (ctx, bad, f, got[bad], want[bad]))


# ---- 5. canonical = the oracle's rows as they stand ------------------------------------------------------------
@pytest.mark.parametrize("size", [(13, 37), (37, 53), (260, 346)])
def test_canonical_rows_equal_the_oracles_unsorted(size):
    H, W = size
    T = 10
    fr, ts = texture_frames(H, W, T, seed=H), [k / 300. for k in range(T)]
    em = _emulator("canonical", max_frames_per_step=24, **CLI_DEFAULTS)
    rows, offs = em.generate_events_batch(fr, ts)
    want, woffs, iters, n_shot, orc = _oracle(em, CLI_DEFAULTS, fr, ts)
    assert len(want) > 200 and max(len(c) for c in iters) >= 2
    assert np.array_equal(offs, woffs)
    _assert_rows(rows, want, offs, "canonical %dx%d" % (W, H))
    assert (em.num_events_on, em.num_events_off, em.num_events_total) == \
        (orc.num_events_on, orc.num_events_off, orc.num_events_total)
    dev, ref = _state(em, True), _state(orc, False)
    assert dev.keys() == ref.keys()
    for k in ref:
        assert dev[k].dtype == ref[k].dtype and np.array_equal(dev[k], ref[k]), k


# ---- 6. shuffled = the oracle's rows in key order ---------------------------------------------------------------
def test_shuffled_rows_equal_the_oracles_in_key_order_and_mix_on_and_off():
    H, W, T = 260, 346, 9
    fr, ts = texture_frames(H, W, T, seed=2), [k / 300. for k in range(T)]
    em = _emulator("shuffled", max_frames_per_step=24, **C3_PARAMS)
    rows, offs = em.generate_events_batch(fr, ts)
    crows, woffs, iters, n_shot, _ = _oracle(em, C3_PARAMS, fr, ts)
    assert np.array_equal(offs, woffs) and n_shot.sum() > 100
    want = _want("shuffled", crows, woffs, iters, n_shot, W)
    _assert_rows(rows, want, offs, "shuffled")
    assert rows.tobytes() != crows.tobytes()
    # ON and OFF rows of a large iteration alternate often; in the canonical order they form two runs
    checked = 0
    for f in range(T):
        a = int(offs[f])
        for c in iters[f]:
            pol = rows[a:a + c, 3]
            n_on = int(np.sum(pol > 0))
            if min(n_on, c - n_on) >= 50:
                runs = 1 + int(np.sum(pol[1:] != pol[:-1]))
                assert runs > 20, (f, runs)
                assert 1 + int(np.sum(np.diff(crows[a:a + c, 3]) != 0)) == 2
                checked += 1
            a += int(c)
    assert checked >= 3
    assert np.all(np.diff(rows[:, 0]) >= 0)                     # timestamps stay non-decreasing


# ---- 7. the bytes do not depend on how the rows were produced ------------------------------------------------
def _jump_clip(H, W, T):
    """A slowly moving texture with one block that jumps from dark to bright in frame 5: enough events of one pixel in
    one frame that refractory_period_s > dt / max_n, so the multi-frame kernels reject the chunk."""
    fr = (texture_frames(H, W, T, seed=11, speed=1.0) // 4 + 90).astype(np.uint8)
    fr[:5, 8:24, 8:40] = 4
    fr[5:, 8:24, 8:40] = 250
    return fr


@pytest.mark.parametrize("mode", MODES)
def test_rows_are_the_same_bytes_on_every_path(mode):
    H, W, T = 64, 96, 12
    fr, ts = _jump_clip(H, W, T), [k / 300. for k in range(T)]
    kw = dict(CLI_DEFAULTS, leak_rate_hz=1.0, shot_noise_rate_hz=20.0)
    runs = {}
    for name, fused, mfps, hint in (("fused", True, 80, None), ("again", True, 80, None), ("classic", False, 80, None),
                                    ("mfps1", True, 1, None), ("mfps3", True, 3, None), ("resume", True, 80, 64),
                                    ("resume_classic", False, 3, 64)):
        em = _emulator(mode, fused=fused, max_frames_per_step=mfps, **kw)
        em.event_rows_hint = hint
        rows, offs = em.generate_events_batch(fr, ts)
        runs[name] = (rows.tobytes(), offs.tolist(), _fused_counters(em), em._ev_dev.shape[0])
    chunks, rejected, multi, single = runs["fused"][2]
    assert chunks >= 1 and rejected >= 1 and multi + single == T - 1, runs["fused"][2]
    assert runs["classic"][2][0] == 0
    assert runs["resume"][3] > 64                                # the 64-row buffer had to grow
    for name, r in runs.items():
        assert r[1] == runs["fused"][1], name
        assert r[0] == runs["fused"][0], name
    # and they are the oracle's
    em = _emulator(mode, max_frames_per_step=80, **kw)
    rows, offs = em.generate_events_batch(fr, ts)
    crows, woffs, iters, n_shot, _ = _oracle(em, kw, fr, ts)
    _assert_rows(rows, _want(mode, crows, woffs, iters, n_shot, W), offs, mode)
    assert rows.tobytes() == runs["fused"][0]
    # frame by frame through generate_events
    em = _emulator(mode, **kw)
    single_rows = [em.generate_events(f, t) for f, t in zip(fr, ts)]
    assert np.concatenate([r for r in single_rows if r is not None]).tobytes() == runs["fused"][0]


# ---- 8. extremes at 1280 x 720 -----------------------------------------------------------------------------------
def _extreme_clip():
    H, W = 720, 1280
    fr = np.empty((6, H, W), np.uint8)
    fr[0] = 100
    fr[1] = 130          # every pixel fires ON once
    fr[2] = 80           # every pixel fires OFF twice
    fr[3] = 80
    fr[3, 700, 1279] = 110   # one event
    fr[4] = fr[3]        # none
    fr[5] = fr[3]
    return fr


@pytest.mark.parametrize("mode", MODES)
def test_extreme_segments_at_1280x720(mode):
    H, W = 720, 1280
    fr, ts = _extreme_clip(), [k / 300. for k in range(6)]
    kw = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.0, cutoff_hz=0.0, leak_rate_hz=0.0, shot_noise_rate_hz=0.0)
    em = _emulator(mode, max_frames_per_step=8, **kw)
    rows, offs = em.generate_events_batch(fr, ts)
    assert np.diff(offs).tolist() == [0, H * W, 2 * H * W, 1, 0, 0]
    assert np.all(rows[:H * W, 3] == 1) and np.all(rows[H * W:3 * H * W, 3] == -1)
    crows, woffs, iters, n_shot, _ = _oracle(em, kw, fr, ts)
    assert [len(c) for c in iters] == [0, 1, 2, 1, 0, 0]
    _assert_rows(rows, _want(mode, crows, woffs, iters, n_shot, W), offs, mode)
    plain, poffs = _emulator(None, max_frames_per_step=8, **kw).generate_events_batch(fr, ts)
    assert np.array_equal(poffs, offs)
    for f in range(6):
        assert np.array_equal(canonical(plain[poffs[f]:poffs[f + 1]]), canonical(rows[offs[f]:offs[f + 1]])), f


@pytest.mark.parametrize("mode", MODES)
def test_shot_noise_only_frames_at_1280x720(mode):
    H, W, T = 720, 1280, 4
    fr, ts = np.full((T, H, W), 120, np.uint8), [k / 300. for k in range(T)]
    kw = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=0.0, leak_rate_hz=0.0, shot_noise_rate_hz=5.0)
    em = _emulator(mode, max_frames_per_step=8, **kw)
    rows, offs = em.generate_events_batch(fr, ts)
    crows, woffs, iters, n_shot, _ = _oracle(em, kw, fr, ts)
    assert n_shot[1:].min() > 1000 and n_shot.sum() > 0.9 * len(crows)             # next to nothing but shot noise
    _assert_rows(rows, _want(mode, crows, woffs, iters, n_shot, W), offs, mode)
    for f in range(T):                                            # shot rows are canonical in both modes
        assert np.array_equal(rows[offs[f + 1] - n_shot[f]:offs[f + 1]], crows[offs[f + 1] - n_shot[f]:offs[f + 1]])
    plain, poffs = _emulator(None, max_frames_per_step=8, **kw).generate_events_batch(fr, ts)
    assert np.array_equal(canonical(plain), canonical(rows)) and np.array_equal(poffs, offs)


# ---- 9. row_order=None is what it was ------------------------------------------------------------------------
def test_no_row_order_leaves_the_groups_and_the_counters_alone():
    H, W, T = 64, 96, 12
    fr, ts = _jump_clip(H, W, T), [k / 300. for k in range(T)]
    kw = dict(CLI_DEFAULTS, leak_rate_hz=1.0, shot_noise_rate_hz=20.0)
    plain = _emulator(None, max_frames_per_step=80, **kw)
    prow, poffs = plain.generate_events_batch(fr, ts)
    assert _order_stats(plain) == (0, 0)                          # nothing allocated, nothing ordered
    for mode in MODES:
        em = _emulator(mode, max_frames_per_step=80, **kw)
        rows, offs = em.generate_events_batch(fr, ts)
        assert np.array_equal(offs, poffs) and _fused_counters(em) == _fused_counters(plain)
        nbytes, nrows = _order_stats(em)
        assert nbytes > 0 and nrows == len(rows)
        crows, woffs, iters, n_shot, _ = _oracle(em, kw, fr, ts)
        for f in range(T):
            # the unordered run holds, group by group, the rows the canonical order holds there
            a = int(poffs[f])
            for c in iters[f]:
                blk, ref = prow[a:a + c], crows[a:a + c]
                n_on = int(np.sum(ref[:, 3] > 0))
                assert np.array_equal(canonical(blk[:n_on]), canonical(ref[:n_on])), (f, "ON")
                assert np.array_equal(canonical(blk[n_on:]), canonical(ref[n_on:])), (f, "OFF")
                a += int(c)
            assert np.array_equal(canonical(prow[a:poffs[f + 1]]), canonical(crows[a:poffs[f + 1]])), (f, "shot")


# ---- 10. labels and the text sink ---------------------------------------------------------------------------
def test_labels_and_text_of_shuffled_rows():
    import text_sink_oracle
    from v2e_b200 import sinks
    H, W, T = 64, 96, 8
    fr, ts = texture_frames(H, W, T, seed=3), [k / 300. for k in range(T)]
    kw = dict(CLI_DEFAULTS, shot_noise_rate_hz=40.0)
    em = _emulator("shuffled", label_signal_noise=True, max_frames_per_step=5, **kw)
    rows, offs, labels = em.generate_events_batch(fr, ts, return_device=True, return_labels=True)
    rows, labels = rows.clone(), labels.clone()
    crows, woffs, iters, n_shot, _ = _oracle(em, kw, fr, ts)
    want = _want("shuffled", crows, woffs, iters, n_shot, W)
    _assert_rows(rows.cpu().numpy(), want, offs, "labels")
    want_lab = np.ones(len(want), bool)
    for f in range(T):
        want_lab[woffs[f + 1] - n_shot[f]:woffs[f + 1]] = False
    assert n_shot.sum() > 20 and np.array_equal(labels.cpu().numpy().astype(bool), want_lab)
    assert sinks.events_to_text(rows).cpu().numpy().tobytes() == text_sink_oracle.text_body(want)
    assert sinks.events_to_text(rows, labels).cpu().numpy().tobytes() == text_sink_oracle.text_body(want, want_lab)
    host = _emulator("shuffled", label_signal_noise=True, max_frames_per_step=5, **kw)
    hrows, _ = host.generate_events_batch(fr, ts, copy=False)
    assert hrows.tobytes() == want.tobytes()


# ---- 11. sharded: bands in key order, merged = unsharded ---------------------------------------------------------
_SHARD_KW = dict(cutoff_hz=300, leak_rate_hz=1.0, shot_noise_rate_hz=20.0, sigma_thres=0.03)


def _band_worker(rank, world, port, q, mode, frames, ts, kw, backend="gloo"):
    import torch.distributed as dist
    if backend == "gloo":
        _init(rank, world, port)
        dev = "cuda:0"
    else:
        import os
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        dev = "cuda:%d" % rank
    try:
        from v2e_b200 import EventEmulator
        H = frames.shape[1]
        em = EventEmulator(device=dev, seed=SEED, rng_mode="device", shard=(rank, world, None), row_order=mode,
                           max_frames_per_step=5, **kw)
        ye0, ye1 = em.ext_band(H)
        rows, offs, keys = em.generate_events_band_batch(np.ascontiguousarray(frames[:, ye0:ye1]), ts, H,
                                                         return_keys=True)
        q.put((rank, (rows, offs, keys, em.last_n_shot)))
    finally:
        dist.destroy_process_group()


def _check_bands(res, world, mode, want, woffs, W):
    from v2e_b200.parallel import merge_by_key
    parts = [res[r] for r in range(world)]
    for rows, offs, keys, n_shot in parts:
        assert keys.dtype == np.uint64 and len(keys) == len(rows) > 0
        for f in range(len(offs) - 1):
            a, b = int(offs[f]), int(offs[f + 1])
            s = b - int(n_shot[f])
            # signal rows by (time, key), shot rows by key
            t, k = rows[a:s, 0], keys[a:s]
            assert np.all((np.diff(t) > 0) | ((np.diff(t) == 0) & (k[1:] > k[:-1])))
            assert np.all(np.diff(keys[s:b].astype(np.int64)) > 0)      # at most 33 bits: (p < 0) << 32 | pixel
    merged, moffs = merge_by_key([p[0] for p in parts], [p[2] for p in parts], [p[1] for p in parts],
                                 [p[3] for p in parts])
    assert np.array_equal(moffs, woffs)
    _assert_rows(merged, want, woffs, "%s over %d bands" % (mode, world))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world,refr", [(2, 0.0), (3, 0.004)])
def test_sharded_bands_merge_into_the_unsharded_rows(world, refr, mode):
    """refr = 0: the multi-frame kernels run every chunk; 0.004: chunks are rejected and replayed frame by frame."""
    H, W, T = 37, 53, 11
    fr, ts = texture_frames(H, W, T, seed=5, speed=2.0), [k * 1e-2 for k in range(T)]
    kw = dict(_SHARD_KW, refractory_period_s=refr)
    one = _emulator(mode, max_frames_per_step=5, **kw)
    want, woffs = one.generate_events_batch(fr, ts)
    assert len(want) > 1000
    res = _spawn(world, _band_worker, mode, fr, ts, kw)
    _check_bands(res, world, mode, want, woffs, W)


def test_sharded_bands_merge_over_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    import socket
    import torch.multiprocessing as mp
    H, W, T = 37, 53, 11
    fr, ts = texture_frames(H, W, T, seed=5, speed=2.0), [k * 1e-2 for k in range(T)]
    want, woffs = _emulator("shuffled", max_frames_per_step=5, **_SHARD_KW).generate_events_batch(fr, ts)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_band_worker, args=(r, 2, port, q, "shuffled", fr, ts, _SHARD_KW, "nccl"))
             for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    _check_bands(res, 2, "shuffled", want, woffs, W)


def test_pipeline_rows_come_out_ordered():
    """V2EPipeline.run passes the emulator through: its rows are the ordered rows of the interpolated frames."""
    from test_sharded_options import _slomo
    from v2e_b200 import V2EPipeline
    rng = np.random.default_rng(0)
    big = np.kron(rng.integers(30, 220, (20, 40)).astype(np.uint8), np.ones((8, 8), np.uint8))
    frames = np.stack([big[5:5 + 96, s:s + 128] for s in (0, 2, 4, 6)])
    sl = _slomo()
    kw = dict(cutoff_hz=200, leak_rate_hz=0.2, shot_noise_rate_hz=10.0, sigma_thres=0.02)
    ev, offs, t, nf = V2EPipeline(sl, _emulator("shuffled", **kw)).run(frames, 0.2, copy=True)
    interp, _, _ = sl.interpolate_frames(frames)
    em = _emulator("shuffled", **kw)
    rows, roffs = em.generate_events_batch(interp, t)
    sl.cleanup()
    assert len(ev) > 0 and np.array_equal(offs, roffs) and ev.tobytes() == rows.tobytes()
    crows, woffs, iters, n_shot, _ = _oracle(em, kw, interp.cpu().numpy(), t)
    _assert_rows(rows, _want("shuffled", crows, woffs, iters, n_shot, frames.shape[2]), roffs, "pipeline")


# ---- 12. refusals ---------------------------------------------------------------------------------------------
def test_row_order_value_errors():
    from v2e_b200 import EventEmulator
    with pytest.raises(ValueError):
        EventEmulator(device="cuda", rng_mode="device", row_order="sorted")
    with pytest.raises(ValueError):
        EventEmulator(device="cuda", rng_mode="replay", row_order="canonical")
    with pytest.raises(ValueError):
        EventEmulator(device="cuda", row_order="shuffled")          # replay is the default mode
    em = EventEmulator(device="cuda", rng_mode="device", shard=(0, 1, None))
    with pytest.raises(ValueError):
        em.generate_events_band_batch(np.zeros((2, 8, 8), np.uint8), [0.0, 1e-3], 8, return_keys=True)
