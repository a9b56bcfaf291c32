"""One clip's pixel model sharded over row bands with the optional models and options of the single-GPU path:
SCIDVS, photoreceptor noise (with and without the centre-surround model), signal / noise labels, and SloMo's auto
upsampling on a pair-sharded clip. Ranks are spawned processes joined by gloo, all sharing the one test GPU (gloo moves
CUDA tensors through the host)."""
import os
import socket

import numpy as np
import pytest

from helpers import EMU_GOLDENS_OPT, TapeRNG, assert_events_equal, canonical, load_golden, split_events

pytestmark = pytest.mark.gpu


def _spawn(world, target, *args, timeout=300):
    """Runs target(rank, world, port, q, *args) on `world` spawned ranks; returns {rank: what the rank put}. A rank
    that raises reports the error instead; the others, which may then wait in a collective, are terminated."""
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_guarded, args=(target, r, world, port, q) + args) for r in range(world)]
    for p in procs:
        p.start()
    res, err = {}, None
    try:
        for _ in range(world):
            r, ok, payload = q.get(timeout=timeout)
            if not ok:
                err = "rank %d: %s" % (r, payload)
                break
            res[r] = payload
    finally:
        for p in procs:
            if err is not None:
                p.terminate()
            p.join(timeout=60)
    assert err is None, err
    for p in procs:
        assert p.exitcode == 0
    return res


def _guarded(target, rank, world, port, q, *args):
    import traceback

    class _Q:
        def put(self, item):
            q.put((item[0], True, item[1]))
    try:
        target(rank, world, port, _Q(), *args)
    except BaseException:
        q.put((rank, False, traceback.format_exc()))
        raise


def _init(rank, world, port):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _own_rows(em, H, t):
    """The rows of state tensor `t` (the handle's rows, halo included) that this rank owns."""
    from v2e_b200.parallel import row_band
    y0, y1 = row_band(H, em.shard[0], em.shard[1])
    ye0 = em.ext_band(H)[0]
    return t.cpu().numpy()[y0 - ye0:y1 - ye0]


_STATES = ("lp_log_frame", "base_log_frame", "photoreceptor_noise_arr", "scidvs_highpass", "scidvs_tau_arr")


def _states(em, H):
    out = {}
    for name in _STATES:
        t = getattr(em, name)
        if t is not None:
            out[name] = _own_rows(em, H, t)
    return out


# ---- 1. replay mode against the reference's goldens ----------------------------------------------------------
def _golden_worker(rank, world, port, q, names, chunk_steps):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator
        from v2e_b200.parallel import row_band
        res = {}
        for name in names:
            g = load_golden(name)
            rng = TapeRNG(g["tape"])
            extra = {"pr_vrms_tape": list(g["pr_vrms"])} if "pr_vrms" in g else {}
            em = EventEmulator(device="cuda:0", shard=(rank, world, None), rng=rng, **extra, **g["kwargs"])
            em.cs_chunk_steps = chunk_steps
            out = [em.generate_events(f, float(t)) for f, t in zip(g["frames"], g["times"])]
            H = g["frames"].shape[1]
            y0, y1 = row_band(H, rank, world)
            res[name] = dict(out=out, on=em.num_events_on, off=em.num_events_off, steps=list(em.cs_steps_taken),
                             states=_states(em, H), band=(y0, y1), K=em.cs_halo_rows(H), exhausted=rng.exhausted())
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_optional_models_match_reference_golden(world):
    """SCIDVS and photoreceptor noise (and both with the centre-surround model) over `world` row bands in replay
    mode: every rank replays the fixture's draws and noise amplitudes. The union of the ranks' rows equals the
    reference's rows per frame, the counters add up to the reference's, and each rank's slice of the state equals the
    reference's (the high-pass within test_optional_models_match_reference_golden's tolerance)."""
    res = _spawn(world, _golden_worker, list(EMU_GOLDENS_OPT), 3)
    for name in EMU_GOLDENS_OPT:
        g = load_golden(name)
        want = split_events(g["events"], g["event_counts"])
        for r in range(world):
            assert res[r][name]["exhausted"], (name, r)
        for i in range(len(want)):
            parts = [res[r][name]["out"][i] for r in range(world) if res[r][name]["out"][i] is not None]
            got = np.concatenate(parts) if parts else None
            assert_events_equal(got, want[i], exact_order=False, ctx="%s frame %d (world %d)" % (name, i, world))
        assert sum(res[r][name]["on"] for r in range(world)) == int(g["num_on"])
        assert sum(res[r][name]["off"] for r in range(world)) == int(g["num_off"])
        for r in range(world):
            y0, y1 = res[r][name]["band"]
            st = res[r][name]["states"]
            for key in ("lp_log_frame", "base_log_frame"):
                assert st[key].dtype == g["state_" + key].dtype and np.array_equal(st[key], g["state_" + key][y0:y1]), (name, r, key)
            if g["kwargs"].get("photoreceptor_noise"):
                assert np.array_equal(st["photoreceptor_noise_arr"], g["state_photoreceptor_noise_arr"][y0:y1]), (name, r)
            if g["kwargs"].get("scidvs"):
                hp = st["scidvs_highpass"]
                tol = 4e-15 if hp.dtype == np.float64 else 2e-6
                assert hp.dtype == g["state_scidvs_highpass"].dtype
                assert np.max(np.abs(hp - g["state_scidvs_highpass"][y0:y1])) <= tol, (name, r)
                assert np.array_equal(st["scidvs_tau_arr"], g["state_scidvs_tau_arr"][y0:y1]), (name, r)
            if "cs_steps_taken" in g:
                assert res[r][name]["steps"] == list(g["cs_steps_taken"]), (name, r)
                assert 0 < res[r][name]["K"] < y1 - y0, (name, r)        # the halo chunk is smaller than the band


# ---- 2. device RNG: sharded equals unsharded ---------------------------------------------------------------
def _frames(H, W, T, seed):
    from test_emulator_gpu import texture_frames
    return texture_frames(H, W, T, seed=seed, speed=2.0)


_DEV_KW = dict(scidvs=True, photoreceptor_noise=True, cutoff_hz=100, leak_rate_hz=0.5, shot_noise_rate_hz=5.0,
               sigma_thres=0.03)
_CS_KW = dict(cs_lambda_pixels=4, cs_tau_p_ms=2.0)


def _device_worker(rank, world, port, q, kw, frames, ts, vrms):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator
        from v2e_b200.parallel import row_band
        H = frames.shape[1]
        em = EventEmulator(device="cuda:0", seed=21, rng_mode="device", shard=(rank, world, None),
                           pr_vrms_tape=[vrms] * len(ts), max_frames_per_step=6, **kw)
        em.cs_chunk_steps = 5
        ye0, ye1 = em.ext_band(H)
        rows, offs = em.generate_events_band_batch(np.ascontiguousarray(frames[:, ye0:ye1]), ts, H)
        draws = {k: em.device_draws(k)["pr_randn"].cpu().numpy() for k in (0, 3)}
        q.put((rank, dict(rows=rows, offs=offs, on=em.num_events_on, off=em.num_events_off, states=_states(em, H),
                          band=row_band(H, rank, world), ext=(ye0, ye1), draws=draws, K=em.cs_halo_rows(H),
                          steps=list(em.cs_steps_taken))))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("centre_surround", [False, True])
def test_sharded_optional_models_device_rng_equal_unsharded(centre_surround):
    """SCIDVS + photoreceptor noise + leak + shot noise in device-RNG mode, 37 x 53 frames over 2 ranks: 53 is not a
    multiple of 4, so the second band starts in the middle of a Philox quad. Rows per frame, counters and the state of
    every owned row equal the unsharded run's bit for bit, and each band's photoreceptor-noise draws are the matching
    rows of the unsharded draws."""
    from v2e_b200 import EventEmulator
    H, W, T, vrms = 37, 53, 12, 0.05
    kw = dict(_DEV_KW, **(_CS_KW if centre_surround else {}))
    fr = _frames(H, W, T, seed=7)
    ts = [k * 1e-3 for k in range(T)]
    one = EventEmulator(device="cuda:0", seed=21, rng_mode="device", pr_vrms_tape=[vrms] * T, max_frames_per_step=6,
                        **kw)
    want, woffs = one.generate_events_batch(fr, ts)
    assert len(want) > 0
    full = {n: getattr(one, n).cpu().numpy() for n in _STATES}
    draws = {k: one.device_draws(k)["pr_randn"].cpu().numpy() for k in (0, 3)}
    res = _spawn(2, _device_worker, kw, fr, ts, vrms)
    assert (res[1]["ext"][0] * W) % 4 != 0                  # a band starts mid-quad
    for i in range(T):
        got = np.concatenate([res[r]["rows"][res[r]["offs"][i]:res[r]["offs"][i + 1]] for r in (0, 1)])
        assert_events_equal(got, want[woffs[i]:woffs[i + 1]], exact_order=False, ctx="frame %d" % i)
    assert sum(res[r]["on"] for r in (0, 1)) == one.num_events_on
    assert sum(res[r]["off"] for r in (0, 1)) == one.num_events_off
    for r in (0, 1):
        y0, y1 = res[r]["band"]
        ye0, ye1 = res[r]["ext"]
        for name in _STATES:
            assert np.array_equal(res[r]["states"][name], full[name][y0:y1]), (r, name)
        for k in draws:
            assert np.array_equal(res[r]["draws"][k], draws[k][ye0:ye1]), (r, k)
        if centre_surround:
            assert res[r]["steps"] == one.cs_steps_taken and 0 < res[r]["K"] < y1 - y0


# ---- 3. one noise amplitude on every rank ---------------------------------------------------------------------
def _vrms_worker(rank, world, port, q, frames, ts):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator
        em = EventEmulator(device="cuda:0", seed=3, rng_mode="device", shard=(rank, world, None),
                           **dict(_DEV_KW, cutoff_hz=30))
        H = frames.shape[1]
        ye0, ye1 = em.ext_band(H)
        vr = []
        for f, t in zip(frames, ts):
            em.generate_events_band(f[ye0:ye1], t, H)
            vr.append(em.photoreceptor_noise_vrms)
        q.put((rank, vr))
    finally:
        dist.destroy_process_group()


def test_sharded_noise_amplitude_is_the_same_on_every_rank():
    """Without a tape the amplitude is calibrated with an unseeded generator (as in the reference); the first rank's
    value is broadcast, so every rank uses the same amplitude after every frame, also when the frame rate changes."""
    T = 8
    fr = _frames(30, 40, T, seed=2)
    ts = [k * 1e-3 for k in range(4)] + [3e-3 + k * 2e-3 for k in range(1, T - 3)]     # 1 kHz, then 500 Hz
    res = _spawn(3, _vrms_worker, fr, ts)
    assert res[0][0] is None and all(v is not None and v > 0 for v in res[0][1:])
    for r in (1, 2):
        assert res[r] == res[0], (r, res[r], res[0])


# ---- 4. signal / noise labels ------------------------------------------------------------------------------
def _labels_worker(rank, world, port, q, kw, frames, ts):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator
        em = EventEmulator(device="cuda:0", seed=21, rng_mode="device", shard=(rank, world, None),
                           label_signal_noise=True, max_frames_per_step=5, **kw)
        H = frames.shape[1]
        ye0, ye1 = em.ext_band(H)
        rows, offs, labels = em.generate_events_band_batch(np.ascontiguousarray(frames[:, ye0:ye1]), ts, H,
                                                           return_labels=True)
        q.put((rank, (rows, offs, labels)))
    finally:
        dist.destroy_process_group()


def _sorted_rows_labels(rows, labels):
    """(t, x, y, p, label) rows in an order-insensitive form."""
    a = np.concatenate([np.asarray(rows, np.float64), np.asarray(labels, np.float64)[:, None]], 1)
    return a[np.lexsort((a[:, 4], a[:, 3], a[:, 1], a[:, 2], a[:, 0]))]


@pytest.mark.parametrize("case", [
    # multi-frame kernels (refractory filter off): shot-noise rows at the end of every band's frame block
    dict(cutoff_hz=300, leak_rate_hz=0.5, shot_noise_rate_hz=20.0),
    # refractory filter on: chunks rejected and replayed frame by frame
    dict(cutoff_hz=200, leak_rate_hz=0.5, shot_noise_rate_hz=20.0, refractory_period_s=0.004, pos_thres=0.05,
         neg_thres=0.05, sigma_thres=0.01),
])
def test_sharded_labels_equal_unsharded(case):
    """label_signal_noise on a row band: per frame, the union over the ranks of (row, label) equals the unsharded
    emulator's, with shot-noise rows (label 0) present."""
    from v2e_b200 import EventEmulator
    H, W, T = 37, 53, 11
    fr = _frames(H, W, T, seed=5)
    ts = [k * 1e-2 for k in range(T)]
    one = EventEmulator(device="cuda:0", seed=21, rng_mode="device", label_signal_noise=True, max_frames_per_step=5,
                        **case)
    want, woffs, wlab = one.generate_events_batch(fr, ts, return_labels=True)
    assert (~wlab).sum() > 0 and wlab.sum() > 0
    res = _spawn(2, _labels_worker, case, fr, ts)
    for i in range(T):
        got_r = np.concatenate([res[r][0][res[r][1][i]:res[r][1][i + 1]] for r in (0, 1)])
        got_l = np.concatenate([res[r][2][res[r][1][i]:res[r][1][i + 1]] for r in (0, 1)])
        a, b = woffs[i], woffs[i + 1]
        assert np.array_equal(_sorted_rows_labels(got_r, got_l), _sorted_rows_labels(want[a:b], wlab[a:b])), i


# ---- 5. auto-upsampled SloMo on a pair-sharded clip ---------------------------------------------------------
_AUTO_KW = dict(cutoff_hz=200, leak_rate_hz=0.2, shot_noise_rate_hz=10.0, refractory_period_s=0.001, sigma_thres=0.02)


def _slomo(auto=True):
    from test_slomo_gpu import _weights
    from v2e_b200 import SuperSloMo
    fc, at = _weights(5)
    return SuperSloMo(model=None, auto_upsample=auto, upsampling_factor=None, batch_size=2,
                      state_dicts={"state_dictFC": fc, "state_dictAT": at})


def _auto_worker(rank, world, port, q, frames):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator, V2EPipeline
        sl = _slomo()
        em = EventEmulator(device="cuda:0", seed=9, rng_mode="device", shard=(rank, world, None),
                           label_signal_noise=True, **_AUTO_KW)
        rows, t, nf, labels = V2EPipeline(sl, em).run_clip_sharded(frames, 0.2, return_labels=True)
        sl.cleanup()
        q.put((rank, (rows, t, nf, labels)))
    finally:
        dist.destroy_process_group()


def _auto_clip(seed):
    """8 frames (7 pairs: batches of 2, 2, 2, 1) whose motion and contrast change from batch to batch."""
    rng = np.random.default_rng(seed)
    big = np.kron(rng.integers(30, 220, (20, 40)).astype(np.uint8), np.ones((8, 8), np.uint8)).astype(np.float32)
    shifts = np.cumsum([0, 1, 1, 6, 6, 14, 2, 2])
    gains = [1.0, 1.0, 0.5, 0.5, 1.0, 1.0, 0.3, 0.3]
    return np.stack([np.clip(128 + g * (big[5:5 + 96, s:s + 128] - 128), 0, 255).astype(np.uint8)
                     for s, g in zip(shifts, gains)])


def test_auto_upsampled_clip_sharded_over_two_ranks_matches_single_gpu():
    """SloMo with a U chosen per batch (v2e's auto timestamp resolution) on a clip sharded over 2 ranks by whole
    batches: the ranks gather each other's U's and build the clip's interpTimes, so the times, the frame count and the
    events (with their signal / noise labels) equal the single-GPU V2EPipeline.run on the whole clip."""
    import torch
    from v2e_b200 import EventEmulator, V2EPipeline
    from v2e_b200.parallel import batch_pair_range
    sl = _slomo()
    frames = None
    for seed in range(8):        # a clip whose batches get at least two different U's
        cand = _auto_clip(seed)
        _, _, _, ups = sl.interpolate_frames(cand, return_ups=True)
        if len(set(ups)) >= 2:
            frames = cand
            break
    assert frames is not None, "no candidate clip with two different per-batch U's"
    p0, p1 = batch_pair_range(frames.shape[0] - 1, 2, 1, 2)
    assert (p1 - p0) % 2 == 1                               # the last rank holds the clip's short final batch
    em = EventEmulator(device="cuda:0", seed=9, rng_mode="device", **_AUTO_KW)
    ev, offs, t, nf = V2EPipeline(sl, em).run(frames, 0.2, copy=True)
    assert ev.shape[0] > 0
    # the labels of the same run
    interp, times, _ = sl.interpolate_frames(frames)
    em2 = EventEmulator(device="cuda:0", seed=9, rng_mode="device", label_signal_noise=True, **_AUTO_KW)
    ev2, _, lab = em2.generate_events_batch(interp, t, return_labels=True)
    assert np.array_equal(canonical(ev2), canonical(ev)) and (~lab).sum() > 0
    sl.cleanup()
    del interp
    torch.cuda.empty_cache()
    res = _spawn(2, _auto_worker, frames)
    for r in (0, 1):
        rows, tr, nfr, _ = res[r]
        assert nfr == nf and np.array_equal(tr, t), r
    rows = np.concatenate([res[r][0] for r in (0, 1)])
    labels = np.concatenate([res[r][3] for r in (0, 1)])
    assert np.array_equal(_sorted_rows_labels(rows, labels), _sorted_rows_labels(ev2, lab))
