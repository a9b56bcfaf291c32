"""GPU: the centre-surround pixel model with a float32 photoreceptor state (cutoff_hz = 0, the class default and what
the 'clean' preset sets) against the CPU oracle and the reference's fixtures, bit for bit, on every device path of its
Euler iteration -- the float32 twin of test_emulator_centre_surround.py:
  - the fixtures of oracle/make_golden_cs32.py in replay mode (rows in the reference's order, counters, state);
  - one cooperative launch per frame (emu_csdvs_iter_kernel<float>), in this process;
  - one kernel per step (emu_csdvs_step_kernel<float> + emu_csdvs_finish_kernel), in a spawned process with
    V2E_CS_COOP=0;
  - generate_events_batch with the device RNG, the oracle fed the device's draws;
  - pixel-sharded row bands (v2e_emu_cs_*, float32 halo exchange) over 2 and 3 gloo ranks on one GPU, and over NCCL on
    two GPUs.
Every case compares rows, cs_steps_taken and float32 cs_surround_frame, lp_log_frame and base_log_frame.

Shapes: 1280x720 with the parameters of the reference's CSDVS_test run configuration (lambda 15 px, tau_p 20 ms,
thresholds 0.15, no noise) at 1/1500 s per frame (38 Euler steps), and 141x141, 141x142, 20x974 and 37x53 on both sides
of the float32 Laplacian's summation-order switch, with per-pixel thresholds, leak, shot noise and the refractory
filter on."""
import functools
import os
import socket

import numpy as np
import pytest
import torch

import bench
from helpers import DeviceDrawRNG, TapeRNG, assert_events_equal, load_golden, run_oracle_with_draws, split_events

pytestmark = pytest.mark.gpu

CS32_GOLDENS = ["emu_cs32_120x176", "emu_cs32_37x53", "emu_cs32_scidvs", "emu_cs32_clean"]
DT = 1 / 1500.
# .idea/runConfigurations/CSDVS_test.xml of the reference
CSDVS_TEST = dict(pos_thres=0.15, neg_thres=0.15, sigma_thres=0, cutoff_hz=0, leak_rate_hz=0, shot_noise_rate_hz=0,
                  cs_lambda_pixels=15, cs_tau_p_ms=20)
NOISY = dict(CSDVS_TEST, sigma_thres=0.03, leak_rate_hz=0.1, shot_noise_rate_hz=2.0, refractory_period_s=1e-4)
SMALL = ["141x141", "141x142", "20x974", "37x53"]
STATES = ("cs_surround_frame", "lp_log_frame", "base_log_frame")
# pixel-sharded runs: world -> [(case, Euler steps per chunk = halo rows K)]. 38 steps per frame: K = 19 ends the full
# iteration on a chunk boundary, the uniform pair's single step ends inside the first chunk; K = 5 / 3 / 7 leave a
# partial last chunk
SHARDED = {2: [("big", 19), ("37x53", 5), ("20x974", 3)], 3: [("big", 16), ("141x142", 7)]}


def case_inputs(name):
    """(frames [T, H, W] uint8, times, kwargs): a uniform pair first (the iteration stops after one step), then the
    block texture of bench.py moving, with one static pair."""
    if name == "big":
        H, W, kw = 720, 1280, CSDVS_TEST
        src = 96 + bench.block_texture_clip(H, W, 3, seed=7, block=32) // 4       # grey levels 96 .. 159
    else:
        H, W = (int(v) for v in name.split("x"))
        kw = NOISY
        src = bench.block_texture_clip(H, W, 3, seed=H * W, block=1, shift=(3, 2))     # high contrast
    grey = np.full((H, W), 128, np.uint8)
    frames = np.stack([grey, grey, src[0], src[1], src[1], src[2]])
    return frames, np.arange(len(frames)) * DT, kw


def _result(em, out, whole_frame=True):
    r = dict(rows=[np.zeros((0, 4), np.float32) if e is None else np.asarray(e) for e in out],
             steps=list(em.cs_steps_taken))
    if whole_frame:
        for k in STATES:
            r[k] = getattr(em, k).cpu().numpy()
        r["paths"] = em.cs_paths()
    return r


def run_device(name):
    from v2e_b200 import EventEmulator
    frames, times, kw = case_inputs(name)
    em = EventEmulator(device="cuda", seed=11, **kw)
    out = [em.generate_events(f, float(t)) for f, t in zip(frames, times)]
    return _result(em, out)


@functools.lru_cache(maxsize=None)
def oracle(name):
    from emu_oracle_cs32 import OracleEmulatorCS32
    frames, times, kw = case_inputs(name)
    em = OracleEmulatorCS32(seed=11, **kw)
    out = [em.generate_events(f, float(t)) for f, t in zip(frames, times)]
    return dict(rows=[np.zeros((0, 4), np.float32) if e is None else e for e in out], steps=list(em.cs_steps_taken),
                cs_surround_frame=em.surround, lp_log_frame=em.lp, base_log_frame=em.base)


def assert_matches(got, want, ctx):
    assert got["steps"] == want["steps"], (ctx, got["steps"], want["steps"])
    assert len(got["rows"]) == len(want["rows"])
    for i, (g, w) in enumerate(zip(got["rows"], want["rows"])):
        assert_events_equal(g, w, exact_order=False, ctx="%s frame %d" % (ctx, i))
    for k in STATES:
        if k in got:
            a, b = got[k], want[k]
            assert a.dtype == np.float32 and b.dtype == np.float32 and a.shape == b.shape, (ctx, k, a.dtype, b.dtype)
            n = int((a.view(np.uint32) != b.view(np.uint32)).sum())
            assert n == 0, "%s: %s differs at %d pixels" % (ctx, k, n)


# ---- the reference's fixtures, replay mode ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", CS32_GOLDENS)
def test_reference_golden_bit_exact_f32(name):
    """Rows (values and order), counters, cs_steps_taken and the float32 lp / base / surround equal to the reference's
    CPU output. emu_cs32_clean takes the reference's gradients_csdvs route: cutoff_hz=300 then set_dvs_params('clean')."""
    from v2e_b200 import EventEmulator
    g = load_golden(name)
    rng = TapeRNG(g["tape"])
    em = EventEmulator(device="cuda", rng=rng, **g["kwargs"])
    if "dvs_params" in g:
        em.set_dvs_params(str(g["dvs_params"]))
    want = split_events(g["events"], g["event_counts"])
    for i, (f, t) in enumerate(zip(g["frames"], g["times"])):
        ev = em.generate_events(f, float(t))
        assert_events_equal(ev, want[i], exact_order=True, ctx="%s frame %d" % (name, i))
    assert rng.exhausted()
    assert em.num_events_on == int(g["num_on"]) and em.num_events_off == int(g["num_off"])
    assert em.cs_steps_taken == list(g["cs_steps_taken"])
    for key, attr in (("state_base_log_frame", "base_log_frame"), ("state_lp_log_frame", "lp_log_frame"),
                      ("state_cs_surround_frame", "cs_surround_frame")):
        got = getattr(em, attr).cpu().numpy()
        assert got.dtype == np.float32 and g[key].dtype == np.float32, key
        assert np.array_equal(got.view(np.uint32), g[key].view(np.uint32)), key


def test_class_defaults_run_centre_surround():
    """EventEmulator(cs_lambda_pixels=15, cs_tau_p_ms=20) with every other argument at its default (cutoff_hz = 0)."""
    from v2e_b200 import EventEmulator
    em = EventEmulator(device="cuda", cs_lambda_pixels=15, cs_tau_p_ms=20)
    frames, times, _ = case_inputs("37x53")
    for f, t in zip(frames, times):
        em.generate_events(f, float(t))
    assert em.cs_surround_frame.dtype == torch.float32 and len(em.cs_steps_taken) == len(frames) - 1


# ---- cooperative launch, this process ---------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def coop(name):
    return run_device(name)


@pytest.mark.parametrize("name", ["big"] + SMALL)
def test_cooperative_path_matches_oracle_f32(name):
    got, want = coop(name), oracle(name)
    assert got["paths"] == (len(want["steps"]), 0), got["paths"]        # one cooperative launch per frame, no fallback
    assert_matches(got, want, name + " cooperative")
    print("%s cooperative: %d rows, cs_steps_taken %s" % (name, sum(len(r) for r in want["rows"]), want["steps"]))
    assert 1 in want["steps"] and max(want["steps"]) == 38, want["steps"]


# ---- one kernel per step, spawned process -----------------------------------------------------------------------------
def _per_step_worker(names, q):
    os.environ["V2E_CS_COOP"] = "0"     # read once, at the first centre-surround frame of the process
    try:
        for name in names:
            q.put((name, run_device(name)))
    except BaseException as e:          # report instead of leaving the parent waiting
        q.put(("error", repr(e)))


def _spawn(target, args_list, n_results):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=a + (q,)) for a in args_list]
    for p in procs:
        p.start()
    res = []
    try:
        for _ in range(n_results):
            res.append(q.get(timeout=900))
            assert res[-1][0] != "error", res[-1]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for p in procs:
        assert p.exitcode == 0, p.exitcode
    return res


@functools.lru_cache(maxsize=None)
def per_step_results():
    names = ["big"] + SMALL
    return dict(_spawn(_per_step_worker, [(names,)], len(names)))


@pytest.mark.parametrize("name", ["big"] + SMALL)
def test_per_step_path_matches_oracle_f32(name):
    got, want = per_step_results()[name], oracle(name)
    assert got["paths"] == (0, len(want["steps"])), got["paths"]       # the fallback ran, the cooperative launch did not
    assert_matches(got, want, name + " per-step")


# ---- batch path, device RNG -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["37x53", "141x142"])
def test_batch_device_rng_matches_oracle_f32(name):
    """generate_events_batch with the device RNG (leak and shot noise on): the oracle draws the device's own Philox
    fields (EventEmulator.device_draws), so rows, steps and state must match bit for bit."""
    from emu_oracle_cs32 import OracleEmulatorCS32
    from v2e_b200 import EventEmulator
    frames, times, kw = case_inputs(name)
    em = EventEmulator(device="cuda", seed=11, rng_mode="device", max_frames_per_step=4, **kw)
    rows, offs = em.generate_events_batch(frames, times)
    got = dict(rows=[rows[offs[i]:offs[i + 1]] for i in range(len(frames))], steps=list(em.cs_steps_taken))
    for k in STATES:
        got[k] = getattr(em, k).cpu().numpy()
    rng = DeviceDrawRNG(lambda k: {n: t.cpu().numpy() for n, t in em.device_draws(k - 1).items()})
    orc = OracleEmulatorCS32(seed=11, rng=rng, shuffle=False, **kw)
    want = dict(rows=run_oracle_with_draws(orc, rng, frames, times), steps=list(orc.cs_steps_taken),
                cs_surround_frame=orc.surround, lp_log_frame=orc.lp, base_log_frame=orc.base)
    assert ("randn", "rand") == tuple(sorted({c[1] for c in rng.calls}, reverse=True))   # the noise took part
    assert_matches(got, want, name + " batch")


# ---- pixel-sharded ----------------------------------------------------------------------------------------------------
def _sharded_worker(rank, world, port, cases, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = 0 if backend == "gloo" else rank
    if backend == "nccl":
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from v2e_b200 import EventEmulator
        from v2e_b200.parallel import row_band
        for name, K in cases:
            frames, times, kw = case_inputs(name)
            em = EventEmulator(device="cuda:%d" % dev, shard=(rank, world, None), seed=11, **kw)
            em.cs_chunk_steps = K
            out = [em.generate_events(f, float(t)) for f, t in zip(frames, times)]
            r = _result(em, out, whole_frame=False)
            r["paths"] = em.cs_paths()
            H = frames.shape[1]
            r["K"] = em.cs_halo_rows(H)
            (y0, y1), ye0 = row_band(H, rank, world), em.ext_band(H)[0]
            r["surround_own"] = em.cs_surround_frame.cpu().numpy()[y0 - ye0:y1 - ye0]   # the band without its halo
            q.put(((name, rank), r))
    except BaseException as e:
        q.put(("error", repr(e)))
    finally:
        dist.destroy_process_group()


@functools.lru_cache(maxsize=None)
def sharded_results(world, backend="gloo"):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cases = SHARDED[world]
    return dict(_spawn(_sharded_worker, [(r, world, port, cases, backend) for r in range(world)], world * len(cases)))


def check_sharded(res, world, name, K):
    want = oracle(name)
    for r in range(world):
        got = res[(name, r)]
        assert got["K"] == K
        assert got["steps"] == want["steps"], (r, got["steps"], want["steps"])
        chunks = sum(-(-s // K) for s in want["steps"])       # every chunk up to the converged one ran
        assert got["paths"][0] >= chunks and got["paths"][1] == 0, (got["paths"], chunks)
    for i in range(len(want["rows"])):
        g = np.concatenate([res[(name, r)]["rows"][i] for r in range(world)])
        assert_events_equal(g, want["rows"][i], exact_order=False, ctx="%s %d ranks frame %d" % (name, world, i))
    h = np.concatenate([res[(name, r)]["surround_own"] for r in range(world)])
    assert h.dtype == np.float32
    n = int((h.view(np.uint32) != want["cs_surround_frame"].view(np.uint32)).sum())
    assert n == 0, "%s %d ranks: cs_surround_frame differs at %d pixels" % (name, world, n)
    ends = [s % K for s in want["steps"]]
    return ends


@pytest.mark.parametrize("world,name", [(w, c) for w in SHARDED for c, _ in SHARDED[w]])
def test_pixel_sharded_matches_oracle_f32(world, name):
    K = dict(SHARDED[world])[name]
    ends = check_sharded(sharded_results(world), world, name, K)
    if name == "big" and world == 2:
        assert 0 in ends and any(e != 0 for e in ends), ends   # on a chunk boundary, and inside a chunk


def test_pixel_sharded_nccl_two_gpus_f32():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    res = sharded_results(2, "nccl")
    for name, K in SHARDED[2]:
        check_sharded(res, 2, name, K)
