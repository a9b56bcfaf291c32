"""GPU: the centre-surround pixel model (emulator.py:1061-1124, BASELINE config 5) against the CPU oracle, bit for bit,
on every device path of its Euler iteration:
  - one cooperative launch per frame (emu_csdvs_iter_kernel), in this process;
  - one kernel per step (emu_csdvs_step_kernel + emu_csdvs_finish_kernel), in a spawned process with V2E_CS_COOP=0
    (the library reads it once per process);
  - pixel-sharded row bands (v2e_emu_cs_*) over 2 and 3 gloo ranks on one GPU;
  - generate_events_batch with the device RNG.
Each case compares the rows of every frame (canonical order), cs_steps_taken and, where the handle holds the whole
frame, cs_surround_frame, lp_log_frame and base_log_frame.

Shapes: config 5 itself (1280x720, bench.C5_PARAMS, frames 1/1500 s apart as at 50x slow-down), and frames at the
float32 Laplacian's summation-order switch and with a non-empty flattened tail (oracle_lap_kernel_order in
oracle/emu_oracle.c): 141x141 (padded 20 449: pairwise, 9-pixel tail), 141x142 (padded 20 592: kernel order),
20x974 (19 480 pixels but padded 21 472: kernel order) and 37x53 (pairwise, 9-pixel tail)."""
import functools
import os
import socket

import numpy as np
import pytest

import bench
from helpers import assert_events_equal

pytestmark = pytest.mark.gpu

C5 = bench.C5_PARAMS
DT = 1 / 1500.
SMALL = ["141x141", "141x142", "20x974", "37x53"]
# pixel-sharded runs: world -> [(case, Euler steps per chunk = halo rows K)]. 2 ranks at 1280x720 with K = 29: 667
# steps are 23 whole chunks, and the frame that converges after 1 step ends inside the first chunk. 3 ranks with
# K = 64: the last chunk is partial. Band + halo offsets of 37x53 (K = 5: 424, 1060) and 20x974 (K = 3: 6818) are not
# multiples of 16 pixels, so the tail test's whole-frame index matters.
SHARDED = {2: [("c5", 29), ("141x141", 7), ("141x142", 7), ("20x974", 3), ("37x53", 5)],
           3: [("c5", 64), ("37x53", 5)]}


def case_inputs(name):
    """(frames [T, H, W] uint8, times). Config 5: two uniform frames first, so that frame 1's iteration converges
    after one step, then the block texture of bench.py moving, with one static frame."""
    if name == "c5":
        H, W = 720, 1280
        src = bench.block_texture_clip(H, W, 3, seed=5)
        grey = np.full((H, W), 128, np.uint8)
        frames = np.stack([grey, grey, src[0], src[1], src[1], src[2]])
    else:
        H, W = (int(v) for v in name.split("x"))
        src = bench.block_texture_clip(H, W, 4, seed=H * W, block=1, shift=(3, 2))     # high contrast
        frames = np.stack([src[0], src[0], src[1], src[2], src[3]])
    return frames, np.arange(len(frames)) * DT


def _result(em, out, whole_frame=True):
    r = dict(rows=[np.zeros((0, 4), np.float32) if e is None else np.asarray(e) for e in out],
             steps=list(em.cs_steps_taken))
    if whole_frame:
        for k in ("cs_surround_frame", "lp_log_frame", "base_log_frame"):
            r[k] = getattr(em, k).cpu().numpy()
        r["paths"] = em.cs_paths()
    return r


def run_device(name, frames_dtype=None):
    from v2e_b200 import EventEmulator
    frames, times = case_inputs(name)
    if frames_dtype is not None:
        frames = frames.astype(frames_dtype) + np.random.default_rng(1).uniform(0, 0.9, frames.shape).astype(frames_dtype)
    em = EventEmulator(device="cuda", seed=11, **C5)
    out = [em.generate_events(f, float(t)) for f, t in zip(frames, times)]
    return _result(em, out)


@functools.lru_cache(maxsize=None)
def oracle(name, legacy_order=0, alpha_h_ulps=0, frames_dtype=None):
    from emu_oracle import OracleEmulator, lib
    frames, times = case_inputs(name)
    if frames_dtype is not None:
        frames = frames.astype(frames_dtype) + np.random.default_rng(1).uniform(0, 0.9, frames.shape).astype(frames_dtype)
    lib().oracle_set_cs_perturbation(legacy_order, alpha_h_ulps)
    try:
        em = OracleEmulator(seed=11, **C5)
        out = [em.generate_events(f, float(t)) for f, t in zip(frames, times)]
    finally:
        lib().oracle_set_cs_perturbation(0, 0)
    return dict(rows=[np.zeros((0, 4), np.float32) if e is None else e for e in out], steps=list(em.cs_steps_taken),
                cs_surround_frame=em.surround, lp_log_frame=em.lp, base_log_frame=em.base)


def assert_matches(got, want, ctx):
    assert got["steps"] == want["steps"], (ctx, got["steps"], want["steps"])
    assert len(got["rows"]) == len(want["rows"])
    for i, (g, w) in enumerate(zip(got["rows"], want["rows"])):
        assert_events_equal(g, w, exact_order=False, ctx="%s frame %d" % (ctx, i))
    for k in ("cs_surround_frame", "lp_log_frame", "base_log_frame"):
        if k in got:
            a, b = got[k], want[k]
            assert a.dtype == b.dtype and a.shape == b.shape, (ctx, k)
            n = int((a.view(np.uint64) != b.view(np.uint64)).sum())
            assert n == 0, "%s: %s differs at %d pixels" % (ctx, k, n)


def differences(got, want):
    """(rows that differ over all frames, surround pixels that differ) -- how far a perturbed oracle moved."""
    from helpers import canonical
    rows = 0
    for g, w in zip(got["rows"], want["rows"]):
        g, w = canonical(g), canonical(w)
        if g.shape != w.shape:
            rows += abs(len(g) - len(w)) + min(len(g), len(w))
        else:
            rows += int((g != w).any(axis=1).sum())
    return rows, int((got["cs_surround_frame"].view(np.uint64) != want["cs_surround_frame"].view(np.uint64)).sum())


@functools.lru_cache(maxsize=None)
def coop(name):
    return run_device(name)


# ---- cooperative launch, this process ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["c5"] + SMALL)
def test_cooperative_path_matches_oracle(name):
    got, want = coop(name), oracle(name)
    assert got["paths"] == (len(want["steps"]), 0), got["paths"]        # one cooperative launch per frame, no fallback
    assert_matches(got, want, name + " cooperative")
    print("%s cooperative: %d rows, cs_steps_taken %s" % (name, sum(len(r) for r in want["rows"]), want["steps"]))
    if name == "c5":
        assert 1 in want["steps"] and max(want["steps"]) == 667, want["steps"]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_float_frames_346x260(dtype):
    """emu_lp_kernel's float32 / float64 frame variants ahead of the surround, config 5 parameters."""
    name = "260x346"
    got, want = run_device(name, dtype), oracle(name, frames_dtype=dtype)
    assert_matches(got, want, "%s %s" % (name, dtype.__name__))


# ---- one kernel per step, spawned process ----------------------------------------------------------------------------
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
    names = ["c5"] + SMALL
    return dict(_spawn(_per_step_worker, [(names,)], len(names)))


@pytest.mark.parametrize("name", ["c5"] + SMALL)
def test_per_step_path_matches_oracle(name):
    got, want = per_step_results()[name], oracle(name)
    assert got["paths"] == (0, len(want["steps"])), got["paths"]       # the fallback ran, the cooperative launch did not
    assert_matches(got, want, name + " per-step")


# ---- batch path ---------------------------------------------------------------------------------------------------
def test_batch_device_rng_matches_oracle_c5():
    """generate_events_batch, device RNG (config 5 has no leak or shot noise, so no draw is used)."""
    from v2e_b200 import EventEmulator
    frames, times = case_inputs("c5")
    want = oracle("c5")
    em = EventEmulator(device="cuda", seed=11, rng_mode="device", max_frames_per_step=4, **C5)
    rows, offs = em.generate_events_batch(frames, times)
    got = dict(rows=[rows[offs[i]:offs[i + 1]] for i in range(len(frames))], steps=list(em.cs_steps_taken))
    for k in ("cs_surround_frame", "lp_log_frame", "base_log_frame"):
        got[k] = getattr(em, k).cpu().numpy()
    assert_matches(got, want, "c5 batch")


# ---- pixel-sharded ---------------------------------------------------------------------------------------------------
def _sharded_worker(rank, world, port, cases, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from v2e_b200 import EventEmulator
        from v2e_b200.parallel import row_band
        for name, K in cases:
            frames, times = case_inputs(name)
            em = EventEmulator(device="cuda:0", shard=(rank, world, None), seed=11, **C5)
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
def sharded_results(world):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cases = SHARDED[world]
    return dict(_spawn(_sharded_worker, [(r, world, port, cases) for r in range(world)], world * len(cases)))


@pytest.mark.parametrize("world,name", [(w, c) for w in SHARDED for c, _ in SHARDED[w]])
def test_pixel_sharded_matches_oracle(world, name):
    res, want = sharded_results(world), oracle(name)
    K = dict(SHARDED[world])[name]
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
    n = int((h.view(np.uint64) != want["cs_surround_frame"].view(np.uint64)).sum())
    assert n == 0, "%s %d ranks: cs_surround_frame differs at %d pixels" % (name, world, n)
    if name == "c5" and world == 2:
        ends = [s % K for s in want["steps"]]
        assert 0 in ends and any(e != 0 for e in ends), ends   # on a chunk boundary, and inside a chunk


# ---- sensitivity: the comparisons above fail when only the oracle is wrong ----------------------------------------
@pytest.mark.parametrize("name", ["141x141", "20x974", "37x53"])
def test_legacy_order_rule_is_caught(name):
    """The rule the oracle and the kernels used before (kernel order iff H*W >= 20000, no tail) in the oracle alone:
    20x974 switches order at every pixel, 141x141 and 37x53 in their 9-pixel tails. (141x142 takes kernel order under
    both rules.)"""
    got, want = coop(name), oracle(name, legacy_order=1)
    rows, px = differences(got, want)
    print("%s, legacy rule in the oracle: %d rows and %d surround pixels differ" % (name, rows, px))
    with pytest.raises(AssertionError):
        assert_matches(got, want, name)


def test_alpha_h_one_ulp_is_caught_c5():
    got, want = coop("c5"), oracle("c5", alpha_h_ulps=1)
    rows, px = differences(got, want)
    print("c5, alpha_h + 1 ulp in the oracle: %d rows and %d surround pixels differ" % (rows, px))
    assert rows > 0
