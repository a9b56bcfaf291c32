"""Event files from the batched and sharded pixel-model paths: EventEmulator.write_events, generate_events_batch and
V2EPipeline.run feeding the sinks, and a sharded clip's bands merged on the device (parallel.merge_by_key_device) and
written by the group's first rank (V2EPipeline.run_clip_sharded(..., write_sinks=True)).

CPU: write_events' and write_sinks' argument checks (gloo ranks, a stub emulator); the AEDAT-2.0 rule that drops leading
'#' records of a writer's first events, as an oracle against the reference's own AEDat2Output and against
emulator._append_aedat2 fed the oracle's words.
GPU: batched files byte-identical to frame-by-frame files and to the oracle; the pipeline's text file; the device merge
bit for bit against the host merge_by_key; sharded files byte-identical to the one-GPU files. The reference's writers
are loaded in subprocesses / spawned ranks (loading the reference stubs modules)."""
import io
import os
import subprocess
import sys
import types

import numpy as np
import pytest

import sinks_oracle
import text_sink_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _have_reference():
    import ref_shim
    return ref_shim.reference_available()


def drop_leading_hashes(body, written):
    """aedat2_output.py:174-180: while the writer has written no event, leading 8-byte records whose first byte is '#'
    are dropped. Returns (bytes written, records dropped)."""
    if written:
        return body, 0
    k = 0
    while body[8 * k:8 * k + 1] == b"#":
        k += 1
    return body[8 * k:], k


def aedat2_body(rows, width, height, labels, written=0):
    """What one AEDat2Output(label_signal_noise=labels is not None).appendEvents(rows, labels) call writes."""
    if labels is None:
        words, _ = sinks_oracle.aedat2_words(np.asarray(rows, np.float32), width, height)
    else:
        words, _ = text_sink_oracle.aedat2_words_labeled(np.asarray(rows, np.float32), width, height, labels)
    return drop_leading_hashes(words.tobytes(), written)[0]


def split_header(data, eol):
    """(header, body) of a file the reference's text or AEDAT-2.0 writer wrote: its header ends with the
    '# User name: ...' line (a body may start with '#' when the writer's first call had only such records)."""
    pos = data.index(eol, data.index(b"# User name: ")) + len(eol)
    return data[:pos], data[pos:]


def hash_rows(n, seed, lead):
    """n rows at 346 x 260 whose first `lead` rows have flipped y >> 2 == 35 (a '#' first byte), the rest not."""
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 346, n)
    y = rng.integers(0, 116, n)                          # flipped y >= 144: first byte >= 36
    y[:lead] = rng.integers(116, 120, lead)              # flipped y in [140, 143]: first byte 35 = '#'
    t = np.sort(rng.uniform(0, 0.05, n))
    return np.stack([t, x, y, rng.choice([-1.0, 1.0], n)], 1).astype(np.float32)


# ---- CPU --------------------------------------------------------------------------------------------------------
def _stub_emulator(monkeypatch, **kw):
    from v2e_b200 import emulator as em_mod
    monkeypatch.setattr(em_mod._lib, "load", lambda *a, **k: object())
    e = em_mod.EventEmulator(device="cuda", **kw)
    e._finalizer.detach()
    return e


def test_write_events_argument_checks(monkeypatch):
    import torch
    em = _stub_emulator(monkeypatch)
    rows = np.zeros((5, 4), np.float32)
    assert em.write_events(rows) == 5
    assert em.write_events(rows, labels=np.ones(5, bool)) == 5
    assert em.write_events(torch.zeros((3, 4), dtype=torch.float32)) == 3
    assert em.write_events(np.zeros((0, 4), np.float32), labels=[]) == 0
    for bad in (np.zeros((5, 4), np.float64), np.zeros((5, 3), np.float32), np.zeros(20, np.float32),
                np.zeros((5, 4, 1), np.float32), torch.zeros((5, 4), dtype=torch.float64), [[0.0, 1.0, 2.0, 1.0]]):
        with pytest.raises(ValueError):
            em.write_events(bad)
    for lab in (np.ones(4, bool), np.ones((5, 1), np.uint8), torch.ones(6, dtype=torch.uint8)):
        with pytest.raises(ValueError):
            em.write_events(rows, labels=lab)


def _sink_check_worker(rank, world, port, q, case):
    import torch.distributed as dist
    from test_sharded_options import _init
    _init(rank, world, port)
    try:
        from v2e_b200 import V2EPipeline
        holds = case == "others_hold_sinks" and rank == world - 1
        em = types.SimpleNamespace(shard=(rank, world, None), label_signal_noise=False, device="cpu",
                                   row_order=None if case == "no_row_order" else "canonical",
                                   _sinks=object() if holds or rank == 0 else None)
        try:
            V2EPipeline(None, em).run_clip_sharded(np.zeros((4, 8, 8), np.uint8), 0.1, group=None, write_sinks=True)
            msg = None
        except ValueError as e:
            msg = str(e)
        q.put((rank, msg))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("case,world", [("no_row_order", 2), ("others_hold_sinks", 2), ("others_hold_sinks", 3)])
def test_run_clip_sharded_write_sinks_refusals(case, world):
    """row_order missing, or sinks on a rank that is not the first: every rank raises ValueError (none is left waiting
    in a collective) before any data moves -- the stub emulator and the missing upsampler are never used."""
    from test_sharded_options import _spawn
    res = _spawn(world, _sink_check_worker, case)
    for r in range(world):
        assert res[r] is not None, r
        assert ("row_order" in res[r]) == (case == "no_row_order"), res[r]


_HASH_REF = r"""
import os, sys
import numpy as np
sys.path[:0] = [{root!r}, os.path.join({root!r}, "oracle"), os.path.join({root!r}, "tests")]
import ref_shim
ref_shim.load_reference()
from v2ecore.output.aedat2_output import AEDat2Output
from test_sinks_batched import _HASH_CASES, hash_rows
out = {out!r}
counts = {{}}
for name, (lab, calls) in _HASH_CASES.items():
    w = AEDat2Output(os.path.join(out, name + ".aedat"), 346, 260, label_signal_noise=lab)
    for n, seed, lead in calls:
        rows = hash_rows(n, seed, lead)
        w.appendEvents(rows, signnoise_label=(np.arange(n) % 3 != 0) if lab else None)
    counts[name] = (w.numEventsWritten, w.numOnEvents, w.numOffEvents)
    w.close()
np.save(os.path.join(out, "counts.npy"), counts, allow_pickle=True)
"""

_HASH_CASES = {"lead2": (True, [(40, 1, 2), (30, 2, 3)]), "all_hash": (False, [(6, 3, 6), (20, 4, 2)]),
               "plain": (True, [(25, 5, 0)])}


def test_hash_record_drop_oracle_equals_reference_writer(tmp_path):
    """The oracle (aedat2_words_labeled + drop_leading_hashes) writes what the reference's AEDat2Output writes: leading
    '#' records of the first non-empty call dropped (all of them when every record is one), none of a later call's."""
    if not _have_reference():
        pytest.skip("reference tree not present")
    subprocess.check_call([sys.executable, "-c", _HASH_REF.format(root=ROOT, out=str(tmp_path))])
    counts = np.load(tmp_path / "counts.npy", allow_pickle=True).item()
    for name, (lab, calls) in _HASH_CASES.items():
        head, body = split_header((tmp_path / (name + ".aedat")).read_bytes(), b"\r\n")
        assert head.startswith(b"#!AER-DAT2.0")
        want, written, n_on = b"", 0, 0
        for n, seed, lead in calls:
            rows = hash_rows(n, seed, lead)
            want += aedat2_body(rows, 346, 260, (np.arange(n) % 3 != 0) if lab else None, written)
            written += n
            n_on += int((rows[:, 3] > 0).sum())
        assert body == want, name
        assert counts[name] == (written, n_on, written - n_on), name


def test_append_aedat2_drops_like_the_oracle(monkeypatch):
    """emulator._append_aedat2 (the writer's counters, the drop of leading '#' records) with the device conversion
    replaced by the oracle's words."""
    import torch
    from v2e_b200 import emulator as em_mod
    from v2e_b200 import sinks

    def fake(ev, w, h, labels=None):
        rows = ev.numpy()
        words, n_on = (sinks_oracle.aedat2_words(rows, w, h) if labels is None else
                       text_sink_oracle.aedat2_words_labeled(rows, w, h, labels.numpy()))
        return torch.from_numpy(words.view(np.int32).copy()), torch.tensor([n_on])
    monkeypatch.setattr(sinks, "events_to_aedat2", fake)
    for name, (lab, calls) in _HASH_CASES.items():
        w = types.SimpleNamespace(file=io.BytesIO(), sizex=346, sizey=260, numEventsWritten=0, numOnEvents=0,
                                  numOffEvents=0)
        want, n_on = b"", 0
        for n, seed, lead in calls:
            rows = hash_rows(n, seed, lead)
            labels = (np.arange(n) % 3 != 0) if lab else None
            want += aedat2_body(rows, 346, 260, labels, w.numEventsWritten)
            n_on += int((rows[:, 3] > 0).sum())
            em_mod._append_aedat2(w, torch.from_numpy(rows),
                                  None if labels is None else torch.from_numpy(labels.astype(np.uint8)))
        written = sum(c[0] for c in calls)
        assert w.file.getvalue() == want, name
        assert (w.numEventsWritten, w.numOnEvents, w.numOffEvents) == (written, n_on, written - n_on), name
    w = types.SimpleNamespace(file=None, numEventsWritten=0)
    em_mod._append_aedat2(w, torch.zeros((2, 4)), None)         # a closed writer takes nothing, counts nothing
    assert w.numEventsWritten == 0


# ---- GPU: batched files -------------------------------------------------------------------------------------------
_KW = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.5, shot_noise_rate_hz=2.0,
           refractory_period_s=0.0005)


def batched_clip(H, W, T=14):
    """A moving texture whose first frame with events changes only a block of rows 116..123: at 346 x 260 the first
    rows of the stream (canonical order: by pixel) have flipped y >> 2 == 35, so the AEDAT-2.0 writer drops them."""
    from test_emulator_device_rng import texture_frames
    base = texture_frames(H, W, T, seed=W, speed=2.0)
    fr = np.empty_like(base)
    fr[0] = base[0]
    fr[1] = base[0]
    fr[1, 116:124, 100:140] = np.clip(base[0, 116:124, 100:140].astype(int) + 80, 0, 255)
    fr[2:] = base[:T - 2]
    return fr, [k / 300. for k in range(T)]


_BATCHED = r"""
import os, sys
import numpy as np
sys.path[:0] = [{root!r}, os.path.join({root!r}, "oracle"), os.path.join({root!r}, "tests")]
try:
    import h5py
except ImportError:
    h5py = None
import ref_shim
ref_shim.load_reference()
import torch
from test_sinks_batched import batched_clip, _KW
from v2e_b200 import EventEmulator
H, W, out = {H}, {W}, {out!r}
fr, ts = batched_clip(H, W)
res = {{}}
for variant in ("host", "device"):
    d = os.path.join(out, variant)
    os.makedirs(os.path.join(d, "batched"))
    os.makedirs(os.path.join(d, "frames"))
    mk = lambda sub, **k: EventEmulator(device="cuda", rng_mode="device", seed=5, row_order="canonical",
                                        label_signal_noise=True, output_folder=os.path.join(d, sub), dvs_text="ev",
                                        dvs_aedat2="ev", dvs_h5="ev" if h5py else None, output_width=W,
                                        output_height=H, **_KW, **k)
    a = mk("batched", max_frames_per_step=4)
    if variant == "host":
        rows, offs, lab = a.generate_events_batch(fr[:7], ts[:7], return_labels=True)
        rows2, offs2, lab2 = a.generate_events_batch(fr[7:], ts[7:], return_labels=True)
        rows, lab = np.concatenate([rows, rows2]), np.concatenate([lab, lab2])
    else:
        r1, _ = a.generate_events_batch(fr[:7], ts[:7], return_device=True, copy=False)
        r1 = r1.clone()
        r2, _ = a.generate_events_batch(fr[7:], ts[7:], return_device=True, copy=False)
        rows = torch.cat([r1, r2]).cpu().numpy()
        lab = None
    b = mk("frames")
    frows, flab = [], []
    for f, t in zip(fr, ts):
        ev = b.generate_events(f, t)
        if ev is not None:
            frows.append(ev)
            flab.append(b.last_signnoise_label)
    frows, flab = np.concatenate(frows), np.concatenate(flab)
    counters = [(e.dvs_text.numEventsWritten, e.dvs_aedat2.numEventsWritten, e.dvs_aedat2.numOnEvents,
                 e.dvs_aedat2.numOffEvents) for e in (a, b)]
    a.cleanup()
    b.cleanup()
    np.savez(os.path.join(d, "rows.npz"), rows=rows, labels=lab if lab is not None else flab, frows=frows, flab=flab,
             counters=np.array(counters), h5=h5py is not None)
"""


@pytest.fixture(scope="module", params=[(260, 346), (480, 640)], ids=["346x260", "640x480"])
def batched_run(request, tmp_path_factory):
    if not _have_reference():
        pytest.skip("v2ecore (the reference's writers) does not import")
    H, W = request.param
    out = tmp_path_factory.mktemp("batched_%dx%d" % (W, H))
    subprocess.check_call([sys.executable, "-c", _BATCHED.format(root=ROOT, H=H, W=W, out=str(out))])
    return H, W, out


def _files(d):
    text = split_header((d / "ev.txt").read_bytes(), b"\n")
    aedat = split_header((d / "ev.aedat").read_bytes(), b"\r\n")
    assert text[0].startswith(b"#!events.txt") and aedat[0].startswith(b"#!AER-DAT2.0")
    return text[1], aedat[1]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["host", "device"])
def test_batched_files_equal_frame_by_frame_files(batched_run, variant):
    """generate_events_batch over chunks (max_frames_per_step 4, two calls) writes the bytes a loop of generate_events
    writes through the reference's writers: the text and AEDAT-2.0 bodies after their headers and the counters; also
    with return_device=True and copy=False."""
    H, W, out = batched_run
    d = out / variant
    r = np.load(d / "rows.npz")
    assert r["rows"].tobytes() == r["frows"].tobytes() and len(r["rows"]) > 1000
    assert (~r["flab"]).sum() > 0 and r["flab"].sum() > 0
    assert _files(d / "batched") == _files(d / "frames")
    ca, cb = r["counters"]
    assert ca.tolist() == cb.tolist() and ca[0] == ca[1] == len(r["rows"]) and ca[2] + ca[3] == ca[0]
    if W == 346:
        # the stream starts with rows the AEDAT-2.0 writer drops ('#' first byte), then keeps the rest
        first = int(np.argmax((259 - r["rows"][:, 2].astype(int)) >> 2 != 35))
        assert first >= 1 and len(_files(d / "batched")[1]) == 8 * (len(r["rows"]) - first)


@pytest.mark.gpu
def test_batched_bodies_equal_the_oracle(batched_run):
    H, W, out = batched_run
    d = out / "host"
    r = np.load(d / "rows.npz")
    rows, labels = r["rows"], r["labels"]
    text, aedat = _files(d / "batched")
    assert text == text_sink_oracle.text_body(rows, labels)
    assert aedat == aedat2_body(rows, W, H, labels)
    if bool(r["h5"]):
        import h5py
        with h5py.File(d / "batched" / "ev.h5", "r") as f:
            assert np.array_equal(f["events"][:], sinks_oracle.h5_rows(rows))


_PIPE = r"""
import os, sys
import numpy as np
sys.path[:0] = [{root!r}, os.path.join({root!r}, "oracle"), os.path.join({root!r}, "tests")]
import ref_shim
ref_shim.load_reference()
from test_sharded_options import _auto_clip, _slomo
from v2e_b200 import EventEmulator, V2EPipeline
out = {out!r}
sl = _slomo()
em = EventEmulator(device="cuda", rng_mode="device", seed=3, output_folder=out, dvs_text="ev", cutoff_hz=200,
                   leak_rate_hz=0.2, shot_noise_rate_hz=10.0, sigma_thres=0.02)
ev, offs, t, nf = V2EPipeline(sl, em).run(_auto_clip(0), 0.2, copy=True)
n = em.dvs_text.numEventsWritten
em.cleanup()
sl.cleanup()
np.savez(os.path.join(out, "rows.npz"), rows=ev, n=n)
"""


@pytest.mark.gpu
def test_pipeline_text_file_holds_the_rows_it_returns(tmp_path):
    if not _have_reference():
        pytest.skip("v2ecore (the reference's writers) does not import")
    subprocess.check_call([sys.executable, "-c", _PIPE.format(root=ROOT, out=str(tmp_path))])
    r = np.load(tmp_path / "rows.npz")
    assert len(r["rows"]) > 0 and int(r["n"]) == len(r["rows"])
    assert split_header((tmp_path / "ev.txt").read_bytes(), b"\n")[1] == text_sink_oracle.text_body(r["rows"])


# ---- GPU: device merge ------------------------------------------------------------------------------------------
def _assert_merge_equal(streams, keys, offsets, n_shot, ctx):
    from v2e_b200.parallel import merge_by_key, merge_by_key_device
    want, woffs = merge_by_key(streams, keys, offsets, n_shot)
    got, goffs = merge_by_key_device(streams, keys, offsets, n_shot)
    assert got.is_cuda and goffs.is_cuda
    assert np.array_equal(goffs.cpu().numpy(), woffs), ctx
    assert got.cpu().numpy().tobytes() == want.tobytes(), ctx
    return len(want)


def _bands_worker(rank, world, port, q, frames, ts):
    import torch.distributed as dist
    from test_sharded_options import _init
    from test_row_order_gpu import _SHARD_KW
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator
        H = frames.shape[1]
        out = {}
        for mode in ("canonical", "shuffled"):
            for refr in (0.0, 0.004):
                em = EventEmulator(device="cuda:0", seed=1234, rng_mode="device", shard=(rank, world, None),
                                   row_order=mode, max_frames_per_step=5, **dict(_SHARD_KW, refractory_period_s=refr))
                ye0, ye1 = em.ext_band(H)
                rows, offs, keys = em.generate_events_band_batch(np.ascontiguousarray(frames[:, ye0:ye1]), ts, H,
                                                                 return_keys=True)
                out[mode, refr] = (rows, offs, keys, em.last_n_shot)
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_device_merge_equals_host_merge_on_band_outputs(world):
    """The bands of gloo ranks sharing the GPU, both row orders, refractory 0 (multi-frame kernels) and 0.004
    (rejected chunks replayed frame by frame)."""
    from test_emulator_device_rng import texture_frames
    from test_sharded_options import _spawn
    H, W, T = 37, 53, 11
    fr, ts = texture_frames(H, W, T, seed=5, speed=2.0), [k * 1e-2 for k in range(T)]
    res = _spawn(world, _bands_worker, fr, ts)
    for case in res[0]:
        parts = [res[r][case] for r in range(world)]
        # a worker's part is (rows, offsets, keys, n_shot)
        n = _assert_merge_equal(*[[p[i] for p in parts] for i in (0, 2, 1, 3)], ctx=case)
        assert n > 1000


def synthetic_bands(world, T, H, W, seed, empty_bands=(), empty_frames=(), shot_only=(), key_range=None, n_max=400):
    """Band outputs with the ordering a band generated with row_order has: per frame, signal rows strictly by
    (t, key) -- a few iterations, keys drawn from key_range (small ranges make keys of different bands collide, so
    the merge falls back to (y, x, p)) -- then shot rows strictly by key = (p < 0) << 32 | pixel."""
    from v2e_b200.parallel import row_band
    rng = np.random.default_rng(seed)
    streams, keys, offsets, n_shot = [], [], [], []
    for r in range(world):
        y0, y1 = row_band(H, r, world)
        rows, ks, offs, ns = [], [], [0], []
        for f in range(T):
            n_sig = 0 if (r in empty_bands or f in empty_frames or f in shot_only) else int(rng.integers(0, n_max))
            n_sh = 0 if (r in empty_bands or f in empty_frames) else int(rng.integers(0, 60)) + (f in shot_only)
            it = rng.integers(0, 3, n_sig)
            t = np.float32(f * 1e-2) + np.float32(1e-3) * it.astype(np.float32)
            k = rng.integers(0, key_range or 2 ** 40, n_sig).astype(np.uint64)
            sig = np.stack([t, rng.integers(0, W, n_sig), rng.integers(y0, max(y1, y0 + 1), n_sig),
                            rng.choice([-1.0, 1.0], n_sig)], 1).astype(np.float32)
            order = np.lexsort((k, t))
            sig, k = sig[order], k[order]
            keep = np.ones(n_sig, bool)
            keep[1:] = (np.diff(sig[:, 0]) != 0) | (np.diff(k.astype(np.int64)) != 0)      # strictly by (t, key)
            sig, k = sig[keep], k[keep]
            pix = rng.choice(max(y1 - y0, 1) * W, size=min(n_sh, max(y1 - y0, 1) * W), replace=False)
            pol = rng.choice([-1.0, 1.0], len(pix))
            sk = ((pol < 0).astype(np.uint64) << np.uint64(32)) | (pix + y0 * W).astype(np.uint64)
            o = np.argsort(sk)
            pix, pol, sk = pix[o], pol[o], sk[o]
            shot = np.stack([np.full(len(pix), np.float32(f * 1e-2)), pix % W, y0 + pix // W, pol], 1).astype(np.float32)
            rows += [sig, shot]
            ks += [k, sk]
            offs.append(offs[-1] + len(sig) + len(shot))
            ns.append(len(shot))
        streams.append(np.concatenate(rows).reshape(-1, 4))
        keys.append(np.concatenate(ks).astype(np.uint64))
        offsets.append(np.asarray(offs, np.int64))
        n_shot.append(np.asarray(ns, np.int64))
    return streams, keys, offsets, n_shot


@pytest.mark.gpu
def test_device_merge_equals_host_merge_on_synthetic_bands():
    import torch
    from v2e_b200.parallel import merge_by_key_device
    cases = [dict(world=3, T=8, H=30, W=40, seed=1, empty_frames=(0, 5), shot_only=(2, 7)),
             dict(world=4, T=6, H=30, W=40, seed=2, empty_bands=(1,), shot_only=(3,), key_range=5),
             dict(world=8, T=5, H=64, W=50, seed=3, empty_bands=(0, 7), key_range=40),
             dict(world=2, T=4, H=20, W=30, seed=4, empty_bands=(0, 1)),
             dict(world=1, T=3, H=20, W=30, seed=5),
             dict(world=5, T=1, H=10, W=30, seed=6, key_range=3)]
    total = 0
    for c in cases:
        total += _assert_merge_equal(*synthetic_bands(**c), ctx=c)
    assert total > 3000
    # many blocks: 8 bands of a 720-row frame, 3 frames
    s, k, o, n = synthetic_bands(8, 3, 720, 1280, seed=9, key_range=1 << 20, n_max=40000)
    assert _assert_merge_equal(s, k, o, n, "720p") > 100000
    # CUDA inputs (int64 keys) give the same
    dev = ([torch.from_numpy(x).cuda() for x in s], [torch.from_numpy(x.view(np.int64)).cuda() for x in k])
    a, ao = merge_by_key_device(dev[0], dev[1], o, n)
    b, bo = merge_by_key_device(s, k, o, n)
    assert torch.equal(a, b) and torch.equal(ao, bo)
    with pytest.raises(ValueError):
        merge_by_key_device(s, k, o[:-1], n)
    with pytest.raises(ValueError):
        merge_by_key_device(s, k, [x[:-1] for x in o], n)


# ---- GPU: sharded clip files --------------------------------------------------------------------------------------
_SH_KW = dict(cutoff_hz=200, leak_rate_hz=0.2, shot_noise_rate_hz=10.0, sigma_thres=0.02)


def _files_worker(rank, world, port, q, out, sharded, backend="gloo"):
    import torch
    import torch.distributed as dist
    if backend == "gloo":
        from test_sharded_options import _init
        _init(rank, world, port)
        dev = "cuda:0"
    else:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        dev = "cuda:%d" % rank
    try:
        import ref_shim
        ref_shim.load_reference()
        from test_sharded_options import _auto_clip, _slomo
        from v2e_b200 import EventEmulator, V2EPipeline
        folder = os.path.join(out, "rank%d" % rank)
        os.makedirs(folder)
        sinks = dict(dvs_text="ev", dvs_aedat2="ev") if rank == 0 else {}
        em = EventEmulator(device=dev, seed=9, rng_mode="device", row_order="canonical", label_signal_noise=True,
                           output_folder=folder, output_width=346, output_height=260,
                           shard=(rank, world, None) if sharded else None, **sinks, **_SH_KW)
        sl = _slomo()
        if sharded:
            rows = V2EPipeline(sl, em).run_clip_sharded(_auto_clip(0), 0.2, write_sinks=True)[0]
        else:
            rows = V2EPipeline(sl, em).run(_auto_clip(0), 0.2, copy=True)[0]
        counters = None
        if rank == 0:
            counters = (em.dvs_text.numEventsWritten, em.dvs_aedat2.numEventsWritten, em.dvs_aedat2.numOnEvents)
        em.cleanup()
        sl.cleanup()
        q.put((rank, (len(rows), counters, sorted(os.listdir(folder)))))
    finally:
        dist.destroy_process_group()


def _compare_sharded(tmp_path, world, backend="gloo"):
    from test_sharded_options import _spawn
    one, sh = tmp_path / "one", tmp_path / "sharded"
    ref = _spawn(1, _files_worker, str(one), False)
    if backend == "gloo":
        res = _spawn(world, _files_worker, str(sh), True)
    else:
        res = _spawn(world, _files_worker, str(sh), True, "nccl")
    n, counters, _ = ref[0]
    assert n > 0 and counters[0] == n
    assert res[0][1] == counters and sum(res[r][0] for r in range(world)) == n
    assert res[0][2] == ["ev.aedat", "ev.txt"]
    for r in range(1, world):
        assert res[r][2] == [], r                                   # the other ranks open no file
    assert _files(sh / "rank0") == _files(one / "rank0")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_files_equal_one_gpu_files(tmp_path, world):
    """run_clip_sharded(write_sinks=True) over gloo ranks sharing the GPU: the first rank's text and AEDAT-2.0 files are
    the one-GPU V2EPipeline.run's after the header, labels included."""
    if not _have_reference():
        pytest.skip("v2ecore (the reference's writers) does not import")
    _compare_sharded(tmp_path, world)


@pytest.mark.gpu
def test_sharded_files_equal_one_gpu_files_over_nccl(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    if not _have_reference():
        pytest.skip("v2ecore (the reference's writers) does not import")
    _compare_sharded(tmp_path, 2, backend="nccl")
