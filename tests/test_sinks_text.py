"""DVS text sink and signal / noise labels (label_signal_noise).

CPU: the oracle (text_sink_oracle.text_body, aedat2_words_labeled) against the bytes the reference's own
DVSTextOutput and AEDat2Output(label_signal_noise=True) wrote (tests/golden/sinks_labeled.npz,
oracle/make_golden_text.py); a host build of the device float formatter (v2e_b200/csrc/shortest_repr.cuh,
tests/shortest_repr_host.cpp) against CPython's repr on whole binades.
GPU: v2e_b200.sinks.events_to_text / events_to_aedat2(labels=) against the fixture and the oracle, and the
emulator's labels against the CPU oracle's per-frame shot counts (replay and device RNG) and end to end through
the file sinks."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import sinks_oracle
import text_sink_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "sinks_labeled.npz"))
SIZES = [(346, 260), (240, 180), (640, 480)]
SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1e-45, -1e-45, 1.1754942e-38, 1.17549435e-38,
                     3.4028235e38, -3.4028235e38, 1e16, 9.999999e15, 1e15, 1e-4, 9.999999e-5, 1e-5, 0.5, 1.0,
                     -2.5, 123456.0, 0.1, 16777216.0, 2.0 ** 63], np.float32)


def binade(e):
    """Every float32 of [2^e, 2^(e+1))."""
    lo = int(np.float32(2.0 ** e).view(np.uint32))
    return np.arange(lo, lo + (1 << 23), dtype=np.uint32).view(np.float32)


# binades around 1e-4 (= 2^-13.3, where the notation switches) and [0.5, 64), then 2 M random finite float32
SWEEP_BINADES = [-14, -13] + list(range(-1, 6))


def random_finite(n=2_000_000, seed=3):
    v = np.random.default_rng(seed).integers(0, 2 ** 32, int(n * 1.01) + 1000, dtype=np.uint64).astype(np.uint32)
    v = v.view(np.float32)
    return v[np.isfinite(v)][:n]


def sweep():
    for e in SWEEP_BINADES:
        yield "binade 2^%d" % e, binade(e)
    yield "random", random_finite()


def repr_lines(v):
    return ("\n".join(map(repr, v.astype(np.float64).tolist())) + "\n").encode()


# ---- CPU --------------------------------------------------------------------------------------------------------
def test_oracle_reproduces_reference_text_bytes():
    ev = G["text_events"]
    assert text_sink_oracle.text_body(ev) == G["text_body"].tobytes()
    assert text_sink_oracle.text_body(ev, G["text_labels"]) == G["text_body_labeled"].tobytes()
    t = ev[:, 0]
    assert (t < 1e-4).sum() > 100 and (t >= 1e-4).sum() > 100 and b"e-" in G["text_body"].tobytes()


@pytest.mark.parametrize("size", SIZES)
def test_oracle_reproduces_reference_labeled_aedat2_bytes(size):
    w, h = size
    ev, lab = G["aedat2_events_%dx%d" % size], G["aedat2_labels_%dx%d" % size]
    words, _ = text_sink_oracle.aedat2_words_labeled(ev, w, h, lab)
    assert words.tobytes() == G["aedat2_body_%dx%d" % size].tobytes()
    assert words.tobytes() != sinks_oracle.aedat2_words(ev, w, h)[0].tobytes()


def test_writer_float_formatting_is_python_repr():
    """The writer formats np.float64 scalars ('{}'.format(t[i]), ae_text_output.py:90-100); the kernels implement
    repr(float(t)). They agree on the fixture's timestamps and the specials."""
    for v in np.concatenate([G["text_events"][:, 0], SPECIALS]).astype(np.float64):
        assert '{}'.format(np.float64(v)) == repr(float(v))


def test_fixture_regenerates_bit_identically(tmp_path):
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("reference tree not present")
    out = tmp_path / "sinks_labeled.npz"
    subprocess.check_call([sys.executable, os.path.join(ROOT, "oracle", "make_golden_text.py"), str(out)],
                          stdout=subprocess.DEVNULL)
    with open(out, "rb") as a, open(os.path.join(ROOT, "tests", "golden", "sinks_labeled.npz"), "rb") as b:
        assert a.read() == b.read()


def test_pow5_tables_are_the_generator_output():
    import runpy
    gen = runpy.run_path(os.path.join(ROOT, "v2e_b200", "csrc", "make_pow5_tables.py"))     # no bytecode in csrc/
    with open(gen["OUT"]) as f:
        assert f.read() == gen["render"]()


@pytest.fixture(scope="module")
def host_formatter(tmp_path_factory):
    cxx = shutil.which(os.environ.get("CXX", "c++")) or shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    so = str(tmp_path_factory.mktemp("repr") / "librepr.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "shortest_repr_host.cpp")])
    lib = ctypes.CDLL(so)
    lib.repr_lines_f32.restype = ctypes.c_int64
    lib.repr_lines_f32.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]

    def run(v):
        v = np.ascontiguousarray(v, np.float32)
        buf = np.empty(25 * len(v) + 1, np.uint8)
        n = lib.repr_lines_f32(v.ctypes.data, len(v), buf.ctypes.data)
        assert n >= 0, "value %d: repr_length disagrees with repr_write" % (-1 - n)
        return buf[:n].tobytes()
    return run


def _first_difference(got, want, v):
    g, w = got.split(b"\n"), want.split(b"\n")
    bad = next(i for i in range(min(len(g), len(w))) if g[i] != w[i])
    return "float32 %r: got %r, repr %r" % (v[bad], g[bad], w[bad])


def test_host_formatter_equals_repr_on_binades_and_random(host_formatter):
    assert host_formatter(SPECIALS) == repr_lines(SPECIALS)
    for name, v in sweep():
        got, want = host_formatter(v), repr_lines(v)
        assert got == want, "%s: %s" % (name, _first_difference(got, want, v))


# ---- GPU --------------------------------------------------------------------------------------------------------
def _text(ev, labels=None):
    import torch
    from v2e_b200 import sinks
    d = torch.from_numpy(np.ascontiguousarray(ev, np.float32)).cuda()
    lab = None if labels is None else torch.from_numpy(np.asarray(labels, np.uint8)).cuda()
    out = sinks.events_to_text(d, lab)
    assert out.is_cuda and out.dtype == torch.uint8
    return out.cpu().numpy().tobytes()


@pytest.mark.gpu
def test_cuda_text_matches_reference_bytes():
    ev = G["text_events"]
    assert _text(ev) == G["text_body"].tobytes()
    assert _text(ev, G["text_labels"]) == G["text_body_labeled"].tobytes()
    assert _text(ev, G["text_labels"].astype(np.uint8)) == text_sink_oracle.text_body(ev, G["text_labels"])


@pytest.mark.gpu
def test_cuda_text_small_and_special_rows():
    import torch
    from v2e_b200 import sinks
    assert _text(np.zeros((0, 4), np.float32)) == b"" and _text(np.zeros((0, 4), np.float32), []) == b""
    one = np.array([[0.1, 3, 7, -1]], np.float32)
    assert _text(one) == b"0.10000000149011612 3 7 0\n"
    assert _text(one, [1]) == b"0.10000000149011612 3 7 0 1\n"
    n = len(SPECIALS)
    rng = np.random.default_rng(1)
    ev = np.stack([SPECIALS, rng.integers(0, 65536, n), rng.integers(0, 65536, n), rng.choice([-1.0, 1.0], n)],
                  1).astype(np.float32)
    ev[:4, 1:3] = [[0, 0], [65535, 65535], [-1, -65535], [2 ** 31 - 128, -2 ** 31]]     # int32 extremes, signs
    lab = rng.integers(0, 256, n).astype(np.uint8)
    assert _text(ev) == text_sink_oracle.text_body(ev)
    assert _text(ev, lab) == text_sink_oracle.text_body(ev, lab)
    with pytest.raises(ValueError):
        sinks.events_to_text(torch.zeros((3, 4), device="cuda"), torch.ones(2, dtype=torch.uint8, device="cuda"))


@pytest.mark.gpu
def test_cuda_text_equals_oracle_on_binades_and_random():
    """The CPU sweep on the device, millions of rows per call (many 256-row blocks and scan runs), x and y over
    [0, 65535], labels on every other call."""
    k = 0
    for name, v in sweep():
        n = len(v)
        idx = np.arange(n, dtype=np.int64)
        ev = np.stack([v, idx % 65536, (idx * 7919) % 65536, np.where(idx % 3 == 0, -1.0, 1.0)], 1).astype(np.float32)
        lab = (idx % 5 != 0) if k % 2 else None
        got, want = _text(ev, lab), text_sink_oracle.text_body(ev, lab)
        assert got == want, "%s: %s" % (name, _first_difference(got, want, v))
        k += 1


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_cuda_labeled_aedat2_matches_reference_bytes(size):
    import torch
    from v2e_b200 import sinks
    w, h = size
    ev = torch.from_numpy(G["aedat2_events_%dx%d" % size]).cuda()
    lab = G["aedat2_labels_%dx%d" % size]
    words, n_on = sinks.events_to_aedat2(ev, w, h, labels=torch.from_numpy(lab).cuda())
    assert words.cpu().numpy().tobytes() == G["aedat2_body_%dx%d" % size].tobytes()
    plain, plain_on = sinks.events_to_aedat2(ev, w, h)
    again, _ = sinks.events_to_aedat2(ev, w, h, labels=None)
    want, want_on = sinks_oracle.aedat2_words(G["aedat2_events_%dx%d" % size], w, h)
    assert plain.cpu().numpy().tobytes() == again.cpu().numpy().tobytes() == want.tobytes()
    assert int(n_on.item()) == int(plain_on.item()) == want_on


def _signnoise(n_rows, n_noise):
    lab = np.ones(n_rows, bool)
    lab[n_rows - n_noise:] = False
    return lab


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["emu_static_leak_shot", "emu_cli_noisy", "emu_refractory_multi"])
def test_replay_labels_mark_the_oracle_shot_rows(name):
    """Replay mode on fixtures with shot noise (the reference's draws from the fixture's tape; the static scene has
    only shot rows, the others signal and shot rows in the same frames): frame by frame the rows equal the
    reference's and last_signnoise_label is 0 on exactly the oracle's shot-noise rows, its last ones."""
    from emu_oracle import OracleEmulator
    from helpers import TapeRNG, load_golden, split_events
    from text_sink_oracle import LabelCountingRNG, frame_labels
    from v2e_b200 import EventEmulator
    g = load_golden(name)
    orc = OracleEmulator(rng=LabelCountingRNG(TapeRNG(g["tape"])), **g["kwargs"])
    em = EventEmulator(device="cuda", rng=TapeRNG(g["tape"]), label_signal_noise=True, **g["kwargs"])
    plain = EventEmulator(device="cuda", rng=TapeRNG(g["tape"]), **g["kwargs"])
    want_rows = split_events(g["events"], g["event_counts"])
    n_noise = n_signal = 0
    for i, (f, t) in enumerate(zip(g["frames"], g["times"])):
        want, want_lab = frame_labels(orc, f, float(t))
        ev = em.generate_events(f, float(t))
        assert plain.last_signnoise_label is None
        plain.generate_events(f, float(t))
        if want is None:
            assert ev is None and em.last_signnoise_label is None
            continue
        assert np.array_equal(ev, want) and np.array_equal(ev, want_rows[i]), "frame %d" % i
        s = int((~want_lab).sum())
        lab = em.last_signnoise_label
        assert np.array_equal(want_lab, _signnoise(len(want), s))
        assert lab.dtype == bool and np.array_equal(lab, want_lab), "frame %d" % i
        n_noise += s
        n_signal += len(want) - s
    assert n_noise > 0 and (n_signal > 0) == (name != "emu_static_leak_shot")
    assert n_noise + n_signal == orc.num_events_total
    assert plain.last_signnoise_label is None


def _texture(H, W, T, seed):
    rng = np.random.default_rng(seed)
    big = np.kron(rng.integers(0, 256, (H // 4 + T + 4, W // 4 + T + 4)), np.ones((4, 4))).astype(np.uint8)
    return np.stack([np.ascontiguousarray(big[k:k + H, 2 * k:2 * k + W]) for k in range(T)])


@pytest.mark.gpu
@pytest.mark.parametrize("mfps", [1, 24])
def test_device_rng_labels_equal_oracle_split(mfps):
    """rng_mode='device', generate_events_batch(return_labels=True): per frame the labels are 1 then 0, the zeros
    being exactly the shot-noise rows of the oracle fed the device's own draws; zeros = sum of the shot counts."""
    import torch
    from emu_oracle import OracleEmulator
    from helpers import DeviceDrawRNG, canonical
    from text_sink_oracle import LabelCountingRNG, frame_labels
    from v2e_b200 import EventEmulator
    kw = dict(cutoff_hz=100, leak_rate_hz=5.0, shot_noise_rate_hz=40.0, refractory_period_s=0.0005)
    frames = _texture(37, 53, 12, seed=4)
    ts = [k * 2e-3 for k in range(len(frames))]
    torch.manual_seed(7)
    em = EventEmulator(device="cuda", rng_mode="device", seed=7, label_signal_noise=True, max_frames_per_step=mfps,
                       **kw)
    rows, offs, lab = em.generate_events_batch(frames, ts, return_labels=True)
    assert lab.dtype == bool and lab.shape == (len(rows),)
    torch.manual_seed(7)
    rng = DeviceDrawRNG(lambda k: em.device_draws(k - 1))
    orc = OracleEmulator(seed=7, rng=LabelCountingRNG(rng), shuffle=False, **kw)
    total_shot = 0
    for k, (f, t) in enumerate(zip(frames, ts)):
        rng.frame = k
        want, want_lab = frame_labels(orc, f, t)
        a, b = int(offs[k]), int(offs[k + 1])
        if want is None:
            assert a == b
            continue
        s = int((~want_lab).sum())
        assert np.array_equal(want_lab, _signnoise(len(want), s))
        assert b - a == len(want) and np.array_equal(lab[a:b], want_lab), "frame %d" % k
        assert np.array_equal(canonical(rows[a:b][~lab[a:b]]), canonical(want[len(want) - s:])), "frame %d" % k
        total_shot += s
    assert total_shot > 0 and int((~lab).sum()) == total_shot
    r2, o2, l2 = EventEmulator(device="cuda", rng_mode="device", seed=7, label_signal_noise=True,
                               **kw).generate_events_batch(frames, ts, return_device=True, return_labels=True)
    assert l2.is_cuda and l2.dtype == torch.uint8 and np.array_equal(l2.cpu().numpy().astype(bool), lab)
    with pytest.raises(ValueError):
        EventEmulator(device="cuda", rng_mode="device", **kw).generate_events_batch(frames, ts, return_labels=True)


_E2E = r"""
import os, sys
import numpy as np
sys.path[:0] = [{root!r}, os.path.join({root!r}, "oracle"), os.path.join({root!r}, "tests")]
import ref_shim
ref_shim.load_reference()
from helpers import TapeRNG, load_golden
from v2e_b200 import EventEmulator
g = load_golden("emu_cli_noisy")
em = EventEmulator(device="cuda", rng=TapeRNG(g["tape"]), output_folder={out!r}, dvs_text="ev", dvs_aedat2="ev",
                   output_width=346, output_height=260, label_signal_noise=True, **g["kwargs"])
assert em.dvs_text is not None and em.dvs_aedat2 is not None
rows, labels = [], []
for f, t in zip(g["frames"], g["times"]):
    ev = em.generate_events(f, float(t))
    if ev is not None:
        rows.append(ev)
        labels.append(em.last_signnoise_label)
n = em.dvs_text.numEventsWritten
em.cleanup()
np.savez(os.path.join({out!r}, "rows.npz"), rows=np.concatenate(rows), labels=np.concatenate(labels), n=n)
"""


@pytest.mark.gpu
def test_emulator_writes_labeled_text_and_aedat2_files(tmp_path):
    """dvs_text + dvs_aedat2 + label_signal_noise through the reference's writers (a subprocess: loading the reference
    stubs modules): the file bodies equal the oracle applied to the returned rows and labels."""
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    subprocess.check_call([sys.executable, "-c", _E2E.format(root=ROOT, out=str(tmp_path))])
    r = np.load(tmp_path / "rows.npz")
    rows, labels = r["rows"], r["labels"]
    assert int(r["n"]) == len(rows) and (~labels).sum() > 0 and labels.sum() > 0
    text = (tmp_path / "ev.txt").read_bytes()
    lines = text.split(b"\n")
    n_head = next(i for i, ln in enumerate(lines) if not ln.startswith(b"#"))
    head = sum(len(ln) + 1 for ln in lines[:n_head])
    assert text.startswith(b"#!events.txt") and b"signal/noise" in text[:head]
    assert text[head:] == text_sink_oracle.text_body(rows, labels)
    words, _ = text_sink_oracle.aedat2_words_labeled(rows, 346, 260, labels)
    aedat = (tmp_path / "ev.aedat").read_bytes()
    assert aedat.startswith(b"#!AER-DAT2.0") and aedat[len(aedat) - 8 * len(rows):] == words.tobytes()
