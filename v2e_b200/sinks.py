"""Event-sink row conversions on the device (SURVEY.md 8f rank 3).

The reference converts the emitted rows on the host, per frame, inside generate_events
(emulator.py:953-975 -> v2ecore/output/aedat2_output.py:133-188, ae_text_output.py:68-101). Here the packed
device rows are converted by CUDA kernels and the caller copies file-ready bytes: 8 per event for AEDAT-2.0
instead of 16 for the float rows, and the exact lines of the DVS text (RPG events.txt) writer. File headers
stay with the writers.

Signal / noise labels (label_signal_noise, emulator.py:889-923) are uint8 CUDA tensors [N], 1 = signal and
0 = shot noise; `signnoise_labels` builds them from per-frame row offsets and shot counts."""
import ctypes
import io

import torch

from . import _lib

# aedat2_output.py:38-60: (width, height) -> yShiftBits, xShiftBits, polShiftBits; flipx = flipy = True
AEDAT2_LAYOUTS = {(346, 260): (22, 12, 11), (240, 180): (22, 12, 11), (640, 480): (11, 1, 0)}


def _check(events):
    if not (isinstance(events, torch.Tensor) and events.is_cuda and events.dtype == torch.float32
            and events.dim() == 2 and events.shape[1] == 4 and events.is_contiguous()):
        raise ValueError("events must be a contiguous CUDA float32 tensor [N, 4]")


def _labels(labels, events):
    """-> the label tensor as contiguous uint8 on the events' device (None stays None)."""
    if labels is None:
        return None
    if not isinstance(labels, torch.Tensor):
        labels = torch.as_tensor(labels)
    if labels.dim() != 1 or labels.shape[0] != events.shape[0]:
        raise ValueError("labels must be [N] for N event rows")
    if labels.device != events.device:
        labels = labels.to(events.device)
    if labels.dtype != torch.uint8:
        labels = labels.to(torch.uint8) if labels.dtype == torch.bool else (labels != 0).to(torch.uint8)
    return labels.contiguous()


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def events_to_h5_rows(events):
    """[N,4] float32 rows [t,x,y,p] -> [N,4] uint32 rows [t_us, x, y, p01] (emulator.py:953-959)."""
    _check(events)
    out = torch.empty((events.shape[0], 4), dtype=torch.int32, device=events.device)
    lib = _lib.load()
    with torch.cuda.device(events.device):
        st = ctypes.c_void_p(torch.cuda.current_stream(events.device).cuda_stream)
        _lib.check(lib.v2e_events_to_h5_rows(ctypes.c_void_p(events.data_ptr()), events.shape[0],
                                             ctypes.c_void_p(out.data_ptr()), st))
    return out.view(torch.int32)    # bit pattern of the uint32 rows (torch has no uint32 arithmetic)


def events_to_aedat2(events, output_width=346, output_height=260, labels=None):
    """[N,4] float32 rows -> ([2N] int32 big-endian words ready for file.write(), number of ON events),
    as AEDat2Output.appendEvents builds them (aedat2_output.py:133-165). Raises ValueError for a size the
    reference's writer does not support (aedat2_output.py:61-63). labels ([N], 0 = shot noise): noise rows
    set the special-event bit 1 << 10 of their address, as AEDat2Output(label_signal_noise=True) does
    (:154-158), also at 640x480 where that bit overlaps x."""
    _check(events)
    key = (int(output_width), int(output_height))
    if key not in AEDAT2_LAYOUTS:
        raise ValueError("AEDAT-2.0 output width=%d height=%d not supported" % key)
    ys, xs, ps = AEDAT2_LAYOUTS[key]
    lab = _labels(labels, events)
    n = events.shape[0]
    out = torch.empty((2 * n,), dtype=torch.int32, device=events.device)
    n_on = torch.zeros((1,), dtype=torch.int64, device=events.device)
    lib = _lib.load()
    with torch.cuda.device(events.device):
        st = ctypes.c_void_p(torch.cuda.current_stream(events.device).cuda_stream)
        _lib.check(lib.v2e_events_to_aedat2(ctypes.c_void_p(events.data_ptr()), n, key[0], key[1], xs, ys, ps, 1, 1,
                                            _ptr(lab), ctypes.c_void_p(out.data_ptr()),
                                            ctypes.c_void_p(n_on.data_ptr()), st))
    return out, n_on


def events_to_text(events, labels=None):
    """[N,4] float32 rows -> uint8 CUDA tensor holding the DVS text body that DVSTextOutput.appendEvents means to
    write (ae_text_output.py:89-101): per row '{} {} {} {}\\n'.format(float(t), int(x), int(y), int((p + 1) / 2)),
    float(t) being repr() of the float32 timestamp as a double, and with labels ([N], 1 = signal, 0 = noise)
    ' {label}' before the newline. Synchronises once, to read the body's length."""
    _check(events)
    lab = _labels(labels, events)
    n = events.shape[0]
    lib = _lib.load()
    with torch.cuda.device(events.device):
        st = ctypes.c_void_p(torch.cuda.current_stream(events.device).cuda_stream)
        offs = torch.empty((int(lib.v2e_events_to_text_scratch(n)),), dtype=torch.int64, device=events.device)
        _lib.check(lib.v2e_events_to_text_layout(_ptr(events), n, _ptr(lab), _ptr(offs), st))
        total = int(offs[-1].item())
        out = torch.empty((total,), dtype=torch.uint8, device=events.device)
        _lib.check(lib.v2e_events_to_text(_ptr(events), n, _ptr(lab), _ptr(offs), _ptr(out), st))
    return out


def write_text(fileobj, events, labels=None):
    """Appends the text lines of device rows `events` (see events_to_text) to an open file: one device-to-host
    copy, one write. A text-mode file (DVSTextOutput.file) gets str, a binary one bytes. Returns the row count."""
    body = events_to_text(events, labels).cpu().numpy().tobytes()
    fileobj.write(body.decode("ascii") if isinstance(fileobj, io.TextIOBase) else body)
    return events.shape[0]


def signnoise_labels(offsets, n_noise, device):
    """Labels [offsets[-1]] uint8 on `device` of a chunk of frames whose rows are [offsets[f], offsets[f+1]) and whose
    last n_noise[f] rows are shot noise (V2eFrameInfo n_shot_on + n_shot_off): 1 = signal, 0 = noise
    (emulator.py:889-923)."""
    offsets = torch.as_tensor(offsets, dtype=torch.int64)
    n_noise = torch.as_tensor(n_noise, dtype=torch.int32)
    T = int(n_noise.shape[0])
    if offsets.shape[0] != T + 1:
        raise ValueError("offsets must have one entry more than n_noise")
    n = int(offsets[-1])
    out = torch.empty((n,), dtype=torch.uint8, device=device)
    if n == 0:
        return out
    o_dev, s_dev = offsets.to(device), n_noise.to(device)
    lib = _lib.load()
    with torch.cuda.device(out.device):
        st = ctypes.c_void_p(torch.cuda.current_stream(out.device).cuda_stream)
        _lib.check(lib.v2e_signnoise_labels(_ptr(o_dev), _ptr(s_dev), T, n, _ptr(out), st))
    return out
