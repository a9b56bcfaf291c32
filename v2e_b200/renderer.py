"""EventRenderer -- drop-in for v2ecore/renderer.py:26 (render_events_to_frames, :161) with the histogram on the GPU
(csrc/render.cu; SURVEY.md 8f rank 4).

Same constructor keywords and the same frames, quirks included (restated and pinned in oracle/render_oracle.py): the
frame being filled is dropped at the start of every call (renderer.py:270), the last event of a packet is never
rendered (:300-303), DURATION boundaries are searchsorted(left / right) over the whole packet so an event exactly on a
boundary lands in both frames. Which rows belong to which frame, and each frame's time, is the frame plan, computed on
the device for all packets of a call at once (v2e_render_plan; AREA_COUNT, a sequential data-dependent scan
(renderer.py:246-261), by one device thread in v2e_render_area_scan); the scatter-add, clip and normalisation run on the
device too, in chunks of RENDER_CHUNK_FRAMES frames. render_events_to_frames renders one packet; render_frame_rows
renders the rows of consecutive pixel-model frames in the packets v2e.py forms. Writing the AVI (`dvs_vid`) is the
reference's job: it is delegated to v2ecore.v2e_utils.video_writer when that imports, otherwise ignored with a warning.
`video_writer` (a factory with that function's signature, e.g. v2e_b200.video.MjpegWriter) replaces it for this object's
video; a writer with write_frames gets each chunk's uint8 frames on the device, with no host copy and no GRAY2BGR.
"""
import ctypes
import logging
import os
from enum import Enum

import numpy as np
import torch

from . import _lib

logger = logging.getLogger(__name__)

# DVS frames rendered per launch: the render's int32 accumulators and uint8 frames hold this many frames whatever a call
# finishes (at 1280x720: 16 x 3.7 MB + 16 x 0.9 MB on the device, and 16 x 0.9 MB of pinned host memory for the video).
RENDER_CHUNK_FRAMES = 16


class ExposureMode(Enum):
    DURATION = 1
    COUNT = 2
    AREA_COUNT = 3
    SOURCE = 4


class EventRenderer(object):
    def __init__(self, full_scale_count=3, output_path=None, dvs_vid=None, preview=False,
                 exposure_mode=ExposureMode.DURATION, exposure_value=1 / 300.0, area_dimension=None,
                 frame_times_suffix='-frame_times.txt', avi_frame_rate=30, device="cuda:0", video_writer=None):
        mode = exposure_mode if isinstance(exposure_mode, ExposureMode) else ExposureMode(getattr(exposure_mode, "value", exposure_mode))
        self.exposure_mode = mode
        self.exposure_value = exposure_value
        self.output_path = output_path
        self.width = self.height = None
        self.full_scale_count = full_scale_count
        self.dvs_frame_times_suffix = frame_times_suffix
        self.frame_rate_hz = self.event_count = self.frameIntevalS = None
        self.avi_frame_rate = avi_frame_rate
        self.area_counts = self.area_count = None
        self.area_dimension = area_dimension
        if mode == ExposureMode.DURATION:
            self.frame_rate_hz = 1 / self.exposure_value           # renderer.py:91-93
            self.frameIntevalS = 1 / self.frame_rate_hz
        elif mode == ExposureMode.COUNT:
            self.event_count = int(self.exposure_value)
            if self.event_count < 1:                      # a frame of 0 events never advances: renderer.py:283-285
                raise ValueError("ExposureMode.COUNT needs an event count of at least 1, got %r" % (exposure_value,))
        elif mode == ExposureMode.AREA_COUNT:
            self.area_count = int(self.exposure_value)
            if not area_dimension:
                raise ValueError("ExposureMode.AREA_COUNT needs area_dimension")
            # the event that closes a frame opens the next one and counts 1 there: with area_count 1 that frame closes
            # on the same event again and the scan never advances (renderer.py:254-265)
            if self.area_count < 2:
                raise ValueError("ExposureMode.AREA_COUNT needs an area count of at least 2, got %r" % (exposure_value,))
        self.video_output_file_name = dvs_vid
        self.video_writer = video_writer
        self.video_output_file = None
        self.frame_times_output_file = None
        self.preview = preview
        if preview:
            logger.warning("preview windows are out of scope here: ignored")
        self.numFramesWritten = 0
        self.currentFrameStartTime = None
        self.currentFrame = None
        self.printed_empty_packet_warning = False
        self.device = torch.device(device)
        self._lib = _lib.load()
        self._bufs = {}                                 # reused plan / chunk buffers (_buf)
        self._plan_frames = 4096                        # DURATION plan capacity, grown when a call finishes more frames
        self._held, self._n_held = None, 0              # rows render_frame_rows holds for the next call's first packet

    def cleanup(self):
        if self.video_output_file is not None:
            self.video_output_file.release()
            self.video_output_file = None
        if self.frame_times_output_file is not None:
            self.frame_times_output_file.close()
            self.frame_times_output_file = None

    def _check_outputs_open(self):
        """renderer.py:141-170, through the reference's own writer when it imports, or the video_writer factory."""
        if self.video_output_file is not None or not (self.output_path and type(self.video_output_file_name) is str):
            return
        if self.video_writer is not None:
            video_writer, checkAddSuffix = self.video_writer, _with_suffix
        else:
            try:
                from v2ecore.v2e_utils import checkAddSuffix, video_writer
            except ImportError as e:
                logger.warning("dvs_vid ignored: v2ecore.v2e_utils.video_writer is not importable (%s)", e)
                self.video_output_file_name = None
                return
        fn = checkAddSuffix(os.path.join(self.output_path, self.video_output_file_name), '.avi')
        self.video_output_file = video_writer(fn, self.height, self.width, frame_rate=self.avi_frame_rate)
        fn = checkAddSuffix(os.path.join(self.output_path, self.video_output_file_name), self.dvs_frame_times_suffix)
        self.frame_times_output_file = open(fn, 'w')
        self.frame_times_output_file.write('# frame times for {}\n# frame# time(s)\n'.format(self.video_output_file_name))

    # -- the frame plan and the frames ----------------------------------------------------------------------------
    def _buf(self, name, n, dtype, pinned=False, shape=()):
        """A reused buffer of at least n entries (device, or pinned host), grown to twice what overflowed it."""
        b = self._bufs.get(name)
        if b is None or b.shape[0] < n or tuple(b.shape[1:]) != tuple(shape):
            size = max(n, 2 * b.shape[0] if b is not None and tuple(b.shape[1:]) == tuple(shape) else n)
            b = (torch.empty((size,) + tuple(shape), dtype=dtype).pin_memory() if pinned else
                 torch.empty((size,) + tuple(shape), dtype=dtype, device=self.device))
            self._bufs[name] = b
        return b

    def _plan(self, rows0, rows, packets):
        """The frame plan of packets (int64 [P, 2] row ranges; packet 0 of rows0 when rows0 is not None, the others of
        rows), one host synchronisation. Returns (frames, largest slice, packet_first [P+1], frame times as the
        frame-times file states them or None without a video); commits the carried DURATION start. Raises ValueError,
        before any state changes, for a DURATION packet spanning 2^20 frame intervals or more."""
        mode, P = self.exposure_mode, len(packets)
        sizes = packets[:, 1] - packets[:, 0]
        if mode == ExposureMode.COUNT:
            cap = int(np.sum(np.maximum(sizes - 2, 0) // self.event_count))
        elif mode == ExposureMode.SOURCE:
            cap = P
        elif mode == ExposureMode.AREA_COUNT:
            # every frame but the first of a packet advances at least area_count - 1 events: the event that closes a
            # frame is counted again as the first of the next one
            cap = int(np.sum(sizes // (self.area_count - 1) + 2))
        else:
            cap = self._plan_frames
        cap = max(cap, 1)
        pk = torch.from_numpy(np.ascontiguousarray(packets, np.int64)).to(self.device)
        want_times = self.video_output_file is not None
        p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
        f64 = False
        while True:
            starts, ends = self._buf("starts", cap, torch.int64), self._buf("ends", cap, torch.int64)
            times, hdr = self._buf("times", cap, torch.float64), self._buf("hdr", 8 + P + 1, torch.int64)
            first = hdr[8:]
            with torch.cuda.device(self.device):
                stream = torch.cuda.current_stream(self.device)
                sp = ctypes.c_void_p(stream.cuda_stream)
                if mode == ExposureMode.AREA_COUNT:
                    if self.area_counts is None:
                        self._cells = (1 + self.width // self.area_dimension, 1 + self.height // self.area_dimension)
                        self.area_counts = torch.zeros(self._cells, dtype=torch.int32, device=self.device)
                    _lib.check(self._lib.v2e_render_area_scan(
                        p(rows0), p(rows), p(pk), P, int(rows0 is not None), int(self.area_dimension),
                        int(self.area_count), self._cells[0], self._cells[1], p(self.area_counts), p(starts), p(ends),
                        p(times), cap, p(hdr), p(first), sp))
                else:
                    cur, has = self.currentFrameStartTime, self.currentFrameStartTime is not None
                    if mode == ExposureMode.DURATION:
                        # the starts accumulate in the dtype numpy gives the first row's float32 time plus the interval
                        f64 = isinstance(np.float32(0) + self.frameIntevalS, np.float64)
                    _lib.check(self._lib.v2e_render_plan(
                        p(rows0), p(rows), p(pk), P, int(rows0 is not None), mode.value,
                        float(self.frameIntevalS or 0.0), int(f64), int(self.event_count or 0),
                        float(cur) if has else 0.0, int(has), p(self._buf("bounds", 2 * cap, torch.float64)),
                        p(starts), p(ends), p(times), cap, p(hdr), p(first), sp))
                hdr_h = self._buf("hdr_host", 8 + P + 1, torch.int64, pinned=True)
                hdr_h[:8 + P + 1].copy_(hdr[:8 + P + 1], non_blocking=True)
                if want_times:
                    times_h = self._buf("times_host", cap, torch.float64, pinned=True)
                    times_h[:cap].copy_(times[:cap], non_blocking=True)
                stream.synchronize()
            h = hdr_h[:8 + P + 1].numpy().copy()
            status, F, big = int(h[0]), int(h[1]), int(h[2])
            if status == 2:
                bits = h[6:8].view(np.float64)
                raise ValueError("a DURATION packet may span at most 2^20 frame intervals of %g s; packet %d of this call "
                                 "runs from %r s to %r s: pass it in shorter packets"
                                 % (self.frameIntevalS, int(h[5]), float(bits[0]), float(bits[1])))
            if status == 1 and mode == ExposureMode.DURATION:
                cap = self._plan_frames = 2 * F                 # the plan is a pure function of its inputs: run it again
                continue
            if status != 0:
                raise RuntimeError("render plan: more frames than its slice table holds")
            break
        if mode == ExposureMode.DURATION and h[4]:
            cur = h[3:4].view(np.float64)[0]
            self.currentFrameStartTime = np.float64(cur) if f64 else np.float32(cur)
        t = times_h[:F].numpy().copy() if want_times else None
        if t is not None and not f64:
            t = t.astype(np.float32)                            # the float32 scalars the reference formats
        return F, big, h[8:], t

    def _render_packets(self, rows0, rows, packets, want_img):
        """Renders packets (see _plan) in chunks of RENDER_CHUNK_FRAMES frames into reused buffers: each chunk's uint8
        frames go to the video (one device-to-host copy per chunk) and, with want_img, its float64 frames into the
        returned [F, H, W] tensor. Returns (F, frames or None)."""
        H, W = int(self.height), int(self.width)
        F, big, first, times = self._plan(rows0, rows, packets)
        want_u8 = self.video_output_file is not None
        if F == 0 or not (want_u8 or want_img):
            return F, None
        on_device = want_u8 and hasattr(self.video_output_file, "write_frames")
        starts, ends = self._bufs["starts"], self._bufs["ends"]
        img = torch.empty((F, H, W), dtype=torch.float64, device=self.device) if want_img else None
        ch = min(RENDER_CHUNK_FRAMES, F)
        acc = self._buf("acc", ch, torch.int32, shape=(H, W))
        u8 = self._buf("u8", ch, torch.uint8, shape=(H, W)) if want_u8 else None
        u8_h = self._buf("u8_host", ch, torch.uint8, pinned=True, shape=(H, W)) if want_u8 and not on_device else None
        p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
        k0 = int(first[1]) if rows0 is not None else 0          # packet 0's frames read rows0
        if want_u8 and not on_device:
            import cv2
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            sp = ctypes.c_void_p(stream.cuda_stream)
            for a, b, src in ((0, k0, rows0), (k0, F, rows)):
                for c in range(a, b, ch):
                    n = min(ch, b - c)
                    _lib.check(self._lib.v2e_render_frames(
                        p(src), ctypes.c_void_p(starts.data_ptr() + 8 * c), ctypes.c_void_p(ends.data_ptr() + 8 * c),
                        n, big, H, W, int(self.full_scale_count), p(acc), None if img is None else p(img[c]), p(u8), sp))
                    if not want_u8:
                        continue
                    if on_device:
                        self.video_output_file.write_frames(u8[:n])
                    else:
                        u8_h[:n].copy_(u8[:n], non_blocking=True)
                        stream.synchronize()
                        host = u8_h[:n].numpy()
                    for f in range(n):
                        if not on_device:
                            self.video_output_file.write(cv2.cvtColor(host[f], cv2.COLOR_GRAY2BGR))
                        self.frame_times_output_file.write('{}\t{:10.6f}\n'.format(self.numFramesWritten, times[c + f]))
                        self.numFramesWritten += 1
        return F, img

    def render_events_to_frames(self, event_arr, height, width, return_frames=False, return_device=False):
        """renderer.py:161: float64 frames [k, height, width] in 0..1 for the frames this packet finished, or None.
        The one-packet case of render_frame_rows' plan."""
        self.width, self.height = width, height
        self._check_outputs_open()
        if event_arr is None or event_arr.shape[0] == 0:
            self.printed_empty_packet_warning = True
            return None
        if isinstance(event_arr, np.ndarray):
            ev = torch.from_numpy(np.ascontiguousarray(event_arr, dtype=np.float32)).to(self.device)
        else:
            ev = event_arr.to(self.device, torch.float32).contiguous()
        self.currentFrame = None                          # renderer.py:270
        k, img = self._render_packets(None, ev, np.array([[0, ev.shape[0]]], np.int64), return_frames or return_device)
        if k == 0:
            return None
        if return_device:
            return img
        return img.cpu().numpy() if return_frames else None

    def render_frame_rows(self, rows, offsets, first_frame, packet_frames, end_of_clip=False, height=None, width=None):
        """Renders the rows of consecutive pixel-model frames first_frame .. first_frame+T-1 in the packets v2e.py's
        stage-3 loop (v2e.py:826-846) hands render_events_to_frames, with batch_size = packet_frames: frame i's rows
        join the packet, and when frame i has rows and i % packet_frames == 0 the packet is rendered. rows: [N, 4]
        float32 (a CUDA tensor, read in place, or an ndarray); frame first_frame + j has rows[offsets[j]:offsets[j+1]]
        (offsets [T+1]). The rows after the call's last packet are held in a buffer the renderer owns and lead the next
        call's first packet; end_of_clip=True renders them as v2e.py's leftover packet. height / width: the frame size
        (default: that of the previous call). Writes the DVS video and its frame-times file when dvs_vid is open, and
        returns the number of frames the packets finished.

        One host synchronisation per call reads the plan, plus one copy per RENDER_CHUNK_FRAMES frames of video; no
        timestamps go to the host, and of the call's rows only the packet that starts in an earlier call is copied.
        Raises ValueError, with nothing of the call written and nothing held, for a DURATION packet spanning 2^20
        frame intervals or more."""
        if height is not None or width is not None:
            self.height, self.width = int(height), int(width)
        if self.height is None or self.width is None:
            raise ValueError("render_frame_rows needs the frame size: pass height and width")
        self._check_outputs_open()
        if isinstance(offsets, torch.Tensor):
            offsets = offsets.cpu().numpy()
        offsets = np.asarray(offsets, np.int64)
        if offsets.ndim != 1 or offsets.shape[0] < 1 or np.any(np.diff(offsets) < 0):
            raise ValueError("offsets must be a non-decreasing [T+1] array")
        if isinstance(rows, np.ndarray):
            rows = torch.from_numpy(np.ascontiguousarray(rows, dtype=np.float32)).to(self.device)
        else:
            rows = rows.to(self.device, torch.float32).contiguous()
        base, n_new, held = int(offsets[0]), int(offsets[-1] - offsets[0]), self._n_held
        if rows.shape[0] < base + n_new:
            raise ValueError("offsets run to row %d of %d rows" % (base + n_new, rows.shape[0]))
        ends, keep = cut_packets(offsets, first_frame, packet_frames, held, end_of_clip)
        call = rows[base:base + n_new]
        if len(ends) == 0:                                      # the call's rows all join the held packet
            self._hold(call, held)
            self._n_held = held + n_new
            return 0
        rows0 = None
        packets = np.stack([np.concatenate([[0], ends[:-1]]), ends], 1) - held
        if held:
            # the packet that straddles the previous call: its head is held, its tail is this call's first rows
            rows0 = self._hold(call[:ends[0] - held], held)
            packets[0] = (0, ends[0])
        self.currentFrame = None                          # renderer.py:270
        k, _ = self._render_packets(rows0, call, packets, False)
        self._n_held = 0
        self._hold(call[keep - held:], 0)
        self._n_held = n_new - (keep - held)
        return k

    def _hold(self, rows, at):
        """Copies rows into the held-row buffer at row `at` (rows before it are kept); returns the buffer."""
        need = at + rows.shape[0]
        buf = self._held
        if buf is None or buf.shape[0] < need:
            grown = torch.empty((max(2 * need, 1024), 4), dtype=torch.float32, device=self.device)
            if at:
                grown[:at].copy_(buf[:at])
            self._held = buf = grown
        if rows.shape[0]:
            buf[at:need].copy_(rows)
        return buf


def _with_suffix(path, suffix):
    """The path with its extension replaced by suffix, unless it already ends in suffix (what the reference's
    checkAddSuffix does to the video and frame-times names)."""
    return path if path.endswith(suffix) else os.path.splitext(path)[0] + suffix


def cut_packets(offsets, first_frame, packet_frames, held=0, end_of_clip=False):
    """The packets v2e.py's stage-3 loop (v2e.py:826-846) renders from the rows of frames first_frame .. first_frame+T-1
    (frame first_frame + j has rows offsets[j] .. offsets[j+1]), behind `held` rows carried from earlier frames: frame
    i's rows join the packet; when frame i has rows and i % packet_frames == 0 the packet is rendered; end_of_clip
    renders what is left when any rows are. Rows are numbered held rows first, then the call's rows. Returns
    (ends, keep): packet j is rows [ends[j-1], ends[j]) (ends[-1] read as 0), and rows keep .. held + N are held for
    the next call."""
    offsets = np.asarray(offsets, np.int64)
    pf = int(packet_frames)
    if pf < 1:
        raise ValueError("packet_frames=%d: a packet needs at least one frame" % pf)
    n = offsets[1:] - offsets[:-1]
    i = int(first_frame) + np.arange(n.shape[0], dtype=np.int64)
    ends = int(held) + offsets[1:][(n > 0) & (i % pf == 0)] - offsets[0]
    total = int(held) + int(offsets[-1] - offsets[0])
    keep = int(ends[-1]) if len(ends) else 0
    if end_of_clip and total > keep:
        ends = np.append(ends, total)
        keep = total
    return ends.astype(np.int64), keep
