"""EventRenderer -- drop-in for v2ecore/renderer.py:26 (render_events_to_frames, :161) with the histogram on the GPU
(csrc/render.cu; SURVEY.md 8f rank 4).

Same constructor keywords and the same frames, quirks included (restated and pinned in oracle/render_oracle.py): the
frame being filled is dropped at the start of every call (renderer.py:270), the last event of a packet is never
rendered (:300-303), DURATION boundaries are searchsorted(left / right) over the whole packet so an event exactly on a
boundary lands in both frames. Host code here decides which rows belong to which frame (exposure bookkeeping); the
scatter-add, clip and normalisation run on the device. AREA_COUNT exposure is a sequential data-dependent scan
(renderer.py:246-261): one device thread walks the packet (v2e_render_area_scan). Writing the AVI (`dvs_vid`) is the reference's job: it is delegated
to v2ecore.v2e_utils.video_writer when that imports, otherwise ignored with a warning.
"""
import ctypes
import logging
import os
from enum import Enum

import numpy as np
import torch

from . import _lib

logger = logging.getLogger(__name__)


class ExposureMode(Enum):
    DURATION = 1
    COUNT = 2
    AREA_COUNT = 3
    SOURCE = 4


class EventRenderer(object):
    def __init__(self, full_scale_count=3, output_path=None, dvs_vid=None, preview=False,
                 exposure_mode=ExposureMode.DURATION, exposure_value=1 / 300.0, area_dimension=None,
                 frame_times_suffix='-frame_times.txt', avi_frame_rate=30, device="cuda:0"):
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

    def cleanup(self):
        if self.video_output_file is not None:
            self.video_output_file.release()
            self.video_output_file = None
        if self.frame_times_output_file is not None:
            self.frame_times_output_file.close()
            self.frame_times_output_file = None

    def _check_outputs_open(self):
        """renderer.py:141-170, through the reference's own writer when it imports."""
        if self.video_output_file is not None or not (self.output_path and type(self.video_output_file_name) is str):
            return
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

    # -- which rows go to which frame (renderer.py:272-330), on the timestamps only ------------------------------
    def _slices(self, ts):
        """ts: float32 device tensor [n], non-decreasing. Returns (starts, ends, t_frame) lists, one entry per FINISHED
        frame of this packet, with the reference's end-of-packet rule."""
        n = ts.shape[0]
        mode = self.exposure_mode
        starts, ends, tmid = [], [], []
        if mode == ExposureMode.SOURCE:
            starts, ends = [0], [n - 1]                     # end >= n - 1 -> end = n - 1; the frame is still emitted
            return starts, ends, [None]
        if mode == ExposureMode.COUNT:
            idx = 0
            while True:
                s, e = idx, idx + self.event_count
                if e >= n - 1:
                    break                                   # the rest stays in the (dropped) current frame
                starts.append(s); ends.append(e); tmid.append((s, e))
                idx = e
            return starts, ends, tmid
        # DURATION: frame k covers [cur_k, cur_k + interval]; cur accumulates in the dtype numpy gives it (the first
        # timestamp is a float32 scalar, renderer.py:205)
        t0, t1 = ts[0].item(), ts[-1].item()
        if self.currentFrameStartTime is None:
            self.currentFrameStartTime = np.float32(t0)
        cur = self.currentFrameStartTime
        curs = [cur]
        while float(curs[-1]) <= t1:
            if len(curs) >= 1 << 20:
                raise ValueError("a DURATION packet may span at most 2^20 frame intervals of %g s; this one runs from "
                                 "%r s to %r s: pass it in shorter packets" % (self.frameIntevalS, float(cur), t1))
            curs.append(curs[-1] + self.frameIntevalS)
        c = torch.tensor(np.asarray(curs, dtype=np.float64), device=ts.device)
        tsd = ts.double()
        left = torch.searchsorted(tsd, c, right=False).tolist()
        right = torch.searchsorted(tsd, c, right=True).tolist()
        k = 0
        while True:
            s, e = left[k], right[k + 1] if k + 1 < len(curs) else n
            if e >= n - 1:
                break
            starts.append(s); ends.append(e)
            self.currentFrameStartTime = curs[k + 1]
            tmid.append(curs[k + 1] + self.frameIntevalS / 2)
            k += 1
        return starts, ends, tmid

    def _area_slices(self, ev, height, width):
        """ExposureMode.AREA_COUNT (renderer.py:213-217, 246-261, 287-291): a frame ends when a cell of
        area_dimension^2 pixels has collected area_count events; the cell counters persist between packets."""
        n = ev.shape[0]
        if self.area_counts is None:
            self._cells = (1 + width // self.area_dimension, 1 + height // self.area_dimension)
            self.area_counts = torch.zeros(self._cells, dtype=torch.int32, device=self.device)
        # every frame but the first advances at least area_count - 1 events: the event that closes a frame is counted
        # again as the first of the next one
        cap = n // (self.area_count - 1) + 2
        st_t = torch.empty((cap,), dtype=torch.int64, device=self.device)
        en_t = torch.empty((cap,), dtype=torch.int64, device=self.device)
        nf = torch.zeros((1,), dtype=torch.int32, device=self.device)
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        with torch.cuda.device(self.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self._lib.v2e_render_area_scan(p(ev), n, int(self.area_dimension), int(self.area_count),
                                                      self._cells[0], self._cells[1], p(self.area_counts), p(st_t), p(en_t),
                                                      cap, p(nf), stream))
        k = int(nf.item())
        if k < 0:
            raise RuntimeError("area-count scan: more frames than its slice table holds")
        starts, ends = st_t[:k].tolist(), en_t[:k].tolist()
        return starts, ends, list(zip(starts, ends)), st_t[:k].contiguous(), en_t[:k].contiguous()

    def render_events_to_frames(self, event_arr, height, width, return_frames=False, return_device=False):
        """renderer.py:161: float64 frames [k, height, width] in 0..1 for the frames this packet finished, or None."""
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
        if self.exposure_mode == ExposureMode.AREA_COUNT:
            starts, ends, tinfo, st_t, en_t = self._area_slices(ev, height, width)
        else:
            starts, ends, tinfo = self._slices(ev[:, 0].contiguous())
            st_t = en_t = None
        k = len(starts)
        if k == 0:
            return None
        if st_t is None:
            st_t = torch.tensor(starts, dtype=torch.int64, device=self.device)
            en_t = torch.tensor(ends, dtype=torch.int64, device=self.device)
        acc = torch.empty((k, height, width), dtype=torch.int32, device=self.device)
        want_u8 = self.video_output_file is not None
        img = torch.empty((k, height, width), dtype=torch.float64, device=self.device) if (return_frames or return_device) else None
        u8 = torch.empty((k, height, width), dtype=torch.uint8, device=self.device) if want_u8 else None
        p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
        with torch.cuda.device(self.device):
            stream = ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self._lib.v2e_render_frames(p(ev), p(st_t), p(en_t), k, max(max(e - s for s, e in zip(starts, ends)), 0),
                                                   int(height), int(width), int(self.full_scale_count), p(acc), p(img),
                                                   p(u8), stream))
        if want_u8:
            import cv2
            host = u8.cpu().numpy()
            ts_host = ev[:, 0].cpu().numpy()
            for f in range(k):
                self.video_output_file.write(cv2.cvtColor(host[f], cv2.COLOR_GRAY2BGR))
                if self.exposure_mode == ExposureMode.SOURCE:
                    t = ts_host[0]
                elif self.exposure_mode in (ExposureMode.COUNT, ExposureMode.AREA_COUNT):
                    t = (ts_host[starts[f]] + ts_host[ends[f]]) / 2
                else:
                    t = tinfo[f]
                self.frame_times_output_file.write('{}\t{:10.6f}\n'.format(self.numFramesWritten, t))
                self.numFramesWritten += 1
        if return_device:
            return img
        return img.cpu().numpy() if return_frames else None
