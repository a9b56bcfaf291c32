"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the reference's EventRenderer.render_events_to_frames
(v2ecore/renderer.py:161-390, accumulate_event_frame :392-430, hist2d_numba_seq v2ecore/v2e_utils.py:474-486), with
its quirks kept, because a drop-in must return the same frames:
  * the frame being filled is dropped at the start of every call (`self.currentFrame = None`, :270);
  * the last event of a packet is never rendered (`end = numEvents - 1`, :300-303; slices are end-exclusive);
  * DURATION: boundaries by searchsorted(ts, frame start, 'left') / (ts, next start, 'right') over the whole packet;
  * a finished frame is clip(hist_on - hist_off, +-full_scale_count), returned as (frame + fs) / (2 fs) in float64.
AREA_COUNT (a sequential, data-dependent scan, renderer.py:246-261) is restated too.

Besides the frames, the oracle keeps what the reference writes when a DVS video is open (renderer.py:337-354): the
frame handed to the video writer, (img * 255) as uint8 repeated into 3 BGR channels (`video_frames`), and the time of
every frame in the frame-times file (`times`, formatted by `frame_times_text`). Those times are numpy scalars of the
dtype the reference computes them in (float32 for float32 events).
Pinned by tests/test_render.py and tests/test_render_packets.py against tests/golden/render_ref.npz
(oracle/make_golden_render.py ran the unmodified class and recorded its video writer and frame-times file).
"""
import numpy as np

DURATION, COUNT, AREA_COUNT, SOURCE = 1, 2, 3, 4


def video_frames(frames, H, W):
    """The uint8 BGR frames the reference hands its video writer for float64 frames [k, H, W] (None: no frames)."""
    if frames is None:
        return np.zeros((0, H, W, 3), np.uint8)
    return np.repeat((frames * 255).astype(np.uint8)[..., None], 3, axis=3)


def frame_times_text(dvs_vid, times):
    """The whole frame-times file for a video named dvs_vid (renderer.py:157-159, 352-353)."""
    head = '# frame times for {}\n# frame# time(s)\n'.format(dvs_vid)
    return head + ''.join('{}\t{:10.6f}\n'.format(i, t) for i, t in enumerate(times))


class RenderOracle:
    def __init__(self, full_scale_count=3, exposure_mode=DURATION, exposure_value=1 / 300.0, area_dimension=None):
        self.mode, self.value, self.fs = exposure_mode, exposure_value, full_scale_count
        self.area_dimension = area_dimension
        self.interval = 1 / (1 / exposure_value) if exposure_mode == DURATION else None      # renderer.py:92-93
        self.cur_start = None
        self.area_counts = None
        self.times = []                 # time of every frame finished so far, as the frame-times file states it
        self.slices = []                # (start, end) rows of the packet rendered into each of those frames

    def _frame(self, ev, H, W):
        """hist2d_numba_seq of the ON rows minus that of the OFF rows: bin int(y), int(x) for 0 <= y < H, 0 <= x < W
        (its delta is 1 / ((H - 0) / H) = 1 exactly); every row whose p is not 1 is OFF."""
        y, x = ev[:, 2].astype(np.float64), ev[:, 1].astype(np.float64)
        keep = (y >= 0) & (y < H) & (x >= 0) & (x < W)
        pix = y[keep].astype(np.int64) * W + x[keep].astype(np.int64)
        on = ev[keep, 3] == 1
        hist = lambda m: np.bincount(pix[m], minlength=H * W).astype(np.float64).reshape(H, W)
        return np.clip(hist(on) - hist(~on), -self.fs, self.fs)

    def _area_scan(self, cells, start):
        """compute_area_counts (renderer.py:254-267) on cells = [(x cell, y cell)] of the packet's rows."""
        counts, a = self.area_counts, int(self.value)
        e = start
        for e in range(start, len(cells)):
            x, y = cells[e]
            c = 1 + counts[x][y]
            counts[x][y] = c
            if c >= a:
                for col in counts:
                    col[:] = [0] * len(col)
                break
        return e

    def render(self, ev, H, W):
        if ev is None or ev.shape[0] == 0:
            return None
        ts = ev[:, 0]
        n = len(ts)
        if self.mode == DURATION:
            if self.cur_start is None:
                self.cur_start = ts[0]
            nxt = self.cur_start + self.interval
        if self.mode == AREA_COUNT:
            if self.area_counts is None:
                self.area_counts = [[0] * (1 + H // self.area_dimension) for _ in range(1 + W // self.area_dimension)]
            d = self.area_dimension
            cells = list(zip((ev[:, 1] // d).astype(np.int64).tolist(), (ev[:, 2] // d).astype(np.int64).tolist()))
        out, idx, done = [], 0, False
        while not done:
            if self.mode == DURATION:
                start = int(np.searchsorted(ts[idx:], self.cur_start, side="left"))
                end = int(np.searchsorted(ts[idx:], nxt, side="right"))
            elif self.mode == COUNT:
                start, end = idx, idx + int(self.value)
            elif self.mode == AREA_COUNT:
                start = idx
                end = self._area_scan(cells, start)
            else:
                start, end = 0, n
            if end >= n - 1:
                done, end = True, n - 1
            frame = self._frame(ev[start:end], H, W)
            if not done or self.mode == SOURCE:
                if self.mode == DURATION:
                    self.cur_start += self.interval
                    nxt = self.cur_start + self.interval
                    self.times.append(self.cur_start + self.interval / 2)
                elif self.mode in (COUNT, AREA_COUNT):
                    idx = end
                    self.times.append((ts[start] + ts[end]) / 2)
                else:
                    self.times.append(ts[0])
                self.slices.append((start, end))
                out.append((frame + self.fs) / float(self.fs * 2))
        return np.stack(out) if out else None
