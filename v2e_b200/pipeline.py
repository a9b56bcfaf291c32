"""Stage 2 + stage 3 of v2e.py (v2e.py:741-846) without the temp folders: source frames ->
SuperSloMo up-sampling -> DVS events, everything device-resident.

The reference hands frames from SloMo to the emulator as 8-bit PNG files in a temp dir
(slomo.py:440-444 -> v2e.py:832 read_image); here the uint8 frames stay in HBM. Times follow
v2e.py:794-797: interpTimes (units of source-frame intervals) scaled to the clip's duration.
Without an upsampler (V2EPipeline(None, emulator): --disable_slomo, or a timestamp resolution that needs no
upsampling) the source frames go to the pixel model themselves, at interpTimes = range(n) (v2e.py:776-797);
run_synthetic runs v2e.py's --synthetic_input loop (v2e.py:580-607).
"""
import logging

import numpy as np
import torch

from .emulator import EventEmulator, _replay_noise
from .slomo import SuperSloMo, batch_times, clip_span

logger = logging.getLogger(__name__)

# Source frame pairs per segment of V2EPipeline.run_segments. Each segment adds one event read-back and one finiteness
# check (two stream synchronisations) to the SloMo work of its pairs; at 64 pairs that is ~640 interpolated frames at
# U = 10, enough to hide them at small frame sizes too. At 1280x720, U = 10 and 0.11 events/px/frame a segment of 64
# pairs adds ~3 GB of device memory (its frames, and an event buffer grown to twice what overflowed it), and
# bench_stream.py measures the same time per frame at 16, 64 and 256 pairs as one run.
DEFAULT_SEGMENT_PAIRS = 64

# Source frames per segment without an upsampler (V2EPipeline(None, ...).run_segments, run_synthetic): the interpolated
# frames of a DEFAULT_SEGMENT_PAIRS segment at U = 10, so that a segment holds as many frames on the device (and as
# large an event buffer) as in the SloMo mode.
DEFAULT_SEGMENT_FRAMES = 10 * DEFAULT_SEGMENT_PAIRS

# v2e.py's --batch_size default: the frames per rendered DVS packet when no upsampler sets it
DEFAULT_BATCH_SIZE = 8


def segment_plan(n_frames, batch_size, segment_pairs=None, world=1, auto_upsample=False, upsampler=True):
    """The segments V2EPipeline.run_segments runs a clip of n_frames source frames in, as pair ranges [(p0, p1)]:
    segment k interpolates pairs p0 .. p1-1 from source frames p0 .. p1, so consecutive segments share one source
    frame. segment_pairs (default DEFAULT_SEGMENT_PAIRS) is rounded up to a multiple of batch_size, which puts every
    boundary on a SloMo batch boundary of the clip; the last segment takes the pairs that are left.

    world > 1: the segments of V2EPipeline.run_segments_sharded over `world` ranks, each one that run_clip_sharded
    accepts: at least `world` pairs, or with auto_upsample (whose batches are dealt to the ranks whole) at least
    `world` batches. segment_pairs is raised to that minimum before it is rounded, a shorter last segment is folded
    into the one before it, and a clip shorter than one segment raises ValueError. world=1 gives the plan above.

    upsampler=False: the segments of a clip that runs without an upsampler, as frame ranges [(a, b)]: segment k runs
    source frames a .. b-1, so segments share no frame. segment_pairs counts frames (default DEFAULT_SEGMENT_FRAMES)
    and is not rounded; each segment holds at least `world` frames. batch_size and auto_upsample are not used. A clip
    still needs two frames: v2e.py divides its duration by n_frames - 1."""
    n_frames, world = int(n_frames), int(world)
    if n_frames < 2:
        raise ValueError("n_frames=%d: a clip needs at least two source frames" % n_frames)
    if world < 1:
        raise ValueError("world=%d: a clip needs at least one rank" % world)
    what = "frame pair" if upsampler else "frame"
    sp = (DEFAULT_SEGMENT_PAIRS if upsampler else DEFAULT_SEGMENT_FRAMES) if segment_pairs is None else int(segment_pairs)
    if sp < 1:
        raise ValueError("segment_pairs=%d: a segment needs at least one %s" % (sp, what))
    auto_upsample = auto_upsample and upsampler
    bs = max(1, int(batch_size)) if upsampler else 1
    unit = bs if auto_upsample else 1                    # pairs per share a rank must get at least one of
    sp = -(-max(sp, world * unit) // bs) * bs
    n_units = n_frames - 1 if upsampler else n_frames
    plan = [(p0, min(p0 + sp, n_units)) for p0 in range(0, n_units, sp)]
    p0, p1 = plan[-1]
    if -(-(p1 - p0) // unit) < world:
        if len(plan) == 1:
            raise ValueError("fewer batches of frame pairs than ranks" if auto_upsample else
                             "fewer %ss than ranks" % what)
        plan[-2:] = [(plan[-2][0], p1)]
    return plan


def sharded_times(n_pairs, batch_size, pairs, ups):
    """interpTimes of pairs p0 .. p1-1 (p0 on a SloMo batch boundary) of a clip of n_pairs frame pairs sharded over
    ranks: these elements of the times run_clip_sharded builds for the whole clip, bit for bit. ups: the fixed U (an
    int: np.arange(n_pairs * U) * (1 / U), slomo.py:391-395 for the whole clip), or the list of U's of the batches in
    [p0, p1) (auto_upsample: each batch's batch_times, as slomo.clip_times concatenates them)."""
    p0, p1 = pairs
    if isinstance(ups, (int, np.integer)):
        U = int(ups)
        return np.arange(p0 * U, p1 * U) * (1.0 / U)
    bs = max(1, min(int(batch_size), n_pairs))
    starts = range(p0, p1, bs)
    if len(ups) != len(starts):
        raise ValueError("%d U's for %d batches" % (len(ups), len(starts)))
    return np.concatenate([batch_times(a, min(bs, n_pairs - a), int(U)) for a, U in zip(starts, ups)])


def sharded_span(n_pairs, batch_size, last_U, auto_upsample):
    """max - min of the times run_clip_sharded builds for a clip of n_pairs frame pairs whose last batch gets last_U
    (the fixed U without auto_upsample): the denominator of v2e.py:794-797, the same double."""
    if auto_upsample:
        return clip_span(n_pairs, batch_size, last_U)
    return (n_pairs * int(last_U) - 1) * (1.0 / int(last_U)) - 0.0


def _describe(x):
    if isinstance(x, (np.ndarray, torch.Tensor)):
        return "%s %s %s" % (type(x).__name__, str(x.dtype).replace("torch.", ""), list(x.shape))
    return type(x).__name__


class V2EPipeline:
    def __init__(self, slomo: SuperSloMo, emulator: EventEmulator, renderer=None, batch_size=None):
        """slomo: the upsampler, or None to run without one, as v2e.py does with --disable_slomo or when the timestamp
        resolution needs no upsampling (v2e.py:414-422, 470-478): the source frames themselves then go to the pixel
        model, frame i at t_offset + i * src_duration_s / (n_frames - 1) (v2e.py:776-797), and no upsampler video is
        written.

        renderer (optional): a v2e_b200.renderer.EventRenderer the runs feed with every segment's rows, in the packets
        v2e.py's stage-3 loop renders (batch_size frames per packet, v2e.py:826-846), so that it writes the DVS
        video and its frame-times file as v2e.py does. The caller owns it and calls its cleanup() after the clip.

        batch_size: v2e.py's --batch_size, the frames per rendered packet. With slomo it is slomo.batch_size, and any
        other value raises ValueError; without, it defaults to DEFAULT_BATCH_SIZE (v2e's default)."""
        if slomo is not None:
            if batch_size is not None and batch_size != slomo.batch_size:
                raise ValueError("batch_size=%r differs from slomo.batch_size=%r: v2e.py renders packets of the "
                                 "upsampler's batch size" % (batch_size, slomo.batch_size))
        elif int(DEFAULT_BATCH_SIZE if batch_size is None else batch_size) < 1:
            raise ValueError("batch_size=%r: a packet needs at least one frame" % (batch_size,))
        self.slomo = slomo
        self.emulator = emulator
        self.renderer = renderer
        self._batch_size = None if slomo is not None else int(DEFAULT_BATCH_SIZE if batch_size is None else batch_size)

    @property
    def batch_size(self):
        """The frames per rendered DVS packet: slomo.batch_size, or the constructor's batch_size without an upsampler."""
        return self.slomo.batch_size if self.slomo is not None else self._batch_size

    def run(self, frames_u8, src_duration_s, t_offset=0.0, return_device=False, copy=False):
        """frames_u8: [N,H,W] uint8 source frames covering `src_duration_s` seconds.
        Returns (events [M,4] float32, frame offsets, interp_times_s, n_interp_frames). Host rows are a
        view of the emulator's pinned staging buffer unless copy=True (valid until the next call).
        The clip is run_segments' single segment."""
        if isinstance(frames_u8, np.ndarray):
            frames_u8 = torch.from_numpy(np.ascontiguousarray(frames_u8))
        n = frames_u8.shape[0]
        (res,) = self.run_segments(lambda a, b: frames_u8[a:b], n, src_duration_s, t_offset,
                                   segment_pairs=max(n - 1, 1) if self.slomo is not None else max(n, 1),
                                   return_device=return_device, copy=copy)
        return res

    def run_segments(self, get_frames, n_frames, src_duration_s, t_offset=0.0, segment_pairs=None,
                     return_device=False, copy=False):
        """Runs a clip of any length segment by segment: a generator that yields, per segment,
        (events [M,4] float32, frame offsets [T+1], interp_times_s [T], n_interp_frames T) -- what run returns, for
        that segment's interpolated frames only (offsets start at 0 in every segment). Concatenated, the segments are
        what one run(all frames, src_duration_s, t_offset) returns on a fresh pipeline: the same frames, times,
        rows, offsets and emulator counters, and the same vid_orig / vid_slomo videos and event files.

        get_frames(a, b) returns source frames a .. b-1 as uint8 [b-a, H, W], an ndarray or a tensor, on the host or
        the device (for an array: lambda a, b: frames[a:b]; raw BGR video goes through InputPrep inside it).
        n_frames >= 2 is the clip's source frame count, src_duration_s its duration.

        segment_pairs: source frame pairs per segment, rounded up to a multiple of slomo.batch_size so that segments
        start on the clip's SloMo batch boundaries (segment_plan). Default DEFAULT_SEGMENT_PAIRS: ~3 GB of device
        memory per segment at 1280x720, U = 10, and as fast per frame as one run. Consecutive segments share one
        source frame: the last of segment k is the first of segment k+1.

        Device and pinned-host memory depend on the segment length, not the clip length: one segment's source and
        interpolated frames are held at a time, and the emulator's event buffers grow to the largest segment. The
        rows are valid until the next iteration (return_device=True: a view of the emulator's device buffer; host
        rows with copy=False: a view of its pinned staging buffer); copy=True returns host rows the caller owns.

        Times: the scale f = src_duration_s / (max - min of the clip's interpTimes) (v2e.py:794-797) depends on the U
        of the clip's last batch and enters every frame interval of the pixel model, so it is known before the first
        segment. With a fixed U it follows from the shapes; with auto_upsample and more than one segment, the flow
        network first runs on the clip's last batch (fetched through get_frames) to pick its U. A single segment
        takes f from its own times, as run does.

        With a renderer, each segment's rows go from the emulator's device buffer to renderer.render_frame_rows before
        the segment is yielded, frame i counted from the clip's first interpolated frame; the packet that straddles a
        segment boundary is held by the renderer, and the clip's last segment renders the leftover packet.

        Without an upsampler (slomo None) the segments are disjoint runs of source frames: segment_pairs counts frames
        (default DEFAULT_SEGMENT_FRAMES, the interpolated frames of a default SloMo segment at U = 10, so as much device
        memory per segment), each segment's frames go to generate_events_batch as they are, and frame i gets the time
        t_offset + f * i with f = src_duration_s / (n_frames - 1) in float64, v2e.py:794-797 over interpTimes =
        range(n_frames). The yields have the same form, n_interp_frames being the segment's frame count. Frames
        get_frames returns on the device are read in place; host frames go up in one copy per segment.

        Raises ValueError, naming the segment, when get_frames returns anything but uint8 [b-a, H, W] with the first
        segment's H, W; RuntimeError, before any work, where generate_events_batch refuses the emulator (replay mode
        with per-frame noise, a sharded emulator: run_clip_sharded takes a clip over ranks)."""
        sl, em = self.slomo, self.emulator
        em.check_batch_path()
        n = int(n_frames)
        if sl is None:
            plan = segment_plan(n, 1, segment_pairs, upsampler=False)
        else:
            plan = segment_plan(n, sl.batch_size, segment_pairs)
        m = len(plan)
        size = []

        def fetch(a, b, k):
            fr = get_frames(a, b)
            if isinstance(fr, np.ndarray):
                fr = torch.from_numpy(np.ascontiguousarray(fr))
            ok = (isinstance(fr, torch.Tensor) and fr.dtype == torch.uint8 and fr.dim() == 3 and fr.shape[0] == b - a
                  and (not size or tuple(fr.shape[1:]) == size[0]))
            if not ok:
                want = "[%d, %d, %d]" % ((b - a,) + size[0]) if size else "[%d, H, W]" % (b - a)
                raise ValueError("segment %d of %d: get_frames(%d, %d) returned %s, expected uint8 %s"
                                 % (k, m, a, b, _describe(fr), want))
            size[:] = [tuple(fr.shape[1:])]
            return fr

        f = u_last = None
        if sl is None:
            f = src_duration_s / np.int64(n - 1)              # v2e.py:794-797 over interpTimes = range(n)
        elif m > 1:
            if sl.auto_upsample:
                bs = max(1, min(int(sl.batch_size), n - 1))
                a = (n - 2) // bs * bs
                u_last = sl.batch_upsampling(fetch(a, n, m - 1), n)
            else:
                u_last = int(sl.upsampling_factor)
            f = src_duration_s / clip_span(n - 1, sl.batch_size, u_last)

        def segment(k):
            nonlocal f
            p0, p1 = plan[k]
            if sl is None:
                return fetch(p0, p1, k), t_offset + f * np.arange(p0, p1), k == m - 1
            fr = fetch(p0, p1 + 1, k)
            interp, times, _, ups = sl.interpolate_frames(fr, return_ups=True, first_pair=p0, clip_frames=n)
            del fr
            if f is None:
                f = src_duration_s / (np.max(times) - np.min(times))          # v2e.py:794-797
            elif k == m - 1 and ups[-1] != u_last:
                raise RuntimeError("the clip's last batch got U=%d, its time-scale pre-pass U=%d" % (ups[-1], u_last))
            return interp, t_offset + f * times, k == m - 1
        yield from self._emulate(segment, 0, return_device, copy)

    def run_synthetic(self, source, segment_frames=None, t_offset=0.0, return_device=False, copy=False):
        """v2e.py's --synthetic_input loop (v2e.py:580-607) segment by segment: a generator that yields, per segment,
        (events [M,4] float32, frame offsets [T+1], times_s [T], T), as run_segments does.

        source: a v2ecore.base_synthetic_input, or anything with its next_frame() -> (frame [H, W] or None at the end,
        time in seconds). Frames may be uint8, float32 or float64 (log_input / HDR frames), ndarrays or tensors, every
        one of the first frame's shape and dtype; other numeric dtypes are read as float64. Each frame gets the
        source's own time plus t_offset. Up to segment_frames frames (default DEFAULT_SEGMENT_FRAMES) are pulled per
        segment and copied as they arrive (a source may reuse its frame array), into a buffer of pinned host memory
        (for host frames) that goes to the device in one copy, and run by one generate_events_batch call. The caller
        owns the source and calls its cleanup().

        With a renderer the rows are rendered in the synthetic loop's packets, which end one frame later than
        stage 3's: that loop counts frame i as i + 1 before its `% batch_size == 0` test, so the packet closes after
        frame i when (i + 1) % batch_size == 0 and frame i has rows, and the leftover rows are rendered at the end.

        Raises ValueError, naming the frame, for a frame of another shape or dtype than the first, or not [H, W];
        RuntimeError, before any work, where generate_events_batch refuses the emulator."""
        em = self.emulator
        em.check_batch_path()
        sf = DEFAULT_SEGMENT_FRAMES if segment_frames is None else int(segment_frames)
        if sf < 1:
            raise ValueError("segment_frames=%d: a segment needs at least one frame" % sf)
        dev = torch.device(em.device)
        nxt = source.next_frame()
        if nxt[0] is None:
            return
        want = []                                           # the first frame's (shape, dtype)
        stage = [None, None]                                # the segment buffer, the event its last upload records
        pulled = 0                                          # frames taken from the source so far

        def segment(k):
            nonlocal nxt, pulled
            buf, uploaded = stage
            if uploaded is not None:
                uploaded.synchronize()                      # the previous segment's frames have left the buffer
            fr, t = nxt
            times = []
            while fr is not None and len(times) < sf:
                x = torch.as_tensor(fr)
                if not want:
                    want[:] = [tuple(x.shape), x.dtype]
                if x.dim() != 2 or tuple(x.shape) != want[0] or x.dtype != want[1]:
                    raise ValueError("frame %d: next_frame() returned %s, expected [H, W] like frame 0 (%s %s)"
                                     % (pulled, _describe(fr), str(want[1]).replace("torch.", ""), list(want[0])))
                if buf is None:
                    dt = x.dtype if x.dtype in (torch.uint8, torch.float32, torch.float64) else torch.float64
                    pin = x.device.type == "cpu" and dev.type == "cuda"
                    buf = stage[0] = torch.empty((sf,) + want[0], dtype=dt, device=x.device, pin_memory=pin)
                buf[len(times)].copy_(x)
                times.append(float(t))
                pulled += 1
                fr, t = source.next_frame()
            nxt = (fr, t)
            frames = buf[:len(times)].to(dev, non_blocking=True)
            if buf.is_pinned():
                stage[1] = torch.cuda.Event()
                stage[1].record(torch.cuda.current_stream(dev))
            return frames, t_offset + np.asarray(times, np.float64), fr is None
        yield from self._emulate(segment, 1, return_device, copy)

    def _emulate(self, segment, first, return_device, copy):
        """The pixel model and the renderer over a clip's segments, what every single-GPU run yields: segment(k)
        returns segment k's frames [T, H, W], their times in seconds and whether it is the clip's last segment. first:
        the index the render loop gives the clip's first frame (v2e.py's stage-3 loop 0, its synthetic loop 1)."""
        em, rd = self.emulator, self.renderer
        k, last = 0, False
        while not last:
            fr, t, last = segment(k)
            em._sinks_continue = k > 0
            try:
                ev, offs = em.generate_events_batch(fr, t, return_device=return_device or rd is not None, copy=copy)
            finally:
                em._sinks_continue = False
            nf = fr.shape[0]
            del fr
            if rd is not None:
                rd.render_frame_rows(ev, offs, first, self.batch_size, end_of_clip=last,
                                     height=em.output_height, width=em.output_width)
                if not return_device:
                    ev = em._rows_to_host(ev.shape[0], copy=copy)
            first += nf
            k += 1
            yield ev, offs, t, nf

    def run_clip_sharded(self, frames_u8, src_duration_s, t_offset=0.0, group=None, return_labels=False,
                         write_sinks=False):
        """ONE clip over the ranks of `group` (BASELINE config 5 layout; SURVEY.md 8e). Every rank passes the
        same source frames; the emulator must have been built with shard=(rank, world, group).
          1. SloMo over this rank's frame pairs (parallel.pair_range) -- no halo, weights replicated. With
             auto_upsample the pairs are whole batches (parallel.batch_pair_range), each rank picks the U of its
             batches, and the ranks all-gather those U's to build the clip's times (slomo.clip_times);
          2. all-to-all of uint8 row bands (parallel.exchange_frame_bands);
          3. pixel model on this rank's rows of every frame (one all-reduce(MAX) of an int32 per frame).
        Returns (rows [M_r, 4] float32 host array of THIS rank's pixel rows (global y), interp_times_s,
        n_interp_frames), and with return_labels (needs label_signal_noise=True) the labels of those rows after them.
        Union over ranks = the events of the clip; parallel.gather_event_streams / merge_by_time assemble them where
        one stream is wanted. Every rank holds only its own frame pairs, so the upsampler writes no vid_orig /
        vid_slomo video here (rank 0 logs a warning when video_path is set).
        write_sinks=True (needs row_order) writes the clip's event files: every rank's rows, sort keys, frame offsets and
        shot counts are gathered on the group's first rank (parallel.gather_band_outputs), which merges the bands on the
        device into the one-GPU stream (parallel.merge_by_key_device) and passes it, with its labels, to its own
        emulator's write_events -- the files a single-GPU V2EPipeline.run writes -- and, when that rank's pipeline has a
        renderer, to the renderer: the DVS video and frame-times file of a single-GPU run. Only that rank's emulator may
        be built with sink keywords (dvs_text, dvs_aedat2, ...) and only its pipeline may hold a renderer; the others
        are built without, since they would open, and truncate, the same paths. The ranks check this together before
        any data moves and all raise ValueError when another rank holds sinks or a renderer. The return values are those
        of write_sinks=False. Without write_sinks no rank renders (rank 0 logs a warning when it holds a renderer).
        The clip is run_segments_sharded's single segment; a clip of any length streams through that."""
        if isinstance(frames_u8, np.ndarray):
            frames_u8 = torch.from_numpy(np.ascontiguousarray(frames_u8))
        n = frames_u8.shape[0]
        (res,) = self.run_segments_sharded(lambda a, b: frames_u8[a:b], n, src_duration_s, t_offset,
                                           segment_pairs=max(n - 1, 1) if self.slomo is not None else max(n, 1),
                                           group=group, return_labels=return_labels, write_sinks=write_sinks)
        return res

    def run_segments_sharded(self, get_frames, n_frames, src_duration_s, t_offset=0.0, segment_pairs=None, group=None,
                             return_labels=False, write_sinks=False):
        """ONE clip of any length over the ranks of `group`, segment by segment: a generator that yields, per segment,
        what run_clip_sharded returns for that segment's interpolated frames -- (rows [M_r, 4] float32 host array of
        this rank's rows (global y), interp_times_s, n_interp_frames), and the labels of the rows with return_labels.
        Concatenated, the segments are what one run_clip_sharded(all frames, src_duration_s, t_offset) returns on a
        fresh pipeline: every rank's rows (in the same order with row_order, the same multiset per frame without), the
        times, frame counts, labels and emulator counters, and with write_sinks the first rank's event files.

        Every rank calls it with the same arguments. get_frames(a, b) returns source frames a .. b-1 as uint8
        [b-a, H, W], an ndarray or a tensor, on the host or the device (run_segments' contract); a rank asks only for
        the frames its own pairs need. segment_pairs (default DEFAULT_SEGMENT_PAIRS per rank) is the segment length in
        source frame pairs of the whole group: segments start on the clip's SloMo batch boundaries and each holds at
        least `world` pairs, or with auto_upsample `world` batches (segment_plan(..., world, auto_upsample)).

        Per segment every rank interpolates its share of the segment's pairs (write_video=False), the row bands are
        exchanged (parallel.exchange_frame_bands) and the band emulator runs one generate_events_band_batch call, or
        frame by frame in replay mode with noise; its state carries over to the next segment. write_sinks: the first
        rank gathers, merges and writes each segment's bands. Device memory on a rank depends on the segment length,
        not the clip length.

        Times: the scale f of v2e.py:794-797 depends on the U of the clip's last batch. With a fixed U it follows from
        the shapes; with auto_upsample and more than one segment the last rank runs the flow network on the clip's last
        batch first (SuperSloMo.batch_upsampling) and broadcasts its U; the segment holding that batch raises
        RuntimeError on every rank when its U differs. A single segment takes f from its own times.

        Without an upsampler (slomo None) the segments are disjoint runs of source frames, segment_pairs counting
        frames (default DEFAULT_SEGMENT_FRAMES per rank, at least `world` per segment); each rank fetches its contiguous
        run of a segment's frames (parallel.pair_range over frames) and passes it to the band exchange; the times are
        run_segments' (t_offset + f * i, f = src_duration_s / (n_frames - 1)).

        Raises, on every rank and before any work, what run_clip_sharded raises: RuntimeError without a shard,
        ValueError for return_labels without label_signal_noise, write_sinks without row_order or with sinks on another
        rank than the first, and too short a clip. The frames a segment's get_frames calls return are checked by one
        all-gather before any frame moves: every rank raises ValueError naming the segment and the rank whose frames
        are not uint8 [b-a, H, W] with the clip's H, W."""
        import torch.distributed as dist
        from . import parallel
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        write_sinks = self._sharded_refusals(group, return_labels, write_sinks)
        if rank == 0 and self.renderer is not None and not write_sinks:
            logger.warning("renderer ignored: a clip sharded over ranks is rendered from the merged stream "
                           "write_sinks=True builds")
        sl, em = self.slomo, self.emulator
        n = int(n_frames)
        if sl is None:
            plan = segment_plan(n, 1, DEFAULT_SEGMENT_FRAMES * world if segment_pairs is None else segment_pairs,
                                world=world, upsampler=False)
            auto = False
        else:
            if n - 1 < world:
                raise ValueError("fewer frame pairs than ranks")
            auto = bool(sl.auto_upsample)
            bs = max(1, min(int(sl.batch_size), n - 1))
            if segment_pairs is None:
                segment_pairs = DEFAULT_SEGMENT_PAIRS * world
            plan = segment_plan(n, sl.batch_size, segment_pairs, world=world, auto_upsample=auto)
        m = len(plan)
        if rank == 0 and sl is not None and sl.writes_video():
            logger.warning("video_path ignored: a clip sharded over ranks writes no upsampler video")
        comm = em.device if dist.get_backend(group) == "nccl" else "cpu"
        size = []

        def fetch(a, b, k, mine=True):
            """get_frames(a, b) on this rank (when mine), checked on every rank by one all-gather of (ok, H, W)."""
            fr, ok, hw = None, 1, (-1, -1)
            if mine:
                fr = get_frames(a, b)
                if isinstance(fr, np.ndarray):
                    fr = torch.from_numpy(np.ascontiguousarray(fr))
                ok = int(isinstance(fr, torch.Tensor) and fr.dtype == torch.uint8 and fr.dim() == 3
                         and fr.shape[0] == b - a)
                if ok:
                    hw = tuple(fr.shape[1:])
            v = torch.tensor([ok, hw[0], hw[1], a, b], dtype=torch.int64, device=comm)
            vs = [torch.empty_like(v) for _ in range(world)]
            dist.all_gather(vs, v, group=group)
            vs = [x.tolist() for x in vs]
            if not size:
                size[:] = [tuple(x[1:3]) for x in vs if x[0] and x[1] >= 0][:1]
            bad = [r for r, x in enumerate(vs) if not x[0] or (x[1] >= 0 and tuple(x[1:3]) != size[0])]
            if bad:
                r = bad[0]
                want = "[%d, %d, %d]" % ((vs[r][4] - vs[r][3],) + size[0]) if size else "[%d, H, W]" % (vs[r][4] - vs[r][3])
                got = "" if r != rank else ": it returned %s" % _describe(fr)
                raise ValueError("segment %d of %d: rank %d's get_frames(%d, %d) did not return uint8 %s%s"
                                 % (k, m, r, vs[r][3], vs[r][4], want, got))
            return fr

        f = u_last = None
        first = 0                                           # the clip's index of the segment's first interpolated frame
        if sl is None:
            f = src_duration_s / np.int64(n - 1)              # v2e.py:794-797 over interpTimes = range(n)
        elif m > 1:
            if auto:
                a = (n - 2) // bs * bs
                fr = fetch(a, n, m - 1, mine=rank == world - 1)
                u = torch.tensor([0 if fr is None else sl.batch_upsampling(fr, n)], dtype=torch.int64, device=comm)
                del fr
                dist.broadcast(u, group=group, group_src=world - 1)
                u_last = int(u.item())
            else:
                u_last = int(sl.upsampling_factor)
            f = src_duration_s / sharded_span(n - 1, sl.batch_size, u_last, auto)
        for k, (s0, s1) in enumerate(plan):
            if auto:
                p0, p1 = parallel.batch_pair_range(s1 - s0, bs, rank, world)
            else:
                p0, p1 = parallel.pair_range(s1 - s0, rank, world)      # without an upsampler: frames
            p0, p1 = p0 + s0, p1 + s0
            fr = fetch(p0, p1 if sl is None else p1 + 1, k)
            H = size[0][0]
            if sl is None:
                local, times = fr.to(em.device, non_blocking=True), np.arange(s0, s1)
            elif auto:
                local, _, _, ups_l = sl.interpolate_frames(fr, return_ups=True, write_video=False, first_pair=p0,
                                                           clip_frames=n)
                # every rank's per-batch U's (a few ints; each rank knows how many batches every rank holds)
                nb = [-(-(b - a) // bs) for a, b in (parallel.batch_pair_range(s1 - s0, bs, r, world)
                                                     for r in range(world))]
                send = torch.zeros(max(nb), dtype=torch.int64, device=local.device)
                send[:len(ups_l)] = torch.tensor(ups_l, dtype=torch.int64)
                recv = [torch.empty_like(send) for _ in range(world)]
                dist.all_gather(recv, send, group=group)
                ups = [u for r in range(world) for u in recv[r][:nb[r]].tolist()]
                times = sharded_times(n - 1, bs, (s0, s1), ups)
                if k == m - 1 and u_last is not None and ups[-1] != u_last:
                    raise RuntimeError("the clip's last batch got U=%d, its time-scale pre-pass U=%d"
                                       % (ups[-1], u_last))
            else:
                local, times_l, _ = sl.interpolate_frames(fr, write_video=False)
                U = int(sl.upsampling_factor)
                times = sharded_times(n - 1, bs, (s0, s1), U)
                assert np.allclose(times_l + p0, times[(p0 - s0) * U:(p1 - s0) * U])
            del fr
            if f is None:
                f = src_duration_s / (np.max(times) - np.min(times))        # v2e.py:794-797
            t = t_offset + f * times
            bands = parallel.exchange_frame_bands(local, H, group=group, halo=em.cs_halo_rows(H))
            del local
            res = self._band_events(bands, t, H, (k > 0, k == m - 1, first), group, return_labels, write_sinks)
            first += bands.shape[0]
            del bands
            yield res

    def _sharded_refusals(self, group, return_labels, write_sinks):
        """run_clip_sharded's refusals, raised on every rank together. Returns whether the group's first rank merges the
        bands: write_sinks and it writes event files or renders the DVS video."""
        import torch.distributed as dist
        world = dist.get_world_size(group)
        em = self.emulator
        if em.shard is None:
            raise RuntimeError("run_clip_sharded needs EventEmulator(shard=(rank, world, group))")
        if return_labels and not em.label_signal_noise:
            raise ValueError("return_labels=True needs label_signal_noise=True")
        if not write_sinks:
            return False
        if em.row_order is None:
            raise ValueError("write_sinks=True needs EventEmulator(row_order='canonical' or 'shuffled'): the bands "
                             "are merged by their sort keys")
        # every rank learns who holds sinks (bit 0) or a renderer (bit 1), so that all of them raise (none waits in a
        # collective)
        nccl = dist.get_backend(group) == "nccl"
        flag = torch.tensor([(em._sinks is not None) | (self.renderer is not None) << 1], dtype=torch.int64,
                            device=em.device if nccl else "cpu")
        flags = [torch.zeros_like(flag) for _ in range(world)]
        dist.all_gather(flags, flag, group=group)
        flags = [int(f.item()) for f in flags]
        bad = [r for r in range(1, world) if flags[r] & 1]
        if bad:
            raise ValueError("write_sinks=True: only the group's first rank may hold sinks, ranks %s do; build "
                             "their emulators without dvs_* keywords" % bad)
        bad = [r for r in range(1, world) if flags[r] & 2]
        if bad:
            raise ValueError("write_sinks=True: only the group's first rank may hold a renderer, ranks %s do; build "
                             "their pipelines without one" % bad)
        return bool(flags[0])

    def _band_events(self, bands, t, H, seg, group, return_labels, write_sinks):
        """The pixel model on this rank's bands of one segment's frames: what run_segments_sharded yields. seg: (the
        segment is not the clip's first (the sinks continue the AEDAT-2.0 rule across segments), it is the clip's last,
        the clip's index of its first frame)."""
        cont = seg[0]
        em = self.emulator
        extra = dict(return_labels=True) if return_labels else {}
        if not _replay_noise(em):
            # chunks of frames through the multi-frame kernels: one all-reduce(MAX) of the frame maxima per chunk
            # (frame by frame -- one all-reduce each -- for a chunk the refractory filter touches, for the
            # centre-surround model, whose Euler iteration exchanges halo rows, and for SCIDVS / photoreceptor noise)
            if not write_sinks:
                res = em.generate_events_band_batch(bands, t, H, **extra)
                return (res[0], t, bands.shape[0]) + tuple(res[2:])
            rows, offs, *labels, keys = em.generate_events_band_batch(bands, t, H, return_device=True,
                                                                      return_keys=True, **extra)
            em._sinks_continue = cont
            try:
                self._write_merged(rows, keys, offs, group, seg, H, bands.shape[-1])
            finally:
                em._sinks_continue = False
            labels = [labels[0].cpu().numpy().astype(bool)] if labels else []
            return (rows.cpu().numpy(), t, bands.shape[0]) + tuple(labels)
        assert not write_sinks, "row_order needs rng_mode='device', which takes the batched path"
        out, labs = [], []
        for k in range(bands.shape[0]):
            ev = em.generate_events_band(bands[k], t[k], H)
            if ev is not None:
                out.append(ev)
                labs.append(em.last_signnoise_label)
        rows = np.concatenate(out, 0) if out else np.zeros((0, 4), np.float32)
        if return_labels:
            return rows, t, bands.shape[0], (np.concatenate(labs) if labs else np.zeros((0,), bool))
        return rows, t, bands.shape[0]

    def _write_merged(self, rows, keys, offs, group, seg, H, W):
        """write_sinks: the bands of every rank to the group's first rank, merged there and written to its sinks and
        rendered by its renderer (seg: see _band_events; H, W: the frame size)."""
        from . import parallel
        from .sinks import signnoise_labels
        em = self.emulator
        g = parallel.gather_band_outputs(rows, keys, offs, em.last_n_shot, dst=0, group=group)
        if g is None:
            return
        streams, ks, os_, ss = g
        merged, moffs = parallel.merge_by_key_device(streams, ks, os_, ss, device=em.device)
        labels = signnoise_labels(moffs, np.sum(ss, axis=0), em.device) if em.label_signal_noise else None
        em.write_events(merged, labels)
        if self.renderer is not None:
            self.renderer.render_frame_rows(merged, moffs, seg[2], self.batch_size, end_of_clip=seg[1],
                                            height=H, width=W)
