"""Stage 2 + stage 3 of v2e.py (v2e.py:741-846) without the temp folders: source frames ->
SuperSloMo up-sampling -> DVS events, everything device-resident.

The reference hands frames from SloMo to the emulator as 8-bit PNG files in a temp dir
(slomo.py:440-444 -> v2e.py:832 read_image); here the uint8 frames stay in HBM. Times follow
v2e.py:794-797: interpTimes (units of source-frame intervals) scaled to the clip's duration.
"""
import logging

import numpy as np
import torch

from .emulator import EventEmulator
from .slomo import SuperSloMo, batch_times, clip_span

logger = logging.getLogger(__name__)

# Source frame pairs per segment of V2EPipeline.run_segments. Each segment adds one event read-back and one finiteness
# check (two stream synchronisations) to the SloMo work of its pairs; at 64 pairs that is ~640 interpolated frames at
# U = 10, enough to hide them at small frame sizes too. At 1280x720, U = 10 and 0.11 events/px/frame a segment of 64
# pairs adds ~3 GB of device memory (its frames, and an event buffer grown to twice what overflowed it), and
# bench_stream.py measures the same time per frame at 16, 64 and 256 pairs as one run.
DEFAULT_SEGMENT_PAIRS = 64


def segment_plan(n_frames, batch_size, segment_pairs=None, world=1, auto_upsample=False):
    """The segments V2EPipeline.run_segments runs a clip of n_frames source frames in, as pair ranges [(p0, p1)]:
    segment k interpolates pairs p0 .. p1-1 from source frames p0 .. p1, so consecutive segments share one source
    frame. segment_pairs (default DEFAULT_SEGMENT_PAIRS) is rounded up to a multiple of batch_size, which puts every
    boundary on a SloMo batch boundary of the clip; the last segment takes the pairs that are left.

    world > 1: the segments of V2EPipeline.run_segments_sharded over `world` ranks, each one that run_clip_sharded
    accepts: at least `world` pairs, or with auto_upsample (whose batches are dealt to the ranks whole) at least
    `world` batches. segment_pairs is raised to that minimum before it is rounded, a shorter last segment is folded
    into the one before it, and a clip shorter than one segment raises ValueError. world=1 gives the plan above."""
    n_frames, world = int(n_frames), int(world)
    if n_frames < 2:
        raise ValueError("n_frames=%d: a clip needs at least two source frames" % n_frames)
    if world < 1:
        raise ValueError("world=%d: a clip needs at least one rank" % world)
    sp = DEFAULT_SEGMENT_PAIRS if segment_pairs is None else int(segment_pairs)
    if sp < 1:
        raise ValueError("segment_pairs=%d: a segment needs at least one frame pair" % sp)
    bs = max(1, int(batch_size))
    unit = bs if auto_upsample else 1                    # pairs per share a rank must get at least one of
    sp = -(-max(sp, world * unit) // bs) * bs
    n_pairs = n_frames - 1
    plan = [(p0, min(p0 + sp, n_pairs)) for p0 in range(0, n_pairs, sp)]
    p0, p1 = plan[-1]
    if -(-(p1 - p0) // unit) < world:
        if len(plan) == 1:
            raise ValueError("fewer batches of frame pairs than ranks" if auto_upsample else
                             "fewer frame pairs than ranks")
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
    def __init__(self, slomo: SuperSloMo, emulator: EventEmulator, renderer=None):
        """renderer (optional): a v2e_b200.renderer.EventRenderer the runs feed with every segment's rows, in the packets
        v2e.py's stage-3 loop renders (slomo.batch_size frames per packet, v2e.py:826-846), so that it writes the DVS
        video and its frame-times file as v2e.py does. The caller owns it and calls its cleanup() after the clip."""
        self.slomo = slomo
        self.emulator = emulator
        self.renderer = renderer

    def run(self, frames_u8, src_duration_s, t_offset=0.0, return_device=False, copy=False):
        """frames_u8: [N,H,W] uint8 source frames covering `src_duration_s` seconds.
        Returns (events [M,4] float32, frame offsets, interp_times_s, n_interp_frames). Host rows are a
        view of the emulator's pinned staging buffer unless copy=True (valid until the next call).
        The clip is run_segments' single segment."""
        if isinstance(frames_u8, np.ndarray):
            frames_u8 = torch.from_numpy(np.ascontiguousarray(frames_u8))
        n = frames_u8.shape[0]
        (res,) = self.run_segments(lambda a, b: frames_u8[a:b], n, src_duration_s, t_offset,
                                   segment_pairs=max(n - 1, 1), return_device=return_device, copy=copy)
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

        Raises ValueError, naming the segment, when get_frames returns anything but uint8 [b-a, H, W] with the first
        segment's H, W; RuntimeError, before any work, where generate_events_batch refuses the emulator (replay mode
        with per-frame noise, a sharded emulator: run_clip_sharded takes a clip over ranks)."""
        sl, em, rd = self.slomo, self.emulator, self.renderer
        em.check_batch_path()
        n = int(n_frames)
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
        first = 0                                           # the clip's index of the segment's first interpolated frame
        if m > 1:
            if sl.auto_upsample:
                bs = max(1, min(int(sl.batch_size), n - 1))
                a = (n - 2) // bs * bs
                u_last = sl.batch_upsampling(fetch(a, n, m - 1), n)
            else:
                u_last = int(sl.upsampling_factor)
            f = src_duration_s / clip_span(n - 1, sl.batch_size, u_last)
        for k, (p0, p1) in enumerate(plan):
            fr = fetch(p0, p1 + 1, k)
            interp, times, _, ups = sl.interpolate_frames(fr, return_ups=True, first_pair=p0, clip_frames=n)
            del fr
            if f is None:
                f = src_duration_s / (np.max(times) - np.min(times))          # v2e.py:794-797
            elif k == m - 1 and ups[-1] != u_last:
                raise RuntimeError("the clip's last batch got U=%d, its time-scale pre-pass U=%d" % (ups[-1], u_last))
            t = t_offset + f * times
            em._sinks_continue = k > 0
            try:
                ev, offs = em.generate_events_batch(interp, t, return_device=return_device or rd is not None, copy=copy)
            finally:
                em._sinks_continue = False
            nf = interp.shape[0]
            del interp
            if rd is not None:
                rd.render_frame_rows(ev, offs, first, sl.batch_size, end_of_clip=k == m - 1,
                                     height=em.output_height, width=em.output_width)
                if not return_device:
                    ev = em._rows_to_host(ev.shape[0], copy=copy)
            first += nf
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
                                           segment_pairs=max(n - 1, 1), group=group, return_labels=return_labels,
                                           write_sinks=write_sinks)
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
        if n - 1 < world:
            raise ValueError("fewer frame pairs than ranks")
        auto = bool(sl.auto_upsample)
        bs = max(1, min(int(sl.batch_size), n - 1))
        if segment_pairs is None:
            segment_pairs = DEFAULT_SEGMENT_PAIRS * world
        plan = segment_plan(n, sl.batch_size, segment_pairs, world=world, auto_upsample=auto)
        m = len(plan)
        if rank == 0 and sl.writes_video():
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
        if m > 1:
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
                p0, p1 = parallel.pair_range(s1 - s0, rank, world)
            p0, p1 = p0 + s0, p1 + s0
            fr = fetch(p0, p1 + 1, k)
            H = size[0][0]
            if auto:
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
        if em.rng_mode == "device" or not (em.leak_rate_hz > 0 or em.shot_noise_rate_hz > 0 or em.photoreceptor_noise):
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
            self.renderer.render_frame_rows(merged, moffs, seg[2], self.slomo.batch_size, end_of_clip=seg[1],
                                            height=H, width=W)
