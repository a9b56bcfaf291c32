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
from .slomo import SuperSloMo

logger = logging.getLogger(__name__)


class V2EPipeline:
    def __init__(self, slomo: SuperSloMo, emulator: EventEmulator):
        self.slomo = slomo
        self.emulator = emulator

    def run(self, frames_u8, src_duration_s, t_offset=0.0, return_device=False, copy=False):
        """frames_u8: [N,H,W] uint8 source frames covering `src_duration_s` seconds.
        Returns (events [M,4] float32, frame offsets, interp_times_s, n_interp_frames). Host rows are a
        view of the emulator's pinned staging buffer unless copy=True (valid until the next call)."""
        interp, times, avg_u = self.slomo.interpolate_frames(frames_u8)
        f = src_duration_s / (np.max(times) - np.min(times))          # v2e.py:794-797
        t = t_offset + f * times
        ev, offs = self.emulator.generate_events_batch(interp, t, return_device=return_device, copy=copy)
        return ev, offs, t, interp.shape[0]

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
        emulator's write_events -- the files a single-GPU V2EPipeline.run writes. Only that rank's emulator may be built
        with sink keywords (dvs_text, dvs_aedat2, ...); the others are built without, since they would open, and
        truncate, the same paths. The ranks check this together before any data moves and all raise ValueError when
        another rank holds sinks. The return values are those of write_sinks=False."""
        import torch.distributed as dist
        from . import parallel
        from .slomo import clip_times
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        em = self.emulator
        if em.shard is None:
            raise RuntimeError("run_clip_sharded needs EventEmulator(shard=(rank, world, group))")
        if return_labels and not em.label_signal_noise:
            raise ValueError("return_labels=True needs label_signal_noise=True")
        if write_sinks:
            if em.row_order is None:
                raise ValueError("write_sinks=True needs EventEmulator(row_order='canonical' or 'shuffled'): the bands "
                                 "are merged by their sort keys")
            # every rank learns who holds sinks, so that all of them raise (none waits in a collective)
            nccl = dist.get_backend(group) == "nccl"
            flag = torch.tensor([0 if em._sinks is None else 1], dtype=torch.int64,
                                device=em.device if nccl else "cpu")
            flags = [torch.zeros_like(flag) for _ in range(world)]
            dist.all_gather(flags, flag, group=group)
            flags = [int(f.item()) for f in flags]
            bad = [r for r in range(1, world) if flags[r]]
            if bad:
                raise ValueError("write_sinks=True: only the group's first rank may hold sinks, ranks %s do; build "
                                 "their emulators without dvs_* keywords" % bad)
            write_sinks = bool(flags[0])
        if isinstance(frames_u8, np.ndarray):
            frames_u8 = torch.from_numpy(np.ascontiguousarray(frames_u8))
        n, H, W = frames_u8.shape
        if n - 1 < world:
            raise ValueError("fewer frame pairs than ranks")
        if rank == 0 and self.slomo.writes_video():
            logger.warning("video_path ignored: a clip sharded over ranks writes no upsampler video")
        if self.slomo.auto_upsample:
            bs = max(1, min(int(self.slomo.batch_size), n - 1))
            p0, p1 = parallel.batch_pair_range(n - 1, bs, rank, world)
            local, _, _, ups_l = self.slomo.interpolate_frames(frames_u8[p0:p1 + 1], return_ups=True,
                                                              write_video=False)
            # every rank's per-batch U's (a few ints; each rank knows how many batches every rank holds)
            nb = [-(-(b - a) // bs) for a, b in (parallel.batch_pair_range(n - 1, bs, r, world) for r in range(world))]
            send = torch.zeros(max(nb), dtype=torch.int64, device=local.device)
            send[:len(ups_l)] = torch.tensor(ups_l, dtype=torch.int64)
            recv = [torch.empty_like(send) for _ in range(world)]
            dist.all_gather(recv, send, group=group)
            ups = [u for r in range(world) for u in recv[r][:nb[r]].tolist()]
            times, _ = clip_times(ups, n - 1, bs)
        else:
            p0, p1 = parallel.pair_range(n - 1, rank, world)
            local, times_l, _ = self.slomo.interpolate_frames(frames_u8[p0:p1 + 1], write_video=False)
            U = int(self.slomo.upsampling_factor)
            times = np.arange((n - 1) * U) * (1.0 / U)                       # slomo.py:391-395 for the whole clip
            assert np.allclose(times_l + p0, times[p0 * U:p1 * U])
        bands = parallel.exchange_frame_bands(local, H, group=group, halo=em.cs_halo_rows(H))
        f = src_duration_s / (np.max(times) - np.min(times))            # v2e.py:794-797
        t = t_offset + f * times
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
            self._write_merged(rows, keys, offs, group)
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

    def _write_merged(self, rows, keys, offs, group):
        """write_sinks: the bands of every rank to the group's first rank, merged there and written to its sinks."""
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
