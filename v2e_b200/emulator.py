"""EventEmulator -- drop-in for v2ecore/emulator.py:35 backed by the sm_90a (H100) kernels.

Same constructor keywords, `generate_events(new_frame, t_frame)` contract, counters and state
attribute names as the reference (emulator.py:86-117, 619-1022; SURVEY.md 8b). Host code here is
plumbing only: it owns no arithmetic of the pixel model. What it does own is the *order of random
draws*, because parity with a seeded reference run requires the same torch CPU-generator calls
in the same order (emulator.py:459-505, 868; emulator_utils.py:122-124, 340-343).

Two RNG modes:
  rng_mode="replay" (default): thresholds / noise-rate / per-frame leak and shot fields are drawn on
      the host exactly like the reference and uploaded; per-iteration `randperm` calls are replayed
      so the returned rows are bit-identical *including order* to the reference's CPU output.
  rng_mode="device": per-frame noise comes from an in-kernel Philox4x32-7 stream; no per-frame
      host work, frames can be batched (`generate_events_batch`). Counts are bit-exact whenever no
      per-frame noise is enabled, statistically equivalent otherwise.

Extra keywords (not in the reference): rng_mode, rng (draw source object), iter_cap,
max_frames_per_step, exact_order, shard, fused, row_order, record_pixels.

Row order in device mode. The kernels put a row inside its (frame, iteration, polarity) group wherever an atomicAdd
placed it, so with row_order=None (default) the order inside a group can change from run to run. row_order="canonical"
orders every frame like the reference before its randperm (iteration-major; ON rows then OFF rows by pixel index
y*W + x; then shot ON, shot OFF by pixel); row_order="shuffled" mixes the ON and OFF rows of each (frame, iteration) in
a pseudo-random order, uniform over permutations, as the reference's randperm leaves them (emulator.py:861-870), shot
rows canonical and last. Both are sorted on the device by a key that is a function of the row alone (DESIGN.md 4.1):
the bytes do not depend on fused / max_frames_per_step / replayed chunks / buffer growth, and a row band of a sharded
clip is a subsequence of the one-GPU stream (v2e_b200.parallel.merge_by_key puts the bands back together).

Sink keywords (dvs_h5, dvs_aedat2, dvs_aedat4, dvs_text; emulator.py:325-357): the files are opened by the
reference's own writer classes (v2ecore.output.*, h5py) when those import, and fed the way the reference feeds
them (emulator.py:953-975); when they do not import the keyword is ignored with a warning. The DVS text body is
formatted on the device (v2e_b200.sinks.events_to_text) and written to the writer's file. generate_events feeds the
sinks frame by frame, generate_events_batch once per call, both through write_events, which builds the text, AEDAT-2.0
and HDF5 bytes on the device and copies only those. label_signal_noise labels every returned row signal (1) or shot noise
(0) -- `last_signnoise_label`, generate_events_batch(..., return_labels=True) -- and passes the labels to the text and
AEDAT-2.0 sinks. A pixel-sharded emulator labels its own rows (generate_events_band(_batch)(..., return_labels=True))
and writes no sink itself: a file needs the merged stream, which V2EPipeline.run_clip_sharded(..., write_sinks=True)
builds on the group's first rank and writes through that rank's write_events.

show_dvs_model_state=[names] (or ['all']) captures, like the reference (emulator.py:41-50, 580-617, 756-767), every
frame but the first: each shown state after the low-pass, noise, SCIDVS, surround and leak updates and before the
events, scaled to its MODEL_STATE_RANGES range and cast to uint8 -- on the device, on every path (DESIGN.md 4.1).
model_state_frames() returns the frames of the last call. No window is opened. save_dvs_model_state=True writes
<output_folder>/<name>.avi through the reference's v2ecore.v2e_utils.video_writer with the reference's text overlay
when that imports (a warning and no files otherwise); a sharded emulator captures its own rows and writes no file.
Two cases where the reference fails mid-run raise ValueError here at construction: save_dvs_model_state with
output_folder=None, and a shown name that is a state tensor without a display range (e.g. 'pos_thres').

record_single_pixel_states=(a, b) records, like the reference (emulator.py:278-302, 985-1009), pixel row a, column b
(the tuple indexes frames as frame[a, b]) after every frame: single_pixel_states, single_pixel_sample_count,
save_recorded_single_pixel_states(), saved to SINGLE_PIXEL_STATES_FILENAME in the current directory at cleanup(), at
exit and when SINGLE_PIXEL_MAX_SAMPLES are full. record_pixels=[(a, b), ...] (extension, up to 64) records the same
ten quantities without a limit (pixel_traces()). The device writes the samples (DESIGN.md 4.1); every path records,
and a sharded emulator records on the rank whose own rows hold the pixel.
"""
import ctypes
import logging
import math
import os
import weakref

import numpy as np
import torch

from . import _lib

logger = logging.getLogger(__name__)


class TorchGlobalRNG:
    """torch's global CPU generator, the calls the reference makes."""

    def normal(self, mean, std, shape):
        return torch.normal(mean, std, size=shape, dtype=torch.float32)

    def randn(self, shape):
        return torch.randn(shape, dtype=torch.float32)

    def rand(self, shape):
        return torch.rand(shape, dtype=torch.float32)

    def randperm(self, n):
        return torch.randperm(n)


class _DevView:
    """Minimal __cuda_array_interface__ wrapper so torch can view library-owned device memory."""

    def __init__(self, ptr, shape, typestr, owner):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr,
                                         "data": (int(ptr), False), "version": 2}
        self._owner = owner


def _linlog_lut():
    # lin_log(0..255) with the reference's expression (emulator_utils.py:18-45): exact by construction
    x = torch.arange(256, dtype=torch.float64)
    f = (1. / 20) * math.log(20)
    y = torch.where(x <= 20, x * f, torch.log(x))
    y = torch.round(y * 1e8) / 1e8
    return y.float().contiguous()


class _Sinks:
    """The reference's event writers, opened and closed the way emulator.py:325-357 / :401-421 does;
    EventEmulator.write_events feeds them."""

    def __init__(self, output_folder, dvs_h5, dvs_aedat2, dvs_aedat4, dvs_text, output_width, output_height,
                 label_signal_noise):
        self.h5 = self.h5_dataset = self.aedat2 = self.aedat4 = self.text = None
        folder = output_folder if output_folder is not None else "."

        def suffix(path, sfx):        # v2e_utils.checkAddSuffix
            return path if path.endswith(sfx) else path + sfx
        if dvs_h5:
            try:
                import h5py
                self.h5 = h5py.File(suffix(os.path.join(folder, dvs_h5), ".h5"), "w")
                self.h5_dataset = self.h5.create_dataset(name="events", shape=(0, 4), maxshape=(None, 4),
                                                         dtype="uint32", compression="gzip")
            except ImportError as e:
                logger.warning("dvs_h5 ignored: h5py is not importable (%s)", e)
        if dvs_aedat2:
            try:
                from v2ecore.output.aedat2_output import AEDat2Output
                self.aedat2 = AEDat2Output(suffix(os.path.join(folder, dvs_aedat2), ".aedat"),
                                           output_width=output_width, output_height=output_height,
                                           label_signal_noise=label_signal_noise)
            except ImportError as e:
                logger.warning("dvs_aedat2 ignored: v2ecore.output.aedat2_output is not importable (%s)", e)
        if dvs_aedat4:
            try:
                from v2ecore.output.aedat4_output import AEDat4Output
                self.aedat4 = AEDat4Output(suffix(os.path.join(folder, dvs_aedat4), ".aedat4"))
            except ImportError as e:
                logger.warning("dvs_aedat4 ignored: v2ecore.output.aedat4_output is not importable (%s)", e)
        if dvs_text:
            try:
                from v2ecore.output.ae_text_output import DVSTextOutput
                self.text = DVSTextOutput(suffix(os.path.join(folder, dvs_text), ".txt"),
                                          label_signal_noise=label_signal_noise)
            except ImportError as e:
                logger.warning("dvs_text ignored: v2ecore.output.ae_text_output is not importable (%s)", e)

    def any(self):
        return any(x is not None for x in (self.h5, self.aedat2, self.aedat4, self.text))

    def close(self):
        for w in (self.h5, self.aedat2, self.aedat4, self.text):
            if w is not None:
                try:
                    w.close()
                except Exception:
                    pass
        self.h5 = self.h5_dataset = self.aedat2 = self.aedat4 = self.text = None


def _append_aedat2(w, ev, labels, dropping=None):
    """AEDat2Output.appendEvents (aedat2_output.py:133-188) for device rows `ev` (labels: uint8 CUDA tensor or None):
    the words come from the device and are the only bytes copied; while nothing has been written, leading 8-byte
    records whose first byte is '#' are dropped (they would read as a header line) but still counted. dropping=True
    applies that rule to a call that continues an earlier one which dropped all its records. Returns True when this
    call applied the rule and dropped every record."""
    from . import sinks
    if w.file is None:
        return False
    n = ev.shape[0]
    words, n_on = sinks.events_to_aedat2(ev, w.sizex, w.sizey, labels=labels)
    body = words.cpu().numpy().view(np.uint8)
    k = 0
    if w.numEventsWritten == 0 or dropping:
        hashes = body[0::8] == 0x23
        k = n if hashes.all() else int(np.argmin(hashes))
        for _ in range(k):
            logger.warning('first event would write a # comment char, dropping it')
        body = body[8 * k:]
    w.file.write(body.tobytes())
    w.numEventsWritten += n
    on = int(n_on.item())
    w.numOnEvents += on
    w.numOffEvents += n - on
    w.file.flush()
    return k == n


def _frame_labels(n, fi):
    """label_signal_noise (emulator.py:889-923): the labels of a frame's n rows, whose control block is fi. Signal rows
    (leak included) come first, labelled True; the frame's last n_shot_on + n_shot_off rows are shot noise, False."""
    label = np.ones(n, dtype=bool)
    label[n - (int(fi.n_shot_on) + int(fi.n_shot_off)):] = False
    return label


def _replay_noise(em):
    """Replay mode with per-frame noise (leak, shot or photoreceptor): the host draws every frame's noise fields in the
    reference's order, so the emulator `em` runs its frames one by one through the single-frame phases."""
    return em.rng_mode == "replay" and (em.leak_rate_hz > 0 or em.shot_noise_rate_hz > 0 or em.photoreceptor_noise)


def _finalize(lib, box, sinks, spx, ms_writers=None):
    """weakref.finalize callback: frees the library handle, closes the writers and saves the single-pixel recording
    of a collected (or exiting) emulator without keeping it alive (the reference registers cleanup with atexit,
    emulator.py:372)."""
    _release_writers(ms_writers)
    h = box[0]
    box[0] = None
    if h:
        try:
            lib.v2e_emu_destroy(h)
        except Exception:
            pass
    if sinks is not None:
        sinks.close()
    if spx["pixel"] is not None and spx["owner"]:
        _save_pixel_states(spx["states"], spx["count"], spx["file"])


def _release_writers(writers):
    """emulator.py:424-426: the model-state video writers are released at cleanup."""
    for w in list((writers or {}).values()):
        try:
            w.release()
        except Exception:
            pass
    if writers:
        writers.clear()


# Display ranges of the model states (emulator.py:41-50): (lo, hi) built as the reference builds them, from the
# float64 scalar np.log(255), so that lo and hi - lo are the same doubles. Keys in EventEmulator.MODEL_STATES order.
_L255 = np.log(255)
_GR, _LG, _SLG = (0, 255), (0, _L255), (-_L255 / 8, _L255 / 8)
MODEL_STATE_RANGES = {'new_frame': _GR, 'log_new_frame': _LG, 'lp_log_frame': _LG, 'scidvs_highpass': _SLG,
                      'photoreceptor_noise_arr': _SLG, 'cs_surround_frame': _LG, 'c_minus_s_frame': _SLG,
                      'base_log_frame': _SLG, 'diff_frame': _SLG}
# state tensors without a display range: the reference raises KeyError when asked to show one
_NO_RANGE_TENSORS = ('pos_thres', 'neg_thres', 'noise_rate_array', 'timestamp_mem', 'scidvs_tau_arr',
                     'scidvs_previous_photo')


# the device's V2eProbeSample (include/v2e_b200.h) and the reference's recorded names (emulator.py:291-302)
_PROBE_DTYPE = np.dtype([("new_frame", "<f8"), ("log_new_frame", "<f8"), ("lp_log_frame", "<f8"),
                         ("base_log_frame", "<f8"), ("diff_frame", "<f8"), ("pos_thres", "<f8"), ("neg_thres", "<f8"),
                         ("final_pos_evts", "<i4"), ("final_neg_evts", "<i4"), ("frame", "<i4"), ("pixel", "<i4")])
_PIXEL_STATE_FIELDS = (("new_frame", "new_frame"), ("base_log_frame", "base_log_frame"),
                       ("lp_log_frame", "lp_log_frame"), ("log_new_frame", "log_new_frame"),
                       ("pos_thres", "pos_thres"), ("neg_thres", "neg_thres"), ("diff_frame", "diff_frame"),
                       ("final_neg_evts_frame", "final_neg_evts"), ("final_pos_evts_frame", "final_pos_evts"))
PIXEL_STATE_NAMES = ("time",) + tuple(k for k, _ in _PIXEL_STATE_FIELDS)


def _save_pixel_states(states, count, filename):
    """emulator.py:428-437: the dict, pickled to `filename` relative to the current directory."""
    import pickle
    try:
        with open(filename, "wb") as outfile:
            pickle.dump(states, outfile, protocol=pickle.HIGHEST_PROTOCOL)
            logger.info(f"saved single pixel states with {count} samples to {filename}")
    except Exception as e:
        logger.error(f"could not save pickled pixel states, got {e}")


def _pixel_list(arg, name):
    if not isinstance(arg, (list, tuple)) or len(arg) > 64:
        raise ValueError(f"{name} must be a list of at most 64 (row, column) tuples")
    out = []
    for p in arg:
        if not (isinstance(p, tuple) and len(p) == 2 and all(type(i) is int for i in p)):
            raise ValueError(f"{name}: {p!r} is not a (row, column) tuple of two ints")
        out.append(p)
    return out


_STATE_IDS = {"lp_log_frame": 0, "base_log_frame": 1, "pos_thres": 2, "neg_thres": 3,
              "noise_rate_array": 4, "timestamp_mem": 5, "cs_surround_frame": 6,
              "scidvs_highpass": 7, "photoreceptor_noise_arr": 8, "scidvs_tau_arr": 9}


class EventEmulator(object):
    MODEL_STATES = ('new_frame', 'log_new_frame', 'lp_log_frame', 'scidvs_highpass',
                    'photoreceptor_noise_arr', 'cs_surround_frame', 'c_minus_s_frame',
                    'base_log_frame', 'diff_frame')
    MAX_CHANGE_TO_TERMINATE_EULER_SURROUND_STEPPING = 1e-5
    SINGLE_PIXEL_STATES_FILENAME = 'pixel-states.dat'
    SINGLE_PIXEL_MAX_SAMPLES = 10000

    def __init__(
            self,
            pos_thres: float = 0.2,
            neg_thres: float = 0.2,
            sigma_thres: float = 0.03,
            cutoff_hz: float = 0.0,
            leak_rate_hz: float = 0.1,
            refractory_period_s: float = 0.0,
            shot_noise_rate_hz: float = 0.0,
            photoreceptor_noise: bool = False,
            leak_jitter_fraction: float = 0.1,
            noise_rate_cov_decades: float = 0.1,
            seed: int = 0,
            output_folder: str = None,
            dvs_h5: str = None,
            dvs_aedat2: str = None,
            dvs_aedat4: str = None,
            dvs_text: str = None,
            show_dvs_model_state: str = None,
            save_dvs_model_state: bool = False,
            output_width: int = None,
            output_height: int = None,
            device: str = "cuda",
            cs_lambda_pixels: float = None,
            cs_tau_p_ms: float = None,
            hdr: bool = False,
            scidvs: bool = False,
            record_single_pixel_states=None,
            label_signal_noise=False,
            # ---- extensions ----
            rng_mode: str = "replay",
            rng=None,
            pr_vrms_tape=None,
            iter_cap: int = 1024,
            max_frames_per_step: int = 64,
            exact_order: bool = True,
            shard=None,
            fused: bool = True,
            row_order: str = None,
            record_pixels=None,
    ):
        if not str(device).startswith("cuda"):
            raise RuntimeError("v2e_b200.EventEmulator runs on a CUDA device only (device=%r); "
                               "there is no CPU fallback" % (device,))
        if photoreceptor_noise and (shot_noise_rate_hz == 0 or cutoff_hz == 0):
            # emulator.py:196-204 logs and calls v2e_quit(1)
            logger.warning("--photoreceptor_noise needs a finite --shot_noise_rate_hz and --cutoff_hz")
            raise SystemExit(1)
        if record_single_pixel_states is not None:          # emulator.py:279-290: same argument checks
            if not (type(record_single_pixel_states) is tuple):
                raise ValueError(f'--record_single_pixel_states {record_single_pixel_states} should be a tuple, e.g. (10,20)')
            if len(record_single_pixel_states) != 2:
                raise ValueError(f'--record_single_pixel_states {record_single_pixel_states} should have two pixel addresses (x,y)')
            for i in record_single_pixel_states:
                if not (type(i) is int):
                    raise ValueError(f'--record_single_pixel_states {record_single_pixel_states} should have two integer-value pixel addresses (x,y)')
        # model-state planes (emulator.py:365-368, 580-617, 756-767): the shown states that exist in this
        # configuration; a name that does not is logged once and skipped, as the reference does
        self.show_dvs_model_state = None
        self.save_dvs_model_state = save_dvs_model_state
        self._ms_names = []
        self._ms_chunks = []          # (frame counters, t_previous, planes [k, states, rows, W]) of the last call
        self._ms_writers = {}         # name -> the reference's video writer
        self._ms_video_writer = None
        if show_dvs_model_state is not None:
            names = list(show_dvs_model_state)
            if len(names) == 1 and names[0] == 'all':
                names = list(MODEL_STATE_RANGES)
            self.show_dvs_model_state = names
            absent = set()
            if not scidvs:
                absent.add('scidvs_highpass')
            if cs_lambda_pixels is None:
                absent.update(('cs_surround_frame', 'c_minus_s_frame'))
            for s in names:
                if s in self._ms_names:
                    continue
                if s in MODEL_STATE_RANGES and s not in absent:
                    self._ms_names.append(s)
                elif s in _NO_RANGE_TENSORS:
                    raise ValueError(f"show_dvs_model_state: {s} has no display range (MODEL_STATE_RANGES)")
                else:
                    logger.error(f'{s} does not exist so we cannot show it')
            if self._ms_names:
                logger.info("show_dvs_model_state: the frames are captured on the device (model_state_frames()); "
                            "no window is opened")
                if save_dvs_model_state and output_folder is None:
                    raise ValueError("save_dvs_model_state needs an output_folder for <output_folder>/<name>.avi")
                if save_dvs_model_state and shard is None:
                    try:
                        from v2ecore.v2e_utils import video_writer
                        self._ms_video_writer = video_writer
                    except ImportError as e:
                        logger.warning("save_dvs_model_state ignored: v2ecore.v2e_utils is not importable (%s)", e)
        # single-pixel recording (emulator.py:278-302, 985-1009): shared with the finalizer, which saves at exit
        self._spx = {"pixel": record_single_pixel_states, "count": 0, "owner": True,
                     "file": self.SINGLE_PIXEL_STATES_FILENAME, "col": None,
                     "states": None if record_single_pixel_states is None else
                     {k: np.empty(self.SINGLE_PIXEL_MAX_SAMPLES) * np.nan for k in PIXEL_STATE_NAMES}}
        self._record_pixels = _pixel_list(record_pixels, "record_pixels") if record_pixels is not None else None
        self._trace_cols = None       # record_pixels: probe index of each (-1: not on this rank's rows)
        self._traces = []             # record_pixels: one (t, samples) per frame
        self._n_probes = 0
        if rng_mode not in ("replay", "device"):
            raise ValueError("rng_mode must be 'replay' or 'device'")
        if row_order not in (None, "canonical", "shuffled"):
            raise ValueError("row_order must be None, 'canonical' or 'shuffled'")
        if row_order is not None and rng_mode == "replay":
            raise ValueError("row_order needs rng_mode='device' (replay mode returns the reference's own order)")
        logger.info("ON/OFF log_e temporal contrast thresholds: {} / {} +/- {}".format(
            pos_thres, neg_thres, sigma_thres))
        self.device = torch.device(device if device != "cuda" else "cuda:0")
        self.sigma_thres = sigma_thres
        self.pos_thres_nominal = pos_thres
        self.neg_thres_nominal = neg_thres
        self.cutoff_hz = cutoff_hz
        self.leak_rate_hz = leak_rate_hz
        self.refractory_period_s = refractory_period_s
        self.shot_noise_rate_hz = shot_noise_rate_hz
        self.photoreceptor_noise = photoreceptor_noise
        self.photoreceptor_noise_vrms = None
        # parity tests: the reference's own amplitudes (its calibration draws from an unseeded generator)
        self._pr_vrms_tape = list(pr_vrms_tape) if pr_vrms_tape is not None else None
        self._vn_cache = [None, None]
        self.leak_jitter_fraction = leak_jitter_fraction
        self.noise_rate_cov_decades = noise_rate_cov_decades
        self.SHOT_NOISE_INTEN_FACTOR = 0.25
        self.output_folder = output_folder
        self.output_width = output_width
        self.output_height = output_height
        self.label_signal_noise = label_signal_noise
        self.last_signnoise_label = None     # label_signal_noise: labels of the rows generate_events last returned
        self.log_input = hdr
        self.scidvs = scidvs
        self.cs_lambda_pixels = cs_lambda_pixels
        self.cs_tau_p_ms = cs_tau_p_ms
        self.csdvs_enabled = cs_lambda_pixels is not None
        self.cs_steps_taken = []
        if self.csdvs_enabled:
            self.cs_tau_h_ms = 0 if (cs_tau_p_ms is None or cs_tau_p_ms == 0) \
                else cs_tau_p_ms / (cs_lambda_pixels ** 2)
        self.rng_mode = rng_mode
        self.rng = rng if rng is not None else TorchGlobalRNG()
        self.iter_cap = int(iter_cap)
        self.max_frames_per_step = int(max_frames_per_step)
        self.exact_order = exact_order
        # shard = (rank, world, process_group): this instance owns a band of rows of every frame
        # (v2e_b200.parallel.row_band); see _first_frame and _phase_frame
        self.shard = shard
        self.event_rows_hint = None   # initial event-buffer rows (default: max(2*H*W, 65536))
        self.seed = seed
        if seed != 0:  # emulator.py:221-224
            import random
            torch.manual_seed(seed)
            np.random.seed(seed)
            random.seed(seed)
        self.fused = bool(fused)
        self.row_order = row_order
        self._want_keys = False      # generate_events_band_batch(return_keys=True) is running
        self._keys_dev = self._last_keys = self.last_n_shot = None
        self.cs_chunk_steps = 64     # pixel-sharded centre-surround model: Euler steps per halo exchange
        self._lib = _lib.load()
        self._hbox = [None]          # the library handle, shared with the finalizer
        self._ev_dev = None
        self._ev_pin = None
        # sink keywords: delegated to the reference's writers when they import (emulator.py:325-357)
        self.dvs_h5 = self.dvs_aedat2 = self.dvs_aedat4 = self.dvs_text = None
        self._sinks = None
        # set by V2EPipeline.run_segments: the next write continues the last one, so AEDAT-2.0 keeps dropping leading
        # '#' records while every record so far was dropped, as one write of both would
        self._sinks_continue = False
        self._aedat2_dropped_all = False
        if dvs_h5 or dvs_aedat2 or dvs_aedat4 or dvs_text:
            sk = _Sinks(output_folder, dvs_h5, dvs_aedat2, dvs_aedat4, dvs_text, output_width, output_height,
                        label_signal_noise)
            if sk.any():
                self._sinks = sk
                self.dvs_h5, self.dvs_aedat2, self.dvs_aedat4, self.dvs_text = sk.h5, sk.aedat2, sk.aedat4, sk.text
        self.reset()
        self.t_previous = 0
        # the reference registers cleanup with atexit (emulator.py:372), which would keep every instance alive
        # until exit; a finalizer frees the device memory when the object is collected AND runs at exit
        self._finalizer = weakref.finalize(self, _finalize, self._lib, self._hbox, self._sinks, self._spx,
                                           self._ms_writers)

    @property
    def _h(self):
        return self._hbox[0]

    @_h.setter
    def _h(self, v):
        self._hbox[0] = v

    # single-pixel recording, by the reference's attribute names. The pixel (a, b) indexes frames as arr[(a, b)]:
    # row a, column b. Setting record_single_pixel_states = None stops recording (and the save at exit).
    record_single_pixel_states = property(lambda self: self._spx["pixel"],
                                          lambda self, v: self._spx.__setitem__("pixel", v))
    single_pixel_states = property(lambda self: self._spx["states"],
                                   lambda self, v: self._spx.__setitem__("states", v))
    single_pixel_sample_count = property(lambda self: self._spx["count"],
                                         lambda self, v: self._spx.__setitem__("count", v))

    def save_recorded_single_pixel_states(self):
        """emulator.py:428-437: pickles single_pixel_states to SINGLE_PIXEL_STATES_FILENAME in the current directory."""
        _save_pixel_states(self._spx["states"], self._spx["count"], self.SINGLE_PIXEL_STATES_FILENAME)

    def pixel_traces(self):
        """record_pixels=[(row, column), ...]: every frame's state of those pixels since construction, without the
        reference's sample limit: a dict of the recorder's names, 'time' as a float64 [frames] array and the others as
        float64 [frames, pixels] arrays (NaN for a pixel outside a sharded emulator's own rows)."""
        if self._record_pixels is None:
            raise RuntimeError("pixel_traces needs record_pixels=[(row, column), ...]")
        P = len(self._record_pixels)
        out = {"time": np.array([t for t, _ in self._traces], dtype=np.float64)}
        for key, field in _PIXEL_STATE_FIELDS:
            a = np.full((len(self._traces), P), np.nan)
            for f, (_, s) in enumerate(self._traces):
                for j, col in enumerate(self._trace_cols or []):
                    if col >= 0:
                        a[f, j] = s[col][field]
            out[key] = a
        return out

    def _set_probes(self, H, W, y0, y1, ye0):
        """The probe pixels of a new handle: the recorded pixels inside this emulator's own rows [y0, y1) of frames of
        H x W pixels, as handle-local indices (the handle's row 0 is frame row ye0)."""
        want = []
        if self._spx["pixel"] is not None:
            want.append(tuple(self._spx["pixel"]))
        want += list(self._record_pixels or [])
        for r, c in want:
            if not (0 <= r < H and 0 <= c < W):
                raise ValueError("recorded pixel (row %d, column %d) is outside the %d x %d frame" % (r, c, H, W))
        local = []
        for r, c in want:
            if y0 <= r < y1 and (r - ye0) * W + c not in local:
                local.append((r - ye0) * W + c)
        col = lambda p: local.index((p[0] - ye0) * W + p[1]) if y0 <= p[0] < y1 else -1
        if self._spx["pixel"] is not None:
            c = col(self._spx["pixel"])
            self._spx["col"] = c if c >= 0 else None
            self._spx["owner"] = c >= 0
        if self._record_pixels is not None:
            self._trace_cols = [col(p) for p in self._record_pixels]
        self._n_probes = len(local)
        if local:
            px = np.asarray(local, dtype=np.int32)
            _lib.check(self._lib.v2e_emu_set_probes(self._h, px.ctypes.data_as(ctypes.c_void_p), len(local)))

    def _drain_probes(self, t_frames):
        """After v2e_emu_collect returned V2E_OK (it synchronised): the probe samples of the step's frames."""
        if not self._n_probes:
            return
        n = self._n_probes
        buf = np.zeros(len(t_frames) * n, dtype=_PROBE_DTYPE)
        nf = ctypes.c_int(0)
        _lib.check(self._lib.v2e_emu_probe_read(self._h, buf.ctypes.data_as(ctypes.c_void_p), buf.size,
                                                ctypes.byref(nf), self._stream()))
        if nf.value != len(t_frames):
            raise RuntimeError("probe samples of %d frames, expected %d" % (nf.value, len(t_frames)))
        self._record(buf.reshape(len(t_frames), n), t_frames)

    def _record(self, samples, t_frames):
        """samples [frames, probes] (_PROBE_DTYPE) of frames at t_frames -> the recorder (emulator.py:985-1009: when
        the counter has reached SINGLE_PIXEL_MAX_SAMPLES the next frame saves the file and stops recording) and the
        record_pixels traces."""
        spx = self._spx
        for f, t in enumerate(t_frames):
            if self._record_pixels is not None:
                self._traces.append((float(t), samples[f].copy()))
            if spx["pixel"] is None or not spx["owner"] or spx["col"] is None:
                continue
            k = spx["count"]
            if k < self.SINGLE_PIXEL_MAX_SAMPLES:
                if k % 250 == 0:
                    logger.info(f"recorded {k} single pixel states")
                s = samples[f, spx["col"]]
                spx["states"]["time"][k] = t
                for key, field in _PIXEL_STATE_FIELDS:
                    spx["states"][key][k] = s[field]
                spx["count"] = k + 1
            else:
                self.save_recorded_single_pixel_states()
                spx["pixel"] = None

    def model_state_frames(self):
        """show_dvs_model_state: the frames the last generate_events / generate_events_batch /
        generate_events_band(_batch) call captured, a dict: 'frame' (the reference's frame_counter of each frame,
        int64 [k]), 't_previous' (the previous frame's time, float64 [k]; the overlay text shows both) and, for each
        shown state, a uint8 CUDA tensor [k, rows, W] of the bytes before the text overlay (a sharded emulator's own
        rows)."""
        if not self._ms_names:
            raise RuntimeError("model_state_frames needs show_dvs_model_state with a state that exists here")
        out = {"frame": np.array([f for c in self._ms_chunks for f in c[0]], np.int64),
               "t_previous": np.array([t for c in self._ms_chunks for t in c[1]], np.float64)}
        order = self._ms_order()
        if self._ms_chunks:
            planes = torch.cat([c[2] for c in self._ms_chunks], 0)
        else:
            planes = torch.zeros((0, len(order), 0, 0), dtype=torch.uint8, device=self.device)
        for name in self._ms_names:
            out[name] = planes[:, order.index(name)].contiguous()
        return out

    def _ms_order(self):
        """The shown states in the device's plane order (MODEL_STATES order)."""
        return [s for s in self.MODEL_STATES if s in self._ms_names]

    def _set_model_states(self):
        order = self._ms_order()
        mask, ls = 0, np.zeros(2 * len(self.MODEL_STATES), np.float64)
        for s in order:
            i = self.MODEL_STATES.index(s)
            lo, hi = MODEL_STATE_RANGES[s]
            mask |= 1 << i
            ls[2 * i], ls[2 * i + 1] = lo, hi - lo          # Python's own lo and hi - lo
        _lib.check(self._lib.v2e_emu_set_model_states(self._h, mask, ls.ctypes.data_as(ctypes.c_void_p)))

    def _drain_states(self, t_frames, fc0):
        """After v2e_emu_collect returned V2E_OK: the planes of the step's frames (frame counters fc0, fc0 + 1, ...;
        self.t_previous is still the time before the step's first frame)."""
        if not self._ms_names:
            return
        k = len(t_frames)
        buf = torch.empty((k, len(self._ms_names), self._own_rows, self._W), dtype=torch.uint8, device=self.device)
        nf = ctypes.c_int(0)
        _lib.check(self._lib.v2e_emu_model_state_read(self._h, ctypes.c_void_p(buf.data_ptr()), buf.numel(),
                                                      ctypes.byref(nf), self._stream()))
        if nf.value != k:
            raise RuntimeError("model-state planes of %d frames, expected %d" % (nf.value, k))
        fcs = list(range(fc0, fc0 + k))
        tps = [float(self.t_previous)] + [float(t) for t in t_frames[:-1]]
        self._ms_chunks.append((fcs, tps, buf))
        if self._ms_video_writer is not None:
            self._write_states(buf, fcs, tps)

    def _write_states(self, buf, fcs, tps):
        """emulator.py:598-617 for the captured bytes: the two putText calls draw 0.0 and 255.0 into the float image,
        which the x255 uint8 cast turns into 0 and 1; drawing 0 and 1 into the bytes gives the same frame."""
        import cv2
        host = buf.cpu().numpy()
        order = self._ms_order()
        for j, (fc, tp) in enumerate(zip(fcs, tps)):
            text = f'fr:{fc} t:{tp:.4f}s'
            for name in self._ms_names:
                img = np.ascontiguousarray(host[j, order.index(name)])
                cv2.putText(img, text, org=(0, self.output_height), fontScale=1.3, color=(0, 0, 0),
                            fontFace=cv2.FONT_HERSHEY_PLAIN, thickness=1)
                cv2.putText(img, text, org=(1, self.output_height - 1), fontScale=1.3, color=(1, 1, 1),
                            fontFace=cv2.FONT_HERSHEY_PLAIN, thickness=1)
                w = self._ms_writers.get(name)
                if w is None:
                    w = self._ms_writers[name] = self._ms_video_writer(
                        os.path.join(self.output_folder, name + '.avi'), self.output_height, self.output_width)
                w.write(cv2.cvtColor(img, cv2.COLOR_GRAY2BGR))

    # ------------------------------------------------------------------------------------------
    def reset(self):
        """emulator.py:558-578: next frame re-initialises the per-pixel state."""
        self.num_events_total = 0
        self.num_events_on = 0
        self.num_events_off = 0
        self.frame_counter = 0
        self._destroy_handle()
        self._initialized = False
        self.last_frame_info = None

    def cleanup(self):
        self._destroy_handle()
        _release_writers(self._ms_writers)
        if self._sinks is not None:
            self._sinks.close()
        if self._spx["pixel"] is not None and self._spx["owner"]:     # emulator.py:425-426
            self.save_recorded_single_pixel_states()

    def prepare_storage(self, n_frames, frame_ts):
        return None  # HDF5 frame storage is a sink (out of scope); kept for call compatibility

    def set_dvs_params(self, model: str):
        """emulator.py:513-556 presets."""
        if model == 'clean':
            self.pos_thres_nominal = self.neg_thres_nominal = 0.2
            self.sigma_thres = 0.02
            self.cutoff_hz = 0
            self.leak_rate_hz = 0
            self.leak_jitter_fraction = 0
            self.noise_rate_cov_decades = 0
            self.shot_noise_rate_hz = 0
            self.refractory_period_s = 0
        elif model == 'noisy':
            self.pos_thres_nominal = self.neg_thres_nominal = 0.2
            self.sigma_thres = 0.05
            self.cutoff_hz = 30
            self.leak_rate_hz = 0.1
            self.shot_noise_rate_hz = 5.0
            self.refractory_period_s = 0
            self.leak_jitter_fraction = 0.1
            self.noise_rate_cov_decades = 0.1
        else:
            logger.warning("dvs_params {} not known: Using commandline assigned options".format(model))
        if self._initialized:
            raise RuntimeError("set_dvs_params must be called before the first frame (or after reset())")

    def _destroy_handle(self):
        box = getattr(self, "_hbox", None)
        if box and box[0]:
            try:
                self._lib.v2e_emu_destroy(box[0])
            except Exception:
                pass
            box[0] = None
        self._cs_cache = None

    # ------------------------------------------------------------------------------------------
    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _to_device_frames(self, frames):
        """-> (contiguous device tensor, dtype code). Accepts uint8 / float32 / float64 ndarrays or
        tensors, [H,W] or [T,H,W] (emulator.py:663 copies on entry; so do we)."""
        if isinstance(frames, np.ndarray):
            if frames.dtype == np.uint8 or frames.dtype == np.float32:
                t = torch.from_numpy(np.ascontiguousarray(frames))
            else:
                t = torch.from_numpy(np.ascontiguousarray(frames, dtype=np.float64))
        elif isinstance(frames, torch.Tensor):
            t = frames
            if t.dtype not in (torch.uint8, torch.float32, torch.float64):
                t = t.to(torch.float64)
        else:
            t = torch.from_numpy(np.ascontiguousarray(np.asarray(frames), dtype=np.float64))
        t = t.to(self.device, non_blocking=True).contiguous()
        code = {torch.uint8: _lib.U8, torch.float32: _lib.F32, torch.float64: _lib.F64}[t.dtype]
        return t, code

    def _create(self, H, W, px_offset=0, own=None, cs_halo=0, full_px=0):
        cfg = _lib.V2eEmuCfg()
        cfg.width, cfg.height = W, H
        cfg.per_pixel_thres = 1 if self.sigma_thres > 0 else 0
        cfg.hdr = 1 if self.log_input else 0
        cfg.pos_thres_nominal, cfg.neg_thres_nominal = self.pos_thres_nominal, self.neg_thres_nominal
        cfg.cutoff_hz = self.cutoff_hz
        cfg.leak_rate_hz = self.leak_rate_hz
        cfg.leak_jitter_fraction = self.leak_jitter_fraction
        cfg.refractory_period_s = self.refractory_period_s
        cfg.shot_noise_rate_hz = self.shot_noise_rate_hz
        cfg.shot_inten_factor = self.SHOT_NOISE_INTEN_FACTOR
        cfg.rng_mode = 0 if self.rng_mode == "replay" else 1
        cfg.iter_cap = self.iter_cap
        cfg.seed = int(self.seed) & 0xFFFFFFFFFFFFFFFF
        cfg.csdvs = 1 if self.csdvs_enabled else 0
        cfg.max_frames_per_step = self.max_frames_per_step
        cfg.scidvs = 1 if self.scidvs else 0
        cfg.photoreceptor_noise = 1 if self.photoreceptor_noise else 0
        cfg.rng_pixel_offset = int(px_offset)
        cfg.full_frame_px = int(full_px)
        if own is not None:
            cfg.own_row0, cfg.own_rows = int(own[0]), int(own[1])
        cfg.cs_halo_rows = int(cs_halo)
        if self.csdvs_enabled:
            abs_min_tau_p = 1e-9  # emulator.py:1068-1073
            cfg.cs_tau_p_s = abs_min_tau_p if (self.cs_tau_p_ms is None or self.cs_tau_p_ms == 0) \
                else self.cs_tau_p_ms * 1e-3
            cfg.cs_tau_h_s = abs_min_tau_p / (self.cs_lambda_pixels ** 2) \
                if (self.cs_tau_h_ms is None or self.cs_tau_h_ms == 0) else self.cs_tau_h_ms * 1e-3
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.v2e_emu_create(ctypes.byref(cfg), ctypes.byref(h)))
            self._h = h
            if not self.fused:
                _lib.check(self._lib.v2e_emu_set_option(h, 0, 0))
            if self.shard is not None:
                # a row band's photoreceptor-noise draws count whole-frame pixels, like its leak / shot draws
                _lib.check(self._lib.v2e_emu_set_option(h, 1, 1))
            if self.row_order is not None:
                _lib.check(self._lib.v2e_emu_set_option(h, 2, 1 if self.row_order == "canonical" else 2))
            lut = _linlog_lut()
            _lib.check(self._lib.v2e_emu_set_linlog_lut(h, ctypes.c_void_p(lut.data_ptr()), self._stream()))
            if self._ms_names:
                self._set_model_states()
        self._H, self._W = H, W
        self._own_rows = H if own is None else int(own[1])
        self.output_width = W if self.output_width is None else self.output_width
        self.output_height = H if self.output_height is None else self.output_height
        self._state_f64 = bool(self._lib.v2e_emu_state_is_f64(h))

    def _grow_event_buffer(self, rows, keep=0):
        """Makes the device event buffer hold at least `rows` rows; a new buffer starts with the old one's first
        `keep` rows."""
        if self._ev_dev is not None and self._ev_dev.shape[0] >= rows:
            return
        old = self._ev_dev if keep else None
        self._ev_dev = None
        self._ev_dev = torch.empty((max(int(rows), 16), 4), dtype=torch.float32, device=self.device)
        if keep:
            self._ev_dev[:keep].copy_(old[:keep])

    def _bind_keys(self):
        """row_order set: tells the library where to leave the sort key of every row it orders (one uint64 per row of
        the event buffer) while generate_events_band_batch(return_keys=True) runs, nowhere otherwise."""
        if self.row_order is None:
            return
        ptr = None
        if self._want_keys:
            if self._keys_dev is None or self._keys_dev.shape[0] < self._ev_dev.shape[0]:
                self._keys_dev = torch.empty(self._ev_dev.shape[0], dtype=torch.int64, device=self.device)
            ptr = ctypes.c_void_p(self._keys_dev.data_ptr())
        _lib.check(self._lib.v2e_emu_set_key_buffer(self._h, ptr))

    def _rows_to_host(self, n_rows, base=0, copy=True):
        """Device rows -> host ndarray through a pinned staging buffer. copy=False returns a view of that
        buffer (valid until the next call) and saves one pass over the rows on the host."""
        if n_rows == 0:
            return np.zeros((0, 4), np.float32)
        if self._ev_pin is None or self._ev_pin.shape[0] < n_rows:   # pinned staging, grown on demand
            self._ev_pin = torch.empty((int(n_rows * 1.25) + 1024, 4), dtype=torch.float32).pin_memory()
        self._ev_pin[:n_rows].copy_(self._ev_dev[base:base + n_rows], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        out = self._ev_pin[:n_rows].numpy()
        return out.copy() if copy else out

    def _frame_times(self, t_frames, T):
        """t_frames as floats, checked: T of them, none earlier than the frame before (the first: t_previous)."""
        t_frames = [float(t) for t in t_frames]
        if len(t_frames) != T:
            raise ValueError("t_frames length mismatch")
        for a, b in zip([self.t_previous] + t_frames[:-1], t_frames):
            if b < a:
                raise ValueError("this frame time={} must be later than previous frame time={}".format(b, a))
        return t_frames

    def _first_frame(self, fr, code, t_frame, H):
        """Creates the handle for rows [ye0, ye1) of frames of H rows (the whole frame; when sharded, this rank's
        band plus the centre-surround halo rows), initialises the state from `fr` (those rows) and draws the
        per-pixel fields in the reference's order (emulator.py:439-511): normal(pos), normal(neg),
        [normal(scidvs tau)], randn(noise_rate). Every field is drawn for the whole frame, so that a band gets the
        values a single-GPU run gets, and keeps rows [ye0, ye1)."""
        from .parallel import band_with_halo, row_band
        rank, world = (0, 1) if self.shard is None else self.shard[:2]
        y0, y1 = row_band(H, rank, world)
        if self.shard is not None and y1 == y0:
            raise ValueError("more ranks than pixel rows")
        K = self.cs_halo_rows(H)
        ye0, ye1 = band_with_halo(H, rank, world, K)
        W = fr.shape[-1]
        # Philox counters and the conv2d summation order refer to the whole frame
        self._create(ye1 - ye0, W, px_offset=ye0 * W, own=(y0 - ye0, y1 - y0) if K else None, cs_halo=K,
                     full_px=H * W)
        self._full_h, self._ye0, self._cs_K = H, ye0, K
        with torch.cuda.device(self.device):
            self._set_probes(H, W, y0, y1, ye0)
        rows = lambda t: t[ye0:ye1].contiguous()
        L, p = self._lib, lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
        with torch.cuda.device(self.device):
            _lib.check(L.v2e_emu_first_frame(self._h, p(fr), code, float(t_frame), float(self.t_previous),
                                             self._stream()))
            pos = neg = nr = None
            if self.sigma_thres > 0:
                pos = rows(torch.clamp(self.rng.normal(self.pos_thres_nominal, self.sigma_thres, (H, W)), min=0.01))
                neg = rows(torch.clamp(self.rng.normal(self.neg_thres_nominal, self.sigma_thres, (H, W)), min=0.01))
            if self.scidvs:     # emulator.py:480-483: SCIDVS_TAU_S * exp(normal(0, SCIDVS_TAU_COV))
                tau = rows(0.01 * torch.exp(self.rng.normal(0, 0.5, (H, W))))
                _lib.check(L.v2e_emu_set_scidvs_tau(self._h, p(tau)))
            if self.leak_rate_hz > 0:
                nr = rows(torch.exp(math.log(10) * self.noise_rate_cov_decades * self.rng.randn((H, W))))
            _lib.check(L.v2e_emu_set_fields(self._h, p(pos), p(neg), p(nr)))
        self._initialized = True
        # the reference returns before `self.t_previous = t_frame` (emulator.py:717 vs :1011)

    # ------------------------------------------------------------------------------------------
    def generate_events(self, new_frame, t_frame):
        """emulator.py:619: returns float32 [N,4] rows [t, x, y, +-1] or None."""
        t_frame = float(t_frame)
        self.frame_counter += 1
        self._frame_times([t_frame], 1)
        self._ms_chunks = []
        fr, code = self._to_device_frames(new_frame)
        if fr.dim() != 2:
            raise ValueError("new_frame must be [height, width]")
        if self.shard is not None:
            ye0, ye1 = self.ext_band(fr.shape[0])
            return self._generate_band(fr[ye0:ye1], code, t_frame, fr.shape[0])
        self.last_signnoise_label = None
        if not self._initialized:
            self._first_frame(fr, code, t_frame, fr.shape[0])
            return None
        if fr.shape != (self._H, self._W):
            raise ValueError("frame size changed")
        if _replay_noise(self) or (self.rng_mode == "replay" and self.exact_order):
            ev = self._phase_frame(fr, code, t_frame)
        else:
            total, _, _ = self._run_step(fr.unsqueeze(0), code, [t_frame], self.frame_counter)
            ev = self._rows_to_host(total)
        self.t_previous = t_frame
        if ev is None or len(ev) == 0:
            return None
        if self.label_signal_noise:
            self.last_signnoise_label = _frame_labels(len(ev), self.last_frame_info)
        if self._sinks is not None:
            self.write_events(ev, self.last_signnoise_label)
        return ev

    def _pr_vrms(self, delta_time):
        """emulator.py:695-697 -> emulator_utils.py:177-295: host-side calibration of the Gaussian noise
        amplitude that gives the requested shot-noise rate after the RC low-pass; cached per sample rate
        (+-10 %). Like the reference it draws from an unseeded numpy generator, so a pixel-sharded emulator takes the
        amplitude of the shard group's first rank, broadcast to every rank (each rank still pops its own tape)."""
        if self.shard is not None:
            import torch.distributed as dist
            group = self.shard[2]
            first = dist.get_global_rank(group, 0) if group is not None else 0
            mine = dist.get_rank() == first
            v = 0.0
            if mine:
                v = self._pr_vrms_local(delta_time)
            elif self._pr_vrms_tape is not None:
                self._pr_vrms_tape.pop(0)
            # the amplitude and the first rank's calibration cache (sample rate, amplitude; nan: empty)
            msg = [v] + [math.nan if c is None else float(c) for c in self._vn_cache]
            vt = torch.tensor(msg, dtype=torch.float64, device=self.device)
            dist.broadcast(vt, src=first, group=group)
            v, rate, cached = vt.tolist()
            self._vn_cache = [None if math.isnan(rate) else rate, None if math.isnan(cached) else cached]
        else:
            v = self._pr_vrms_local(delta_time)
        self.photoreceptor_noise_vrms = v
        return v

    def _pr_vrms_local(self, delta_time):
        if self._pr_vrms_tape is not None:
            v = float(self._pr_vrms_tape.pop(0))
        else:
            rate = 1.0 / delta_time
            if self._vn_cache[0] is not None and abs(rate / self._vn_cache[0] - 1) < 0.1:
                v = self._vn_cache[1]
            else:
                f3db = self.cutoff_hz
                x = math.log10((self.shot_noise_rate_hz / f3db) / 2)
                y = -0.0026 * x ** 3 - 0.036 * x ** 2 - 0.1949 * x + 0.321
                n_s = 300
                pos = self.pos_thres_nominal + self.sigma_thres * np.random.default_rng().standard_normal(n_s)
                neg = self.neg_thres_nominal + self.sigma_thres * np.random.default_rng().standard_normal(n_s)
                vn = float(np.mean(np.minimum(pos, neg) / (10 ** y)))
                tau = 1 / (f3db * 2 * math.pi)
                dt = 1 / rate
                rin = vn * np.random.default_rng().standard_normal(np.arange(0, 1000 * tau, dt).shape)
                eps = dt / tau
                rout = np.zeros_like(rin)
                acc = 0.0
                for i in range(1, len(rin)):
                    acc = acc * (1 - eps) + rin[i] * eps
                    rout[i] = acc
                v = float(np.std(rin) / np.std(rout) * vn)
                self._vn_cache = [rate, v]
        return v

    # one frame through the single-frame phase functions, host draws interleaved like the reference's ---------
    def _phase_frame(self, fr, code, t_frame, return_device=False):
        """One frame -- this handle's rows of it -- through the single-frame phases: every frame of a sharded
        emulator, and unsharded frames in replay mode. In replay mode the host draws the per-frame fields and replays
        the per-iteration randperm calls in the reference's order (emulator.py:694-698, 868, 897). Sharded, the
        frame-global maximum (emulator.py:773-775) is all-reduced (MAX) between the update and the refractory filter.
        Returns the rows (y of the whole frame) in the canonical order -- unsharded with exact_order, the reference's
        own order -- on the host, or on the device with return_device, where device-RNG rows keep the kernels' order.
        With row_order set the library has ordered the rows and they are returned as they are. None when there are
        none."""
        import torch.distributed as dist
        sharded, replay = self.shard is not None, self.rng_mode == "replay"
        group = self.shard[2] if sharded else None
        H, W, ye0 = self._full_h, self._W, self._ye0
        L, h = self._lib, self._h
        shot_pending = replay and self.shot_noise_rate_hz > 0 and not self.photoreceptor_noise      # emulator.py:893
        tp = float(self.t_previous)
        p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())

        def field(draw):
            # drawn for the whole frame, so that a band gets the values a single-GPU run gets; this handle's rows
            return draw((H, W))[ye0:ye0 + self._H].contiguous().to(self.device)
        with torch.cuda.device(self.device):
            st = self._stream()
            if self.photoreceptor_noise:
                # emulator.py:694-698: amplitude, then the randn draw (replay mode; device mode draws it in the kernel),
                # before the leak's
                vr = (ctypes.c_double * 1)(self._pr_vrms(t_frame - tp))
                pr_dev = field(self.rng.randn) if replay else None
                _lib.check(L.v2e_emu_set_pr_noise(h, p(pr_dev), vr, 1))
            lr_dev = field(self.rng.randn) if replay and self.leak_rate_hz > 0 else None
            self._grow_event_buffer(self.event_rows_hint or max(4 * self._H * W, 1 << 16))
            self._bind_keys()
            cap = self._ev_dev.shape[0]
            fp = ctypes.c_void_p(fr.data_ptr())
            if not sharded:
                _lib.check(L.v2e_emu_phase_count(h, fp, code, t_frame, tp, p(lr_dev), None, 1 if shot_pending else 0,
                                                 cap, 0, st))
            else:
                if self._cs_K:
                    self._cs_iterate(fp, code, t_frame, tp, cap, p(lr_dev), st, W)
                else:
                    _lib.check(L.v2e_emu_phase_update(h, fp, code, t_frame, tp, p(lr_dev), None, cap, 0, st))
                mx = torch.as_tensor(_DevView(L.v2e_emu_max_n_dev(h), (1,), "<i4", self), device=self.device)
                dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=group)
                _lib.check(L.v2e_emu_phase_filter(h, t_frame, tp, cap, 0 if shot_pending else 1, st))
            counts = perms = None
            if replay or not (return_device or self.row_order is not None):
                # per-(iteration, polarity) counts on the host (one synchronisation): the replayed randperm draws and
                # the canonical row order need them
                max_n = ctypes.c_int32(0)
                counts = np.zeros(2 * self.iter_cap, np.uint32)
                _lib.check(L.v2e_emu_read_counts(h, ctypes.byref(max_n), counts.ctypes.data_as(ctypes.c_void_p),
                                                 counts.size, st))
                counts = counts[:2 * max_n.value].astype(np.int64)
            if replay:
                # one randperm(n_i) per iteration, n_i = the events of the WHOLE frame (emulator.py:868): summed over
                # the ranks when sharded, so that the seeded generator stays in step with an unsharded run
                tot = counts
                if sharded and len(counts):
                    tot = torch.from_numpy(counts.copy()).to(self.device)
                    dist.all_reduce(tot, op=dist.ReduceOp.SUM, group=group)
                    tot = tot.cpu().numpy()
                perms = []
                for it in range(len(counts) // 2):
                    k = int(tot[2 * it] + tot[2 * it + 1])
                    perms.append(self.rng.randperm(k).numpy() if k > 0 else None)
            if shot_pending:
                sr_dev = field(self.rng.rand)
                _lib.check(L.v2e_emu_phase_shot(h, fp, code, t_frame, tp, p(sr_dev), cap, st))
            _lib.check(L.v2e_emu_phase_emit(h, t_frame, tp, p(self._ev_dev), cap, st))

            def resume(first, base):        # a capacity abort left the frame counted: only its emission runs again
                _lib.check(L.v2e_emu_step(h, fp, code, 1, (ctypes.c_double * 1)(t_frame), tp, None, None,
                                          p(self._ev_dev), self._ev_dev.shape[0], base, first, 1, st))
            fi = self._collect([t_frame], self.frame_counter, resume)[1][0]
            self.last_frame_info = fi
            n_ev = int(fi.n_events)
            ev = self._ev_dev[:n_ev].clone() if counts is None and return_device else self._rows_to_host(n_ev)
            self._last_keys = self._keys_dev[:n_ev].clone() if self._want_keys else None
        self._account(fi)
        if n_ev == 0:
            return None
        if counts is not None:
            # a band's rows cannot take the reference's order: that shuffles the whole frame's rows
            ev = self._canonical_then_shuffle(ev, counts, perms if not sharded and self.exact_order else None,
                                              int(fi.n_shot_on), int(fi.n_shot_off))
        if ye0:
            ev[:, 2] += ye0
        return torch.from_numpy(ev).to(self.device) if return_device and counts is not None else ev

    def _collect(self, t_frames, fc0, relaunch, keep=False):
        """Collects the step just launched over the frames at t_frames (frame counters fc0, fc0 + 1, ...). On
        V2E_E_CAPACITY (frames done..T-1 counted, nothing emitted from frame `done` on) the event buffer grows to at
        least twice the rows those frames need, keeping the rows before frame `done` when `keep`, and
        relaunch(done, row) emits again into it, from frame `done` at `row`; then the step is collected again.
        Returns (rc, control blocks [T], done, rows) of the last collect: rc is V2E_OK, the step's probe samples and
        model-state planes drained, or V2E_E_FALLBACK, which only a v2e_emu_fused_emit chunk returns."""
        T = len(t_frames)
        info = (_lib.V2eFrameInfo * T)()
        done, rows = ctypes.c_int(0), ctypes.c_uint64(0)
        st = self._stream()
        while True:
            rc = self._lib.v2e_emu_collect(self._h, info, T, ctypes.byref(done), ctypes.byref(rows), st)
            if rc != _lib.V2E_E_CAPACITY:
                break
            first = done.value
            base = int(info[first].ev_base)
            # a multi-frame (fused) step reports the rows of every frame of the chunk; the frame-by-frame
            # kernels only those up to the frame that did not fit
            need = max(int(info[f].ev_base) + int(info[f].n_events) for f in range(first, T))
            grow = 2 * max(need, self._ev_dev.shape[0])
            if keep:
                self._grow_event_buffer(grow, keep=base)
            else:
                self._grow_event_buffer(grow)
            self._bind_keys()
            relaunch(first, base)
        if rc != _lib.V2E_E_FALLBACK:
            _lib.check(rc)
            self._drain_probes(t_frames)
            self._drain_states(t_frames, fc0)
        return rc, info, done.value, int(rows.value)

    # pixel-sharded path (SURVEY.md 8e, BASELINE config 5): this rank owns rows [y0, y1) ---------------
    def cs_halo_rows(self, H):
        """Halo rows K of the pixel-sharded centre-surround model = Euler steps between two halo exchanges
        (0 when this emulator is not a sharded centre-surround one). Bounded by the smallest band."""
        if self.shard is None or not self.csdvs_enabled:
            return 0
        from .parallel import row_band
        _, world, _ = self.shard
        smallest = min(row_band(H, r, world)[1] - row_band(H, r, world)[0] for r in range(world))
        return max(1, min(int(self.cs_chunk_steps), smallest))

    def ext_band(self, H):
        """Rows [ye0, ye1) this rank's handle covers: its own band plus the halo rows of the neighbours."""
        from .parallel import band_with_halo
        return band_with_halo(H, self.shard[0], self.shard[1], self.cs_halo_rows(H))

    def generate_events_band(self, band_frame, t_frame, full_height, return_labels=False):
        """Pixel-sharded operation with the rows already cut: band_frame is [y1-y0, W], this rank's rows
        (v2e_b200.parallel.row_band) of a frame of `full_height` rows -- what the frame exchange of
        V2EPipeline.run_clip_sharded delivers. Same contract as generate_events otherwise.
        return_labels=True (needs label_signal_noise=True) returns (rows, labels): the band's labels, a bool ndarray
        aligned with its rows (None with the rows)."""
        if self.shard is None:
            raise RuntimeError("generate_events_band needs shard=(rank, world, group)")
        if return_labels and not self.label_signal_noise:
            raise ValueError("return_labels=True needs label_signal_noise=True")
        t_frame = float(t_frame)
        self.frame_counter += 1
        self._frame_times([t_frame], 1)
        self._ms_chunks = []
        fr, code = self._to_device_frames(band_frame)
        y0, y1 = self.ext_band(int(full_height))       # the band (+ halo rows for the centre-surround model)
        if fr.dim() != 2 or fr.shape[0] != y1 - y0:
            raise ValueError("band_frame must hold rows [%d, %d) of the frame" % (y0, y1))
        ev = self._generate_band(fr, code, t_frame, int(full_height))
        return (ev, self.last_signnoise_label) if return_labels else ev

    def _generate_band(self, fr, code, t_frame, H, return_device=False):
        """Rows ext_band(H) of one frame of H rows. With label_signal_noise, last_signnoise_label labels the band's
        rows: its last n_shot_on + n_shot_off rows are the shot noise of the band (emulator.py:889-923)."""
        self.last_signnoise_label = None
        if not self._initialized:
            self._first_frame(fr, code, t_frame, H)
            return None
        ev = self._phase_frame(fr, code, t_frame, return_device)
        self.t_previous = t_frame
        if ev is not None and self.label_signal_noise:
            self.last_signnoise_label = _frame_labels(len(ev), self.last_frame_info)
        return ev

    def _cs_iterate(self, fp, code, t_frame, tp, cap, lrp, st, W):
        """Centre-surround model over row bands (emulator.py:1061-1124; BASELINE config 5): the Euler iteration in
        chunks of K steps. Per chunk: the K own rows next to each band edge go to the neighbours (their halo rows),
        K steps run on the band, then ONE all-reduce(MAX) of the chunk's per-step max|change| decides -- on the
        device, identically on every rank -- whether the iteration ended inside the chunk (the first step whose
        global maximum is <= 1e-5 is the last one applied: `cs_steps_taken` equals the single-GPU run's)."""
        import torch.distributed as dist
        rank, world, group = self.shard
        L, h, K = self._lib, self._h, self._cs_K
        ns = ctypes.c_int(0)
        _lib.check(L.v2e_emu_cs_begin(h, fp, code, t_frame, tp, cap, 0, ctypes.byref(ns), st))
        ns = ns.value
        c = getattr(self, "_cs_cache", None)
        if c is None:                # views of the library's exchange buffers (state dtype), made once per handle
            nccl = dist.get_backend(group) == "nccl"
            dtype, typestr = (torch.float64, "<f8") if self._state_f64 else (torch.float32, "<f4")
            c = self._cs_cache = dict(
                nccl=nccl,
                send=torch.as_tensor(_DevView(L.v2e_emu_cs_send_dev(h), (2, K, W), typestr, self), device=self.device),
                mxv=torch.as_tensor(_DevView(L.v2e_emu_cs_max_dev(h), (8192,), "<i8", self), device=self.device),
                gathered=torch.empty((world, 2, K, W), dtype=dtype, device=self.device))
        send, mxv, gathered = c["send"], c["mxv"], c["gathered"]
        row_bytes = 2 * K * W * gathered.element_size()
        # the upper neighbour's bottom edge / the lower neighbour's top edge, where the all-gather leaves them
        above = ctypes.c_void_p(gathered.data_ptr() + (rank - 1) * row_bytes + row_bytes // 2) if rank > 0 else None
        below = ctypes.c_void_p(gathered.data_ptr() + (rank + 1) * row_bytes) if rank < world - 1 else None
        for s0 in range(0, ns, K):
            s1 = min(ns, s0 + K)
            _lib.check(L.v2e_emu_cs_pack(h, st))
            if c["nccl"]:
                dist.all_gather_into_tensor(gathered, send, group=group)
            else:
                dist.all_gather(list(gathered.unbind(0)), send.clone(), group=group)
            _lib.check(L.v2e_emu_cs_unpack_from(h, above, below, st))
            _lib.check(L.v2e_emu_cs_chunk(h, s0, s1, st))
            dist.all_reduce(mxv[s0:s1], op=dist.ReduceOp.MAX, group=group)
            _lib.check(L.v2e_emu_cs_advance(h, s0, s1, st))
        _lib.check(L.v2e_emu_cs_update(h, fp, code, lrp, None, st))

    def generate_events_band_batch(self, band_frames, t_frames, full_height, return_device=False, return_labels=False,
                                   return_keys=False):
        """Pixel-sharded, batched (BASELINE config 5 without per-frame host work): band_frames [T, y1-y0, W] uint8,
        this rank's rows of T consecutive frames. The multi-frame kernels run the whole chunk with per-pixel state in
        registers; the only exchange is ONE all-reduce(MAX) of the T frame maxima (SURVEY.md 8e "batch as a [T]
        vector"). A chunk in which the refractory filter would run is replayed frame by frame (one all-reduce per
        frame), identically on every rank; so is every chunk with SCIDVS or photoreceptor noise, which the multi-frame
        kernels do not take. Needs rng_mode='device' when leak / shot / photoreceptor noise is on.
        Returns (rows [N,4] float32 with global y, offsets [T+1]) like generate_events_batch; return_labels=True (needs
        label_signal_noise=True) adds the band's labels like generate_events_batch(..., return_labels=True).
        return_keys=True (needs row_order) adds, last, the uint64 sort key of every row, computed by the library while
        it ordered the rows (a uint64 ndarray; with return_device a CUDA int64 tensor holding the same bits): what
        v2e_b200.parallel.merge_by_key needs, with `last_n_shot` (the shot-noise rows that end each frame of this call),
        to put the bands of all ranks into the one-GPU order."""
        if self.shard is None:
            raise RuntimeError("generate_events_band_batch needs shard=(rank, world, group)")
        if return_labels and not self.label_signal_noise:
            raise ValueError("return_labels=True needs label_signal_noise=True")
        if return_keys and self.row_order is None:
            raise ValueError("return_keys=True needs row_order='canonical' or 'shuffled'")
        if _replay_noise(self):
            raise RuntimeError("batched sharded operation with per-frame noise needs rng_mode='device'")
        self._want_keys = bool(return_keys)
        self._ms_chunks = []
        try:
            return self._band_batch(band_frames, t_frames, full_height, return_device, return_labels, return_keys)
        finally:
            self._want_keys = False

    def _band_batch(self, band_frames, t_frames, full_height, return_device, return_labels, return_keys):
        import torch.distributed as dist
        rank, world, group = self.shard
        fr, code = self._to_device_frames(band_frames)
        H = int(full_height)
        y0, y1 = self.ext_band(H)        # = the band, unless the centre-surround model adds halo rows
        if fr.dim() != 3 or fr.shape[1] != y1 - y0:
            raise ValueError("band_frames must be [T, %d, W]: rows [%d, %d) of every frame" % (y1 - y0, y0, y1))
        T = fr.shape[0]
        t_frames = self._frame_times(t_frames, T)
        L = self._lib
        out, offs, n_shot, keys = [], [0], [], []
        state = {"total": 0}
        n = (y1 - y0) * fr.shape[2]

        def fused_piece(a, b):
            """Multi-frame kernels over frames [a, b). Returns None when accepted, else the index (relative to a)
            of the first frame that breaks the assumption (-1: the configuration does not qualify)."""
            Tc = b - a
            chunk = fr[a:b]
            ts = (ctypes.c_double * Tc)(*t_frames[a:b])
            with torch.cuda.device(self.device):
                st = self._stream()
                self._grow_event_buffer(self.event_rows_hint or max(2 * n, 1 << 16))
                self._bind_keys()
                rc = L.v2e_emu_fused_count(self._h, ctypes.c_void_p(chunk.data_ptr()), code, Tc, ts,
                                           float(self.t_previous), st)
                if rc == _lib.V2E_E_UNSUPPORTED:
                    return -1
                _lib.check(rc)
                # the one exchange of the chunk: frame maxima (emulator.py:773-775), MAX over the ranks
                mx = torch.as_tensor(_DevView(L.v2e_emu_max_vec_dev(self._h), (Tc,), "<i4", self), device=self.device)
                dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=group)

                def emit(*_):               # after a capacity abort: the whole chunk again, from row 0
                    _lib.check(L.v2e_emu_fused_emit(self._h, ctypes.c_void_p(self._ev_dev.data_ptr()),
                                                    self._ev_dev.shape[0], 0, st))
                emit()
                rc, info, done, nrows = self._collect(t_frames[a:b], self.frame_counter + 1, emit)
                if rc == _lib.V2E_E_FALLBACK:
                    return done
                for k in range(Tc):
                    self._account(info[k])
                    offs.append(state["total"] + int(info[k].ev_base) + int(info[k].n_events))
                    n_shot.append(int(info[k].n_shot_on) + int(info[k].n_shot_off))
                ev = self._ev_dev[:nrows].clone()
                ev[:, 2] += y0
                out.append(ev)
                if return_keys:
                    keys.append(self._keys_dev[:nrows].clone())
                state["total"] += nrows
                self.last_frame_info = info[Tc - 1]
                self.t_previous = t_frames[b - 1]
                self.frame_counter += Tc
            return None

        def frame_by_frame(a, b):
            for k in range(a, b):
                self.frame_counter += 1
                evk = self._generate_band(fr[k], code, t_frames[k], H, return_device=True)
                fi = self.last_frame_info
                if evk is not None:
                    out.append(evk)
                    if return_keys:
                        keys.append(self._last_keys)
                    state["total"] += len(evk)
                offs.append(state["total"])
                n_shot.append(0 if evk is None else int(fi.n_shot_on) + int(fi.n_shot_off))

        f = 0
        if not self._initialized:
            frame_by_frame(0, 1)
            f = 1
        while f < T:
            e = min(T, f + self.max_frames_per_step)
            bad = -1 if (e - f < 2 or not self.fused) else fused_piece(f, e)
            if bad is not None:
                # rejected (identically on every rank): the frames before the first offending one go through the
                # multi-frame kernels again, the rest of the chunk frame by frame (one all-reduce per frame)
                g = f
                if bad >= 2:
                    again = fused_piece(f, f + bad)
                    assert again is None, "a prefix of a rejected chunk must be accepted"
                    g = f + bad
                frame_by_frame(g, e)
            f = e
        offs = np.asarray(offs, np.int64)
        self.last_n_shot = np.asarray(n_shot, np.int64)      # shot-noise rows that end each frame of this call
        rows = torch.cat(out, 0) if out else torch.zeros((0, 4), dtype=torch.float32, device=self.device)
        labels = None
        if return_labels:
            from .sinks import signnoise_labels
            labels = signnoise_labels(offs, n_shot, self.device)
            if not return_device:
                labels = labels.cpu().numpy().astype(bool)
        if not return_device:
            rows = rows.cpu().numpy()
        res = (rows, offs, labels) if return_labels else (rows, offs)
        if return_keys:
            k = torch.cat(keys, 0) if keys else torch.zeros((0,), dtype=torch.int64, device=self.device)
            res += (k if return_device else k.cpu().numpy().view(np.uint64),)
        return res

    def _canonical_then_shuffle(self, ev, counts, perms, shot_on, shot_off):
        """Device rows of one (iteration, polarity) group come in no particular order. The reference
        builds each iteration as ON rows then OFF rows in row-major pixel order and shuffles it with
        randperm (emulator.py:861-870, 1024-1059); shot rows are appended unshuffled (:906-919).
        perms: the replayed permutation of every iteration, or None to keep the rows in that canonical order."""
        W = self._W
        out = np.empty_like(ev)
        off = 0
        for it in range(len(counts) // 2):
            c_on, c_off = int(counts[2 * it]), int(counts[2 * it + 1])
            k = c_on + c_off
            if k == 0:
                continue
            blk = ev[off:off + k]
            key = blk[:, 2].astype(np.int64) * W + blk[:, 1].astype(np.int64)
            key[c_on:] += (1 << 40)   # keep OFF rows after ON rows
            blk = blk[np.argsort(key, kind="stable")]
            out[off:off + k] = blk if perms is None else blk[perms[it]]
            off += k
        for c in (shot_on, shot_off):
            if c:
                blk = ev[off:off + c]
                key = blk[:, 2].astype(np.int64) * W + blk[:, 1].astype(np.int64)
                out[off:off + c] = blk[np.argsort(key, kind="stable")]
                off += c
        assert off == len(ev)
        return out

    def _account(self, fi):
        if self.csdvs_enabled:
            self.cs_steps_taken.append(int(fi.cs_steps))
        self.num_events_on += int(fi.n_on)
        self.num_events_off += int(fi.n_off)
        self.num_events_total += int(fi.n_events)

    # batched path ------------------------------------------------------------------------------
    def _run_step(self, frames_dev, code, t_frames, fc0, base_row=0):
        """frames_dev: [T,H,W] device tensor, T <= max_frames_per_step, of frame counters fc0, fc0 + 1, ... Appends
        this chunk's rows to the device event buffer starting at base_row; returns (end_row, absolute offsets[T+1],
        shot-noise rows [T])."""
        T = frames_dev.shape[0]
        L, h = self._lib, self._h
        n = self._H * self._W
        ts = (ctypes.c_double * T)(*[float(t) for t in t_frames])
        with torch.cuda.device(self.device):
            st = self._stream()
            self._grow_event_buffer(self.event_rows_hint or max(2 * n, 1 << 16))
            if self.photoreceptor_noise:
                tps = [float(self.t_previous)] + [float(t) for t in t_frames[:-1]]
                vr = (ctypes.c_double * T)(*[self._pr_vrms(float(t) - tp_) for t, tp_ in zip(t_frames, tps)])
                _lib.check(L.v2e_emu_set_pr_noise(h, None, vr, T))

            def step(first, base, resume=1):
                _lib.check(L.v2e_emu_step(h, ctypes.c_void_p(frames_dev.data_ptr()), code, T, ts,
                                          float(self.t_previous), None, None,
                                          ctypes.c_void_p(self._ev_dev.data_ptr()), self._ev_dev.shape[0],
                                          base, first, resume, st))
            step(0, int(base_row), 0)
            # on a capacity abort the rows already written are kept and the step resumes at the frame that did not fit
            _, info, _, total = self._collect(t_frames, fc0, step, keep=True)
            offsets = np.array([int(info[f].ev_base) for f in range(T)] + [total], np.int64)
            n_shot = np.array([int(info[f].n_shot_on) + int(info[f].n_shot_off) for f in range(T)], np.int64)
            for f in range(T):
                self._account(info[f])
            self.last_frame_info = info[T - 1]
            return total, offsets, n_shot

    def check_batch_path(self):
        """Raises RuntimeError where generate_events_batch cannot run this emulator: replay mode with per-frame noise,
        or a sharded emulator."""
        if _replay_noise(self):
            raise RuntimeError("generate_events_batch with per-frame noise needs rng_mode='device' "
                               "(replay mode must interleave host draws frame by frame)")
        if self.shard is not None:
            raise RuntimeError("generate_events_batch runs whole frames; a sharded emulator takes "
                               "generate_events_band_batch")

    def generate_events_batch(self, frames, t_frames, return_device=False, copy=True, return_labels=False):
        """Fast path (not in the reference): all frames of a clip in a few launches per frame and no
        per-frame host synchronisation. frames: [T,H,W]; t_frames: [T] seconds, non-decreasing.
        Returns (rows [N,4] float32, offsets [T+1]) -- rows of frame f are rows[offsets[f]:offsets[f+1]].
        With return_device=True rows is a view of the emulator's device buffer (valid until the next
        call); with copy=False the host rows are a view of the pinned staging buffer (same lifetime). The first frame of a fresh emulator only initialises state (zero rows), as in the
        reference. Needs rng_mode="device" when leak or shot noise is on.
        return_labels=True (needs label_signal_noise=True) returns (rows, offsets, labels): labels [N], 1 for a signal
        row and 0 for a shot-noise row, as a uint8 CUDA tensor with return_device, else a bool ndarray.
        The call's rows (and, with label_signal_noise, their labels) go to the open sinks through write_events."""
        if return_labels and not self.label_signal_noise:
            raise ValueError("return_labels=True needs label_signal_noise=True")
        self.check_batch_path()
        fr, code = self._to_device_frames(frames)
        if fr.dim() != 3:
            raise ValueError("frames must be [T, height, width]")
        T = fr.shape[0]
        t_frames = self._frame_times(t_frames, T)
        self._ms_chunks = []
        offs, n_shot = [0], []
        start = 0
        if not self._initialized:
            self._first_frame(fr[0], code, t_frames[0], fr.shape[1])
            self.frame_counter += 1
            offs.append(0)
            n_shot.append(0)
            start = 1
        f, row = start, 0
        while f < T:
            e = min(T, f + self.max_frames_per_step)
            row, o, s = self._run_step(fr[f:e], code, t_frames[f:e], self.frame_counter + 1, base_row=row)
            offs.extend(o[1:].tolist())
            n_shot.extend(s.tolist())
            self.t_previous = t_frames[e - 1]
            self.frame_counter += e - f
            f = e
        offs = np.asarray(offs, np.int64)
        labels = None
        if return_labels or (self._sinks is not None and self.label_signal_noise):
            from .sinks import signnoise_labels
            labels = signnoise_labels(offs, n_shot, self.device)
        if self._sinks is not None:
            # the call's rows, straight from the device buffer, to the open sinks
            self.write_events(self._ev_dev[:row] if row else torch.zeros((0, 4), dtype=torch.float32), labels)
        if not return_labels:
            labels = None
        elif not return_device:
            labels = labels.cpu().numpy().astype(bool)
        if return_device:
            if self._ev_dev is None:
                rows = torch.zeros((0, 4), dtype=torch.float32, device=self.device)
            else:
                rows = self._ev_dev[:row]
        else:
            rows = self._rows_to_host(row, copy=copy)
        return (rows, offs, labels) if return_labels else (rows, offs)

    def write_events(self, rows, labels=None):
        """Appends event rows to this emulator's open sinks (dvs_text, dvs_aedat2, dvs_h5, dvs_aedat4) and returns their
        count N: what generate_events_batch does with the rows of every call, for rows that come from elsewhere (e.g.
        the merged bands of a sharded clip). rows: [N, 4] float32 [t, x, y, +-1], a CUDA tensor or a host ndarray;
        labels: [N] (1 = signal, 0 = shot noise) or None, used only with label_signal_noise. The files get the bytes the
        reference's writers write for one appendEvents(rows, labels) call (emulator.py:953-975): the text and AEDAT-2.0
        bodies and the HDF5 rows are built on the device and only they are copied to the host; AEDAT-4 gets host rows.
        Without sinks nothing is written. Raises ValueError for rows that are not [N, 4] float32 or labels that are not
        [N]."""
        if isinstance(rows, torch.Tensor):
            ok = rows.dtype == torch.float32
        else:
            ok = isinstance(rows, np.ndarray) and rows.dtype == np.float32
        if not (ok and rows.ndim == 2 and rows.shape[1] == 4):
            raise ValueError("rows must be a float32 [N, 4] CUDA tensor or ndarray")
        n = int(rows.shape[0])
        if labels is not None and (np.ndim(labels) != 1 or len(labels) != n):
            raise ValueError("labels must be [N] for N rows")
        sk = self._sinks
        if sk is None or n == 0:
            return n
        from . import sinks
        if isinstance(rows, torch.Tensor):
            ev = rows.to(self.device).contiguous()
        else:
            ev = torch.from_numpy(np.ascontiguousarray(rows)).to(self.device)
        lab = sinks._labels(labels, ev) if self.label_signal_noise and labels is not None else None
        with torch.cuda.device(self.device):
            if sk.h5 is not None:
                # on the device: past 2^32 us the reference's numpy cast depends on the array's length (DESIGN.md 2)
                tmp = sinks.events_to_h5_rows(ev).cpu().numpy().view(np.uint32)
                sk.h5_dataset.resize(sk.h5_dataset.shape[0] + n, axis=0)
                sk.h5_dataset[-n:] = tmp
            if sk.aedat2 is not None:
                self._aedat2_dropped_all = _append_aedat2(sk.aedat2, ev, lab,
                                                          self._sinks_continue and self._aedat2_dropped_all)
            if sk.aedat4 is not None:
                sk.aedat4.appendEvents(ev.cpu().numpy(), signnoise_label=None)
            if sk.text is not None:
                if sk.text.file is None:
                    raise Exception('output file closed already')
                sk.text.numEventsWritten += sinks.write_text(sk.text.file, ev, lab)
        return n

    # state tensors by the reference's attribute names (emulator.py:756-764 reads them via getattr)
    def _state(self, name):
        if not self._initialized:
            return None
        which = _STATE_IDS[name]
        ptr = self._lib.v2e_emu_state_ptr(self._h, which)
        if not ptr:
            return None
        f64 = which in (0, 1, 6, 7) and self._state_f64      # lp, base, surround, high-pass: the state dtype
        view = _DevView(ptr, (self._H, self._W), "<f8" if f64 else "<f4", self)
        torch.cuda.current_stream(self.device).synchronize()
        # a copy: the library owns the memory and frees it at reset() / cleanup()
        return torch.as_tensor(view, device=self.device).clone()

    def cs_paths(self):
        """Centre-surround model: (cooperative, per_step) = how many Euler iterations (frames; chunks when
        pixel-sharded) ran as one cooperative launch and how many as one kernel per step."""
        coop, per_step = ctypes.c_longlong(0), ctypes.c_longlong(0)
        _lib.check(self._lib.v2e_emu_cs_paths(self._h, ctypes.byref(coop), ctypes.byref(per_step)))
        return coop.value, per_step.value

    def device_draws(self, frame_index):
        """rng_mode='device': the Philox draws of `frame_index` for every pixel of this emulator's handle, as [H, W]
        float32 CUDA tensors: 'leak_randn' (leak jitter normal), 'shot_u01' (shot-noise uniform) and 'pr_randn'
        (photoreceptor-noise normal). Frame k >= 1 of a clip uses frame_index k - 1 (frame 0 only initialises),
        whichever of generate_events / generate_events_batch ran it. For checking the kernels against a CPU model
        fed with the same draws; nothing here takes part in generating events."""
        if not self._h:
            raise RuntimeError("device_draws needs the handle the first frame creates")
        out = {k: torch.empty((self._H, self._W), dtype=torch.float32, device=self.device)
               for k in ("leak_randn", "shot_u01", "pr_randn")}
        with torch.cuda.device(self.device):
            _lib.check(self._lib.v2e_emu_draw_noise(
                self._h, int(frame_index) & 0xFFFFFFFF, *(ctypes.c_void_p(out[k].data_ptr())
                                                        for k in ("leak_randn", "shot_u01", "pr_randn")),
                self._stream()))
        return out

    lp_log_frame = property(lambda self: self._state("lp_log_frame"))
    base_log_frame = property(lambda self: self._state("base_log_frame"))
    timestamp_mem = property(lambda self: self._state("timestamp_mem"))
    noise_rate_array = property(lambda self: self._state("noise_rate_array"))
    cs_surround_frame = property(lambda self: self._state("cs_surround_frame"))
    scidvs_highpass = property(lambda self: self._state("scidvs_highpass"))
    photoreceptor_noise_arr = property(lambda self: self._state("photoreceptor_noise_arr"))
    scidvs_tau_arr = property(lambda self: self._state("scidvs_tau_arr"))

    @property
    def pos_thres(self):
        t = self._state("pos_thres") if self._initialized else None
        return t if t is not None else self.pos_thres_nominal

    @property
    def neg_thres(self):
        t = self._state("neg_thres") if self._initialized else None
        return t if t is not None else self.neg_thres_nominal
