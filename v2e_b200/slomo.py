"""SuperSloMo -- drop-in for v2ecore/slomo.py:37 backed by the sm_90a (H100) kernels.

Same constructor and `interpolate(source_frame_path, output_folder, frame_size)` contract as the
reference (slomo.py:44-54, 231-495): reads `*.npy` luma frames from a folder, writes `<index>.png`
frames, returns `(interpTimes, avgUpsampling)`. Everything between the two file formats runs on the
GPU through the C ABI (include/v2e_b200.h): Pillow-exact LANCZOS down-resize (dataloader.py:142),
flow UNet, per-t interpolation UNet + warps + blend (slomo.py:404-433), uint8 quantisation
(slomo.py:437) and Pillow-exact BILINEAR up-resize (slomo.py:438).

`interpolate_frames()` is the in-memory fast path (not in the reference): uint8 frames in, uint8
interpolated frames out (device tensors), no temp folders -- what the event emulator consumes.

The reference's CPU branch skips the 0.428 mean normalisation (slomo.py:154-156); like the
reference on a CUDA machine, this class always applies it.

With `video_path` set, both paths write the reference's two videos (slomo.py:288-303, 468-491): `vid_orig`, the
source frames, and `vid_slomo`, the interpolated frames in output order, each converted GRAY2BGR on the host and
written through v2ecore.v2e_utils.video_writer (its codec) when that imports; otherwise a warning and no files.
`video_writer` (a factory with that function's signature, e.g. v2e_b200.video.MjpegWriter) replaces it for this object's
videos; writers with write_frames get each batch's uint8 frames on the device, with no host copy and no GRAY2BGR.
`preview` windows are not opened.
"""
import atexit
import ctypes
import glob
import logging
import os

import numpy as np
import torch

from . import _lib

logger = logging.getLogger(__name__)

# forward order of the 23 convolutions (model.py:184-196) as state_dict prefixes
LAYER_NAMES = (["conv1", "conv2"] +
               ["down%d.conv%d" % (d, c) for d in range(1, 6) for c in (1, 2)] +
               ["up%d.conv%d" % (u, c) for u in range(1, 6) for c in (1, 2)] +
               ["conv3"])


def unet_layer_shapes(in_ch, out_ch):
    """[(cout, cin, k)] for UNet(in_ch, out_ch) in LAYER_NAMES order (model.py:184-196)."""
    ch = [32, 64, 128, 256, 512, 512]
    dk = [5, 3, 3, 3, 3]
    s = [(32, in_ch, 7), (32, 32, 7)]
    for d in range(5):
        s += [(ch[d + 1], ch[d], dk[d]), (ch[d + 1], ch[d + 1], dk[d])]
    uo, ui = [512, 256, 128, 64, 32], [512, 512, 256, 128, 64]
    for k in range(5):
        s += [(uo[k], ui[k], 3), (uo[k], 2 * uo[k], 3)]
    s += [(out_ch, 32, 3)]
    return s


def batch_times(in_ctr, b, U):
    """interpTimes of one batch of b pairs starting at pair in_ctr, up-sampled U times (slomo.py:391-395)."""
    return in_ctr + np.array(range(U * b)) * (1 / U)


def clip_times(ups, n_pairs, batch_size):
    """(interpTimes, avgUpsampling) of a clip of n_pairs frame pairs interpolated in batches of batch_size consecutive
    pairs (the last one short) with U = ups[i] for batch i: what SuperSloMo.interpolate_frames returns for the whole
    clip, assembled from the per-batch U's alone (a pair-sharded clip gathers them from its ranks)."""
    bs = max(1, min(int(batch_size), n_pairs))
    starts = range(0, n_pairs, bs)
    if len(ups) != len(starts):
        raise ValueError("%d U's for %d batches" % (len(ups), len(starts)))
    times = [batch_times(a, min(bs, n_pairs - a), int(U)) for a, U in zip(starts, ups)]
    return np.concatenate(times), sum(ups) / len(ups)


def clip_span(n_pairs, batch_size, last_U):
    """max(interpTimes) - min(interpTimes) of a clip of n_pairs frame pairs in batches of batch_size whose last batch is
    up-sampled last_U times: the denominator of v2e.py:794-797, known before any other batch is interpolated. The same
    double as for clip_times(...)[0]: the times start at 0.0 and increase, so the span is the last batch's last time."""
    bs = max(1, min(int(batch_size), n_pairs))
    a = (n_pairs - 1) // bs * bs
    return batch_times(a, n_pairs - a, int(last_U))[-1] - 0.0


def _write_gray(writer, frames):
    """Writes host [H, W] uint8 frames to a video writer as cv2.cvtColor(frame, GRAY2BGR) (slomo.py:480-490): the
    three channels are made on the host, so the device-to-host copy moves one. Returns how many were written."""
    import cv2
    n = 0
    for f in frames:
        writer.write(cv2.cvtColor(f, cv2.COLOR_GRAY2BGR))
        n += 1
    return n


def _write_device(writer, frames):
    """Hands a writer with write_frames uint8 [n, H, W] frames (a tensor, host or device); returns n."""
    writer.write_frames(frames)
    return int(frames.shape[0])


def _weights_struct(state_dict, in_ch, out_ch, keep):
    st = _lib.V2eUNetWeights()
    for i, (name, (co, ci, k)) in enumerate(zip(LAYER_NAMES, unet_layer_shapes(in_ch, out_ch))):
        w = state_dict[name + ".weight"].detach().to("cpu", torch.float32).contiguous()
        b = state_dict[name + ".bias"].detach().to("cpu", torch.float32).contiguous()
        if tuple(w.shape) != (co, ci, k, k) or tuple(b.shape) != (co,):
            raise ValueError("checkpoint tensor %s has shape %s, expected %s" % (name, tuple(w.shape), (co, ci, k, k)))
        keep += [w, b]
        st.w[i] = w.data_ptr()
        st.b[i] = b.data_ptr()
    return st


class SloMoEngine:
    """Device-side interpolator for frames of one size: resizers + the two UNets."""

    def __init__(self, state_dict_fc, state_dict_at, ori_dim, max_batch, device):
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.ori_w, self.ori_h = int(ori_dim[0]), int(ori_dim[1])
        self.w, self.h = int(self.ori_w / 32) * 32, int(self.ori_h / 32) * 32     # dataloader.py:122-123
        if self.w < 32 or self.h < 32:
            raise ValueError("frame size %s is smaller than one 32x32 network cell" % (ori_dim,))
        self.max_batch = int(max_batch)
        keep = []
        fc = _weights_struct(state_dict_fc, 2, 4, keep)
        at = _weights_struct(state_dict_at, 12, 5, keep)
        self._h = ctypes.c_void_p()
        self._rin = ctypes.c_void_p()
        self._rout = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.v2e_slomo_create(self.h, self.w, self.max_batch, ctypes.byref(fc), ctypes.byref(at),
                                                 ctypes.byref(self._h)))
            _lib.check(self.lib.v2e_resize_create(self.ori_w, self.ori_h, self.w, self.h, 1, self.max_batch + 1,
                                                  ctypes.byref(self._rin)))      # LANCZOS, dataloader.py:142
            _lib.check(self.lib.v2e_resize_create(self.w, self.h, self.ori_w, self.ori_h, 0, self.max_batch,
                                                  ctypes.byref(self._rout)))     # BILINEAR, slomo.py:438
        self._net_in = torch.empty((self.max_batch + 1, self.h, self.w), dtype=torch.uint8, device=self.device)
        self._net_out = torch.empty((self.max_batch, self.h, self.w), dtype=torch.uint8, device=self.device)
        self.cur_b = 0

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def close(self):
        if self._h:
            self.lib.v2e_slomo_destroy(self._h)
            self.lib.v2e_resize_destroy(self._rin)
            self.lib.v2e_resize_destroy(self._rout)
            self._h = None

    def set_pairs(self, frames_u8_dev):
        """frames_u8_dev: [B+1, ori_h, ori_w] uint8 device tensor of consecutive source frames."""
        b = frames_u8_dev.shape[0] - 1
        assert 1 <= b <= self.max_batch and frames_u8_dev.dtype == torch.uint8 and frames_u8_dev.is_contiguous()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.v2e_resize_run(self._rin, ctypes.c_void_p(frames_u8_dev.data_ptr()),
                                               ctypes.c_void_p(self._net_in.data_ptr()), b + 1, self._stream()))
            _lib.check(self.lib.v2e_slomo_set_pairs(self._h, ctypes.c_void_p(self._net_in.data_ptr()), b,
                                                    self._stream()))
        self.cur_b = b

    def max_flow(self):
        v = ctypes.c_float(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.v2e_slomo_max_flow(self._h, ctypes.byref(v), self._stream()))
        return float(v.value)

    def interp(self, t, out_u8_dev, ft_f32_dev=None):
        """out_u8_dev: [B, ori_h, ori_w] uint8 device view whose images are contiguous; the images themselves may
        be strided (out[k::U] of the output clip: frame of pair b at step k lands at U*b + k, slomo.py:440)."""
        b = self.cur_b
        assert out_u8_dev.shape == (b, self.ori_h, self.ori_w) and out_u8_dev[0].is_contiguous()
        stride = out_u8_dev.stride(0) if b > 1 else self.ori_h * self.ori_w
        with torch.cuda.device(self.device):
            _lib.check(self.lib.v2e_slomo_interp(self._h, float(t), ctypes.c_void_p(self._net_out.data_ptr()),
                                                 None if ft_f32_dev is None else ctypes.c_void_p(ft_f32_dev.data_ptr()),
                                                 self._stream()))
            _lib.check(self.lib.v2e_resize_run_strided(self._rout, ctypes.c_void_p(self._net_out.data_ptr()),
                                                       ctypes.c_void_p(out_u8_dev.data_ptr()), b, stride, self._stream()))

    def check_finite(self):
        """Raises FloatingPointError if a network head or a blended pixel was inf / nan since the last check: the
        convolutions run on fp16 operands (fp32 accumulation), a checkpoint whose activations exceed 65504 overflows.
        One small D2H read (synchronises the stream)."""
        bad = ctypes.c_int(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.v2e_slomo_check_finite(self._h, ctypes.byref(bad), self._stream()))
        if bad.value:
            raise FloatingPointError("SuperSloMo produced non-finite values: fp16 activations overflowed "
                                     "(this checkpoint needs a wider dynamic range than the fp16 tensor-core path has)")

    def _view(self, ptr_fn):
        from .emulator import _DevView
        ptr = ptr_fn(self._h)
        v = _DevView(ptr, (self.cur_b, self.h, self.w, 8), "<f4", self)
        return torch.as_tensor(v, device=self.device)

    def flow_out(self):
        return self._view(self.lib.v2e_slomo_flow_ptr)

    def intrp_out(self):
        return self._view(self.lib.v2e_slomo_intrp_ptr)

    # engine internals for layer-by-layer tests: v2e_slomo_buffer_ptr / v2e_slomo_layer_kernel (include/v2e_b200.h)
    _BUFS = {"in16": 0, "x0": 1, "s1": 2, "pool": 3, "da": 4, "s": 5, "up": 6, "ua": 7, "ub": 8, "img": 9}
    KERNELS = {0: None, 1: "tap", 2: "strip", 3: "strip_pool", 4: "up2"}

    def activations(self):
        """Views (no copies) of the engine's buffers for the current batch: fp16 NHWC "in16", "x0", "s1", lists of
        five "pool", "da", "s" (level l at 1/2^(l+1) resolution) and "up", "ua", "ub" (up block k at 1/2^(4-k)), and
        the fp32 normalised frames "img" [B+1, H, W]. The flow and interpolation networks share these buffers: read the
        flow network's after set_pairs and before interp. up[k] is stale when up block k ran fused (layer_kernels)."""
        from .emulator import _DevView
        b, H, W = self.cur_b, self.h, self.w
        shapes = unet_layer_shapes(12, 5)

        def view(name, index, shape, typestr="<f2"):
            ptr = self.lib.v2e_slomo_buffer_ptr(self._h, self._BUFS[name], index)
            if not ptr:
                raise RuntimeError("v2e_slomo_buffer_ptr: no buffer %s[%d]" % (name, index))
            return torch.as_tensor(_DevView(ptr, shape, typestr, self), device=self.device)

        a = {"in16": view("in16", 0, (b, H, W, 16)), "x0": view("x0", 0, (b, H, W, 32)),
             "s1": view("s1", 0, (b, H, W, 32)), "img": view("img", 0, (b + 1, H, W), "<f4")}
        for name, first, lvl in (("pool", 2, lambda l: l + 1), ("da", 2, lambda l: l + 1), ("s", 3, lambda l: l + 1),
                                 ("up", 12, lambda k: 4 - k), ("ua", 12, lambda k: 4 - k), ("ub", 13, lambda k: 4 - k)):
            a[name] = []
            for i in range(5):
                co, ci, _ = shapes[first + 2 * i]
                c = ci if name in ("pool", "up") else co
                a[name].append(view(name, i, (b, H >> lvl(i), W >> lvl(i), c)))
        return a

    def layer_kernels(self):
        """{"flow": [...], "interp": [...]}: per layer (forward order), the kernel that ran it in the last forward pass
        of that network: "tap", "strip", "strip_pool" (pool of the next down block from the epilogue), "up2" (fused x2
        up-sampling), or None (not run yet)."""
        out = {}
        for net, name in ((0, "flow"), (1, "interp")):
            codes = [self.lib.v2e_slomo_layer_kernel(self._h, net, i) for i in range(len(LAYER_NAMES))]
            for c in codes:
                if c < 0:
                    _lib.check(c)
            out[name] = [self.KERNELS[c] for c in codes]
        return out


class SuperSloMo(object):
    def __init__(self, model: str, auto_upsample: bool, upsampling_factor: object, batch_size=1,
                 video_path=None, vid_orig='original.avi', vid_slomo='slomo.avi', preview=False,
                 avi_frame_rate=30, device="cuda:0", state_dicts=None, video_writer=None):
        """`model`: checkpoint path as in the reference (slomo.py:44-54); `state_dicts` (extension):
        a dict with 'state_dictFC' / 'state_dictAT' used instead of loading `model`; `video_writer` (extension): the
        factory that opens vid_orig / vid_slomo instead of v2ecore.v2e_utils.video_writer."""
        if not torch.cuda.is_available():
            raise RuntimeError("v2e_b200.SuperSloMo needs a CUDA device; there is no CPU fallback")
        self.device = device
        self.checkpoint = model
        self.batch_size = batch_size
        if not auto_upsample and (not isinstance(upsampling_factor, int) or upsampling_factor < 2):
            raise ValueError('upsampling_factor={} but must be an int value>1 when auto_upsample=True'
                             .format(upsampling_factor))
        self.upsampling_factor = upsampling_factor
        self.auto_upsample = auto_upsample
        if preview:
            logger.warning("preview windows are out of scope here: ignored")
        self.video_path, self.vid_orig, self.vid_slomo = video_path, vid_orig, vid_slomo
        self.preview, self.avi_frame_rate = preview, avi_frame_rate
        self.ori_writer = self.slomo_writer = None      # opened on the first batch (slomo.py:288-303)
        self._writers_opened = False
        self.video_writer = video_writer
        self.numOrigVideoFramesWritten = self.numSlomoVideoFramesWritten = 0
        self._state_dicts = state_dicts
        self._engine = None
        self.model_loaded = False
        atexit.register(self.cleanup)

    def cleanup(self):
        """slomo.py:127-138: logs the video frame counts and releases the writers; frees the device engine."""
        if self.ori_writer is not None:
            logger.info('closing original video AVI {} after writing {} frames'.format(
                self.vid_orig, self.numOrigVideoFramesWritten))
            self.ori_writer.release()
            self.ori_writer = None
        if self.slomo_writer is not None:
            logger.info('closing slomo video AVI {} after writing {} frames'.format(
                self.vid_slomo, self.numSlomoVideoFramesWritten))
            self.slomo_writer.release()
            self.slomo_writer = None
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    # -- vid_orig / vid_slomo ------------------------------------------------------------------
    def writes_video(self):
        """True when video_path and at least one of vid_orig / vid_slomo are set."""
        return self.video_path is not None and (self.vid_orig is not None or self.vid_slomo is not None)

    def _open_writers(self, H, W):
        """slomo.py:288-303: the reference's video_writer for each of vid_orig / vid_slomo that is set, at the output
        frame size. Once per object: later calls append to the same writers, and after cleanup() nothing reopens (and
        so truncates) a finished file."""
        if self._writers_opened or not self.writes_video():
            return
        self._writers_opened = True
        video_writer = self.video_writer
        if video_writer is None:
            try:
                from v2ecore.v2e_utils import video_writer
            except ImportError as e:
                logger.warning("video_path ignored: v2ecore.v2e_utils is not importable (%s)", e)
                return
        if self.vid_orig is not None:
            self.ori_writer = video_writer(os.path.join(self.video_path, self.vid_orig), H, W,
                                           frame_rate=self.avi_frame_rate)
        if self.vid_slomo is not None:
            self.slomo_writer = video_writer(os.path.join(self.video_path, self.vid_slomo), H, W,
                                             frame_rate=self.avi_frame_rate)

    # -- model ---------------------------------------------------------------------------------
    def _load_state(self):
        if self._state_dicts is not None:
            return self._state_dicts
        if not os.path.isfile(str(self.checkpoint)):
            raise FileNotFoundError('SuperSloMo model checkpoint ' + str(self.checkpoint) +
                                    ' does not exist or is not readable')
        logger.info('loading SuperSloMo model from ' + str(self.checkpoint))
        return torch.load(self.checkpoint, map_location="cpu", weights_only=False)   # slomo.py:225

    def _engine_for(self, ori_dim, batch):
        e = self._engine
        if e is None or (e.ori_w, e.ori_h) != (int(ori_dim[0]), int(ori_dim[1])) or e.max_batch < batch:
            if e is not None:
                e.close()
            sd = self._load_state()
            self._engine = SloMoEngine(sd['state_dictFC'], sd['state_dictAT'], ori_dim, batch, self.device)
            self.model_loaded = True
        return self._engine

    # -- in-memory path ------------------------------------------------------------------------
    def _upsampling(self, eng):
        """U of the batch set on `eng` (slomo.py:366-385): the flow network's ceil(max |flow|) with auto_upsample,
        floored at upsampling_factor, else upsampling_factor; at least 2."""
        if self.auto_upsample:
            U = int(np.ceil(eng.max_flow()))                          # slomo.py:366-372
            if self.upsampling_factor is not None and self.upsampling_factor > U:
                U = self.upsampling_factor
        else:
            U = self.upsampling_factor
        return max(U, 2)                                                # slomo.py:383-385

    def _batches(self, get_frames, n, H, W, out=None, pairs=None):
        """The reference's loop over batches of consecutive frame pairs (slomo.py:330-444) of a clip of n source frames.
        get_frames(a, b) returns source frames a .. b-1 as a uint8 [b-a, H, W] tensor (host or device). pairs=(p0, p1)
        runs pairs p0 .. p1-1 only (p0 on a batch boundary): batches and times are still the whole clip's. Yields, per
        batch, (frames [U*b, H, W] uint8 device, interpTimes of the batch, U): with `out` (fixed U) the frames are a
        view of out[U*(in_ctr-p0) : U*(in_ctr-p0+b)], otherwise a fresh block."""
        bs = max(1, min(int(self.batch_size), n - 1))
        p0, p1 = (0, n - 1) if pairs is None else pairs
        eng = self._engine_for((W, H), bs)
        in_ctr = p0
        while in_ctr < p1:
            b = min(bs, p1 - in_ctr)
            fr = get_frames(in_ctr, in_ctr + b + 1).to(self.device, non_blocking=True).contiguous()
            eng.set_pairs(fr)
            U = self._upsampling(eng)
            if out is not None:
                blk = out[U * (in_ctr - p0): U * (in_ctr - p0 + b)]
            else:
                blk = torch.empty((U * b, H, W), dtype=torch.uint8, device=self.device)
            for k in range(U):
                t = (k + 0.5) / U                                       # slomo.py:405
                # frame of pair bi at step k goes to index U*bi + k of the batch (slomo.py:440): written in place
                eng.interp(t, blk[k: U * b: U])
            yield blk, batch_times(in_ctr, b, U), U                     # slomo.py:391-395
            in_ctr += b

    def batch_upsampling(self, frames, clip_frames):
        """U that one batch gets: frames, uint8 [b+1, H, W] (tensor, host or device), are the source frames of one
        batch of a clip of clip_frames frames. Runs the flow network alone (slomo.py:343-385) and raises
        FloatingPointError if it overflowed."""
        n, H, W = frames.shape
        eng = self._engine_for((W, H), max(1, min(int(self.batch_size), clip_frames - 1)))
        eng.set_pairs(frames.to(self.device, non_blocking=True).contiguous())
        U = self._upsampling(eng)
        eng.check_finite()
        return U

    def interpolate_frames(self, frames, out=None, return_ups=False, write_video=True, first_pair=0, clip_frames=None):
        """frames: [N, H, W] uint8 (ndarray or tensor, host or device), N >= 2.
        Returns (out_u8 [M, H, W] device tensor, interpTimes [M] float64, avgUpsampling), and with return_ups the
        list of per-batch U's after them. Frame order and times follow slomo.py:391-400, 440: output index =
        counter + U*b + k holds the frame synthesised at t=(k+0.5)/U between source frames b and b+1, labelled with
        time b + k/U.

        first_pair / clip_frames: `frames` are source frames first_pair .. first_pair + N - 1 of a clip of clip_frames
        frames (a segment of it; first_pair on a batch boundary of the clip). The batches, their U's and the times are
        then those of the whole clip, restricted to the segment's pairs.

        With video_path set (and write_video), vid_slomo gets the returned frames in order, one device-to-host copy
        per batch, and vid_orig the N source frames (without the first when first_pair > 0: the segment before wrote
        it); the writes are synchronous. write_video=False writes neither: a rank of a sharded clip holds only part
        of it."""
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(np.ascontiguousarray(frames))
        if frames.dtype != torch.uint8 or frames.dim() != 3:
            raise ValueError("frames must be uint8 [N, H, W]")
        n, H, W = frames.shape
        if n < 2:
            raise ValueError("need at least two frames")
        clip_n = n if clip_frames is None else int(clip_frames)
        if first_pair < 0 or first_pair + n > clip_n:
            raise ValueError("frames %d .. %d are not in a clip of %d" % (first_pair, first_pair + n - 1, clip_n))
        if out is None and not self.auto_upsample:
            out = torch.empty(((n - 1) * int(self.upsampling_factor), H, W), dtype=torch.uint8, device=self.device)
        fixed = out if not self.auto_upsample else None
        chunks, times, ups = [], [], []
        for blk, tt, U in self._batches(lambda a, b: frames[a - first_pair:b - first_pair], clip_n, H, W, out=fixed,
                                        pairs=(first_pair, first_pair + n - 1)):
            times.append(tt)
            ups.append(U)
            if fixed is None:
                chunks.append(blk)
            if write_video:
                self._open_writers(H, W)
                if hasattr(self.slomo_writer, "write_frames"):
                    self.numSlomoVideoFramesWritten += _write_device(self.slomo_writer, blk)
                elif self.slomo_writer is not None:
                    self.numSlomoVideoFramesWritten += _write_gray(self.slomo_writer, blk.cpu().numpy())
        if fixed is None:
            out = torch.cat(chunks, 0)
        if write_video and hasattr(self.ori_writer, "write_frames"):
            self.numOrigVideoFramesWritten += _write_device(self.ori_writer, frames[1 if first_pair else 0:])
        elif write_video and self.ori_writer is not None:
            self.numOrigVideoFramesWritten += _write_gray(self.ori_writer, frames[1 if first_pair else 0:].cpu().numpy())
        self._engine.check_finite()
        if return_ups:
            return out, np.concatenate(times), sum(ups) / len(ups), ups
        return out, np.concatenate(times), sum(ups) / len(ups)

    # -- reference file API ----------------------------------------------------------------------
    def interpolate(self, source_frame_path, output_folder, frame_size):
        """slomo.py:231: .npy frames in, <idx>.png frames out; returns (interpTimes, avgUpsampling). Streams batch by
        batch like the reference: only one batch of source frames and its interpolated frames are resident.

        With video_path set, vid_orig gets every source .npy frame in sorted order after the last batch
        (slomo.py:471-482) and vid_slomo the frames this call writes as PNG, in output-index order, from the host copy
        each batch makes for the PNGs. The reference instead re-reads every PNG in output_folder (slomo.py:484-490);
        the two agree unless output_folder held PNGs before the call (v2e.py passes a fresh temporary directory)."""
        from PIL import Image
        if not output_folder:
            raise ValueError('output_folder is None; it must be supplied to store the interpolated frames')
        files = sorted(glob.glob("{}".format(source_frame_path) + "/*.npy"))    # dataloader.py:116
        nframes = len(os.listdir(source_frame_path))
        if nframes / self.batch_size < 2:                                       # slomo.py:276-280
            logger.warning(f'only {nframes} input frames with batch_size={self.batch_size}, '
                           'automatically reducing batch size to provide at least 2 batches')
            while nframes / self.batch_size < 2:
                self.batch_size = int(self.batch_size / 2)
        n_pairs = len(files) - 1
        if self.batch_size < 1 or -(-n_pairs // max(self.batch_size, 1)) < 2:   # slomo.py:323-324
            raise Exception('there are only {} batches in {} and we need at least 2; maybe you need to '
                            'reduce batch size or increase number of input frames'.format(
                                0 if self.batch_size < 1 else -(-n_pairs // self.batch_size), source_frame_path))
        W, H = int(frame_size[0]), int(frame_size[1])

        def get_frames(a, b):
            fr = np.stack([np.load(f) for f in files[a:b]])
            if fr.shape[1:] != (H, W):
                raise ValueError("frames on disk are %s, frame_size says %s" % (fr.shape[1:], (H, W)))
            return torch.from_numpy(np.ascontiguousarray(fr.astype(np.uint8, copy=False)))
        os.makedirs(output_folder, exist_ok=True)
        times, ups, out_ctr = [], [], 0
        for blk, tt, U in self._batches(get_frames, len(files), H, W):
            self._open_writers(H, W)
            if hasattr(self.slomo_writer, "write_frames"):
                self.numSlomoVideoFramesWritten += _write_device(self.slomo_writer, blk)
            host = blk.cpu().numpy()
            for i in range(host.shape[0]):
                Image.fromarray(host[i]).save(os.path.join(output_folder, str(out_ctr + i) + ".png"))
            if self.slomo_writer is not None and not hasattr(self.slomo_writer, "write_frames"):
                self.numSlomoVideoFramesWritten += _write_gray(self.slomo_writer, host)
            out_ctr += host.shape[0]
            times.append(tt)
            ups.append(U)
        if hasattr(self.ori_writer, "write_frames"):
            for a in range(0, len(files), 64):             # the source frames in blocks of 64 per encode
                self.numOrigVideoFramesWritten += _write_device(self.ori_writer, get_frames(a, min(a + 64, len(files))))
        elif self.ori_writer is not None:
            self.numOrigVideoFramesWritten += _write_gray(self.ori_writer, (np.load(f) for f in files))
        self._engine.check_finite()
        interp_times, avg = np.concatenate(times), sum(ups) / len(ups)
        logger.info('Wrote {} frames and returning {} frame times.\nAverage upsampling factor={:5.1f}'.format(
            out_ctr, len(interp_times), avg))
        return interp_times, avg

    def get_interpolated_timestamps(self, ts):
        """slomo.py:540-564."""
        new_ts = []
        for i in range(ts.shape[0] - 1):
            start, end = ts[i], ts[i + 1]
            new_ts.append(np.linspace(start, end, self.upsampling_factor, endpoint=False) +
                          0.5 * (end - start) / self.upsampling_factor)
        return np.hstack(new_ts)
