"""Motion-JPEG AVI video on the device: MjpegWriter encodes greyscale frames with the CUDA encoder (csrc/mjpeg.cu, the
format in DESIGN.md §4.4) and moves only the compressed bytes to the host, where AviWriter puts them in an AVI file.

MjpegWriter(output_path, height, width, frame_rate) has the signature of the reference's v2ecore.v2e_utils.video_writer
and the cv2.VideoWriter methods v2e calls (write, isOpened, release), so it can stand wherever that factory does, e.g.
`v2ecore.v2e_utils.video_writer = MjpegWriter` in v2e.py, or `video_writer=MjpegWriter` for SuperSloMo and
EventRenderer, which then hand it their device frames through write_frames.

The container: RIFF 'AVI ' (hdrl: avih, strl with strh 'vids'/'MJPG', strf BITMAPINFOHEADER 'MJPG', an OpenDML super
index 'indx'; odml/dmlh), movi with one '00dc' chunk per frame, an OpenDML 'ix00' index per movi and the legacy idx1.
Past RIFF_LIMIT bytes the file continues in 'AVIX' RIFF segments, each with its own movi and ix00; the frame counts
are patched in at release()."""
import ctypes
import struct

import numpy as np
import torch

from . import _lib

RIFF_LIMIT = 1 << 30                  # bytes per RIFF segment (OpenDML readers take more; 1 GB keeps every reader happy)
SUPER_INDEX_ENTRIES = 256             # room for 256 RIFF segments in the super index
_KEYFRAME = 0x10


def _chunk(tag, data):
    return tag + struct.pack("<I", len(data)) + data + (b"\0" if len(data) % 2 else b"")


def _list(tag, data):
    return b"LIST" + struct.pack("<I", len(data) + 4) + tag + data


class AviWriter:
    """Writes JPEG frames into an MJPG AVI file as they come. add(jpeg) appends one frame; close() writes the indexes
    and patches the headers."""

    def __init__(self, path, width, height, frame_rate):
        self.width, self.height = int(width), int(height)
        fr = float(frame_rate)
        self.scale, self.rate = (1, int(fr)) if fr.is_integer() else (1000, int(round(fr * 1000)))
        if self.rate < 1:
            raise ValueError("frame_rate must be positive, got %r" % (frame_rate,))
        self.f = open(path, "wb")
        self.frames = 0
        self.max_chunk = 0
        self.segments = []                          # (ix00 offset, ix00 size, frames) of every finished segment
        self._write_headers()
        self._open_segment(first=True)

    def _write_headers(self):
        w, h = self.width, self.height
        avih = struct.pack("<10I4I", int(round(1e6 * self.scale / self.rate)), 0, 0, _KEYFRAME, 0, 0, 1, 0, w, h,
                           0, 0, 0, 0)
        strh = b"vids" + b"MJPG" + struct.pack("<IHHIIIIIIIIhhhh", 0, 0, 0, 0, self.scale, self.rate, 0, 0, 0,
                                               0xFFFFFFFF, 0, 0, 0, w, h)
        strf = struct.pack("<IiiHH4sIiiII", 40, w, h, 1, 24, b"MJPG", w * h * 3, 0, 0, 0, 0)
        indx = struct.pack("<HBBI4s3I", 4, 0, 0, 0, b"00dc", 0, 0, 0) + bytes(16 * SUPER_INDEX_ENTRIES)
        strl = _list(b"strl", _chunk(b"strh", strh) + _chunk(b"strf", strf) + _chunk(b"indx", indx))
        odml = _list(b"odml", _chunk(b"dmlh", bytes(248)))
        hdrl = _list(b"hdrl", _chunk(b"avih", avih) + strl + odml)
        head = b"RIFF" + struct.pack("<I", 0) + b"AVI " + hdrl
        self.f.write(head)
        # where the counters live, for close()
        self._avih_frames = 12 + 12 + 8 + 16
        self._avih_bufsize = self._avih_frames + 12
        strh_at = head.index(b"strh") + 8
        self._strh_length = strh_at + 32
        self._strh_bufsize = strh_at + 36
        self._indx_at = head.index(b"indx") + 8
        self._dmlh_at = head.index(b"dmlh") + 8

    def _open_segment(self, first):
        self.riff_at = self.f.tell()
        if not first:
            self.f.write(b"RIFF" + struct.pack("<I", 0) + b"AVIX")
        self.movi_at = self.f.tell()
        self.f.write(b"LIST" + struct.pack("<I", 0) + b"movi")
        self.seg_offsets, self.seg_sizes = [], []     # data offsets (absolute) and sizes of this segment's frames
        self.first = first

    def _riff_bytes(self, extra):
        """This segment's RIFF size (from its 'RIFF' tag) once `extra` more bytes and its indexes are written."""
        n = len(self.seg_sizes) + 1
        idx = 32 + 8 * n + (8 + 16 * n if self.first else 0)
        start = 0 if self.first else self.riff_at
        return self.f.tell() - start + extra + idx

    def add(self, jpeg):
        """Appends one frame's JPEG bytes (bytes or any buffer)."""
        n = len(jpeg)
        if self.seg_sizes and self._riff_bytes(8 + n + n % 2) > RIFF_LIMIT:
            self._close_segment()
            self._open_segment(first=False)
        self.seg_offsets.append(self.f.tell() + 8)
        self.seg_sizes.append(n)
        self.f.write(b"00dc" + struct.pack("<I", n))
        self.f.write(jpeg)
        if n % 2:
            self.f.write(b"\0")
        self.frames += 1
        self.max_chunk = max(self.max_chunk, len(jpeg))

    def _close_segment(self):
        n = len(self.seg_sizes)
        base = self.movi_at
        ix_at = self.f.tell()
        rel = np.asarray(self.seg_offsets, np.int64) - base
        entries = np.stack([rel, np.asarray(self.seg_sizes, np.int64)], 1).astype("<u4").tobytes()
        ix = struct.pack("<HBBI4sqI", 2, 0, 1, n, b"00dc", base, 0) + entries
        self.f.write(_chunk(b"ix00", ix))
        self.segments.append((ix_at, 8 + len(ix), n))
        end = self.f.tell()
        self._patch(self.movi_at + 4, end - self.movi_at - 8)
        if self.first:
            # idx1: offsets from the 'movi' tag, for readers without OpenDML
            rel = np.asarray(self.seg_offsets, np.int64) - 8 - (self.movi_at + 8)
            e = np.zeros((n, 4), "<u4")
            e[:, 0] = struct.unpack("<I", b"00dc")[0]
            e[:, 1] = _KEYFRAME
            e[:, 2] = rel
            e[:, 3] = self.seg_sizes
            self.f.write(_chunk(b"idx1", e.tobytes()))
            self.first_frames = n
            end = self.f.tell()
            self._patch(4, end - 8)
        else:
            self._patch(self.riff_at + 4, end - self.riff_at - 8)

    def _patch(self, at, value):
        here = self.f.tell()
        self.f.seek(at)
        self.f.write(struct.pack("<I", value))
        self.f.seek(here)

    def close(self):
        if self.f is None:
            return
        self._close_segment()
        if len(self.segments) > SUPER_INDEX_ENTRIES:
            raise ValueError("the AVI has %d RIFF segments; its super index holds %d"
                             % (len(self.segments), SUPER_INDEX_ENTRIES))
        self._patch(self._avih_frames, self.first_frames)
        self._patch(self._avih_bufsize, self.max_chunk + 8)
        self._patch(self._strh_length, self.frames)
        self._patch(self._strh_bufsize, self.max_chunk + 8)
        self._patch(self._dmlh_at, self.frames)
        self.f.seek(self._indx_at + 4)
        self.f.write(struct.pack("<I", len(self.segments)))
        self.f.seek(self._indx_at + 24)
        for at, size, n in self.segments:
            self.f.write(struct.pack("<qII", at, size, n))
        self.f.close()
        self.f = None


class MjpegWriter:
    """A greyscale Motion-JPEG AVI writer whose encoder runs on the device.

    write_frames(frames): uint8 [n, H, W] frames (a CUDA tensor is read in place; host tensors and ndarrays are copied
    to the device): one encode and one device-to-host copy of the compressed bytes per call.
    write(frame): cv2.VideoWriter.write -- uint8 [H, W, 3] BGR or [H, W], host or device; BGR is reduced to luma with
    the pixel pipeline's integer rule, which gives g back for a GRAY2BGR frame.
    A frame of the wrong size or dtype raises ValueError (cv2.VideoWriter drops such frames silently)."""

    def __init__(self, output_path, height, width, frame_rate=30, quality=95, device="cuda:0"):
        if not 1 <= int(quality) <= 100:
            raise ValueError("quality must be 1..100, got %r" % (quality,))
        if not (1 <= int(width) <= 65535 and 1 <= int(height) <= 65535):
            raise ValueError("frame size %dx%d: each side must be 1..65535" % (width, height))
        self.height, self.width, self.quality = int(height), int(width), int(quality)
        self.device = torch.device(device)
        self._lib = _lib.load()
        self._enc, self._cap = None, 0
        self._out = self._sizes = self._sizes_host = None
        self._avi = AviWriter(output_path, self.width, self.height, frame_rate)

    def isOpened(self):
        return self._avi is not None

    def _encoder(self, n):
        if n <= self._cap:
            return
        self._free()
        cap = max(n, 2 * self._cap)
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.v2e_mjpeg_create(self.width, self.height, self.quality, cap, ctypes.byref(h)))
        self._enc, self._cap = h, cap
        bound = self._lib.v2e_mjpeg_bound(self.width, self.height, cap)
        self._out = torch.empty(bound, dtype=torch.uint8, device=self.device)
        self._sizes = torch.empty(cap, dtype=torch.int64, device=self.device)
        self._sizes_host = torch.empty(cap, dtype=torch.int64).pin_memory()

    def _free(self):
        if self._enc is not None:
            self._lib.v2e_mjpeg_destroy(self._enc)
            self._enc, self._cap = None, 0

    def encode(self, frames):
        """The JPEGs of uint8 [n, H, W] frames: (a host uint8 tensor of their bytes, one after another; their sizes)."""
        if self._avi is None:
            raise ValueError("the writer is released")
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or frames.dim() != 3 or \
                tuple(frames.shape[1:]) != (self.height, self.width):
            raise ValueError("frames must be uint8 [n, %d, %d], got %s %s" % (
                self.height, self.width, getattr(frames, "dtype", type(frames)), tuple(getattr(frames, "shape", ()))))
        n = frames.shape[0]
        if n == 0:
            return torch.empty(0, dtype=torch.uint8), np.zeros(0, np.int64)
        frames = frames.to(self.device).contiguous()
        self._encoder(n)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            _lib.check(self._lib.v2e_mjpeg_encode(self._enc, ctypes.c_void_p(frames.data_ptr()), n,
                                                  ctypes.c_void_p(self._out.data_ptr()),
                                                  ctypes.c_void_p(self._sizes.data_ptr()),
                                                  ctypes.c_void_p(stream.cuda_stream)))
            self._sizes_host[:n].copy_(self._sizes[:n], non_blocking=True)
            stream.synchronize()                       # the one synchronisation: the sizes size the copy
            sizes = self._sizes_host[:n].numpy().copy()
            data = self._out[:int(sizes.sum())].cpu()
        return data, sizes

    def write_frames(self, frames):
        data, sizes = self.encode(frames)
        buf = memoryview(data.numpy())
        o = 0
        for s in sizes:
            self._avi.add(buf[o:o + s])
            o += s

    def write(self, frame):
        if isinstance(frame, np.ndarray):
            frame = torch.from_numpy(frame)
        if not isinstance(frame, torch.Tensor) or frame.dtype != torch.uint8 or \
                tuple(frame.shape[:2]) != (self.height, self.width) or \
                not (frame.dim() == 2 or (frame.dim() == 3 and frame.shape[2] == 3)):
            raise ValueError("frame must be uint8 [%d, %d] or [%d, %d, 3], got %s %s" % (
                self.height, self.width, self.height, self.width, getattr(frame, "dtype", type(frame)),
                tuple(getattr(frame, "shape", ()))))
        if frame.dim() == 3:
            frame = bgr_to_luma(frame)
        self.write_frames(frame[None])

    def release(self):
        if self._avi is not None:
            self._avi.close()
            self._avi = None
        self._free()
        self._out = self._sizes = self._sizes_host = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def bgr_to_luma(bgr):
    """uint8 [..., 3] BGR -> uint8 luma: (B*3735 + G*19235 + R*9798 + 2^14) >> 15, the integer rule of the pixel
    pipeline's BGR2GRAY (csrc/prep.cu). The weights sum to 2^15, so a GRAY2BGR frame gives its grey back."""
    x = bgr.to(torch.int32)
    return ((x[..., 0] * 3735 + x[..., 1] * 19235 + x[..., 2] * 9798 + (1 << 14)) >> 15).to(torch.uint8)
