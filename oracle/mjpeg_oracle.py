"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the greyscale Motion-JPEG encoder (v2e_b200/csrc/mjpeg.cu), byte
for byte. DESIGN.md §4.4 states the format; this module is its executable definition:

  * baseline sequential JPEG, 8-bit, one component, 1x1 sampling; markers SOI, APP0 (JFIF 1.1), DQT, SOF0, DHT (DC 0),
    DHT (AC 0), DRI, SOS, the scan, EOI;
  * a frame whose width or height is not a multiple of 8 is padded by repeating its last column and row;
  * quantisation: ITU T.81 table K.1 scaled by the IJG quality rule, s = q < 50 ? 5000 / q : 200 - 2q,
    entry clamp((K1 * s + 50) / 100, 1, 255) (integer division);
  * forward DCT, integer only: X = pixel - 128; C[u][x] = round(8192 a(u) cos((2x + 1) u pi / 16)), a(0) = sqrt(1/8),
    a(u > 0) = 1/2 (DCT_MATRIX); row pass T[y][u] = (sum_x C[u][x] X[y][x] + 2^10) >> 11 (arithmetic shift);
    column pass F[v][u] = sum_y C[v][y] T[y][u], which is the orthonormal DCT scaled by 2^15; quantised coefficient
    sign(F) * ((|F| + (Q << 14)) // (Q << 15)), round half away from zero; AC coefficients clamped to +-1023 (the
    largest magnitude table K.5 codes). Every intermediate fits int32;
  * Huffman coding with the typical tables K.3 (DC) and K.5 (AC), no per-frame optimisation;
  * restart interval one MCU row (DRI = ceil(W / 8)): the DC prediction restarts at 0 on every row, every row's bits
    are padded with 1-bits to a byte, bytes 0xFF are stuffed with 0x00, and RST0..RST7 (cycling) separate the rows.
"""
import numpy as np

# ITU T.81 K.1, natural (row-major) order
K1_LUMA = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)

# ITU T.81 K.3 (DC luminance) and K.5 (AC luminance): code counts per length 1..16, then the symbols
DC_BITS = [0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]
DC_VALS = list(range(12))
AC_BITS = [0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d]
AC_VALS = [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
    0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa]


def dct_matrix():
    a = lambda u: np.sqrt(1 / 8) if u == 0 else 0.5
    return np.array([[int(round(8192 * a(u) * np.cos((2 * x + 1) * u * np.pi / 16))) for x in range(8)]
                     for u in range(8)], np.int64)


# the constants the CUDA kernel holds as literals (a CPU test checks them against dct_matrix())
DCT_MATRIX = np.array([
    [2896, 2896, 2896, 2896, 2896, 2896, 2896, 2896], [4017, 3406, 2276, 799, -799, -2276, -3406, -4017],
    [3784, 1567, -1567, -3784, -3784, -1567, 1567, 3784], [3406, -799, -4017, -2276, 2276, 4017, 799, -3406],
    [2896, -2896, -2896, 2896, 2896, -2896, -2896, 2896], [2276, -4017, 799, 3406, -3406, -799, 4017, -2276],
    [1567, -3784, 3784, -1567, -1567, 3784, -3784, 1567], [799, -2276, 3406, -4017, 4017, -3406, 2276, -799]],
    np.int64)


def zigzag():
    """Natural index of zigzag position k (T.81 figure A.6)."""
    order = sorted(((y, x) for y in range(8) for x in range(8)),
                   key=lambda p: (p[0] + p[1], p[0] if (p[0] + p[1]) % 2 else p[1]))
    return np.array([y * 8 + x for y, x in order], np.int64)


ZIGZAG = zigzag()


def quant_table(quality):
    q = int(quality)
    if not 1 <= q <= 100:
        raise ValueError("quality must be 1..100, got %r" % (quality,))
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((K1_LUMA * s + 50) // 100, 1, 255)


def huffman_codes(bits, vals):
    """T.81 Annex C: (code, length) of every symbol."""
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


DC_CODES = huffman_codes(DC_BITS, DC_VALS)
AC_CODES = huffman_codes(AC_BITS, AC_VALS)
_AC_CODE = np.zeros(256, np.int64)
_AC_LEN = np.zeros(256, np.int64)
for _s, (_c, _l) in AC_CODES.items():
    _AC_CODE[_s], _AC_LEN[_s] = _c, _l
_DC_CODE = np.array([DC_CODES[c][0] for c in range(12)], np.int64)
_DC_LEN = np.array([DC_CODES[c][1] for c in range(12)], np.int64)


def header(width, height, quality):
    """Everything before the scan: SOI, APP0, DQT, SOF0, DHT x2, DRI, SOS."""
    def seg(marker, body):
        return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + bytes(body)
    q = quant_table(quality)[ZIGZAG]
    out = b"\xff\xd8"
    out += seg(0xE0, b"JFIF\x00" + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0]))
    out += seg(0xDB, bytes([0]) + bytes(int(v) for v in q))
    out += seg(0xC0, bytes([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([1, 1, 0x11, 0]))
    out += seg(0xC4, bytes([0x00] + DC_BITS + DC_VALS))
    out += seg(0xC4, bytes([0x10] + AC_BITS + AC_VALS))
    out += seg(0xDD, (-(-width // 8)).to_bytes(2, "big"))
    out += seg(0xDA, bytes([1, 1, 0x00, 0, 63, 0]))
    return out


def coefficients(frame, quality):
    """Quantised coefficients of every block, [rows, cols, 64] int64 in zigzag order."""
    f = np.asarray(frame)
    if f.dtype != np.uint8 or f.ndim != 2:
        raise ValueError("frame must be uint8 [H, W]")
    H, W = f.shape
    by, bx = -(-H // 8), -(-W // 8)
    p = np.pad(f, ((0, by * 8 - H), (0, bx * 8 - W)), mode="edge").astype(np.int64) - 128
    X = p.reshape(by, 8, bx, 8).transpose(0, 2, 1, 3)               # [by, bx, y, x]
    C = DCT_MATRIX
    T = (np.einsum("abyx,ux->abyu", X, C) + 1024) >> 11
    F = np.einsum("vy,abyu->abvu", C, T).reshape(by, bx, 64)
    D = quant_table(quality) << 15
    c = np.sign(F) * ((np.abs(F) + (D >> 1)) // D)
    c = c[..., ZIGZAG]
    c[..., 1:] = np.clip(c[..., 1:], -1023, 1023)
    return c


def _bit_length(a):
    return (np.abs(a)[..., None] >= (1 << np.arange(12))).sum(-1)


def _value_bits(v, size):
    return np.where(v >= 0, v, v + (1 << size) - 1)


def _row_codes(c):
    """(codes, lengths) of one MCU row's blocks c [n, 64], in stream order."""
    n = c.shape[0]
    dc = c[:, 0]
    diff = dc - np.concatenate([[0], dc[:-1]])
    cat = _bit_length(diff)
    keys = [np.arange(n) * 1024]
    codes = [(_DC_CODE[cat] << cat) | _value_bits(diff, cat)]
    lens = [_DC_LEN[cat] + cat]
    b, k = np.nonzero(c[:, 1:])
    k = k + 1
    if len(b):
        v = c[b, k]
        first = np.concatenate([[True], b[1:] != b[:-1]])
        prev = np.where(first, 0, np.concatenate([[0], k[:-1]]))
        run = k - prev - 1
        size = _bit_length(v)
        sym = ((run & 15) << 4) | size
        keys.append(b * 1024 + k * 8 + 4)
        codes.append((_AC_CODE[sym] << size) | _value_bits(v, size))
        lens.append(_AC_LEN[sym] + size)
        nz = run >> 4                                                 # ZRLs (16 zeros) ahead of the coefficient
        if nz.any():
            i = np.repeat(np.arange(len(b)), nz)
            j = np.arange(len(i)) - np.repeat(np.cumsum(nz) - nz, nz)
            keys.append(b[i] * 1024 + k[i] * 8 + j)
            codes.append(np.full(len(i), _AC_CODE[0xF0]))
            lens.append(np.full(len(i), _AC_LEN[0xF0]))
    last = np.zeros(n, np.int64)
    if len(b):
        last[b] = k                                                   # k is ascending within a block
    e = np.nonzero(last < 63)[0]
    keys.append(e * 1024 + 1000)
    codes.append(np.full(len(e), _AC_CODE[0x00]))
    lens.append(np.full(len(e), _AC_LEN[0x00]))
    order = np.argsort(np.concatenate(keys), kind="stable")
    return np.concatenate(codes)[order], np.concatenate(lens)[order]


def _pack(codes, lens):
    """The row's bits, MSB first, padded with 1-bits to a byte."""
    total = int(lens.sum())
    off = np.cumsum(lens) - lens
    idx = np.repeat(np.arange(len(codes)), lens)
    j = np.arange(total) - off[idx]
    bits = (codes[idx] >> (lens[idx] - 1 - j)) & 1
    bits = np.concatenate([bits, np.ones(-total % 8, np.int64)]).astype(np.uint8)
    return np.packbits(bits).tobytes()


def encode(frame, quality=95):
    """The JPEG bytes of one uint8 [H, W] frame."""
    f = np.asarray(frame)
    c = coefficients(f, quality)
    H, W = f.shape
    out = [header(W, H, quality)]
    for r in range(c.shape[0]):
        out.append(_pack(*_row_codes(c[r])).replace(b"\xff", b"\xff\x00"))
        if r + 1 < c.shape[0]:
            out.append(bytes([0xFF, 0xD0 + (r & 7)]))
    out.append(b"\xff\xd9")
    return b"".join(out)


def luma(bgr):
    """BGR uint8 [..., 3] -> uint8 luma with the pixel pipeline's integer rule (v2e_b200/csrc/prep.cu, cv2's
    BGR2GRAY): (B*3735 + G*19235 + R*9798 + 2^14) >> 15; equal channels give that channel back."""
    x = np.asarray(bgr).astype(np.int64)
    return ((x[..., 0] * 3735 + x[..., 1] * 19235 + x[..., 2] * 9798 + (1 << 14)) >> 15).astype(np.uint8)
