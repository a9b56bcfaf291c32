// Greyscale Motion-JPEG encoder for sm_90a (H100): a batch of uint8 [n][H][W] device frames becomes n baseline JPEGs,
// one after another in one device buffer, with no host work per frame. The format, bit for bit, is DESIGN.md §4.4 and
// oracle/mjpeg_oracle.py. Restart interval = one MCU row, so every row's bitstream is independent:
//   1. mjpeg_dct_kernel    one warp per 8x8 block: level shift, integer DCT, quantise, zigzag; the block's AC bits.
//   2. mjpeg_row_kernel    one CTA per row: the DC differences, a scan of the blocks' bit lengths -> bit offsets;
//                          zeroes the row's words of the bit buffer.
//   3. mjpeg_pack_kernel   one warp per block: every code ORed into the row's bit buffer at its offset; the row's last
//                          block pads the row to a byte with 1-bits.
//   4. mjpeg_count_kernel  one CTA per row: the row's 0xFF bytes -> its stuffed length (+ RST marker).
//   5. mjpeg_scan_kernel   one CTA: a scan over every row of every frame -> each row's output offset, each frame's size.
//   6. mjpeg_write_kernel  one CTA per row: the stuffed bytes, RSTn; the header before row 0, EOI after the last row.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/v2e_b200.h"

int v2e_set_error(int code, const char *fmt, const char *detail);
#define CU(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess) return v2e_set_error(V2E_E_CUDA, #call ": %s", cudaGetErrorString(e_)); \
    } while (0)

namespace {

// a block codes at most 20 DC bits + 63 x (16-bit code + 10 value bits) = 1658 bits < 208 bytes
constexpr int BLOCK_BYTES = 208;
constexpr int BLOCK_WORDS = BLOCK_BYTES / 4;
constexpr int HEADER_BYTES = 334;             // SOI 2, APP0 18, DQT 69, SOF0 13, DHT 33 + 183, DRI 6, SOS 10

// C[u][x] = round(8192 a(u) cos((2x + 1) u pi / 16))
constexpr int16_t kDct[64] = {
    2896, 2896, 2896, 2896, 2896, 2896, 2896, 2896, 4017, 3406, 2276, 799, -799, -2276, -3406, -4017,
    3784, 1567, -1567, -3784, -3784, -1567, 1567, 3784, 3406, -799, -4017, -2276, 2276, 4017, 799, -3406,
    2896, -2896, -2896, 2896, 2896, -2896, -2896, 2896, 2276, -4017, 799, 3406, -3406, -799, 4017, -2276,
    1567, -3784, 3784, -1567, -1567, 3784, -3784, 1567, 799, -2276, 3406, -4017, 4017, -3406, 2276, -799};
// natural index of zigzag position k
constexpr uint8_t kZigzag[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47,
    55, 62, 63};
constexpr uint8_t kK1[64] = {
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51,
    87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101,
    72, 92, 95, 98, 112, 100, 103, 99};
// ITU T.81 K.3 / K.5: code counts per length 1..16, then the symbols
constexpr uint8_t kDcBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
constexpr uint8_t kAcVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
    0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// per-encoder tables in device memory: quantiser divisors (natural order), DCT rows, zigzag, Huffman codes as
// code | length << 16
struct Tables {
    int32_t q[64];
    int32_t dct[64];
    int32_t zz[64];
    uint32_t ac[256];
    uint32_t dc[12];
};

struct Geometry {
    int W, H, nbx, nby;
    int64_t blocks_per_frame;
};

__device__ __forceinline__ int bit_length(int a) { return a ? 32 - __clz(a) : 0; }
__device__ __forceinline__ uint32_t value_bits(int v, int size) { return (uint32_t)(v >= 0 ? v : v + (1 << size) - 1); }

// the code of AC coefficient c at zigzag position k >= 1, after the nonzero mask m of the block's AC positions:
// ZRLs for each 16 zeros of the run, then the run/size symbol and the value bits (at most 3 x 11 + 16 + 10 bits)
__device__ __forceinline__ int ac_code(const Tables &t, int k, int c, uint64_t m, uint64_t &code) {
    const uint64_t below = m & ((1ull << k) - 1);
    const int prev = below ? 63 - __clzll(below) : 0;
    const int run = k - prev - 1, size = bit_length(abs(c));
    const uint32_t zrl = t.ac[0xF0], sym = t.ac[((run & 15) << 4) | size];
    uint64_t v = 0;
    int len = 0;
    for (int r = 0; r < (run >> 4); ++r) {
        v = (v << (zrl >> 16)) | (zrl & 0xFFFF);
        len += zrl >> 16;
    }
    v = (v << (sym >> 16)) | (sym & 0xFFFF);
    v = (v << size) | value_bits(c, size);
    code = v;
    return len + (int)(sym >> 16) + size;
}

__device__ __forceinline__ void block_of(const Geometry &g, int64_t b, int64_t &f, int &by, int &bx) {
    f = b / g.blocks_per_frame;
    const int r = (int)(b - f * g.blocks_per_frame);
    by = r / g.nbx;
    bx = r - by * g.nbx;
}

__global__ void __launch_bounds__(256)
mjpeg_dct_kernel(const uint8_t *__restrict__ frames, Geometry g, int64_t n_blocks, const Tables *__restrict__ tab,
                 int16_t *__restrict__ coef, int32_t *__restrict__ dc, int32_t *__restrict__ ac_bits) {
    __shared__ Tables t;
    __shared__ int32_t xs[8][64], ts[8][64];
    for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 4); i += blockDim.x)
        ((int32_t *)&t)[i] = ((const int32_t *)tab)[i];
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * 8 + w;
    if (b >= n_blocks) return;
    int64_t f;
    int by, bx;
    block_of(g, b, f, by, bx);
    const uint8_t *src = frames + f * g.H * (int64_t)g.W;
    int32_t *X = xs[w], *T = ts[w];
#pragma unroll
    for (int h = 0; h < 2; ++h) {                       // edge padding: the last row / column repeat
        const int i = lane + 32 * h;
        const int y = min(by * 8 + (i >> 3), g.H - 1), x = min(bx * 8 + (i & 7), g.W - 1);
        X[i] = (int)src[(int64_t)y * g.W + x] - 128;
    }
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {                       // rows: T[y][u] = (sum_x C[u][x] X[y][x] + 2^10) >> 11
        const int i = lane + 32 * h, y = i >> 3, u = i & 7;
        int s = 0;
#pragma unroll
        for (int x = 0; x < 8; ++x) s += t.dct[u * 8 + x] * X[y * 8 + x];
        T[i] = (s + 1024) >> 11;
    }
    __syncwarp();
    int c[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {                       // columns, quantised, in zigzag position k
        const int k = lane + 32 * h, i = t.zz[k], v = i >> 3, u = i & 7;
        int s = 0;
#pragma unroll
        for (int y = 0; y < 8; ++y) s += t.dct[v * 8 + y] * T[y * 8 + u];
        const int d = t.q[i] << 15;
        int a = (abs(s) + (d >> 1)) / d;
        if (k) a = min(a, 1023);
        c[h] = s < 0 ? -a : a;
        coef[b * 64 + k] = (int16_t)c[h];
    }
    const uint64_t m = (uint64_t)(__ballot_sync(~0u, c[0] != 0) & ~1u) | ((uint64_t)__ballot_sync(~0u, c[1] != 0) << 32);
    int bits = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int k = lane + 32 * h;
        uint64_t code;
        if (k && c[h]) bits += ac_code(t, k, c[h], m, code);
    }
    bits = __reduce_add_sync(~0u, bits);
    if (lane == 0) {
        dc[b] = c[0];
        ac_bits[b] = bits + (m >> 63 ? 0 : (int)(t.ac[0x00] >> 16));     // EOB unless position 63 is coded
    }
}

// exclusive scan of v over the CTA (blockDim.x a multiple of 32, at most 1024); *total gets the sum
template <typename T>
__device__ __forceinline__ T cta_exclusive_scan(T v, T *warp_sums, T *total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(~0u, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[w] = x;
    __syncthreads();
    if (w == 0) {
        T s = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(~0u, s, o);
            if (lane >= o) s += y;
        }
        if (lane < nw) warp_sums[lane] = s;
    }
    __syncthreads();
    const T before = (w ? warp_sums[w - 1] : 0) + x - v;
    *total = warp_sums[nw - 1];
    __syncthreads();
    return before;
}

__global__ void __launch_bounds__(256)
mjpeg_row_kernel(Geometry g, const int32_t *__restrict__ dc, const int32_t *__restrict__ ac_bits,
                 const Tables *__restrict__ tab, int32_t *__restrict__ bit_off, int32_t *__restrict__ row_bits,
                 uint32_t *__restrict__ words) {
    __shared__ int32_t sums[32];
    const int64_t r = blockIdx.x, b0 = r * g.nbx;        // the row's blocks are consecutive
    int carry = 0;
    for (int j0 = 0; j0 < g.nbx; j0 += blockDim.x) {
        const int j = j0 + threadIdx.x;
        int bits = 0;
        if (j < g.nbx) {
            const int diff = dc[b0 + j] - (j ? dc[b0 + j - 1] : 0);
            const int cat = bit_length(abs(diff));
            bits = ac_bits[b0 + j] + (int)(tab->dc[cat] >> 16) + cat;
        }
        int total;
        const int before = cta_exclusive_scan(bits, sums, &total);
        if (j < g.nbx) bit_off[b0 + j] = carry + before;
        carry += total;
    }
    uint32_t *rw = words + r * g.nbx * BLOCK_WORDS;
    for (int i = threadIdx.x; i < (carry + 31) / 32; i += blockDim.x) rw[i] = 0;
    if (threadIdx.x == 0) row_bits[r] = carry;
}

// ORs the len <= 64 - 31 low bits of code into the big-endian bit stream `words` at bit pos
__device__ __forceinline__ void put_bits(uint32_t *words, int pos, uint64_t code, int len) {
    if (len <= 0) return;
    const int s = pos & 31;
    uint32_t *w = words + (pos >> 5);
    int left = len;                                     // bits of code not yet written
    int room = 32 - s;
    while (left > 0) {
        const int take = min(room, left);
        const uint32_t part = (uint32_t)((code >> (left - take)) & ((1ull << take) - 1));
        const uint32_t word = part << (room - take);
        atomicOr(w, __byte_perm(word, 0, 0x0123));      // stream bytes in address order
        left -= take;
        ++w;
        room = 32;
    }
}

__global__ void __launch_bounds__(256)
mjpeg_pack_kernel(Geometry g, int64_t n_blocks, const int16_t *__restrict__ coef, const int32_t *__restrict__ dc,
                  const Tables *__restrict__ tab, const int32_t *__restrict__ bit_off,
                  const int32_t *__restrict__ row_bits, uint32_t *__restrict__ words) {
    __shared__ Tables t;
    for (int i = threadIdx.x; i < (int)(sizeof(Tables) / 4); i += blockDim.x)
        ((int32_t *)&t)[i] = ((const int32_t *)tab)[i];
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * 8 + w;
    if (b >= n_blocks) return;
    const int64_t r = b / g.nbx;
    const int j = (int)(b - r * g.nbx);
    uint32_t *rw = words + r * g.nbx * BLOCK_WORDS;
    const int c0 = coef[b * 64 + lane], c1 = coef[b * 64 + 32 + lane];
    const uint64_t m = (uint64_t)(__ballot_sync(~0u, c0 != 0) & ~1u) | ((uint64_t)__ballot_sync(~0u, c1 != 0) << 32);
    uint64_t code0 = 0, code1 = 0;
    int len0 = 0, len1 = 0;
    if (lane == 0) {
        const int diff = c0 - (j ? dc[b - 1] : 0);
        const int cat = bit_length(abs(diff));
        code0 = ((uint64_t)(t.dc[cat] & 0xFFFF) << cat) | value_bits(diff, cat);
        len0 = (int)(t.dc[cat] >> 16) + cat;
    } else if (c0) {
        len0 = ac_code(t, lane, c0, m, code0);
    }
    if (c1) len1 = ac_code(t, lane + 32, c1, m, code1);
    // bit offsets: positions 0..31 (lane order), then 32..63
    int x0 = len0, x1 = len1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y0 = __shfl_up_sync(~0u, x0, o), y1 = __shfl_up_sync(~0u, x1, o);
        if (lane >= o) x0 += y0, x1 += y1;
    }
    const int tot0 = __shfl_sync(~0u, x0, 31), tot1 = __shfl_sync(~0u, x1, 31);
    const int base = bit_off[b];
    put_bits(rw, base + x0 - len0, code0, len0);
    put_bits(rw, base + tot0 + x1 - len1, code1, len1);
    if (lane == 31) {
        int end = base + tot0 + tot1;
        if (!(m >> 63)) {                               // EOB
            const uint32_t eob = t.ac[0x00];
            put_bits(rw, end, eob & 0xFFFF, (int)(eob >> 16));
            end += eob >> 16;
        }
        if (j == g.nbx - 1) {                           // the row's end: 1-bits to the byte
            const int pad = (8 - (row_bits[r] & 7)) & 7;
            put_bits(rw, row_bits[r], (1u << pad) - 1, pad);
        }
    }
}

__global__ void __launch_bounds__(256)
mjpeg_count_kernel(Geometry g, const int32_t *__restrict__ row_bits, const uint32_t *__restrict__ words,
                   int32_t *__restrict__ row_len) {
    __shared__ int32_t sums[32];
    const int64_t r = blockIdx.x;
    const int nbytes = (row_bits[r] + 7) >> 3;
    const uint8_t *bytes = (const uint8_t *)(words + r * g.nbx * BLOCK_WORDS);
    int n = 0;
    for (int i = threadIdx.x; i < nbytes; i += blockDim.x) n += bytes[i] == 0xFF;
    int total;
    cta_exclusive_scan(n, sums, &total);
    if (threadIdx.x == 0) row_len[r] = nbytes + total + ((r % g.nby) == g.nby - 1 ? 0 : 2);
}

// one CTA: row_out[r] = where row r's bytes start in the output; sizes[f] = frame f's bytes
__global__ void __launch_bounds__(1024)
mjpeg_scan_kernel(Geometry g, int n_frames, const int32_t *__restrict__ row_len, int64_t *__restrict__ row_out,
                  int64_t *__restrict__ sizes) {
    __shared__ int64_t sums[32];
    const int64_t n_rows = (int64_t)n_frames * g.nby;
    int64_t carry = 0;
    for (int64_t r0 = 0; r0 < n_rows; r0 += blockDim.x) {
        const int64_t r = r0 + threadIdx.x;
        const int64_t v = r < n_rows ? row_len[r] : 0;
        int64_t total;
        const int64_t before = cta_exclusive_scan(v, sums, &total);
        if (r < n_rows) {
            const int64_t f = r / g.nby;
            row_out[r] = carry + before + (f + 1) * HEADER_BYTES + f * 2;
        }
        carry += total;
    }
    __syncthreads();
    for (int f = threadIdx.x; f < n_frames; f += blockDim.x) {
        const int64_t start = row_out[(int64_t)f * g.nby];
        const int64_t end = f + 1 < n_frames ? row_out[(int64_t)(f + 1) * g.nby] - HEADER_BYTES
                                             : carry + (int64_t)n_frames * (HEADER_BYTES + 2);
        sizes[f] = end - start + HEADER_BYTES;
    }
}

__global__ void __launch_bounds__(256)
mjpeg_write_kernel(Geometry g, const int32_t *__restrict__ row_bits, const uint32_t *__restrict__ words,
                   const int64_t *__restrict__ row_out, const uint8_t *__restrict__ header, uint8_t *__restrict__ out) {
    __shared__ int32_t sums[32];
    const int64_t r = blockIdx.x;
    const int y = (int)(r % g.nby);
    const int nbytes = (row_bits[r] + 7) >> 3;
    const uint8_t *bytes = (const uint8_t *)(words + r * g.nbx * BLOCK_WORDS);
    uint8_t *o = out + row_out[r];
    int carry = 0;                                      // 0xFF bytes before this tile
    for (int i0 = 0; i0 < nbytes; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        const uint8_t v = i < nbytes ? bytes[i] : 0;
        int total;
        const int before = cta_exclusive_scan(i < nbytes && v == 0xFF ? 1 : 0, sums, &total);
        if (i < nbytes) {
            o[i + carry + before] = v;
            if (v == 0xFF) o[i + carry + before + 1] = 0x00;
        }
        carry += total;
    }
    if (threadIdx.x == 0) {
        uint8_t *e = o + nbytes + carry;
        e[0] = 0xFF;
        e[1] = y == g.nby - 1 ? 0xD9 : (uint8_t)(0xD0 + (y & 7));     // EOI after the last row, else RSTn
    }
    if (y == 0)
        for (int i = threadIdx.x; i < HEADER_BYTES; i += blockDim.x) o[i - HEADER_BYTES] = header[i];
}

}  // namespace

struct V2eMjpeg {
    Geometry g;
    int max_frames;
    Tables *tables;
    uint8_t *header;
    int16_t *coef;
    int32_t *dc, *ac_bits, *bit_off, *row_bits, *row_len;
    int64_t *row_out;
    uint32_t *words;
};

static int64_t frame_bound(int W, int H) {
    const int64_t nbx = (W + 7) / 8, nby = (H + 7) / 8;
    return HEADER_BYTES + 2 + nby * (2 * nbx * BLOCK_BYTES + 2);   // every byte stuffed, a marker per row
}

static void huffman(const uint8_t *bits, const uint8_t *vals, uint32_t *out) {
    uint32_t code = 0;
    int k = 0;
    for (int len = 1; len <= 16; ++len) {
        for (int i = 0; i < bits[len - 1]; ++i) out[vals[k++]] = code++ | (uint32_t)len << 16;
        code <<= 1;
    }
}

static void build_header(int W, int H, const Tables &t, uint8_t *h) {
    int n = 0;
    auto put = [&](int v) { h[n++] = (uint8_t)v; };
    auto put16 = [&](int v) { put(v >> 8); put(v & 0xFF); };
    put(0xFF); put(0xD8);
    put(0xFF); put(0xE0); put16(16);
    const char jfif[] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    for (char c : jfif) put(c);
    put(0xFF); put(0xDB); put16(67); put(0);
    for (int k = 0; k < 64; ++k) put(t.q[t.zz[k]]);
    put(0xFF); put(0xC0); put16(11); put(8); put16(H); put16(W); put(1); put(1); put(0x11); put(0);
    put(0xFF); put(0xC4); put16(2 + 1 + 16 + 12); put(0x00);
    for (uint8_t v : kDcBits) put(v);
    for (uint8_t v : kDcVals) put(v);
    put(0xFF); put(0xC4); put16(2 + 1 + 16 + 162); put(0x10);
    for (uint8_t v : kAcBits) put(v);
    for (uint8_t v : kAcVals) put(v);
    put(0xFF); put(0xDD); put16(4); put16((W + 7) / 8);
    put(0xFF); put(0xDA); put16(8); put(1); put(1); put(0x00); put(0); put(63); put(0);
}

extern "C" int64_t v2e_mjpeg_bound(int width, int height, int n_frames) {
    if (width < 1 || height < 1 || width > 65535 || height > 65535 || n_frames < 0) return -1;
    return frame_bound(width, height) * n_frames;
}

extern "C" int v2e_mjpeg_destroy(void *handle) {
    V2eMjpeg *e = (V2eMjpeg *)handle;
    if (!e) return V2E_OK;
    void *bufs[] = {e->tables, e->header, e->coef, e->dc, e->ac_bits, e->bit_off, e->row_bits, e->row_len, e->row_out,
                    e->words};
    for (void *b : bufs)
        if (b) cudaFree(b);
    free(e);
    return V2E_OK;
}

extern "C" int v2e_mjpeg_create(int width, int height, int quality, int max_frames, void **handle) {
    if (!handle || width < 1 || height < 1 || width > 65535 || height > 65535 || quality < 1 || quality > 100 ||
        max_frames < 1)
        return v2e_set_error(V2E_E_INVALID, "bad MJPEG encoder arguments%s", "");
    *handle = nullptr;
    V2eMjpeg *e = (V2eMjpeg *)calloc(1, sizeof(V2eMjpeg));
    if (!e) return v2e_set_error(V2E_E_INVALID, "out of host memory%s", "");
    const int nbx = (width + 7) / 8, nby = (height + 7) / 8;
    e->g = Geometry{width, height, nbx, nby, (int64_t)nbx * nby};
    e->max_frames = max_frames;
    const int64_t blocks = e->g.blocks_per_frame * max_frames, rows = (int64_t)nby * max_frames;
    Tables t;
    memset(&t, 0, sizeof t);
    const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int i = 0; i < 64; ++i) {
        const int v = (kK1[i] * s + 50) / 100;
        t.q[i] = v < 1 ? 1 : v > 255 ? 255 : v;
        t.dct[i] = kDct[i];
        t.zz[i] = kZigzag[i];
    }
    huffman(kDcBits, kDcVals, t.dc);
    huffman(kAcBits, kAcVals, t.ac);
    uint8_t hdr[HEADER_BYTES];
    build_header(width, height, t, hdr);
    cudaError_t err = cudaSuccess;
    auto alloc = [&](auto **p, size_t bytes) {
        if (err == cudaSuccess) err = cudaMalloc((void **)p, bytes);
    };
    alloc(&e->tables, sizeof(Tables));
    alloc(&e->header, HEADER_BYTES);
    alloc(&e->coef, blocks * 64 * sizeof(int16_t));
    alloc(&e->dc, blocks * sizeof(int32_t));
    alloc(&e->ac_bits, blocks * sizeof(int32_t));
    alloc(&e->bit_off, blocks * sizeof(int32_t));
    alloc(&e->row_bits, rows * sizeof(int32_t));
    alloc(&e->row_len, rows * sizeof(int32_t));
    alloc(&e->row_out, rows * sizeof(int64_t));
    alloc(&e->words, (size_t)blocks * BLOCK_BYTES);
    if (err == cudaSuccess) err = cudaMemcpy(e->tables, &t, sizeof t, cudaMemcpyHostToDevice);
    if (err == cudaSuccess) err = cudaMemcpy(e->header, hdr, HEADER_BYTES, cudaMemcpyHostToDevice);
    if (err != cudaSuccess) {
        v2e_mjpeg_destroy(e);
        return v2e_set_error(V2E_E_CUDA, "v2e_mjpeg_create: %s", cudaGetErrorString(err));
    }
    *handle = e;
    return V2E_OK;
}

extern "C" int v2e_mjpeg_encode(void *handle, const uint8_t *frames_dev, int n_frames, uint8_t *out_dev,
                                int64_t *sizes_dev, void *stream) {
    V2eMjpeg *e = (V2eMjpeg *)handle;
    if (!e || !frames_dev || !out_dev || !sizes_dev || n_frames < 1)
        return v2e_set_error(V2E_E_INVALID, "bad MJPEG encode arguments%s", "");
    if (n_frames > e->max_frames)
        return v2e_set_error(V2E_E_CAPACITY, "more frames than the encoder was created for%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    const Geometry g = e->g;
    const int64_t blocks = g.blocks_per_frame * n_frames, rows = (int64_t)g.nby * n_frames;
    const unsigned warp_ctas = (unsigned)((blocks + 7) / 8);
    mjpeg_dct_kernel<<<warp_ctas, 256, 0, st>>>(frames_dev, g, blocks, e->tables, e->coef, e->dc, e->ac_bits);
    mjpeg_row_kernel<<<(unsigned)rows, 256, 0, st>>>(g, e->dc, e->ac_bits, e->tables, e->bit_off, e->row_bits, e->words);
    mjpeg_pack_kernel<<<warp_ctas, 256, 0, st>>>(g, blocks, e->coef, e->dc, e->tables, e->bit_off, e->row_bits,
                                                 e->words);
    mjpeg_count_kernel<<<(unsigned)rows, 256, 0, st>>>(g, e->row_bits, e->words, e->row_len);
    mjpeg_scan_kernel<<<1, 1024, 0, st>>>(g, n_frames, e->row_len, e->row_out, sizes_dev);
    mjpeg_write_kernel<<<(unsigned)rows, 256, 0, st>>>(g, e->row_bits, e->words, e->row_out, e->header, out_dev);
    CU(cudaGetLastError());
    return V2E_OK;
}
