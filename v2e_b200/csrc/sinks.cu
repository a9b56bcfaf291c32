// Event-sink row conversions on the device (SURVEY.md 8f rank 3): the packed float32 rows [t, x, y, p] that the
// pixel model emits become what the reference's writers put into files, so that the host copies 8 (AEDAT-2.0),
// 16 (HDF5) or one text line's bytes per event straight into the sink instead of converting row by row on the host.
//
// Replaces (reference = SensorsINI/v2e):
//   v2ecore/emulator.py:953-959              HDF5 "events" dataset rows: uint32 [t_us, x, y, p01]
//   v2ecore/output/aedat2_output.py:133-168  AEDAT-2.0: int32 address / int32 timestamp pairs, big endian; noise
//                                            rows OR in the special-event bit 1 << 10 when labelled
//   v2ecore/output/ae_text_output.py:68-101  DVS text (RPG events.txt) lines 't x y p[ label]\n'
//   v2ecore/emulator.py:889-923              signal / shot-noise labels of the rows (1 = signal, 0 = noise)
// File headers, h5py and the '#'-first-byte check of aedat2_output.py:166-172 stay with the caller.
// A sharded clip's row bands are merged back into the one-GPU row order here too (v2e_merge_bands), so that the file
// is written from device rows.
// The HDF5 and AEDAT-2.0 conversions are pure streaming (16 B read per event): HBM bound, one thread per event.
// The text body takes three launches (DESIGN.md 4.3): line lengths summed per block, one scan of the block sums,
// then each block formats its lines into shared memory and stores its bytes contiguously at the block's offset.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/v2e_b200.h"
#include "shortest_repr.cuh"

extern int v2e_set_error(int code, const char *fmt, const char *detail);

namespace {

// numpy float32 -> uint32 / int32 casts truncate toward zero. Past 2^32 the uint32 value here wraps mod 2^32 (through
// int64); numpy's own result there depends on the array's length (DESIGN.md 2).
__device__ __forceinline__ uint32_t f2u_trunc(float v) { return (uint32_t)(int64_t)v; }

// numpy's float32 -> int32 cast on x86-64: truncation toward zero inside [-2^31, 2^31), INT32_MIN outside it and for
// NaN (cvttss2si's "integer indefinite"). A plain (int32_t) cast compiles to cvt.rzi.s32.f32, which saturates.
__device__ __forceinline__ int32_t f2i_trunc_x86(float v) {
    return (v >= -2147483648.0f && v < 2147483648.0f) ? (int32_t)v : INT32_MIN;
}

__global__ void __launch_bounds__(256) h5_rows_kernel(const float4 *__restrict__ ev, uint64_t n, uint4 *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 e = ev[i];
    // emulator.py:955-958: temp[:,0] *= 1e6 in float32; p == -1 -> 0; astype(uint32)
    const float t_us = __fmul_rn(e.x, 1e6f);
    const float p = e.w == -1.0f ? 0.0f : e.w;
    out[i] = make_uint4(f2u_trunc(t_us), f2u_trunc(e.y), f2u_trunc(e.z), f2u_trunc(p));
}

__global__ void __launch_bounds__(256)
aedat2_kernel(const float4 *__restrict__ ev, const uint8_t *__restrict__ labels, uint64_t n, int size_x, int size_y,
              int xs, int ys, int ps, int flip_x, int flip_y, uint2 *__restrict__ out, unsigned long long *__restrict__ n_on) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int on = 0;
    if (i < n) {
        const float4 e = ev[i];
        const int32_t t = f2i_trunc_x86(__fmul_rn(1e6f, e.x));        // aedat2_output.py:144
        int32_t x = (int32_t)e.y, y = (int32_t)e.z;
        if (flip_x) x = (size_x - 1) - x;                             // :148
        if (flip_y) y = (size_y - 1) - y;                             // :150
        const int32_t p = (int32_t)__fdiv_rn(__fadd_rn(e.w, 1.0f), 2.0f);   // :151
        uint32_t a = ((uint32_t)x << xs) | ((uint32_t)y << ys) | ((uint32_t)p << ps);         // :153
        // :154-158: noise rows set bit 10, also where it overlaps x (640x480: x << 1 reaches bits 1-10)
        if (labels && labels[i] == 0) a |= 1u << 10;
        // address then timestamp, each byte-swapped to big endian (:160-162)
        out[i] = make_uint2(__byte_perm(a, 0, 0x0123), __byte_perm((uint32_t)t, 0, 0x0123));
        on = p != 0;
    }
    if (n_on) {
        const unsigned m = __ballot_sync(0xffffffffu, on);
        if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_on, (unsigned long long)__popc(m));
    }
}

// ---- DVS text body (ae_text_output.py:89-101) ----------------------------------------------------------------------
// Line of row i: '{} {} {} {}\n'.format(float(t), int(x), int(y), int((p + 1) / 2)) with x, y, p cast like numpy's
// astype(np.int32) (truncation) and (p + 1) / 2 evaluated in float32; with labels ' {}'.format(label) before the
// newline. float(t) is repr() of the float32 timestamp widened to double (shortest_repr.cuh).
constexpr int TEXT_ROWS = 256;       // rows per block = threads per block
constexpr int TEXT_LINE_MAX = 64;    // '-' + 17 digits + '.' + 'e-45' = 23, three int32 of 11, label of 3, 4 separators, '\n'

struct TextLine {
    v2e_repr::Repr t;
    int32_t x, y, p, label;          // label < 0: no label column
    int32_t len;
};

__device__ __forceinline__ TextLine text_line(const float4 *__restrict__ ev, const uint8_t *__restrict__ labels, uint64_t i) {
    const float4 e = ev[i];
    TextLine l;
    l.t = v2e_repr::repr_prepare((uint64_t)__double_as_longlong((double)e.x));
    l.x = (int32_t)e.y;
    l.y = (int32_t)e.z;
    l.p = (int32_t)__fdiv_rn(__fadd_rn(e.w, 1.0f), 2.0f);
    l.label = labels ? (int32_t)labels[i] : -1;
    l.len = v2e_repr::repr_length(l.t) + 1 + v2e_repr::int_length(l.x) + 1 + v2e_repr::int_length(l.y) + 1 +
            v2e_repr::int_length(l.p) + (l.label >= 0 ? 1 + v2e_repr::int_length(l.label) : 0) + 1;
    return l;
}

__device__ __forceinline__ void text_write(const TextLine &l, char *dst) {
    int32_t o = v2e_repr::repr_write(l.t, dst);
    dst[o++] = ' ';
    o += v2e_repr::int_write(l.x, dst + o);
    dst[o++] = ' ';
    o += v2e_repr::int_write(l.y, dst + o);
    dst[o++] = ' ';
    o += v2e_repr::int_write(l.p, dst + o);
    if (l.label >= 0) {
        dst[o++] = ' ';
        o += v2e_repr::int_write(l.label, dst + o);
    }
    dst[o] = '\n';
}

// Exclusive prefix sum of v over the block (TEXT_ROWS threads); *total = the block's sum. warp_sums: shared [8].
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *warp_sums, uint32_t *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < TEXT_ROWS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < TEXT_ROWS / 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < TEXT_ROWS / 32) warp_sums[lane] = w;
    }
    __syncthreads();
    *total = warp_sums[TEXT_ROWS / 32 - 1];
    return (warp ? warp_sums[warp - 1] : 0) + x - v;
}

// Pass 1: bytes of each block's lines.
__global__ void __launch_bounds__(TEXT_ROWS)
text_length_kernel(const float4 *__restrict__ ev, const uint8_t *__restrict__ labels, uint64_t n,
                   unsigned long long *__restrict__ block_bytes) {
    __shared__ uint32_t warp_sums[TEXT_ROWS / 32];
    const uint64_t i = (uint64_t)blockIdx.x * TEXT_ROWS + threadIdx.x;
    const uint32_t len = i < n ? (uint32_t)text_line(ev, labels, i).len : 0u;
    uint32_t total;
    block_exclusive_scan(len, warp_sums, &total);
    if (threadIdx.x == 0) block_bytes[blockIdx.x] = total;
}

// Pass 2 (one block of 1024 threads): block_bytes[0, nb) -> exclusive offsets in place, block_bytes[nb] = total.
// Thread k sums a contiguous run of ceil(nb / 1024) entries, the runs are scanned across the block, then each thread
// rewrites its run.
__global__ void __launch_bounds__(1024) text_scan_kernel(unsigned long long *__restrict__ block_bytes, uint64_t nb) {
    __shared__ unsigned long long warp_sums[32];
    const uint64_t per = (nb + 1023) / 1024;
    const uint64_t b0 = min(nb, (uint64_t)threadIdx.x * per), b1 = min(nb, b0 + per);
    unsigned long long s = 0;
    for (uint64_t b = b0; b < b1; ++b) s += block_bytes[b];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = warp_sums[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        warp_sums[lane] = w;
    }
    __syncthreads();
    unsigned long long run = (warp ? warp_sums[warp - 1] : 0ull) + x - s;
    for (uint64_t b = b0; b < b1; ++b) {
        const unsigned long long v = block_bytes[b];
        block_bytes[b] = run;
        run += v;
    }
    if (threadIdx.x == 1023) block_bytes[nb] = run;
}

// Pass 3: each block formats its lines into shared memory at their scanned offsets and stores the block's bytes at
// block_offsets[blockIdx.x], consecutive threads storing consecutive bytes.
__global__ void __launch_bounds__(TEXT_ROWS)
text_write_kernel(const float4 *__restrict__ ev, const uint8_t *__restrict__ labels, uint64_t n,
                  const unsigned long long *__restrict__ block_offsets, uint8_t *__restrict__ out) {
    __shared__ uint32_t warp_sums[TEXT_ROWS / 32];
    __shared__ char stage[TEXT_ROWS * TEXT_LINE_MAX];
    const uint64_t i = (uint64_t)blockIdx.x * TEXT_ROWS + threadIdx.x;
    TextLine l;
    l.len = 0;
    if (i < n) l = text_line(ev, labels, i);
    uint32_t total;
    const uint32_t at = block_exclusive_scan((uint32_t)l.len, warp_sums, &total);
    if (i < n) text_write(l, stage + at);
    __syncthreads();
    uint8_t *dst = out + block_offsets[blockIdx.x];
    for (uint32_t k = threadIdx.x; k < total; k += TEXT_ROWS) dst[k] = (uint8_t)stage[k];
}

// ---- signal / noise labels (emulator.py:889-923) ---------------------------------------------------------------------
// Row i of frame f (offsets[f] <= i < offsets[f + 1]) is shot noise (0) when it is one of the frame's last n_noise[f]
// rows, signal (1) otherwise.
__global__ void __launch_bounds__(256)
signnoise_labels_kernel(const int64_t *__restrict__ offsets, const uint32_t *__restrict__ n_noise, int n_frames,
                        uint64_t n, uint8_t *__restrict__ labels) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int lo = 0, hi = n_frames - 1;           // the last frame f with offsets[f] <= i
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((uint64_t)offsets[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    labels[i] = i < (uint64_t)offsets[lo + 1] - n_noise[lo] ? 1 : 0;
}

// ---- merge of a sharded clip's row bands (v2e_b200.parallel.merge_by_key) -------------------------------------------
// Per frame the merged stream holds every band's signal rows by (t, key, y, x, p < 0), then every band's shot rows by
// (key, y, x, p < 0); equal tuples keep band order. Each band's frame segment is already sorted that way (a band orders
// its signal rows strictly by (t, key) and its shot rows by key), so a row's place is a co-rank: its index in its own
// segment plus, for every other band, how many rows of that band's segment of the same frame and class precede it --
// one binary search per other band. One thread per row; the rows are scattered to their places (DESIGN.md 4.3).
// bo: [n_bands][n_frames + 1] absolute row offsets of the bands' frames; shot: [n_bands][n_frames].
struct MergeRow {
    float4 e;
    uint64_t key;
};

// a before b in the merged order of one frame's signal (or, ignoring t, shot) rows
__device__ __forceinline__ bool merge_less(const MergeRow &a, const MergeRow &b, bool shot) {
    if (!shot && a.e.x != b.e.x) return a.e.x < b.e.x;
    if (a.key != b.key) return a.key < b.key;
    if (a.e.z != b.e.z) return a.e.z < b.e.z;
    if (a.e.y != b.e.y) return a.e.y < b.e.y;
    return (a.e.w < 0.0f) < (b.e.w < 0.0f);
}

__global__ void __launch_bounds__(256) merge_offsets_kernel(const int64_t *__restrict__ bo, int n_bands, int n_frames,
                                                            int64_t *__restrict__ out_offsets) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f > n_frames) return;
    int64_t s = 0;
    for (int q = 0; q < n_bands; ++q) s += bo[(int64_t)q * (n_frames + 1) + f] - bo[(int64_t)q * (n_frames + 1)];
    out_offsets[f] = s;
}

__global__ void __launch_bounds__(256)
merge_bands_kernel(const float4 *__restrict__ rows, const uint64_t *__restrict__ keys, uint64_t n, int n_bands,
                   int n_frames, const int64_t *__restrict__ bo, const int64_t *__restrict__ shot,
                   float4 *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t stride = n_frames + 1;
    int r = 0;                                   // the band holding row i (empty bands hold none)
    while ((uint64_t)bo[r * stride + n_frames] <= i) ++r;
    const int64_t *o = bo + r * stride;
    int lo = 0, hi = n_frames - 1;               // the last frame f with o[f] <= i
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((uint64_t)o[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    const int f = lo;
    const int64_t s_r = o[f + 1] - shot[r * n_frames + f];
    const bool is_shot = (int64_t)i >= s_r;
    const MergeRow me{rows[i], keys[i]};
    int64_t pos = (int64_t)i - (is_shot ? s_r : o[f]);
    for (int q = 0; q < n_bands; ++q) {
        const int64_t *oq = bo + q * stride;
        const int64_t sq = oq[f + 1] - shot[q * n_frames + f];
        pos += oq[f] - oq[0];                                    // the merged frame's first row
        if (is_shot) pos += sq - oq[f];                          // after every band's signal rows of the frame
        if (q == r) continue;
        // rows of band q's segment before me: strictly smaller ones, and equal ones of an earlier band
        int64_t a = is_shot ? sq : oq[f], b = is_shot ? oq[f + 1] : sq;
        while (a < b) {
            const int64_t mid = a + ((b - a) >> 1);
            const MergeRow other{rows[mid], keys[mid]};
            const bool before = q < r ? !merge_less(me, other, is_shot) : merge_less(other, me, is_shot);
            if (before) a = mid + 1;
            else b = mid;
        }
        pos += a - (is_shot ? sq : oq[f]);
    }
    out[pos] = me.e;
}

}  // namespace

extern "C" int v2e_events_to_h5_rows(const float *events_dev, uint64_t n, uint32_t *rows_dev, void *stream) {
    if (n == 0) return V2E_OK;
    if (!events_dev || !rows_dev) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    if (((uintptr_t)events_dev | (uintptr_t)rows_dev) & 15) return v2e_set_error(V2E_E_INVALID, "buffers must be 16-byte aligned%s", "");
    const uint64_t blocks = (n + 255) / 256;
    if (blocks > 0x7fffffffull) return v2e_set_error(V2E_E_INVALID, "too many events for one call%s", "");
    h5_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const float4 *)events_dev, n, (uint4 *)rows_dev);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "h5_rows_kernel: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_events_to_aedat2(const float *events_dev, uint64_t n, int size_x, int size_y, int x_shift,
                                    int y_shift, int pol_shift, int flip_x, int flip_y, const uint8_t *labels_dev,
                                    uint32_t *words_dev, uint64_t *n_on_dev, void *stream) {
    if (n == 0) return V2E_OK;
    if (!events_dev || !words_dev) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    if (((uintptr_t)events_dev & 15) || ((uintptr_t)words_dev & 7)) return v2e_set_error(V2E_E_INVALID, "misaligned buffer%s", "");
    if (x_shift < 0 || y_shift < 0 || pol_shift < 0 || x_shift > 31 || y_shift > 31 || pol_shift > 31)
        return v2e_set_error(V2E_E_INVALID, "bad shift%s", "");
    const uint64_t blocks = (n + 255) / 256;
    if (blocks > 0x7fffffffull) return v2e_set_error(V2E_E_INVALID, "too many events for one call%s", "");
    aedat2_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const float4 *)events_dev, labels_dev, n, size_x,
                                                                       size_y, x_shift, y_shift, pol_shift, flip_x, flip_y,
                                                                       (uint2 *)words_dev, (unsigned long long *)n_on_dev);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "aedat2_kernel: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" uint64_t v2e_events_to_text_scratch(uint64_t n) { return (n + TEXT_ROWS - 1) / TEXT_ROWS + 1; }

extern "C" int v2e_events_to_text_layout(const float *events_dev, uint64_t n, const uint8_t *labels_dev,
                                         uint64_t *block_offsets_dev, void *stream) {
    if (!block_offsets_dev) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    const uint64_t nb = (n + TEXT_ROWS - 1) / TEXT_ROWS;
    if (nb > 0x7fffffffull) return v2e_set_error(V2E_E_INVALID, "too many events for one call%s", "");
    if (n && !events_dev) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    if ((uintptr_t)events_dev & 15) return v2e_set_error(V2E_E_INVALID, "events must be 16-byte aligned%s", "");
    if ((uintptr_t)block_offsets_dev & 7) return v2e_set_error(V2E_E_INVALID, "misaligned block offsets%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long *bo = (unsigned long long *)block_offsets_dev;
    if (nb) text_length_kernel<<<(unsigned)nb, TEXT_ROWS, 0, st>>>((const float4 *)events_dev, labels_dev, n, bo);
    text_scan_kernel<<<1, 1024, 0, st>>>(bo, nb);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "text layout: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_events_to_text(const float *events_dev, uint64_t n, const uint8_t *labels_dev,
                                  const uint64_t *block_offsets_dev, uint8_t *text_dev, void *stream) {
    if (n == 0) return V2E_OK;
    if (!events_dev || !block_offsets_dev || !text_dev) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    const uint64_t nb = (n + TEXT_ROWS - 1) / TEXT_ROWS;
    if (nb > 0x7fffffffull) return v2e_set_error(V2E_E_INVALID, "too many events for one call%s", "");
    if ((uintptr_t)events_dev & 15) return v2e_set_error(V2E_E_INVALID, "events must be 16-byte aligned%s", "");
    text_write_kernel<<<(unsigned)nb, TEXT_ROWS, 0, (cudaStream_t)stream>>>(
        (const float4 *)events_dev, labels_dev, n, (const unsigned long long *)block_offsets_dev, text_dev);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "text_write_kernel: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_signnoise_labels(const int64_t *offsets_dev, const uint32_t *n_noise_dev, int n_frames,
                                    uint64_t n_rows, uint8_t *labels_dev, void *stream) {
    if (n_rows == 0) return V2E_OK;
    if (!offsets_dev || !n_noise_dev || !labels_dev || n_frames < 1)
        return v2e_set_error(V2E_E_INVALID, "null argument or no frames%s", "");
    const uint64_t blocks = (n_rows + 255) / 256;
    if (blocks > 0x7fffffffull) return v2e_set_error(V2E_E_INVALID, "too many events for one call%s", "");
    signnoise_labels_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(offsets_dev, n_noise_dev, n_frames,
                                                                                n_rows, labels_dev);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "signnoise_labels_kernel: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_merge_bands(const float *rows_dev, const uint64_t *keys_dev, uint64_t n, int n_bands, int n_frames,
                               const int64_t *band_offsets_dev, const int64_t *n_shot_dev, float *out_rows_dev,
                               int64_t *out_offsets_dev, void *stream) {
    if (n_bands < 1 || n_frames < 0 || !band_offsets_dev || !out_offsets_dev || (n_frames && !n_shot_dev))
        return v2e_set_error(V2E_E_INVALID, "bad band / frame counts or null argument%s", "");
    if (n && (!rows_dev || !keys_dev || !out_rows_dev || n_frames < 1))
        return v2e_set_error(V2E_E_INVALID, "null argument or no frames%s", "");
    if (((uintptr_t)rows_dev | (uintptr_t)out_rows_dev) & 15) return v2e_set_error(V2E_E_INVALID, "rows must be 16-byte aligned%s", "");
    if (((uintptr_t)keys_dev | (uintptr_t)band_offsets_dev | (uintptr_t)n_shot_dev | (uintptr_t)out_offsets_dev) & 7)
        return v2e_set_error(V2E_E_INVALID, "misaligned keys or offsets%s", "");
    const uint64_t blocks = (n + 255) / 256;
    if (blocks > 0x7fffffffull) return v2e_set_error(V2E_E_INVALID, "too many events for one call%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    merge_offsets_kernel<<<(n_frames + 256) / 256, 256, 0, st>>>(band_offsets_dev, n_bands, n_frames, out_offsets_dev);
    if (n)
        merge_bands_kernel<<<(unsigned)blocks, 256, 0, st>>>((const float4 *)rows_dev, keys_dev, n, n_bands, n_frames,
                                                             band_offsets_dev, n_shot_dev, (float4 *)out_rows_dev);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "merge_bands_kernel: %s", cudaGetErrorString(e));
    return V2E_OK;
}
