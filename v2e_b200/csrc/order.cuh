// Row order of the batched pixel-model path (v2e_emu_set_option option 2) -- included by emu.cu only.
//
// The emit kernels place a row inside its (frame, iteration, polarity) group wherever an atomicAdd put it. With a row
// order set, v2e_emu_collect sorts every segment of the finished step on the device by a key that is a pure function
// of the row, so the result cannot depend on how the rows were produced:
//   PIXEL segments  (canonical: every (frame, iteration, polarity) group; both modes: shot ON, shot OFF):
//       key = polarity bit << 32 | whole-frame pixel index y * W + x
//   RANDOM segments (shuffled: the ON and OFF rows of one (frame, iteration) together):
//       key = words 0, 1 of Philox4x32-7(counter = (2 * pixel + polarity bit, Philox frame index, iteration, "rord"),
//             key = seed), ties broken by 2 * pixel + polarity bit
// Segments and their iteration numbers come from segoff / FrameCtrl, never from timestamps.
//
// Four passes over the rows of a step, all on the caller's stream:
//   setup   (1 block)  segment table from segoff / ctrl, buckets per segment, bucket bases (exclusive scan)
//   count   read row (16 B), key, bucket -> atomicAdd on the bucket's counter
//   scan    (1 block)  exclusive scan of the bucket counters: bucket b of segment s starts at the row its segment
//                      starts at plus the rows of the segment's earlier buckets -- one scan over all buckets of all
//                      segments, because segments are contiguous and in row order
//   scatter read row (16 B), key again, write row + key into the bucket's range of the scratch (24 B)
//   sort    one block per bucket: read rows + keys (24 B), rank every row by counting smaller keys held in shared
//           memory, write it to its final place (16 B, + 8 B key when the caller asked for keys)
// = 96 B of HBM traffic per row. A bucket is a monotone function of the key: pixel / width (width >= 256 pixels, chosen
// so that a segment of n rows has about n / 32 buckets) or the top bits of the uniform key (64 rows expected per
// bucket). A bucket of more than kOrdTile rows (PIXEL segments whose rows crowd into a small part of the frame) takes
// the same code in tiles -- every tile of rows is ranked against every tile of keys -- which is quadratic in the
// bucket but exact.
#pragma once

constexpr int kOrdThreads = 128;
constexpr int kOrdRows = 4;                          // rows per thread and tile
constexpr int kOrdTile = kOrdThreads * kOrdRows;     // keys held in shared memory at a time
constexpr uint32_t kOrdTag = 0x726f7264u;            // "rord": counter word 3 of the ROW_ORDER stream

struct OrdSeg {
    uint32_t start, n;                  // rows [start, start + n) relative to the step's first row
    uint32_t bucket0, nb;               // its buckets are [bucket0, bucket0 + nb)
    uint32_t width;                     // PIXEL: pixels per bucket; 0: RANDOM
    uint32_t frame_index, iter;         // RANDOM: Philox counter words 1, 2
};

__device__ __forceinline__ void ord_key(const EmuDev &d, const OrdSeg &sg, const float4 row, uint64_t &key, uint32_t &bucket) {
    const uint32_t local = (uint32_t)row.z * (uint32_t)d.W + (uint32_t)row.y;      // row = (t, x, y, p)
    const uint32_t pix = d.px_off + local, pol = row.w < 0.0f ? 1u : 0u;
    if (sg.width) {
        key = ((uint64_t)pol << 32) | pix;
        bucket = local / sg.width;
    } else {
        const uint2 k = make_uint2((uint32_t)d.seed, (uint32_t)(d.seed >> 32));
        const uint4 r = philox4x32<kPhiloxRounds>(make_uint4(2u * pix + pol, sg.frame_index, sg.iter, kOrdTag), k);
        key = ((uint64_t)r.x << 32) | r.y;
        bucket = __umulhi(r.x, sg.nb);
    }
}
__device__ __forceinline__ uint32_t ord_id(const EmuDev &d, const float4 row) {
    return 2u * (d.px_off + (uint32_t)row.z * (uint32_t)d.W + (uint32_t)row.y) + (row.w < 0.0f ? 1u : 0u);
}
// last segment whose start is <= r: the one that holds row r (empty segments share their successor's start)
__device__ __forceinline__ int ord_find(const OrdSeg *__restrict__ segs, int S, uint32_t r) {
    int lo = 0, hi = S;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (segs[mid].start <= r) lo = mid; else hi = mid;
    }
    return lo;
}

// exclusive scan over the 1024 threads of a block; *total = the block's sum
__device__ __forceinline__ uint32_t ord_block_scan(uint32_t v, uint32_t *s_warp, uint32_t *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = s_warp[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        s_warp[lane] = wi - w;
        if (lane == 31) s_warp[32] = wi;
    }
    __syncthreads();
    *total = s_warp[32];
    return s_warp[warp] + incl - v;
}

// hdr[0] = segments, hdr[1] = buckets; seg0[f] = first segment of frame f (scratch, [T + 1])
__global__ void __launch_bounds__(1024)
order_setup_kernel(EmuDev d, int T, int mode, const uint32_t *__restrict__ frame_index, uint32_t *seg0, OrdSeg *segs,
                   uint32_t *hdr) {
    __shared__ uint32_t s_warp[33];
    const int tid = threadIdx.x;
    if (tid == 0) {
        uint32_t s = 0;
        for (int f = 0; f < T; f++) {
            seg0[f] = s;
            const uint32_t m = (uint32_t)d.ctrl[f].max_n;
            s += (mode == 1 ? 2u * m : m) + 2u;
        }
        seg0[T] = s;
        hdr[0] = s;
    }
    __syncthreads();
    const uint64_t row0 = d.ctrl[0].ev_base;
    const uint32_t npx = (uint32_t)d.n;
    for (int f = 0; f < T; f++) {
        const FrameCtrl *c = d.ctrl + f;
        const uint32_t *off = d.segoff + (size_t)f * d.seg_stride;
        const int m = c->max_n, nsig = mode == 1 ? 2 * m : m, ns = nsig + 2;
        const uint32_t base = (uint32_t)(c->ev_base - row0), sig_end = off[2 * d.iter_cap];
        for (int j = tid; j < ns; j += blockDim.x) {
            OrdSeg sg;
            uint32_t a, b;
            bool pixel = true;
            if (j < nsig) {
                if (mode == 1) { a = off[j]; b = j + 1 < 2 * m ? off[j + 1] : sig_end; sg.iter = (uint32_t)(j >> 1); }
                else { a = off[2 * j]; b = j + 1 < m ? off[2 * j + 2] : sig_end; sg.iter = (uint32_t)j; pixel = false; }
            } else if (j == nsig) { a = sig_end; b = off[2 * d.iter_cap + 1]; sg.iter = 0; }
            else { a = off[2 * d.iter_cap + 1]; b = c->n_events; sg.iter = 0; }
            const uint32_t n = b - a;
            sg.start = base + a;
            sg.n = n;
            sg.frame_index = frame_index[f];
            sg.bucket0 = 0;
            if (pixel) {
                uint32_t nbp = (n + 31u) / 32u;
                const uint32_t most = (npx + 255u) / 256u;
                if (nbp > most) nbp = most;
                if (nbp < 1u) nbp = 1u;
                sg.width = (npx + nbp - 1u) / nbp;
                sg.nb = n ? (npx + sg.width - 1u) / sg.width : 0u;
            } else {
                sg.width = 0;
                sg.nb = (n + 63u) / 64u;
            }
            segs[seg0[f] + j] = sg;
        }
    }
    __syncthreads();
    const uint32_t S = seg0[T];
    uint32_t run = 0;
    for (uint32_t s0 = 0; s0 < S; s0 += blockDim.x) {
        const uint32_t s = s0 + tid;
        const uint32_t v = s < S ? segs[s].nb : 0u;
        uint32_t tot;
        const uint32_t ex = ord_block_scan(v, s_warp, &tot);
        if (s < S) segs[s].bucket0 = run + ex;
        run += tot;
    }
    if (tid == 0) hdr[1] = run;
}

__global__ void __launch_bounds__(256)
order_count_kernel(EmuDev d, const float4 *__restrict__ rows, uint32_t n_rows, const OrdSeg *__restrict__ segs,
                   const uint32_t *__restrict__ hdr, uint32_t *boff) {
    const uint32_t r = blockIdx.x * 256u + threadIdx.x;
    if (r >= n_rows) return;
    const OrdSeg sg = segs[ord_find(segs, (int)hdr[0], r)];
    uint64_t key;
    uint32_t b;
    ord_key(d, sg, rows[r], key, b);
    atomicAdd(&boff[sg.bucket0 + b], 1u);
}

// in-place exclusive scan of boff[0 .. hdr[1])
__global__ void __launch_bounds__(1024) order_scan_kernel(const uint32_t *__restrict__ hdr, uint32_t *boff) {
    __shared__ uint32_t s_warp[33];
    const uint32_t nb = hdr[1];
    uint32_t run = 0;
    for (uint32_t b0 = 0; b0 < nb; b0 += 4096u) {
        const uint32_t b = b0 + 4u * threadIdx.x;
        uint32_t v[4], sum = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) { v[k] = b + k < nb ? boff[b + k] : 0u; sum += v[k]; }
        uint32_t tot;
        uint32_t ex = run + ord_block_scan(sum, s_warp, &tot);
#pragma unroll
        for (int k = 0; k < 4; k++) { if (b + k < nb) boff[b + k] = ex; ex += v[k]; }
        run += tot;
    }
}

// after this kernel boff[b] is the END of bucket b (its start is the end of bucket b - 1)
__global__ void __launch_bounds__(256)
order_scatter_kernel(EmuDev d, const float4 *__restrict__ rows, uint32_t n_rows, const OrdSeg *__restrict__ segs,
                     const uint32_t *__restrict__ hdr, uint32_t *boff, float4 *__restrict__ tmp_rows,
                     uint64_t *__restrict__ tmp_keys) {
    const uint32_t r = blockIdx.x * 256u + threadIdx.x;
    if (r >= n_rows) return;
    const OrdSeg sg = segs[ord_find(segs, (int)hdr[0], r)];
    const float4 row = rows[r];
    uint64_t key;
    uint32_t b;
    ord_key(d, sg, row, key, b);
    const uint32_t pos = atomicAdd(&boff[sg.bucket0 + b], 1u);
    tmp_rows[pos] = row;
    tmp_keys[pos] = key;
}

__global__ void __launch_bounds__(kOrdThreads)
order_sort_kernel(EmuDev d, const uint32_t *__restrict__ hdr, const uint32_t *__restrict__ boff,
                  const float4 *__restrict__ tmp_rows, const uint64_t *__restrict__ tmp_keys, float4 *__restrict__ rows,
                  uint64_t *__restrict__ keys_out) {
    __shared__ uint64_t s_key[kOrdTile];
    __shared__ uint32_t s_id[kOrdTile];
    const int tid = threadIdx.x;
    const uint32_t nb = hdr[1];
    for (uint32_t b = blockIdx.x; b < nb; b += gridDim.x) {
        const uint32_t start = b ? boff[b - 1] : 0u, n = boff[b] - start;
        for (uint32_t r0 = 0; r0 < n; r0 += kOrdTile) {
            float4 row[kOrdRows];
            uint64_t key[kOrdRows];
            uint32_t id[kOrdRows], rank[kOrdRows];
#pragma unroll
            for (int k = 0; k < kOrdRows; k++) {
                const uint32_t i = r0 + tid + k * kOrdThreads;
                rank[k] = 0;
                if (i < n) {
                    row[k] = tmp_rows[start + i];
                    key[k] = tmp_keys[start + i];
                    id[k] = ord_id(d, row[k]);
                }
            }
            for (uint32_t t0 = 0; t0 < n; t0 += kOrdTile) {
                __syncthreads();
#pragma unroll
                for (int k = 0; k < kOrdRows; k++) {
                    const uint32_t j = t0 + tid + k * kOrdThreads;
                    if (j < n) {
                        if (t0 == r0) { s_key[tid + k * kOrdThreads] = key[k]; s_id[tid + k * kOrdThreads] = id[k]; }
                        else { s_key[tid + k * kOrdThreads] = tmp_keys[start + j]; s_id[tid + k * kOrdThreads] = ord_id(d, tmp_rows[start + j]); }
                    }
                }
                __syncthreads();
                const uint32_t m = n - t0 < (uint32_t)kOrdTile ? n - t0 : (uint32_t)kOrdTile;
#pragma unroll
                for (int k = 0; k < kOrdRows; k++) {
                    if (r0 + tid + k * kOrdThreads < n) {
                        const uint64_t mk = key[k];
                        const uint32_t mi = id[k];
                        uint32_t c = 0;
                        for (uint32_t j = 0; j < m; j++) {
                            const uint64_t o = s_key[j];
                            c += (o < mk || (o == mk && s_id[j] < mi)) ? 1u : 0u;
                        }
                        rank[k] += c;
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < kOrdRows; k++) {
                if (r0 + tid + k * kOrdThreads < n) {
                    rows[start + rank[k]] = row[k];
                    if (keys_out) keys_out[start + rank[k]] = key[k];
                }
            }
        }
    }
}
