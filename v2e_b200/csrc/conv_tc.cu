// Implicit-GEMM convolution + bias + LeakyReLU on the Hopper tensor cores (sm_90a, wgmma).
//
// Replaces the 23 conv2d+leaky_relu pairs of the reference's UNet (v2ecore/model.py:10-226, called
// from v2ecore/slomo.py:343, 415-419), which the reference runs as stock cuDNN kernels.
//
//   D[pixel, cout] = sum_{tap=(r,s)} sum_{c} X[n, y+r-ph, x+s-pw, c] * Wt[cout, tap, c]      (+bias, lrelu)
//
// Layout: activations NHWC fp16 (C padded to a multiple of 16), weights [Cout_pad][KH*KW*Ctot] fp16
// (K index = tap*Ctot + c), accumulation fp32 in registers.
// One CTA computes a 128-pixel (8 rows x 16 columns) x BN-channel output tile:
//   warp 8      : TMA producer. For every filter tap and every KC-channel slab it issues one 4-D tiled
//                 load of the *shifted* 8x16 window (cp.async.bulk.tensor, 128B/64B/32B swizzle) --
//                 out-of-bounds rows/columns are zero-filled by TMA, which is exactly the conv's zero
//                 padding, so no im2col buffer and no halo logic -- plus one 2-D load of the BN x KC
//                 weight slab. A concatenated input (up-blocks: cat(x, skip), model.py:150-153) is
//                 read from two tensor maps, so the concat is never materialised.
//   warps 0..7  : two consumer warpgroups; warpgroup g issues wgmma (M=64, N=BN, K=16) for pixels
//                 64g..64g+63 of the tile from the swizzled shared-memory stages, keeps one stage of MMAs
//                 in flight, releases the stage before it, and finally applies bias + LeakyReLU(0.1) and
//                 stores NHWC (fp16) or the first channels as fp32 (network outputs) from its registers.
// Pipeline: a kStages-deep mbarrier ring between the producer and the two warpgroups.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "../../include/v2e_b200.h"
#include "common.cuh"
#include "tc_common.cuh"

namespace {

constexpr int kTileH = 8, kTileW = 16, kBM = kTileH * kTileW;   // 128 pixels = two wgmma M = 64 halves
constexpr int kStages = 4;
constexpr int kConvThreads = 288;      // warps 0..3 and 4..7: consumer warpgroups, warp 8: TMA producer
constexpr int kProducerWarp = 8;
constexpr int kConsumerWarps = 8;      // every consumer warp arrives once on an empty barrier

struct ConvParams {
    int N, H, W;
    int C1, C2;                 // padded channel counts of the two inputs (C2 = 0: single input)
    int KH, KW;
    int KC;                     // channels per K slab: 64 / 32 / 16  -> swizzle 128B / 64B / 32B
    int BN;                     // output channels per CTA (wgmma N)
    int stages;                 // depth of the producer / consumer ring (<= kStages)
    int co_fast;                // grid order: 1 = output-channel blocks in gridDim.x
    int tiles_x, tiles_y;
    int n_tiles;                // pixel tiles
    int out_cstride;            // channel stride (elements) of the fp16 NHWC output
    int out_mode;               // 0: fp16 NHWC; 1: fp32 [N,H,W,8], first co_real channels
    int co_real;
    float slope;
    const float *bias;          // [Cout_pad]
    void *out;
};

__device__ __forceinline__ uint8_t *align1024(uint8_t *p) { return (uint8_t *)(((uintptr_t)p + 1023) & ~(uintptr_t)1023); }

__device__ __forceinline__ float lrelu(float x, float slope) { return x > 0.f ? x : x * slope; }

// Row i (0 / 1) of this thread's share of a 64 x BN accumulator (layout: tc_common.cuh, wgmma): bias, LeakyReLU and
// the store of output pixel `pix`. out_mode 0: fp16, channels co0 + column at stride cstride; 1: fp32 [.., 8], the
// first 8 columns. The fp16 values are returned in h (for the pooled epilogue).
template <int BN>
__device__ __forceinline__ void epilogue_row(const float (&d)[BN / 2], int i, bool inb, size_t pix, int lane,
                                             const float *bias, float slope, int out_mode, void *out, int cstride,
                                             int co0, __half2 (&h)[BN / 8]) {
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const int c = 8 * j + 2 * (lane & 3);
        const float x0 = lrelu(d[4 * j + 2 * i] + __ldg(bias + c), slope);
        const float x1 = lrelu(d[4 * j + 2 * i + 1] + __ldg(bias + c + 1), slope);
        h[j] = __floats2half2_rn(x0, x1);
        if (inb) {
            if (out_mode == 0) *(__half2 *)((__half *)out + pix * cstride + co0 + c) = h[j];
            else if (j == 0) *(float2 *)((float *)out + pix * 8 + c) = make_float2(x0, x1);
        }
    }
}

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmB, const ConvParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // carve: stages of [A 128 x KC fp16][B BN x KC fp16], 1024-byte aligned
    uint8_t *smem = align1024(smem_raw);
    const uint32_t a_bytes = kBM * p.KC * 2;
    const uint32_t b_bytes_raw = BN * p.KC * 2;
    const uint32_t b_bytes = (b_bytes_raw + 1023) & ~1023u;
    const uint32_t stage_bytes = a_bytes + b_bytes;
    __shared__ __align__(8) uint64_t full_bar[kStages], empty_bar[kStages];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // output-channel block fastest (gridDim.x when p.co_fast): the CTAs that share an input window run together, so
    // the window comes from DRAM once and from L2 for its siblings
    const int tile = p.co_fast ? blockIdx.y : blockIdx.x;
    const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, n = tile / (p.tiles_x * p.tiles_y);
    const int x0 = tx * kTileW, y0 = ty * kTileH;
    const int n0 = (p.co_fast ? blockIdx.x : blockIdx.y) * BN;
    const int Ctot = p.C1 + p.C2;
    const int slabs = Ctot / p.KC;
    const int k_iters = p.KH * p.KW * slabs;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        fence_barrier_init();
    }
    if (warp == kProducerWarp && lane == 0) {
        prefetch_tmap(&tmA);
        if (p.C2) prefetch_tmap(&tmA2);
        prefetch_tmap(&tmB);
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ===== TMA producer =====
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            const int ph = p.KH / 2, pw = p.KW / 2;
            for (int tap = 0; tap < p.KH * p.KW; tap++) {
                const int r = tap / p.KW, s = tap % p.KW;
                for (int sl = 0; sl < slabs; sl++) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t *sa = smem + stage * stage_bytes, *sb = sa + a_bytes;
                    mbar_expect_tx(&full_bar[stage], a_bytes + b_bytes_raw);
                    const int c = sl * p.KC;
                    if (c < p.C1) tma_load_4d(sa, &tmA, &full_bar[stage], c, x0 + s - pw, y0 + r - ph, n);
                    else tma_load_4d(sa, &tmA2, &full_bar[stage], c - p.C1, x0 + s - pw, y0 + r - ph, n);
                    tma_load_2d(sb, &tmB, &full_bar[stage], tap * Ctot + c, n0);
                    if (++stage == p.stages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===== consumer warpgroup g: pixels 64g .. 64g+63 of the tile =====
        const int g = warp >> 2;
        const uint64_t d0 = make_smem_desc(smem_u32(smem), swizzle_layout(p.KC), 8u * p.KC * 2u);
        const uint32_t stage16 = stage_bytes >> 4, a16 = a_bytes >> 4, half16 = (64u * p.KC * 2u) >> 4;
        const int ksteps = p.KC / 16;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int it = 0; it < k_iters; it++) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t base = (uint32_t)stage * stage16;
            wgmma_fence();
            for (int j = 0; j < ksteps; j++)
                wgmma_f16<BN>(acc, desc_add(d0, base + (uint32_t)g * half16 + 2u * j), desc_add(d0, base + a16 + 2u * j),
                              (uint32_t)((it | j) != 0));
            wgmma_commit();
            wgmma_wait<1>();                 // the stage before this one has been read: hand it back
            if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
            prev = stage;
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        __half2 hv[BN / 8];
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int m = 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * i;
            const int py = y0 + m / kTileW, px = x0 + m % kTileW;
            const bool inb = py < p.H && px < p.W;
            const size_t pix = ((size_t)n * p.H + py) * p.W + px;
            epilogue_row<BN>(acc, i, inb, pix, lane, p.bias + n0, p.slope, p.out_mode, p.out, p.out_cstride, n0, hv);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Wide per-tap kernel: conv_tc_kernel's producer / two-consumer structure with 128 fp32 accumulators per consumer
// thread, so that every (tap, slab) stage feeds twice the MMAs of the 128 x 128 tile. The tile is
//   MH = 1: 128 pixels (8x16) x BN = 256 channels; a warpgroup runs one m64n256 chain over its 64 pixels,
//   MH = 2: 256 pixels (16x16) x BN = 128 channels; a warpgroup runs two m64n128 chains (its two 64-pixel quarters)
//           over the same B slab.
// Every output element accumulates its terms in the order (tap, slab, k16) of conv_tc_kernel.
// ---------------------------------------------------------------------------------------------
template <int MH, int BN>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmB, const ConvParams p) {
    constexpr int TH = kTileH * MH, BM = kBM * MH;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = align1024(smem_raw);
    const uint32_t a_bytes = BM * p.KC * 2;
    const uint32_t b_bytes = BN * p.KC * 2;           // a multiple of 1024 (BN >= 128, KC >= 16)
    const uint32_t stage_bytes = a_bytes + b_bytes;
    __shared__ __align__(8) uint64_t full_bar[kStages], empty_bar[kStages];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = p.co_fast ? blockIdx.y : blockIdx.x;
    const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, n = tile / (p.tiles_x * p.tiles_y);
    const int x0 = tx * kTileW, y0 = ty * TH;
    const int n0 = (p.co_fast ? blockIdx.x : blockIdx.y) * BN;
    const int Ctot = p.C1 + p.C2;
    const int slabs = Ctot / p.KC;
    const int k_iters = p.KH * p.KW * slabs;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        fence_barrier_init();
    }
    if (warp == kProducerWarp && lane == 0) {
        prefetch_tmap(&tmA);
        if (p.C2) prefetch_tmap(&tmA2);
        prefetch_tmap(&tmB);
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ===== TMA producer =====
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            const int ph = p.KH / 2, pw = p.KW / 2;
            for (int tap = 0; tap < p.KH * p.KW; tap++) {
                const int r = tap / p.KW, s = tap % p.KW;
                for (int sl = 0; sl < slabs; sl++) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t *sa = smem + stage * stage_bytes, *sb = sa + a_bytes;
                    mbar_expect_tx(&full_bar[stage], a_bytes + b_bytes);
                    const int c = sl * p.KC;
                    if (c < p.C1) tma_load_4d(sa, &tmA, &full_bar[stage], c, x0 + s - pw, y0 + r - ph, n);
                    else tma_load_4d(sa, &tmA2, &full_bar[stage], c - p.C1, x0 + s - pw, y0 + r - ph, n);
                    tma_load_2d(sb, &tmB, &full_bar[stage], tap * Ctot + c, n0);
                    if (++stage == p.stages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===== consumer warpgroup g: pixels BM/2 * g .. BM/2 * (g+1) - 1 of the tile, MH 64-pixel quarters =====
        const int g = __shfl_sync(0xffffffffu, warp >> 2, 0);       // warp-uniform to ptxas (see strip_pair_mma)
        const uint64_t d0 = make_smem_desc(smem_u32(smem), swizzle_layout(p.KC), 8u * p.KC * 2u);
        const uint32_t stage16 = stage_bytes >> 4, a16 = a_bytes >> 4, q16 = (64u * p.KC * 2u) >> 4;
        const int ksteps = p.KC / 16;
        float acc[MH][BN / 2];
#pragma unroll
        for (int h = 0; h < MH; h++) {
#pragma unroll
            for (int i = 0; i < BN / 2; i++) acc[h][i] = 0.f;
            wgmma_fence_regs(acc[h]);
        }
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int it = 0; it < k_iters; it++) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t base = (uint32_t)stage * stage16;
            wgmma_fence();
            for (int j = 0; j < ksteps; j++) {
#pragma unroll
                for (int h = 0; h < MH; h++)
                    wgmma_f16<BN>(acc[h], desc_add(d0, base + (uint32_t)(g * MH + h) * q16 + 2u * j),
                                  desc_add(d0, base + a16 + 2u * j), (uint32_t)((it | j) != 0));
            }
            wgmma_commit();
            wgmma_wait<1>();                 // the stage before this one has been read: hand it back
            if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
            prev = stage;
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < MH; h++) wgmma_fence_regs(acc[h]);
        // bias + LeakyReLU + fp16 store of both rows of each 8-column group at once (one bias load per group keeps the
        // 128 accumulators and the addresses within the register budget)
        const float *bias = p.bias + n0;
        __half *out = (__half *)p.out + n0;
#pragma unroll
        for (int h = 0; h < MH; h++) {
            size_t pix[2];
            bool inb[2];
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int m = 64 * (g * MH + h) + 16 * (warp & 3) + (lane >> 2) + 8 * i;
                const int py = y0 + m / kTileW, px = x0 + m % kTileW;
                inb[i] = py < p.H && px < p.W;
                pix[i] = (((size_t)n * p.H + py) * p.W + px) * p.out_cstride;
            }
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
                const int c = 8 * j + 2 * (lane & 3);
                const float2 b = __ldg((const float2 *)(bias + c));
#pragma unroll
                for (int i = 0; i < 2; i++)
                    if (inb[i])
                        *(__half2 *)(out + pix[i] + c) = __floats2half2_rn(lrelu(acc[h][4 * j + 2 * i] + b.x, p.slope),
                                                                           lrelu(acc[h][4 * j + 2 * i + 1] + b.y, p.slope));
            }
        }
    }
}


constexpr int kRowTile = 128;

// ---------------------------------------------------------------------------------------------
// Strip kernel: the full-resolution layers (Cout_pad <= 64, 7x7 / 5x5 / 3x3) that dominate the UNet.
// A CTA walks down a 128-pixel-wide column strip. The layer's weights (or the slice of the output channels
// this CTA class computes) stay resident in shared memory; input rows live in a ring of NSLOT row buffers
// ([128+KW-1 pixels] x KC channels per slab, TMA-swizzled). Moving one output row down costs ONE new input
// row from L2 (instead of KH rows with a per-tile halo, or KH*KW windows with per-tap loads); every filter
// tap (r, s) is a descriptor offset: ring slot of input row y+r-ph, start + s pixels.
//   warp 8     : TMA producer: the weights once per CTA, then one row (all slabs) per ring slot.
//   warps 0..7 : two consumer warpgroups, taking turns over PAIRS of output rows of an item (warpgroup g:
//                pairs g, g+2, ...). Per 64-pixel half of the strip, the pair's wgmmas are one asynchronous chain
//                over the KH+1 input rows: two of M = 64, N = BN per input row (strip_pair_mma), or, with the
//                weight tiles stacked in shared memory (STACK), one of N = 2 * BN (strip_stack_mma); then bias,
//                LeakyReLU and the store. A ring slot is released by both warpgroups (every row of the item exactly
//                once each) when neither needs it any more.
// POOL: F.avg_pool2d(out, 2) written beside the output (model.py:71: the pool that opens a down block). A pair
// is rows (2k, 2k+1) of the item (items start on even rows), so both rows of a 2x2 window are in the same
// registers; the horizontal neighbour is the lane 4 apart.
// ---------------------------------------------------------------------------------------------
struct StripParams {
    int N, H, W;
    int C1, C2;
    int KH, KW;
    int KC, BN;
    int tiles_x, seg_h, n_seg, n_items;
    int nslot;
    void *pool_out;                // POOL: [N, H/2, W/2, pool_cstride] fp16
    int pool_cstride;
    int n_split, cout_pad;         // output channels split over n_split CTA classes of BN = cout_pad / n_split
                                   // (layers whose whole weight tensor does not fit in shared memory)
    int slab_bytes;                // bytes of one row buffer of one slab (1024-aligned)
    int w_bytes;                   // resident weights
    int out_cstride, out_mode, co_real;
    float slope;
    const float *bias;
    void *out;
};
constexpr int kMaxSlot = 12;
constexpr int kStripThreads = 288;      // warps 0..3 and 4..7: consumer warpgroups, warp 8: TMA producer

// Ring bookkeeping of one consumer warpgroup over the input rows of one item: rows are waited for in order and
// released in order, each exactly once (a slot's empty barrier counts the arrivals of all eight consumer warps).
struct RowRing {
    uint64_t *full, *empty;
    uint32_t nslot, cnt;           // cnt: ring rows filled before this item (all items)
    int waited, released;
    __device__ __forceinline__ uint32_t slot(int i) const { return (cnt + (uint32_t)i) % nslot; }
    __device__ __forceinline__ void wait_upto(int n) {
        for (; waited < n; waited++) {
            const uint32_t g = cnt + (uint32_t)waited;
            mbar_wait(&full[g % nslot], (g / nslot) & 1u);
        }
    }
    // every wgmma that read rows < n has completed (wgmma_wait) before this is called
    __device__ __forceinline__ void release_upto(int n, int lane) {
        wait_upto(n);              // observe every fill, so that a later wait on the slot cannot alias this phase
        __syncwarp();
        for (; released < n; released++)
            if (lane == 0) mbar_arrive(&empty[slot(released)]);
    }
};

// The wgmmas of input rows row0+rp0 .. row0+rp1-1 for output rows (row0, row0+1) of a strip item over one 64-pixel
// half (a_off: its start in a row buffer); the caller zeroes the accumulators, fences and commits, so that a pair's
// chain can be committed in several groups (conv_strip_kernel). Input row row0+r' (r' = 0..KH) feeds row0 with tap r'
// and row0+1 with tap r'-1, so the two rows' MMAs interleave in one chain over the KH+1 input rows. An odd last row of
// an item has no input row row0+KH in the ring: last = KH-1 reads row row0+KH-1 in its place, and the epilogue drops
// the row row0+1 this makes. Every output element accumulates its terms in the order (r, slab, s, channel).
// The accumulators are zeroed before the fence and never copied inside the chain: a register move that ptxas places
// between two wgmmas (zeroing sunk past the fence, a path that skips a loop, accumulators merged from two code
// paths, or one accumulator used by wgmmas of two widths) makes it wait for each wgmma before the next. Hence the
// zeroing pinned by wgmma_fence_regs, the slab loop that runs at least once and is never unrolled (its remainder
// would be a second path), and one code path for both row counts.
template <int KW, int KC, int BN>
__device__ __forceinline__ void strip_pair_mma(float (&acc)[2][BN / 2], const RowRing &rr, int row0, int last, int slabs,
                                                uint64_t dr, uint64_t dw, uint32_t a_off, uint32_t row16, uint32_t slab16,
                                                int rp0, int rp1) {
    constexpr int KH = KW, taps = KH * KW;
    constexpr uint32_t rowb16 = (KC * 2u) >> 4, tile16 = (BN * KC * 2u) >> 4;
#pragma unroll
    for (int rp = rp0; rp < rp1; rp++) {
        const uint32_t a_row = rr.slot(row0 + (rp < KH ? rp : last)) * row16 + a_off;
        int sl = 0;
#pragma unroll 1
        do {
            const uint32_t a_lo = a_row + (uint32_t)sl * slab16;
#pragma unroll
            for (int s = 0; s < KW; s++) {
#pragma unroll
                for (int j = 0; j < KC / 16; j++) {
                    const uint64_t ad = desc_add(dr, a_lo + (uint32_t)s * rowb16 + 2u * j);
                    if (rp < KH) wgmma_f16<BN>(acc[0], ad, desc_add(dw, (uint32_t)(sl * taps + rp * KW + s) * tile16 + 2u * j), 1u);
                    if (rp > 0) wgmma_f16<BN>(acc[1], ad, desc_add(dw, (uint32_t)(sl * taps + (rp - 1) * KW + s) * tile16 + 2u * j), 1u);
                }
            }
        } while (++sl < slabs);
    }
}

// Stacked weight tiles (STACK = true): per slab, shared memory holds Z, (s = 0: r = KH-1 .. 0), Z, (s = 1: r = KH-1
// .. 0), Z, ..., Z -- KW * (KH+1) + 1 tiles of BN x KC, Z a zero tile. Tile (r', s) and the one after it are then
// taps (r', s) and (r'-1, s), with Z standing for the tap r' = KH of the upper row and r'-1 = -1 of the lower row, so
// the 2 * BN contiguous rows from tile (r', s) are the B operand of both output rows at once.
template <int KW>
__device__ __forceinline__ constexpr int stack_tiles() { return KW * (KW + 1) + 1; }
// tile of tap (r, s) in its slab's stack; r = KH is the zero tile in front of column s
template <int KW>
__device__ __forceinline__ constexpr int stack_index(int r, int s) { return s * (KW + 1) + KW - r; }

// strip_pair_mma over stacked weight tiles: input row row0+r' feeds both output rows through ONE wgmma of N = 2 * BN
// per (slab, s, k16) -- the A window is read once, and every wgmma of the chain has the same width. acc is that
// wgmma's fragment: columns 0..BN-1 (row row0) in acc[0 .. BN/2), BN..2BN-1 (row row0+1) in acc[BN/2 .. BN), the
// layout of strip_pair_mma' acc[2][BN/2]. The extra terms (Z at r' = KH for the upper row, at r' = 0 for the lower
// row) are exact zeros added to an accumulator that starts at +0 and, absent Inf / NaN inputs, never is -0, so
// every output element is bit-identical to strip_pair_mma', summed in the same (r, slab, s, channel) order.
template <int KW, int KC, int BN>
__device__ __forceinline__ void strip_stack_mma(float (&acc)[BN], const RowRing &rr, int row0, int last, int slabs,
                                                 uint64_t dr, uint64_t dw, uint32_t a_off, uint32_t row16, uint32_t slab16,
                                                 int rp0, int rp1) {
    constexpr int KH = KW;
    constexpr uint32_t rowb16 = (KC * 2u) >> 4, tile16 = (BN * KC * 2u) >> 4, wslab16 = stack_tiles<KW>() * tile16;
#pragma unroll
    for (int rp = rp0; rp < rp1; rp++) {
        const uint32_t a_row = rr.slot(row0 + (rp < KH ? rp : last)) * row16 + a_off;
        int sl = 0;
#pragma unroll 1
        do {
            const uint32_t a_lo = a_row + (uint32_t)sl * slab16;
            const uint32_t w_lo = (uint32_t)sl * wslab16 + (uint32_t)stack_index<KW>(rp, 0) * tile16;
#pragma unroll
            for (int s = 0; s < KW; s++) {
#pragma unroll
                for (int j = 0; j < KC / 16; j++)
                    wgmma_f16<2 * BN>(acc, desc_add(dr, a_lo + (uint32_t)s * rowb16 + 2u * j),
                                      desc_add(dw, w_lo + (uint32_t)(s * (KH + 1)) * tile16 + 2u * j), 1u);
            }
        } while (++sl < slabs);
    }
}

template <int KW, int KC, int BN, bool POOL, bool STACK>
__global__ void __launch_bounds__(kStripThreads, 1)
conv_strip_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                  const __grid_constant__ CUtensorMap tmB, const StripParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = align1024(smem_raw);
    __shared__ __align__(8) uint64_t full_bar[kMaxSlot], empty_bar[kMaxSlot], w_bar;

    constexpr int KH = KW, ph = KH / 2, pw = KW / 2, taps = KH * KW;
    constexpr int PW = kRowTile + KW - 1;
    constexpr uint32_t tile_bytes = BN * KC * 2;            // one (slab, tap) weight tile
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slabs = (p.C1 + p.C2) / KC;
    const uint32_t row_bytes = (uint32_t)p.slab_bytes * slabs;       // one ring slot (all slabs)
    uint8_t *ring = smem + ((p.w_bytes + 1023) & ~1023);
    // CTA class: which slice of the output channels this CTA computes (weights resident per slice)
    const int split = (int)blockIdx.x % p.n_split, co_off = split * BN;
    const int item0 = (int)blockIdx.x / p.n_split, item_step = (int)gridDim.x / p.n_split;

    if constexpr (STACK) {
        // the zero tiles of the stacks, before any wgmma can read them (the fence hands them to the async proxy)
        constexpr int z_vec = (int)tile_bytes / 16, z_per_slab = KW + 1;
        for (int i = threadIdx.x; i < slabs * z_per_slab * z_vec; i += blockDim.x) {
            const int z = i / z_vec, sl = z / z_per_slab, s = z % z_per_slab;
            ((uint4 *)(smem + ((size_t)sl * stack_tiles<KW>() + (size_t)s * (KH + 1)) * tile_bytes))[i % z_vec] =
                make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async();
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < p.nslot; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        mbar_init(&w_bar, 1);
        fence_barrier_init();
    }
    if (warp == kProducerWarp && lane == 0) {
        prefetch_tmap(&tmA);
        if (p.C2) prefetch_tmap(&tmA2);
        prefetch_tmap(&tmB);
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ===== TMA producer =====
        if (lane == 0) {
            mbar_expect_tx(&w_bar, (uint32_t)(slabs * taps) * tile_bytes);
            for (int t = 0; t < slabs * taps; t++) {            // tile (slab, tap) of this CTA's output channels
                const int sl = t / taps, tap = t % taps;
                const int dst = STACK ? sl * stack_tiles<KW>() + stack_index<KW>(tap / KW, tap % KW) : t;
                tma_load_2d(smem + (size_t)dst * tile_bytes, &tmB, &w_bar, 0, t * p.cout_pad + co_off);
            }
            uint32_t cnt = 0;                                   // input rows loaded so far (all items)
            for (int item = item0; item < p.n_items; item += item_step) {
                const int tx = item % p.tiles_x, rest = item / p.tiles_x;
                const int seg = rest % p.n_seg, n = rest / p.n_seg;
                const int ya = seg * p.seg_h, yb = min(p.H, ya + p.seg_h);
                const int x0 = tx * kRowTile;
                for (int i = ya - ph; i < yb + ph; i++, cnt++) {
                    const int slot = (int)(cnt % (uint32_t)p.nslot);
                    mbar_wait(&empty_bar[slot], ((cnt / (uint32_t)p.nslot) & 1u) ^ 1u);
                    mbar_expect_tx(&full_bar[slot], (uint32_t)(PW * KC * 2 * slabs));
                    uint8_t *dst = ring + (size_t)slot * row_bytes;
                    for (int sl = 0; sl < slabs; sl++) {
                        const int c = sl * KC;
                        if (c < p.C1) tma_load_4d(dst + (size_t)sl * p.slab_bytes, &tmA, &full_bar[slot], c, x0 - pw, i, n);
                        else tma_load_4d(dst + (size_t)sl * p.slab_bytes, &tmA2, &full_bar[slot], c - p.C1, x0 - pw, i, n);
                    }
                }
            }
        }
    } else {
        // ===== consumer warpgroup g =====
        // g broadcast from lane 0: ptxas then sees warp-uniform control flow around the wgmma chains (a chain under
        // a branch it takes for divergent is serialised, one wait per wgmma)
        const int g = __shfl_sync(0xffffffffu, warp >> 2, 0);
        constexpr uint32_t sbo = 8u * KC * 2u, half16 = (64u * KC * 2u) >> 4;
        // the second 64-pixel half's chain runs during the first half's epilogue where both halves' accumulators
        // (2 x BN registers) fit within the 168-register budget; BN = 64 runs the halves one after the other
        constexpr bool kOverlap = BN <= 32;
        const uint64_t dw = make_smem_desc(smem_u32(smem), swizzle_layout(KC), sbo);
        const uint64_t dr = make_smem_desc(smem_u32(ring), swizzle_layout(KC), sbo);
        const uint32_t row16 = row_bytes >> 4, slab16 = (uint32_t)p.slab_bytes >> 4;
        mbar_wait(&w_bar, 0);
        RowRing rr{full_bar, empty_bar, (uint32_t)p.nslot, 0u, 0, 0};
        for (int item = item0; item < p.n_items; item += item_step) {
            const int tx = item % p.tiles_x, rest = item / p.tiles_x;
            const int seg = rest % p.n_seg, n = rest / p.n_seg;
            const int ya = seg * p.seg_h, yb = min(p.H, ya + p.seg_h);
            const int rows_out = yb - ya, rows_in = rows_out + 2 * ph;
            rr.waited = 0; rr.released = 0;
            for (int q = g; 2 * q < rows_out; q += 2) {
                rr.release_upto(2 * q, lane);                   // rows only the other warpgroup needed
                const bool two = 2 * q + 1 < rows_out;          // an odd last row is the pair's upper row alone
                rr.wait_upto(2 * q + KH + (two ? 1 : 0));
                // [64-pixel half][output row 2q in 0 .. BN/2-1, row 2q+1 in BN/2 .. BN-1] (strip_stack_mma' fragment)
                float acc[2][BN];
                auto rows = [&](int hf) -> float (&)[2][BN / 2] { return *reinterpret_cast<float (*)[2][BN / 2]>(acc[hf]); };
                auto zero = [&](int hf) {
#pragma unroll
                    for (int i = 0; i < BN; i++) acc[hf][i] = 0.f;
                    wgmma_fence_regs(acc[hf]);
                };
                // the wgmmas of input rows 2q+rp0 .. 2q+rp1-1 for half hf
                auto issue = [&](int hf, int rp0, int rp1) {
                    if constexpr (STACK)
                        strip_stack_mma<KW, KC, BN>(acc[hf], rr, 2 * q, two ? KH : KH - 1, slabs, dr, dw, hf * half16,
                                                     row16, slab16, rp0, rp1);
                    else
                        strip_pair_mma<KW, KC, BN>(rows(hf), rr, 2 * q, two ? KH : KH - 1, slabs, dr, dw, hf * half16,
                                                    row16, slab16, rp0, rp1);
                };
                const int y = ya + 2 * q;
                auto epilogue = [&](int hf) {
#pragma unroll
                    for (int i = 0; i < 2; i++) {
                        const int m = 64 * hf + 16 * (warp & 3) + (lane >> 2) + 8 * i;
                        const int px = tx * kRowTile + m;
                        const bool inb = px < p.W;
                        const size_t pix = ((size_t)n * p.H + y) * p.W + px;
                        __half2 h0[BN / 8], h1[BN / 8];
                        epilogue_row<BN>(rows(hf)[0], i, inb, pix, lane, p.bias + co_off, p.slope, p.out_mode, p.out,
                                         p.out_cstride, co_off, h0);
                        if (two) {
                            epilogue_row<BN>(rows(hf)[1], i, inb, pix + p.W, lane, p.bias + co_off, p.slope, p.out_mode, p.out,
                                             p.out_cstride, co_off, h1);
                            if (POOL) {
                                // 2x2 average of the stored (fp16) activations; pixel m+1 is the lane 4 apart
                                __half2 *pl = (__half2 *)((__half *)p.pool_out +
                                    (((size_t)n * (p.H / 2) + y / 2) * (p.W / 2) + px / 2) * p.pool_cstride + co_off);
#pragma unroll
                                for (int j = 0; j < BN / 8; j++) {
                                    const float2 a = __half22float2(h1[j]), b = __half22float2(h0[j]);
                                    float s0 = a.x + b.x, s1 = a.y + b.y;       // exact: fp16 values in float32
                                    s0 += __shfl_xor_sync(0xffffffffu, s0, 4);
                                    s1 += __shfl_xor_sync(0xffffffffu, s1, 4);
                                    if (inb && (lane & 4) == 0)
                                        pl[(8 * j + 2 * (lane & 3)) / 2] = __floats2half2_rn(s0 * 0.25f, s1 * 0.25f);
                                }
                            }
                        }
                    }
                };
                if constexpr (kOverlap) {
                    // one chain over both halves in three commit groups: input rows 2q, 2q+1 of both halves, the rest
                    // of half 0, the rest of half 1. Rows 2q and 2q+1 are this pair's alone (the other warpgroup's
                    // pairs start at 2q-2 and 2q+2), so they go back to the producer as soon as the first group has
                    // completed: with a short ring (split layers: 4 or 7 slots where two pairs in flight need KH+3)
                    // the rows of the other warpgroup's next pair then load while this pair's chain still runs,
                    // instead of after it. Half 0's epilogue runs under half 1's remaining wgmmas.
                    zero(0);
                    zero(1);
                    wgmma_fence();
                    issue(0, 0, 2);
                    issue(1, 0, 2);
                    wgmma_commit();
                    issue(0, 2, KH + 1);
                    wgmma_commit();
                    issue(1, 2, KH + 1);
                    wgmma_commit();
                    wgmma_wait<2>();
                    rr.release_upto(2 * q + 2, lane);
                    wgmma_wait<1>();
                    wgmma_fence_regs(acc[0]);
                    epilogue(0);
                    wgmma_wait<0>();
                    wgmma_fence_regs(acc[1]);
                    rr.release_upto(min(rows_in, 2 * q + 4), lane);    // next pair starts at 2q+4
                    epilogue(1);
                } else {
#pragma unroll
                    for (int hf = 0; hf < 2; hf++) {
                        zero(hf);
                        wgmma_fence();
                        issue(hf, 0, KH + 1);
                        wgmma_commit();
                        wgmma_wait<0>();
                        wgmma_fence_regs(acc[hf]);
                        if (hf == 1) rr.release_upto(min(rows_in, 2 * q + 4), lane);
                        epilogue(hf);
                    }
                }
            }
            rr.release_upto(rows_in, lane);
            rr.cnt += (uint32_t)rows_in;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Fused up-sampling convolution: conv3x3(bilinear_up2(L)) + bias + LeakyReLU without materialising the
// up-sampled tensor (model.py:140-147: up.forward = interpolate(x, scale_factor=2, mode='bilinear') -> conv1 ->
// leaky_relu).
//
// The x2 bilinear up-sampling (align_corners=False) is linear and shift-invariant with period 2, so it folds
// into the convolution: out[2m+py][2j+px] = sum_{a,b in -1..1} Wf[py][px][a][b] . L[m+a][j+b] -- four
// phase-specific 3x3 filters over the LOW-resolution tensor (Wf = W combined with the 0.25/0.75 coefficients,
// built in float32 on the host). Same MACs as the convolution over the up-sampled tensor, a quarter of the
// input bytes, no upsample kernel. The kernel walks a strip of 128 low-resolution columns like the strip kernel:
// a consumer warpgroup takes a pair of output rows (2m, 2m+1), both read low rows m-1..m+1, and each row is
// one asynchronous wgmma chain per 64-pixel half whose N = 128 columns are the four phases (px, py) x 32 output
// channels (they read the same low-resolution window); phase px is written to pixels 2j+px. Only the 2-pixel
// frame of the image differs (bilinear clamping and the conv's zero padding are not shift-invariant there); a
// small direct kernel rewrites it afterwards.
// Folded weight tiles in global memory: [slab][px][b][q][Cout_pad][64], q = py + 2*(1-a); in shared memory:
// [slab][b][a][px][py][Cout_pad][64].
// ---------------------------------------------------------------------------------------------
constexpr int kUpBlocks = 6;

__global__ void __launch_bounds__(kStripThreads, 1)
conv_up2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const StripParams p) {
    constexpr int KC = 64, KW = 3, BN = 32;
    constexpr int PW = kRowTile + KW - 1;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = align1024(smem_raw);
    __shared__ __align__(8) uint64_t full_bar[kMaxSlot], empty_bar[kMaxSlot], w_bar;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slabs = p.C1 / KC;
    uint8_t *ring = smem + ((p.w_bytes + 1023) & ~1023);
    const uint32_t row_bytes = (uint32_t)p.slab_bytes * slabs;
    const int hl = p.H / 2, wl = p.W / 2;                     // low-resolution input size

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.nslot; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        mbar_init(&w_bar, 1);
        fence_barrier_init();
    }
    if (warp == kProducerWarp && lane == 0) { prefetch_tmap(&tmA); prefetch_tmap(&tmB); }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ===== TMA producer: folded weights (already in tile order), then low-resolution rows =====
        if (lane == 0) {
            mbar_expect_tx(&w_bar, (uint32_t)p.w_bytes);
            // blocks [slab][b][t][px] of the tiles py = 0, 1 (adjacent in the host layout: q = py + 2*(2-t)), so
            // that the four phases of a window (slab, b, t) are 4*BN consecutive rows: one N = 128 B descriptor
            for (int l = 0; l < slabs * 3 * 3 * 2; l++) {
                const int sl = l / 18, b = (l / 6) % 3, t = (l / 2) % 3, px = l % 2;
                tma_load_2d(smem + (size_t)l * 2 * BN * KC * 2, &tmB, &w_bar, 0,
                            (((sl * 2 + px) * KW + b) * kUpBlocks + 2 * (2 - t)) * BN);
            }
            uint32_t cnt = 0;
            for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
                const int tx = item % p.tiles_x, rest = item / p.tiles_x;
                const int seg = rest % p.n_seg, n = rest / p.n_seg;
                const int ka = seg * p.seg_h, kb = min(hl, ka + p.seg_h);
                const int j0 = tx * kRowTile;
                for (int k = ka - 1; k <= kb; k++, cnt++) {
                    const int slot = (int)(cnt % (uint32_t)p.nslot);
                    mbar_wait(&empty_bar[slot], ((cnt / (uint32_t)p.nslot) & 1u) ^ 1u);
                    mbar_expect_tx(&full_bar[slot], (uint32_t)(PW * KC * 2 * slabs));
                    for (int sl = 0; sl < slabs; sl++)
                        tma_load_4d(ring + (size_t)slot * row_bytes + (size_t)sl * p.slab_bytes, &tmA, &full_bar[slot],
                                    sl * KC, j0 - 1, k, n);
                }
            }
        }
    } else {
        // ===== consumer warpgroup g: output row pairs g, g+2, ... of an item =====
        const int g = __shfl_sync(0xffffffffu, warp >> 2, 0);     // warp-uniform to ptxas (see strip_pair_mma)
        constexpr uint32_t sbo = 8u * KC * 2u, rowb16 = (KC * 2u) >> 4, half16 = (64u * KC * 2u) >> 4;
        constexpr uint32_t blk16 = (2u * BN * KC * 2u) >> 4;      // one weight block (slab, b, t, px)
        const uint64_t dw = make_smem_desc(smem_u32(smem), swizzle_layout(KC), sbo);
        const uint64_t dr = make_smem_desc(smem_u32(ring), swizzle_layout(KC), sbo);
        const uint32_t row16 = row_bytes >> 4, slab16 = (uint32_t)p.slab_bytes >> 4;
        mbar_wait(&w_bar, 0);
        RowRing rr{full_bar, empty_bar, (uint32_t)p.nslot, 0u, 0, 0};
        for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
            const int tx = item % p.tiles_x, rest = item / p.tiles_x;
            const int seg = rest % p.n_seg, n = rest / p.n_seg;
            const int ka = seg * p.seg_h, kb = min(hl, ka + p.seg_h);
            const int pairs = kb - ka, rows_in = pairs + 2;    // low rows ka-1 .. kb
            rr.waited = 0; rr.released = 0;
            for (int q = g; q < pairs; q += 2) {
                rr.release_upto(q, lane);
                rr.wait_upto(q + 3);                            // low rows ka-1+q .. ka+1+q
#pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    // one 64-pixel half, all four phases: columns [(2 px + py) * BN, +BN) are phase (px, py); every
                    // output element accumulates its terms in the order (t, slab, b, channel). Zeroed and chained
                    // as in strip_pair_mma, so that the wgmmas issue back to back.
                    float acc[4 * BN / 2];
#pragma unroll
                    for (int i = 0; i < 4 * BN / 2; i++) acc[i] = 0.f;
                    wgmma_fence_regs(acc);
                    wgmma_fence();
#pragma unroll
                    for (int t = 0; t < 3; t++) {
                        const uint32_t a_row = rr.slot(q + t) * row16 + (uint32_t)hf * half16;
                        int sl = 0;
#pragma unroll 1
                        do {
                            const uint32_t a_lo = a_row + (uint32_t)sl * slab16;
#pragma unroll
                            for (int b = 0; b < KW; b++) {
#pragma unroll
                                for (int j = 0; j < KC / 16; j++)
                                    wgmma_f16<4 * BN>(acc, desc_add(dr, a_lo + (uint32_t)b * rowb16 + 2u * j),
                                                      desc_add(dw, (uint32_t)(((sl * KW + b) * 3 + t) * 2) * blk16 + 2u * j), 1u);
                            }
                        } while (++sl < slabs);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_regs(acc);
                    if (hf == 1) rr.release_upto(min(rows_in, q + 2), lane);        // next pair starts at q+2
#pragma unroll
                    for (int ph = 0; ph < 4; ph++) {
                        const int px = ph >> 1, py = ph & 1;
                        const float (&d)[BN / 2] = *reinterpret_cast<const float (*)[BN / 2]>(&acc[ph * BN / 2]);
                        const int y = 2 * (ka + q) + py;
#pragma unroll
                        for (int i = 0; i < 2; i++) {
                            const int jl = tx * kRowTile + 64 * hf + 16 * (warp & 3) + (lane >> 2) + 8 * i;
                            const size_t pix = ((size_t)n * p.H + y) * p.W + (size_t)(2 * jl + px);
                            __half2 hv[BN / 8];
                            epilogue_row<BN>(d, i, jl < wl, pix, lane, p.bias, p.slope, 0, p.out, p.out_cstride, 0, hv);
                        }
                    }
                }
            }
            rr.release_upto(rows_in, lane);
            rr.cnt += (uint32_t)rows_in;
        }
    }
}

// The 2-pixel frame of conv3x3(up2(L)): direct evaluation with the unfolded weights [Cout_pad][9*C] (K index =
// tap*C + c), the bilinear sample rounded to fp16 like the materialised tensor would be, zero outside the
// up-sampled image. C = 64, Cout_pad = 32. One warp per frame pixel: a lane holds two channels (one half2) of
// the nine bilinear samples; the 32 output channels are 32 dot products over (tap, channel) against weights
// staged in shared memory. A lane's 18 products per output channel are accumulated with HFMA2 (the frame is
// 1.4 % of the layer's pixels; the partial sums are ~0.2 in magnitude, fp16 rounding of them stays below
// 1e-3 absolute), widened to float32 for the cross-lane reduction: a halving butterfly after which lane co holds
// output channel co.
// Latency-bound (a warp's pixel is a serial chain of gathers, half2 FMAs and shuffles): 4 warps x 4 blocks per SM.
constexpr int kBorderThreads = 128, kBorderBlocks = 4;

__global__ void __launch_bounds__(kBorderThreads, kBorderBlocks)
conv_up2_border_kernel(const __half *__restrict__ L, const __half *__restrict__ wgt, const float *__restrict__ bias,
                       __half *__restrict__ out, int N, int H, int W, int out_cstride, float slope) {
    constexpr int C = 64, BN = 32;
    extern __shared__ __align__(16) unsigned char s_wraw[];
    __half2 *s_w = (__half2 *)s_wraw;                          // [co][tap][32 lanes] half2
    for (int i = threadIdx.x; i < BN * 9 * 32; i += blockDim.x) s_w[i] = ((const __half2 *)wgt)[i];
    __syncthreads();
    const int hl = H / 2, wl = W / 2;
    const int per_img = 4 * W + 4 * (H - 4);                  // rows 0,1,H-2,H-1 and columns 0,1,W-2,W-1 of the rest
    const long total = (long)N * per_img;
    const int lane = threadIdx.x & 31;
    const long warp0 = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nwarps = (long)gridDim.x * (blockDim.x >> 5);
    const float bias_l = bias[lane];
    const __half2 *base = (const __half2 *)L + lane;
    for (long pi = warp0; pi < total; pi += nwarps) {
        const int n = (int)(pi / per_img), f = (int)(pi % per_img);
        int y, x;
        if (f < 4 * W) { const int r = f / W; y = r < 2 ? r : H - 4 + r; x = f % W; }
        else { const int g = f - 4 * W; const int c = g % 4; y = 2 + g / 4; x = c < 2 ? c : W - 4 + c; }
        __half2 smp[9];
#pragma unroll
        for (int t = 0; t < 9; t++) {
            const int uy = y + t / 3 - 1, ux = x + t % 3 - 1;
            __half2 v = __floats2half2_rn(0.f, 0.f);
            if (uy >= 0 && uy < H && ux >= 0 && ux < W) {
                const float sy = fmaxf(0.f, (uy + 0.5f) * 0.5f - 0.5f), sx = fmaxf(0.f, (ux + 0.5f) * 0.5f - 0.5f);
                const int y0 = (int)sy, y1 = min(y0 + 1, hl - 1), x0 = (int)sx, x1 = min(x0 + 1, wl - 1);
                const float ly = sy - (float)y0, lx = sx - (float)x0;
                const float2 a = __half22float2(base[(((size_t)n * hl + y0) * wl + x0) * (C / 2)]);
                const float2 b = __half22float2(base[(((size_t)n * hl + y0) * wl + x1) * (C / 2)]);
                const float2 c = __half22float2(base[(((size_t)n * hl + y1) * wl + x0) * (C / 2)]);
                const float2 d = __half22float2(base[(((size_t)n * hl + y1) * wl + x1) * (C / 2)]);
                const float v0 = (1.f - ly) * ((1.f - lx) * a.x + lx * b.x) + ly * ((1.f - lx) * c.x + lx * d.x);
                const float v1 = (1.f - ly) * ((1.f - lx) * a.y + lx * b.y) + ly * ((1.f - lx) * c.y + lx * d.y);
                v = __floats2half2_rn(v0, v1);
            }
            smp[t] = v;
        }
        // two groups of 16 output channels (keeps 16 accumulators live): partial dot products, a halving
        // butterfly over lane bits 3..0 (lane keeps channel lane & 15 of the group), then the two 16-lane halves
        // are added; the half whose index equals the group writes
        float res = 0.f;
#pragma unroll
        for (int g = 0; g < 2; g++) {
            float acc[16];
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const int co = g * 16 + j;
                __half2 h = __hmul2(smp[0], s_w[(co * 9) * 32 + lane]);
#pragma unroll
                for (int t = 1; t < 9; t++) h = __hfma2(smp[t], s_w[(co * 9 + t) * 32 + lane], h);
                const float2 hf = __half22float2(h);
                acc[j] = hf.x + hf.y;
            }
#pragma unroll
            for (int o = 8; o >= 1; o >>= 1) {
                const bool up = (lane & o) != 0;
#pragma unroll
                for (int j = 0; j < o; j++) {
                    const float mine = up ? acc[j + o] : acc[j];
                    const float send = up ? acc[j] : acc[j + o];
                    acc[j] = mine + __shfl_xor_sync(0xffffffffu, send, o);
                }
            }
            const float tot = acc[0] + __shfl_xor_sync(0xffffffffu, acc[0], 16);
            if ((lane >> 4) == g) res = tot;                   // channel g*16 + (lane & 15) == lane
        }
        const float v = res + bias_l;
        out[(((size_t)n * H + y) * W + x) * out_cstride + lane] = __float2half_rn(fmaxf(v, v * slope));
    }
}

}  // namespace

// =============================================================================================
// host side
// =============================================================================================
static thread_local char g_conv_err[512];
extern int v2e_set_error(int code, const char *fmt, const char *detail);

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

static CUtensorMapSwizzle swizzle_for(int kc) {
    return kc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (kc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// NHWC fp16 activation [N,H,W,C]: box = KC channels x 16 columns x tile_h rows x 1 image
static int make_act_tmap_h(CUtensorMap *tm, const void *ptr, int N, int H, int W, int C, int KC, int tile_h) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled unavailable%s", "");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)kTileW, (cuuint32_t)tile_h, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void *)ptr, dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(KC), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        snprintf(g_conv_err, sizeof(g_conv_err), "activation map N=%d H=%d W=%d C=%d KC=%d CUresult=%d", N, H, W, C, KC, (int)r);
        return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled failed: %s", g_conv_err);
    }
    return V2E_OK;
}
int v2e_make_act_tmap(CUtensorMap *tm, const void *ptr, int N, int H, int W, int C, int KC) {
    return make_act_tmap_h(tm, ptr, N, H, W, C, KC, kTileH);
}

// weights [Cout_pad][Ktot] fp16: box = KC x BN
int v2e_make_wgt_tmap(CUtensorMap *tm, const void *ptr, int Cout_pad, int Ktot, int KC, int BN) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled unavailable%s", "");
    cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)Cout_pad};
    cuuint64_t strides[1] = {(cuuint64_t)Ktot * 2};
    cuuint32_t box[2] = {(cuuint32_t)KC, (cuuint32_t)BN};
    cuuint32_t es[2] = {1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)ptr, dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(KC), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        snprintf(g_conv_err, sizeof(g_conv_err), "weight map Cout=%d K=%d KC=%d BN=%d CUresult=%d", Cout_pad, Ktot, KC, BN, (int)r);
        return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled failed: %s", g_conv_err);
    }
    return V2E_OK;
}

int v2e_conv_pick_kc(int C1, int C2) {
    int g = C2 ? (C1 < C2 ? C1 : C2) : C1;
    return g % 64 == 0 ? 64 : (g % 32 == 0 ? 32 : 16);
}
int v2e_conv_pick_bn(int Cout_pad) { return Cout_pad >= 128 ? 128 : Cout_pad; }

// Per-tap tiles (pixels x output channels): V2E_CONV_TILE_LEGACY = 128 x min(Cout_pad, 128) (conv_tc_kernel),
// V2E_CONV_TILE_256x128 and V2E_CONV_TILE_128x256 (conv_wide_kernel, MH = 2 / 1).
static void tile_shape(int tile, int Cout_pad, int *mh, int *bn) {
    *mh = tile == V2E_CONV_TILE_256x128 ? 2 : 1;
    *bn = tile == V2E_CONV_TILE_128x256 ? 256 : (tile == V2E_CONV_TILE_256x128 ? 128 : v2e_conv_pick_bn(Cout_pad));
}

// Wave-aware choice of the tile. A CTA's time per (tap, slab) stage is
// the larger of its L2-to-shared-memory bytes at ~24 B/clk per SM (6-7 TB/s over 132 SMs, the rate the 128 x 128
// tile runs at) and its MMAs at 4096 dense fp16 FLOP/clk per SM; every tile runs the same stages per CTA, so a layer
// costs waves x (time per stage). One CTA per SM (the stages fill the shared memory). Ties go to the 128 x 128 tile.
// The wide tiles need 64-channel slabs.
extern "C" int v2e_conv_pick_tile(int C1, int C2, int Cout_pad, int KH, int KW, int N, int H, int W, int n_sms) {
    (void)KH; (void)KW;
    const int kc = v2e_conv_pick_kc(C1, C2);
    if (n_sms < 1) n_sms = 1;
    int best = V2E_CONV_TILE_LEGACY;
    double best_cost = 0.0;
    for (int tile = V2E_CONV_TILE_LEGACY; tile <= V2E_CONV_TILE_128x256; tile++) {
        int mh, bn;
        tile_shape(tile, Cout_pad, &mh, &bn);
        const bool wide = tile != V2E_CONV_TILE_LEGACY;
        // one wide candidate per layer: 16x16 pixels for Cout_pad = 128, 256 channels from Cout_pad = 256 on
        if (wide && (kc != 64 || Cout_pad % bn || (tile == V2E_CONV_TILE_256x128) != (Cout_pad == 128))) continue;
        long tiles = (long)((W + kTileW - 1) / kTileW) * ((H + kTileH * mh - 1) / (kTileH * mh)) * N;
        const long ctas = tiles * (Cout_pad / bn);
        const long waves = (ctas + n_sms - 1) / n_sms;
        const double a_bytes = (double)kBM * mh * kc * 2, b_bytes = (double)bn * kc * 2;
        const double flops = 2.0 * kBM * mh * bn * kc;
        const double per_stage = fmax((a_bytes + b_bytes) / 24.0, flops / 4096.0);
        const double cost = (double)waves * per_stage;
        if (tile == V2E_CONV_TILE_LEGACY || cost < best_cost) { best = tile; best_cost = cost; }
    }
    return best;
}

struct V2eConvLaunch {
    CUtensorMap tmA, tmA2, tmB;
    ConvParams p;
    dim3 grid;
    int mh;
    size_t smem;
};

int v2e_conv_prepare(V2eConvLaunch *L, const void *x1, int C1, const void *x2, int C2, const void *wgt,
                     const float *bias, int Cout_pad, int KH, int KW, int N, int H, int W, void *out,
                     int out_cstride, int out_mode, int co_real, float slope, int tile, int n_sms) {
    if (C1 % 16 || C2 % 16 || !(Cout_pad == 16 || Cout_pad == 32 || Cout_pad == 64 || (Cout_pad > 0 && Cout_pad % 128 == 0)))
        return v2e_set_error(V2E_E_INVALID, "conv: channel counts must be padded to 16 (Cout to 16/32/64/128k)%s", "");
    if (tile == V2E_CONV_TILE_AUTO) tile = v2e_conv_pick_tile(C1, C2, Cout_pad, KH, KW, N, H, W, n_sms);
    if (tile < V2E_CONV_TILE_LEGACY || tile > V2E_CONV_TILE_128x256)
        return v2e_set_error(V2E_E_INVALID, "conv: unknown tile%s", "");
    memset(L, 0, sizeof(*L));
    ConvParams &p = L->p;
    int mh, bn;
    tile_shape(tile, Cout_pad, &mh, &bn);
    const bool wide = tile != V2E_CONV_TILE_LEGACY;
    p.N = N; p.H = H; p.W = W; p.C1 = C1; p.C2 = C2; p.KH = KH; p.KW = KW;
    p.KC = v2e_conv_pick_kc(C1, C2);
    p.BN = bn;
    if (wide && (Cout_pad % bn || out_mode != 0))
        return v2e_set_error(V2E_E_INVALID, "conv: the wide tiles need fp16 output and Cout_pad a multiple of their width%s", "");
    p.stages = kStages;
    p.tiles_x = (W + kTileW - 1) / kTileW;
    p.tiles_y = (H + kTileH * mh - 1) / (kTileH * mh);
    p.n_tiles = p.tiles_x * p.tiles_y * N;
    p.out_cstride = out_cstride; p.out_mode = out_mode; p.co_real = co_real; p.slope = slope;
    p.bias = bias; p.out = out;
    L->mh = mh;
    int rc;
    if ((rc = make_act_tmap_h(&L->tmA, x1, N, H, W, C1, p.KC, kTileH * mh))) return rc;
    if (C2) { if ((rc = make_act_tmap_h(&L->tmA2, x2, N, H, W, C2, p.KC, kTileH * mh))) return rc; }
    else L->tmA2 = L->tmA;
    if ((rc = v2e_make_wgt_tmap(&L->tmB, wgt, Cout_pad, KH * KW * (C1 + C2), p.KC, bn))) return rc;
    const unsigned tiles = (unsigned)p.n_tiles, cob = (unsigned)(Cout_pad / p.BN);
    p.co_fast = (cob > 1 && tiles <= 65535u) ? 1 : 0;
    L->grid = p.co_fast ? dim3(cob, tiles, 1) : dim3(tiles, cob, 1);
    size_t stage = (size_t)kBM * mh * p.KC * 2 + (((size_t)p.BN * p.KC * 2 + 1023) & ~(size_t)1023);
    L->smem = stage * p.stages + 1024;
    return V2E_OK;
}

template <int BN>
static cudaError_t conv_launch_bn(const V2eConvLaunch *L, cudaStream_t st) {
    static PerDeviceOnce attr_once;
    if (attr_once.first()) cudaFuncSetAttribute(conv_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    conv_tc_kernel<BN><<<L->grid, kConvThreads, L->smem, st>>>(L->tmA, L->tmA2, L->tmB, L->p);
    return cudaGetLastError();
}

template <int MH, int BN>
static cudaError_t conv_launch_wide(const V2eConvLaunch *L, cudaStream_t st) {
    static PerDeviceOnce attr_once;
    if (attr_once.first())
        cudaFuncSetAttribute(conv_wide_kernel<MH, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    conv_wide_kernel<MH, BN><<<L->grid, kConvThreads, L->smem, st>>>(L->tmA, L->tmA2, L->tmB, L->p);
    return cudaGetLastError();
}

int v2e_conv_launch(const V2eConvLaunch *L, cudaStream_t st) {
    cudaError_t e;
    if (L->mh == 2 && L->p.BN == 128) e = conv_launch_wide<2, 128>(L, st);
    else if (L->mh == 1 && L->p.BN == 256) e = conv_launch_wide<1, 256>(L, st);
    else switch (L->p.BN) {
        case 16: e = conv_launch_bn<16>(L, st); break;
        case 32: e = conv_launch_bn<32>(L, st); break;
        case 64: e = conv_launch_bn<64>(L, st); break;
        case 128: e = conv_launch_bn<128>(L, st); break;
        default: return v2e_set_error(V2E_E_UNSUPPORTED, "conv_tc_kernel: unsupported tile width%s", "");
    }
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "conv_tc_kernel launch: %s", cudaGetErrorString(e));
    return V2E_OK;
}

size_t v2e_conv_launch_size(void) { return sizeof(V2eConvLaunch); }

// ---- standalone C-ABI entry (tests, and integrators who bring their own network driver) -------------
static int device_sms() {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

extern "C" int v2e_conv2d_lrelu_sm100_tile(const void *x1_dev, int C1, const void *x2_dev, int C2,
                                           const void *wgt_dev, const float *bias_dev, int Cout_pad, int KH, int KW,
                                           int N, int H, int W, void *out_dev, int out_cstride, int out_mode,
                                           int co_real, float slope, int tile, void *stream) {
    V2eConvLaunch L;
    int rc = v2e_conv_prepare(&L, x1_dev, C1, x2_dev, C2, wgt_dev, bias_dev, Cout_pad, KH, KW, N, H, W, out_dev,
                              out_cstride, out_mode, co_real, slope, tile, device_sms());
    if (rc) return rc;
    return v2e_conv_launch(&L, (cudaStream_t)stream);
}

extern "C" int v2e_conv2d_lrelu_sm100(const void *x1_dev, int C1, const void *x2_dev, int C2,
                                      const void *wgt_dev, const float *bias_dev, int Cout_pad, int KH, int KW,
                                      int N, int H, int W, void *out_dev, int out_cstride, int out_mode,
                                      int co_real, float slope, void *stream) {
    return v2e_conv2d_lrelu_sm100_tile(x1_dev, C1, x2_dev, C2, wgt_dev, bias_dev, Cout_pad, KH, KW, N, H, W, out_dev,
                                       out_cstride, out_mode, co_real, slope, V2E_CONV_TILE_AUTO, stream);
}

// ---- strip kernel host side ------------------------------------------------------------------------
struct V2eStripLaunch {
    CUtensorMap tmA, tmA2, tmB;
    StripParams p;
    int stacked;                  // conv_strip_kernel<.., STACK>
    int grid;
    size_t smem;
};

// one input row of the strip: KC channels x (128+KW-1) columns
static int make_rowseg_tmap(CUtensorMap *tm, const void *ptr, int N, int H, int W, int C, int KC, int KW) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled unavailable%s", "");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)(kRowTile + KW - 1), 1, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void *)ptr, dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(KC), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled failed for a strip row map%s", "");
    return V2E_OK;
}

// Shared memory of one CTA (227 KB on sm_90, 228 KB per SM): the whole budget, or half of it for two CTAs per SM.
constexpr size_t kSmemFull = 222 * 1024, kSmemHalf = 110 * 1024;

// Resident weights of one CTA class: KH*KW tiles of BN x KC per slab, or KW*(KH+1)+1 with the zero tiles of the
// stacked layout (strip_stack_mma).
static size_t strip_w_bytes(int slabs, int KH, int KW, int bn, int kc, int stacked) {
    return (size_t)slabs * (stacked ? KW * (KH + 1) + 1 : KH * KW) * bn * kc * 2;
}

// Strip configuration of a layer and chain: ring slots (one input row, all slabs, each), CTAs per SM, output-channel
// split. Returns 0 when the layer does not fit (resident weights of a slice of >= 16 output channels + KH+1 ring rows:
// the rows a pair of output rows reads). Two CTAs per SM when the weights and KH+3 rows (both warpgroups busy)
// fit in half of the shared memory.
static int strip_config(int C1, int C2, int Cout_pad, int KH, int KW, int kc, int stacked, int *nslot, int *ctas_per_sm,
                        int *n_split) {
    if (Cout_pad > 64) return 0;
    const int slabs = (C1 + C2) / kc;
    const size_t row = (((size_t)(kRowTile + KW - 1) * kc * 2 + 1023) & ~(size_t)1023) * slabs;
    for (int split = 1; split <= 2; split++) {
        const int bn = Cout_pad / split;
        if (bn < 16 || bn % 16) break;
        const size_t wb = (strip_w_bytes(slabs, KH, KW, bn, kc, stacked) + 1023) & ~(size_t)1023;
        const int two = wb + 2048 + (size_t)(KH + 3) * row <= kSmemHalf;
        const size_t budget = two ? kSmemHalf : kSmemFull;
        if (wb + 2048 + (size_t)(KH + 1) * row > budget) continue;
        int ns = (int)((budget - wb - 2048) / row);
        if (ns > kMaxSlot) ns = kMaxSlot;
        *nslot = ns; *ctas_per_sm = two ? 2 : 1; *n_split = split;
        return 1;
    }
    return 0;
}

// wide layers only: narrow rows waste part of the last 128-pixel strip (320 = 2.5 strips) and the per-tap kernel's
// 8x16 tiles take over
constexpr int kStripMinW = 2 * kRowTile;

// Slab width for the strip kernel; returns KC (0: layer does not qualify), *nslot_out.
int v2e_strip_pick(int C1, int C2, int Cout_pad, int KH, int KW, int W, int *nslot_out) {
    if (Cout_pad > 64 || KH != KW || W < kStripMinW || (KW != 3 && KW != 5 && KW != 7)) return 0;
    const int g = C2 ? (C1 < C2 ? C1 : C2) : C1;
    const int kc = g % 64 == 0 ? 64 : (g % 32 == 0 ? 32 : 16);
    int ns, cps, nsp;
    if (!strip_config(C1, C2, Cout_pad, KH, KW, kc, 0, &ns, &cps, &nsp)) return 0;
    if (nslot_out) *nslot_out = ns;
    return kc;
}

// The chain V2E_STRIP_CHAIN_AUTO runs: stacked (strip_stack_mma) where a CTA class has BN <= 32 output channels and the
// stacked weights fit with the CTAs per SM and the output-channel split of the paired chain. Per input row and k16 the
// paired chain reads 2 x (2 KB of A + BN x 32 B of B) and the stacked one 2 KB + 2 x BN x 32 B: a third fewer operand
// bytes at BN = 32, 40 % at BN = 16, but only a quarter at BN = 64, which does not pay for the (KH+1)/KH MACs there
// (down1.conv1 measured 1-2.5 % slower stacked; conv2 11-14 % and conv3 9 % faster, bench_strip.py, DESIGN.md 5).
static int strip_auto_stacked(int C1, int C2, int Cout_pad, int KH, int KW, int kc) {
    int ns0, cps0, nsp0, ns1, cps1, nsp1;
    if (!strip_config(C1, C2, Cout_pad, KH, KW, kc, 0, &ns0, &cps0, &nsp0) || Cout_pad / nsp0 > 32 ||
        !strip_config(C1, C2, Cout_pad, KH, KW, kc, 1, &ns1, &cps1, &nsp1))
        return 0;
    return cps1 == cps0 && nsp1 == nsp0;
}

// Plan of a layer that qualifies (kc from v2e_strip_pick) under a chain request; 0 when a stacked chain was asked
// for and its weights do not fit.
static int strip_plan(int C1, int C2, int Cout_pad, int KH, int KW, int kc, int chain, int *nslot, int *ctas_per_sm,
                      int *n_split, int *stacked) {
    *stacked = chain == V2E_STRIP_CHAIN_AUTO ? strip_auto_stacked(C1, C2, Cout_pad, KH, KW, kc)
                                             : chain == V2E_STRIP_CHAIN_STACKED;
    return strip_config(C1, C2, Cout_pad, KH, KW, kc, *stacked, nslot, ctas_per_sm, n_split);
}

extern "C" int v2e_conv_strip_pick_chain(int C1, int C2, int Cout_pad, int KH, int KW, int W) {
    const int kc = v2e_strip_pick(C1, C2, Cout_pad, KH, KW, W, nullptr);
    return kc ? strip_auto_stacked(C1, C2, Cout_pad, KH, KW, kc) : -1;
}

size_t v2e_strip_launch_size(void) { return sizeof(V2eStripLaunch); }

// a pooled epilogue (conv_strip_kernel<KW, KC, BN, true, .>) exists for these: one CTA per SM (the pooled variant keeps
// a row of activations in registers), >= 32 output channels per CTA class, even image size
static bool strip_pool_ok(int KW, int KC, int H, int W, int ctas_per_sm, int bn) {
    return !(H & 1) && !(W & 1) && ((KW == 7 && KC == 32) || (KW == 5 && KC == 64)) && ctas_per_sm == 1 && bn >= 32;
}

// 1 when the layer's strip configuration (V2E_STRIP_CHAIN_AUTO) has a pooled epilogue
int v2e_strip_pool_supported(int C1, int C2, int Cout_pad, int KH, int KW, int H, int W) {
    const int KC = v2e_strip_pick(C1, C2, Cout_pad, KH, KW, W, nullptr);
    int ns, cps, nsp, st;
    if (!KC || !strip_plan(C1, C2, Cout_pad, KH, KW, KC, V2E_STRIP_CHAIN_AUTO, &ns, &cps, &nsp, &st)) return 0;
    return strip_pool_ok(KW, KC, H, W, cps, Cout_pad / nsp);
}

int v2e_strip_prepare(V2eStripLaunch *L, const void *x1, int C1, const void *x2, int C2, const void *wgt_row,
                      const float *bias, int Cout_pad, int KH, int KW, int N, int H, int W, void *out,
                      int out_cstride, int out_mode, int co_real, float slope, int n_sms, void *pool_out,
                      int pool_cstride, int chain) {
    memset(L, 0, sizeof(*L));
    StripParams &p = L->p;
    if (chain < V2E_STRIP_CHAIN_AUTO || chain > V2E_STRIP_CHAIN_STACKED)
        return v2e_set_error(V2E_E_INVALID, "strip: unknown chain%s", "");
    const int KC = v2e_strip_pick(C1, C2, Cout_pad, KH, KW, W, nullptr);
    int nslot = 0, ctas_per_sm = 0, n_split = 0, stacked = 0;
    if (!KC || !strip_plan(C1, C2, Cout_pad, KH, KW, KC, chain, &nslot, &ctas_per_sm, &n_split, &stacked))
        return v2e_set_error(V2E_E_INVALID, "layer does not qualify for the strip kernel (with this chain)%s", "");
    L->stacked = stacked;
    p.N = N; p.H = H; p.W = W; p.C1 = C1; p.C2 = C2; p.KH = KH; p.KW = KW; p.KC = KC;
    p.n_split = n_split; p.cout_pad = Cout_pad; p.BN = Cout_pad / n_split;
    p.tiles_x = (W + kRowTile - 1) / kRowTile;
    // segment height: enough items to balance the SMs (>= ~6 per SM), at least 4*KH rows per item
    int seg_h = H;
    const int strips = p.tiles_x * N;
    while (seg_h > 4 * KH && (long)strips * ((H + seg_h - 1) / seg_h) < 6L * n_sms) seg_h = (seg_h + 1) / 2;
    if (pool_out) {
        if (out_mode != 0 || !strip_pool_ok(KW, KC, H, W, ctas_per_sm, p.BN))
            return v2e_set_error(V2E_E_UNSUPPORTED, "strip: this layer has no pooled epilogue%s", "");
        seg_h = (seg_h + 1) & ~1;                      // 2x2 windows never straddle two items
    }
    p.pool_out = pool_out;
    p.pool_cstride = pool_cstride;
    p.seg_h = seg_h;
    p.n_seg = (H + seg_h - 1) / seg_h;
    p.n_items = strips * p.n_seg;
    p.nslot = nslot;
    const int slabs = (C1 + C2) / KC, taps = KH * KW;
    p.slab_bytes = (int)(((size_t)(kRowTile + KW - 1) * KC * 2 + 1023) & ~(size_t)1023);
    p.w_bytes = (int)strip_w_bytes(slabs, KH, KW, p.BN, KC, stacked);   // resident per CTA: its output channels
    p.out_cstride = out_cstride; p.out_mode = out_mode; p.co_real = co_real; p.slope = slope;
    p.bias = bias; p.out = out;
    int rc;
    if ((rc = make_rowseg_tmap(&L->tmA, x1, N, H, W, C1, KC, KW))) return rc;
    if (C2) { if ((rc = make_rowseg_tmap(&L->tmA2, x2, N, H, W, C2, KC, KW))) return rc; }
    else L->tmA2 = L->tmA;
    {
        // weights [slabs][taps][Cout_pad][KC]: one box per (slab, tap) tile of this CTA class's BN output channels
        EncodeTiledFn fn = encode_fn();
        const int rows_total = slabs * taps * Cout_pad;
        cuuint64_t dims[2] = {(cuuint64_t)KC, (cuuint64_t)rows_total};
        cuuint64_t strides[1] = {(cuuint64_t)KC * 2};
        cuuint32_t box[2] = {(cuuint32_t)KC, (cuuint32_t)p.BN};
        cuuint32_t es[2] = {1, 1};
        CUresult r = fn(&L->tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)wgt_row, dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(KC), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled failed for strip weights%s", "");
    }
    L->smem = (size_t)((p.w_bytes + 1023) & ~1023) + (size_t)p.nslot * p.slab_bytes * slabs + 1024;
    // every CTA class walks all items
    int per = ctas_per_sm * n_sms / p.n_split;
    if (per > p.n_items) per = p.n_items;
    if (per < 1) per = 1;
    L->grid = per * p.n_split;
    return V2E_OK;
}

template <int KW, int KC, int BN, bool POOL, bool STACK>
static cudaError_t strip_launch_s(const V2eStripLaunch *L, cudaStream_t st) {
    static PerDeviceOnce attr_once;
    if (attr_once.first())
        cudaFuncSetAttribute(conv_strip_kernel<KW, KC, BN, POOL, STACK>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    conv_strip_kernel<KW, KC, BN, POOL, STACK><<<L->grid, kStripThreads, L->smem, st>>>(L->tmA, L->tmA2, L->tmB, L->p);
    return cudaGetLastError();
}

template <int KW, int KC, int BN, bool POOL>
static cudaError_t strip_launch_t(const V2eStripLaunch *L, cudaStream_t st) {
    return L->stacked ? strip_launch_s<KW, KC, BN, POOL, true>(L, st) : strip_launch_s<KW, KC, BN, POOL, false>(L, st);
}

template <int KW, int KC>
static int strip_launch_kc(const V2eStripLaunch *L, cudaStream_t st, cudaError_t *e) {
    const StripParams &p = L->p;
    if (p.KW != KW || p.KC != KC) return 0;
    if (p.pool_out) {
        // the two layers that are followed by the pool of a down block at full / half resolution (conv2, down1.conv2)
        if constexpr ((KW == 7 && KC == 32) || (KW == 5 && KC == 64)) {
            if (p.BN == 32) { *e = strip_launch_t<KW, KC, 32, true>(L, st); return 1; }
            if (p.BN == 64) { *e = strip_launch_t<KW, KC, 64, true>(L, st); return 1; }
        }
        return 0;
    }
    if (p.BN == 16) { *e = strip_launch_t<KW, KC, 16, false>(L, st); return 1; }
    if (p.BN == 32) { *e = strip_launch_t<KW, KC, 32, false>(L, st); return 1; }
    if (p.BN == 64) { *e = strip_launch_t<KW, KC, 64, false>(L, st); return 1; }
    return 0;
}

int v2e_strip_launch(const V2eStripLaunch *L, cudaStream_t st) {
    cudaError_t e = cudaSuccess;
    const int launched = strip_launch_kc<3, 16>(L, st, &e) || strip_launch_kc<3, 32>(L, st, &e) ||
                         strip_launch_kc<3, 64>(L, st, &e) || strip_launch_kc<5, 16>(L, st, &e) ||
                         strip_launch_kc<5, 32>(L, st, &e) || strip_launch_kc<5, 64>(L, st, &e) ||
                         strip_launch_kc<7, 16>(L, st, &e) || strip_launch_kc<7, 32>(L, st, &e) ||
                         strip_launch_kc<7, 64>(L, st, &e);
    if (!launched) return v2e_set_error(V2E_E_UNSUPPORTED, "strip kernel: unsupported filter width / slab / pooled epilogue%s", "");
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "conv_strip_kernel launch: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_conv2d_lrelu_sm100_strip_chain(const void *x1_dev, int C1, const void *x2_dev, int C2,
                                                  const void *wgt_row_dev, const float *bias_dev, int Cout_pad, int KH,
                                                  int KW, int N, int H, int W, void *out_dev, int out_cstride,
                                                  int out_mode, int co_real, float slope, int chain, void *stream) {
    V2eStripLaunch L;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int rc = v2e_strip_prepare(&L, x1_dev, C1, x2_dev, C2, wgt_row_dev, bias_dev, Cout_pad, KH, KW, N, H, W,
                               out_dev, out_cstride, out_mode, co_real, slope, sms, nullptr, 0, chain);
    if (rc) return rc;
    return v2e_strip_launch(&L, (cudaStream_t)stream);
}

extern "C" int v2e_conv2d_lrelu_sm100_strip(const void *x1_dev, int C1, const void *x2_dev, int C2,
                                            const void *wgt_row_dev, const float *bias_dev, int Cout_pad, int KH,
                                            int KW, int N, int H, int W, void *out_dev, int out_cstride,
                                            int out_mode, int co_real, float slope, void *stream) {
    return v2e_conv2d_lrelu_sm100_strip_chain(x1_dev, C1, x2_dev, C2, wgt_row_dev, bias_dev, Cout_pad, KH, KW, N, H, W,
                                              out_dev, out_cstride, out_mode, co_real, slope, V2E_STRIP_CHAIN_AUTO, stream);
}


// ---- fused up-sample + 3x3 convolution host side ------------------------------------------------------
struct V2eUpLaunch {
    CUtensorMap tmA, tmB;
    StripParams p;
    int grid;
    size_t smem;
    const __half *low;            // border kernel inputs
    const __half *w_plain;
    int C;
};

// 64-channel slabs, Cout_pad = 32, folded weights resident: slabs * 36 tiles of 32 x 64 fp16, + 3 ring rows
int v2e_conv_up2_supported(int C, int Cout_pad, int W_out) {
    if (C != 64 || Cout_pad != 32 || W_out % 2 || W_out < 2 * kStripMinW) return 0;   // the frame kernel is written for C = 64
    const size_t wb = (size_t)(C / 64) * 2 * 3 * kUpBlocks * Cout_pad * 64 * 2;
    const size_t slab = ((size_t)(kRowTile + 2) * 64 * 2 + 1023) & ~(size_t)1023;
    return wb + 2048 + 3 * slab * (C / 64) <= kSmemFull;
}

// Folds the x2 bilinear up-sampling into the 3x3 filter (see conv_up2_kernel). w: float32 [cout][cin][3][3]
// (the reference's state_dict layout); out: fp16 [C_pad/64][2 px][3 b][6 q][Cout_pad][64], zero padded.
extern "C" int v2e_conv_up2_fold_weights(const float *w, int cout, int cin, int Cout_pad, int C_pad, void *out_host) {
    if (!w || !out_host || C_pad % 64 || cin > C_pad || cout > Cout_pad) return v2e_set_error(V2E_E_INVALID, "bad argument%s", "");
    __half *o = (__half *)out_host;
    auto coef = [](int i, int a) -> float {      // weight of low index m+a in up-sampled index 2m+i (interior)
        const int t = i >= 0 ? i / 2 : -((1 - i) / 2), odd = i - 2 * t;
        if (!odd) return a == t - 1 ? 0.25f : (a == t ? 0.75f : 0.f);
        return a == t ? 0.75f : (a == t + 1 ? 0.25f : 0.f);
    };
    const int slabs = C_pad / 64;
    for (int sl = 0; sl < slabs; sl++)
        for (int px = 0; px < 2; px++)
            for (int b = 0; b < 3; b++)
                for (int q = 0; q < kUpBlocks; q++) {
                    const int py = q & 1, a = 1 - (q >> 1);
                    for (int co = 0; co < Cout_pad; co++)
                        for (int c = 0; c < 64; c++) {
                            const int ci = sl * 64 + c;
                            float v = 0.f;
                            if (co < cout && ci < cin)
                                for (int r = 0; r < 3; r++)
                                    for (int s2 = 0; s2 < 3; s2++)
                                        v += w[(((size_t)co * cin + ci) * 3 + r) * 3 + s2] * coef(py + r - 1, a) * coef(px + s2 - 1, b - 1);
                            o[((((size_t)(sl * 2 + px) * 3 + b) * kUpBlocks + q) * Cout_pad + co) * 64 + c] = __float2half_rn(v);
                        }
                }
    return V2E_OK;
}

size_t v2e_conv_up2_launch_size(void) { return sizeof(V2eUpLaunch); }

int v2e_conv_up2_prepare(V2eUpLaunch *L, const void *x_low, int C, const void *wgt_fold, const void *wgt_plain,
                         const float *bias, int Cout_pad, int N, int H, int W, void *out, int out_cstride, float slope,
                         int n_sms) {
    memset(L, 0, sizeof(*L));
    if (!v2e_conv_up2_supported(C, Cout_pad, W) || H % 2) return v2e_set_error(V2E_E_INVALID, "layer does not qualify for the fused up-sampling convolution%s", "");
    if (!(slope >= 0.f && slope <= 1.f)) return v2e_set_error(V2E_E_INVALID, "slope must be in [0, 1]%s", "");
    StripParams &p = L->p;
    const int hl = H / 2, wl = W / 2, KC = 64;
    p.N = N; p.H = H; p.W = W; p.C1 = C; p.C2 = 0; p.KH = 3; p.KW = 3; p.KC = KC; p.BN = Cout_pad;
    p.tiles_x = (wl + kRowTile - 1) / kRowTile;
    const int strips = p.tiles_x * N;
    int n_seg = (6 * n_sms + strips - 1) / strips;
    if (n_seg < 1) n_seg = 1;
    int seg_h = (hl + n_seg - 1) / n_seg;
    if (seg_h < 8) seg_h = hl < 8 ? hl : 8;
    p.seg_h = seg_h;
    p.n_seg = (hl + seg_h - 1) / seg_h;
    p.n_items = strips * p.n_seg;
    p.n_split = 1; p.cout_pad = Cout_pad;
    const int slabs = C / KC;
    p.slab_bytes = (int)(((size_t)(kRowTile + 2) * KC * 2 + 1023) & ~(size_t)1023);
    p.w_bytes = slabs * 2 * 3 * kUpBlocks * Cout_pad * KC * 2;
    const int rows_total = slabs * 2 * 3 * kUpBlocks * Cout_pad;
    int ns = (int)((kSmemFull - (size_t)p.w_bytes - 2048) / ((size_t)p.slab_bytes * slabs));
    if (ns > kMaxSlot) ns = kMaxSlot;
    if (ns < 3) return v2e_set_error(V2E_E_INVALID, "fused up-sampling convolution: weights leave no room for the input ring%s", "");
    p.nslot = ns;
    p.out_cstride = out_cstride; p.out_mode = 0; p.co_real = Cout_pad; p.slope = slope;
    p.bias = bias; p.out = out;
    int rc;
    if ((rc = make_rowseg_tmap(&L->tmA, x_low, N, hl, wl, C, KC, 3))) return rc;
    {
        EncodeTiledFn fn = encode_fn();
        cuuint64_t dims[2] = {(cuuint64_t)KC, (cuuint64_t)rows_total};
        cuuint64_t strides[1] = {(cuuint64_t)KC * 2};
        cuuint32_t box[2] = {(cuuint32_t)KC, (cuuint32_t)(2 * Cout_pad)};     // the tiles py = 0, 1 of one (slab, px, b, a)
        cuuint32_t es[2] = {1, 1};
        CUresult r = fn(&L->tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)wgt_fold, dims, strides, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(KC), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return v2e_set_error(V2E_E_CUDA, "cuTensorMapEncodeTiled failed for folded weights%s", "");
    }
    L->smem = (size_t)((p.w_bytes + 1023) & ~1023) + (size_t)p.nslot * p.slab_bytes * slabs + 1024;
    L->grid = p.n_items < n_sms ? p.n_items : n_sms;
    L->low = (const __half *)x_low;
    L->w_plain = (const __half *)wgt_plain;
    L->C = C;
    return V2E_OK;
}

int v2e_conv_up2_launch(const V2eUpLaunch *L, cudaStream_t st) {
    static PerDeviceOnce attr_once;
    if (attr_once.first()) cudaFuncSetAttribute(conv_up2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    conv_up2_kernel<<<L->grid, kStripThreads, L->smem, st>>>(L->tmA, L->tmB, L->p);
    // the 2-pixel frame, where clamping / zero padding break the shift invariance the folding relies on
    const StripParams &p = L->p;
    const size_t bsm = 32 * 9 * 64 * 2;
    static PerDeviceOnce battr_once;
    if (battr_once.first()) cudaFuncSetAttribute(conv_up2_border_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bsm);
    conv_up2_border_kernel<<<L->grid * kBorderBlocks, kBorderThreads, bsm, st>>>(L->low, L->w_plain, p.bias, (__half *)p.out,
                                                                                 p.N, p.H, p.W, p.out_cstride, p.slope);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "conv_up2_kernel launch: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_conv2d_up2_lrelu_sm100(const void *x_low_dev, int C, const void *wgt_fold_dev, const void *wgt_plain_dev,
                                          const float *bias_dev, int Cout_pad, int N, int H_out, int W_out, void *out_dev,
                                          int out_cstride, float slope, void *stream) {
    V2eUpLaunch L;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int rc = v2e_conv_up2_prepare(&L, x_low_dev, C, wgt_fold_dev, wgt_plain_dev, bias_dev, Cout_pad, N, H_out, W_out, out_dev,
                                  out_cstride, slope, sms);
    if (rc) return rc;
    return v2e_conv_up2_launch(&L, (cudaStream_t)stream);
}

extern "C" int v2e_conv_up2_supported_c(int C, int Cout_pad, int W_out) { return v2e_conv_up2_supported(C, Cout_pad, W_out); }

extern "C" int v2e_conv_strip_pick_kc(int C1, int C2, int Cout_pad, int KH, int KW, int W) {
    return v2e_strip_pick(C1, C2, Cout_pad, KH, KW, W, nullptr);
}
