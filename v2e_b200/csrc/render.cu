// DVS frame rendering for sm_90a (H100) (SURVEY.md 8f rank 4): the reference's
// EventRenderer.render_events_to_frames (v2ecore/renderer.py:161-430 -> accumulate_event_frame :392-430 ->
// hist2d_numba_seq, v2ecore/v2e_utils.py:474-486) over many packets per call.
//   1. The frame plan (v2e_render_plan; v2e_render_area_scan for AREA_COUNT): which rows of which packet every finished
//      frame takes (exposure by duration / count / area / source frame, with the reference's end-of-packet rule), and
//      the time the frame-times file states for it.
//   2. The frames (v2e_render_frames, over chunks of the plan): per frame, ON count minus OFF count per pixel of the
//      frame's slice (scatter-add with integer atomics), clipped to +-full_scale_count, returned as (frame + fs) / (2 fs)
//      in float64 and, for the video file, (img * 255) truncated to uint8 (renderer.py:345-347).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/v2e_b200.h"

int v2e_set_error(int code, const char *fmt, const char *detail);
#define CU(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess) return v2e_set_error(V2E_E_CUDA, #call ": %s", cudaGetErrorString(e_)); \
    } while (0)

namespace {

// frames grid-stride in y (a packet may finish more frames than gridDim.y can hold); events [start, end) of a frame,
// grid-stride in x
__global__ void __launch_bounds__(256)
render_scatter_kernel(const float4 *__restrict__ ev, const int64_t *__restrict__ starts, const int64_t *__restrict__ ends,
                      int n_frames, int H, int W, int32_t *__restrict__ acc) {
    for (int f = blockIdx.y; f < n_frames; f += gridDim.y) {
        const int64_t s = starts[f], e = ends[f];
        int32_t *a = acc + (size_t)f * H * W;
        for (int64_t i = s + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (int64_t)gridDim.x * blockDim.x) {
            const float4 r = ev[i];                     // [t, x, y, p]
            // hist2d_numba_seq: i = y * delta with delta = 1 / ((H - 0) / H) = 1: bin = int(y) if 0 <= y < H
            const double yy = (double)r.z, xx = (double)r.y;
            if (yy >= 0.0 && yy < (double)H && xx >= 0.0 && xx < (double)W)
                atomicAdd(&a[(int)yy * W + (int)xx], r.w == 1.0f ? 1 : -1);     // pol_on = (p == 1), everything else is OFF
        }
    }
}

__global__ void __launch_bounds__(256)
render_finish_kernel(const int32_t *__restrict__ acc, size_t n, int fs, double *__restrict__ img, uint8_t *__restrict__ u8) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int v = acc[i];
    v = v < -fs ? -fs : (v > fs ? fs : v);                                  // np.clip, renderer.py:427-429
    const double x = ((double)v + (double)fs) / (double)(fs * 2);           // normalize_frame, renderer.py:239-241
    if (img) img[i] = x;
    if (u8) u8[i] = (uint8_t)(x * 255.0);                                   // (img * 255).astype(np.uint8)
}

// ---- the frame plan: which rows of which packet each finished frame takes, and the time the frame-times file states
// A call renders P packets, each a row range [b, e) of one of two row arrays: packet 0 of rows0 when first_from_rows0
// (the packet that straddles the previous call, assembled by the caller), every other of rows. The plan is, for every
// frame any packet finishes, in packet order: starts / ends (row indices into the packet's array; end-exclusive), the
// frame time (double, holding the float32 or float64 value the reference computes) and, in hdr, the status, the frame
// count, the largest slice and the carried DURATION state. packet_first[p] is the index of packet p's first frame.
enum { PLAN_OK = 0, PLAN_CAPACITY = 1, PLAN_SPAN = 2 };
enum { H_STATUS, H_FRAMES, H_MAX_SLICE, H_CUR, H_HAS_CUR, H_BAD_PACKET, H_BAD_FROM, H_BAD_TO, H_WORDS };
enum { MODE_DURATION = 1, MODE_COUNT = 2, MODE_AREA_COUNT = 3, MODE_SOURCE = 4 };
constexpr int64_t kMaxSpan = int64_t(1) << 20;          // frame intervals one DURATION packet may span

__device__ __forceinline__ const float4 *packet_rows(const float4 *rows0, const float4 *rows, int first_from_rows0, int p) {
    return p == 0 && first_from_rows0 ? rows0 : rows;
}

__device__ __forceinline__ int64_t as_bits(double v) { return __double_as_longlong(v); }

// next DURATION frame start: cur + interval in the dtype the reference accumulates it in (float32 for a Python-float
// interval added to the first row's float32 time, renderer.py:205, 316; float64 for a float64 interval)
__device__ __forceinline__ double next_start(double c, double interval, float interval_f, int f64) {
    return f64 ? __dadd_rn(c, interval) : (double)__fadd_rn((float)c, interval_f);
}

// Serial part of DURATION / COUNT / SOURCE (one thread): the frame counts of every packet and, for DURATION, the chain
// of frame starts. The starts form one sequence over the clip (c(m+1) = c(m) + interval, from the first row's time);
// each packet resumes at the first start it did not finish. Frame j of a packet of n rows is finished iff
// searchsorted(ts, c(j+1), 'right') < n - 1, i.e. c(j+1) < ts[n - 2]; the packet's chain runs while c <= ts[n - 1],
// and more than kMaxSpan starts there refuse the call (renderer.py:316-326).
__global__ void render_plan_kernel(const float4 *__restrict__ rows0, const float4 *__restrict__ rows,
                                   const int64_t *__restrict__ packets, int P, int first_from_rows0, int mode,
                                   double interval, float interval_f, int f64, int64_t count, double cur, int has_cur,
                                   double2 *__restrict__ bounds, int64_t max_frames, int64_t *__restrict__ hdr,
                                   int64_t *__restrict__ packet_first) {
    if (blockIdx.x || threadIdx.x) return;
    int64_t F = 0;
    int status = PLAN_OK;
    for (int p = 0; p < P; p++) {
        packet_first[p] = F;
        const float4 *ev = packet_rows(rows0, rows, first_from_rows0, p);
        const int64_t b = packets[2 * p], n = packets[2 * p + 1] - b;
        if (n <= 0) continue;
        if (mode == MODE_SOURCE) {
            F += 1;                                                 // [0, n - 1), emitted even when empty
        } else if (mode == MODE_COUNT) {
            F += n >= 2 ? (n - 2) / count : 0;                      // frame j finished iff (j + 1) count < n - 1
        } else {
            if (!has_cur) {
                cur = (double)ev[b].x;
                has_cur = 1;
            }
            const double t1 = (double)ev[b + n - 1].x;
            const bool any = n >= 2;
            const double stop = any ? (double)ev[b + n - 2].x : 0.0;
            double c = cur, prev = cur, next = cur;
            for (int64_t m = 0; c <= t1; m++) {
                if (m + 1 >= kMaxSpan) {
                    status = PLAN_SPAN;
                    hdr[H_BAD_PACKET] = p;
                    hdr[H_BAD_FROM] = as_bits(cur);
                    hdr[H_BAD_TO] = as_bits(t1);
                    break;
                }
                if (m >= 1 && any && c < stop) {                    // frame m - 1 = [prev, c] is finished
                    if (F < max_frames) bounds[F] = make_double2(prev, c);
                    F++;
                    next = c;
                }
                prev = c;
                c = next_start(c, interval, interval_f, f64);
            }
            if (status != PLAN_OK) break;
            cur = next;
        }
    }
    for (int p = status == PLAN_OK ? P : 0; p <= P; p++) packet_first[p] = F;
    if (status == PLAN_OK && F > max_frames) status = PLAN_CAPACITY;
    hdr[H_STATUS] = status;
    hdr[H_FRAMES] = F;
    hdr[H_MAX_SLICE] = 0;
    hdr[H_CUR] = as_bits(cur);
    hdr[H_HAS_CUR] = has_cur;
}

// ExposureMode.AREA_COUNT (renderer.py:246-261, 287-291): a frame ends when any area_dimension x area_dimension cell
// has collected area_count events. Inherently sequential (every event depends on the counters the previous ones left,
// and the counters are cleared when a frame ends), so ONE thread walks the P packets in order; the counters persist
// between packets and calls like the reference's self.area_counts. Writes the slices of the finished frames with the
// reference's end-of-packet rule per packet (end >= n - 1 -> stop; the last event of a packet is never rendered).
__global__ void render_area_scan_kernel(const float4 *__restrict__ rows0, const float4 *__restrict__ rows,
                                        const int64_t *__restrict__ packets, int P, int first_from_rows0, int area_dim,
                                        int area_count, int nw, int nh, int32_t *__restrict__ counts,
                                        int64_t *__restrict__ starts, int64_t *__restrict__ ends, int64_t max_frames,
                                        int64_t *__restrict__ hdr, int64_t *__restrict__ packet_first) {
    if (blockIdx.x || threadIdx.x) return;
    int64_t k = 0;
    for (int p = 0; p < P; p++) {
        packet_first[p] = k;
        const float4 *ev = packet_rows(rows0, rows, first_from_rows0, p) + packets[2 * p];
        const int64_t n = packets[2 * p + 1] - packets[2 * p];
        int64_t idx = 0;
        while (n > 0) {
            int64_t e = idx;
            for (e = idx; e < n; e++) {
                const float4 r = ev[e];
                const int x = (int)floorf(r.y / (float)area_dim), y = (int)floorf(r.z / (float)area_dim);
                if (x < 0 || x >= nw || y < 0 || y >= nh) continue;     // cannot happen for in-frame events
                const int c = 1 + counts[x * nh + y];
                counts[x * nh + y] = c;
                if (c >= area_count) {
                    for (int i = 0; i < nw * nh; i++) counts[i] = 0;
                    break;
                }
            }
            int64_t end = e < n ? e : n - 1;                            // numba leaves the loop variable at the last index
            if (idx >= n) end = idx;                                    // empty range: ev_idx = start
            if (end >= n - 1) break;                                    // the rest stays in the (dropped) current frame
            if (k < max_frames) {
                starts[k] = packets[2 * p] + idx;
                ends[k] = packets[2 * p] + end;
            }
            k++;
            idx = end;
        }
    }
    packet_first[P] = k;
    hdr[H_STATUS] = k > max_frames ? PLAN_CAPACITY : PLAN_OK;
    hdr[H_FRAMES] = k;
    hdr[H_MAX_SLICE] = 0;
}

// Parallel part, one thread per planned frame: its packet (binary search of packet_first), its slice (DURATION: the
// searchsorted left / right of its two starts over the packet's rows; COUNT: j * count .. (j + 1) * count; SOURCE:
// 0 .. n - 1), its time and the largest slice. AREA_COUNT frames come with their slices; only time and size here.
__global__ void __launch_bounds__(256)
render_plan_slices_kernel(const float4 *__restrict__ rows0, const float4 *__restrict__ rows,
                          const int64_t *__restrict__ packets, int P, int first_from_rows0, int mode, double half,
                          float half_f, int f64, int64_t count, const double2 *__restrict__ bounds,
                          int64_t *__restrict__ starts, int64_t *__restrict__ ends, double *__restrict__ times,
                          int64_t *__restrict__ hdr, const int64_t *__restrict__ packet_first) {
    if (hdr[H_STATUS] != PLAN_OK) return;
    const int64_t F = hdr[H_FRAMES];
    int64_t big = 0;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = P;                                             // last p with packet_first[p] <= f
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (packet_first[mid] <= f) lo = mid; else hi = mid;
        }
        const int p = lo;
        const float4 *ev = packet_rows(rows0, rows, first_from_rows0, p);
        const int64_t b = packets[2 * p], n = packets[2 * p + 1] - b;
        const int64_t j = f - packet_first[p];
        int64_t s, e;
        double t;
        if (mode == MODE_DURATION) {
            const double2 c = bounds[f];
            int64_t a0 = 0, a1 = n;                                     // first row with ts >= c.x
            while (a0 < a1) {
                const int64_t m = (a0 + a1) >> 1;
                if ((double)ev[b + m].x < c.x) a0 = m + 1; else a1 = m;
            }
            s = a0;
            a1 = n;                                                     // first row with ts > c.y (c.y > c.x)
            while (a0 < a1) {
                const int64_t m = (a0 + a1) >> 1;
                if ((double)ev[b + m].x <= c.y) a0 = m + 1; else a1 = m;
            }
            e = a0;
            t = f64 ? __dadd_rn(c.y, half) : (double)__fadd_rn((float)c.y, half_f);
        } else if (mode == MODE_SOURCE) {
            s = 0;
            e = n - 1;
            t = (double)ev[b].x;
        } else {
            if (mode == MODE_COUNT) {
                s = j * count;
                e = s + count;
            } else {
                s = starts[f] - b;
                e = ends[f] - b;
            }
            t = (double)__fdiv_rn(__fadd_rn(ev[b + s].x, ev[b + e].x), 2.0f);     // float32 (ts[s] + ts[e]) / 2
        }
        starts[f] = b + s;
        ends[f] = b + e;
        times[f] = t;
        big = e - s > big ? e - s : big;
    }
    if (big > 0) atomicMax((unsigned long long *)&hdr[H_MAX_SLICE], (unsigned long long)big);
}

}  // namespace

static int plan_slices(const float4 *rows0, const float4 *rows, const int64_t *packets, int P, int first_from_rows0,
                       int mode, double half, int f64, int64_t count, const double2 *bounds, int64_t *starts,
                       int64_t *ends, double *times, int64_t max_frames, int64_t *hdr, const int64_t *packet_first,
                       cudaStream_t st) {
    int blocks = (int)((max_frames + 255) / 256);
    blocks = blocks < 1 ? 1 : (blocks > 264 ? 264 : blocks);
    render_plan_slices_kernel<<<blocks, 256, 0, st>>>(rows0, rows, packets, P, first_from_rows0, mode, half, (float)half,
                                                      f64, count, bounds, starts, ends, times, hdr, packet_first);
    CU(cudaGetLastError());
    return V2E_OK;
}

extern "C" int v2e_render_plan(const float *rows0_dev, const float *rows_dev, const int64_t *packets_dev, int n_packets,
                               int first_from_rows0, int exposure_mode, double interval, int f64_starts, int64_t count,
                               double cur, int has_cur, double *bounds_dev, int64_t *starts_dev, int64_t *ends_dev,
                               double *times_dev, int64_t max_frames, int64_t *hdr_dev, int64_t *packet_first_dev,
                               void *stream) {
    if (!packets_dev || n_packets < 1 || !starts_dev || !ends_dev || !times_dev || !hdr_dev || !packet_first_dev ||
        max_frames < 1 || (first_from_rows0 && !rows0_dev) || (n_packets > (first_from_rows0 ? 1 : 0) && !rows_dev) ||
        (exposure_mode != MODE_DURATION && exposure_mode != MODE_COUNT && exposure_mode != MODE_SOURCE) ||
        (exposure_mode == MODE_DURATION && (!bounds_dev || !(interval > 0.0))) || (exposure_mode == MODE_COUNT && count < 1))
        return v2e_set_error(V2E_E_INVALID, "bad render-plan arguments%s", "");
    if (((uintptr_t)rows0_dev & 15) || ((uintptr_t)rows_dev & 15))
        return v2e_set_error(V2E_E_INVALID, "rows must be 16-byte aligned device arrays%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    const float4 *r0 = (const float4 *)rows0_dev, *r = (const float4 *)rows_dev;
    // interval / 2 as the reference adds it: a Python float, rounded to float32 for a float32 chain
    const double half = f64_starts ? interval / 2 : (double)(float)(interval / 2);
    render_plan_kernel<<<1, 32, 0, st>>>(r0, r, packets_dev, n_packets, first_from_rows0, exposure_mode, interval,
                                         (float)interval, f64_starts, count, cur, has_cur, (double2 *)bounds_dev,
                                         max_frames, hdr_dev, packet_first_dev);
    CU(cudaGetLastError());
    return plan_slices(r0, r, packets_dev, n_packets, first_from_rows0, exposure_mode, half, f64_starts, count,
                       (const double2 *)bounds_dev, starts_dev, ends_dev, times_dev, max_frames, hdr_dev,
                       packet_first_dev, st);
}

extern "C" int v2e_render_area_scan(const float *rows0_dev, const float *rows_dev, const int64_t *packets_dev,
                                    int n_packets, int first_from_rows0, int area_dimension, int area_count,
                                    int cells_w, int cells_h, int32_t *counts_dev, int64_t *starts_dev,
                                    int64_t *ends_dev, double *times_dev, int64_t max_frames, int64_t *hdr_dev,
                                    int64_t *packet_first_dev, void *stream) {
    if (!packets_dev || n_packets < 1 || !counts_dev || !starts_dev || !ends_dev || !times_dev || !hdr_dev ||
        !packet_first_dev || area_dimension < 1 || area_count < 1 || cells_w < 1 || cells_h < 1 || max_frames < 1 ||
        (first_from_rows0 && !rows0_dev) || (n_packets > (first_from_rows0 ? 1 : 0) && !rows_dev))
        return v2e_set_error(V2E_E_INVALID, "bad area-scan arguments%s", "");
    if (((uintptr_t)rows0_dev & 15) || ((uintptr_t)rows_dev & 15))
        return v2e_set_error(V2E_E_INVALID, "rows must be 16-byte aligned device arrays%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    const float4 *r0 = (const float4 *)rows0_dev, *r = (const float4 *)rows_dev;
    render_area_scan_kernel<<<1, 32, 0, st>>>(r0, r, packets_dev, n_packets, first_from_rows0, area_dimension, area_count,
                                              cells_w, cells_h, counts_dev, starts_dev, ends_dev, max_frames, hdr_dev,
                                              packet_first_dev);
    CU(cudaGetLastError());
    return plan_slices(r0, r, packets_dev, n_packets, first_from_rows0, MODE_AREA_COUNT, 0.0, 0, 0, nullptr, starts_dev,
                       ends_dev, times_dev, max_frames, hdr_dev, packet_first_dev, st);
}

extern "C" int v2e_render_frames(const float *events_dev, const int64_t *starts_dev, const int64_t *ends_dev, int n_frames,
                                 int64_t max_events_per_frame, int height, int width, int full_scale_count,
                                 int32_t *acc_dev, double *frames_f64_dev, uint8_t *frames_u8_dev, void *stream) {
    if (!starts_dev || !ends_dev || !acc_dev || n_frames < 1 || height < 1 || width < 1 || full_scale_count < 1)
        return v2e_set_error(V2E_E_INVALID, "bad render arguments%s", "");
    if (max_events_per_frame > 0 && (!events_dev || ((uintptr_t)events_dev & 15)))
        return v2e_set_error(V2E_E_INVALID, "events must be a 16-byte aligned device array%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)n_frames * height * width;
    CU(cudaMemsetAsync(acc_dev, 0, n * sizeof(int32_t), st));
    if (max_events_per_frame > 0) {
        int gx = (int)((max_events_per_frame + 255) / 256);
        if (gx > 1184) gx = 1184;
        if (gx < 1) gx = 1;
        dim3 grid(gx, n_frames < 65535 ? n_frames : 65535);
        render_scatter_kernel<<<grid, 256, 0, st>>>((const float4 *)events_dev, starts_dev, ends_dev, n_frames, height, width,
                                                    acc_dev);
    }
    render_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(acc_dev, n, full_scale_count, frames_f64_dev, frames_u8_dev);
    CU(cudaGetLastError());
    return V2E_OK;
}
