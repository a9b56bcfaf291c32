// DVS frame rendering for sm_90a (H100) (SURVEY.md 8f rank 4): the histogram part of the reference's
// EventRenderer.render_events_to_frames (v2ecore/renderer.py:161-430 -> accumulate_event_frame :392-430 ->
// hist2d_numba_seq, v2ecore/v2e_utils.py:474-486): per output frame, ON count minus OFF count per pixel of the events
// of the frame's slice, clipped to +-full_scale_count, returned as (frame + fs) / (2 fs) in float64 (and, for the
// video file, (img * 255) truncated to uint8, renderer.py:345-347). Which events belong to which frame (exposure by
// duration / count / source frame, and the reference's end-of-packet rule) is decided by the caller
// (v2e_b200/renderer.py); here: scatter-add with integer atomics, then one normalising pass.
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

// ExposureMode.AREA_COUNT (renderer.py:246-261, 287-291): a frame ends when any area_dimension x area_dimension
// cell has collected area_count events. Inherently sequential (every event depends on the counters the previous ones
// left, and the counters are cleared when a frame ends), so ONE thread walks the packet; the counters persist between
// packets like the reference's self.area_counts. Writes the slices of the finished frames with the reference's
// end-of-packet rule (end >= n - 1 -> stop; the last event of a packet is never rendered).
__global__ void render_area_scan_kernel(const float4 *__restrict__ ev, int64_t n, int area_dim, int area_count, int nw, int nh,
                                        int32_t *__restrict__ counts, int64_t *__restrict__ starts, int64_t *__restrict__ ends,
                                        int max_frames, int32_t *__restrict__ n_frames) {
    if (blockIdx.x || threadIdx.x) return;
    int k = 0;
    int64_t idx = 0;
    bool overflow = false;
    while (true) {
        int64_t e = idx;
        for (e = idx; e < n; e++) {
            const float4 r = ev[e];
            const int x = (int)floorf(r.y / (float)area_dim), y = (int)floorf(r.z / (float)area_dim);
            if (x < 0 || x >= nw || y < 0 || y >= nh) continue;         // cannot happen for in-frame events
            const int c = 1 + counts[x * nh + y];
            counts[x * nh + y] = c;
            if (c >= area_count) {
                for (int i = 0; i < nw * nh; i++) counts[i] = 0;
                break;
            }
        }
        int64_t end = e < n ? e : n - 1;                                // numba leaves the loop variable at the last index
        if (idx >= n) end = idx;                                        // empty range: ev_idx = start
        if (end >= n - 1) break;                                        // the rest stays in the (dropped) current frame
        if (k >= max_frames) { overflow = true; break; }
        starts[k] = idx;
        ends[k] = end;
        k++;
        idx = end;
    }
    *n_frames = overflow ? -1 : k;
}

}  // namespace

extern "C" int v2e_render_area_scan(const float *events_dev, int64_t n, int area_dimension, int area_count, int cells_w,
                                    int cells_h, int32_t *counts_dev, int64_t *starts_dev, int64_t *ends_dev,
                                    int max_frames, int32_t *n_frames_dev, void *stream) {
    if (!events_dev || !counts_dev || !starts_dev || !ends_dev || !n_frames_dev || n < 1 || area_dimension < 1 ||
        area_count < 1 || cells_w < 1 || cells_h < 1 || max_frames < 1)
        return v2e_set_error(V2E_E_INVALID, "bad area-scan arguments%s", "");
    render_area_scan_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((const float4 *)events_dev, n, area_dimension, area_count, cells_w,
                                                                 cells_h, counts_dev, starts_dev, ends_dev, max_frames, n_frames_dev);
    CU(cudaGetLastError());
    return V2E_OK;
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
