// Stage-1 input preparation for sm_90a (H100) (SURVEY.md 8f rank 2): v2e.py:687-737 --
//     frame[c_t:c_b, c_l:c_r] -> cv2.resize(dsize, interpolation=cv2.INTER_AREA) -> cv2.cvtColor(BGR2GRAY)
// for 8-bit frames, bit-exact with OpenCV 4.x (restated in oracle/prep_oracle.py, pinned against cv2's own output):
//   * integer scale factors (resize.cpp, resizeAreaFast_Invoker): integer box sum * float32(1/area), rounded half to
//     even; the 2x2 box is (s + 2) >> 2 (its SIMD path);
//   * fractional shrink (computeResizeAreaTab + ResizeArea_Invoker): float32 accumulation, horizontally
//     buf += S * alpha in table order, vertically sum += beta * buf in row order, separate multiply and add;
//   * luma (RGB2Gray<uchar>): (B * 3735 + G * 19235 + R * 9798 + (1 << 14)) >> 15.
// HBM-bound streaming kernel: one thread per output pixel reads its (scale_x x scale_y) source box once -- the box of
// the neighbouring thread is adjacent, so a warp reads contiguous source rows -- and writes one byte.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../include/v2e_b200.h"

int v2e_set_error(int code, const char *fmt, const char *detail);
#define CU(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess) return v2e_set_error(V2E_E_CUDA, #call ": %s", cudaGetErrorString(e_)); \
    } while (0)

namespace {

struct Tap { int32_t si; float alpha; };       // source index (pixels), weight

struct PrepDev {
    int sw, sh, cn, pitch;                      // cropped source size, channels, bytes per source row (uncropped)
    long img_stride;                            // bytes between source images
    long src_off;                               // byte offset of the crop's first pixel
    int dw, dh;
    int mode;                                   // 0 copy (no resize), 1 integer boxes, 2 fractional shrink
    int isx, isy;                               // mode 1
    float inv_area;
    const int32_t *xofs, *yofs;                 // mode 2: [dw + 1] / [dh + 1] offsets into the tap tables
    const Tap *xtab, *ytab;
};

__device__ __forceinline__ uint8_t round_u8(float v) {          // saturate_cast<uchar>: cvRound, clamped
    int r = __float2int_rn(v);
    return (uint8_t)(r < 0 ? 0 : (r > 255 ? 255 : r));
}
__device__ __forceinline__ uint8_t luma(int b, int g, int r) {
    return (uint8_t)((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15);
}

template <int CN>
__global__ void __launch_bounds__(256) prep_kernel(PrepDev p, const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, int n_img) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long per = (long)p.dw * p.dh;
    if (i >= per * n_img) return;
    const int img = (int)(i / per);
    const int dy = (int)((i - (long)img * per) / p.dw), dx = (int)(i % p.dw);
    const uint8_t *s = src + (long)img * p.img_stride + p.src_off;
    int v[CN];
    if (p.mode == 0) {
#pragma unroll
        for (int c = 0; c < CN; c++) v[c] = s[(long)dy * p.pitch + dx * CN + c];
    } else if (p.mode == 1) {
        int sum[CN];
#pragma unroll
        for (int c = 0; c < CN; c++) sum[c] = 0;
        for (int yy = 0; yy < p.isy; yy++) {
            const uint8_t *row = s + (long)(dy * p.isy + yy) * p.pitch + (long)dx * p.isx * CN;
            for (int xx = 0; xx < p.isx; xx++)
#pragma unroll
                for (int c = 0; c < CN; c++) sum[c] += row[xx * CN + c];
        }
#pragma unroll
        for (int c = 0; c < CN; c++)
            v[c] = (p.isx == 2 && p.isy == 2) ? ((sum[c] + 2) >> 2) : (int)round_u8(__fmul_rn((float)sum[c], p.inv_area));
    } else {
        float acc[CN];
        const int y0 = p.yofs[dy], y1 = p.yofs[dy + 1], x0 = p.xofs[dx], x1 = p.xofs[dx + 1];
        for (int j = y0; j < y1; j++) {
            const Tap ty = p.ytab[j];
            const uint8_t *row = s + (long)ty.si * p.pitch;
            float buf[CN];
#pragma unroll
            for (int c = 0; c < CN; c++) buf[c] = 0.f;
            for (int k = x0; k < x1; k++) {
                const Tap tx = p.xtab[k];
#pragma unroll
                for (int c = 0; c < CN; c++)
                    buf[c] = __fadd_rn(buf[c], __fmul_rn((float)row[tx.si * CN + c], tx.alpha));      // no fused multiply-add
            }
#pragma unroll
            for (int c = 0; c < CN; c++) {
                const float t = __fmul_rn(ty.alpha, buf[c]);
                acc[c] = j == y0 ? t : __fadd_rn(acc[c], t);
            }
        }
#pragma unroll
        for (int c = 0; c < CN; c++) v[c] = round_u8(acc[c]);
    }
    dst[i] = CN == 3 ? luma(v[0], v[1], v[2]) : (uint8_t)v[0];
}

// computeResizeAreaTab (resize.cpp), per destination index
void area_tab(int ssize, int dsize, double scale, std::vector<int32_t> &ofs, std::vector<Tap> &tab) {
    ofs.assign((size_t)dsize + 1, 0);
    tab.clear();
    for (int dx = 0; dx < dsize; dx++) {
        ofs[dx] = (int32_t)tab.size();
        const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
        const double cell = scale < ssize - fsx1 ? scale : ssize - fsx1;
        int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
        if (sx2 > ssize - 1) sx2 = ssize - 1;
        if (sx1 > sx2) sx1 = sx2;
        if (sx1 - fsx1 > 1e-3) tab.push_back({sx1 - 1, (float)((sx1 - fsx1) / cell)});
        for (int sx = sx1; sx < sx2; sx++) tab.push_back({sx, float(1.0 / cell)});
        if (fsx2 - sx2 > 1e-3) {
            double w = fsx2 - sx2;
            if (w > 1.) w = 1.;
            if (w > cell) w = cell;
            tab.push_back({sx2, (float)(w / cell)});
        }
    }
    ofs[dsize] = (int32_t)tab.size();
}

}  // namespace

struct V2ePrep {
    PrepDev d;
    int full_w, full_h;
    void *bufs[4];
};

extern "C" int v2e_prep_create(int src_w, int src_h, int channels, int crop_left, int crop_right, int crop_top,
                               int crop_bottom, int dst_w, int dst_h, V2ePrep **out) {
    if (!out || src_w < 1 || src_h < 1 || dst_w < 1 || dst_h < 1) return v2e_set_error(V2E_E_INVALID, "bad size%s", "");
    if (channels != 1 && channels != 3) return v2e_set_error(V2E_E_INVALID, "channels must be 1 (grey) or 3 (BGR)%s", "");
    // v2e.py:646-649, 702: frame[c_t:c_b, c_l:c_r] with c_r = -right, c_b = -bottom
    const int cl = crop_left > 0 ? crop_left : 0, cr = crop_right > 0 ? crop_right : 0;
    const int ct = crop_top > 0 ? crop_top : 0, cb = crop_bottom > 0 ? crop_bottom : 0;
    const int sw = src_w - cl - cr, sh = src_h - ct - cb;
    if (sw < 1 || sh < 1) return v2e_set_error(V2E_E_INVALID, "crop is larger than the frame%s", "");
    const double scale_x = (double)sw / dst_w, scale_y = (double)sh / dst_h;
    V2ePrep *h = new V2ePrep();
    memset(h, 0, sizeof(*h));
    PrepDev &d = h->d;
    h->full_w = src_w;
    h->full_h = src_h;
    d.sw = sw; d.sh = sh; d.cn = channels; d.pitch = src_w * channels;
    d.img_stride = (long)src_w * src_h * channels;
    d.src_off = (long)ct * d.pitch + (long)cl * channels;
    d.dw = dst_w; d.dh = dst_h;
    if (sw == dst_w && sh == dst_h) {
        d.mode = 0;
    } else {
        if (scale_x < 1.0 || scale_y < 1.0) {
            delete h;
            return v2e_set_error(V2E_E_UNSUPPORTED, "INTER_AREA enlargement (OpenCV's bilinear path) is not built%s", "");
        }
        const int isx = (int)lrint(scale_x), isy = (int)lrint(scale_y);
        if (fabs(scale_x - isx) < 2.220446049250313e-16 && fabs(scale_y - isy) < 2.220446049250313e-16) {
            d.mode = 1; d.isx = isx; d.isy = isy;
            d.inv_area = 1.f / (float)(isx * isy);
        } else {
            d.mode = 2;
            std::vector<int32_t> xo, yo;
            std::vector<Tap> xt, yt;
            area_tab(sw, dst_w, scale_x, xo, xt);
            area_tab(sh, dst_h, scale_y, yo, yt);
            const void *hs[4] = {xo.data(), yo.data(), xt.data(), yt.data()};
            const size_t bs[4] = {xo.size() * 4, yo.size() * 4, xt.size() * sizeof(Tap), yt.size() * sizeof(Tap)};
            for (int i = 0; i < 4; i++) {
                if (cudaMalloc(&h->bufs[i], bs[i]) != cudaSuccess ||
                    cudaMemcpy(h->bufs[i], hs[i], bs[i], cudaMemcpyHostToDevice) != cudaSuccess) {
                    for (int k = 0; k <= i; k++) if (h->bufs[k]) cudaFree(h->bufs[k]);
                    delete h;
                    return v2e_set_error(V2E_E_CUDA, "v2e_prep_create: %s", cudaGetErrorString(cudaGetLastError()));
                }
            }
            d.xofs = (const int32_t *)h->bufs[0]; d.yofs = (const int32_t *)h->bufs[1];
            d.xtab = (const Tap *)h->bufs[2]; d.ytab = (const Tap *)h->bufs[3];
        }
    }
    *out = h;
    return V2E_OK;
}

extern "C" int v2e_prep_destroy(V2ePrep *h) {
    if (!h) return V2E_OK;
    for (int i = 0; i < 4; i++) if (h->bufs[i]) cudaFree(h->bufs[i]);
    delete h;
    return V2E_OK;
}

extern "C" int v2e_prep_run(V2ePrep *h, const uint8_t *src_dev, int n_images, uint8_t *dst_dev, void *stream) {
    if (!h || !src_dev || !dst_dev || n_images < 1) return v2e_set_error(V2E_E_INVALID, "bad argument%s", "");
    const long n = (long)h->d.dw * h->d.dh * n_images;
    const int grid = (int)((n + 255) / 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (h->d.cn == 3) prep_kernel<3><<<grid, 256, 0, st>>>(h->d, src_dev, dst_dev, n_images);
    else prep_kernel<1><<<grid, 256, 0, st>>>(h->d, src_dev, dst_dev, n_images);
    CU(cudaGetLastError());
    return V2E_OK;
}
