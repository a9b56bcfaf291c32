// SuperSloMo frame interpolation for sm_90a (H100): everything of v2ecore/slomo.py:330-444 and
// v2ecore/model.py:158-300 that runs per frame pair, behind the C ABI in include/v2e_b200.h.
//
//   set_pairs : uint8 frames (net resolution) -> normalised fp32 images (slomo.py:148-162: x/255 - 0.428)
//               -> flow UNet(2,4) (slomo.py:343) -> F_0_1 | F_1_0 (fp32)
//   interp(t) : flow coefficients, two back-warps, 12-channel input (slomo.py:405-419)
//               -> interpolation UNet(12,5) -> residual flows, visibility, two back-warps, blend
//               (slomo.py:421-433) -> (x+0.428)*255 -> uint8 truncation (slomo.py:437, torchvision ToPILImage)
// UNet convolutions: conv_tc.cu (wgmma implicit GEMM, fp16 operands, fp32 accumulate). avg_pool2d
// (model.py:72) and bilinear x2 (model.py:137-140) are NHWC fp16 streaming kernels here; the channel
// concat of the up-blocks (model.py:150-153) is never materialised (the conv reads two tensors).
// Also here: Pillow-exact 8-bit resampling (dataloader.py:142 LANCZOS, slomo.py:438 BILINEAR).
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

// ---- from conv_tc.cu ------------------------------------------------------------------------------
struct V2eConvLaunch;
int v2e_conv_prepare(V2eConvLaunch *L, const void *x1, int C1, const void *x2, int C2, const void *wgt,
                     const float *bias, int Cout_pad, int KH, int KW, int N, int H, int W, void *out,
                     int out_cstride, int out_mode, int co_real, float slope, int tile, int n_sms);
int v2e_conv_launch(const V2eConvLaunch *L, cudaStream_t st);
size_t v2e_conv_launch_size(void);
struct V2eStripLaunch;
int v2e_strip_pick(int C1, int C2, int Cout_pad, int KH, int KW, int W, int *nslot_out);
size_t v2e_strip_launch_size(void);
int v2e_strip_pool_supported(int C1, int C2, int Cout_pad, int KH, int KW, int H, int W);
int v2e_strip_prepare(V2eStripLaunch *L, const void *x1, int C1, const void *x2, int C2, const void *wgt_row,
                      const float *bias, int Cout_pad, int KH, int KW, int N, int H, int W, void *out,
                      int out_cstride, int out_mode, int co_real, float slope, int n_sms, void *pool_out,
                      int pool_cstride, int chain);
int v2e_strip_launch(const V2eStripLaunch *L, cudaStream_t st);
struct V2eUpLaunch;
int v2e_conv_up2_supported(int C, int Cout_pad, int W_out);
extern "C" int v2e_conv_up2_fold_weights(const float *w, int cout, int cin, int Cout_pad, int C_pad, void *out_host);
size_t v2e_conv_up2_launch_size(void);
int v2e_conv_up2_prepare(V2eUpLaunch *L, const void *x_low, int C, const void *wgt_fold, const void *wgt_plain,
                         const float *bias, int Cout_pad, int N, int H, int W, void *out, int out_cstride, float slope,
                         int n_sms);
int v2e_conv_up2_launch(const V2eUpLaunch *L, cudaStream_t st);
int v2e_set_error(int code, const char *fmt, const char *detail);

#define CU(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess) return v2e_set_error(V2E_E_CUDA, #call ": %s", cudaGetErrorString(e_)); \
    } while (0)

namespace {

constexpr float kMean = 0.428f;         // slomo.py:148
constexpr float kSlope = 0.1f;          // model.py: negative_slope=0.1 everywhere

// ---------------------------------------------------------------------------------------------
// elementwise kernels
// ---------------------------------------------------------------------------------------------
// uint8 frames [B+1,H,W] -> fp32 images [B+1,H,W] (ToTensor + Normalize) and the flow-net input
// NHWC16 fp16 [B,H,W,16]: ch0 = I[b], ch1 = I[b+1] (slomo.py:343 cat((I0, I1), dim=1))
__global__ void prep_pairs_kernel(const uint8_t *__restrict__ frames, float *__restrict__ img,
                                  __half *__restrict__ flow_in, int B, int HW) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)(B + 1) * HW;
    if (i >= total) return;
    const float v = (float)frames[i] / 255.0f - kMean;
    img[i] = v;
    const int b = (int)(i / HW);
    const long px = i % HW;
    if (b < B) {                       // frame b is I0 of pair b, frame b + 1 its I1: one 32-byte pixel record per thread
        const float v1 = (float)frames[i + HW] / 255.0f - kMean;
        const __half2 h01 = __floats2half2_rn(v, v1);
        uint4 lo = make_uint4(*(const uint32_t *)&h01, 0u, 0u, 0u), hi = make_uint4(0u, 0u, 0u, 0u);
        uint4 *d = (uint4 *)(flow_in + ((long)b * HW + px) * 16);
        d[0] = lo;
        d[1] = hi;
    }
}

// F.avg_pool2d(x, 2) on NHWC fp16, 8 channels per thread
__global__ void avgpool2_kernel(const __half *__restrict__ in, __half *__restrict__ out, int N, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2, C8 = C / 8;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)N * Ho * Wo * C8;
    if (i >= total) return;
    const int c8 = (int)(i % C8);
    long r = i / C8;
    const int x = (int)(r % Wo); r /= Wo;
    const int y = (int)(r % Ho);
    const int n = (int)(r / Ho);
    const __half *p = in + (((long)n * H + 2 * y) * W + 2 * x) * C + c8 * 8;
    uint4 a = *(const uint4 *)p, b = *(const uint4 *)(p + C), c = *(const uint4 *)(p + (long)W * C),
          d = *(const uint4 *)(p + (long)W * C + C);
    const __half2 *ha = (const __half2 *)&a, *hb = (const __half2 *)&b, *hc = (const __half2 *)&c, *hd = (const __half2 *)&d;
    uint4 o;
    __half2 *ho = (__half2 *)&o;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]), fc = __half22float2(hc[j]), fd = __half22float2(hd[j]);
        ho[j] = __floats2half2_rn((fa.x + fb.x + fc.x + fd.x) * 0.25f, (fa.y + fb.y + fc.y + fd.y) * 0.25f);
    }
    *(uint4 *)(out + (((long)n * Ho + y) * Wo + x) * C + c8 * 8) = o;
}

// F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) on NHWC fp16.
// Output rows 2k+1 and 2k+2 both interpolate input rows k and k+1 (weights .75/.25 and .25/.75), same
// for columns, so one thread loads a 2x2 input patch (8 channels each) and writes the 2x2 output block
// (2k+1..2k+2, 2m+1..2m+2): one 16-byte load per 16-byte store. k = -1 and k = H-1 are the clamped borders
// (PyTorch clamps the source index, which makes output rows 0 and 2H-1 copies of input rows 0 and H-1).
__global__ void upsample2_kernel(const __half *__restrict__ in, __half *__restrict__ out, int N, int H, int W, int C) {
    const int C8 = C / 8, Hb = H + 1, Wb = W + 1;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)N * Hb * Wb * C8;
    if (i >= total) return;
    const int c8 = (int)(i % C8);
    long r = i / C8;
    const int m = (int)(r % Wb) - 1; r /= Wb;
    const int k = (int)(r % Hb) - 1;
    const int n = (int)(r / Hb);
    const int y0 = k < 0 ? 0 : k, y1 = k + 1 > H - 1 ? H - 1 : k + 1;
    const int x0 = m < 0 ? 0 : m, x1 = m + 1 > W - 1 ? W - 1 : m + 1;
    const __half *base = in + (long)n * H * W * C + c8 * 8;
    const uint4 a = *(const uint4 *)(base + ((long)y0 * W + x0) * C), b = *(const uint4 *)(base + ((long)y0 * W + x1) * C),
                c = *(const uint4 *)(base + ((long)y1 * W + x0) * C), d = *(const uint4 *)(base + ((long)y1 * W + x1) * C);
    const __half2 *ha = (const __half2 *)&a, *hb = (const __half2 *)&b, *hc = (const __half2 *)&c, *hd = (const __half2 *)&d;
    float2 fa[4], fb[4], fc[4], fd[4];
#pragma unroll
    for (int j = 0; j < 4; j++) { fa[j] = __half22float2(ha[j]); fb[j] = __half22float2(hb[j]); fc[j] = __half22float2(hc[j]); fd[j] = __half22float2(hd[j]); }
    const int Ho = 2 * H, Wo = 2 * W;
#pragma unroll
    for (int dy = 0; dy < 2; dy++) {
        const int oy = 2 * k + 1 + dy;
        if (oy < 0 || oy >= Ho) continue;
        // lambda of the lower row: 0.25 for output row 2k+1, 0.75 for 2k+2 (exactly PyTorch's src - floor(src))
        const float ly = dy ? 0.75f : 0.25f, hy = 1.f - ly;
#pragma unroll
        for (int dx = 0; dx < 2; dx++) {
            const int ox = 2 * m + 1 + dx;
            if (ox < 0 || ox >= Wo) continue;
            const float lx = dx ? 0.75f : 0.25f, hx = 1.f - lx;
            uint4 o;
            __half2 *ho = (__half2 *)&o;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                float vx = hy * (hx * fa[j].x + lx * fb[j].x) + ly * (hx * fc[j].x + lx * fd[j].x);
                float vy = hy * (hx * fa[j].y + lx * fb[j].y) + ly * (hx * fc[j].y + lx * fd[j].y);
                ho[j] = __floats2half2_rn(vx, vy);
            }
            *(uint4 *)(out + (((long)n * Ho + oy) * Wo + ox) * C + c8 * 8) = o;
        }
    }
}

// backWarp.forward (model.py:268-300) for one output pixel: grid_sample(img, bilinear, zeros,
// align_corners=False) at ((x+u), (y+v)) after the reference's normalise / un-normalise round trip,
// i.e. at (x+u-0.5, y+v-0.5).
__device__ __forceinline__ float backwarp(const float *__restrict__ img, int H, int W, int x, int y, float u, float v) {
    float gx = 2.0f * (((float)x + u) / (float)W - 0.5f);
    float gy = 2.0f * (((float)y + v) / (float)H - 0.5f);
    float ix = ((gx + 1.0f) * (float)W - 1.0f) * 0.5f;
    float iy = ((gy + 1.0f) * (float)H - 1.0f) * 0.5f;
    float fx = floorf(ix), fy = floorf(iy);
    int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    float wx1 = ix - fx, wy1 = iy - fy, wx0 = 1.0f - wx1, wy0 = 1.0f - wy1;
    float acc = 0.f;
    const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
    if (vy0 && vx0) acc += img[(long)y0 * W + x0] * (wx0 * wy0);
    if (vy0 && vx1) acc += img[(long)y0 * W + x1] * (wx1 * wy0);
    if (vy1 && vx0) acc += img[(long)y1 * W + x0] * (wx0 * wy1);
    if (vy1 && vx1) acc += img[(long)y1 * W + x1] * (wx1 * wy1);
    return acc;
}

struct FlowCoef { float c00, c01, c10, c11, w0, w1; };   // slomo.py:405-410, 428

// slomo.py:405-419: builds the 12-channel interpolator input (NHWC16 fp16)
__global__ void pre_interp_kernel(const float *__restrict__ img, const float *__restrict__ flow,
                                  __half *__restrict__ out, int B, int H, int W, FlowCoef k) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long HW = (long)H * W;
    if (i >= (long)B * HW) return;
    const int b = (int)(i / HW);
    const long px = i % HW;
    const int y = (int)(px / W), x = (int)(px % W);
    const float *I0 = img + (long)b * HW, *I1 = I0 + HW;
    const float4 f = *(const float4 *)(flow + i * 8);          // F01x F01y F10x F10y
    const float ft0x = k.c00 * f.x + k.c01 * f.z, ft0y = k.c00 * f.y + k.c01 * f.w;
    const float ft1x = k.c10 * f.x + k.c11 * f.z, ft1y = k.c10 * f.y + k.c11 * f.w;
    const float g0 = backwarp(I0, H, W, x, y, ft0x, ft0y);
    const float g1 = backwarp(I1, H, W, x, y, ft1x, ft1y);
    __half2 h[8];
    h[0] = __floats2half2_rn(I0[px], I1[px]);
    h[1] = __floats2half2_rn(f.x, f.y);
    h[2] = __floats2half2_rn(f.z, f.w);
    h[3] = __floats2half2_rn(ft1x, ft1y);
    h[4] = __floats2half2_rn(ft0x, ft0y);
    h[5] = __floats2half2_rn(g1, g0);
    h[6] = __floats2half2_rn(0.f, 0.f);
    h[7] = h[6];
    uint4 *d = (uint4 *)(out + i * 16);
    d[0] = *(uint4 *)&h[0];
    d[1] = *(uint4 *)&h[4];
}

// slomo.py:421-437: refined flows, visibility, warps, blend, de-normalise, uint8 truncation
__global__ void post_interp_kernel(const float *__restrict__ img, const float *__restrict__ flow,
                                   const float *__restrict__ intrp, uint8_t *__restrict__ out,
                                   float *__restrict__ out_f32, int B, int H, int W, FlowCoef k, int *nonfinite) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long HW = (long)H * W;
    if (i >= (long)B * HW) return;
    const int b = (int)(i / HW);
    const long px = i % HW;
    const int y = (int)(px / W), x = (int)(px % W);
    const float *I0 = img + (long)b * HW, *I1 = I0 + HW;
    const float4 f = *(const float4 *)(flow + i * 8);
    const float4 r0 = *(const float4 *)(intrp + i * 8);
    const float vlogit = intrp[i * 8 + 4];
    const float ft0x = k.c00 * f.x + k.c01 * f.z + r0.x, ft0y = k.c00 * f.y + k.c01 * f.w + r0.y;
    const float ft1x = k.c10 * f.x + k.c11 * f.z + r0.z, ft1y = k.c10 * f.y + k.c11 * f.w + r0.w;
    const float v0 = 1.0f / (1.0f + expf(-vlogit)), v1 = 1.0f - v0;
    const float g0 = backwarp(I0, H, W, x, y, ft0x, ft0y);
    const float g1 = backwarp(I1, H, W, x, y, ft1x, ft1y);
    const float ft = (k.w0 * v0 * g0 + k.w1 * v1 * g1) / (k.w0 * v0 + k.w1 * v1);
    if (out_f32) out_f32[i] = ft;
    // fp16 activations that overflowed (a checkpoint whose dynamic range exceeds 65504) surface here as inf / nan in
    // the fp32 network heads or in the blended value: flag it, v2e_slomo_check_finite reports it (fail loudly)
    if (!(isfinite(f.x) && isfinite(f.y) && isfinite(f.z) && isfinite(f.w) && isfinite(r0.x) && isfinite(r0.y) &&
          isfinite(r0.z) && isfinite(r0.w) && isfinite(vlogit) && isfinite(ft)))
        *nonfinite = 1;
    // revNormalize then ToPILImage: (x + 0.428).mul(255).byte() -- CPU float->uint8 conversion
    // truncates toward zero and wraps modulo 256
    const float s = (ft + kMean) * 255.0f;
    out[i] = (uint8_t)((int)s & 0xFF);
}

// max over pixels of |F01| and |F10| (slomo.py:358-366)
__global__ void max_speed_kernel(const float *__restrict__ flow, long n, float *out) {
    float m = 0.f;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float4 f = *(const float4 *)(flow + i * 8);
        m = fmaxf(m, fmaxf(sqrtf(f.x * f.x + f.y * f.y), sqrtf(f.z * f.z + f.w * f.w)));
    }
    m = warp_reduce_max(m);
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax((int *)out, __float_as_int(m));   // m >= 0: int order == float order
}

// ---------------------------------------------------------------------------------------------
// Pillow 8-bit resampling (Pillow src/libImaging/Resample.c, ImagingResampleHorizontal_8bpc /
// ImagingResampleVertical_8bpc): 22-bit fixed-point coefficients computed on the host in double
// exactly like precompute_coeffs() + normalize_coeffs_8bpc(), integer accumulation here.
// ---------------------------------------------------------------------------------------------
// dst_stride: distance in bytes between consecutive destination images (dense: rows * width)
__global__ void resample_h_u8_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, int n_img, int sw,
                                     int sh, int dw, const int *__restrict__ bounds, const int *__restrict__ kk, int ksize,
                                     long dst_stride) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n_img * sh * dw) return;
    const int xx = (int)(i % dw);
    const long row = i / dw;
    const int xmin = bounds[2 * xx], xmax = bounds[2 * xx + 1];
    const uint8_t *s = src + row * sw + xmin;
    const int *k = kk + (long)xx * ksize;
    int ss = 1 << 21;
    for (int x = 0; x < xmax; x++) ss += (int)s[x] * k[x];
    ss >>= 22;
    const long per = (long)sh * dw;
    dst[(i / per) * dst_stride + i % per] = (uint8_t)(ss < 0 ? 0 : (ss > 255 ? 255 : ss));
}
__global__ void resample_v_u8_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, int n_img, int w,
                                     int sh, int dh, const int *__restrict__ bounds, const int *__restrict__ kk, int ksize,
                                     long dst_stride) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n_img * dh * w) return;
    const int x = (int)(i % w);
    const long r = i / w;
    const int yy = (int)(r % dh);
    const long img = r / dh;
    const int ymin = bounds[2 * yy], ymax = bounds[2 * yy + 1];
    const uint8_t *s = src + (img * sh + ymin) * w + x;
    const int *k = kk + (long)yy * ksize;
    int ss = 1 << 21;
    for (int y = 0; y < ymax; y++) ss += (int)s[(long)y * w] * k[y];
    ss >>= 22;
    dst[img * dst_stride + (long)yy * w + x] = (uint8_t)(ss < 0 ? 0 : (ss > 255 ? 255 : ss));
}

static double bilinear_filter(double x) { if (x < 0.0) x = -x; return x < 1.0 ? 1.0 - x : 0.0; }
static double sinc_filter(double x) { if (x == 0.0) return 1.0; x = x * M_PI; return sin(x) / x; }
static double lanczos_filter(double x) { return (-3.0 <= x && x < 3.0) ? sinc_filter(x) * sinc_filter(x / 3) : 0.0; }

static int precompute_coeffs(int inSize, int outSize, int filter, std::vector<int> &bounds, std::vector<int> &kk) {
    const double support0 = filter == 1 ? 3.0 : 1.0;
    double (*fn)(double) = filter == 1 ? lanczos_filter : bilinear_filter;
    double scale = (double)inSize / outSize, filterscale = scale;
    if (filterscale < 1.0) filterscale = 1.0;
    const double support = support0 * filterscale;
    const int ksize = (int)ceil(support) * 2 + 1;
    bounds.assign((size_t)outSize * 2, 0);
    kk.assign((size_t)outSize * ksize, 0);
    std::vector<double> pre(ksize);
    for (int xx = 0; xx < outSize; xx++) {
        double center = (xx + 0.5) * scale, ww = 0.0, ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > inSize) xmax = inSize;
        xmax -= xmin;
        int x;
        for (x = 0; x < xmax; x++) { double w = fn((x + xmin - center + 0.5) * ss); pre[x] = w; ww += w; }
        for (x = 0; x < xmax; x++) if (ww != 0.0) pre[x] /= ww;
        for (; x < ksize; x++) pre[x] = 0;
        for (x = 0; x < ksize; x++)
            kk[(size_t)xx * ksize + x] = pre[x] < 0 ? (int)(-0.5 + pre[x] * (1 << 22)) : (int)(0.5 + pre[x] * (1 << 22));
        bounds[2 * xx] = xmin;
        bounds[2 * xx + 1] = xmax;
    }
    return ksize;
}

inline int cdiv(long a, int b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------------------------------------
// UNet (model.py:158-226)
// ---------------------------------------------------------------------------------------------
struct LayerSpec { int cin1, cin2, cout, k; };

struct UNet {
    int in_ch, out_ch;
    LayerSpec L[23];
    __half *w[23];
    __half *w_row[23];           // [slabs][taps][Cout_pad][KC] for layers that run on the strip kernel
    int row_kc[23];              // slab width of the strip kernel; 0: per-tap kernel
    __half *w_fold[23];          // up-block conv1 with the x2 bilinear up-sampling folded in (conv_up2_kernel), or null
    float *b[23];
    int cout_pad[23], c1p[23], c2p[23];
};

int pad16(int c) { return (c + 15) / 16 * 16; }
int cout_padded(int c) { int p = pad16(c); return p <= 16 ? 16 : (p <= 32 ? 32 : (p <= 64 ? 64 : (p + 127) / 128 * 128)); }

void unet_spec(UNet &u, int in_ch, int out_ch) {
    u.in_ch = in_ch; u.out_ch = out_ch;
    const int ch[6] = {32, 64, 128, 256, 512, 512};
    int i = 0;
    u.L[i++] = {in_ch, 0, 32, 7};
    u.L[i++] = {32, 0, 32, 7};
    const int dk[5] = {5, 3, 3, 3, 3};
    for (int d = 0; d < 5; d++) { u.L[i++] = {ch[d], 0, ch[d + 1], dk[d]}; u.L[i++] = {ch[d + 1], 0, ch[d + 1], dk[d]}; }
    const int uo[5] = {512, 256, 128, 64, 32}, ui[5] = {512, 512, 256, 128, 64};
    for (int k = 0; k < 5; k++) { u.L[i++] = {ui[k], 0, uo[k], 3}; u.L[i++] = {uo[k], uo[k], uo[k], 3}; }
    u.L[i++] = {32, 0, out_ch, 3};
}

}  // namespace

struct V2eSlomo {
    int H, W, maxB;
    UNet flow, interp;
    // activations (NHWC fp16), sized for maxB
    __half *in16;                 // [B,H,W,16]
    __half *x0, *s1;              // full res 32
    __half *pool[5], *da[5], *s[5];   // level l+1 (1/2^(l+1)): pooled, conv1 out, conv2 out (s2..s5, x5)
    __half *up[5], *ua[5], *ub[5];    // up-block k: upsampled, conv1 out, conv2 out
    float *flow_out, *intrp_out;  // [B,H,W,8] fp32
    float *img;                   // [B+1,H,W] fp32
    float *maxspeed;              // device scalar
    int *nonfinite;               // device flag: a network head or a blended pixel was inf / nan
    int curB;
    std::vector<char> launch_mem, row_mem, up_mem;
    int n_sms, no_fused_pool;
    int dev_sms;                  // the device's SM count; n_sms plans the launches (option 3 lowers it)
    int8_t ran[2][23];            // [flow, interp][layer]: V2E_SLOMO_KERNEL_* of the last launch (test hook)
    // measurement hooks: CUDA events around every conv launch
    int profile;
    std::vector<cudaEvent_t> ev;
    size_t ev_used;
    double conv_flops;           // algorithmic FLOPs (2*MAC, unpadded channels) of the bracketed launches
    std::vector<int> ev_layer;   // UNet layer index (0..22) of every bracketed launch
    std::vector<double> ev_flops;
};

// spatial level (power of two divisor) at which layer i runs
static int layer_level(int i) {
    if (i < 2 || i == 22) return 0;
    if (i < 12) return (i - 2) / 2 + 1;            // down1..down5 -> 1..5
    return 4 - (i - 12) / 2;                       // up1..up5 -> 4..0
}

static int upload_unet(UNet &u, const V2eUNetWeights *wts, int W) {
    for (int i = 0; i < 23; i++) {
        const LayerSpec &l = u.L[i];
        const int c1p = pad16(l.cin1), c2p = l.cin2 ? pad16(l.cin2) : 0, cp = cout_padded(l.cout), taps = l.k * l.k;
        u.c1p[i] = c1p; u.c2p[i] = c2p; u.cout_pad[i] = cp;
        const int cin = l.cin1 + l.cin2, ktot = taps * (c1p + c2p);
        std::vector<__half> packed((size_t)cp * ktot, __float2half(0.f));
        const float *src = wts->w[i];   // [cout][cin][k][k]
        if (!src || !wts->b[i]) return v2e_set_error(V2E_E_INVALID, "missing UNet weight%s", "");
        for (int o = 0; o < l.cout; o++)
            for (int c = 0; c < cin; c++) {
                const int cc = c < l.cin1 ? c : c1p + (c - l.cin1);
                for (int t = 0; t < taps; t++)
                    packed[(size_t)o * ktot + (size_t)t * (c1p + c2p) + cc] = __float2half_rn(src[((size_t)o * cin + c) * taps + t]);
            }
        std::vector<float> bias(cp, 0.f);
        for (int o = 0; o < l.cout; o++) bias[o] = wts->b[i][o];
        u.w_fold[i] = nullptr;
        if (i >= 12 && i < 22 && (i & 1) == 0 && l.k == 3 && !c2p && v2e_conv_up2_supported(c1p, cp, W >> layer_level(i))) {
            // conv1 of an up block: its input is interpolate(x, 2, bilinear) (model.py:140-147)
            std::vector<__half> fold((size_t)(c1p / 64) * 2 * 3 * 6 * cp * 64);
            int frc = v2e_conv_up2_fold_weights(src, l.cout, l.cin1, cp, c1p, fold.data());
            if (frc) return frc;
            CU(cudaMalloc((void **)&u.w_fold[i], fold.size() * sizeof(__half)));
            CU(cudaMemcpy(u.w_fold[i], fold.data(), fold.size() * sizeof(__half), cudaMemcpyHostToDevice));
        }
        u.w_row[i] = nullptr;
        u.row_kc[i] = v2e_strip_pick(c1p, c2p, cp, l.k, l.k, W >> layer_level(i), nullptr);
        if (u.row_kc[i]) {
            const int kc = u.row_kc[i], slabs = (c1p + c2p) / kc;
            std::vector<__half> rowp((size_t)slabs * taps * cp * kc);
            for (int sl = 0; sl < slabs; sl++)
                for (int t = 0; t < taps; t++)
                    for (int o = 0; o < cp; o++)
                        for (int c = 0; c < kc; c++)
                            rowp[(((size_t)sl * taps + t) * cp + o) * kc + c] =
                                packed[(size_t)o * ktot + (size_t)t * (c1p + c2p) + sl * kc + c];
            CU(cudaMalloc((void **)&u.w_row[i], rowp.size() * sizeof(__half)));
            CU(cudaMemcpy(u.w_row[i], rowp.data(), rowp.size() * sizeof(__half), cudaMemcpyHostToDevice));
        }
        CU(cudaMalloc((void **)&u.w[i], packed.size() * sizeof(__half)));
        CU(cudaMalloc((void **)&u.b[i], bias.size() * sizeof(float)));
        CU(cudaMemcpy(u.w[i], packed.data(), packed.size() * sizeof(__half), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(u.b[i], bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    return V2E_OK;
}

extern "C" int v2e_slomo_create(int H, int W, int max_batch, const V2eUNetWeights *flow, const V2eUNetWeights *interp,
                                V2eSlomo **out) {
    if (!flow || !interp || !out) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    if (H % 32 || W % 32 || H <= 0 || W <= 0) return v2e_set_error(V2E_E_INVALID, "network dims must be multiples of 32 (dataloader.py:122-123)%s", "");
    if (max_batch < 1) return v2e_set_error(V2E_E_INVALID, "max_batch < 1%s", "");
    V2eSlomo *h = new V2eSlomo();
    h->H = H; h->W = W; h->maxB = max_batch; h->curB = 0;
    h->profile = 0; h->ev_used = 0; h->conv_flops = 0;
    unet_spec(h->flow, 2, 4);
    unet_spec(h->interp, 12, 5);
    int rc;
    if ((rc = upload_unet(h->flow, flow, W)) || (rc = upload_unet(h->interp, interp, W))) { delete h; return rc; }
    const size_t B = max_batch, HW = (size_t)H * W;
    auto alloc16 = [&](__half **p, size_t elems) { return cudaMalloc((void **)p, elems * sizeof(__half)); };
    const int ch[6] = {32, 64, 128, 256, 512, 512};
    CU(alloc16(&h->in16, B * HW * 16));
    CU(alloc16(&h->x0, B * HW * 32));
    CU(alloc16(&h->s1, B * HW * 32));
    for (int l = 0; l < 5; l++) {
        const size_t hw = HW >> (2 * (l + 1));
        CU(alloc16(&h->pool[l], B * hw * ch[l]));
        CU(alloc16(&h->da[l], B * hw * ch[l + 1]));
        CU(alloc16(&h->s[l], B * hw * ch[l + 1]));
    }
    const int uo[5] = {512, 256, 128, 64, 32}, ui[5] = {512, 512, 256, 128, 64};
    for (int k = 0; k < 5; k++) {
        const size_t hw = HW >> (2 * (4 - k));
        CU(alloc16(&h->up[k], B * hw * ui[k]));
        CU(alloc16(&h->ua[k], B * hw * uo[k]));
        CU(alloc16(&h->ub[k], B * hw * uo[k]));
    }
    CU(cudaMalloc((void **)&h->flow_out, B * HW * 8 * sizeof(float)));
    CU(cudaMalloc((void **)&h->intrp_out, B * HW * 8 * sizeof(float)));
    CU(cudaMalloc((void **)&h->img, (B + 1) * HW * sizeof(float)));
    CU(cudaMalloc((void **)&h->maxspeed, sizeof(float)));
    CU(cudaMalloc((void **)&h->nonfinite, sizeof(int)));
    CU(cudaMemset(h->nonfinite, 0, sizeof(int)));
    h->launch_mem.resize(v2e_conv_launch_size());
    h->row_mem.resize(v2e_strip_launch_size());
    { int dev = 0; cudaGetDevice(&dev); h->n_sms = 132; cudaDeviceGetAttribute(&h->n_sms, cudaDevAttrMultiProcessorCount, dev); }
    h->dev_sms = h->n_sms;
    h->no_fused_pool = 0;
    h->up_mem.resize(v2e_conv_up2_launch_size());
    memset(h->ran, V2E_SLOMO_KERNEL_NONE, sizeof(h->ran));
    *out = h;
    return V2E_OK;
}

extern "C" int v2e_slomo_destroy(V2eSlomo *h) {
    if (!h) return V2E_OK;
    for (UNet *u : {&h->flow, &h->interp})
        for (int i = 0; i < 23; i++) { if (u->w[i]) cudaFree(u->w[i]); if (u->b[i]) cudaFree(u->b[i]); if (u->w_row[i]) cudaFree(u->w_row[i]); if (u->w_fold[i]) cudaFree(u->w_fold[i]); }
    void *ptrs[] = {h->in16, h->x0, h->s1, h->flow_out, h->intrp_out, h->img, h->maxspeed, h->nonfinite};
    for (void *p : ptrs) if (p) cudaFree(p);
    for (int l = 0; l < 5; l++) {
        cudaFree(h->pool[l]); cudaFree(h->da[l]); cudaFree(h->s[l]);
        cudaFree(h->up[l]); cudaFree(h->ua[l]); cudaFree(h->ub[l]);
    }
    for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
    delete h;
    return V2E_OK;
}

// pool_out != null: the caller has checked pool_fusable(); F.avg_pool2d(out, 2) is written by the same kernel
static int conv(V2eSlomo *h, const UNet &u, int li, const __half *x1, const __half *x2, int B, int H, int W, void *out,
                int out_mode, cudaStream_t st, __half *pool_out = nullptr) {
    int rc;
    const bool row = u.row_kc[li] != 0;
    V2eConvLaunch *L = (V2eConvLaunch *)h->launch_mem.data();
    V2eStripLaunch *R = (V2eStripLaunch *)h->row_mem.data();
    h->ran[&u == &h->interp][li] = row ? (pool_out ? V2E_SLOMO_KERNEL_STRIP_POOL : V2E_SLOMO_KERNEL_STRIP)
                                       : V2E_SLOMO_KERNEL_TAP;
    if (row)
        rc = v2e_strip_prepare(R, x1, u.c1p[li], x2, x2 ? u.c2p[li] : 0, u.w_row[li], u.b[li], u.cout_pad[li], u.L[li].k,
                               u.L[li].k, B, H, W, out, u.cout_pad[li], out_mode, u.L[li].cout, kSlope, h->n_sms,
                               pool_out, u.cout_pad[li], V2E_STRIP_CHAIN_AUTO);
    else
        rc = v2e_conv_prepare(L, x1, u.c1p[li], x2, x2 ? u.c2p[li] : 0, u.w[li], u.b[li], u.cout_pad[li], u.L[li].k,
                              u.L[li].k, B, H, W, out, u.cout_pad[li], out_mode, u.L[li].cout, kSlope,
                              V2E_CONV_TILE_AUTO, h->n_sms);
    if (rc) return rc;
    if (h->profile) {
        if (h->ev_used + 2 > h->ev.size()) {
            size_t old = h->ev.size();
            h->ev.resize(old + 512);
            for (size_t i = old; i < h->ev.size(); i++) cudaEventCreate(&h->ev[i]);
        }
        cudaEventRecord(h->ev[h->ev_used], st);
    }
    rc = row ? v2e_strip_launch(R, st) : v2e_conv_launch(L, st);
    if (h->profile) {
        cudaEventRecord(h->ev[h->ev_used + 1], st);
        h->ev_used += 2;
        const LayerSpec &l = u.L[li];
        const double fl = 2.0 * B * H * W * (double)l.cout * (l.cin1 + l.cin2) * l.k * l.k;
        h->conv_flops += fl;
        h->ev_layer.push_back(li);
        h->ev_flops.push_back(fl);
    }
    return rc;
}

static int conv_up2(V2eSlomo *h, const UNet &u, int li, const __half *x_low, int B, int H, int W, void *out, cudaStream_t st) {
    V2eUpLaunch *L = (V2eUpLaunch *)h->up_mem.data();
    h->ran[&u == &h->interp][li] = V2E_SLOMO_KERNEL_UP2;
    int rc = v2e_conv_up2_prepare(L, x_low, u.c1p[li], u.w_fold[li], u.w[li], u.b[li], u.cout_pad[li], B, H, W, out,
                                  u.cout_pad[li], kSlope, h->n_sms);
    if (rc) return rc;
    if (h->profile) {
        if (h->ev_used + 2 > h->ev.size()) {
            size_t old = h->ev.size();
            h->ev.resize(old + 512);
            for (size_t i = old; i < h->ev.size(); i++) cudaEventCreate(&h->ev[i]);
        }
        cudaEventRecord(h->ev[h->ev_used], st);
    }
    rc = v2e_conv_up2_launch(L, st);
    if (h->profile) {
        cudaEventRecord(h->ev[h->ev_used + 1], st);
        h->ev_used += 2;
        const LayerSpec &l = u.L[li];
        const double fl = 2.0 * B * H * W * (double)l.cout * l.cin1 * 9;
        h->conv_flops += fl;
        h->ev_layer.push_back(li);
        h->ev_flops.push_back(fl);
    }
    return rc;
}

// the average pool that opens a down block (model.py:71) can ride in the epilogue of the convolution before it
static bool pool_fusable(const V2eSlomo *h, const UNet &u, int li, int H, int W) {
    if (h->no_fused_pool || !u.row_kc[li] || u.cout_pad[li] != u.L[li].cout) return false;
    return v2e_strip_pool_supported(u.c1p[li], u.c2p[li], u.cout_pad[li], u.L[li].k, u.L[li].k, H, W) != 0;
}

// UNet.forward (model.py:198-226). in: NHWC16 fp16 [B,H,W,16]; out: fp32 [B,H,W,8]
static int unet_forward(V2eSlomo *h, const UNet &u, const __half *in, float *out, int B, cudaStream_t st) {
    const int H = h->H, W = h->W;
    int rc;
    if ((rc = conv(h, u, 0, in, nullptr, B, H, W, h->x0, 0, st))) return rc;
    bool pooled = pool_fusable(h, u, 1, H, W);           // conv2 also writes pool[0]
    if ((rc = conv(h, u, 1, h->x0, nullptr, B, H, W, h->s1, 0, st, pooled ? h->pool[0] : nullptr))) return rc;
    const int ch[6] = {32, 64, 128, 256, 512, 512};
    const __half *prev = h->s1;
    for (int l = 0; l < 5; l++) {                       // down blocks (model.py:55-77)
        const int hi = H >> l, wi = W >> l, ho = hi / 2, wo = wi / 2;
        if (!pooled) {
            const long n = (long)B * ho * wo * (ch[l] / 8);
            avgpool2_kernel<<<cdiv(n, 256), 256, 0, st>>>(prev, h->pool[l], B, hi, wi, ch[l]);
        }
        if ((rc = conv(h, u, 2 + 2 * l, h->pool[l], nullptr, B, ho, wo, h->da[l], 0, st))) return rc;
        pooled = l < 4 && pool_fusable(h, u, 3 + 2 * l, ho, wo);        // this block's conv2 writes the next pool
        if ((rc = conv(h, u, 3 + 2 * l, h->da[l], nullptr, B, ho, wo, h->s[l], 0, st, pooled ? h->pool[l + 1] : nullptr))) return rc;
        prev = h->s[l];
    }
    const int ui[5] = {512, 512, 256, 128, 64};
    const __half *x = h->s[4];                          // output of down5
    for (int k = 0; k < 5; k++) {                       // up blocks (model.py:125-155)
        const int lvl = 5 - k;                          // x lives at 1/2^lvl
        const int hi = H >> lvl, wi = W >> lvl, ho = hi * 2, wo = wi * 2;
        const __half *skip = k < 4 ? h->s[3 - k] : h->s1;
        const int li = 12 + 2 * k;
        if (u.w_fold[li]) {
            // interpolate + conv1 in one kernel: the up-sampled tensor is never written
            if ((rc = conv_up2(h, u, li, x, B, ho, wo, h->ua[k], st))) return rc;
        } else {
            const long n = (long)B * (hi + 1) * (wi + 1) * (ui[k] / 8);
            upsample2_kernel<<<cdiv(n, 256), 256, 0, st>>>(x, h->up[k], B, hi, wi, ui[k]);
            if ((rc = conv(h, u, li, h->up[k], nullptr, B, ho, wo, h->ua[k], 0, st))) return rc;
        }
        if ((rc = conv(h, u, 13 + 2 * k, h->ua[k], skip, B, ho, wo, h->ub[k], 0, st))) return rc;
        x = h->ub[k];
    }
    if ((rc = conv(h, u, 22, x, nullptr, B, H, W, out, 1, st))) return rc;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "unet_forward: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_slomo_set_pairs(V2eSlomo *h, const uint8_t *frames_u8_dev, int B, void *stream) {
    if (!h || !frames_u8_dev) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    if (B < 1 || B > h->maxB) return v2e_set_error(V2E_E_INVALID, "batch out of range%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    const int HW = h->H * h->W;
    prep_pairs_kernel<<<cdiv((long)(B + 1) * HW, 256), 256, 0, st>>>(frames_u8_dev, h->img, h->in16, B, HW);
    h->curB = B;
    return unet_forward(h, h->flow, h->in16, h->flow_out, B, st);
}

extern "C" int v2e_slomo_max_flow(V2eSlomo *h, float *max_speed_host, void *stream) {
    if (!h || !max_speed_host || h->curB < 1) return v2e_set_error(V2E_E_STATE, "v2e_slomo_set_pairs must run first%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    CU(cudaMemsetAsync(h->maxspeed, 0, sizeof(float), st));
    max_speed_kernel<<<296, 256, 0, st>>>(h->flow_out, (long)h->curB * h->H * h->W, h->maxspeed);
    CU(cudaMemcpyAsync(max_speed_host, h->maxspeed, sizeof(float), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return V2E_OK;
}

extern "C" int v2e_slomo_interp(V2eSlomo *h, double t, uint8_t *out_u8_dev, float *out_f32_dev, void *stream) {
    if (!h || !out_u8_dev || h->curB < 1) return v2e_set_error(V2E_E_STATE, "v2e_slomo_set_pairs must run first%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    const int B = h->curB;
    const long n = (long)B * h->H * h->W;
    // slomo.py:405-410, 428: Python doubles, rounded to float32 when they meet the tensors
    const double temp = -t * (1 - t);
    FlowCoef k;
    k.c00 = (float)temp; k.c01 = (float)(t * t); k.c10 = (float)((1 - t) * (1 - t)); k.c11 = (float)temp;
    k.w0 = (float)(1 - t); k.w1 = (float)t;
    pre_interp_kernel<<<cdiv(n, 256), 256, 0, st>>>(h->img, h->flow_out, h->in16, B, h->H, h->W, k);
    int rc = unet_forward(h, h->interp, h->in16, h->intrp_out, B, st);
    if (rc) return rc;
    post_interp_kernel<<<cdiv(n, 256), 256, 0, st>>>(h->img, h->flow_out, h->intrp_out, out_u8_dev, out_f32_dev, B, h->H, h->W, k,
                                                     h->nonfinite);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "v2e_slomo_interp: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_slomo_check_finite(V2eSlomo *h, int *nonfinite_host, void *stream) {
    if (!h || !nonfinite_host) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    CU(cudaMemcpyAsync(nonfinite_host, h->nonfinite, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaMemsetAsync(h->nonfinite, 0, sizeof(int), st));
    CU(cudaStreamSynchronize(st));
    return V2E_OK;
}

extern "C" int v2e_slomo_set_option(V2eSlomo *h, int option, int value) {
    if (!h) return v2e_set_error(V2E_E_INVALID, "null handle%s", "");
    if (option == 2) { h->no_fused_pool = value; return V2E_OK; }
    if (option == 3) {
        // plan as if the device had `value` SMs; never more than it has, so a persistent grid cannot oversubscribe it
        if (value < 0 || value > h->dev_sms) return v2e_set_error(V2E_E_INVALID, "SM count out of range%s", "");
        h->n_sms = value ? value : h->dev_sms;
        return V2E_OK;
    }
    return v2e_set_error(V2E_E_INVALID, "unknown option%s", "");
}

extern "C" int v2e_slomo_profile(V2eSlomo *h, int enable) {
    if (!h) return v2e_set_error(V2E_E_INVALID, "null handle%s", "");
    h->profile = enable ? 1 : 0;
    h->ev_used = 0;
    h->conv_flops = 0;
    h->ev_layer.clear();
    h->ev_flops.clear();
    return V2E_OK;
}

static int profile_collect(V2eSlomo *h, float *conv_ms, int *conv_launches, double *conv_flops, float *ms23, int *n23,
                           double *flops23, void *stream) {
    CU(cudaStreamSynchronize((cudaStream_t)stream));
    float tot = 0.f;
    if (ms23) for (int i = 0; i < 23; i++) { ms23[i] = 0.f; n23[i] = 0; flops23[i] = 0.0; }
    for (size_t i = 0, k = 0; i + 1 < h->ev_used; i += 2, k++) {
        float ms = 0.f;
        CU(cudaEventElapsedTime(&ms, h->ev[i], h->ev[i + 1]));
        tot += ms;
        if (ms23 && k < h->ev_layer.size()) {
            const int li = h->ev_layer[k];
            ms23[li] += ms; n23[li] += 1; flops23[li] += h->ev_flops[k];
        }
    }
    if (conv_ms) *conv_ms = tot;
    if (conv_launches) *conv_launches = (int)(h->ev_used / 2);
    if (conv_flops) *conv_flops = h->conv_flops;
    h->ev_used = 0;
    h->conv_flops = 0;
    h->ev_layer.clear();
    h->ev_flops.clear();
    return V2E_OK;
}
extern "C" int v2e_slomo_profile_read(V2eSlomo *h, float *conv_ms, int *conv_launches, double *conv_flops, void *stream) {
    if (!h || !conv_ms || !conv_launches || !conv_flops) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    return profile_collect(h, conv_ms, conv_launches, conv_flops, nullptr, nullptr, nullptr, stream);
}
extern "C" int v2e_slomo_profile_read_layers(V2eSlomo *h, float *ms23, int *launches23, double *flops23, float *conv_ms,
                                             int *conv_launches, double *conv_flops, void *stream) {
    if (!h || !ms23 || !launches23 || !flops23) return v2e_set_error(V2E_E_INVALID, "null argument%s", "");
    return profile_collect(h, conv_ms, conv_launches, conv_flops, ms23, launches23, flops23, stream);
}

extern "C" const float *v2e_slomo_flow_ptr(V2eSlomo *h) { return h ? h->flow_out : nullptr; }
extern "C" const float *v2e_slomo_intrp_ptr(V2eSlomo *h) { return h ? h->intrp_out : nullptr; }

extern "C" void *v2e_slomo_buffer_ptr(V2eSlomo *h, int which, int index) {
    if (!h) return nullptr;
    const bool level = index >= 0 && index < 5;
    switch (which) {
        case V2E_SLOMO_BUF_IN16: return h->in16;
        case V2E_SLOMO_BUF_X0: return h->x0;
        case V2E_SLOMO_BUF_S1: return h->s1;
        case V2E_SLOMO_BUF_POOL: return level ? h->pool[index] : nullptr;
        case V2E_SLOMO_BUF_DA: return level ? h->da[index] : nullptr;
        case V2E_SLOMO_BUF_S: return level ? h->s[index] : nullptr;
        case V2E_SLOMO_BUF_UP: return level ? h->up[index] : nullptr;
        case V2E_SLOMO_BUF_UA: return level ? h->ua[index] : nullptr;
        case V2E_SLOMO_BUF_UB: return level ? h->ub[index] : nullptr;
        case V2E_SLOMO_BUF_IMG: return h->img;
        default: return nullptr;
    }
}

extern "C" int v2e_slomo_layer_kernel(V2eSlomo *h, int net, int layer) {
    if (!h || net < 0 || net > 1 || layer < 0 || layer >= 23) return v2e_set_error(V2E_E_INVALID, "bad net / layer%s", "");
    return h->ran[net][layer];
}

// ---- Pillow-exact uint8 resize -------------------------------------------------------------------
struct V2eResizer {
    int sw, sh, dw, dh, filter, max_images;
    int *bounds_h, *kk_h, *bounds_v, *kk_v;
    int ks_h, ks_v;
    uint8_t *tmp;
};

extern "C" int v2e_resize_create(int sw, int sh, int dw, int dh, int filter, int max_images, V2eResizer **out) {
    if (!out || sw < 1 || sh < 1 || dw < 1 || dh < 1 || max_images < 1 || (filter != 0 && filter != 1))
        return v2e_set_error(V2E_E_INVALID, "bad resize arguments%s", "");
    V2eResizer *r = new V2eResizer();
    memset(r, 0, sizeof(*r));
    r->sw = sw; r->sh = sh; r->dw = dw; r->dh = dh; r->filter = filter; r->max_images = max_images;
    std::vector<int> b, k;
    if (sw != dw) {     // Pillow skips a pass whose size does not change (Resample.c: need_horizontal)
        r->ks_h = precompute_coeffs(sw, dw, filter, b, k);
        CU(cudaMalloc((void **)&r->bounds_h, b.size() * 4)); CU(cudaMalloc((void **)&r->kk_h, k.size() * 4));
        CU(cudaMemcpy(r->bounds_h, b.data(), b.size() * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(r->kk_h, k.data(), k.size() * 4, cudaMemcpyHostToDevice));
    }
    if (sh != dh) {
        r->ks_v = precompute_coeffs(sh, dh, filter, b, k);
        CU(cudaMalloc((void **)&r->bounds_v, b.size() * 4)); CU(cudaMalloc((void **)&r->kk_v, k.size() * 4));
        CU(cudaMemcpy(r->bounds_v, b.data(), b.size() * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(r->kk_v, k.data(), k.size() * 4, cudaMemcpyHostToDevice));
    }
    if (sw != dw && sh != dh) CU(cudaMalloc((void **)&r->tmp, (size_t)max_images * sh * dw));
    *out = r;
    return V2E_OK;
}

extern "C" int v2e_resize_destroy(V2eResizer *r) {
    if (!r) return V2E_OK;
    void *p[] = {r->bounds_h, r->kk_h, r->bounds_v, r->kk_v, r->tmp};
    for (void *q : p) if (q) cudaFree(q);
    delete r;
    return V2E_OK;
}

extern "C" int v2e_resize_run_strided(V2eResizer *r, const uint8_t *src_dev, uint8_t *dst_dev, int n_images,
                                      long dst_image_stride, void *stream) {
    if (!r || !src_dev || !dst_dev || n_images < 1 || n_images > r->max_images)
        return v2e_set_error(V2E_E_INVALID, "bad resize arguments%s", "");
    const long dense = (long)r->dw * r->dh;
    if (dst_image_stride < dense) return v2e_set_error(V2E_E_INVALID, "destination image stride smaller than an image%s", "");
    cudaStream_t st = (cudaStream_t)stream;
    const bool nh = r->sw != r->dw, nv = r->sh != r->dh;
    if (!nh && !nv) {
        CU(cudaMemcpy2DAsync(dst_dev, (size_t)dst_image_stride, src_dev, (size_t)dense, (size_t)dense, (size_t)n_images,
                             cudaMemcpyDeviceToDevice, st));
        return V2E_OK;
    }
    const uint8_t *cur = src_dev;
    if (nh) {
        uint8_t *d = nv ? r->tmp : dst_dev;
        const long n = (long)n_images * r->sh * r->dw;
        resample_h_u8_kernel<<<cdiv(n, 256), 256, 0, st>>>(cur, d, n_images, r->sw, r->sh, r->dw, r->bounds_h, r->kk_h, r->ks_h,
                                                           nv ? (long)r->sh * r->dw : dst_image_stride);
        cur = d;
    }
    if (nv) {
        const long n = (long)n_images * r->dh * r->dw;
        resample_v_u8_kernel<<<cdiv(n, 256), 256, 0, st>>>(cur, dst_dev, n_images, r->dw, r->sh, r->dh, r->bounds_v, r->kk_v, r->ks_v,
                                                           dst_image_stride);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return v2e_set_error(V2E_E_CUDA, "v2e_resize_run: %s", cudaGetErrorString(e));
    return V2E_OK;
}

extern "C" int v2e_resize_run(V2eResizer *r, const uint8_t *src_dev, uint8_t *dst_dev, int n_images, void *stream) {
    if (!r) return v2e_set_error(V2E_E_INVALID, "bad resize arguments%s", "");
    return v2e_resize_run_strided(r, src_dev, dst_dev, n_images, (long)r->dw * r->dh, stream);
}
