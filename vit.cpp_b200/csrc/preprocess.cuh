// preprocess.cuh -- vit_image_preprocess on the GPU (SURVEY.md 8(f) rank 1): u8 RGB image of any size -> bicubic (default) or
// bilinear resize to img_size^2 -> round to u8 -> (v - mean_c) / std_c -> image_f32 (HWC f32, vit.h:98-103), written straight
// into the engine's input buffer.  One thread per output pixel (three channels).
//
// The arithmetic reproduces the reference build operation for operation, including its quirks (reference vit.cpp:204-287):
//  * sampling position tx*j with NO half-pixel offset, clamp-to-edge taps, no anti-aliasing;
//  * cubic coefficients evaluated in DOUBLE (the literals -1.0/3, 1.0/6 promote the expression) and narrowed to float;
//  * the float polynomial a0 + a1 t + a2 t^2 + a3 t^3 with the fused multiply-adds gcc emits under -ffp-contract=fast
//    (checked in the disassembly of the reference build): fma(a1,t,a0); fma(a2*t,t,.); fma((a3*t)*t,t,.);
//  * the result is rounded to u8 (round half away from zero, clamped) BEFORE normalisation (vit.cpp:279-280);
//  * bilinear (vit.cpp:130-196) uses half-pixel centres: sx = fma(x+0.5, scale, -0.5).  (gcc fused the reference's three
//    unrolled channel iterations differently from each other; that per-channel pattern is not replicated, so a few values
//    per 10^4 differ by one u8 level in bilinear mode.  Bicubic, the default, matches the reference build.)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vitb200 {

struct PreImage
{
    size_t offset; // byte offset of this image's RGB data in the staging buffer
    int nx, ny;
};

__device__ __forceinline__ int pre_clipi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__device__ __forceinline__ float pre_cubic(float p0, float p1, float p2, float p3, float t)
{
    const float d0 = p0 - p1, d2 = p2 - p1, d3 = p3 - p1, a0 = p1;
    const float a1 = (float)fma(-(1.0 / 6), (double)d3, fma(-1.0 / 3, (double)d0, (double)d2));
    const float a2 = (float)fma(1.0 / 2, (double)d0, (1.0 / 2) * (double)d2);
    const float a3 = (float)fma(1.0 / 6, (double)d3, fma(-(1.0 / 2), (double)d2, (-1.0 / 6) * (double)d0));
    float r = __fmaf_rn(a1, t, a0);
    r = __fmaf_rn(__fmul_rn(a2, t), t, r);
    r = __fmaf_rn(__fmul_rn(__fmul_rn(a3, t), t), t, r);
    return r;
}

// out (image_f32 batch, may be NULL) and/or patches (may be NULL): the f16 patch matrix the patch-embedding GEMM reads through TMA,
// row = (image, patch), k = c*P*P + ky*P + kx (ggml.c:11597-11599), row pitch ldk -- written directly so that the f32 image never
// exists in HBM on the u8 path (the reference rounds the pixels to f16 for the conv anyway, ggml.c:11599).
__global__ void preprocess_kernel(const uint8_t *__restrict__ staging, const PreImage *__restrict__ imgs, float *__restrict__ out,
                                  int S, int bilinear, __half *__restrict__ patches, int P, int ldk)
{
    const int b = blockIdx.y;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= S * S) return;
    const int i = idx / S, j = idx - i * S; // output row, column
    const PreImage im = imgs[b];
    const uint8_t *src = staging + im.offset;
    const int nx = im.nx, ny = im.ny;
    const float m3[3] = {123.675f, 116.280f, 103.530f}; // vit.cpp:233-234
    const float s3[3] = {58.395f, 57.120f, 57.375f};
    float px3[3];
    float *dst = px3;
    if (!bilinear)
    {
        const float tx = __fdiv_rn((float)nx, (float)S), ty = __fdiv_rn((float)ny, (float)S);
        const float fx = __fmul_rn(tx, (float)j), fy = __fmul_rn(ty, (float)i);
        const int x = (int)fx, y = (int)fy;
        const float dx = fx - (float)x, dy = fy - (float)y;
        const int xs[4] = {pre_clipi(x - 1, 0, nx - 1), pre_clipi(x, 0, nx - 1), pre_clipi(x + 1, 0, nx - 1), pre_clipi(x + 2, 0, nx - 1)};
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            float C[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj)
            {
                const uint8_t *row = src + (size_t)pre_clipi(y - 1 + jj, 0, ny - 1) * nx * 3;
                C[jj] = pre_cubic((float)row[xs[0] * 3 + k], (float)row[xs[1] * 3 + k], (float)row[xs[2] * 3 + k], (float)row[xs[3] * 3 + k], dx);
            }
            const float Cc = pre_cubic(C[0], C[1], C[2], C[3], dy);
            const float v = fminf(fmaxf(roundf(Cc), 0.0f), 255.0f);
            dst[k] = __fdiv_rn((float)(uint8_t)v - m3[k], s3[k]);
        }
    }
    else
    {
        const float x_scale = __fdiv_rn((float)nx, (float)S), y_scale = __fdiv_rn((float)ny, (float)S);
        const float sx = __fmaf_rn((float)j + 0.5f, x_scale, -0.5f), sy = __fmaf_rn((float)i + 0.5f, y_scale, -0.5f);
        const int x0 = max(0, (int)floorf(sx)), y0 = max(0, (int)floorf(sy));
        const int x1 = min(x0 + 1, nx - 1), y1 = min(y0 + 1, ny - 1);
        const float dx = sx - (float)x0, dy = sy - (float)y0;
#pragma unroll
        for (int k = 0; k < 3; ++k)
        {
            const float v00 = src[3 * ((size_t)y0 * nx + x0) + k], v01 = src[3 * ((size_t)y0 * nx + x1) + k];
            const float v10 = src[3 * ((size_t)y1 * nx + x0) + k], v11 = src[3 * ((size_t)y1 * nx + x1) + k];
            const float v0 = __fmaf_rn(v00, 1.0f - dx, __fmul_rn(v01, dx));
            const float v1 = __fmaf_rn(v10, 1.0f - dx, __fmul_rn(v11, dx));
            const float v = __fmaf_rn(v1, dy, __fmul_rn(v0, 1.0f - dy));
            const float r = fminf(fmaxf(roundf(v), 0.0f), 255.0f);
            dst[k] = __fdiv_rn((float)(uint8_t)r - m3[k], s3[k]);
        }
    }
    if (out)
    {
        float *o = out + ((size_t)b * S * S + idx) * 3;
        o[0] = px3[0]; o[1] = px3[1]; o[2] = px3[2];
    }
    if (patches)
    {
        const int G = S / P, py = i / P, ky = i - py * P, pxi = j / P, kx = j - pxi * P;
        __half *row = patches + ((size_t)b * G * G + (size_t)py * G + pxi) * ldk + ky * P + kx;
#pragma unroll
        for (int k = 0; k < 3; ++k) row[k * P * P] = __float2half_rn(px3[k]);
    }
}

// ---- The ViTSTR extension's vit_image_preprocess (reference extensions/vitstr.cpp:128-201): u8 RGB -> grayscale -> bilinear resize
// to img_size^2 -> (v / 255 - 0.5) * 2, 1 channel, no rounding to u8 in between.  Operation for operation as the extension's build
// (gcc -O3 -mavx2 -mfma, -std=gnu++11 so contraction is on) computes it, read off its disassembly:
//  * rgb_to_grayscale (vitstr.cpp:128-132, an out-of-line scalar function) in DOUBLE: fma(0.114, b, fma(0.299, r, 0.587 * g)),
//    truncated to u8.  Not an identity on gray pixels: 75 of the 256 levels (v, v, v) come out as v - 1 (0.99...9 truncates);
//  * the resize (vitstr.cpp:150-172) in float, sampling at x * (nx / S) with NO half-pixel offset; u = gx - (int)gx is taken
//    BEFORE the clamp px0 = max(0, min(gxi, nx - 2)) and not recomputed after it, so the last columns / rows extrapolate towards
//    px0 + 1 <= nx - 1.  The four products are summed as fma(g11, u*v, fma(g10, (1-u)*v, fma(g00, (1-u)*(1-v), (u*(1-v)) * g01)));
//  * normalisation (vitstr.cpp:175): val / 255 - 0.5, times 2.  The padding loops (vitstr.cpp:181-198) never run.
// Images narrower or shorter than 2 pixels are rejected on the host (the extension reads outside such an image).
__device__ __forceinline__ float gray_level(const uint8_t *rgb)
{
    const double y = __fma_rn(0.114, (double)rgb[2], __fma_rn(0.299, (double)rgb[0], __dmul_rn(0.587, (double)rgb[1])));
    return (float)(uint8_t)(int)y;
}

// out (float32 [B][S][S], may be NULL) and/or patches (may be NULL): the 1-channel f16 patch matrix of the patch-embedding GEMM,
// k = ky*P + kx, row pitch ldk.  Same staging layout (PreImage table + interleaved RGB u8) as preprocess_kernel.
__global__ void preprocess_gray_kernel(const uint8_t *__restrict__ staging, const PreImage *__restrict__ imgs, float *__restrict__ out,
                                       int S, __half *__restrict__ patches, int P, int ldk)
{
    const int b = blockIdx.y;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= S * S) return;
    const int y = idx / S, x = idx - y * S; // output row, column
    const PreImage im = imgs[b];
    const uint8_t *src = staging + im.offset;
    const int nx = im.nx, ny = im.ny;
    const float x_scale = __fdiv_rn((float)nx, (float)S), y_scale = __fdiv_rn((float)ny, (float)S);
    const float gx = __fmul_rn((float)x, x_scale), gy = __fmul_rn((float)y, y_scale);
    const int gxi = (int)gx, gyi = (int)gy;
    const float u = __fsub_rn(gx, (float)gxi), v = __fsub_rn(gy, (float)gyi);
    const int px0 = max(0, min(gxi, nx - 2)), py0 = max(0, min(gyi, ny - 2));
    const uint8_t *r0 = src + (size_t)py0 * nx * 3, *r1 = r0 + (size_t)nx * 3;
    const float g00 = gray_level(r0 + px0 * 3), g01 = gray_level(r0 + px0 * 3 + 3);
    const float g10 = gray_level(r1 + px0 * 3), g11 = gray_level(r1 + px0 * 3 + 3);
    const float omu = __fsub_rn(1.0f, u), omv = __fsub_rn(1.0f, v);
    float val = __fmul_rn(__fmul_rn(u, omv), g01);
    val = __fmaf_rn(__fmul_rn(omu, omv), g00, val);
    val = __fmaf_rn(__fmul_rn(omu, v), g10, val);
    val = __fmaf_rn(__fmul_rn(u, v), g11, val);
    val = __fmul_rn(__fsub_rn(__fdiv_rn(val, 255.0f), 0.5f), 2.0f);
    if (out) out[(size_t)b * S * S + idx] = val;
    if (patches)
    {
        const int G = S / P, py = y / P, ky = y - py * P, pxi = x / P, kx = x - pxi * P;
        patches[((size_t)b * G * G + (size_t)py * G + pxi) * ldk + ky * P + kx] = __float2half_rn(val);
    }
}

// The extension's greedy decode (vitstr.cpp:1020-1054), one thread per image: the arg-max of token rows 1 .. TH-1 in order (top1_idx /
// top1_val: softmax_topk_kernel with k = 1, whose tie rule -- lowest index among equal maxima -- is the extension's `>` scan from
// class 0), stopping at the first row whose arg-max is class 1 ([s], end of sentence).  chars [B][TH-1] (-1 past the end),
// lengths [B], scores [B] = the product of the emitted maxima in double, multiplied in token order (`conf *= max_value`; 1 if empty).
__global__ void vitstr_decode_kernel(const int32_t *__restrict__ top1_idx, const float *__restrict__ top1_val, int B, int TH,
                                     int32_t *__restrict__ chars, int32_t *__restrict__ lengths, double *__restrict__ scores)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int n = TH - 1;
    double conf = 1.0;
    int len = 0;
    bool eos = false;
    for (int t = 1; t < TH; ++t)
    {
        const size_t row = (size_t)b * TH + t;
        const int id = top1_idx[row];
        eos = eos || id == 1;
        chars[(size_t)b * n + t - 1] = eos ? -1 : id;
        if (eos) continue;
        conf = __dmul_rn(conf, (double)top1_val[row]);
        ++len;
    }
    lengths[b] = len;
    scores[b] = conf;
}

} // namespace vitb200
