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
    // a size the patch does not divide (SigLIP's floor grid): pixels at or past G P belong to no patch, and a row for them would be the
    // next image's
    const int G = S / P;
    if (patches && i < G * P && j < G * P)
    {
        const int py = i / P, ky = i - py * P, pxi = j / P, kx = j - pxi * P;
        __half *row = patches + ((size_t)b * G * G + (size_t)py * G + pxi) * ldk + ky * P + kx;
#pragma unroll
        for (int k = 0; k < 3; ++k) row[k * P * P] = __float2half_rn(px3[k]);
    }
}

// ---- Hugging Face's PIL image processors (vitb200_image_proc; CLIPImageProcessor, SiglipImageProcessor, BitImageProcessor with the
// PIL backend): Pillow's 8-bit ImagingResample (bicubic a = -0.5 or bilinear, anti-aliased when downscaling) to the resized size, HF's
// centre crop, x = f32(f64(v) * rescale_factor), y = (x - mean_c) / std_c in f32.  Two kernels, only over the crop window (an output
// pixel depends on its own taps alone, so this gives Pillow's bits for the whole image cropped afterwards):
//   image_proc_h_kernel  the horizontal pass: the crop's S columns of the source rows the vertical taps reach, rounded to u8, into a
//                        per-slot scratch [rows][S][3];
//   image_proc_v_kernel  the vertical pass over that scratch, rounded to u8, then rescale and normalise, written like preprocess_kernel.
// Pillow runs the horizontal pass first and rounds in between, so the order is fixed.  It skips a pass whose axis keeps its size; here
// such a pass is one tap of weight 1 << 22, the identity, which is what Pillow's coefficients would be too.
// Coefficients are Pillow's precompute_coeffs + normalize_coeffs_8bpc in double, operation for operation with explicit roundings: a
// contracted multiply-add moves a coefficient, and one coefficient moves a pixel by a level.  Each CTA computes the ones it needs into
// shared memory, laid out [tap][row or column] so that the threads of a warp read different banks.
constexpr int PIL_PRECISION_BITS = 22;   // Pillow's 32 - 8 - 2
constexpr int IMG_PROC_H_COLS = 32;      // output columns per CTA of the horizontal pass (one per lane)
constexpr int IMG_PROC_H_ROWS = 64;      // source rows per CTA of the horizontal pass (8 warps, 8 rows each)
constexpr int IMG_PROC_V_ROWS = 8;       // output rows per CTA of the vertical pass

// Per image, computed on the host in 64-bit integers: the resized size, the crop's offset in it, and the source rows the horizontal
// pass writes (y0 .. y0 + rows - 1) at byte offset tmp of the scratch
struct ProcGeom
{
    size_t tmp;
    int ow, oh, left, top, y0, rows;
};

struct ProcNorm
{
    double rescale;
    float mean[3], std_[3];
};

__device__ __forceinline__ double pil_filter(double x, int resample)
{
    x = fabs(x);
    if (resample == 2) return x < 1.0 ? __dsub_rn(1.0, x) : 0.0; // bilinear_filter
    // bicubic_filter, a = -0.5: ((a + 2) x - (a + 3)) x x + 1 and (((x - 5) x + 8) x - 4) a
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
    return 0.0;
}

// Fixed-point taps of output index xx of a resize in -> out along one axis, into k[t * stride] (t < K); *first = the first source index,
// *n = the tap count.  in == out: the identity tap.
__device__ void pil_coeffs(int in, int out, int xx, int resample, int K, int *k, int stride, int *first, int *n)
{
    if (in == out)
    {
        *first = xx; *n = 1; k[0] = 1 << PIL_PRECISION_BITS;
        return;
    }
    const double scale = __ddiv_rn((double)in, (double)out);
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = __dmul_rn(resample == 2 ? 1.0 : 2.0, filterscale);
    const double ss = __ddiv_rn(1.0, filterscale);
    const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), scale);
    int xmin = (int)__dadd_rn(__dsub_rn(center, support), 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)__dadd_rn(__dadd_rn(center, support), 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    if (xmax > K) xmax = K; // cannot happen: K = ceil(support) * 2 + 1 bounds Pillow's tap count
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) ww = __dadd_rn(ww, pil_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss), resample));
    for (int x = 0; x < xmax; ++x)
    {
        double w = pil_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss), resample);
        if (ww != 0.0) w = __ddiv_rn(w, ww);
        const double f = __dmul_rn(w, (double)(1 << PIL_PRECISION_BITS));
        k[x * stride] = w < 0 ? (int)__dadd_rn(-0.5, f) : (int)__dadd_rn(0.5, f);
    }
    *first = xmin; *n = xmax;
}

__device__ __forceinline__ uint8_t pil_clip8(int v) { return (uint8_t)(v <= 0 ? 0 : (v >> PIL_PRECISION_BITS > 255 ? 255 : v >> PIL_PRECISION_BITS)); }

// grid (ceil(S / 32), ceil(max rows / 64), batch), 256 threads; dynamic shared memory 32 * (K + 2) ints
__global__ void image_proc_h_kernel(const uint8_t *__restrict__ staging, const PreImage *__restrict__ imgs, const ProcGeom *__restrict__ geo,
                                    uint8_t *__restrict__ tmp, int S, int resample, int K)
{
    extern __shared__ int pil_k[]; // [K][32] taps, then first[32], n[32]
    const int b = blockIdx.z;
    const ProcGeom g = geo[b];
    const int r0 = blockIdx.y * IMG_PROC_H_ROWS;
    if (r0 >= g.rows) return;
    const PreImage im = imgs[b];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * IMG_PROC_H_COLS + lane;
    int *first = pil_k + K * IMG_PROC_H_COLS, *count = first + IMG_PROC_H_COLS;
    if (warp == 0 && j < S) pil_coeffs(im.nx, g.ow, g.left + j, resample, K, pil_k + lane, IMG_PROC_H_COLS, first + lane, count + lane);
    __syncthreads();
    if (j >= S) return;
    const int x0 = first[lane], n = count[lane];
    const int r1 = min(r0 + IMG_PROC_H_ROWS, g.rows);
    for (int r = r0 + warp; r < r1; r += 8)
    {
        const uint8_t *src = staging + im.offset + ((size_t)(g.y0 + r) * im.nx + x0) * 3;
        int s0 = 1 << (PIL_PRECISION_BITS - 1), s1 = s0, s2 = s0;
        for (int t = 0; t < n; ++t)
        {
            const int k = pil_k[t * IMG_PROC_H_COLS + lane];
            s0 += (int)src[3 * t] * k; s1 += (int)src[3 * t + 1] * k; s2 += (int)src[3 * t + 2] * k;
        }
        uint8_t *o = tmp + g.tmp + ((size_t)r * S + j) * 3;
        o[0] = pil_clip8(s0); o[1] = pil_clip8(s1); o[2] = pil_clip8(s2);
    }
}

// grid (ceil(S / 8), batch), 256 threads; dynamic shared memory 8 * (K + 2) ints.  Launched programmatically: the taps are computed
// while the horizontal pass finishes, the scratch is read after griddepcontrol.wait.  out / patches as preprocess_kernel.
__global__ void image_proc_v_kernel(const uint8_t *__restrict__ tmp, const PreImage *__restrict__ imgs, const ProcGeom *__restrict__ geo,
                                    float *__restrict__ out, int S, int resample, int K, ProcNorm nm, __half *__restrict__ patches, int P, int ldk)
{
    extern __shared__ int pil_k[]; // [K][8] taps, then first[8], n[8]
    const int b = blockIdx.y;
    const ProcGeom g = geo[b];
    const PreImage im = imgs[b];
    const int i0 = blockIdx.x * IMG_PROC_V_ROWS;
    int *first = pil_k + K * IMG_PROC_V_ROWS, *count = first + IMG_PROC_V_ROWS;
    if (threadIdx.x < IMG_PROC_V_ROWS && i0 + (int)threadIdx.x < S)
        pil_coeffs(im.ny, g.oh, g.top + i0 + threadIdx.x, resample, K, pil_k + threadIdx.x, IMG_PROC_V_ROWS, first + threadIdx.x,
                   count + threadIdx.x);
    __syncthreads();
    ptx::grid_dep_wait();
    const int G = S / P;
    for (int p = threadIdx.x; p < IMG_PROC_V_ROWS * S; p += blockDim.x)
    {
        const int il = p / S, j = p - il * S, i = i0 + il;
        if (i >= S) break;
        const int n = count[il];
        const int y = min(max(first[il] - g.y0, 0), g.rows - n); // always first - y0; clamped so the reads stay in the scratch
        const uint8_t *src = tmp + g.tmp + ((size_t)y * S + j) * 3;
        int s[3] = {1 << (PIL_PRECISION_BITS - 1), 1 << (PIL_PRECISION_BITS - 1), 1 << (PIL_PRECISION_BITS - 1)};
        for (int t = 0; t < n; ++t)
        {
            const int k = pil_k[t * IMG_PROC_V_ROWS + il];
            const uint8_t *q = src + (size_t)t * S * 3;
            s[0] += (int)q[0] * k; s[1] += (int)q[1] * k; s[2] += (int)q[2] * k;
        }
        float px3[3];
#pragma unroll
        for (int c = 0; c < 3; ++c)
        {
            const float x = (float)__dmul_rn((double)pil_clip8(s[c]), nm.rescale);
            px3[c] = __fdiv_rn(__fsub_rn(x, nm.mean[c]), nm.std_[c]);
        }
        if (out)
        {
            float *o = out + ((size_t)b * S * S + (size_t)i * S + j) * 3;
            o[0] = px3[0]; o[1] = px3[1]; o[2] = px3[2];
        }
        if (patches && i < G * P && j < G * P) // pixels past the floor grid belong to no patch (preprocess_kernel)
        {
            const int py = i / P, ky = i - py * P, pxi = j / P, kx = j - pxi * P;
            __half *row = patches + ((size_t)b * G * G + (size_t)py * G + pxi) * ldk + ky * P + kx;
#pragma unroll
            for (int c = 0; c < 3; ++c) row[c * P * P] = __float2half_rn(px3[c]);
        }
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
