// kernels.cuh -- the non-GEMM kernels of the forward path (all HBM-bound except attention):
//   patchify_f16_kernel      reference im2col for stride==kernel conv (ggml.c:11528-11608) without the buffer
//                            reshuffle: pixels HWC f32 -> f16 patch rows, K order c*P*P + ky*P + kx
//   cls_rows_kernel          token 0 = cls_token + pos_embed[0] (vit.cpp:794-797), and the register tokens after it
//   cls_patch_mean_kernel    DINOv2's classifier input: LN(token 0) || the mean of LN(patch rows), one CTA per image; without a class
//                            token (SigLIP) the mean alone
//   attention_pool_kernel    SigLIP's attention-pooling head: one learned query attending over an image's token rows, per head
//                            (head dims 64 and 72)
//   token_embed_kernel       text towers: token rows = the token table's row of each id + pos_embed, replacing the patch embedding
//   text_pool_kernel         text towers: the pooled row of each sequence (CLIP's EOS row, SigLIP's last row) through the final LayerNorm
//   layernorm_f16_kernel     ggml_norm * w + b (ggml.c:8959-9008, vit.cpp:808-812) emitting the f16 A operand; its f32 / bf16
//                            and un-normalised forms write the encoder features (vitb200_features), its e4m3 form the FP8 A operand
//   layernorm_inplace_kernel the same arithmetic in place on f32 rows (the pre-norm of CLIP towers)
//   attention_kernel         per (image, head): S = QK^T / sqrt(hd), softmax with the reference's f16-exp
//                            semantics (ggml.c:10536-10558), O = P V   (vit.cpp:826-866)
//   softmax_topk_kernel      final soft-max (vit.cpp:931) + top-k (replaces the host std::sort, vit.cpp:1047-1057); its sigmoid form
//                            for SigLIP's zero-shot head
//   zero_shot_kernel         the zero-shot head (vitb200_set_zero_shot): cosine similarity of each head row with the class matrix, scaled
#pragma once
#include "ptx.cuh"

#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <type_traits>

namespace vitb200 {

// ------------------------------------------------------------------------------------------------
// images [B][S][S][C] f32 (HWC, vit.h:98-103; C = 1 for the ViTSTR extension's grayscale input) -> A [B*G*G][ldk] f16,
// k = c*P*P + ky*P + kx.  One thread per (image, patch row py, kernel row ky, patch column px): reads P*C contiguous floats.
template <int P, int C = 3>
__global__ void patchify_f16_kernel(const float *__restrict__ img, __half *__restrict__ A, int B, int S, int G, int ldk)
{
    const long long total = (long long)B * G * P * G;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x)
    {
        const int px = (int)(idx % G);
        long long r = idx / G;
        const int ky = (int)(r % P);
        r /= P;
        const int py = (int)(r % G);
        const int b = (int)(r / G);
        const float *src = img + (((size_t)b * S + (size_t)(py * P + ky)) * S + (size_t)px * P) * C;
        float v[P * C];
        if constexpr ((P * C) % 4 == 0 && (P % 4) == 0)
        {
#pragma unroll
            for (int i = 0; i < P * C / 4; ++i)
            {
                const float4 f = __ldg(reinterpret_cast<const float4 *>(src) + i);
                v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w;
            }
        }
        else
        {
#pragma unroll
            for (int i = 0; i < P * C; ++i) v[i] = __ldg(src + i);
        }
        __half *dst = A + ((size_t)b * G * G + (size_t)py * G + px) * ldk + ky * P;
#pragma unroll
        for (int c = 0; c < C; ++c)
        {
            __half2 *d2 = reinterpret_cast<__half2 *>(dst + c * P * P);
#pragma unroll
            for (int kx = 0; kx < P; kx += 2)
                d2[kx >> 1] = __floats2half2_rn(v[kx * C + c], v[(kx + 1) * C + c]); // RNE, ggml.c:11599
        }
    }
}

// P = 16, 3 channels: one WARP per patch.  Lane (ky = lane / 2, half = lane % 2) reads the 8 pixels x 3 channels (96 contiguous bytes)
// of its half kernel row and writes, per channel, the 8 f16 values at k = c*256 + ky*16 + half*8: the warp's stores are three fully
// coalesced 512-byte runs of the patch's A row, its loads sixteen 192-byte row segments.  (The thread-per-kernel-row mapping above
// scatters 32-byte stores over 32 different A rows per warp: 1.5 TB/s at batch 256.)
__global__ void patchify16_warp_kernel(const float *__restrict__ img, __half *__restrict__ A, int n_patches, int S, int G, int ldk)
{
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int pidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; pidx < n_patches; pidx += warps)
    {
        const int b = pidx / (G * G), pp = pidx - b * G * G, py = pp / G, px = pp - py * G;
        const int ky = lane >> 1, half = lane & 1;
        const float4 *src = reinterpret_cast<const float4 *>(img + (((size_t)b * S + (size_t)(py * 16 + ky)) * S + (size_t)px * 16 + half * 8) * 3);
        float v[24];
#pragma unroll
        for (int i = 0; i < 6; ++i)
        {
            const float4 f = __ldg(src + i);
            v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w;
        }
        __half *dst = A + (size_t)pidx * ldk + ky * 16 + half * 8;
#pragma unroll
        for (int c = 0; c < 3; ++c)
        {
            uint32_t w[4];
#pragma unroll
            for (int e = 0; e < 4; ++e)
            {
                const __half2 h2 = __floats2half2_rn(v[(2 * e) * 3 + c], v[(2 * e + 1) * 3 + c]); // RNE, ggml.c:11599
                w[e] = *reinterpret_cast<const uint32_t *>(&h2);
            }
            *reinterpret_cast<uint4 *>(dst + c * 256) = make_uint4(w[0], w[1], w[2], w[3]);
        }
    }
}

// The prefix rows r = 0 .. rows-1 of every image: x[b*ntok + r][:] = prefix[r][:] + pos[r][:], prefix = [cls_token; reg_token]
// (rows = 1 + vitb200_arch.reg_tokens; the patch GEMM writes the rows after them)
__global__ void cls_rows_kernel(float *__restrict__ x, const float *__restrict__ prefix, const float *__restrict__ pos, int B, int rows, int ntok,
                                int D)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * rows * D) return;
    const int b = i / (rows * D), o = i - b * rows * D; // o = r D + column
    x[(size_t)b * ntok * D + o] = __fadd_rn(prefix[o], pos[o]);
}

// ------------------------------------------------------------------------------------------------
// The LayerNorm arithmetic, written once for every LayerNorm kernel below: f32 mean and biased variance (the reference sums in
// double; the difference is ~1e-7 relative), y = ((x - mean) * scale) * w + b as three separately rounded f32 ops like the reference's
// NORM, MUL, ADD nodes, and the FP8 engine's per-row e4m3 quantisation of y.  A warp holds a row, float4 j of lane l being float4
// l + 32 j of the row.

// Butterfly reductions over the 32 lanes: every lane gets the result
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// A lane's part of the row sum
__device__ __forceinline__ float sum4(float4 v) { return (v.x + v.y) + (v.z + v.w); }

// Centres the lane's float4 of the row (those with index < nvec) on the row mean, given the lane's part of the row sum, and returns
// scale = 1 / sqrt(biased variance + eps)
template <int MAXV>
__device__ __forceinline__ float ln_center(float4 (&v)[MAXV], float sum, int lane, int nvec, int D, float eps)
{
    const float mean = warp_sum(sum) / (float)D;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
    {
        if (lane + 32 * j < nvec)
        {
            v[j].x -= mean; v[j].y -= mean; v[j].z -= mean; v[j].w -= mean;
            sq += (v[j].x * v[j].x + v[j].y * v[j].y) + (v[j].z * v[j].z + v[j].w * v[j].w);
        }
    }
    return 1.0f / sqrtf(warp_sum(sq) / (float)D + eps);
}

// The affine of a centred float4: (v * scale) * w + b, each op rounded
__device__ __forceinline__ float4 ln_affine(float4 v, float scale, float4 w, float4 b)
{
    return make_float4(__fadd_rn(__fmul_rn(__fmul_rn(v.x, scale), w.x), b.x), __fadd_rn(__fmul_rn(__fmul_rn(v.y, scale), w.y), b.y),
                       __fadd_rn(__fmul_rn(__fmul_rn(v.z, scale), w.z), b.z), __fadd_rn(__fmul_rn(__fmul_rn(v.w, scale), w.w), b.w));
}

// e4m3 rows: amax = max |y| over the row (abs_max4: a lane's part, then warp_max), the row's scale amax / 448 and
// y = e4m3_rn_satfinite(y (448 / amax)); an all-zero row gets scale 1.  (The scale and the multiplier are two functions: one function
// computing both changes the code the compiler generates for its callers.)
__device__ __forceinline__ float abs_max4(float4 v) { return fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))); }
__device__ __forceinline__ float e4m3_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f; }
__device__ __forceinline__ float e4m3_multiplier(float amax) { return amax > 0.f ? __fdiv_rn(448.f, amax) : 1.f; }

__device__ __forceinline__ uint32_t e4m3x4(float4 v, float inv)
{
    return ptx::cvt_e4m3x4(__fmul_rn(v.x, inv), __fmul_rn(v.y, inv), __fmul_rn(v.z, inv), __fmul_rn(v.w, inv));
}

// Four f32 values rounded to nearest even f16 or bf16 (OutT), packed in order
template <typename OutT>
__device__ __forceinline__ uint2 pack4(float4 v)
{
    uint2 u;
    if constexpr (std::is_same<OutT, __half>::value)
    {
        const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
        u.x = *reinterpret_cast<const uint32_t *>(&h0);
        u.y = *reinterpret_cast<const uint32_t *>(&h1);
    }
    else
    {
        const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
        u.x = *reinterpret_cast<const uint32_t *>(&h0);
        u.y = *reinterpret_cast<const uint32_t *>(&h1);
    }
    return u;
}

// Four f32 results -> OutT, stored at float4 index i of a row.  16-bit outputs pair up neighbouring lanes (lanes 2k and 2k+1 hold
// consecutive float4 indices) so that the even lane issues one 16-byte store for both; `vec16` requires an even float4 count per row.
// Every lane of the warp must call this (shuffles), `live` says whether its own index is inside the row.
template <typename OutT>
__device__ __forceinline__ void store4(OutT *__restrict__ yr, int i, bool live, bool vec16, float o0, float o1, float o2, float o3)
{
    if constexpr (sizeof(OutT) == 4)
    {
        if (live) reinterpret_cast<float4 *>(yr)[i] = make_float4(o0, o1, o2, o3);
    }
    else
    {
        const uint2 u = pack4<OutT>(make_float4(o0, o1, o2, o3));
        if (vec16)
        {
            const uint32_t nx = __shfl_xor_sync(0xffffffffu, u.x, 1), ny = __shfl_xor_sync(0xffffffffu, u.y, 1);
            if (live && !(threadIdx.x & 1)) reinterpret_cast<uint4 *>(yr)[i >> 1] = make_uint4(u.x, u.y, nx, ny);
        }
        else if (live)
            reinterpret_cast<uint2 *>(yr)[i] = u;
    }
}

// One warp per row: the LayerNorm above, then RNE to f16 (the GEMM's src1 conversion, ggml.c:9493-9506).
// OutT = float stores the f32 values before that rounding, __nv_bfloat16 rounds them to nearest even bf16 instead.
// NORM = false skips the normalisation: the selected rows of x are converted and stored as they are (w and b are not read).
// OutT = __nv_fp8_e4m3 (FP8 engine, NORM only) quantises each row with its own scale, y_scale[row].
// The body is a device function so that the in-place form below can run it with y == x: a warp holds its whole row in registers
// before it writes any of it, and no two warps share a row.
template <int MAXV, typename OutT, bool NORM>
__device__ __forceinline__ void layernorm_row_warp(const float *x, size_t x_row_stride, int rows_per_group, size_t group_stride, const float *w,
                                                   const float *b, OutT *y, int rows, int D, float eps, float *y_scale)
{
    constexpr bool kE4M3 = std::is_same<OutT, __nv_fp8_e4m3>::value;
    static_assert(!kE4M3 || NORM, "e4m3 output: normalised rows only");
    const int warps_per_block = blockDim.x >> 5;
    // rows are taken LAST FIRST: the producing GEMM wrote them in ascending order, so the tail of X is what the 50 MB L2 still
    // holds when this kernel starts (and the GEMM that follows, walking up from row 0, meets this kernel's freshest output)
    const int row = rows - 1 - (blockIdx.x * warps_per_block + (threadIdx.x >> 5));
    if (row < 0) return;
    const int lane = threadIdx.x & 31;
    const int nvec = D >> 2;
    // input row = group g (an image), member t (a token): all T rows are one group for the block LayerNorms; the pooled head
    // takes the first rows_per_group tokens of every image (token 0: vit.cpp:910; 25 tokens: vitstr.cpp:864-883)
    const int g = row / rows_per_group, t = row - g * rows_per_group;
    const float4 *xr = reinterpret_cast<const float4 *>(x + (size_t)g * group_stride + (size_t)t * x_row_stride);
    float4 v[MAXV];
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
    {
        const int i = lane + 32 * j;
        if (i < nvec)
        {
            v[j] = xr[i];
            sum += sum4(v[j]);
        }
    }
    float scale = 1.f;
    if constexpr (NORM) scale = ln_center(v, sum, lane, nvec, D, eps);
    const float4 *w4 = reinterpret_cast<const float4 *>(w);
    const float4 *b4 = reinterpret_cast<const float4 *>(b);
    const bool vec16 = (nvec & 1) == 0;
    OutT *yr = y + (size_t)row * D;
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
    {
        const int i = lane + 32 * j;
        float o0 = 0.f, o1 = 0.f, o2 = 0.f, o3 = 0.f; // four floats, not a float4: that reorders the f16 / bf16 packing
        if (i < nvec)
        {
            float4 o = v[j];
            if constexpr (NORM) o = ln_affine(v[j], scale, __ldg(w4 + i), __ldg(b4 + i));
            o0 = o.x; o1 = o.y; o2 = o.z; o3 = o.w;
        }
        if constexpr (kE4M3)
        {
            v[j] = make_float4(o0, o1, o2, o3);
            amax = fmaxf(amax, abs_max4(v[j]));
        }
        else store4(yr, i, i < nvec, vec16, o0, o1, o2, o3);
    }
    if constexpr (kE4M3)
    {
        amax = warp_max(amax);
        const float inv = e4m3_multiplier(amax);
        if (lane == 0) y_scale[row] = e4m3_row_scale(amax);
#pragma unroll
        for (int j = 0; j < MAXV; ++j)
        {
            const int i = lane + 32 * j;
            if (i < nvec) reinterpret_cast<uint32_t *>(yr)[i] = e4m3x4(v[j], inv);
        }
    }
}

template <int MAXV, typename OutT = __half, bool NORM = true>
__global__ void layernorm_f16_kernel(const float *__restrict__ x, size_t x_row_stride, int rows_per_group, size_t group_stride,
                                     const float *__restrict__ w, const float *__restrict__ b, OutT *__restrict__ y, int rows,
                                     int D, float eps, float *__restrict__ y_scale)
{
    ptx::grid_dep_launch(); // PDL: blocks may be resident before the producing GEMM has drained
    ptx::grid_dep_wait();
    layernorm_row_warp<MAXV, OutT, NORM>(x, x_row_stride, rows_per_group, group_stride, w, b, y, rows, D, eps, y_scale);
}

// The same LayerNorm in place on `rows` consecutive f32 rows of x (the pre-norm of CLIP towers, on the residual stream before block 0):
// f32 in, f32 out, no rounding to f16
template <int MAXV>
__global__ void layernorm_inplace_kernel(float *x, const float *__restrict__ w, const float *__restrict__ b, int rows, int D, float eps)
{
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();
    layernorm_row_warp<MAXV, float, true>(x, (size_t)D, rows, 0, w, b, x, rows, D, eps, nullptr);
}

// ------------------------------------------------------------------------------------------------
// DINOv2's classifier input (vitb200_arch.pool = 1): per image, y[0 .. D) = LN(token 0) and y[D .. 2 D) = the mean over the patch rows
// first_patch .. ntok-1 of LN(row) (the register rows between them are left out), LN = layernorm_row_regs
// (NORM = false: the rows as they are).  first_patch = 0 (no class token, vitb200_arch.pool = 3): y[0 .. D) = the mean over all ntok rows,
// rows of D.  One CTA of 8 warps per image: warp w normalises patch rows w, w + 8, ... and keeps its column
// sums in registers in that order; the eight partial sums then meet in shared memory and are added warp 0 first, 7 last, and divided
// by the patch count.  No atomics and nothing shared between images: an image gives the same bits alone as in any batch.
// OutT: __half (the head GEMM's A operand [B][2 D] or [B][D]), float or __nv_bfloat16 (the features' prelogits).  Dynamic shared memory
// 8 D floats.
constexpr int POOL_WARPS = 8;

template <typename OutT>
__device__ __forceinline__ OutT to_out(float v)
{
    if constexpr (std::is_same<OutT, __half>::value) return __float2half_rn(v);
    else if constexpr (std::is_same<OutT, __nv_bfloat16>::value) return __float2bfloat16_rn(v);
    else return v;
}

// One row of D floats into a warp's registers, normalised (NORM = false: as it is): lane l holds float4 l + 32 j of the row in o[j]
template <int MAXV, bool NORM>
__device__ __forceinline__ void layernorm_row_regs(const float *__restrict__ xrow, const float *__restrict__ w, const float *__restrict__ b,
                                                   int D, float eps, int lane, float4 (&o)[MAXV])
{
    const int nvec = D >> 2;
    const float4 *xr = reinterpret_cast<const float4 *>(xrow);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
    {
        const int i = lane + 32 * j;
        o[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < nvec)
        {
            o[j] = xr[i];
            sum += sum4(o[j]);
        }
    }
    if constexpr (NORM)
    {
        const float scale = ln_center(o, sum, lane, nvec, D, eps);
        const float4 *w4 = reinterpret_cast<const float4 *>(w);
        const float4 *b4 = reinterpret_cast<const float4 *>(b);
#pragma unroll
        for (int j = 0; j < MAXV; ++j)
        {
            const int i = lane + 32 * j;
            if (i < nvec) o[j] = ln_affine(o[j], scale, __ldg(w4 + i), __ldg(b4 + i));
        }
    }
}

template <int MAXV, typename OutT = __half, bool NORM = true>
__global__ void __launch_bounds__(POOL_WARPS * 32)
cls_patch_mean_kernel(const float *__restrict__ x, int ntok, int first_patch, const float *__restrict__ w, const float *__restrict__ b,
                      OutT *__restrict__ y, int D, float eps)
{
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();
    extern __shared__ float4 s_part[]; // [POOL_WARPS][D / 4]
    const int img = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nvec = D >> 2;
    const float *xi = x + (size_t)img * ntok * D;
    const int cls = first_patch > 0 ? 1 : 0; // 1: the row starts with LN(token 0)
    OutT *yi = y + (size_t)img * (1 + cls) * D;
    float4 o[MAXV], acc[MAXV];
#pragma unroll
    for (int j = 0; j < MAXV; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = first_patch + warp; r < ntok; r += POOL_WARPS)
    {
        layernorm_row_regs<MAXV, NORM>(xi + (size_t)r * D, w, b, D, eps, lane, o);
#pragma unroll
        for (int j = 0; j < MAXV; ++j)
        {
            acc[j].x = __fadd_rn(acc[j].x, o[j].x); acc[j].y = __fadd_rn(acc[j].y, o[j].y);
            acc[j].z = __fadd_rn(acc[j].z, o[j].z); acc[j].w = __fadd_rn(acc[j].w, o[j].w);
        }
    }
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
        if (lane + 32 * j < nvec) s_part[warp * nvec + lane + 32 * j] = acc[j];
    if (cls && warp == 0)
    {
        // the class row, under the other warps' wait at the barrier
        layernorm_row_regs<MAXV, NORM>(xi, w, b, D, eps, lane, o);
#pragma unroll
        for (int j = 0; j < MAXV; ++j)
        {
            const int i = lane + 32 * j;
            if (i < nvec)
            {
                yi[4 * i] = to_out<OutT>(o[j].x); yi[4 * i + 1] = to_out<OutT>(o[j].y);
                yi[4 * i + 2] = to_out<OutT>(o[j].z); yi[4 * i + 3] = to_out<OutT>(o[j].w);
            }
        }
    }
    __syncthreads();
    const float count = (float)(ntok - first_patch);
    const float *part = reinterpret_cast<const float *>(s_part);
    for (int c = threadIdx.x; c < D; c += POOL_WARPS * 32)
    {
        float s = part[c];
#pragma unroll
        for (int k = 1; k < POOL_WARPS; ++k) s = __fadd_rn(s, part[k * D + c]);
        yi[cls * D + c] = to_out<OutT>(__fdiv_rn(s, count));
    }
}

// ------------------------------------------------------------------------------------------------
// Text towers (vitb200_create_text): the token rows of sequence b are x[b N + t][:] = f32(tok[ids[b][t]][:]) + pos[t][:], tok the f16
// token table [V][D].  A sequence holding an id outside [0, V) gets NaN in every one of its rows and the table is not read for it, so
// no batch mate changes.  One CTA per (position, sequence): it first checks the sequence's N ids, then writes its row 4 columns per
// thread.  D % 4 == 0.
constexpr int TOKEN_EMBED_THREADS = 128;

__global__ void __launch_bounds__(TOKEN_EMBED_THREADS)
token_embed_kernel(const int32_t *__restrict__ ids, const __half *__restrict__ tok, const float *__restrict__ pos, float *__restrict__ x,
                   int N, int D, int V)
{
    const int t = blockIdx.x, b = blockIdx.y;
    const int32_t *seq = ids + (size_t)b * N;
    int bad = 0;
    for (int i = threadIdx.x; i < N; i += TOKEN_EMBED_THREADS) bad |= seq[i] < 0 || seq[i] >= V;
    bad = __syncthreads_or(bad);
    const int id = seq[t];
    float4 *xr = reinterpret_cast<float4 *>(x + ((size_t)b * N + t) * D);
    const float4 *pr = reinterpret_cast<const float4 *>(pos + (size_t)t * D);
    const uint2 *tr = reinterpret_cast<const uint2 *>(tok + (size_t)(bad ? 0 : id) * D);
    for (int c = threadIdx.x; c < D / 4; c += TOKEN_EMBED_THREADS)
    {
        if (bad) { xr[c] = make_float4(NAN, NAN, NAN, NAN); continue; }
        const uint2 u = __ldg(tr + c);
        const float4 p = __ldg(pr + c);
        const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&u.x)), e = __half22float2(*reinterpret_cast<const __half2 *>(&u.y));
        xr[c] = make_float4(__fadd_rn(a.x, p.x), __fadd_rn(a.y, p.y), __fadd_rn(e.x, p.z), __fadd_rn(e.y, p.w));
    }
}

// Text towers: one warp per sequence picks the pooled row of its N ids and writes it through the final LayerNorm (layernorm_row_regs)
// as the head's f16 A operand y [B][D].  pool 0: the first position whose id is eos, row 0 when there is none;
// 1: the first position of the largest id; 2: row N - 1 (vitb200_text_arch.pool).  Ties go to the first position, as torch's argmax.
constexpr int TEXT_POOL_WARPS = 4;

template <int MAXV>
__global__ void __launch_bounds__(TEXT_POOL_WARPS * 32)
text_pool_kernel(const float *__restrict__ x, const int32_t *__restrict__ ids, int B, int N, int pool, int eos, const float *__restrict__ w,
                 const float *__restrict__ b, __half *__restrict__ y, int D, float eps)
{
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();
    const int seq = blockIdx.x * TEXT_POOL_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (seq >= B) return;
    const int32_t *s = ids + (size_t)seq * N;
    // (key, position) of this lane's best candidate; a smaller key wins, then the smaller position
    constexpr long long kNone = 0x7fffffffffffffffll;
    long long best = kNone;
    for (int t = lane; t < N; t += 32)
    {
        const long long pos = t;
        if (pool == 0 && s[t] == eos) best = min(best, pos);
        else if (pool == 1) best = min(best, ((0x7fffffffll - max(s[t], 0)) << 32) | pos); // the largest id first
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    const int row = pool == 2 ? N - 1 : best == kNone ? 0 : (int)(best & 0xffffffffll);
    float4 o[MAXV];
    layernorm_row_regs<MAXV, true>(x + ((size_t)seq * N + row) * D, w, b, D, eps, lane, o);
    __half *yr = y + (size_t)seq * D;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
    {
        const int i = lane + 32 * j;
        if (i < (D >> 2)) reinterpret_cast<uint2 *>(yr)[i] = pack4<__half>(o[j]);
    }
}

// ------------------------------------------------------------------------------------------------
// SigLIP's attention-pooling head (vitb200_arch.pool = 2), its attention: per (image, head), one query q_h (f32 [HD], the learned probe
// projected once at load) against the image's P key rows, o = sum_j softmax_j(q_h . k_j / sqrt(HD)) v_j, f32 throughout, max subtracted.
// HD = 64: k and v are the head-major planes the k | v GEMM writes ([2 H planes][plane_rows][64] f16: planes 0 .. H-1 keys, H .. 2H-1
// values), and the scale is the exact 1 / 8.  HD = 72 (So400m): the row-major [rows][2 D] buffer the k | v GEMM writes for that head dim,
// head h's k at column 72 h and its v at D + 72 h (plane_rows is not read), scale f32(1 / sqrtf(72)).  Only rows 0 .. P-1 of the image
// are read, so nothing of another image reaches a sum.  o -> f16 at column HD h of out [B][D] (merged heads).
// HBM-bound (2 x 2 HD B per key, no reuse): 16-byte loads, eight lanes per key row, APOOL_CHUNK keys per CTA pass.  Lane seg of a key
// row holds its columns 8 seg .. 8 seg + 7; at HD = 72 lane 0 also holds the ninth segment, columns 64 .. 71.  The score of key j is
// its lanes' products summed in a fixed butterfly, the output column sums are added chunk row by chunk row in a fixed order, so an image
// gives the same bits alone as in any batch.  Dynamic shared memory: P scores.
constexpr int APOOL_THREADS = 256;
constexpr int APOOL_CHUNK = APOOL_THREADS / 8; // key rows per pass

template <int HD>
__global__ void __launch_bounds__(APOOL_THREADS)
attention_pool_kernel(const __half *__restrict__ kv, size_t plane_rows, const float *__restrict__ q, __half *__restrict__ out, int P, int H)
{
    static_assert(HD == 64 || HD == 72, "head dims 64 (head-major k | v) and 72 (row-major)");
    constexpr bool kTail = HD == 72; // lane 0 of each key row takes the ninth 16-B segment
    extern __shared__ float s_score[]; // [P]
    __shared__ float s_red[APOOL_THREADS / 32];
    __shared__ float s_part[APOOL_CHUNK][HD + 1];
    const int img = blockIdx.x / H, h = blockIdx.x - img * H, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int seg = tid & 7, r0 = tid >> 3; // 16-byte segment (8 columns) of a row; first key row of this thread
    // a key row's stride in 16-B segments, and segment 0 of this head's k and v in key row 0 of the image
    const size_t ld16 = kTail ? (size_t)H * HD / 4 : 8;
    const uint4 *kp, *vp;
    if constexpr (kTail)
    {
        kp = reinterpret_cast<const uint4 *>(kv + (size_t)img * P * 2 * H * HD + (size_t)h * HD);
        vp = kp + (size_t)H * HD / 8;
    }
    else
    {
        kp = reinterpret_cast<const uint4 *>(kv + ((size_t)h * plane_rows + (size_t)img * P) * 64);
        vp = reinterpret_cast<const uint4 *>(kv + ((size_t)(H + h) * plane_rows + (size_t)img * P) * 64);
    }
    const float qscale = kTail ? 1.0f / sqrtf((float)HD) : 0.125f; // 1 / sqrt(64), exact
    float qr[8], qt[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) qr[i] = __ldg(q + HD * h + 8 * seg + i) * qscale;
    if constexpr (kTail)
    {
#pragma unroll
        for (int i = 0; i < 8; ++i) qt[i] = __ldg(q + HD * h + 64 + i) * qscale;
    }
    // scores, and the running maximum of the keys this thread saw
    // (the whole warp takes every pass, so that its shuffles see all 32 lanes; rows past P are neither read nor scored)
    float mx = -INFINITY;
    for (int j0 = 0; j0 < P; j0 += APOOL_CHUNK)
    {
        const int j = j0 + r0;
        const bool live = j < P;
        const uint4 u = live ? __ldg(kp + (size_t)j * ld16 + seg) : make_uint4(0u, 0u, 0u, 0u);
        const __half2 *k2 = reinterpret_cast<const __half2 *>(&u);
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i)
        {
            const float2 f = __half22float2(k2[i]);
            d = fmaf(qr[2 * i], f.x, d);
            d = fmaf(qr[2 * i + 1], f.y, d);
        }
        if constexpr (kTail)
        {
            if (live && seg == 0)
            {
                const uint4 ut = __ldg(kp + (size_t)j * ld16 + 8);
                const __half2 *t2 = reinterpret_cast<const __half2 *>(&ut);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                {
                    const float2 f = __half22float2(t2[i]);
                    d = fmaf(qt[2 * i], f.x, d);
                    d = fmaf(qt[2 * i + 1], f.y, d);
                }
            }
        }
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        d += __shfl_xor_sync(0xffffffffu, d, 2);
        d += __shfl_xor_sync(0xffffffffu, d, 4);
        if (live)
        {
            if (seg == 0) s_score[j] = d;
            mx = fmaxf(mx, d);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_red[warp] = mx;
    __syncthreads(); // also orders the s_score writes before their reads
    mx = s_red[0];
#pragma unroll
    for (int w = 1; w < APOOL_THREADS / 32; ++w) mx = fmaxf(mx, s_red[w]);
    // o = sum_j e_j v_j / sum_j e_j, e_j = exp(s_j - max): this thread's 8 columns over key rows r0, r0 + CHUNK, ...
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, acc_t[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, esum = 0.f;
    for (int j = r0; j < P; j += APOOL_CHUNK)
    {
        const float e = expf(s_score[j] - mx);
        const uint4 u = __ldg(vp + (size_t)j * ld16 + seg);
        const __half2 *v2 = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i)
        {
            const float2 f = __half22float2(v2[i]);
            acc[2 * i] = fmaf(e, f.x, acc[2 * i]);
            acc[2 * i + 1] = fmaf(e, f.y, acc[2 * i + 1]);
        }
        if constexpr (kTail)
        {
            if (seg == 0)
            {
                const uint4 ut = __ldg(vp + (size_t)j * ld16 + 8);
                const __half2 *t2 = reinterpret_cast<const __half2 *>(&ut);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                {
                    const float2 f = __half22float2(t2[i]);
                    acc_t[2 * i] = fmaf(e, f.x, acc_t[2 * i]);
                    acc_t[2 * i + 1] = fmaf(e, f.y, acc_t[2 * i + 1]);
                }
            }
        }
        esum += e;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s_part[r0][8 * seg + i] = acc[i];
    if constexpr (kTail)
    {
        if (seg == 0)
        {
#pragma unroll
            for (int i = 0; i < 8; ++i) s_part[r0][64 + i] = acc_t[i];
        }
    }
    __syncthreads(); // every s_red[w] has been read: it takes the exp sums next
    // the exp sum: each key row's e was added by its 8 segment lanes alike, so lanes with seg == 0 hold the sums
    float es = seg == 0 ? esum : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) es += __shfl_xor_sync(0xffffffffu, es, o);
    if (lane == 0) s_red[warp] = es;
    __syncthreads();
    if (tid < HD)
    {
        float den = s_red[0];
#pragma unroll
        for (int w = 1; w < APOOL_THREADS / 32; ++w) den += s_red[w];
        float o = s_part[0][tid];
        for (int r = 1; r < APOOL_CHUNK; ++r) o += s_part[r][tid];
        out[(size_t)img * H * HD + HD * h + tid] = __float2half_rn(__fdiv_rn(o, den));
    }
}

// ------------------------------------------------------------------------------------------------
// The same LayerNorm for the block LayerNorms (all T rows consecutive, D % 128 == 0, D <= 1024) as a PERSISTENT kernel on bulk copies:
// CTAs (2 per SM) walk 8-row blocks of X (8 D floats = one contiguous run) last block first; warp 8 streams them into a 3-deep
// shared-memory ring with cp.async.bulk + mbarrier, warps 0-7 each normalise one row out of shared memory (w / b kept in registers for
// the whole launch) into a double-buffered staging block that leaves as ONE contiguous bulk store of 8 f16 rows.  Purpose: the
// row-per-warp kernel above reaches 5.9 TB/s alone but 4.8 TB/s inside the step (6 304 short blocks ramping up and draining between two
// persistent GEMMs).  OutT = __nv_fp8_e4m3: the FP8 engine's per-row quantisation; the row scales go straight to y_scale.
constexpr int LN_TMA_ROWS = 8, LN_TMA_STAGES = 3, LN_TMA_THREADS = 288;
__host__ __device__ inline int layernorm_tma_smem_bytes(int D) { return 128 + LN_TMA_STAGES * LN_TMA_ROWS * D * 4 + 2 * LN_TMA_ROWS * D * 2 + 64; }

template <int NV, typename OutT = __half> // float4 per lane = D / 128
__global__ void __launch_bounds__(LN_TMA_THREADS, 2)
layernorm_tma_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ b, OutT *__restrict__ y, int rows, float eps,
                     float *__restrict__ y_scale)
{
    constexpr int D = NV * 128;
    constexpr bool kE4M3 = std::is_same<OutT, __nv_fp8_e4m3>::value;
    extern __shared__ uint8_t ln_smem_raw[];
    const uint32_t base = (ptx::smem_u32(ln_smem_raw) + 127u) & ~127u;
    uint8_t *smem = ln_smem_raw + (base - ptx::smem_u32(ln_smem_raw));
    constexpr uint32_t IN_BYTES = LN_TMA_ROWS * D * 4, OUT_BYTES = LN_TMA_ROWS * D * sizeof(OutT);
    const uint32_t s_in = base, s_out = base + LN_TMA_STAGES * IN_BYTES, bars = s_out + 2 * OUT_BYTES;
    auto full_bar = [&](int st) { return bars + 8u * st; };
    auto empty_bar = [&](int st) { return bars + 8u * (LN_TMA_STAGES + st); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0)
    {
        for (int st = 0; st < LN_TMA_STAGES; ++st) { ptx::mbar_init(full_bar(st), 1); ptx::mbar_init(empty_bar(st), LN_TMA_ROWS); }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    ptx::grid_dep_launch(); // PDL: resident before the producing GEMM has drained
    ptx::grid_dep_wait();
    const int nblk = (rows + LN_TMA_ROWS - 1) / LN_TMA_ROWS;
    if (warp == LN_TMA_ROWS)
    {
        // ---- producer: 8-row blocks, LAST block first (the tail of X is what the L2 still holds)
        if (lane == 0)
        {
            int st = 0;
            uint32_t ph = 0;
            for (int k = blockIdx.x; k < nblk; k += gridDim.x)
            {
                const int row0 = (nblk - 1 - k) * LN_TMA_ROWS;
                const int nr = rows - row0 < LN_TMA_ROWS ? rows - row0 : LN_TMA_ROWS;
                ptx::mbar_wait(empty_bar(st), ph ^ 1);
                ptx::mbar_arrive_expect_tx(full_bar(st), (uint32_t)(nr * D * 4));
                // the input rows are read once (the output is what the next GEMM reads again and again): evict them first
                ptx::bulk_load_1d_hint(s_in + st * IN_BYTES, x + (size_t)row0 * D, (uint32_t)(nr * D * 4), full_bar(st), ptx::L2_EVICT_FIRST);
                if (++st == LN_TMA_STAGES) { st = 0; ph ^= 1; }
            }
        }
    }
    else
    {
        float4 ww[NV], bb[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j)
        {
            ww[j] = __ldg(reinterpret_cast<const float4 *>(w) + lane + 32 * j);
            bb[j] = __ldg(reinterpret_cast<const float4 *>(b) + lane + 32 * j);
        }
        int st = 0, it = 0;
        uint32_t ph = 0;
        for (int k = blockIdx.x; k < nblk; k += gridDim.x, ++it)
        {
            const int row0 = (nblk - 1 - k) * LN_TMA_ROWS;
            const int nr = rows - row0 < LN_TMA_ROWS ? rows - row0 : LN_TMA_ROWS;
            ptx::mbar_wait(full_bar(st), ph);
            float4 v[NV];
            const float4 *xr = reinterpret_cast<const float4 *>(smem + (size_t)st * IN_BYTES + (size_t)warp * D * 4);
            float sum = 0.f;
            if (warp < nr)
            {
#pragma unroll
                for (int j = 0; j < NV; ++j) { v[j] = xr[lane + 32 * j]; sum += sum4(v[j]); }
            }
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(empty_bar(st)); // this row is in registers: the slot may be refilled once all eight have left it
            const float scale = ln_center(v, sum, lane, NV * 32, D, eps);
            // the staging block of two iterations ago must have left shared memory before it is overwritten
            const uint32_t ob = s_out + (uint32_t)(it & 1) * OUT_BYTES;
            if (threadIdx.x == 0) ptx::tma_store_wait_read<1>();
            ptx::named_bar_sync(1, 32 * LN_TMA_ROWS);
            if constexpr (kE4M3)
            {
                if (warp < nr)
                {
                    float amax = 0.f;
#pragma unroll
                    for (int j = 0; j < NV; ++j)
                    {
                        v[j] = ln_affine(v[j], scale, ww[j], bb[j]);
                        amax = fmaxf(amax, abs_max4(v[j]));
                    }
                    amax = warp_max(amax);
                    const float inv = e4m3_multiplier(amax);
                    if (lane == 0) y_scale[row0 + warp] = e4m3_row_scale(amax);
                    uint32_t *yr = reinterpret_cast<uint32_t *>(smem + (ob - base) + (size_t)warp * D);
#pragma unroll
                    for (int j = 0; j < NV; ++j) yr[lane + 32 * j] = e4m3x4(v[j], inv);
                }
            }
            else if (warp < nr)
            {
                uint2 *yr = reinterpret_cast<uint2 *>(smem + (ob - base) + (size_t)warp * D * 2);
#pragma unroll
                for (int j = 0; j < NV; ++j) yr[lane + 32 * j] = pack4<OutT>(ln_affine(v[j], scale, ww[j], bb[j]));
            }
            ptx::fence_proxy_async_smem();
            ptx::named_bar_sync(1, 32 * LN_TMA_ROWS);
            if (threadIdx.x == 0)
            {
                ptx::bulk_store_1d(y + (size_t)row0 * D, ob, (uint32_t)(nr * D * sizeof(OutT)));
                ptx::tma_store_commit();
            }
            if (++st == LN_TMA_STAGES) { st = 0; ph ^= 1; }
        }
        if (threadIdx.x == 0) ptx::tma_store_wait_all();
    }
}

// exp with the reference's f16 table semantics: f16(expf(f32(f16(x))))  (ggml.c:10547-10549, 2200)
__device__ __forceinline__ __half exp_f16_semantics(float x)
{
    const float xr = __half2float(__float2half_rn(x));
    return __float2half_rn(ptx::ex2_approx(xr * 1.4426950408889634f));
}

// ------------------------------------------------------------------------------------------------
// Attention for head dim 64.  Replaces the reference's reshape/permute/CONT nodes + mul_mat(K,Q) + scale + soft_max_inplace +
// mul_mat(V,P) + head merge (reference vit.cpp:826-866; CPU kernels ggml.c:1163-1198 (f32 dot), 10498-10567 (soft-max)).
// qkv: the head-major buffer the qkv GEMM writes, out [T][D] f16.  One CTA per (image, head); K and V of that head live in shared
// memory (XOR-swizzled 16-B chunks); each warp owns 16-query tiles.  Two passes over the keys so the soft-max uses the TRUE row maximum (the f16 rounding of x - max makes online rescaling inexact,
// SURVEY.md H2): pass 1 = row max of QK^T, pass 2 = P = exp(...), l = sum P, O += P V.  Tensor-core work is mma.sync m16n8k16
// (f16 in, f32 acc).  Used beyond 224 tokens; attention_wgmma.cuh covers N <= 224.
// Precision of the split-precision attention (attention_wgmma.cuh): the reference feeds F32 q, k, v to both attention mat-muls
// (vit.cpp:848,858).  The qkv GEMM then leaves every value as TWO f16 numbers, hi = f16(x) and lo = f16(x - hi) (hi + lo carries ~22
// significant bits), and the tensor cores run
//   S = Ql Kh^T + Qh Kl^T + Qh Kh^T   (the Ql Kl^T term is below 2^-22 relative)        O = P Vl + P Vh   (P is exactly f16)
// with f32 accumulation: rounding q, k or v to f16 alone costs ~17 % of the logit-parity budget (DESIGN.md section 4).
constexpr int ATT_KC = 32; // keys per chunk

__device__ __forceinline__ void att_scores(float (&s)[ATT_KC / 8][4], const uint32_t (&qa)[4][4], uint32_t sK, int kc, int lane)
{
#pragma unroll
    for (int nt = 0; nt < ATT_KC / 8; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
    const int mi = lane >> 3, lr = lane & 7;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
    {
#pragma unroll
        for (int ntp = 0; ntp < ATT_KC / 16; ++ntp)
        {
            const int key = kc + (2 * ntp + (mi >> 1)) * 8 + lr;
            const int ch = ks * 2 + (mi & 1);
            uint32_t b0, b1, b2, b3;
            ptx::ldmatrix_x4(sK + key * 128 + ((ch ^ (key & 7)) << 4), b0, b1, b2, b3);
            ptx::mma_m16n8k16_f16(s[2 * ntp], qa[ks], b0, b1);
            ptx::mma_m16n8k16_f16(s[2 * ntp + 1], qa[ks], b2, b3);
        }
    }
}

template <int NWARPS>
__global__ void __launch_bounds__(NWARPS * 32)
attention_kernel(const __half *__restrict__ qkv, size_t plane_rows, __half *__restrict__ out, int N, int D, int H, int Npad, float scale)
// qkv: the head-major buffer the qkv GEMM writes, [3 H planes][plane_rows][64]: q of head h in plane h, k in H + h, v in 2 H + h
{
    extern __shared__ __align__(16) uint8_t att_smem[];
    // launched with programmatic dependent launch: q, k, v are read only once the qkv GEMM has completed
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();
    const int b = blockIdx.x / H, h = blockIdx.x - b * H;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint4 *sK4 = reinterpret_cast<uint4 *>(att_smem);
    uint4 *sV4 = sK4 + Npad * 8;
    const size_t row_stride = 64;
    const __half *base = qkv + ((size_t)h * plane_rows + (size_t)b * N) * 64;       // q rows of this (image, head)
    const size_t k_off = (size_t)H * plane_rows * 64, v_off = 2 * k_off;           // same rows in the k / v planes
    for (int idx = tid; idx < Npad * 8; idx += NWARPS * 32)
    {
        const int t = idx >> 3, c = idx & 7;
        uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
        if (t < N)
        {
            kv = __ldg(reinterpret_cast<const uint4 *>(base + k_off + (size_t)t * row_stride) + c);
            vv = __ldg(reinterpret_cast<const uint4 *>(base + v_off + (size_t)t * row_stride) + c);
        }
        sK4[t * 8 + (c ^ (t & 7))] = kv;
        sV4[t * 8 + (c ^ (t & 7))] = vv;
    }
    __syncthreads();
    const uint32_t sK = ptx::smem_u32(sK4), sV = ptx::smem_u32(sV4);
    const int g = lane >> 2, t4 = lane & 3;
    const int n_qtiles = (N + 15) >> 4;
    for (int qt = warp; qt < n_qtiles; qt += NWARPS)
    {
        const int r0 = qt * 16 + g, r1 = r0 + 8;
        uint32_t qa[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
        {
            const int col = ks * 16 + 2 * t4;
            qa[ks][0] = r0 < N ? __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)r0 * row_stride + col)) : 0u;
            qa[ks][1] = r1 < N ? __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)r1 * row_stride + col)) : 0u;
            qa[ks][2] = r0 < N ? __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)r0 * row_stride + col + 8)) : 0u;
            qa[ks][3] = r1 < N ? __ldg(reinterpret_cast<const uint32_t *>(base + (size_t)r1 * row_stride + col + 8)) : 0u;
        }
        // ---- pass 1: true row maximum (ggml.c:10533-10534)
        float mx0 = -INFINITY, mx1 = -INFINITY;
        for (int kc = 0; kc < Npad; kc += ATT_KC)
        {
            float s[ATT_KC / 8][4];
            att_scores(s, qa, sK, kc, lane);
#pragma unroll
            for (int nt = 0; nt < ATT_KC / 8; ++nt)
            {
                const int key = kc + nt * 8 + 2 * t4;
                if (key < N) { mx0 = fmaxf(mx0, s[nt][0]); mx1 = fmaxf(mx1, s[nt][2]); }
                if (key + 1 < N) { mx0 = fmaxf(mx0, s[nt][1]); mx1 = fmaxf(mx1, s[nt][3]); }
            }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        mx0 *= scale; // ggml_scale_inplace (vit.cpp:851-854): exact for hd = 64 (0.125)
        mx1 *= scale;
        // ---- pass 2: P = f16 exp(f16(s*scale - max)), l = sum P, O += P V
        float o[8][4];
#pragma unroll
        for (int dt = 0; dt < 8; ++dt) { o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f; }
        float l0 = 0.f, l1 = 0.f;
        for (int kc = 0; kc < Npad; kc += ATT_KC)
        {
            float s[ATT_KC / 8][4];
            att_scores(s, qa, sK, kc, lane);
            uint32_t pa[ATT_KC / 16][4];
#pragma unroll
            for (int nt = 0; nt < ATT_KC / 8; ++nt)
            {
                const int key = kc + nt * 8 + 2 * t4;
                const bool v0 = key < N, v1 = key + 1 < N;
                const __half p00 = v0 ? exp_f16_semantics(__fmul_rn(s[nt][0], scale) - mx0) : __float2half_rn(0.f);
                const __half p01 = v1 ? exp_f16_semantics(__fmul_rn(s[nt][1], scale) - mx0) : __float2half_rn(0.f);
                const __half p10 = v0 ? exp_f16_semantics(__fmul_rn(s[nt][2], scale) - mx1) : __float2half_rn(0.f);
                const __half p11 = v1 ? exp_f16_semantics(__fmul_rn(s[nt][3], scale) - mx1) : __float2half_rn(0.f);
                l0 += __half2float(p00) + __half2float(p01);
                l1 += __half2float(p10) + __half2float(p11);
                const __half2 h0 = __halves2half2(p00, p01), h1 = __halves2half2(p10, p11);
                pa[nt >> 1][(nt & 1) * 2 + 0] = *reinterpret_cast<const uint32_t *>(&h0);
                pa[nt >> 1][(nt & 1) * 2 + 1] = *reinterpret_cast<const uint32_t *>(&h1);
            }
            const int mi = lane >> 3, lr = lane & 7;
#pragma unroll
            for (int j = 0; j < ATT_KC / 16; ++j)
            {
#pragma unroll
                for (int dt = 0; dt < 8; dt += 2)
                {
                    const int key = kc + j * 16 + (mi & 1) * 8 + lr;
                    const int ch = dt + (mi >> 1);
                    uint32_t b0, b1, b2, b3;
                    ptx::ldmatrix_x4_trans(sV + key * 128 + ((ch ^ (key & 7)) << 4), b0, b1, b2, b3);
                    ptx::mma_m16n8k16_f16(o[dt], pa[j], b0, b1);
                    ptx::mma_m16n8k16_f16(o[dt + 1], pa[j], b2, b3);
                }
            }
        }
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
        l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1; // p_i = e_i * (1/sum)  (ggml.c:10556-10558)
        __half *o0 = out + ((size_t)b * N + r0) * D + h * 64 + 2 * t4;
        __half *o1 = out + ((size_t)b * N + r1) * D + h * 64 + 2 * t4;
#pragma unroll
        for (int dt = 0; dt < 8; ++dt)
        {
            if (r0 < N) *reinterpret_cast<__half2 *>(o0 + dt * 8) = __floats2half2_rn(o[dt][0] * inv0, o[dt][1] * inv0);
            if (r1 < N) *reinterpret_cast<__half2 *>(o1 + dt * 8) = __floats2half2_rn(o[dt][2] * inv1, o[dt][3] * inv1);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Attention for the row-major head dims HD = 80 (ViT-H/14) and 72 (SigLIP So400m), every token count up to the engine's limit for HD
// (ATT80_MAX_TOKENS, ATT72_MAX_TOKENS).  The soft-max of attention_kernel: two passes, the TRUE row maximum,
// e = f16(exp(f16(s * scale - max))), l = sum e in f32, O = (P V) * (1 / l).  scale = 1 / sqrtf(HD) is not a power of two, but f32
// rounding is monotone, so f32(max(s) * scale) == max(f32(s * scale)) still holds exactly.
// qkv: the row-major [T][3 D] buffer the qkv GEMM writes for these head dims (q | k | v, head h at columns h HD, D + h HD and
// 2 D + h HD), out [T][D] f16.  One CTA per (image, head); it reads only the image's own N rows.  K and V live in shared memory in
// rows of att_row_bytes(HD) whose length in 16-B units is odd, so the 8 row starts of an ldmatrix fall in 8 distinct 16-B bank
// groups: 80 columns take 160 B of data and 16 B of padding (stride 11 x 16 B), 72 columns 144 B and none (stride 9 x 16 B).  Rows
// past N are zero.  S = Q K^T is HD / 16 k16 steps per 8-key tile and, at 72, one k8 step for columns 64..71; O = P V is HD / 8 n8
// tiles, in pairs from ldmatrix_x4_trans and, at 72, a last one from ldmatrix_x2_trans.
// SPLIT (N <= 224, like the wgmma kernel for head dim 64): qkv and qkv_lo hold hi = f16(x) and lo = f16(x - hi) of every value, and
// S = Ql Kh^T + Qh Kl^T + Qh Kh^T, O = P Vl + P Vh (hi and lo of K and V in shared memory).  Otherwise the f16 values of qkv.
constexpr int ATT80_HD = 80, ATT72_HD = 72;
__host__ __device__ constexpr int att_row_bytes(int hd) { return (hd / 8) % 2 ? 2 * hd : 2 * hd + 16; }
constexpr int ATT80_ROW_BYTES = att_row_bytes(ATT80_HD);
static_assert(ATT80_ROW_BYTES == 176 && att_row_bytes(ATT72_HD) == 144);

template <int HD, bool SPLIT>
__device__ __forceinline__ void att_rm_scores(float (&s)[ATT_KC / 8][4], const uint32_t (&qh)[(HD + 15) / 16][4],
                                              const uint32_t (&ql)[(HD + 15) / 16][4], uint32_t sKh, uint32_t sKl, int kc, int lane)
{
    constexpr int KS = HD / 16, ROW = att_row_bytes(HD);
#pragma unroll
    for (int nt = 0; nt < ATT_KC / 8; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
    const int mi = lane >> 3, lr = lane & 7;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
    {
#pragma unroll
        for (int ntp = 0; ntp < ATT_KC / 16; ++ntp)
        {
            const int key = kc + (2 * ntp + (mi >> 1)) * 8 + lr;
            const uint32_t off = (uint32_t)(key * ROW + (ks * 2 + (mi & 1)) * 16);
            uint32_t b0, b1, b2, b3;
            ptx::ldmatrix_x4(sKh + off, b0, b1, b2, b3);
            if constexpr (SPLIT)
            {
                uint32_t c0, c1, c2, c3;
                ptx::ldmatrix_x4(sKl + off, c0, c1, c2, c3);
                ptx::mma_m16n8k16_f16(s[2 * ntp], ql[ks], b0, b1);
                ptx::mma_m16n8k16_f16(s[2 * ntp + 1], ql[ks], b2, b3);
                ptx::mma_m16n8k16_f16(s[2 * ntp], qh[ks], c0, c1);
                ptx::mma_m16n8k16_f16(s[2 * ntp + 1], qh[ks], c2, c3);
            }
            ptx::mma_m16n8k16_f16(s[2 * ntp], qh[ks], b0, b1);
            ptx::mma_m16n8k16_f16(s[2 * ntp + 1], qh[ks], b2, b3);
        }
    }
    if constexpr (HD % 16 == 8)
    {
        // columns HD - 8 .. HD - 1, one k8 step per 8-key tile: lanes 0-7 give the rows of key tile 2 ntp, lanes 8-15 of tile 2 ntp + 1
#pragma unroll
        for (int ntp = 0; ntp < ATT_KC / 16; ++ntp)
        {
            const uint32_t off = (uint32_t)((kc + (2 * ntp + (mi & 1)) * 8 + lr) * ROW + KS * 32);
            uint32_t b0, b1;
            ptx::ldmatrix_x2(sKh + off, b0, b1);
            if constexpr (SPLIT)
            {
                uint32_t c0, c1;
                ptx::ldmatrix_x2(sKl + off, c0, c1);
                ptx::mma_m16n8k8_f16(s[2 * ntp], ql[KS][0], ql[KS][1], b0);
                ptx::mma_m16n8k8_f16(s[2 * ntp + 1], ql[KS][0], ql[KS][1], b1);
                ptx::mma_m16n8k8_f16(s[2 * ntp], qh[KS][0], qh[KS][1], c0);
                ptx::mma_m16n8k8_f16(s[2 * ntp + 1], qh[KS][0], qh[KS][1], c1);
            }
            ptx::mma_m16n8k8_f16(s[2 * ntp], qh[KS][0], qh[KS][1], b0);
            ptx::mma_m16n8k8_f16(s[2 * ntp + 1], qh[KS][0], qh[KS][1], b1);
        }
    }
}

template <int HD, int NWARPS, bool SPLIT>
__global__ void __launch_bounds__(NWARPS * 32)
attention_rowmajor_kernel(const __half *__restrict__ qkv, const __half *__restrict__ qkv_lo, __half *__restrict__ out, int N, int D, int H,
                          int Npad, float scale)
{
    static_assert(HD % 8 == 0 && HD > 64 && HD <= 128, "row-major head dims: whole 16-B segments, more than the 64 of attention_kernel");
    constexpr int ROW = att_row_bytes(HD);
    constexpr int KQ = (HD + 15) / 16; // q fragments per row: HD / 16 k16 steps, and a k8 step for the last 8 columns when HD % 16 == 8
    constexpr int DT = HD / 8;         // n8 tiles of O = P V
    extern __shared__ __align__(16) uint8_t att_rm_smem[];
    // launched with programmatic dependent launch: q, k, v are read only once the qkv GEMM has completed
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();
    const int b = blockIdx.x / H, h = blockIdx.x - b * H;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int kParts = SPLIT ? 2 : 1;
    const size_t ld = 3 * (size_t)D;                                     // row stride of qkv
    const size_t q_off = (size_t)b * N * ld + (size_t)h * HD;            // q of row 0 of this (image, head); k and v D and 2 D further
    const uint32_t part_bytes = (uint32_t)Npad * ROW;
    // [part] K | [part] V, part 0 = hi (or the f16 values), part 1 = lo
    for (int part = 0; part < kParts; ++part)
    {
        const __half *src = (part ? qkv_lo : qkv) + q_off;
        uint8_t *dK = att_rm_smem + part * part_bytes, *dV = att_rm_smem + (kParts + part) * part_bytes;
        for (int idx = tid; idx < Npad * (HD / 8); idx += NWARPS * 32)
        {
            const int t = idx / (HD / 8), c = idx - t * (HD / 8);
            uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
            if (t < N)
            {
                kv = __ldg(reinterpret_cast<const uint4 *>(src + (size_t)t * ld + D) + c);
                vv = __ldg(reinterpret_cast<const uint4 *>(src + (size_t)t * ld + 2 * (size_t)D) + c);
            }
            *reinterpret_cast<uint4 *>(dK + t * ROW + c * 16) = kv;
            *reinterpret_cast<uint4 *>(dV + t * ROW + c * 16) = vv;
        }
    }
    __syncthreads();
    const uint32_t sKh = ptx::smem_u32(att_rm_smem), sKl = sKh + part_bytes;
    const uint32_t sVh = sKh + kParts * part_bytes, sVl = sVh + part_bytes;
    const int g = lane >> 2, t4 = lane & 3;
    const int n_qtiles = (N + 15) >> 4;
    for (int qt = warp; qt < n_qtiles; qt += NWARPS)
    {
        const int r0 = qt * 16 + g, r1 = r0 + 8;
        uint32_t qh[KQ][4], ql[KQ][4];
#pragma unroll
        for (int part = 0; part < kParts; ++part)
        {
            const __half *src = (part ? qkv_lo : qkv) + q_off;
#pragma unroll
            for (int ks = 0; ks < KQ; ++ks)
            {
                const int col = ks * 16 + 2 * t4;
                uint32_t(&qa)[4] = part ? ql[ks] : qh[ks];
                qa[0] = r0 < N ? __ldg(reinterpret_cast<const uint32_t *>(src + (size_t)r0 * ld + col)) : 0u;
                qa[1] = r1 < N ? __ldg(reinterpret_cast<const uint32_t *>(src + (size_t)r1 * ld + col)) : 0u;
                if (ks * 16 + 16 <= HD) // the k8 step reads a[0] and a[1] only
                {
                    qa[2] = r0 < N ? __ldg(reinterpret_cast<const uint32_t *>(src + (size_t)r0 * ld + col + 8)) : 0u;
                    qa[3] = r1 < N ? __ldg(reinterpret_cast<const uint32_t *>(src + (size_t)r1 * ld + col + 8)) : 0u;
                }
            }
        }
        // ---- pass 1: true row maximum of the unscaled scores
        float mx0 = -INFINITY, mx1 = -INFINITY;
        for (int kc = 0; kc < Npad; kc += ATT_KC)
        {
            float s[ATT_KC / 8][4];
            att_rm_scores<HD, SPLIT>(s, qh, ql, sKh, sKl, kc, lane);
#pragma unroll
            for (int nt = 0; nt < ATT_KC / 8; ++nt)
            {
                const int key = kc + nt * 8 + 2 * t4;
                if (key < N) { mx0 = fmaxf(mx0, s[nt][0]); mx1 = fmaxf(mx1, s[nt][2]); }
                if (key + 1 < N) { mx0 = fmaxf(mx0, s[nt][1]); mx1 = fmaxf(mx1, s[nt][3]); }
            }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        mx0 = __fmul_rn(mx0, scale); // == the maximum of the scaled scores (monotone rounding)
        mx1 = __fmul_rn(mx1, scale);
        // ---- pass 2: P = f16 exp(f16(s*scale - max)), l = sum P, O += P V
        float o[DT][4];
#pragma unroll
        for (int dt = 0; dt < DT; ++dt) { o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f; }
        float l0 = 0.f, l1 = 0.f;
        for (int kc = 0; kc < Npad; kc += ATT_KC)
        {
            float s[ATT_KC / 8][4];
            att_rm_scores<HD, SPLIT>(s, qh, ql, sKh, sKl, kc, lane);
            uint32_t pa[ATT_KC / 16][4];
#pragma unroll
            for (int nt = 0; nt < ATT_KC / 8; ++nt)
            {
                const int key = kc + nt * 8 + 2 * t4;
                const bool v0 = key < N, v1 = key + 1 < N;
                const __half p00 = v0 ? exp_f16_semantics(__fmul_rn(s[nt][0], scale) - mx0) : __float2half_rn(0.f);
                const __half p01 = v1 ? exp_f16_semantics(__fmul_rn(s[nt][1], scale) - mx0) : __float2half_rn(0.f);
                const __half p10 = v0 ? exp_f16_semantics(__fmul_rn(s[nt][2], scale) - mx1) : __float2half_rn(0.f);
                const __half p11 = v1 ? exp_f16_semantics(__fmul_rn(s[nt][3], scale) - mx1) : __float2half_rn(0.f);
                l0 += __half2float(p00) + __half2float(p01);
                l1 += __half2float(p10) + __half2float(p11);
                const __half2 h0 = __halves2half2(p00, p01), h1 = __halves2half2(p10, p11);
                pa[nt >> 1][(nt & 1) * 2 + 0] = *reinterpret_cast<const uint32_t *>(&h0);
                pa[nt >> 1][(nt & 1) * 2 + 1] = *reinterpret_cast<const uint32_t *>(&h1);
            }
            const int mi = lane >> 3, lr = lane & 7;
#pragma unroll
            for (int j = 0; j < ATT_KC / 16; ++j)
            {
#pragma unroll
                for (int dt = 0; dt + 1 < DT; dt += 2)
                {
                    const int key = kc + j * 16 + (mi & 1) * 8 + lr;
                    const uint32_t off = (uint32_t)(key * ROW + (dt + (mi >> 1)) * 16);
                    uint32_t b0, b1, b2, b3;
                    if constexpr (SPLIT)
                    {
                        ptx::ldmatrix_x4_trans(sVl + off, b0, b1, b2, b3);
                        ptx::mma_m16n8k16_f16(o[dt], pa[j], b0, b1);
                        ptx::mma_m16n8k16_f16(o[dt + 1], pa[j], b2, b3);
                    }
                    ptx::ldmatrix_x4_trans(sVh + off, b0, b1, b2, b3);
                    ptx::mma_m16n8k16_f16(o[dt], pa[j], b0, b1);
                    ptx::mma_m16n8k16_f16(o[dt + 1], pa[j], b2, b3);
                }
                if constexpr (DT % 2)
                {
                    // the last n8 tile: its 16 keys as two 8x8 matrices (lanes 0-7 and 8-15 give the row addresses)
                    const int key = kc + j * 16 + (mi & 1) * 8 + lr;
                    const uint32_t off = (uint32_t)(key * ROW + (DT - 1) * 16);
                    uint32_t b0, b1;
                    if constexpr (SPLIT)
                    {
                        ptx::ldmatrix_x2_trans(sVl + off, b0, b1);
                        ptx::mma_m16n8k16_f16(o[DT - 1], pa[j], b0, b1);
                    }
                    ptx::ldmatrix_x2_trans(sVh + off, b0, b1);
                    ptx::mma_m16n8k16_f16(o[DT - 1], pa[j], b0, b1);
                }
            }
        }
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
        l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1; // p_i = e_i * (1/sum)  (ggml.c:10556-10558)
        __half *o0 = out + ((size_t)b * N + r0) * D + h * HD + 2 * t4;
        __half *o1 = out + ((size_t)b * N + r1) * D + h * HD + 2 * t4;
#pragma unroll
        for (int dt = 0; dt < DT; ++dt)
        {
            if (r0 < N) *reinterpret_cast<__half2 *>(o0 + dt * 8) = __floats2half2_rn(o[dt][0] * inv0, o[dt][1] * inv0);
            if (r1 < N) *reinterpret_cast<__half2 *>(o1 + dt * 8) = __floats2half2_rn(o[dt][2] * inv1, o[dt][3] * inv1);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// One CTA per classifier row: probs = softmax(logits) with the reference's f16-exp semantics, then top-k (value descending, index
// ascending on ties) by k rounds of block arg-max.  logits rows have pitch ldl (>= C: the head GEMM pads the class count to a
// multiple of 4), probs rows are dense.  The working copy of the row lives in dynamic shared memory when C floats fit (the
// launcher opts in up to the 227 KB limit), otherwise in `scratch` (global, [rows][C]); entries r >= C of a top-k list (k > C)
// are (-1, 0), and so is every entry of a row whose probabilities are NaN (a NaN logit, or +Inf: Inf - Inf).
// SIGMOID (the zero-shot head's mode 1, SigLIP): probs = 1 / (1 + exp(-x)) per class, evaluated in f64 as exp(x) / (1 + exp(x)) below 0
// so that small probabilities keep their relative precision, and the top-k ranks the LOGITS (the probability rounds to 1.0f above about
// 17, which would tie distinct classes) and reports the probability of each; a NaN logit is never ranked, so a NaN row gives (-1, 0).
template <bool SIGMOID>
__global__ void softmax_topk_kernel(const float *__restrict__ logits, int ldl, float *__restrict__ probs, int32_t *__restrict__ topk_idx,
                                    float *__restrict__ topk_val, int C, int k, float *__restrict__ scratch)
{
    extern __shared__ float sp_smem[];
    __shared__ float red_v[32];
    __shared__ int red_i[32];
    const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    float *sp = scratch ? scratch + (size_t)img * C : sp_smem;
    const float *lg = logits + (size_t)img * ldl;
    // in f64, rounded once to f32: within 2^-24 relative of the exact sigmoid of the f32 logit (expf's 2 ulp would not be)
    auto sigmoid = [](float x) {
        const double e = exp(-fabs((double)x));
        return (float)((x >= 0.f ? 1.0 : e) / (1.0 + e));
    };
    if constexpr (SIGMOID)
    {
        for (int i = tid; i < C; i += blockDim.x)
        {
            const float v = lg[i];
            sp[i] = v;
            if (probs) probs[(size_t)img * C + i] = sigmoid(v);
        }
    }
    else
    {
        float mx = -INFINITY;
        for (int i = tid; i < C; i += blockDim.x) { const float v = lg[i]; sp[i] = v; mx = fmaxf(mx, v); }
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) red_v[warp] = mx;
        __syncthreads();
        mx = red_v[0];
        for (int w = 1; w < nw; ++w) mx = fmaxf(mx, red_v[w]);
        __syncthreads();
        float sum = 0.f;
        for (int i = tid; i < C; i += blockDim.x)
        {
            const float e = __half2float(exp_f16_semantics(sp[i] - mx));
            sp[i] = e;
            sum += e;
        }
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) red_v[warp] = sum;
        __syncthreads();
        sum = 0.f;
        for (int w = 0; w < nw; ++w) sum += red_v[w];
        const float inv = 1.0f / sum;
        __syncthreads();
        for (int i = tid; i < C; i += blockDim.x)
        {
            const float pr = __fmul_rn(sp[i], inv);
            sp[i] = pr;
            if (probs) probs[(size_t)img * C + i] = pr;
        }
    }
    __syncthreads();
    // probabilities are >= 0 and a taken entry becomes -2; logits may be -Inf, so the sigmoid form starts below every logit and marks a
    // taken entry NaN
    constexpr float kNone = SIGMOID ? -INFINITY : -1.f;
    for (int r = 0; r < k; ++r)
    {
        if (r >= C) // fewer classes than requested entries
        {
            if (tid == 0)
            {
                if (topk_idx) topk_idx[(size_t)img * k + r] = -1;
                if (topk_val) topk_val[(size_t)img * k + r] = 0.f;
            }
            continue;
        }
        float bv = kNone;
        int bi = 0x7fffffff;
        for (int i = tid; i < C; i += blockDim.x)
        {
            const float v = sp[i];
            if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
        }
        for (int o = 16; o > 0; o >>= 1)
        {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
        __syncthreads();
        if (tid == 0)
        {
            for (int w = 1; w < nw; ++w)
                if (red_v[w] > bv || (red_v[w] == bv && red_i[w] < bi)) { bv = red_v[w]; bi = red_i[w]; }
            if (bi == 0x7fffffff) { bi = -1; bv = 0.f; } // nothing compares >= the floor: a NaN row
            else if constexpr (SIGMOID) bv = sigmoid(bv);
            if (topk_idx) topk_idx[(size_t)img * k + r] = bi;
            if (topk_val) topk_val[(size_t)img * k + r] = bv;
            if (bi >= 0 && bi < C) sp[bi] = SIGMOID ? __int_as_float(0x7fffffff) : -2.f;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// The zero-shot head (vitb200_set_zero_shot): out[r][c] = s * (x_r . t_c) / ||x_r|| + b for the R head rows x (pitch ldx, E columns) and
// the C unit rows of the class matrix t [C][E] (dense); out rows have pitch ldo.  One CTA per ZS_TILE rows x ZS_TILE classes, 256 threads
// of 4 x 4 outputs, operands staged through shared memory ZS_BK columns at a time.  Each dot product is one thread's f32 FFMA chain over
// k = 0 .. E-1 in order, and ||x_r|| is a lane-strided sum of squares with a fixed xor tree, so a row's scores depend on that row alone:
// not on its batch mates, its position in the grid or the batch size.  A NaN or Inf in x_r (or a zero x_r) gives a NaN row.
constexpr int ZS_TILE = 64, ZS_BK = 16, ZS_THREADS = 256;
__global__ void __launch_bounds__(ZS_THREADS)
zero_shot_kernel(const float *__restrict__ x, int ldx, const float *__restrict__ t, float *__restrict__ out, int ldo, int R, int E, int C, float s,
                 float b)
{
    // [k][row] and [k][class]; rows of ZS_TILE + 4 keep the 16-byte reads aligned and spread the transposing stores over the banks
    __shared__ __align__(16) float sx[ZS_BK][ZS_TILE + 4], st[ZS_BK][ZS_TILE + 4];
    __shared__ float nrm[ZS_TILE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tx = tid & 15, ty = tid >> 4;
    const int r0 = blockIdx.x * ZS_TILE, c0 = blockIdx.y * ZS_TILE;
    for (int i = warp; i < ZS_TILE; i += ZS_THREADS / 32)
    {
        float ss = 0.f;
        if (r0 + i < R)
            for (int k = lane; k < E; k += 32) { const float v = x[(size_t)(r0 + i) * ldx + k]; ss = fmaf(v, v, ss); }
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        if (lane == 0) nrm[i] = sqrtf(ss);
    }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < E; k0 += ZS_BK)
    {
        for (int i = tid; i < ZS_TILE * ZS_BK; i += ZS_THREADS)
        {
            const int kk = i % ZS_BK, rr = i / ZS_BK, k = k0 + kk;
            sx[kk][rr] = (r0 + rr < R && k < E) ? x[(size_t)(r0 + rr) * ldx + k] : 0.f;
            st[kk][rr] = (c0 + rr < C && k < E) ? t[(size_t)(c0 + rr) * E + k] : 0.f;
        }
        __syncthreads();
        // past E both operands are 0: fmaf(0, 0, acc) leaves acc as it is
#pragma unroll
        for (int kk = 0; kk < ZS_BK; ++kk)
        {
            const float4 a = *reinterpret_cast<const float4 *>(&sx[kk][ty * 4]);
            const float4 w = *reinterpret_cast<const float4 *>(&st[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        const int r = r0 + ty * 4 + i;
        if (r >= R) continue;
        const float n = nrm[ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j)
        {
            const int c = c0 + tx * 4 + j;
            if (c < C) out[(size_t)r * ldo + c] = fmaf(s, __fdiv_rn(acc[i][j], n), b);
        }
    }
}

} // namespace vitb200
