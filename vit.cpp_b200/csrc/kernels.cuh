// kernels.cuh -- the non-GEMM kernels of the forward path (all HBM-bound except attention):
//   patchify_f16_kernel      reference im2col for stride==kernel conv (ggml.c:11528-11608) without the buffer
//                            reshuffle: pixels HWC f32 -> f16 patch rows, K order c*P*P + ky*P + kx
//   cls_rows_kernel          token 0 = cls_token + pos_embed[0]                      (vit.cpp:794-797)
//   layernorm_f16_kernel     ggml_norm * w + b (ggml.c:8959-9008, vit.cpp:808-812) emitting the f16 A operand
//   attention_kernel         per (image, head): S = QK^T / sqrt(hd), softmax with the reference's f16-exp
//                            semantics (ggml.c:10536-10558), O = P V   (vit.cpp:826-866)
//   softmax_topk_kernel      final soft-max (vit.cpp:931) + top-k (replaces the host std::sort, vit.cpp:1047-1057)
#pragma once
#include "ptx.cuh"

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

// x[b*ntok + 0][:] = cls[:] + pos[0][:]
__global__ void cls_rows_kernel(float *__restrict__ x, const float *__restrict__ cls, const float *__restrict__ pos, int B, int ntok, int D)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * D) return;
    const int b = i / D, o = i - b * D;
    x[(size_t)b * ntok * D + o] = __fadd_rn(cls[o], pos[o]);
}

// ------------------------------------------------------------------------------------------------
// One warp per row.  mean / biased variance in f32 (the reference sums in double; the difference is
// ~1e-7 relative), then y = ((x-mean)*scale)*w + b as three separately rounded f32 ops like the
// reference's NORM, MUL, ADD nodes, then RNE to f16 (the GEMM's src1 conversion, ggml.c:9493-9506).
template <int MAXV>
__global__ void layernorm_f16_kernel(const float *__restrict__ x, size_t x_row_stride, int rows_per_group, size_t group_stride,
                                     const float *__restrict__ w, const float *__restrict__ b, __half *__restrict__ y, int rows,
                                     int D, float eps)
{
    ptx::grid_dep_launch(); // PDL: blocks may be resident before the producing GEMM has drained
    ptx::grid_dep_wait();
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
            sum += (v[j].x + v[j].y) + (v[j].z + v[j].w);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)D;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
    {
        const int i = lane + 32 * j;
        if (i < nvec)
        {
            v[j].x -= mean; v[j].y -= mean; v[j].z -= mean; v[j].w -= mean;
            sq += (v[j].x * v[j].x + v[j].y * v[j].y) + (v[j].z * v[j].z + v[j].w * v[j].w);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float var = sq / (float)D;
    const float scale = 1.0f / sqrtf(var + eps);
    const float4 *w4 = reinterpret_cast<const float4 *>(w);
    const float4 *b4 = reinterpret_cast<const float4 *>(b);
    uint2 *yr = reinterpret_cast<uint2 *>(y + (size_t)row * D);
#pragma unroll
    for (int j = 0; j < MAXV; ++j)
    {
        const int i = lane + 32 * j;
        if (i < nvec)
        {
            const float4 ww = __ldg(w4 + i), bb = __ldg(b4 + i);
            const float o0 = __fadd_rn(__fmul_rn(__fmul_rn(v[j].x, scale), ww.x), bb.x);
            const float o1 = __fadd_rn(__fmul_rn(__fmul_rn(v[j].y, scale), ww.y), bb.y);
            const float o2 = __fadd_rn(__fmul_rn(__fmul_rn(v[j].z, scale), ww.z), bb.z);
            const float o3 = __fadd_rn(__fmul_rn(__fmul_rn(v[j].w, scale), ww.w), bb.w);
            const __half2 h0 = __floats2half2_rn(o0, o1), h1 = __floats2half2_rn(o2, o3);
            uint2 u;
            u.x = *reinterpret_cast<const uint32_t *>(&h0);
            u.y = *reinterpret_cast<const uint32_t *>(&h1);
            yr[i] = u;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// The same LayerNorm for the block LayerNorms (all T rows consecutive, D % 128 == 0, D <= 1024) as a PERSISTENT kernel on bulk copies:
// CTAs (2 per SM) walk 8-row blocks of X (8 D floats = one contiguous run) last block first; warp 8 streams them into a 3-deep
// shared-memory ring with cp.async.bulk + mbarrier, warps 0-7 each normalise one row out of shared memory (identical arithmetic to the
// kernel above, w / b kept in registers for the whole launch) into a double-buffered staging block that leaves as ONE contiguous
// bulk store of 8 f16 rows.  Purpose: the row-per-warp kernel above reaches 5.9 TB/s alone but 4.8 TB/s inside the step (6 304 short
// blocks ramping up and draining between two persistent GEMMs).
constexpr int LN_TMA_ROWS = 8, LN_TMA_STAGES = 3, LN_TMA_THREADS = 288;
__host__ __device__ inline int layernorm_tma_smem_bytes(int D) { return 128 + LN_TMA_STAGES * LN_TMA_ROWS * D * 4 + 2 * LN_TMA_ROWS * D * 2 + 64; }

template <int NV> // float4 per lane = D / 128
__global__ void __launch_bounds__(LN_TMA_THREADS, 2)
layernorm_tma_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ b, __half *__restrict__ y, int rows, float eps,
                     unsigned long long load_policy, unsigned long long store_policy) // L2 eviction hints of the bulk copies (0 = none)
{
    constexpr int D = NV * 128;
    extern __shared__ uint8_t ln_smem_raw[];
    const uint32_t base = (ptx::smem_u32(ln_smem_raw) + 127u) & ~127u;
    uint8_t *smem = ln_smem_raw + (base - ptx::smem_u32(ln_smem_raw));
    constexpr uint32_t IN_BYTES = LN_TMA_ROWS * D * 4, OUT_BYTES = LN_TMA_ROWS * D * 2;
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
                if (load_policy) ptx::bulk_load_1d_hint(s_in + st * IN_BYTES, x + (size_t)row0 * D, (uint32_t)(nr * D * 4), full_bar(st), load_policy);
                else ptx::bulk_load_1d(s_in + st * IN_BYTES, x + (size_t)row0 * D, (uint32_t)(nr * D * 4), full_bar(st));
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
                for (int j = 0; j < NV; ++j) { v[j] = xr[lane + 32 * j]; sum += (v[j].x + v[j].y) + (v[j].z + v[j].w); }
            }
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(empty_bar(st)); // this row is in registers: the slot may be refilled once all eight have left it
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            const float mean = sum / (float)D;
            float sq = 0.f;
#pragma unroll
            for (int j = 0; j < NV; ++j)
            {
                v[j].x -= mean; v[j].y -= mean; v[j].z -= mean; v[j].w -= mean;
                sq += (v[j].x * v[j].x + v[j].y * v[j].y) + (v[j].z * v[j].z + v[j].w * v[j].w);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
            const float scale = 1.0f / sqrtf(sq / (float)D + eps);
            // the staging block of two iterations ago must have left shared memory before it is overwritten
            const uint32_t ob = s_out + (uint32_t)(it & 1) * OUT_BYTES;
            if (threadIdx.x == 0) ptx::tma_store_wait_read<1>();
            ptx::named_bar_sync(1, 32 * LN_TMA_ROWS);
            if (warp < nr)
            {
                uint2 *yr = reinterpret_cast<uint2 *>(smem + (ob - base) + (size_t)warp * D * 2);
#pragma unroll
                for (int j = 0; j < NV; ++j)
                {
                    const __half2 h0 = __floats2half2_rn(__fadd_rn(__fmul_rn(__fmul_rn(v[j].x, scale), ww[j].x), bb[j].x), __fadd_rn(__fmul_rn(__fmul_rn(v[j].y, scale), ww[j].y), bb[j].y));
                    const __half2 h1 = __floats2half2_rn(__fadd_rn(__fmul_rn(__fmul_rn(v[j].z, scale), ww[j].z), bb[j].z), __fadd_rn(__fmul_rn(__fmul_rn(v[j].w, scale), ww[j].w), bb[j].w));
                    uint2 u;
                    u.x = *reinterpret_cast<const uint32_t *>(&h0);
                    u.y = *reinterpret_cast<const uint32_t *>(&h1);
                    yr[lane + 32 * j] = u;
                }
            }
            ptx::fence_proxy_async_smem();
            ptx::named_bar_sync(1, 32 * LN_TMA_ROWS);
            if (threadIdx.x == 0)
            {
                if (store_policy) ptx::bulk_store_1d_hint(y + (size_t)row0 * D, ob, (uint32_t)(nr * D * 2), store_policy);
                else ptx::bulk_store_1d(y + (size_t)row0 * D, ob, (uint32_t)(nr * D * 2));
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
// One CTA per classifier row: probs = softmax(logits) with the reference's f16-exp semantics, then top-k (value descending, index
// ascending on ties) by k rounds of block arg-max.  logits rows have pitch ldl (>= C: the head GEMM pads the class count to a
// multiple of 4), probs rows are dense.  The working copy of the row lives in dynamic shared memory when C floats fit (the
// launcher opts in up to the 227 KB limit), otherwise in `scratch` (global, [rows][C]); entries r >= C of a top-k list (k > C)
// are (-1, 0).
__global__ void softmax_topk_kernel(const float *__restrict__ logits, int ldl, float *__restrict__ probs, int32_t *__restrict__ topk_idx,
                                    float *__restrict__ topk_val, int C, int k, float *__restrict__ scratch)
{
    extern __shared__ float sp_smem[];
    __shared__ float red_v[32];
    __shared__ int red_i[32];
    const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    float *sp = scratch ? scratch + (size_t)img * C : sp_smem;
    const float *lg = logits + (size_t)img * ldl;
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
    __syncthreads();
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
        float bv = -1.f;
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
            if (topk_idx) topk_idx[(size_t)img * k + r] = bi;
            if (topk_val) topk_val[(size_t)img * k + r] = bv;
            if (bi >= 0 && bi < C) sp[bi] = -2.f;
        }
        __syncthreads();
    }
}

} // namespace vitb200
