// gemm_wgmma.cuh -- the linear-layer kernel: C[M,N] = A[M,K] * W[N,K]^T with a fused epilogue.
//
// Replaces ggml_mul_mat + ggml_add_inplace (+ ggml_gelu) (+ residual ggml_add) of the reference graph
// (reference vit.cpp:820-821, 868-873, 889-900, 927-928, and the conv GEMM of vit.cpp:772-797) and the CPU
// kernel behind them (ggml.c:9388-9597 with ggml_vec_dot_f16, ggml.c:1200-1236).
// Numerics follow the reference recipe: A = activations already rounded to f16 (RNE, ggml.c:9493-9506),
// W = the f16 weights as stored in the model file (ne0 = K contiguous, vit.cpp:531-543), fp32 accumulation.
//
// Structure (sm_90a): one CTA per 128 x BN tile of C, three warpgroups:
//   warpgroup 0     TMA producer: one thread streams the 128 x 64 A tile and the BN x 64 W tile of every k-block (SWIZZLE_128B)
//                   into a kStages-deep shared-memory ring; its registers are handed to the MMA warpgroups (setmaxnreg)
//   warpgroups 1-2  MMA + epilogue: each owns 64 rows of the tile and issues 4 x wgmma.m64nBNk16 per k-block with the f32 accumulator
//                   in registers, then applies bias / GELU / hi-lo split / residual / position embedding on those registers and
//                   stores straight to global memory (rows >= M and columns >= N are not written)
// Pipeline: per ring slot a full mbarrier (TMA transaction bytes) and an empty mbarrier (one arrival per MMA warpgroup once the
// wgmma reading the slot has retired).
#pragma once
#include "ptx.cuh"

namespace vitb200 {

enum GemmEpilogue
{
    EPI_BIAS_F16 = 0,       // out f16 = f16(acc + bias)                              (qkv)
    EPI_BIAS_GELU_F16 = 1,  // out f16 = f16(gelu_tanh(f32(f16(acc + bias))))           (fc1; ggml.c:1418-1441)
    EPI_BIAS_RESID_F32 = 2, // out f32 = (acc + bias) + resid                         (proj, fc2; vit.cpp:873,900)
    EPI_PATCH_F32 = 3,      // out f32[token row] = (acc + bias) + pos_embed           (patch embed; vit.cpp:773-797)
    EPI_BIAS_F32 = 4,       // out f32 = acc + bias                                   (head logits)
    EPI_BIAS_F16_HILO = 6,  // x = acc + bias kept to ~22 significant bits as TWO f16 tensors: out = hi = f16(x), out2 = lo = f16(x - hi)
                            // (qkv in front of the split-precision attention: the reference feeds f32 q, k, v to both attention mat-muls,
                            // vit.cpp:848,858; hi + lo lets the f16 tensor cores reproduce that with split-precision MMAs)
};

struct GemmParams
{
    int M, N, K;        // valid extents (rows of A / rows of W / reduction); N % 4 == 0
    const float *bias;  // [N]
    void *out;          // f16 or f32, row-major, leading dimension ldo
    void *out2;         // EPI_BIAS_F16_HILO: the lo halves, same shape as out
    int ldo;
    int headmajor;      // f16 epilogues: 1 = the output is HEAD-MAJOR, [N / 64 planes][plane_rows][64]: every head's q / k / v slice is one
                        // contiguous run of rows, which is what the attention kernel reads (qkv; DESIGN.md section 2)
    size_t plane_rows;  // headmajor: rows per plane
    const float *resid; // EPI_BIAS_RESID_F32: [M][ldo] (may alias out)
    const float *pos;   // EPI_PATCH_F32: pos_embed [ntok][N]
    int np, ntok;       // EPI_PATCH_F32: patches / tokens per image
    // EPI_BIAS_RESID_F32 with a fused LayerNorm (N == hidden size, N % 128 == 0, N <= 1024): the LayerNorm that follows the residual add
    // (vit.cpp:881-885 after proj, vit.cpp:808-812 of the next block after fc2) is applied to a 128-row M tile by the CTA that stores the
    // last of its column tiles (ln_count: one counter per M tile, zero on entry and left zero), while the rows are still in L2; ln_out
    // receives the f16 rows [M][N].  NULL = no fusion.
    __half *ln_out;
    const float *ln_w, *ln_b;
    int *ln_count;
    float ln_eps;
};

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;

template <int BN>
struct GemmCfg
{
    static constexpr int kThreads = 384;                 // producer warpgroup + two MMA warpgroups
    static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
    static constexpr int B_BYTES = BN * GEMM_BK * 2;
    static constexpr int kSmemLimit = 232448;            // 227 KB per CTA
    static constexpr int kStagesFit = (kSmemLimit - 1024 - 256) / (A_BYTES + B_BYTES);
    static constexpr int kStages = kStagesFit > 6 ? 6 : kStagesFit; // operand ring depth: whatever fits, at most 6
    static constexpr int SMEM_BYTES = 1024 /*align slack*/ + kStages * (A_BYTES + B_BYTES) + 256 /*barriers*/;
    static_assert(SMEM_BYTES <= kSmemLimit, "exceeds the 227 KB per-CTA shared memory limit");
};

// GELU, tanh form (the reference's formula, ggml.c:1418-1424) on an f16-valued input, evaluated in f32 as
//   0.5 x (1 + tanh(u)) = x / (1 + e^{-2u}),   u = sqrt(2/pi) x (1 + 0.044715 x^2)
// (algebraically identical; 5 FMA-pipe ops + MUFU.EX2 + MUFU.RCP, relative error ~3e-7, i.e. the f16 rounding the caller
// applies next (table semantics, ggml.c:2197) differs from the host table in well under 0.1 % of inputs, by one ulp).
__device__ __forceinline__ float gelu_tanh_f32(float x)
{
    // -2u log2(e) = x (k0 + k1 x^2), k0 = -2 sqrt(2/pi) log2(e), k1 = 0.044715 k0: FMUL, FFMA, FMUL, EX2, FADD, RCP, FMUL
    const float w = fmaf(x * x, -0.10294323958083856f, -2.3022081981625516f);
    const float e = ptx::ex2_approx(x * w);                      // e^{-2u}
    return x * ptx::rcp_approx(1.0f + e);
}

// One warp normalises one row of X (f32, already complete in L2) into the f16 A operand of the next GEMM: the arithmetic of
// layernorm_f16_kernel (kernels.cuh) -- f32 two-pass mean / biased variance, then ((x - mean) * scale) * w + b as three separately
// rounded operations (the reference's NORM, MUL, ADD nodes, ggml.c:8959-9008, vit.cpp:808-812), RNE to f16 -- with w and b read from
// global memory and the row read past L1 (ld.global.cg: other SMs wrote it).  nv = D / 128 float4 per lane (<= 8).
__device__ __forceinline__ void ln_row_load(const float *xrow, int nv, int lane, float4 (&v)[8])
{
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nv) v[j] = __ldcg(reinterpret_cast<const float4 *>(xrow) + lane + 32 * j);
}
__device__ __forceinline__ void ln_row_finish(float4 (&v)[8], int nv, int D, int lane, const float4 *w4, const float4 *b4, float eps, __half *yrow)
{
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nv) sum += (v[j].x + v[j].y) + (v[j].z + v[j].w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)D;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nv)
        {
            v[j].x -= mean; v[j].y -= mean; v[j].z -= mean; v[j].w -= mean;
            sq += (v[j].x * v[j].x + v[j].y * v[j].y) + (v[j].z * v[j].z + v[j].w * v[j].w);
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float scale = 1.0f / sqrtf(sq / (float)D + eps);
    uint2 *yr = reinterpret_cast<uint2 *>(yrow);
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (j < nv)
        {
            const int i = lane + 32 * j;
            const float4 ww = w4[i], bb = b4[i];
            const __half2 h0 = __floats2half2_rn(__fadd_rn(__fmul_rn(__fmul_rn(v[j].x, scale), ww.x), bb.x), __fadd_rn(__fmul_rn(__fmul_rn(v[j].y, scale), ww.y), bb.y));
            const __half2 h1 = __floats2half2_rn(__fadd_rn(__fmul_rn(__fmul_rn(v[j].z, scale), ww.z), bb.z), __fadd_rn(__fmul_rn(__fmul_rn(v[j].w, scale), ww.w), bb.w));
            uint2 u;
            u.x = *reinterpret_cast<const uint32_t *>(&h0);
            u.y = *reinterpret_cast<const uint32_t *>(&h1);
            yr[i] = u;
        }
}

template <int BN>
__device__ __forceinline__ void wgmma_k16(float (&acc)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    if constexpr (BN == 256) ptx::wgmma_m64n256k16_f16(acc, adesc, bdesc, accumulate);
    else ptx::wgmma_m64n128k16_f16(acc, adesc, bdesc, accumulate);
}

template <int BN, int EPI>
__global__ void __launch_bounds__(384, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p)
{
    static_assert(BN == 128 || BN == 256, "BN");
    using Cfg = GemmCfg<BN>;
    constexpr int kStages = Cfg::kStages;
    constexpr bool kOutF16 = (EPI == EPI_BIAS_F16 || EPI == EPI_BIAS_GELU_F16 || EPI == EPI_BIAS_F16_HILO);

    extern __shared__ uint8_t smem_raw[];
    __shared__ int s_ln_last;
    const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u; // SWIZZLE_128B wants 1024-B aligned tiles
    const uint32_t sA = smem_base;
    const uint32_t sB = sA + kStages * Cfg::A_BYTES;
    const uint32_t bars = sB + kStages * Cfg::B_BYTES;
    auto full_bar = [&](int s) { return bars + 8u * s; };
    auto empty_bar = [&](int s) { return bars + 8u * (kStages + s); };

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int n_tiles = (p.N + BN - 1) / BN;
    const int m_blk = blockIdx.x / n_tiles, n_blk = blockIdx.x - m_blk * n_tiles;
    const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;

    if (threadIdx.x == 0)
    {
        ptx::prefetch_tensormap(&tmA);
        ptx::prefetch_tensormap(&tmB);
        for (int s = 0; s < kStages; ++s)
        {
            ptx::mbar_init(full_bar(s), 1);
            ptx::mbar_init(empty_bar(s), 2); // one arrival per MMA warpgroup
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    // prologue done (it overlapped the previous kernel's tail under PDL); from here on the kernel touches upstream data
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();

    if (wg == 0)
    {
        // ===================== TMA producer =====================
        ptx::setmaxnreg_dec<40>();
        if (tid == 0)
        {
            const int a_row = m_blk * GEMM_BM, b_row = n_blk * BN;
            for (int kb = 0; kb < num_kb; ++kb)
            {
                const int s = kb % kStages;
                ptx::mbar_wait(empty_bar(s), ((kb / kStages) & 1) ^ 1);
                // out-of-range rows / columns are zero-filled and still count their bytes
                ptx::mbar_arrive_expect_tx(full_bar(s), Cfg::A_BYTES + Cfg::B_BYTES);
                ptx::tma_load_2d(sA + s * Cfg::A_BYTES, &tmA, full_bar(s), kb * GEMM_BK, a_row);
                ptx::tma_load_2d(sB + s * Cfg::B_BYTES, &tmB, full_bar(s), kb * GEMM_BK, b_row);
            }
        }
        return;
    }

    // ===================== MMA warpgroups =====================
    ptx::setmaxnreg_inc<232>();
    const int cw = wg - 1; // rows 64 cw .. 64 cw + 63 of the tile
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb)
    {
        const int s = kb % kStages;
        ptx::mbar_wait(full_bar(s), (kb / kStages) & 1);
        const uint64_t adesc = ptx::wgmma_desc_kmajor_sw128(sA + s * Cfg::A_BYTES + cw * 64 * 128);
        const uint64_t bdesc = ptx::wgmma_desc_kmajor_sw128(sB + s * Cfg::B_BYTES);
        ptx::fence_regs(acc);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_k16<BN>(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0); // +32 B along K
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>(); // the previous k-block's MMAs have retired: its slot can be refilled
        ptx::fence_regs(acc);
        if (kb > 0 && tid == 0) ptx::mbar_arrive(empty_bar((kb - 1) % kStages));
    }
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);

    // ===================== epilogue, straight from the accumulator registers =====================
    // wgmma m64nN layout: thread (warp w, lane l) holds rows 16 w + l / 4 (+ 8) and, per 8-column group j, columns 8 j + 2 (l % 4) (+ 1)
    const int warp = tid >> 5, lane = tid & 31;
    const int row0 = m_blk * GEMM_BM + cw * 64 + warp * 16 + (lane >> 2);
    const int col0 = n_blk * BN + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
    {
        const int col = col0 + 8 * j;
        if (col >= p.N) continue; // N % 4 == 0: a column pair is all-in or all-out
        const float2 b = __ldg(reinterpret_cast<const float2 *>(p.bias + col));
#pragma unroll
        for (int h = 0; h < 2; ++h)
        {
            const int row = row0 + 8 * h;
            if (row >= p.M) continue;
            const float x0 = __fadd_rn(acc[4 * j + 2 * h], b.x), x1 = __fadd_rn(acc[4 * j + 2 * h + 1], b.y);
            if constexpr (kOutF16)
            {
                const size_t off = p.headmajor ? ((size_t)(col >> 6) * p.plane_rows + (size_t)row) * 64 + (col & 63) : (size_t)row * p.ldo + col;
                __half2 hv;
                if constexpr (EPI == EPI_BIAS_GELU_F16)
                {
                    const float2 r = __half22float2(__floats2half2_rn(x0, x1)); // ggml.c:1434-1441: y = f16(gelu(f32(f16(x))))
                    hv = __floats2half2_rn(gelu_tanh_f32(r.x), gelu_tanh_f32(r.y));
                }
                else hv = __floats2half2_rn(x0, x1);
                *reinterpret_cast<__half2 *>(reinterpret_cast<__half *>(p.out) + off) = hv;
                if constexpr (EPI == EPI_BIAS_F16_HILO)
                {
                    const float2 hf = __half22float2(hv); // lo = f16(x - hi): exact difference, |lo| <= 2^-11 |x|
                    *reinterpret_cast<__half2 *>(reinterpret_cast<__half *>(p.out2) + off) = __floats2half2_rn(__fsub_rn(x0, hf.x), __fsub_rn(x1, hf.y));
                }
            }
            else if constexpr (EPI == EPI_PATCH_F32)
            {
                const int img = row / p.np, pp = row - img * p.np;
                const float2 pe = __ldg(reinterpret_cast<const float2 *>(p.pos + (size_t)(1 + pp) * p.N + col));
                *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out) + ((size_t)img * p.ntok + 1 + pp) * p.ldo + col) =
                    make_float2(__fadd_rn(x0, pe.x), __fadd_rn(x1, pe.y));
            }
            else
            {
                float *o = reinterpret_cast<float *>(p.out) + (size_t)row * p.ldo + col;
                if constexpr (EPI == EPI_BIAS_RESID_F32)
                {
                    const float2 r = *reinterpret_cast<const float2 *>(p.resid + (size_t)row * p.ldo + col); // (mul_mat + b) + inpL, vit.cpp:869,873
                    *reinterpret_cast<float2 *>(o) = make_float2(__fadd_rn(x0, r.x), __fadd_rn(x1, r.y));
                }
                else *reinterpret_cast<float2 *>(o) = make_float2(x0, x1);
            }
        }
    }

    if constexpr (EPI == EPI_BIAS_RESID_F32)
    {
        if (p.ln_out != nullptr)
        {
            // fused LayerNorm: the CTA that completes the last column tile of this M tile normalises its rows
            __threadfence(); // this thread's stores are visible GPU-wide before the counter moves
            ptx::named_bar_sync(1, 256);
            if (threadIdx.x == 128)
            {
                const int last = atomicAdd(p.ln_count + m_blk, 1) == n_tiles - 1;
                if (last) p.ln_count[m_blk] = 0;
                s_ln_last = last;
            }
            ptx::named_bar_sync(1, 256);
            if (s_ln_last)
            {
                __threadfence();
                const float *X = reinterpret_cast<const float *>(p.out);
                const float4 *w4 = reinterpret_cast<const float4 *>(p.ln_w), *b4 = reinterpret_cast<const float4 *>(p.ln_b);
                const int rows = min(GEMM_BM, p.M - m_blk * GEMM_BM), nv = p.N >> 7;
                for (int r = (threadIdx.x - 128) >> 5; r < rows; r += 8)
                {
                    const size_t grow = (size_t)m_blk * GEMM_BM + r;
                    float4 v[8];
                    ln_row_load(X + grow * p.ldo, nv, lane, v);
                    ln_row_finish(v, nv, p.N, lane, w4, b4, p.ln_eps, p.ln_out + grow * p.N);
                }
            }
        }
    }
}

} // namespace vitb200
