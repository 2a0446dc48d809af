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
//                   into a kStages-deep shared-memory ring; the other warps load the tile's bias into shared memory once and, for
//                   the residual epilogue, prefetch the tile's residual rows into L2; its registers are handed to the MMA
//                   warpgroups (setmaxnreg)
//   warpgroups 1-2  MMA + epilogue: each owns 64 rows of the tile and issues 4 x wgmma.m64nBNk16 per k-block with the f32 accumulator
//                   in registers, then applies bias / GELU / hi-lo split / residual / position embedding on those registers
// Pipeline: per ring slot a full mbarrier (TMA transaction bytes) and an empty mbarrier (one arrival per MMA warpgroup once the
// wgmma reading the slot has retired).
// Staged epilogue (qkv, proj, fc1, fc2): once both MMA warpgroups' wgmmas have retired the operand ring is free; each warpgroup
// writes its 64 result rows into it as 64-row x 128-B boxes (SWIZZLE_128B, so the fragment-layout writes are free of bank
// conflicts) and one thread stores them with TMA.  The residual epilogue first TMA-loads its residual rows into the same boxes and
// adds them there.  The store maps cover exactly M rows and N columns, so rows >= M and columns >= N are not written.  The patch
// and head epilogues store straight from registers.
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
    void *out;          // f16 or f32, row-major, leading dimension ldo (16-B aligned rows for the staged epilogues)
    void *out2;         // EPI_BIAS_F16_HILO: the lo halves, same shape as out
    int ldo;
    int headmajor;      // f16 epilogues: 1 = the output is HEAD-MAJOR, [N / 64 planes][plane_rows][64]: every head's q / k / v slice is one
                        // contiguous run of rows, which is what the attention kernel reads (qkv; DESIGN.md section 2)
    size_t plane_rows;  // headmajor: rows per plane
    const float *resid; // EPI_BIAS_RESID_F32: [M][ldo] (may alias out)
    const float *pos;   // EPI_PATCH_F32: pos_embed [ntok][N]
    int np, ntok;       // EPI_PATCH_F32: patches / tokens per image
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

template <int BN>
__device__ __forceinline__ void wgmma_k16(float (&acc)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    if constexpr (BN == 256) ptx::wgmma_m64n256k16_f16(acc, adesc, bdesc, accumulate);
    else ptx::wgmma_m64n128k16_f16(acc, adesc, bdesc, accumulate);
}

// Epilogues whose result goes out through shared memory and TMA stores (the rest store from registers)
__host__ __device__ constexpr bool gemm_epi_staged(int epi)
{
    return epi == EPI_BIAS_F16 || epi == EPI_BIAS_GELU_F16 || epi == EPI_BIAS_F16_HILO || epi == EPI_BIAS_RESID_F32;
}

// Staged-epilogue geometry: each MMA warpgroup's 64 x BN result leaves as boxes of 64 rows x 128 B (64 f16 or 32 f32 columns),
// one box set per output tensor (hi and lo for EPI_BIAS_F16_HILO), in the operand ring it no longer needs
template <int BN, int EPI>
struct GemmStage
{
    static constexpr bool kF16 = (EPI == EPI_BIAS_F16 || EPI == EPI_BIAS_GELU_F16 || EPI == EPI_BIAS_F16_HILO);
    static constexpr int kBoxCols = kF16 ? 64 : 32;
    static constexpr int kBoxes = BN / kBoxCols;   // boxes per output tensor and warpgroup
    static constexpr int kBoxBytes = 64 * 128;
    static constexpr int kOuts = EPI == EPI_BIAS_F16_HILO ? 2 : 1;
    static constexpr int kWgBytes = kOuts * kBoxes * kBoxBytes;
    static_assert(2 * kWgBytes <= GemmCfg<BN>::kStages * (GemmCfg<BN>::A_BYTES + GemmCfg<BN>::B_BYTES), "staged tile exceeds the ring");
};

// tmOut: the store map of out (f16: box 64 columns x 64 rows, 2-D [M][N] or, head-major, 3-D {64, M, N / 64 planes}; f32: box
// 32 columns x 64 rows over [M][N]), SWIZZLE_128B.  tmAux: the same map over out2 (EPI_BIAS_F16_HILO) or the load map of resid
// (EPI_BIAS_RESID_F32).  Both unused by the register epilogues.
template <int BN, int EPI>
__global__ void __launch_bounds__(384, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                  const __grid_constant__ CUtensorMap tmAux, const GemmParams p)
{
    static_assert(BN == 128 || BN == 256, "BN");
    using Cfg = GemmCfg<BN>;
    constexpr int kStages = Cfg::kStages;
    constexpr bool kStaged = gemm_epi_staged(EPI);

    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(16) float s_bias[BN]; // the tile's bias, zero past N
    const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u; // SWIZZLE_128B wants 1024-B aligned tiles
    const uint32_t sA = smem_base;
    const uint32_t sB = sA + kStages * Cfg::A_BYTES;
    const uint32_t bars = sB + kStages * Cfg::B_BYTES;
    auto full_bar = [&](int s) { return bars + 8u * s; };
    auto empty_bar = [&](int s) { return bars + 8u * (kStages + s); };
    const uint32_t bias_bar = bars + 8u * (2 * kStages);
    auto resid_bar = [&](int cw) { return bars + 8u * (2 * kStages + 1 + cw); };

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int n_tiles = (p.N + BN - 1) / BN;
    const int m_blk = blockIdx.x / n_tiles, n_blk = blockIdx.x - m_blk * n_tiles;
    const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;
    const int m0 = m_blk * GEMM_BM, n0 = n_blk * BN;

    if (threadIdx.x == 0)
    {
        ptx::prefetch_tensormap(&tmA);
        ptx::prefetch_tensormap(&tmB);
        if constexpr (kStaged)
        {
            ptx::prefetch_tensormap(&tmOut);
            if constexpr (EPI == EPI_BIAS_F16_HILO || EPI == EPI_BIAS_RESID_F32) ptx::prefetch_tensormap(&tmAux);
        }
        for (int s = 0; s < kStages; ++s)
        {
            ptx::mbar_init(full_bar(s), 1);
            ptx::mbar_init(empty_bar(s), 2); // one arrival per MMA warpgroup
        }
        ptx::mbar_init(bias_bar, 96); // producer warps 1-3
        ptx::mbar_init(resid_bar(0), 1);
        ptx::mbar_init(resid_bar(1), 1);
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
            for (int kb = 0; kb < num_kb; ++kb)
            {
                const int s = kb % kStages;
                ptx::mbar_wait(empty_bar(s), ((kb / kStages) & 1) ^ 1);
                // out-of-range rows / columns are zero-filled and still count their bytes
                ptx::mbar_arrive_expect_tx(full_bar(s), Cfg::A_BYTES + Cfg::B_BYTES);
                ptx::tma_load_2d(sA + s * Cfg::A_BYTES, &tmA, full_bar(s), kb * GEMM_BK, m0);
                ptx::tma_load_2d(sB + s * Cfg::B_BYTES, &tmB, full_bar(s), kb * GEMM_BK, n0);
            }
        }
        else if (tid >= 32)
        {
            if constexpr (EPI == EPI_BIAS_RESID_F32)
            {
                // the residual rows are read once, by the epilogue: start pulling them into L2 while the main loop runs
                if (tid == 32)
                    for (int h = 0; h < 2; ++h)
                        if (m0 + 64 * h < p.M)
                            for (int c = n0; c < min(n0 + BN, p.N); c += 32) ptx::tma_prefetch_2d(&tmAux, c, m0 + 64 * h);
            }
            for (int c = tid - 32; c < BN; c += 96) s_bias[c] = n0 + c < p.N ? __ldg(p.bias + n0 + c) : 0.f;
            ptx::mbar_arrive(bias_bar);
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
    ptx::mbar_wait(bias_bar, 0);

    // wgmma m64nN layout: thread (warp w, lane l) holds rows 16 w + l / 4 (+ 8) and, per 8-column group j, columns 8 j + 2 (l % 4) (+ 1)
    const int warp = tid >> 5, lane = tid & 31;
    if constexpr (kStaged)
    {
        // ===================== staged epilogue: registers -> swizzled boxes in the free ring -> TMA stores =====================
        using St = GemmStage<BN, EPI>;
        const int wm0 = m0 + cw * 64;                                                  // first row of this warpgroup
        const bool live = wm0 < p.M;                                                   // any of its rows inside M
        const int nbox = min(St::kBoxes, (p.N - n0 + St::kBoxCols - 1) / St::kBoxCols); // boxes that start inside N
        const uint32_t stage = smem_base + cw * St::kWgBytes;
        ptx::named_bar_sync(1, 256); // both warpgroups' wgmmas have retired: nothing reads the ring any more
        if constexpr (EPI == EPI_BIAS_RESID_F32)
        {
            if (live)
            {
                if (tid == 0)
                {
                    ptx::mbar_arrive_expect_tx(resid_bar(cw), nbox * St::kBoxBytes); // partial boxes count in full (zero fill)
                    for (int b = 0; b < nbox; ++b) ptx::tma_load_2d(stage + b * St::kBoxBytes, &tmAux, resid_bar(cw), n0 + 32 * b, wm0);
                }
                ptx::mbar_wait(resid_bar(cw), 0);
            }
        }
        // row r of a box lives at r * 128 B with its 16-B chunks permuted by chunk ^ (r % 8); r % 8 == lane / 4 for every row here
        const int rr = warp * 16 + (lane >> 2), sw = lane >> 2, q = lane & 3;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
        {
            const float2 b = *reinterpret_cast<const float2 *>(&s_bias[8 * j + 2 * q]);
#pragma unroll
            for (int h = 0; h < 2; ++h)
            {
                const uint32_t row = stage + (uint32_t)(rr + 8 * h) * 128u;
                const float x0 = __fadd_rn(acc[4 * j + 2 * h], b.x), x1 = __fadd_rn(acc[4 * j + 2 * h + 1], b.y);
                if constexpr (St::kF16)
                {
                    const uint32_t a = row + (j / 8) * St::kBoxBytes + (((j % 8) ^ sw) << 4) + 4 * q;
                    __half2 hv;
                    if constexpr (EPI == EPI_BIAS_GELU_F16)
                    {
                        const float2 r = __half22float2(__floats2half2_rn(x0, x1)); // ggml.c:1434-1441: y = f16(gelu(f32(f16(x))))
                        hv = __floats2half2_rn(gelu_tanh_f32(r.x), gelu_tanh_f32(r.y));
                    }
                    else hv = __floats2half2_rn(x0, x1);
                    ptx::st_shared_b32(a, *reinterpret_cast<const uint32_t *>(&hv));
                    if constexpr (EPI == EPI_BIAS_F16_HILO)
                    {
                        const float2 hf = __half22float2(hv); // lo = f16(x - hi): exact difference, |lo| <= 2^-11 |x|
                        const __half2 lo = __floats2half2_rn(__fsub_rn(x0, hf.x), __fsub_rn(x1, hf.y));
                        ptx::st_shared_b32(a + St::kBoxes * St::kBoxBytes, *reinterpret_cast<const uint32_t *>(&lo));
                    }
                }
                else
                {
                    const uint32_t a = row + (j / 4) * St::kBoxBytes + (((2 * (j % 4) + (q >> 1)) ^ sw) << 4) + 8 * (q & 1);
                    if constexpr (EPI == EPI_BIAS_RESID_F32)
                    {
                        const float2 r = ptx::ld_shared_v2_f32(a); // (mul_mat + b) + inpL, vit.cpp:869,873
                        ptx::st_shared_v2_f32(a, __fadd_rn(x0, r.x), __fadd_rn(x1, r.y));
                    }
                    else ptx::st_shared_v2_f32(a, x0, x1);
                }
            }
        }
        ptx::fence_proxy_async_smem(); // the writes above are seen by the TMA engine
        ptx::named_bar_sync(2 + cw, 128);
        if (tid == 0 && live)
        {
            for (int b = 0; b < nbox; ++b)
            {
                const uint32_t src = stage + b * St::kBoxBytes;
                if constexpr (St::kF16)
                {
                    if (p.headmajor)
                    {
                        const int plane = (n0 >> 6) + b;
                        ptx::tma_store_3d(&tmOut, src, 0, wm0, plane);
                        if constexpr (EPI == EPI_BIAS_F16_HILO) ptx::tma_store_3d(&tmAux, src + St::kBoxes * St::kBoxBytes, 0, wm0, plane);
                    }
                    else
                    {
                        ptx::tma_store_2d(&tmOut, src, n0 + 64 * b, wm0);
                        if constexpr (EPI == EPI_BIAS_F16_HILO) ptx::tma_store_2d(&tmAux, src + St::kBoxes * St::kBoxBytes, n0 + 64 * b, wm0);
                    }
                }
                else ptx::tma_store_2d(&tmOut, src, n0 + 32 * b, wm0);
            }
            ptx::tma_store_commit();
            ptx::tma_store_wait_read<0>(); // the shared memory must outlive the reads of the stores
        }
    }
    else
    {
        // ===================== register epilogue (patch embedding, head) =====================
        const int row0 = m0 + cw * 64 + warp * 16 + (lane >> 2);
        const int col0 = n0 + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
        {
            const int col = col0 + 8 * j;
            if (col >= p.N) continue; // N % 4 == 0: a column pair is all-in or all-out
            const float2 b = *reinterpret_cast<const float2 *>(&s_bias[col - n0]);
#pragma unroll
            for (int h = 0; h < 2; ++h)
            {
                const int row = row0 + 8 * h;
                if (row >= p.M) continue;
                const float x0 = __fadd_rn(acc[4 * j + 2 * h], b.x), x1 = __fadd_rn(acc[4 * j + 2 * h + 1], b.y);
                if constexpr (EPI == EPI_PATCH_F32)
                {
                    const int img = row / p.np, pp = row - img * p.np;
                    const float2 pe = __ldg(reinterpret_cast<const float2 *>(p.pos + (size_t)(1 + pp) * p.N + col));
                    *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out) + ((size_t)img * p.ntok + 1 + pp) * p.ldo + col) =
                        make_float2(__fadd_rn(x0, pe.x), __fadd_rn(x1, pe.y));
                }
                else *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out) + (size_t)row * p.ldo + col) = make_float2(x0, x1);
            }
        }
    }
}

} // namespace vitb200
