// gemm_wgmma.cuh -- the linear-layer kernel: C[M,N] = A[M,K] * W[N,K]^T with a fused epilogue.
//
// Replaces ggml_mul_mat + ggml_add_inplace (+ ggml_gelu) (+ residual ggml_add) of the reference graph
// (reference vit.cpp:820-821, 868-873, 889-900, 927-928, and the conv GEMM of vit.cpp:772-797) and the CPU
// kernel behind them (ggml.c:9388-9597 with ggml_vec_dot_f16, ggml.c:1200-1236).
// Numerics follow the reference recipe: A = activations already rounded to f16 (RNE, ggml.c:9493-9506),
// W = the f16 weights as stored in the model file (ne0 = K contiguous, vit.cpp:531-543), fp32 accumulation.
//
// Structure (sm_90a): a persistent grid of as many two-CTA clusters as fit at once.  C is cut into 128 x 128 tiles; two
// neighbouring column tiles form a pair, pairs are numbered with N fastest within an M band, and cluster c takes pairs c,
// c + clusters, ..., CTA r of the cluster the column tile 2 j + r of each (a tile past N when the count is odd is computed and never
// stored).  The two CTAs share the pair's A tile: each loads half of it into both with a TMA multicast, so a k-block moves 24 KB from
// L2 per CTA instead of 32 KB (the 128 x 128 tile alone made the main loop L2-bandwidth bound).  Each CTA hands its tiles
// alternately to its two MMA warpgroups (ping-pong):
//   warpgroup 0     TMA producer: one thread streams the A half and the 128 x 64 W tile of every k-block of every tile of the CTA, in
//                   the order the MMA warpgroups consume them, into a ring of 32 KB stages (SWIZZLE_128B); for the residual
//                   epilogue it also prefetches each tile's residual rows into L2 when it starts the tile; before exiting it waits
//                   until both CTAs have released every slot; its registers are handed to the MMA warpgroups (setmaxnreg)
//   warpgroups 1-2  MMA + epilogue: each owns a whole tile at a time and issues 2 x wgmma.m64n128k16 (rows 0-63 and 64-127) per k16
//                   step with the 128 f32 accumulators per thread in registers, then applies bias / GELU / hi-lo split / residual /
//                   position embedding to them
// Pipeline: per ring slot a full mbarrier (TMA transaction bytes, both A halves and the W tile) and an empty mbarrier (two arrivals:
// the warpgroup that consumed the slot, in this CTA and in the peer, once the wgmma reading it has retired; the peer's multicast
// writes into the slot too).  Slots and their phases run on across tile boundaries, so the ring does not drain between tiles.  The
// two warpgroups' main loops take turns on the tensor cores through a pair of named barriers: a warpgroup starts tile i's k-loop
// once the other one has issued tile i-1's, and runs tile i's epilogue while the other runs tile i+1's k-loop.
// Ring depth (template STAGES, chosen by K on the host): 6 stages with 16 KB staging buffers for K >= GEMM_DEEP_K, whose main loop
// dominates and needs the deeper ring to hide its load latency; 5 stages with 32 KB buffers otherwise, where the epilogue's share
// is larger and fewer, larger passes shorten it.
// Operand format (template OP): f16 x f16, or e4m3 x e4m3 for the FP8 engine's qkv and fc1.  A 128-B swizzled row holds 64 f16 or
// 128 e4m3 values, so an e4m3 k-block is 128 elements with the same stage bytes, TMA boxes and multicast; each k-block issues
// 4 x 2 wgmma.m64n128k32.e4m3 instead of 4 x 2 m64n128k16.f16.  The e4m3 operands carry one scale per A row (token) and one for
// all of W, so C[m][n] = a_scale[m] w_scale sum_k qa[m][k] qw[n][k]: the main loop is a plain f32-accumulated MMA and the scale is one
// multiply in the epilogue, x = acc (a_scale[m] w_scale), after which the epilogue runs unchanged on x.
// Staged epilogue (qkv, proj, fc1, fc2): each MMA warpgroup has its own staging buffer outside the ring.  The tile leaves in passes
// of one 64-row half x 64 or 128 columns: the warpgroup writes a pass as 64-row x 128-B boxes (SWIZZLE_128B, so the fragment-layout
// writes are free of bank conflicts) and one thread stores them with TMA.  A pass reuses buffer space only once the stores of the
// pass that used it have read it.  The residual epilogue first TMA-loads the pass's residual rows into the same boxes and adds them
// there; the first pass's residual is loaded at tile start, under the k-loop.  The store maps cover exactly M rows and N columns,
// so rows >= M and columns >= N are not written; a tile reads and writes only its own rows and columns, so the residual may alias
// the output.  The patch and head epilogues store straight from registers.
#pragma once
#include "ptx.cuh"

namespace vitb200 {

enum GemmOperand
{
    GEMM_OP_F16 = 0,  // A and W f16, k-block of 64
    GEMM_OP_E4M3 = 1, // A and W e4m3 with a per-row A scale and a per-tensor W scale (GemmParams), k-block of 128
};

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
    EPI_BIAS_GELU_ERF_F16 = 7,   // out f16 = f16(gelu_erf(acc + bias)), x in f32 without rounding to f16 first   (fc1 of LAION CLIP)
    EPI_BIAS_QUICK_GELU_F16 = 8, // out f16 = f16(quick_gelu(acc + bias)), likewise                               (fc1 of OpenAI CLIP)
    EPI_BIAS_SCALE_RESID_F32 = 9, // out f32 = f32((acc + bias) * gamma[n]) + resid: LayerScale, HF's order    (proj, fc2 of DINOv2)
    EPI_BIAS_GELU_PYTORCH_TANH_F16 = 10, // out f16 = f16(gelu_tanh(acc + bias)), x in f32 without rounding to f16 first (fc1 of SigLIP)
    EPI_BIAS_SWIGLU_F16 = 11, // out f16 [M][F] = f16(silu(x1) * x2), x = acc + bias in f32, W interleaved by 64 (fc1 of DINOv2 ViT-g; below)
};
constexpr int GEMM_EPI_END = EPI_BIAS_SWIGLU_F16 + 1; // one past the largest id: a new epilogue takes this id and moves it on

// What each epilogue is: the kernel, its launch and dispatch and the test hooks derive every per-epilogue choice from this.  staged:
// stored through shared memory with TMA (else from registers); f16 output (else f32); resid: adds the TMA-loaded residual stream; hilo:
// outputs hi and lo; swiglu: W interleaved by SWIGLU_GROUP, F of the N columns stored; e4m3: has an e4m3-operand form.  5: valid = false.
struct GemmEpiDesc { bool valid, staged, f16, resid, hilo, swiglu, e4m3; };
__host__ __device__ constexpr GemmEpiDesc gemm_epi(int epi)
{
    switch (epi) //                                valid  staged f16    resid  hilo   swiglu e4m3
    {
    case EPI_BIAS_F16:                   return {true, true,  true,  false, false, false, true};
    case EPI_BIAS_GELU_F16:              return {true, true,  true,  false, false, false, true};
    case EPI_BIAS_RESID_F32:             return {true, true,  false, true,  false, false, false};
    case EPI_PATCH_F32:                  return {true, false, false, false, false, false, false};
    case EPI_BIAS_F32:                   return {true, false, false, false, false, false, false};
    case EPI_BIAS_F16_HILO:              return {true, true,  true,  false, true,  false, true};
    case EPI_BIAS_GELU_ERF_F16:          return {true, true,  true,  false, false, false, true};
    case EPI_BIAS_QUICK_GELU_F16:        return {true, true,  true,  false, false, false, true};
    case EPI_BIAS_SCALE_RESID_F32:       return {true, true,  false, true,  false, false, false};
    case EPI_BIAS_GELU_PYTORCH_TANH_F16: return {true, true,  true,  false, false, false, true};
    case EPI_BIAS_SWIGLU_F16:            return {true, true,  true,  false, false, true,  true};
    default:                             return {};
    }
}

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
    const float *a_scale; // GEMM_OP_E4M3: [M] f32, the scale of each A row
    float w_scale;        // GEMM_OP_E4M3: the scale of W
    const float *gamma;   // EPI_BIAS_SCALE_RESID_F32: [N] f32, the LayerScale of each output column
    int F;                // EPI_BIAS_SWIGLU_F16: the columns of out; N = 2 round_up(F, 64)
};

constexpr int GEMM_BM = 128; // rows of a tile
constexpr int GEMM_BN = 128; // columns of a tile (the W map's box rows)
constexpr int GEMM_A_BOX_ROWS = GEMM_BM / 2; // the A map's box: each CTA of a cluster pair loads half of the A tile they share
constexpr int GEMM_BK = 64; // f16 elements of a k-block (128 B per row); e4m3 k-blocks hold twice as many

// Shared memory holds six 32 KB ring stages and two 16 KB staging buffers, or five stages and two 32 KB buffers.  A long reduction
// (K >= GEMM_DEEP_K) is main-loop bound and wants the deeper ring to hide the L2 latency of its loads; a short one spends a larger
// share in the epilogue, which wants the larger buffer (fewer store / residual round trips per tile).
constexpr int GEMM_DEEP_K = 2048;

template <int STAGES>
struct GemmCfg
{
    static_assert(STAGES == 5 || STAGES == 6, "ring depth");
    static constexpr int kThreads = 384;                 // producer warpgroup + two MMA warpgroups
    static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
    static constexpr int B_BYTES = GEMM_BN * GEMM_BK * 2;
    static constexpr int kStages = STAGES;               // operand ring depth
    static constexpr int kStageBytes = STAGES == 6 ? 16384 : 32768; // epilogue staging buffer per MMA warpgroup
    static constexpr int kSmemLimit = 232448;            // 227 KB per CTA
    static constexpr int SMEM_BYTES = 1024 /*align slack*/ + kStages * (A_BYTES + B_BYTES) + 2 * kStageBytes + 256 /*barriers*/;
    static_assert(SMEM_BYTES + 2 * GEMM_BN * 4 /*s_bias*/ <= kSmemLimit, "exceeds the 227 KB per-CTA shared memory limit");
    static_assert(STAGES != 6 || SMEM_BYTES + 2 * GEMM_BN * 4 + 2 * 64 * 4 /*s_bias, s_gamma*/ <= kSmemLimit, "LayerScale: exceeds 227 KB");
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

// GELU, erf form: 0.5 x (1 + erf(x / sqrt 2)) = x Phi(x), evaluated as x * normcdff(x).  normcdff is erfc-based, so the left tail keeps
// its relative accuracy where 1 + erf(x / sqrt 2) would cancel; for x << 0 it underflows to 0 and the result is -0.
__device__ __forceinline__ float gelu_erf_f32(float x) { return x * normcdff(x); }

// QuickGELU (OpenAI CLIP): x sigma(1.702 x) = x / (1 + e^{-1.702 x}).  For x << 0, e^{-1.702 x} is +inf, its reciprocal 0 and the
// result -0; never NaN for a finite x.
__device__ __forceinline__ float quick_gelu_f32(float x)
{
    const float e = ptx::ex2_approx(x * -2.4554670f); // -1.702 log2(e)
    return x * ptx::rcp_approx(1.0f + e);
}

// SiLU, SwiGLU's gate: x sigma(x) = x / (1 + e^{-x}), in the form of quick_gelu_f32.  For x << 0, e^{-x} is +inf, its reciprocal 0 and
// the result -0; never NaN for a finite x.
__device__ __forceinline__ float silu_f32(float x)
{
    const float e = ptx::ex2_approx(x * -1.4426950408889634f); // -log2(e)
    return x * ptx::rcp_approx(1.0f + e);
}

// SwiGLU (EPI_BIAS_SWIGLU_F16).  HF's fc1 is [2 F][K]: rows 0 .. F-1 give x1, rows F .. 2F-1 its partners x2, h = silu(x1) x2.  The
// weights and the bias are interleaved at upload in groups of 64 hidden units (swiglu_interleave in engine.cu): rows 128 g .. 128 g + 63
// are x1 rows 64 g .., rows 128 g + 64 .. 128 g + 127 the matching x2 rows, rows past F zero, so the GEMM runs with N = 2 round_up(F, 64).
// Each 128-column tile then holds, in the same thread, x1 in its 8-column groups j < 8 and the partner x2 in group j + 8; a pass (one
// 64-row half) stores one 64-column f16 box at column n0 / 2 of out [M][F], and the store map covers F columns, so padding is never stored.
constexpr int SWIGLU_GROUP = 64;

// Staged-epilogue geometry: a warpgroup's 128 x 128 result leaves in passes of one 64-row half x kPassCols columns; a pass is
// kColBoxes boxes of 64 rows x 128 B (64 f16 or 32 f32 columns) per output tensor (hi and lo for EPI_BIAS_F16_HILO) and fills the
// staging buffer
template <int EPI, int STAGES>
struct GemmStage
{
    using Cfg = GemmCfg<STAGES>;
    static constexpr bool kF16 = gemm_epi(EPI).f16;
    static constexpr bool kSwiglu = gemm_epi(EPI).swiglu;
    static constexpr int kOuts = gemm_epi(EPI).hilo ? 2 : 1;
    static constexpr int kBoxCols = kF16 ? 64 : 32;
    static constexpr int kBoxBytes = 64 * 128;
    static constexpr int kFitCols = Cfg::kStageBytes / (64 * kOuts * (kF16 ? 2 : 4));
    static constexpr int kPassCols = kFitCols < GEMM_BN ? kFitCols : GEMM_BN; // 16 KB: 128 (f16), 64 (hi + lo, f32); 32 KB: 128
    static_assert(!kSwiglu || kPassCols == GEMM_BN, "SwiGLU: a pass holds both halves of its 64 outputs");
    static constexpr int kStoreCols = kSwiglu ? kPassCols / 2 : kPassCols; // output columns a pass stores
    static constexpr int kColGroups = GEMM_BN / kPassCols;
    static constexpr int kPasses = 2 * kColGroups; // row half outer, column group inner
    static constexpr int kColBoxes = kStoreCols / kBoxCols;
    static constexpr int kPassBytes = kOuts * kColBoxes * kBoxBytes;
    static constexpr int kSlots = Cfg::kStageBytes / kPassBytes; // passes the buffer holds at once (2: f16 in 32 KB)
    static_assert(kSlots * kPassBytes == Cfg::kStageBytes, "passes tile the staging buffer");
    // offset of box (output o, column box c) in the staging buffer
    __host__ __device__ static constexpr uint32_t box(int o, int c) { return (uint32_t)((o * kColBoxes + c) * kBoxBytes); }
};

// tmOut: the store map of out (f16: box 64 columns x 64 rows, 2-D [M][N] or, head-major, 3-D {64, M, N / 64 planes}; f32: box
// 32 columns x 64 rows over [M][N]), SWIZZLE_128B.  tmAux: the same map over out2 (EPI_BIAS_F16_HILO) or the load map of resid
// (EPI_BIAS_RESID_F32, EPI_BIAS_SCALE_RESID_F32).  Both unused by the register epilogues.
template <int EPI, int STAGES, int OP = GEMM_OP_F16>
__global__ void __launch_bounds__(384, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                  const __grid_constant__ CUtensorMap tmAux, const GemmParams p)
{
    using Cfg = GemmCfg<STAGES>;
    constexpr int kStages = Cfg::kStages;
    constexpr bool kStaged = gemm_epi(EPI).staged;
    constexpr bool kE4M3 = OP == GEMM_OP_E4M3;
    static_assert(gemm_epi(EPI).valid && (!kE4M3 || (kStaged && gemm_epi(EPI).e4m3)), "an epilogue; e4m3: a staged one with an e4m3 form");
    constexpr int kKb = kE4M3 ? 2 * GEMM_BK : GEMM_BK; // K elements per k-block
    constexpr int kBarTurn = 1; // + warpgroup: named barrier "this warpgroup may start its next k-loop"
    constexpr int kBarWg = 3;   // + warpgroup: the warpgroup's own epilogue barrier

    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(16) float s_bias[2][GEMM_BN]; // per MMA warpgroup: its current tile's bias, zero past N
    const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u; // SWIZZLE_128B wants 1024-B aligned tiles
    const uint32_t sA = smem_base;
    const uint32_t sB = sA + kStages * Cfg::A_BYTES;
    const uint32_t sStage = sB + kStages * Cfg::B_BYTES;
    const uint32_t bars = sStage + 2 * Cfg::kStageBytes;
    auto full_bar = [&](int s) { return bars + 8u * s; };
    auto empty_bar = [&](int s) { return bars + 8u * (kStages + s); };
    auto resid_bar = [&](int cw) { return bars + 8u * (2 * kStages + cw); };
    using St = GemmStage<EPI, STAGES>;
    // residual epilogues: TMA-load the residual of one pass (64 rows from `row`, the column boxes from c0 that start inside N) into
    // the staging buffer `dst` of warpgroup cw, completing on resid_bar(cw); partial boxes are zero-filled and count in full
    auto resid_load = [&](uint32_t dst, int c0, int row, int cw) {
        const int ncb = min(St::kColBoxes, (p.N - c0 + St::kBoxCols - 1) / St::kBoxCols);
        ptx::mbar_arrive_expect_tx(resid_bar(cw), ncb * St::kBoxBytes);
        for (int c = 0; c < ncb; ++c) ptx::tma_load_2d(dst + St::box(0, c), &tmAux, resid_bar(cw), c0 + 32 * c, row);
    };

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    // the two CTAs of a cluster take the two column tiles of a pair (a tile past N when the count is odd: computed, never stored)
    const unsigned rank = ptx::cluster_ctarank();
    const unsigned cluster = blockIdx.x >> 1, clusters = gridDim.x >> 1;
    const unsigned n_pairs = (unsigned)(p.N + 2 * GEMM_BN - 1) / (2 * GEMM_BN);
    // pair u exists (its M band starts inside M); tested against p.M rather than a pair count, which would hold a register
    auto pair_exists = [&](unsigned u) { return (int)(u / n_pairs) * GEMM_BM < p.M; };
    const int num_kb = (p.K + kKb - 1) / kKb;

    if (threadIdx.x == 0)
    {
        ptx::prefetch_tensormap(&tmA);
        ptx::prefetch_tensormap(&tmB);
        if constexpr (kStaged)
        {
            ptx::prefetch_tensormap(&tmOut);
            if constexpr (gemm_epi(EPI).hilo || gemm_epi(EPI).resid) ptx::prefetch_tensormap(&tmAux);
        }
        for (int s = 0; s < kStages; ++s)
        {
            ptx::mbar_init(full_bar(s), 1);
            ptx::mbar_init(empty_bar(s), 2); // the MMA warpgroup that consumed the slot, in this CTA and in the peer
        }
        ptx::mbar_init(resid_bar(0), 1);
        ptx::mbar_init(resid_bar(1), 1);
        ptx::fence_barrier_init();
    }
    ptx::cluster_sync(); // the peer multicasts into this CTA's ring and arrives on its empty barriers
    // prologue done (it overlapped the previous kernel's tail under PDL); from here on the kernel touches upstream data
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();

    if (wg == 0)
    {
        // ===================== TMA producer =====================
        ptx::setmaxnreg_dec<40>();
        if (tid == 0)
        {
            int s = 0;
            uint32_t ph = 0;
            for (unsigned u = cluster; pair_exists(u); u += clusters)
            {
                const unsigned m_blk = u / n_pairs;
                const int m0 = (int)m_blk * GEMM_BM, n0 = (int)(2 * (u - m_blk * n_pairs) + rank) * GEMM_BN;
                if constexpr (gemm_epi(EPI).resid)
                {
                    // the residual rows are read once, by the epilogue: start pulling them into L2 while the tile's main loop runs
                    for (int h = 0; h < 2; ++h)
                        if (m0 + 64 * h < p.M)
                            for (int c = n0; c < min(n0 + GEMM_BN, p.N); c += 32) ptx::tma_prefetch_2d(&tmAux, c, m0 + 64 * h);
                }
                for (int kb = 0; kb < num_kb; ++kb)
                {
                    ptx::mbar_wait(empty_bar(s), ph ^ 1); // free in both CTAs: the A half below lands in both
                    // out-of-range rows / columns are zero-filled and still count their bytes; the A tile is shared by the pair,
                    // each CTA loads 64 of its rows into both CTAs
                    ptx::mbar_arrive_expect_tx(full_bar(s), Cfg::A_BYTES + Cfg::B_BYTES);
                    ptx::tma_load_2d_multicast(sA + s * Cfg::A_BYTES + rank * (Cfg::A_BYTES / 2), &tmA, full_bar(s), kb * kKb,
                                               m0 + rank * GEMM_A_BOX_ROWS, 0x3);
                    ptx::tma_load_2d(sB + s * Cfg::B_BYTES, &tmB, full_bar(s), kb * kKb, n0);
                    if (++s == kStages) { s = 0; ph ^= 1; }
                }
            }
            // every slot released by both CTAs: no arrival from the peer is still on its way when this CTA exits
            for (int k = 0; k < kStages; ++k)
            {
                ptx::mbar_wait(empty_bar(s), ph ^ 1);
                if (++s == kStages) { s = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ===================== MMA warpgroups =====================
    ptx::setmaxnreg_inc<232>();
    const int cw = wg - 1;
    // wgmma m64nN layout: thread (warp w, lane l) holds rows 16 w + l / 4 (+ 8) and, per 8-column group j, columns 8 j + 2 (l % 4) (+ 1)
    const int warp = tid >> 5, lane = tid & 31;
    uint32_t resid_ph = 0;
    float acc[2][GEMM_BN / 2]; // rows 0-63 and 64-127 of the tile
    // i: the tile's place in this CTA's sequence; tiles i and i + 1 go to different warpgroups
    for (unsigned i = cw, u = cluster + cw * clusters; pair_exists(u); i += 2, u += 2 * clusters)
    {
        const unsigned m_blk = u / n_pairs;
        const int m0 = (int)m_blk * GEMM_BM, n0 = (int)(2 * (u - m_blk * n_pairs) + rank) * GEMM_BN;
        const float bias_v = n0 + tid < p.N ? __ldg(p.bias + n0 + tid) : 0.f; // lands while the other warpgroup's k-loop runs
        if constexpr (kStaged)
        {
            // the staging buffer is free once the previous tile's last stores have read it (that overlaps the wait for this
            // warpgroup's turn); the residual of the first pass then lands in it while the k-loop runs
            if (tid == 0)
            {
                ptx::tma_store_wait_read<0>();
                if constexpr (gemm_epi(EPI).resid)
                    if (n0 < p.N) resid_load(sStage + cw * Cfg::kStageBytes, n0, m0, cw);
            }
        }

        // the tile's k-blocks sit at positions i * num_kb ... of the ring sequence
        const int g0 = i * num_kb;
        int s = g0 % kStages, s_prev = 0;
        uint32_t ph = (uint32_t)(g0 / kStages) & 1;
        if (i > 0) ptx::named_bar_sync(kBarTurn + cw, 256); // the other warpgroup has issued tile i-1's k-loop
        // every earlier reader of s_bias[cw] (tile i-2's epilogue) passed the barrier above before this write
        s_bias[cw][tid] = bias_v;
        for (int kb = 0; kb < num_kb; ++kb)
        {
            ptx::mbar_wait(full_bar(s), ph);
            const uint64_t adesc0 = ptx::wgmma_desc_kmajor_sw128(sA + s * Cfg::A_BYTES);
            const uint64_t adesc1 = ptx::wgmma_desc_kmajor_sw128(sA + s * Cfg::A_BYTES + 64 * 128);
            const uint64_t bdesc = ptx::wgmma_desc_kmajor_sw128(sB + s * Cfg::B_BYTES);
            ptx::fence_regs(acc[0]);
            ptx::fence_regs(acc[1]);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) // +32 B along K per step: k16 (f16) or k32 (e4m3)
            {
                if constexpr (kE4M3)
                {
                    ptx::wgmma_m64n128k32_e4m3(acc[0], adesc0 + 2 * k, bdesc + 2 * k, (kb | k) != 0);
                    ptx::wgmma_m64n128k32_e4m3(acc[1], adesc1 + 2 * k, bdesc + 2 * k, (kb | k) != 0);
                }
                else
                {
                    ptx::wgmma_m64n128k16_f16(acc[0], adesc0 + 2 * k, bdesc + 2 * k, (kb | k) != 0);
                    ptx::wgmma_m64n128k16_f16(acc[1], adesc1 + 2 * k, bdesc + 2 * k, (kb | k) != 0);
                }
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>(); // the previous k-block's MMAs have retired: its slot can be refilled
            ptx::fence_regs(acc[0]);
            ptx::fence_regs(acc[1]);
            if (kb > 0 && tid == 0) { ptx::mbar_arrive(empty_bar(s_prev)); ptx::mbar_arrive_cluster(empty_bar(s_prev), rank ^ 1); }
            s_prev = s;
            if (++s == kStages) { s = 0; ph ^= 1; }
        }
        if (pair_exists(u + clusters)) ptx::named_bar_arrive(kBarTurn + (cw ^ 1), 256); // tile i+1 may start its k-loop
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc[0]);
        ptx::fence_regs(acc[1]);
        if (tid == 0) { ptx::mbar_arrive(empty_bar(s_prev)); ptx::mbar_arrive_cluster(empty_bar(s_prev), rank ^ 1); }

        if constexpr (kStaged)
        {
            // ===================== staged epilogue: registers -> swizzled boxes -> TMA stores =====================
            const uint32_t stage = sStage + cw * Cfg::kStageBytes;
            // row r of a box lives at r * 128 B with its 16-B chunks permuted by chunk ^ (r % 8); r % 8 == lane / 4 for every row here
            const int rr = warp * 16 + (lane >> 2), sw = lane >> 2, q = lane & 3;
#pragma unroll
            for (int ps = 0; ps < St::kPasses; ++ps)
            {
                const int hm = ps / St::kColGroups, cg = ps % St::kColGroups; // rows 64 hm .., columns cg * kPassCols ..
                const int c0 = n0 + cg * St::kPassCols;
                if (c0 >= p.N || m0 + 64 * hm >= p.M) continue; // nothing of this pass is stored (uniform over the warpgroup)
                const int ncb = min(St::kColBoxes, (p.N - c0 + St::kBoxCols - 1) / St::kBoxCols); // boxes that start inside N
                const uint32_t buf = stage + (ps % St::kSlots) * St::kPassBytes;
                // e4m3: the scales of this thread's two rows of the pass (rr and rr + 8 of row half hm) times the W scale, rows past M
                // not stored; read per pass (four held from the k-loop on cost the split epilogue a spill), under the barrier below
                float row_scale[2];
                if constexpr (kE4M3)
                {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                    {
                        const int row = m0 + 64 * hm + rr + 8 * h;
                        row_scale[h] = row < p.M ? __fmul_rn(__ldg(p.a_scale + row), p.w_scale) : 0.f;
                    }
                }
                // LayerScale gamma of the pass's columns (zero past N): staged in shared memory per pass where a pass is at most 64
                // columns (6-stage ring; a 1 KB whole-tile array beside s_bias would take the CTA past the 227 KB of shared memory by
                // 256 bytes, and loads held in registers across the pass spill there), read through L1 at its use otherwise (5-stage
                // ring, 128-column passes).  The end-of-pass barrier below orders these writes after the previous pass's reads.
                constexpr bool kGammaSmem = EPI == EPI_BIAS_SCALE_RESID_F32 && St::kPassCols <= 64;
                __shared__ __align__(16) float s_gamma[2][kGammaSmem ? St::kPassCols : 1];
                if constexpr (kGammaSmem)
                    if (tid < St::kPassCols) s_gamma[cw][tid] = c0 + tid < p.N ? __ldg(p.gamma + c0 + tid) : 0.f;
                if (ps > 0 && tid == 0)
                {
                    if (ps >= St::kSlots) ptx::tma_store_wait_read<St::kSlots - 1>(); // the stores of the pass that used buf have read it
                    if constexpr (gemm_epi(EPI).resid) resid_load(buf, c0, m0 + 64 * hm, cw);
                }
                ptx::named_bar_sync(kBarWg + cw, 128); // pass 0: s_bias[cw] is written
                if constexpr (gemm_epi(EPI).resid)
                {
                    ptx::mbar_wait(resid_bar(cw), resid_ph);
                    resid_ph ^= 1;
                }
#pragma unroll
                for (int jj = 0; jj < St::kStoreCols / 8; ++jj)
                {
                    const int j = cg * (St::kPassCols / 8) + jj; // 8-column group of the tile
                    const float2 b = *reinterpret_cast<const float2 *>(&s_bias[cw][8 * j + 2 * q]);
                    float2 b2 = make_float2(0.f, 0.f); // SwiGLU: the bias of the x2 partners (group j + 8)
                    if constexpr (St::kSwiglu) b2 = *reinterpret_cast<const float2 *>(&s_bias[cw][8 * (j + 8) + 2 * q]);
                    float2 g = make_float2(0.f, 0.f); // LayerScale: the column pair's gamma (columns past N are never stored)
                    if constexpr (kGammaSmem) g = *reinterpret_cast<const float2 *>(&s_gamma[cw][8 * jj + 2 * q]);
                    else if constexpr (EPI == EPI_BIAS_SCALE_RESID_F32)
                        if (n0 + 8 * j + 2 * q < p.N) g = __ldg(reinterpret_cast<const float2 *>(p.gamma + n0 + 8 * j + 2 * q));
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                    {
                        float a0 = acc[hm][4 * j + 2 * h], a1 = acc[hm][4 * j + 2 * h + 1];
                        if constexpr (kE4M3) { a0 = __fmul_rn(a0, row_scale[h]); a1 = __fmul_rn(a1, row_scale[h]); }
                        const float x0 = __fadd_rn(a0, b.x), x1 = __fadd_rn(a1, b.y);
                        const uint32_t row = buf + (uint32_t)(rr + 8 * h) * 128u;
                        if constexpr (St::kF16)
                        {
                            const uint32_t a = row + (((jj % 8) ^ sw) << 4) + 4 * q;
                            __half2 hv;
                            if constexpr (EPI == EPI_BIAS_GELU_F16)
                            {
                                const float2 r = __half22float2(__floats2half2_rn(x0, x1)); // ggml.c:1434-1441: y = f16(gelu(f32(f16(x))))
                                hv = __floats2half2_rn(gelu_tanh_f32(r.x), gelu_tanh_f32(r.y));
                            }
                            else if constexpr (EPI == EPI_BIAS_GELU_ERF_F16) hv = __floats2half2_rn(gelu_erf_f32(x0), gelu_erf_f32(x1));
                            else if constexpr (EPI == EPI_BIAS_QUICK_GELU_F16) hv = __floats2half2_rn(quick_gelu_f32(x0), quick_gelu_f32(x1));
                            else if constexpr (EPI == EPI_BIAS_GELU_PYTORCH_TANH_F16) // PyTorch's tanh GELU: x itself, no f16 table
                                hv = __floats2half2_rn(gelu_tanh_f32(x0), gelu_tanh_f32(x1));
                            else if constexpr (St::kSwiglu) // x0, x1 are x1 of two columns; their x2 partners sit 64 columns on
                            {
                                float g0 = acc[hm][4 * (j + 8) + 2 * h], g1 = acc[hm][4 * (j + 8) + 2 * h + 1];
                                if constexpr (kE4M3) { g0 = __fmul_rn(g0, row_scale[h]); g1 = __fmul_rn(g1, row_scale[h]); }
                                hv = __floats2half2_rn(__fmul_rn(silu_f32(x0), __fadd_rn(g0, b2.x)), __fmul_rn(silu_f32(x1), __fadd_rn(g1, b2.y)));
                            }
                            else hv = __floats2half2_rn(x0, x1);
                            ptx::st_shared_b32(a + St::box(0, jj / 8), *reinterpret_cast<const uint32_t *>(&hv));
                            if constexpr (EPI == EPI_BIAS_F16_HILO)
                            {
                                const float2 hf = __half22float2(hv); // lo = f16(x - hi): exact difference, |lo| <= 2^-11 |x|
                                const __half2 lo = __floats2half2_rn(__fsub_rn(x0, hf.x), __fsub_rn(x1, hf.y));
                                ptx::st_shared_b32(a + St::box(1, jj / 8), *reinterpret_cast<const uint32_t *>(&lo));
                            }
                        }
                        else
                        {
                            const uint32_t a = row + St::box(0, jj / 4) + (((2 * (jj % 4) + (q >> 1)) ^ sw) << 4) + 8 * (q & 1);
                            if constexpr (EPI == EPI_BIAS_RESID_F32)
                            {
                                const float2 r = ptx::ld_shared_v2_f32(a); // (mul_mat + b) + inpL, vit.cpp:869,873
                                ptx::st_shared_v2_f32(a, __fadd_rn(x0, r.x), __fadd_rn(x1, r.y));
                            }
                            else if constexpr (EPI == EPI_BIAS_SCALE_RESID_F32)
                            {
                                const float2 r = ptx::ld_shared_v2_f32(a); // x + gamma * (mul_mat + b), HF Dinov2Layer's order
                                ptx::st_shared_v2_f32(a, __fadd_rn(__fmul_rn(x0, g.x), r.x), __fadd_rn(__fmul_rn(x1, g.y), r.y));
                            }
                            else ptx::st_shared_v2_f32(a, x0, x1);
                        }
                    }
                }
                ptx::fence_proxy_async_smem(); // the writes above are seen by the TMA engine
                ptx::named_bar_sync(kBarWg + cw, 128);
                if (tid == 0)
                {
                    const int row = m0 + 64 * hm;
                    for (int c = 0; c < ncb; ++c)
                    {
                        const uint32_t src = buf + St::box(0, c);
                        if constexpr (St::kF16)
                        {
                            if (p.headmajor)
                            {
                                const int plane = (c0 >> 6) + c;
                                ptx::tma_store_3d(&tmOut, src, 0, row, plane);
                                if constexpr (EPI == EPI_BIAS_F16_HILO) ptx::tma_store_3d(&tmAux, buf + St::box(1, c), 0, row, plane);
                            }
                            else if constexpr (St::kSwiglu) ptx::tma_store_2d(&tmOut, src, c0 / 2, row);
                            else
                            {
                                ptx::tma_store_2d(&tmOut, src, c0 + 64 * c, row);
                                if constexpr (EPI == EPI_BIAS_F16_HILO) ptx::tma_store_2d(&tmAux, buf + St::box(1, c), c0 + 64 * c, row);
                            }
                        }
                        else ptx::tma_store_2d(&tmOut, src, c0 + 32 * c, row);
                    }
                    ptx::tma_store_commit();
                }
            }
        }
        else
        {
            // ===================== register epilogue (patch embedding, head) =====================
            ptx::named_bar_sync(kBarWg + cw, 128); // s_bias[cw] is written
            const int col0 = n0 + 2 * (lane & 3);
#pragma unroll
            for (int hm = 0; hm < 2; ++hm)
            {
                const int row0 = m0 + 64 * hm + warp * 16 + (lane >> 2);
#pragma unroll
                for (int j = 0; j < GEMM_BN / 8; ++j)
                {
                    const int col = col0 + 8 * j;
                    if (col >= p.N) continue; // N % 4 == 0: a column pair is all-in or all-out
                    const float2 b = *reinterpret_cast<const float2 *>(&s_bias[cw][col - n0]);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                    {
                        const int row = row0 + 8 * h;
                        if (row >= p.M) continue;
                        const float x0 = __fadd_rn(acc[hm][4 * j + 2 * h], b.x), x1 = __fadd_rn(acc[hm][4 * j + 2 * h + 1], b.y);
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
    }
    if constexpr (kStaged)
        if (tid == 0) ptx::tma_store_wait_read<0>(); // the shared memory must outlive the reads of the last stores
}

} // namespace vitb200
