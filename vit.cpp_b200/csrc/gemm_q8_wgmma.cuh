// gemm_q8_wgmma.cuh -- the reference's q8_0 x q8_0 linear layer on the INTEGER tensor cores: prototype (BASELINE.json configs[4]).
//
// Reference semantics (q8_0 model files): every mul_mat with a quantised weight first quantises its f32 activation rows to
// q8_0 blocks of 32 (quantize_row_q8_0, ggml-quants.c:702-790: d = amax / 127 stored as f16, q = rint(x * 127 / amax)) and then
// evaluates, per output element (ggml_vec_dot_q8_0_q8_0, ggml-quants.c:3521+; block layout ggml-quants.h:42-46)
//     y = sum over blocks b of  (d_w[b] * d_x[b]) * (sum over the block's 32 elements of q_w * q_x)      accumulated in f32.
// One f32 scale per 32-element block of BOTH operands means an int32 accumulator can span exactly one block:
// wgmma.m64n128k32.s32.s8.s8 has K = 32 per instruction == one q8_0 block, so every MMA writes a FRESH integer accumulator, which the
// same warpgroup converts to f32 (exact: |sum| <= 32 * 127 * 127 < 2^24) and folds in as acc = fma(d_w * d_x, sum, acc) -- the
// reference's own arithmetic up to the order of the eight partial f32 lanes of its AVX2 kernel.
// Data layout (repacked once at upload -- the 34-byte block_q8_0 is TMA-hostile): int8 planes A [M][K] and W [N][K] (K contiguous,
// 128-byte SWIZZLE_128B rows = 4 blocks per pipeline stage), scale planes Ad [M][K/32] f32 and WdT [K/32][N] f32 (transposed so a
// block's 128 column scales are one contiguous shared-memory row), all four moved by TMA under one mbarrier per stage.
// Warpgroup 0 is the TMA producer; warpgroups 1-2 each own 64 rows of the 128 x 128 tile.
//
// What this prototype is for (DESIGN.md section 3): the per-element correction costs FP32-pipe work per block against one K = 32 MMA,
// so the kernel is bound by the FP32 pipe, not the int8 tensor rate.  Kept as a tested kernel, not wired into the forward schedule.
#pragma once
#include "ptx.cuh"

namespace vitb200 {

struct Q8GemmParams
{
    int M, N, K;       // K % 128 == 0 (4 blocks per stage), N % 4 == 0
    const float *bias; // [N]
    float *out;        // [M][ldo] f32
    int ldo;
};

constexpr int Q8_BM = 128, Q8_BN = 128, Q8_BK = 128; // tile; K bytes (= int8 elements) per stage
constexpr int Q8_STAGES = 5;
constexpr int Q8_THREADS = 384; // warpgroup 0 TMA, warpgroups 1-2 MMA + correction
constexpr int Q8_A_BYTES = Q8_BM * Q8_BK, Q8_W_BYTES = Q8_BN * Q8_BK;
constexpr int Q8_AD_BYTES = Q8_BM * 4 * 4, Q8_WD_BYTES = 4 * Q8_BN * 4;
constexpr int Q8_STAGE_BYTES = Q8_A_BYTES + Q8_W_BYTES + Q8_AD_BYTES + Q8_WD_BYTES;
constexpr int Q8_SMEM_BYTES = 1024 + Q8_STAGES * Q8_STAGE_BYTES + 256;

// f32 activations [M][K] -> q8_0: int8 plane + per-block scale (the f16-rounded d, widened back to f32 as the dot product uses it).
// Bit-exact restatement of quantize_row_q8_0's AVX2 branch (ggml-quants.c:722-742): IEEE divisions, round-half-even.
// Eight lanes per block (one float4 each); a warp covers 128 consecutive elements per step.
__global__ void quantize_q8_0_kernel(const float *__restrict__ x, int8_t *__restrict__ q, float *__restrict__ d_out, long long n_blocks)
{
    const long long gthread = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long blk = gthread >> 3;
    const int sub = (int)(gthread & 7);
    const bool ok = blk < n_blocks;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) v = __ldg(reinterpret_cast<const float4 *>(x + blk * 32) + sub);
    float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float d = __fdiv_rn(amax, 127.f);
    const float id = amax != 0.0f ? __fdiv_rn(127.f, amax) : 0.0f;
    if (!ok) return;
    const int q0 = __float2int_rn(__fmul_rn(v.x, id)), q1 = __float2int_rn(__fmul_rn(v.y, id));
    const int q2 = __float2int_rn(__fmul_rn(v.z, id)), q3 = __float2int_rn(__fmul_rn(v.w, id));
    const uint32_t packed = (uint32_t)(q0 & 0xFF) | ((uint32_t)(q1 & 0xFF) << 8) | ((uint32_t)(q2 & 0xFF) << 16) | ((uint32_t)(q3 & 0xFF) << 24);
    reinterpret_cast<uint32_t *>(q + blk * 32)[sub] = packed;
    if (sub == 0) d_out[blk] = __half2float(__float2half_rn(d));
}

__global__ void __launch_bounds__(Q8_THREADS, 1)
gemm_q8_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                     const __grid_constant__ CUtensorMap tmAd, const __grid_constant__ CUtensorMap tmWd, const Q8GemmParams p)
{
    extern __shared__ uint8_t q8_smem_raw[];
    const uint32_t smem_base = (ptx::smem_u32(q8_smem_raw) + 1023u) & ~1023u;
    uint8_t *smem = q8_smem_raw + (smem_base - ptx::smem_u32(q8_smem_raw));
    auto sA = [&](int s) { return smem_base + (uint32_t)s * Q8_STAGE_BYTES; };
    auto sW = [&](int s) { return sA(s) + Q8_A_BYTES; };
    auto sAd = [&](int s) { return sW(s) + Q8_W_BYTES; };
    auto sWd = [&](int s) { return sAd(s) + Q8_AD_BYTES; };
    const uint32_t bars = smem_base + Q8_STAGES * Q8_STAGE_BYTES;
    auto full_bar = [&](int s) { return bars + 8u * s; };
    auto empty_bar = [&](int s) { return bars + 8u * (Q8_STAGES + s); };

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
    const int n_tiles = (p.N + Q8_BN - 1) / Q8_BN;
    const int m0 = (blockIdx.x / n_tiles) * Q8_BM, n0 = (blockIdx.x % n_tiles) * Q8_BN;
    const int num_kb = p.K / Q8_BK;

    if (threadIdx.x == 0)
    {
        ptx::prefetch_tensormap(&tmA);
        ptx::prefetch_tensormap(&tmW);
        ptx::prefetch_tensormap(&tmAd);
        ptx::prefetch_tensormap(&tmWd);
        for (int s = 0; s < Q8_STAGES; ++s)
        {
            ptx::mbar_init(full_bar(s), 1);
            ptx::mbar_init(empty_bar(s), 2);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0)
    {
        // ===================== TMA producer: int8 operand tiles + both scale tiles of a stage under one barrier =====================
        ptx::setmaxnreg_dec<40>();
        if (tid == 0)
        {
            for (int kb = 0; kb < num_kb; ++kb)
            {
                const int s = kb % Q8_STAGES;
                ptx::mbar_wait(empty_bar(s), ((kb / Q8_STAGES) & 1) ^ 1);
                ptx::mbar_arrive_expect_tx(full_bar(s), Q8_STAGE_BYTES);
                ptx::tma_load_2d(sA(s), &tmA, full_bar(s), kb * Q8_BK, m0);
                ptx::tma_load_2d(sW(s), &tmW, full_bar(s), kb * Q8_BK, n0);
                ptx::tma_load_2d(sAd(s), &tmAd, full_bar(s), kb * 4, m0);
                ptx::tma_load_2d(sWd(s), &tmWd, full_bar(s), n0, kb * 4);
            }
        }
        return;
    }

    // ===================== MMA warpgroups: one K = 32 MMA per q8_0 block, folded into f32 with the block scales =====================
    ptx::setmaxnreg_inc<232>();
    const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
    const int r0 = cw * 64 + warp * 16 + (lane >> 2); // tile rows r0, r0 + 8 of this thread
    const int c0 = 2 * (lane & 3);                    // tile columns 8 j + c0 (+ 1)
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb)
    {
        const int s = kb % Q8_STAGES;
        ptx::mbar_wait(full_bar(s), (kb / Q8_STAGES) & 1);
        const uint64_t adesc = ptx::wgmma_desc_kmajor_sw128(sA(s) + cw * 64 * 128);
        const uint64_t bdesc = ptx::wgmma_desc_kmajor_sw128(sW(s));
        const float *ad = reinterpret_cast<const float *>(smem + (size_t)s * Q8_STAGE_BYTES + Q8_A_BYTES + Q8_W_BYTES); // [128 rows][4]
        const float *wd = ad + Q8_AD_BYTES / 4;                                                                      // [4][128 columns]
#pragma unroll
        for (int j = 0; j < 4; ++j)
        {
            uint32_t isum[64];
            ptx::wgmma_fence();
            ptx::wgmma_m64n128k32_s8(isum, adesc + 2 * j, bdesc + 2 * j); // 32 int8 = 32 B along K: +2 in the (addr >> 4) field
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(isum[i])::"memory");
            const float ad0 = ad[r0 * 4 + j], ad1 = ad[(r0 + 8) * 4 + j];
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
            {
                const float2 w = *reinterpret_cast<const float2 *>(wd + j * Q8_BN + jj * 8 + c0);
                // d = d_w * d_x (ggml-quants.c:3521+); the integer block sum converts to f32 exactly
                acc[4 * jj + 0] = __fmaf_rn(__fmul_rn(w.x, ad0), (float)(int)isum[4 * jj + 0], acc[4 * jj + 0]);
                acc[4 * jj + 1] = __fmaf_rn(__fmul_rn(w.y, ad0), (float)(int)isum[4 * jj + 1], acc[4 * jj + 1]);
                acc[4 * jj + 2] = __fmaf_rn(__fmul_rn(w.x, ad1), (float)(int)isum[4 * jj + 2], acc[4 * jj + 2]);
                acc[4 * jj + 3] = __fmaf_rn(__fmul_rn(w.y, ad1), (float)(int)isum[4 * jj + 3], acc[4 * jj + 3]);
            }
        }
        if (tid == 0) ptx::mbar_arrive(empty_bar(s));
    }
    // bias + store
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
    {
        const int gcol = n0 + jj * 8 + c0;
        if (gcol >= p.N) continue; // N % 4 == 0
        const float2 b = __ldg(reinterpret_cast<const float2 *>(p.bias + gcol));
#pragma unroll
        for (int h = 0; h < 2; ++h)
        {
            const int grow = m0 + r0 + 8 * h;
            if (grow < p.M)
                *reinterpret_cast<float2 *>(p.out + (size_t)grow * p.ldo + gcol) =
                    make_float2(__fadd_rn(acc[4 * jj + 2 * h], b.x), __fadd_rn(acc[4 * jj + 2 * h + 1], b.y));
        }
    }
}

} // namespace vitb200
