// attention_wgmma.cuh -- fused attention for one (image, head) per CTA on the Hopper warpgroup tensor cores, N <= 224 tokens.
//
// Replaces the reference's reshape/permute/CONT nodes + mul_mat(K,Q) + scale + soft_max_inplace + mul_mat(V,P) + head merge
// (reference vit.cpp:826-866) for the 197-token geometries.  Same soft-max semantics as attention_kernel (kernels.cuh): the TRUE row
// maximum, e = f16(exp(f16(s * scale - max))), l = sum e in f32, O = (P V) * (1 / l).
//
//   TMA       one thread loads the q tiles (64 rows each) and the whole K and V of the head (224 rows, zero-filled / masked past N)
//             out of the head-major QKV buffers, SWIZZLE_128B, under one mbarrier -- hi and, with HILO, lo halves
//   S = QK^T  wgmma.m64n224k16, A = Q tile and B = K from shared memory, f32 accumulators in registers (one warpgroup per 64-query
//             tile; two warpgroups, each taking every other tile).  HILO: S = Ql Kh^T + Qh Kl^T + Qh Kh^T (kernels.cuh explains why)
//   softmax   in registers: each row lives in one quad of lanes; P is packed to f16 in place, already in the A-fragment layout
//   O = P V   wgmma.m64n64k16 with A = P from registers and B = V (MN-major) from shared memory; HILO: O = P Vl + P Vh
#pragma once
#include "kernels.cuh"

namespace vitb200 {

constexpr int ATTW_KEYS = 224;                       // keys per problem (wgmma N), N <= ATTW_KEYS
constexpr int ATTW_THREADS = 256;                    // two warpgroups
constexpr int ATTW_QTILE_BYTES = 64 * 128;           // 64 query rows x 64 dims f16
constexpr int ATTW_KV_BYTES = ATTW_KEYS * 128;       // 224 rows x 64 dims f16 (28 KB, 1024-B multiple)

__host__ __device__ inline int attention_wgmma_smem_bytes(bool hilo)
{
    return 1024 + (hilo ? 2 : 1) * (4 * ATTW_QTILE_BYTES + 2 * ATTW_KV_BYTES) + 64;
}

template <bool HILO>
__global__ void __launch_bounds__(ATTW_THREADS, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                       const __grid_constant__ CUtensorMap tmQl, const __grid_constant__ CUtensorMap tmKVl,
                       __half *__restrict__ out, int N, int D, int H, float scale)
// tmQ / tmQl: 3-D maps {64, rows, 3 H planes} of the hi / lo QKV buffers with 64-row boxes; tmKV / tmKVl: the same with 224-row boxes
{
    extern __shared__ uint8_t attw_smem_raw[];
    const uint32_t base = (ptx::smem_u32(attw_smem_raw) + 1023u) & ~1023u;
    constexpr int kParts = HILO ? 2 : 1;
    // [part][4 q tiles] | [part] K | [part] V | barrier
    auto sQ = [&](int part, int t) { return base + (uint32_t)(part * 4 + t) * ATTW_QTILE_BYTES; };
    auto sK = [&](int part) { return base + kParts * 4 * ATTW_QTILE_BYTES + (uint32_t)part * ATTW_KV_BYTES; };
    auto sV = [&](int part) { return base + kParts * 4 * ATTW_QTILE_BYTES + (uint32_t)(kParts + part) * ATTW_KV_BYTES; };
    const uint32_t bar = base + kParts * (4 * ATTW_QTILE_BYTES + 2 * ATTW_KV_BYTES);

    const int b = blockIdx.x / H, h = blockIdx.x - b * H;
    const int n_mt = (N + 63) >> 6;
    const int row0 = b * N; // this image's first token row in every plane
    if (threadIdx.x == 0)
    {
        ptx::prefetch_tensormap(&tmQ);
        ptx::prefetch_tensormap(&tmKV);
        ptx::mbar_init(bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();
    // launched with programmatic dependent launch: q, k, v are read only once the qkv GEMM has completed
    ptx::grid_dep_launch();
    ptx::grid_dep_wait();
    if (threadIdx.x == 0)
    {
        ptx::mbar_arrive_expect_tx(bar, (uint32_t)(kParts * (n_mt * ATTW_QTILE_BYTES + 2 * ATTW_KV_BYTES)));
        for (int part = 0; part < kParts; ++part)
        {
            const CUtensorMap *mq = part ? &tmQl : &tmQ, *mkv = part ? &tmKVl : &tmKV;
            for (int t = 0; t < n_mt; ++t) ptx::tma_load_3d(sQ(part, t), mq, bar, 0, row0 + 64 * t, h);
            ptx::tma_load_3d(sK(part), mkv, bar, 0, row0, H + h);
            ptx::tma_load_3d(sV(part), mkv, bar, 0, row0, 2 * H + h);
        }
    }
    ptx::mbar_wait(bar, 0);

    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31;
    const int c0 = 2 * (lane & 3); // key / dim columns 8 j + c0 (+ 1) of this thread
    for (int mt = wg; mt < n_mt; mt += 2)
    {
        // ---- S = Q K^T (f32, registers)
        float s[ATTW_KEYS / 2];
#pragma unroll
        for (int i = 0; i < ATTW_KEYS / 2; ++i) s[i] = 0.f;
        ptx::fence_regs(s);
        ptx::wgmma_fence();
        const uint64_t qh = ptx::wgmma_desc_kmajor_sw128(sQ(0, mt)), kh = ptx::wgmma_desc_kmajor_sw128(sK(0));
#pragma unroll
        for (int k = 0; k < 4; ++k) // 64 dims = 4 x K 16 (+32 B each)
        {
            if constexpr (HILO)
            {
                const uint64_t ql = ptx::wgmma_desc_kmajor_sw128(sQ(1, mt)), kl = ptx::wgmma_desc_kmajor_sw128(sK(1));
                ptx::wgmma_m64n224k16_f16(s, ql + 2 * k, kh + 2 * k, k != 0);
                ptx::wgmma_m64n224k16_f16(s, qh + 2 * k, kl + 2 * k, 1);
                ptx::wgmma_m64n224k16_f16(s, qh + 2 * k, kh + 2 * k, 1);
            }
            else ptx::wgmma_m64n224k16_f16(s, qh + 2 * k, kh + 2 * k, k != 0);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(s);

        // ---- soft-max over the valid keys: rows r (s[4j], s[4j+1]) and r + 8 (s[4j+2], s[4j+3]) of this quad
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < ATTW_KEYS / 8; ++j)
        {
            const int key = 8 * j + c0;
            if (key < N) { mx0 = fmaxf(mx0, s[4 * j]); mx1 = fmaxf(mx1, s[4 * j + 2]); }
            if (key + 1 < N) { mx0 = fmaxf(mx0, s[4 * j + 1]); mx1 = fmaxf(mx1, s[4 * j + 3]); }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        mx0 *= scale; // ggml_scale_inplace (vit.cpp:851-854): exact for hd = 64 (0.125)
        mx1 *= scale;
        float l0 = 0.f, l1 = 0.f;
#pragma unroll
        for (int j = 0; j < ATTW_KEYS / 8; ++j)
        {
            const int key = 8 * j + c0;
            const bool v0 = key < N, v1 = key + 1 < N;
            const __half p00 = v0 ? exp_f16_semantics(__fmul_rn(s[4 * j], scale) - mx0) : __float2half_rn(0.f);
            const __half p01 = v1 ? exp_f16_semantics(__fmul_rn(s[4 * j + 1], scale) - mx0) : __float2half_rn(0.f);
            const __half p10 = v0 ? exp_f16_semantics(__fmul_rn(s[4 * j + 2], scale) - mx1) : __float2half_rn(0.f);
            const __half p11 = v1 ? exp_f16_semantics(__fmul_rn(s[4 * j + 3], scale) - mx1) : __float2half_rn(0.f);
            l0 += __half2float(p00) + __half2float(p01);
            l1 += __half2float(p10) + __half2float(p11);
            const __half2 h0 = __halves2half2(p00, p01), h1 = __halves2half2(p10, p11);
            s[4 * j] = __uint_as_float(*reinterpret_cast<const uint32_t *>(&h0)); // P packed in place: row r pair, row r + 8 pair
            s[4 * j + 2] = __uint_as_float(*reinterpret_cast<const uint32_t *>(&h1));
        }
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
        l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

        // ---- O = P V: keys 16 kk .. 16 kk + 15 are the A fragment {row r k 0-7, row r+8 k 0-7, row r k 8-15, row r+8 k 8-15}
        float o[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = 0.f;
        ptx::fence_regs(o);
        ptx::fence_regs(s);
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < ATTW_KEYS / 16; ++kk)
        {
            const uint32_t a0 = __float_as_uint(s[8 * kk]), a1 = __float_as_uint(s[8 * kk + 2]);
            const uint32_t a2 = __float_as_uint(s[8 * kk + 4]), a3 = __float_as_uint(s[8 * kk + 6]);
            const uint64_t vh = ptx::wgmma_desc_mnmajor_sw128(sV(0) + (uint32_t)kk * 2048u);
            if constexpr (HILO)
            {
                ptx::wgmma_m64n64k16_f16_rs_tb(o, a0, a1, a2, a3, ptx::wgmma_desc_mnmajor_sw128(sV(1) + (uint32_t)kk * 2048u), kk != 0);
                ptx::wgmma_m64n64k16_f16_rs_tb(o, a0, a1, a2, a3, vh, 1);
            }
            else ptx::wgmma_m64n64k16_f16_rs_tb(o, a0, a1, a2, a3, vh, kk != 0);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(o);

        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1; // p_i = e_i * (1/sum)  (ggml.c:10556-10558)
        const int r0 = mt * 64 + warp * 16 + (lane >> 2), r1 = r0 + 8;
        __half *o0 = out + ((size_t)b * N + r0) * D + h * 64 + c0;
        __half *o1 = out + ((size_t)b * N + r1) * D + h * 64 + c0;
#pragma unroll
        for (int dt = 0; dt < 8; ++dt)
        {
            if (r0 < N) *reinterpret_cast<__half2 *>(o0 + dt * 8) = __floats2half2_rn(o[4 * dt] * inv0, o[4 * dt + 1] * inv0);
            if (r1 < N) *reinterpret_cast<__half2 *>(o1 + dt * 8) = __floats2half2_rn(o[4 * dt + 2] * inv1, o[4 * dt + 3] * inv1);
        }
    }
}

} // namespace vitb200
