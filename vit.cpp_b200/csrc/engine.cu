// engine.cu -- host side of the C ABI in include/vitb200.h: weight upload/repack, the static device arena,
// TMA descriptors, and the fixed kernel schedule that replaces the reference's per-image graph build +
// ggml_allocr + ggml_graph_compute thread pool (reference vit.cpp:1004-1075, ggml.c:15774-16039).
#include "../../include/vitb200.h"

#include "gemm_wgmma.cuh"
#include "kernels.cuh"
#include "gemm_q8_wgmma.cuh"
#include "attention_wgmma.cuh"
#include "gguf_file.hpp"
#include "preprocess.cuh"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

using namespace vitb200;

namespace {

thread_local std::string g_err;

int fail(const char *fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    fprintf(stderr, "vitb200: %s\n", buf); // reference convention: message on stderr + non-zero return
    return 1;
}

// The C ABI promises "non-zero return, never abort": nothing may unwind through an extern "C" frame.  Host-side allocations
// (std::vector staging buffers sized from a model file, the graph cache, debug taps) can throw; every exported function that can
// reach one runs its body through this.
template <class F>
int guarded(const char *fn, F &&body) noexcept
{
    try
    {
        return body();
    }
    catch (const std::exception &ex) { return fail("%s: %s", fn, ex.what()); }
    catch (...) { return fail("%s: unknown exception", fn); }
}

#define CUDA_TRY(x)                                                                       \
    do                                                                                    \
    {                                                                                     \
        cudaError_t e_ = (x);                                                             \
        if (e_ != cudaSuccess)                                                            \
        {                                                                                 \
            (void)cudaGetLastError(); /* do not leave it for an unrelated later check */  \
            return fail("%s failed: %s", #x, cudaGetErrorString(e_));                     \
        }                                                                                 \
    } while (0)

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                        const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_tmapEncodeTiled tmap_encoder()
{
    static PFN_tmapEncodeTiled fn = nullptr;
    if (!fn)
    {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
    }
    return fn;
}

// A 2-D or 3-D tensor map over ptr: dims and box in elements, innermost first; strides in bytes, of dimensions 1 .. rank-1.  Dense
// elements, L2 promotion of 256 B, out-of-bounds elements read as zero.  The GEMM operands and the attention's q / k / v tiles use
// SWIZZLE_128B with a box one 128-byte row wide: the layout the wgmma K-major SWIZZLE_128B shared-memory descriptor reads.
template <int R>
int make_tmap(CUtensorMap *m, CUtensorMapDataType dt, const void *ptr, const cuuint64_t (&dims)[R], const cuuint64_t (&strides)[R - 1],
              const cuuint32_t (&box)[R], CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B)
{
    static_assert(R == 2 || R == 3, "2-D and 3-D maps only");
    PFN_tmapEncodeTiled enc = tmap_encoder();
    if (!enc) return fail("cuTensorMapEncodeTiled entry point not available");
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(m, dt, R, const_cast<void *>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail("cuTensorMapEncodeTiled failed (%d): dims {%llu, %llu, %llu}, row stride %llu B, box {%u, %u, %u}", (int)r,
                    (unsigned long long)dims[0], (unsigned long long)dims[1], R > 2 ? (unsigned long long)dims[R - 1] : 1ull,
                    (unsigned long long)strides[0], box[0], box[1], R > 2 ? box[R - 1] : 1u);
    return 0;
}

struct Linear
{
    __half *w = nullptr; // [n_out][ld] f16, K contiguous (ggml ne0 = K)
    uint8_t *w8 = nullptr; // FP8 engine, qkv and fc1: [n_out][ld] e4m3 instead of w; the weight is w8 * w_scale
    float w_scale = 1.f;
    float *b = nullptr;  // [n_out]
    int n_out = 0, n_in = 0, ld = 0;
    CUtensorMap tm;  // box = one k-block (64 f16 or 128 e4m3 = 128 B) x GEMM_BN rows: the W tile of one k-block
};

struct Layer
{
    float *n1w = nullptr, *n1b = nullptr, *n2w = nullptr, *n2b = nullptr;
    float *ls1 = nullptr, *ls2 = nullptr; // vitb200_arch.layer_scale: the LayerScale gamma [D] of proj and of fc2
    Linear qkv, proj, fc1, fc2;
};

// Argument set of one cached CUDA graph: a classification forward (layers = -1) or an encoder-features call
struct GraphKey
{
    const void *img; int batch; void *probs, *logits, *tidx, *tval; int k;
    int layers, norm, dtype; void *tok, *pre;
    bool operator==(const GraphKey &o) const
    {
        return img == o.img && batch == o.batch && probs == o.probs && logits == o.logits && tidx == o.tidx && tval == o.tval && k == o.k &&
               layers == o.layers && norm == o.norm && dtype == o.dtype && tok == o.tok && pre == o.pre;
    }
};

// One of the two host-pipeline slots (vitb200_forward_async, the u8 and recognition entry points): call n uses slot n & 1, so its
// H2D copy on the copy stream can overlap call n - 1's kernels on the compute stream
// The image processor's layout of one u8 call (plan_proc): per-image geometry, the tap-table widths of the two passes, the most source
// rows of one image and the scratch bytes of the horizontal pass
struct ProcPlan
{
    std::vector<ProcGeom> geo;
    int kh = 1, kv = 1, max_rows = 1;
    size_t tmp_total = 0;
};

struct Slot
{
    float *img = nullptr, *probs = nullptr, *logits = nullptr, *topk_val = nullptr;
    int32_t *topk_idx = nullptr;
    // text recognition (1-channel models with head_tokens >= 2): decoded class ids [max_batch][head_tokens - 1], lengths, scores
    int32_t *chars = nullptr, *len = nullptr;
    double *score = nullptr;
    // GPU preprocessing: a PINNED host staging buffer (the caller's images are packed into it, followed by the per-image
    // descriptors) and its device twin; grown only when a batch needs more than any batch before it
    uint8_t *h_u8 = nullptr, *d_u8 = nullptr;
    size_t u8_cap = 0;
    // the image processor's horizontal pass (vitb200_set_image_proc): [rows][img_size][3] u8 per image, grown like the staging buffer
    uint8_t *d_proc = nullptr;
    size_t proc_cap = 0;
    int32_t *ids = nullptr; // text engines: the token ids of the call [max_batch][N]
    cudaEvent_t ev_h2d = nullptr, ev_done = nullptr;
};

} // namespace

struct vitb200_engine
{
    vitb200_hparams hp;
    vitb200_arch arch{}; // pre-norm, MLP activation, LayerScale, register tokens, head pooling; all zero is the reference's architecture
    float *npre_w = nullptr, *npre_b = nullptr; // arch.pre_norm: norm_pre.weight / norm_pre.bias
    int device = 0, max_batch = 0, num_sms = 132;
    int N = 0, NP = 0, G = 0, KP = 0, KPp = 0; // N = prefix_rows(arch) + NP token rows per image
    int F = 0;            // the MLP's hidden width: 4 D, or SwiGLU's F (arch.activation = 4, read from block 0's fc1)
    int Cp = 0;           // num_classes rounded up to a multiple of 4: pitch of the internal logits rows (128-bit epilogue stores)
    float *d_sm_scratch = nullptr; // soft-max working rows in global memory, only when num_classes floats exceed shared memory
    int C = 3;            // input channels: 3 (vit.cpp) or 1 (ViTSTR extension, vitstr.cpp:713), taken from the patch kernel's shape
    int head_tokens = 1;  // tokens the classifier head reads per image: 1 (token 0, vit.cpp:910) or 25 (vitstr.cpp:864-903)
    int KH = 0;           // the head's K: D, or 2 D with arch.pool = 1 (CLS16 rows are [LN(cls) || mean of LN(patches)])
    // SigLIP's attention-pooling head (arch.pool = 2): the probe's query pool_q [D] (latent Wq^T + bq, f32), k | v, out_proj, the
    // head's LayerNorm and MLP; POOL32 [max_batch][D] f32 holds the pooled rows (out_proj's output, then + the MLP's)
    float *pool_q = nullptr, *pool_nw = nullptr, *pool_nb = nullptr, *POOL32 = nullptr;
    Linear pool_kv, pool_proj, pool_fc1, pool_fc2;
    // FP8 engine (vitb200_create_fp8): LayerNorms 1 and 2 write e4m3 rows A8 with per-row scales SA, and the qkv and fc1 GEMMs run
    // e4m3 x e4m3 against per-tensor-scaled e4m3 weights; everything else is the f16 engine's schedule
    bool fp8 = false;
    uint8_t *A8 = nullptr;
    float *SA = nullptr;
    CUtensorMap tmA8;
    cudaStream_t stream = nullptr;
    std::vector<void *> allocs;
    // weights
    float *cls = nullptr, *pos = nullptr, *norm_w = nullptr, *norm_b = nullptr; // cls: [1 + reg_tokens][D], cls_token then reg_token
    // text towers (vitb200_create_text): the token table tok [V][D] f16 replaces the patch embedding; TOKS stages the host call's token
    // rows ([max_batch][N][D] f32 at most), which are written mid-schedule, while H16 is still in use
    bool text = false;
    vitb200_text_arch text_arch{};
    __half *tok = nullptr;
    int V = 0;
    uint8_t *TOKS = nullptr;
    Linear patch, head;
    std::vector<Layer> layers;
    // activations (static arena, sized for max_batch)
    float *X = nullptr, *d_logits = nullptr;
    __half *A16 = nullptr, *QKV16 = nullptr, *H16 = nullptr, *CLS16 = nullptr, *PA = nullptr;
    // lo halves of q, k, v (x - f16(x), as f16): the split-precision operands of the wgmma attention.  Allocated exactly when that
    // kernel runs (N <= 224); then the qkv GEMM emits hi + lo and the attention runs the 3 + 2 term products.
    __half *QKV16L = nullptr;
    CUtensorMap tmA_D, tmA_H, tmA_P, tmA_C;
    CUtensorMap tmQ, tmKV, tmQl, tmKVl; // attention operand maps (N <= 224: attention_wgmma_kernel)
    CUtensorMap tmKVp, tmKVpl;          // k and v maps of attention_wgmma_persistent_kernel (N <= ATTP_KEYS): ATTP_ROWS-row boxes
    int max_k = 16;
    int launches = 0;
    std::map<int, std::string> labels;
    // host-buffer pipeline (vitb200_forward_async): 2 input/output slots, H2D on a copy stream overlapping the previous
    // call's kernels on the compute stream
    cudaStream_t copy_stream = nullptr;
    Slot slot[2];
    unsigned long long submits = 0;
    // Hugging Face's image preprocessing for the RGB u8 entry points (vitb200_set_image_proc); proc_geom is the per-call host table
    bool has_proc = false;
    vitb200_image_proc proc{};
    ProcPlan proc_plan;
    // the zero-shot head (vitb200_set_zero_shot): zs_C > 0 classes, the unit class rows ZS_T [zs_C][num_classes] f32, the internal score
    // rows ZS_S [max_batch][zs_C] (when the caller takes no logits), s = f32(exp(logit_scale)), b = logit_bias (0 for NaN), mode 0
    // soft-max / 1 sigmoid; the arguments as set are kept for vitb200_get_zero_shot.  out_cols / sm_cols: the floats per row of the slot
    // probs and logits and of the soft-max scratch, grown to zs_C when a head needs more
    int zs_C = 0, zs_mode = 0;
    float zs_s = 0.f, zs_b = 0.f, zs_logit_scale = 0.f, zs_logit_bias = 0.f;
    float *ZS_T = nullptr, *ZS_S = nullptr;
    int out_cols = 0, sm_cols = 0;
    // CUDA-graph cache for the kernel schedule of one forward, keyed by its arguments (launch-bound inner loop: ~90 kernels)
    struct GraphEntry { GraphKey key; int state; int launches; cudaGraphExec_t exec; };
    std::vector<GraphEntry> graphs;
    bool use_graph = true;
    // optional per-kernel timing (bench.py roofline): CUDA event pairs around tracked launches
    bool profile = false;
    struct ProfRec { int kind; cudaEvent_t a, b; double flops; };
    std::vector<ProfRec> prof;
    std::vector<cudaEvent_t> event_pool;
};

namespace {

template <typename T>
int dev_alloc(vitb200_engine *e, T **p, size_t count)
{
    void *q = nullptr;
    CUDA_TRY(cudaMalloc(&q, count * sizeof(T) + 256));
    e->allocs.push_back(q);
    // zeroed once, so that no buffer starts out holding NaN bit patterns; no kernel relies on it afterwards (the attention kernels read
    // only the current image's rows: TMA zero fill past N in the wgmma kernel, explicit zeros in the mma.sync kernels)
    CUDA_TRY(cudaMemset(q, 0, count * sizeof(T) + 256));
    *p = reinterpret_cast<T *>(q);
    return 0;
}

// Frees the engine-owned buffer *p (from dev_alloc, or NULL) and sets it to NULL
template <typename T>
void dev_free(vitb200_engine *e, T **p)
{
    if (!*p) return;
    e->allocs.erase(std::remove(e->allocs.begin(), e->allocs.end(), (void *)*p), e->allocs.end());
    cudaFree(*p);
    *p = nullptr;
}

const vitb200_tensor *find_tensor(const vitb200_tensor *t, int n, const std::string &name)
{
    for (int i = 0; i < n; ++i)
        if (t[i].name && name == t[i].name) return &t[i];
    return nullptr;
}

// the reference keeps tensors in a std::map keyed by name (vit.h:88), so a name can only occur once; a caller-built list with a
// repeated name is rejected instead of silently taking the first
int check_unique_names(const vitb200_tensor *t, int n)
{
    std::map<std::string, int> seen;
    for (int i = 0; i < n; ++i)
    {
        if (!t[i].name || !t[i].data) return fail("tensor %d has a null name or data pointer", i);
        if (t[i].n_dims < 1 || t[i].n_dims > 4) return fail("tensor '%s' has %d dimensions", t[i].name, t[i].n_dims);
        if (seen.count(t[i].name)) return fail("duplicate tensor '%s' in model", t[i].name);
        seen[t[i].name] = i;
    }
    return 0;
}

int64_t dim_of(const vitb200_tensor *t, int i) { return i < t->n_dims ? t->ne[i] : 1; }

// the reference loader's shape check (vit.cpp:633-641): all four ggml extents must match the tensor the model declares
int check_shape(const vitb200_tensor *x, const std::string &name, int64_t e0, int64_t e1, int64_t e2, int64_t e3)
{
    if (dim_of(x, 0) != e0 || dim_of(x, 1) != e1 || dim_of(x, 2) != e2 || dim_of(x, 3) != e3)
        return fail("tensor '%s' has wrong shape in model file: got [%lld, %lld, %lld, %lld], expected [%lld, %lld, %lld, %lld]", name.c_str(),
                    (long long)dim_of(x, 0), (long long)dim_of(x, 1), (long long)dim_of(x, 2), (long long)dim_of(x, 3),
                    (long long)e0, (long long)e1, (long long)e2, (long long)e3);
    return 0;
}

int64_t nelem(const vitb200_tensor *t)
{
    int64_t n = 1;
    for (int i = 0; i < t->n_dims && i < 4; ++i) n *= t->ne[i];
    return n;
}

// f32 tensor with the reference's declared extents {e0, e1, e2, e3} (vit.cpp:510-574), NULL (with the error set) when it is missing or
// does not match
const vitb200_tensor *f32_tensor(const vitb200_tensor *t, int n, const std::string &name, int64_t e0, int64_t e1, int64_t e2, int64_t e3)
{
    const vitb200_tensor *x = find_tensor(t, n, name);
    if (!x) return fail("missing tensor '%s'", name.c_str()), nullptr;
    if (x->type != 0) return fail("tensor '%s' must be f32 (type %d)", name.c_str(), x->type), nullptr;
    const int64_t expect = e0 * e1 * e2 * e3;
    if (nelem(x) != expect)
        return fail("tensor '%s' has wrong size in model file: got %lld, expected %lld", name.c_str(), (long long)nelem(x), (long long)expect), nullptr;
    if (check_shape(x, name, e0, e1, e2, e3)) return nullptr;
    return x;
}

// f32 tensor uploaded as it is stored; `padded` >= the element count allocates a zero-filled tail (the classifier bias when
// num_classes is not a multiple of 4)
int upload_f32(vitb200_engine *e, const vitb200_tensor *t, int n, const std::string &name, int64_t e0, int64_t e1, int64_t e2, int64_t e3,
               float **dst, int64_t padded = 0)
{
    const vitb200_tensor *x = f32_tensor(t, n, name, e0, e1, e2, e3);
    if (!x) return 1;
    const int64_t expect = e0 * e1 * e2 * e3;
    if (dev_alloc(e, dst, (size_t)(padded > expect ? padded : expect))) return 1;
    CUDA_TRY(cudaMemcpy(*dst, x->data, (size_t)expect * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

// IEEE f32 -> f16 round-to-nearest-even on the host (upload-time conversions only)
uint16_t host_f32_to_f16(float f) { const __half h = __float2half_rn(f); uint16_t u; memcpy(&u, &h, 2); return u; }
float host_f16_to_f32(uint16_t u) { __half h; memcpy(&h, &u, 2); return __half2float(h); }

// The FP8 engine's weight quantisation: one scale for the whole tensor, sw = amax / 448 (1 when amax = 0), and
// q = e4m3_rn_satfinite(w (448 / amax)), from the f16 values the f16 engine would store.  Returns sw.
float quantize_e4m3(const uint16_t *w, size_t n, uint8_t *q)
{
    float amax = 0.f;
    for (size_t i = 0; i < n; ++i) amax = std::max(amax, std::fabs(host_f16_to_f32(w[i])));
    const float inv = amax > 0.f ? 448.f / amax : 1.f;
    for (size_t i = 0; i < n; ++i) q[i] = (uint8_t)__nv_cvt_float_to_fp8(host_f16_to_f32(w[i]) * inv, __NV_SATFINITE, __NV_E4M3);
    return amax > 0.f ? amax / 448.f : 1.f;
}

// ggml block formats of 32 weights (ggml-quants.h:11-47), keyed by ggml_type / file ftype (vit.cpp:645-672).
size_t quant_block_bytes(int type)
{
    switch (type)
    {
    case 2: return 18; // q4_0 { f16 d; u8 qs[16] }
    case 3: return 20; // q4_1 { f16 d; f16 m; u8 qs[16] }
    case 6: return 22; // q5_0 { f16 d; u8 qh[4]; u8 qs[16] }
    case 7: return 24; // q5_1 { f16 d; f16 m; u8 qh[4]; u8 qs[16] }
    case 8: return 34; // q8_0 { f16 d; i8 qs[32] }
    default: return 0;
    }
}

// One block -> 32 floats, the arithmetic of ggml's dequantize_row_q* (ggml-quants.c:1074-1185): low nibbles are elements
// 0..15, high nibbles 16..31, the q5 formats take their fifth bit from qh; the *_1 formats add the block minimum m.
void dequant_block(int type, const uint8_t *blk, float *y)
{
    uint16_t du = 0, mu = 0;
    memcpy(&du, blk, 2);
    const float d = host_f16_to_f32(du);
    if (type == 8)
    {
        const int8_t *q = (const int8_t *)(blk + 2);
        for (int i = 0; i < 32; ++i) y[i] = d * (float)q[i];
        return;
    }
    const bool has_min = type == 3 || type == 7, five = type == 6 || type == 7;
    float m = 0.f;
    if (has_min) { memcpy(&mu, blk + 2, 2); m = host_f16_to_f32(mu); }
    const uint8_t *p = blk + (has_min ? 4 : 2);
    uint32_t qh = 0;
    if (five) { memcpy(&qh, p, 4); p += 4; }
    for (int j = 0; j < 16; ++j)
    {
        int x0 = p[j] & 0x0F, x1 = p[j] >> 4;
        if (five)
        {
            x0 |= (int)(((qh >> j) << 4) & 0x10);
            x1 |= (int)((qh >> (j + 12)) & 0x10);
        }
        if (has_min) { y[j] = (float)x0 * d + m; y[j + 16] = (float)x1 * d + m; }
        else
        {
            const int off = five ? 16 : 8;
            y[j] = (float)(x0 - off) * d; y[j + 16] = (float)(x1 - off) * d;
        }
    }
}

// SwiGLU's fc1 (vitb200_arch.activation = 4) in the layout the EPI_BIAS_SWIGLU_F16 epilogue reads (gemm_wgmma.cuh): HF's [2 F] rows
// of row_elems values, x1 rows 0 .. F-1 then x2 rows, become [2 Fp] rows, Fp = round_up(F, 64): group g of 64 hidden units holds x1
// rows 64 g .. 64 g + 63 at 128 g and their x2 rows at 128 g + 64, rows past F zero.  Besides the epilogue this is the only code that
// knows the layout: the f16 and e4m3 weights, the bias and both GEMM test hooks go through it.
int swiglu_rows(int F) { return 2 * ((F + SWIGLU_GROUP - 1) / SWIGLU_GROUP * SWIGLU_GROUP); }

template <typename T>
std::vector<T> swiglu_interleave(const T *src, int F, size_t row_elems)
{
    std::vector<T> out((size_t)swiglu_rows(F) * row_elems, T(0));
    for (int f = 0; f < F; ++f)
        for (int half = 0; half < 2; ++half)
        {
            const size_t dst = (size_t)(2 * SWIGLU_GROUP * (f / SWIGLU_GROUP) + SWIGLU_GROUP * half + f % SWIGLU_GROUP);
            memcpy(&out[dst * row_elems], src + ((size_t)half * F + f) * row_elems, row_elems * sizeof(T));
        }
    return out;
}

// Weight matrix [n_out][n_in] -> device f16, row pitch padded to ld (zero filled), + its TMA descriptor.
//   type 1 (F16): used as stored -- the reference's own operand (ggml.c:1200-1236).
//   type 8 (Q8_0, blocks of {f16 d; int8 q[32]}, ggml-quants.h:42-46): dequantised once to f16(d * q).  The reference
//          multiplies int8 x dynamically quantised int8 activations (ggml-quants.c:3521); this W8A16 form stays within the
//          q8_0 noise floor of that path (SURVEY.md 7.4: 1.6e-2 either way); an int8 tensor-core path is future work.
//   types 2/3/6/7 (Q4_0, Q4_1, Q5_0, Q5_1): same treatment -- dequantised once with ggml's dequantize_row arithmetic and
//          rounded to f16 (exact for q4_0/q5_0 whenever d*q is a normal f16: a 5-bit integer times an f16).  The reference
//          dots them against activations quantised on the fly to q8_0/q8_1 (ggml.c type traits vec_dot_type).
//   type 0 (F32): rounded once to f16 (the reference keeps f32 weights AND f32 activations, ggml.c:1163-1198).
//   type 30 (BF16, GGUF containers): widened to f32, then as type 0.
// e4m3: the f16 values are quantised once more (quantize_e4m3) and only the e4m3 copy goes to the device.
// swiglu: SwiGLU's fc1, n_out = 2 F rows in HF's order; the f16 rows and the bias are interleaved (swiglu_interleave) before the e4m3
// quantisation, so the device holds swiglu_rows(F) rows.
int upload_linear(vitb200_engine *e, const vitb200_tensor *t, int n, const std::string &wname, const std::string &bname,
                  int n_out, int n_in, int ld, Linear *L, int conv_p = 0, bool e4m3 = false, bool swiglu = false)
{
    const vitb200_tensor *w = find_tensor(t, n, wname);
    if (!w) return fail("missing tensor '%s'", wname.c_str());
    if (w->type != 0 && w->type != 1 && w->type != 30 && quant_block_bytes(w->type) == 0)
        return fail("tensor '%s': weight type %d is not supported (f32, f16, bf16, q4_0, q4_1, q5_0, q5_1, q8_0 only)", wname.c_str(), w->type);
    if (nelem(w) != (int64_t)n_out * n_in) return fail("tensor '%s' has wrong size in model file: got %lld, expected %lld", wname.c_str(), (long long)nelem(w), (long long)n_out * n_in);
    if (conv_p > 0) { if (check_shape(w, wname, conv_p, conv_p, n_in / (conv_p * conv_p), n_out)) return 1; } // [P, P, C, D], vit.cpp:515
    else if (check_shape(w, wname, n_in, n_out, 1, 1)) return 1;                                             // [in, out], vit.cpp:531-543
    if (quant_block_bytes(w->type) && n_in % 32 != 0) return fail("tensor '%s': quantised rows must be a multiple of 32", wname.c_str());
    const vitb200_tensor *swiglu_b = swiglu ? f32_tensor(t, n, bname, n_out, 1, 1, 1) : nullptr;
    if (swiglu && !swiglu_b) return 1;
    const int F = n_out / 2;
    const void *src = w->data;
    std::vector<uint16_t> conv;
    if (w->type != 1)
    {
        conv.resize((size_t)n_out * n_in);
        if (w->type == 0)
        {
            // Rounded once to f16.  A bf16 checkpoint widened to f32 (the only way this container can carry bf16,
            // BASELINE.json configs[2]) converts EXACTLY for every weight with |w| >= 2^-14 (8-bit mantissa fits in 11).
            // Keeping such weights as bf16 would need bf16 activations too (one wgmma takes one operand type), and bf16
            // activations cost 5e-3 parity (SURVEY.md 7.4).
            const float *f = (const float *)w->data;
            for (size_t i = 0; i < conv.size(); ++i) conv[i] = host_f32_to_f16(f[i]);
        }
        else if (w->type == 30)
        {
            // BF16 tensors (GGUF containers only): widened to f32 (exact) and rounded to f16 like the f32 case above
            const uint16_t *h = (const uint16_t *)w->data;
            for (size_t i = 0; i < conv.size(); ++i)
            {
                const uint32_t u = (uint32_t)h[i] << 16;
                float f;
                memcpy(&f, &u, 4);
                conv[i] = host_f32_to_f16(f);
            }
        }
        else
        {
            const uint8_t *blk = (const uint8_t *)w->data;
            const size_t nb = conv.size() / 32, bs = quant_block_bytes(w->type);
            float y[32];
            for (size_t b = 0; b < nb; ++b)
            {
                dequant_block(w->type, blk + b * bs, y);
                for (int i = 0; i < 32; ++i) conv[b * 32 + i] = host_f32_to_f16(y[i]);
            }
        }
        src = conv.data();
    }
    std::vector<uint16_t> inter;
    if (swiglu)
    {
        inter = swiglu_interleave((const uint16_t *)src, F, (size_t)n_in);
        src = inter.data();
        n_out = swiglu_rows(F);
    }
    L->n_out = n_out; L->n_in = n_in; L->ld = ld;
    if (e4m3)
    {
        std::vector<uint8_t> q((size_t)n_out * n_in);
        L->w_scale = quantize_e4m3((const uint16_t *)src, q.size(), q.data());
        if (dev_alloc(e, &L->w8, (size_t)n_out * ld)) return 1;
        CUDA_TRY(cudaMemcpy2D(L->w8, (size_t)ld, q.data(), (size_t)n_in, (size_t)n_in, (size_t)n_out, cudaMemcpyHostToDevice));
    }
    else
    {
        if (dev_alloc(e, &L->w, (size_t)n_out * ld)) return 1;
        CUDA_TRY(cudaMemset(L->w, 0, (size_t)n_out * ld * sizeof(__half)));
        CUDA_TRY(cudaMemcpy2D(L->w, (size_t)ld * 2, src, (size_t)n_in * 2, (size_t)n_in * 2, (size_t)n_out, cudaMemcpyHostToDevice));
    }
    if (swiglu)
    {
        const std::vector<float> b = swiglu_interleave((const float *)swiglu_b->data, F, 1);
        if (dev_alloc(e, &L->b, b.size())) return 1;
        CUDA_TRY(cudaMemcpy(L->b, b.data(), b.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    // conv bias is declared [1, 1, D] (vit.cpp:516), every other bias [n_out]; the tail up to a multiple of 4 stays zero
    else if (conv_p > 0 ? upload_f32(e, t, n, bname, 1, 1, n_out, 1, &L->b) : upload_f32(e, t, n, bname, n_out, 1, 1, 1, &L->b, (n_out + 3) / 4 * 4)) return 1;
    const cuuint64_t cols = (cuuint64_t)ld, rows = (cuuint64_t)n_out;
    if (e4m3) return make_tmap(&L->tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, L->w8, {cols, rows}, {cols}, {2 * GEMM_BK, GEMM_BN});
    return make_tmap(&L->tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, L->w, {cols, rows}, {2 * cols}, {GEMM_BK, GEMM_BN});
}

// the largest dynamic shared memory one CTA may opt in to on sm_90 (227 KB)
constexpr int kSmemOptinMax = 232448;
// dynamic shared memory the soft-max kernel may use for its working row (the per-CTA limit minus its static arrays)
constexpr size_t kSoftmaxSmemMax = kSmemOptinMax - 1024;

enum ProfKind { PK_PATCH = 0, PK_QKV, PK_PROJ, PK_FC1, PK_FC2, PK_HEAD, PK_ATTN, PK_LN, PK_POOL, PK_COUNT };

struct ProfScope
{
    vitb200_engine *e;
    cudaStream_t s;
    cudaEvent_t b = nullptr;
    ProfScope(vitb200_engine *e_, int kind, double flops, cudaStream_t s_) : e(e_), s(s_)
    {
        if (!e || !e->profile) { e = nullptr; return; }
        cudaEvent_t a = nullptr;
        auto get = [&](cudaEvent_t *ev) {
            if (!e->event_pool.empty()) { *ev = e->event_pool.back(); e->event_pool.pop_back(); }
            else cudaEventCreate(ev);
        };
        get(&a);
        get(&b);
        cudaEventRecord(a, s);
        e->prof.push_back({kind, a, b, flops});
    }
    ~ProfScope()
    {
        if (e) cudaEventRecord(b, s);
    }
};

// Launch attributes of `launch`, or-ed together: programmatic dependent launch, and clusters of two CTAs
enum : unsigned { LAUNCH_PLAIN = 0, LAUNCH_PDL = 1, LAUNCH_CLUSTER2 = 2 };

struct LaunchConfig
{
    cudaLaunchConfig_t cfg{};
    cudaLaunchAttribute attr[2];
    LaunchConfig(dim3 grid, dim3 block, size_t smem, cudaStream_t s, unsigned attrs)
    {
        cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s; cfg.attrs = attr;
        if (attrs & LAUNCH_CLUSTER2)
        {
            cudaLaunchAttribute &a = attr[cfg.numAttrs++];
            a.id = cudaLaunchAttributeClusterDimension;
            a.val.clusterDim.x = 2; a.val.clusterDim.y = 1; a.val.clusterDim.z = 1;
        }
        if (attrs & LAUNCH_PDL)
        {
            cudaLaunchAttribute &a = attr[cfg.numAttrs++];
            a.id = cudaLaunchAttributeProgrammaticStreamSerialization;
            a.val.programmaticStreamSerializationAllowed = 1;
        }
    }
    LaunchConfig(const LaunchConfig &) = delete; // cfg.attrs points into this object
};

// Opts `kern` in to `bytes` of dynamic shared memory on the current device, and raises that limit when a later launch needs more.
// The attribute belongs to the process and device, not to an engine, so one table serves every engine on every host thread.  It is
// set on a kernel's first eager run, never inside a graph capture (run_graphed captures an argument set's second call only).
// cluster_cfg: also counts, once, the clusters of that launch configuration that fit on the device at a time, into *clusters.
struct KernelAttr
{
    int smem = 0, clusters = 0;
};
std::mutex g_attr_mutex;
std::map<std::pair<const void *, int>, KernelAttr> g_attr;

int smem_optin(const void *kern, int bytes, const cudaLaunchConfig_t *cluster_cfg = nullptr, int *clusters = nullptr)
{
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_attr_mutex);
    KernelAttr &a = g_attr[{kern, dev}];
    if (bytes > a.smem)
    {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        if (cluster_cfg) CUDA_TRY(cudaOccupancyMaxActiveClusters(&a.clusters, kern, cluster_cfg));
        a.smem = bytes;
    }
    if (clusters) *clusters = a.clusters;
    return 0;
}

// Every kernel of the engine and of the test hooks is launched here: with the attributes `attrs` selects, opted in through smem_optin
// when it needs more than the default 48 KB of dynamic shared memory, checked, and counted in e->launches.
// LAUNCH_PDL lets the kernel start while the kernel before it on the stream is still running.  Only a kernel that calls
// griddepcontrol.wait (ptx.cuh) before it touches memory its predecessor writes is correct under it: the GEMM, the attention kernels
// and the LayerNorms, whose barrier init and descriptor prefetch then run on the SMs the previous kernel has already left.
template <typename... KArgs, typename... Args>
int launch(vitb200_engine *e, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, unsigned attrs, Args &&...args)
{
    if (smem > 48 * 1024 && smem_optin((const void *)kern, (int)smem)) return 1;
    LaunchConfig c(grid, block, smem, s, attrs);
    const cudaError_t err = cudaLaunchKernelEx(&c.cfg, kern, std::forward<Args>(args)...);
    if (err != cudaSuccess)
    {
        (void)cudaGetLastError();
        return fail("kernel launch (grid %u x %u, block %u, %zu B shared memory) failed: %s", grid.x, grid.y, block.x, smem, cudaGetErrorString(err));
    }
    e->launches++;
    return 0;
}

template <int EPI, int STAGES, int OP = GEMM_OP_F16>
int launch_gemm_t(vitb200_engine *e, const CUtensorMap &tmA, const CUtensorMap &tmB, const GemmParams &p, cudaStream_t s)
{
    using Cfg = GemmCfg<STAGES>;
    auto kern = gemm_wgmma_kernel<EPI, STAGES, OP>;
    // clusters of two CTAs that share the A tile (multicast)
    constexpr unsigned attrs = LAUNCH_CLUSTER2 | LAUNCH_PDL;
    int max_clusters = 0;
    {
        const LaunchConfig c(dim3(2), dim3((unsigned)Cfg::kThreads), Cfg::SMEM_BYTES, s, attrs);
        if (smem_optin((const void *)kern, Cfg::SMEM_BYTES, &c.cfg, &max_clusters)) return 1;
    }
    if (max_clusters < 1)
    {
        int dev = 0;
        CUDA_TRY(cudaGetDevice(&dev));
        return fail("GEMM: no cluster of two CTAs fits on device %d", dev);
    }
    // the staged epilogues' TMA maps over exactly M rows and N columns of the output (and of the residual), encoded per launch:
    // a captured graph keeps them by value
    CUtensorMap tmO{}, tmX{};
    if constexpr (gemm_epi(EPI).staged)
    {
        using St = GemmStage<EPI, STAGES>;
        // SwiGLU stores F columns of the N / 2 it computes
        const cuuint64_t M = (cuuint64_t)p.M, N = (cuuint64_t)(St::kSwiglu ? p.F : p.N), ldo = (cuuint64_t)p.ldo;
        auto out_map = [&](CUtensorMap *m, const void *ptr) -> int {
            if (!St::kF16) return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, ptr, {N, M}, {4 * ldo}, {32, 64});
            if (p.headmajor)
            {
                // [N / 64 head planes][plane_rows][64], as the attention reads it
                if (p.N % 64 != 0) return fail("GEMM: head-major output needs N %% 64 == 0 (N = %d)", p.N);
                return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ptr, {64, M, N / 64}, {128, 128 * (cuuint64_t)p.plane_rows}, {64, 64, 1});
            }
            return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ptr, {N, M}, {2 * ldo}, {64, 64});
        };
        if (out_map(&tmO, p.out)) return 1;
        if (gemm_epi(EPI).hilo && out_map(&tmX, p.out2)) return 1;
        if (gemm_epi(EPI).resid && out_map(&tmX, p.resid)) return 1;
    }
    // persistent: as many clusters as fit at once, each walking the pairs of column tiles cluster, cluster + clusters, ...
    const int pairs = ((p.M + GEMM_BM - 1) / GEMM_BM) * ((p.N + 2 * GEMM_BN - 1) / (2 * GEMM_BN));
    return launch(e, kern, dim3(2u * (unsigned)std::min(pairs, max_clusters)), dim3((unsigned)Cfg::kThreads), Cfg::SMEM_BYTES, s, attrs, tmA, tmB,
                  tmO, tmX, p);
}

// The instantiation for epilogue epi, found by walking the ids from EPI at compile time (e4m3: the ones gemm_epi gives an e4m3 form)
template <int OP, int EPI = 0>
int launch_gemm_dispatch(vitb200_engine *e, int epi, const CUtensorMap &tmA, const CUtensorMap &tmB, const GemmParams &p, cudaStream_t s)
{
    if constexpr (EPI == GEMM_EPI_END)
        return fail(OP == GEMM_OP_E4M3 ? "no e4m3 GEMM instantiation for epilogue=%d" : "no GEMM instantiation for epilogue=%d", epi);
    else
    {
        if constexpr (gemm_epi(EPI).valid && (OP == GEMM_OP_F16 || gemm_epi(EPI).e4m3))
            if (epi == EPI) return p.K >= GEMM_DEEP_K ? launch_gemm_t<EPI, 6, OP>(e, tmA, tmB, p, s) : launch_gemm_t<EPI, 5, OP>(e, tmA, tmB, p, s);
        return launch_gemm_dispatch<OP, EPI + 1>(e, epi, tmA, tmB, p, s);
    }
}

// tmB: the weight map, box = one k-block x GEMM_BN rows.  e4m3: A and W are e4m3 maps, p.a_scale / p.w_scale their
// scales; the f16-output epilogues only (qkv and fc1 of the FP8 engine)
int launch_gemm(vitb200_engine *e, int epi, const CUtensorMap &tmA, const CUtensorMap &tmB, const GemmParams &p, cudaStream_t s, bool e4m3 = false)
{
    if (p.N % 4 != 0) return fail("GEMM: N = %d is not a multiple of 4", p.N);
    if (epi == EPI_BIAS_SWIGLU_F16 && (p.F < 1 || p.N != swiglu_rows(p.F)))
        return fail("SwiGLU GEMM: N = %d is not the interleaved width %d of F = %d", p.N, p.F < 1 ? 0 : swiglu_rows(p.F), p.F);
    if (e4m3 && !p.a_scale) return fail("e4m3 GEMM: no A scales");
    return e4m3 ? launch_gemm_dispatch<GEMM_OP_E4M3>(e, epi, tmA, tmB, p, s) : launch_gemm_dispatch<GEMM_OP_F16>(e, epi, tmA, tmB, p, s);
}

// The patchify kernel for patch size P and C input channels, NULL for a size it has none for (vitb200_create rejects those)
using PatchifyKernel = void (*)(const float *, __half *, int, int, int, int);
PatchifyKernel patchify_kernel(int P, int C)
{
    if (C == 1) return P == 8 ? patchify_f16_kernel<8, 1> : P == 16 ? patchify_f16_kernel<16, 1> : nullptr;
    switch (P)
    {
    case 8: return patchify_f16_kernel<8>;
    case 14: return patchify_f16_kernel<14>;
    case 16: return patchify16_warp_kernel;
    case 32: return patchify_f16_kernel<32>;
    }
    return nullptr;
}
inline bool patchify_supports(int P, int C) { return patchify_kernel(P, C) != nullptr; }
// Whether the patchify kernel of patch size P reads pixel rows in 16-byte loads (patchify16_warp_kernel, and patchify_f16_kernel's
// float4 path, taken when P % 4 == 0): the row starts (b S + y) S C floats must then be 16-byte aligned, i.e. img_size % 4 == 0.  A
// patch that divides img_size guarantees it; the floor grid of pools 2 and 3 does not.
inline bool patchify_reads_16b(int P) { return P % 4 == 0; }
inline const char *patchify_sizes(int C) { return C == 1 ? "8, 16" : "8, 14, 16, 32"; }

int launch_patchify(vitb200_engine *e, const float *img, __half *A, int B, cudaStream_t s)
{
    const PatchifyKernel kern = patchify_kernel(e->hp.patch_size, e->C);
    if (!kern) return fail("%d-channel input: patch size %d not supported (%s)", e->C, e->hp.patch_size, patchify_sizes(e->C));
    if (kern == patchify16_warp_kernel)
    {
        const int n_patches = B * e->G * e->G; // one warp per patch, grid-stride over a few waves
        return launch(e, kern, dim3(std::min((n_patches + 7) / 8, e->num_sms * 16)), dim3(256), 0, s, LAUNCH_PLAIN, img, A, n_patches,
                      e->hp.img_size, e->G, e->KPp);
    }
    const long long total = (long long)B * e->G * e->hp.patch_size * e->G;
    return launch(e, kern, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, LAUNCH_PLAIN, img, A, B, e->hp.img_size, e->G, e->KPp);
}

// The row-per-warp kernel: the LayerNorms the bulk-copy kernel below does not take (pooled rows, hidden sizes that are not a multiple
// of 128) and, with an f32 / bf16 output or NORM = false, the encoder features.  rows_per_group <= 0: all rows are one group.
// OutT = __nv_fp8_e4m3: y_scale receives the per-row scales.  A lane holds up to LN_ROWS_MAX_V float4 of its row, which bounds the
// hidden size the engine accepts.
constexpr int LN_ROWS_MAX_V = 16;
constexpr int LN_MAX_HIDDEN = LN_ROWS_MAX_V * 128;
// register tokens a model may have (vitb200_arch.reg_tokens; DINOv2 with registers has 4)
constexpr int VB_MAX_REG_TOKENS = 16;

// Token rows in front of an image's patch rows: the class token and the registers, or none with SigLIP's pools (vitb200_arch.pool 2, 3)
int prefix_rows(const vitb200_arch &a) { return a.pool >= 2 ? 0 : 1 + a.reg_tokens; }

// Launches kernel(std::integral_constant<int, MAXV>), a kernel holding rows in registers, MAXV = 4, 8 or LN_ROWS_MAX_V as D needs
template <class Kernel, typename... Args>
int launch_rows_kernel(vitb200_engine *e, Kernel kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args &&...args)
{
    const int D = e->hp.hidden_size;
    if (D > LN_MAX_HIDDEN) return fail("hidden size %d not supported (max %d)", D, LN_MAX_HIDDEN);
    const auto kern = D <= 4 * 128 ? kernel(std::integral_constant<int, 4>())
                    : D <= 8 * 128 ? kernel(std::integral_constant<int, 8>()) : kernel(std::integral_constant<int, LN_ROWS_MAX_V>());
    return launch(e, kern, grid, block, smem, s, LAUNCH_PDL, std::forward<Args>(args)...);
}

template <bool NORM, typename OutT>
int launch_layernorm_rows(vitb200_engine *e, const float *x, size_t x_row_stride, const float *w, const float *b, OutT *y, int rows,
                          cudaStream_t s, int rows_per_group, size_t group_stride, float *y_scale = nullptr)
{
    if (rows_per_group <= 0) rows_per_group = rows > 0 ? rows : 1; // one group: plain consecutive rows
    const int threads = 256, rows_per_block = threads / 32;
    const int blocks = (rows + rows_per_block - 1) / rows_per_block;
    return launch_rows_kernel(e, [](auto V) { return layernorm_f16_kernel<V(), OutT, NORM>; }, dim3(blocks), dim3(threads), 0, s, x, x_row_stride,
                              rows_per_group, group_stride, w, b, y, rows, e->hp.hidden_size, e->hp.eps, y_scale);
}

// OutT = __half: the f16 A operand; __nv_fp8_e4m3: the FP8 engine's e4m3 A operand and its row scales y_scale
template <typename OutT = __half>
int launch_layernorm(vitb200_engine *e, const float *x, size_t x_row_stride, const float *w, const float *b, OutT *y, int rows, cudaStream_t s,
                     int rows_per_group = 0, size_t group_stride = 0, float *y_scale = nullptr)
{
    const int D = e->hp.hidden_size;
    // block LayerNorms (all rows consecutive): the persistent bulk-copy kernel
    // (two CTAs per SM must fit: with one, as for D = 1024, it is slower than the row-per-warp kernel -- 4.98 against 3.9 ms per ViT-L forward)
    if (rows_per_group <= 0 && x_row_stride == (size_t)D && D % 128 == 0 && 2 * (layernorm_tma_smem_bytes(D) + 1024) <= 233472 && rows >= 8)
    {
        const int smem = layernorm_tma_smem_bytes(D);
        const int nblk = (rows + LN_TMA_ROWS - 1) / LN_TMA_ROWS;
        const int grid = std::min(nblk, 2 * e->num_sms);
        // by float4 per lane, D / 128 (at most 7 here: two CTAs per SM hold rows of up to 896 floats)
        using Kern = decltype(&layernorm_tma_kernel<1, OutT>);
        const Kern kernels[8] = {layernorm_tma_kernel<1, OutT>, layernorm_tma_kernel<2, OutT>, layernorm_tma_kernel<3, OutT>, layernorm_tma_kernel<4, OutT>,
                                 layernorm_tma_kernel<5, OutT>, layernorm_tma_kernel<6, OutT>, layernorm_tma_kernel<7, OutT>, layernorm_tma_kernel<8, OutT>};
        return launch(e, kernels[D / 128 - 1], dim3(grid), dim3(LN_TMA_THREADS), (size_t)smem, s, LAUNCH_PDL, x, w, b, y, rows, e->hp.eps, y_scale);
    }
    return launch_layernorm_rows<true>(e, x, x_row_stride, w, b, y, rows, s, rows_per_group, group_stride, y_scale);
}

// The pre-norm: the row-per-warp LayerNorm in place on `rows` consecutive f32 rows of x
int launch_layernorm_inplace(vitb200_engine *e, float *x, const float *w, const float *b, int rows, cudaStream_t s)
{
    const int threads = 256, blocks = (rows + threads / 32 - 1) / (threads / 32);
    return launch_rows_kernel(e, [](auto V) { return layernorm_inplace_kernel<V()>; }, dim3(blocks), dim3(threads), 0, s, x, w, b, rows,
                              e->hp.hidden_size, e->hp.eps);
}

// DINOv2's classifier input (vitb200_arch.pool = 1): per image, [LN(token 0) || mean of LN(patch rows)] into y [B][2 D] (NORM = false:
// the rows as they are), rows 1 .. reg_tokens left out.  SigLIP's (pool = 3, no class token): the mean of LN(every row) into y [B][D]
template <bool NORM, typename OutT>
int launch_pool(vitb200_engine *e, OutT *y, int B, cudaStream_t s)
{
    const int D = e->hp.hidden_size;
    return launch_rows_kernel(e, [](auto V) { return cls_patch_mean_kernel<V(), OutT, NORM>; }, dim3(B), dim3(POOL_WARPS * 32),
                              (size_t)POOL_WARPS * D * sizeof(float), s, e->X, e->N, prefix_rows(e->arch), e->norm_w, e->norm_b, y, D, e->hp.eps);
}

// The fc1 epilogue of the model's MLP activation (vitb200_arch.activation)
int fc1_epilogue(const vitb200_engine *e)
{
    switch (e->arch.activation)
    {
    case 1: return EPI_BIAS_GELU_ERF_F16;
    case 2: return EPI_BIAS_QUICK_GELU_F16;
    case 3: return EPI_BIAS_GELU_PYTORCH_TANH_F16;
    case 4: return EPI_BIAS_SWIGLU_F16;
    }
    return EPI_BIAS_GELU_F16;
}

// The residual epilogue of proj and fc2: with LayerScale (vitb200_arch.layer_scale) the branch is scaled by gamma before the add
int resid_epilogue(const vitb200_engine *e) { return e->arch.layer_scale ? EPI_BIAS_SCALE_RESID_F32 : EPI_BIAS_RESID_F32; }

// Attention kernels (the `kernel` argument of vitb200_test_attention): ATT_MMA8 = the two-pass mma.sync kernel with 8 warps per CTA, any
// token count; ATT_WGMMA = the split-precision wgmma kernel the engine picks for N <= 224: attention_wgmma_persistent_kernel up to
// ATTP_KEYS tokens (not causal), attention_wgmma_kernel beyond; ATT_WGMMA_HEAD = attention_wgmma_kernel (one CTA per problem) at any
// N <= 224; ATT_MMA16 = the mma.sync kernel with 16 warps, 128 < N <= 640.  The engine uses the wgmma kernels up to 224 tokens, 16
// warps up to 640 and 8 beyond.  Head dim 80 has one kernel, ATT_MMA80 = attention_rowmajor_kernel<80> (split precision up to 224
// tokens, f16 operands beyond), which ATT_AUTO picks for it.  Head dim 72 runs attention_rowmajor_kernel<72> alike, through ATT_AUTO
// only.
enum { ATT_AUTO = 0, ATT_MMA8 = 1, ATT_WGMMA = 2, ATT_MMA16 = 3, ATT_MMA80 = 4, ATT_WGMMA_HEAD = 5 };
constexpr int ATT_MAX_KEYS_16 = 640;

// q / k / v tensor maps (hi and lo halves) of the wgmma attention over planes of max_batch * N token rows
int make_attention_maps(vitb200_engine *e)
{
    // the head-major buffer [3 H planes][max_batch][N][64], seen as 3 H max_batch slices of N rows: slice p max_batch + b is image b of
    // plane p.  A box is 64 query rows or ATTW_KEYS key rows of one slice; rows past N are out of bounds and read as zero, never as
    // the next image's rows.
    const cuuint64_t N = (cuuint64_t)e->N, slices = 3 * (cuuint64_t)e->hp.num_attention_heads * (cuuint64_t)e->max_batch;
    auto map = [&](CUtensorMap *m, const __half *ptr, cuuint32_t box_rows) {
        return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ptr, {64, N, slices}, {128, 128 * N}, {64, box_rows, 1});
    };
    if (map(&e->tmQ, e->QKV16, 64) || map(&e->tmKV, e->QKV16, ATTW_KEYS) || map(&e->tmQl, e->QKV16L, 64) || map(&e->tmKVl, e->QKV16L, ATTW_KEYS))
        return 1;
    if (map(&e->tmKVp, e->QKV16, ATTP_ROWS) || map(&e->tmKVpl, e->QKV16L, ATTP_ROWS)) return 1;
    return 0;
}

static_assert(attention_persistent_smem_bytes() <= kSmemOptinMax, "two K V buffers fit one SM's shared memory");

// per_head: attention_wgmma_kernel even where the persistent kernel would run (the test hooks compare the two); probe: the kernels'
// phase probe into g_attn_probe (vitb200_test_attention_phases, not causal)
int launch_attention_wgmma(vitb200_engine *e, int B, cudaStream_t s, bool per_head = false, bool probe = false)
{
    const int H = e->hp.num_attention_heads;
    const bool causal = e->text && e->text_arch.causal;
    if (!per_head && !causal && e->N <= ATTP_KEYS)
        return launch(e, probe ? attention_wgmma_persistent_kernel<true> : attention_wgmma_persistent_kernel<false>,
                      dim3(std::min(B * H, e->num_sms)), dim3(ATTP_THREADS), (size_t)attention_persistent_smem_bytes(), s, LAUNCH_PDL, e->tmKVp, e->tmKVpl,
                      static_cast<const __half *>(e->QKV16), static_cast<const __half *>(e->QKV16L), e->A16, e->N, e->hp.hidden_size, H, e->max_batch, B * H, 1.0f / sqrtf((float)(e->hp.hidden_size / H)));
    const auto kern = causal ? attention_wgmma_kernel<true> : probe ? attention_wgmma_kernel<false, true> : attention_wgmma_kernel<false>;
    return launch(e, kern, dim3(B * H), dim3(ATTW_THREADS), (size_t)attention_wgmma_smem_bytes(), s, LAUNCH_PDL, e->tmQ, e->tmKV, e->tmQl,
                  e->tmKVl, e->A16, e->N, e->hp.hidden_size, H, e->max_batch, 1.0f / sqrtf((float)(e->hp.hidden_size / H)));
}

// The mma.sync kernels hold K and V of one (image, head) problem in shared memory: N tokens padded to whole key chunks, 64 f16 each.
// That bounds the token count the engine accepts.
constexpr int attention_smem_bytes(int N) { return 2 * ((N + ATT_KC - 1) / ATT_KC * ATT_KC) * 128; }
constexpr int ATT_MAX_TOKENS = kSmemOptinMax / (2 * 128) / ATT_KC * ATT_KC;
static_assert(attention_smem_bytes(ATT_MAX_TOKENS) <= kSmemOptinMax && attention_smem_bytes(ATT_MAX_TOKENS + 1) > kSmemOptinMax);

// attention_rowmajor_kernel holds K and V (and, split, their lo halves) of one problem in rows of att_row_bytes(hd), N padded to whole
// key chunks.  Its f16 form bounds the token count of a head-dim-80 or -72 model; the split form runs up to ATTW_KEYS tokens.
constexpr int attention_rm_smem_bytes(int hd, int N, bool split) { return (split ? 4 : 2) * ((N + ATT_KC - 1) / ATT_KC * ATT_KC) * att_row_bytes(hd); }
constexpr int attention_hd80_smem_bytes(int N, bool split) { return attention_rm_smem_bytes(ATT80_HD, N, split); }
constexpr int ATT80_MAX_TOKENS = kSmemOptinMax / (2 * ATT80_ROW_BYTES) / ATT_KC * ATT_KC;
static_assert(attention_hd80_smem_bytes(ATT80_MAX_TOKENS, false) <= kSmemOptinMax &&
              attention_hd80_smem_bytes(ATT80_MAX_TOKENS + 1, false) > kSmemOptinMax);
static_assert(attention_hd80_smem_bytes(ATTW_KEYS, true) <= kSmemOptinMax);
// head dim 72: 2 x 144 B per padded key in the f16 form, 800 tokens (So400m at 384 px: 729 tokens, padded to 736, 211 968 B)
constexpr int ATT72_MAX_TOKENS = kSmemOptinMax / (2 * att_row_bytes(ATT72_HD)) / ATT_KC * ATT_KC;
static_assert(ATT72_MAX_TOKENS == 800 && attention_rm_smem_bytes(ATT72_HD, ATT72_MAX_TOKENS, false) <= kSmemOptinMax &&
              attention_rm_smem_bytes(ATT72_HD, ATT72_MAX_TOKENS + 1, false) > kSmemOptinMax);
static_assert(attention_rm_smem_bytes(ATT72_HD, ATTW_KEYS, true) <= kSmemOptinMax);

int head_dim(const vitb200_engine *e) { return e->hp.hidden_size / e->hp.num_attention_heads; }

// the most tokens an image engine of head dim hd accepts
constexpr int max_tokens(int hd) { return hd == ATT80_HD ? ATT80_MAX_TOKENS : hd == ATT72_HD ? ATT72_MAX_TOKENS : ATT_MAX_TOKENS; }

// head dims 80 and 72: split precision exactly when the qkv GEMM writes lo halves (N <= ATTW_KEYS), 8 warps; f16 operands with 16 warps
template <int HD>
int launch_attention_rowmajor(vitb200_engine *e, int B, cudaStream_t s)
{
    const int N = e->N, D = e->hp.hidden_size, H = e->hp.num_attention_heads;
    const int Npad = (N + ATT_KC - 1) / ATT_KC * ATT_KC;
    const bool split = e->QKV16L != nullptr;
    if (split && N > ATTW_KEYS) return fail("split-precision head-dim-%d attention needs N <= %d (got %d)", HD, ATTW_KEYS, N);
    const int smem = attention_rm_smem_bytes(HD, N, split);
    if (smem > kSmemOptinMax)
        return fail("attention: %d tokens do not fit in shared memory (max %d at head dim %d)", N, max_tokens(HD), HD);
    const float scale = 1.0f / sqrtf((float)HD);
    if (split)
        return launch(e, attention_rowmajor_kernel<HD, 8, true>, dim3(B * H), dim3(8 * 32), (size_t)smem, s, LAUNCH_PDL, e->QKV16, e->QKV16L,
                      e->A16, N, D, H, Npad, scale);
    return launch(e, attention_rowmajor_kernel<HD, 16, false>, dim3(B * H), dim3(16 * 32), (size_t)smem, s, LAUNCH_PDL, e->QKV16,
                  static_cast<const __half *>(nullptr), e->A16, N, D, H, Npad, scale);
}

template <int NW>
int launch_attention_t(vitb200_engine *e, int B, cudaStream_t s)
{
    const int N = e->N, D = e->hp.hidden_size, H = e->hp.num_attention_heads;
    const int Npad = (N + ATT_KC - 1) / ATT_KC * ATT_KC;
    const int smem = attention_smem_bytes(N);
    if (smem > kSmemOptinMax) return fail("attention: %d tokens do not fit in shared memory (max %d)", N, ATT_MAX_TOKENS);
    return launch(e, attention_kernel<NW>, dim3(B * H), dim3(NW * 32), (size_t)smem, s, LAUNCH_PDL, e->QKV16, (size_t)e->max_batch * N, e->A16,
                  N, D, H, Npad, 1.0f / sqrtf((float)(D / H)));
}

int launch_attention(vitb200_engine *e, int B, cudaStream_t s, int kernel = ATT_AUTO, bool probe = false)
{
    if (head_dim(e) == ATT80_HD)
    {
        if (kernel != ATT_AUTO && kernel != ATT_MMA80) return fail("attention kernel %d does not run head dim 80", kernel);
        return launch_attention_rowmajor<ATT80_HD>(e, B, s);
    }
    if (head_dim(e) == ATT72_HD)
    {
        if (kernel != ATT_AUTO) return fail("attention kernel %d does not run head dim 72", kernel);
        return launch_attention_rowmajor<ATT72_HD>(e, B, s);
    }
    if (kernel == ATT_MMA80) return fail("attention kernel %d runs head dim 80 only", kernel);
    if (kernel == ATT_AUTO) kernel = e->N <= ATTW_KEYS ? ATT_WGMMA : (e->N <= ATT_MAX_KEYS_16 ? ATT_MMA16 : ATT_MMA8);
    if (kernel == ATT_WGMMA || kernel == ATT_WGMMA_HEAD) return launch_attention_wgmma(e, B, s, kernel == ATT_WGMMA_HEAD, probe);
    if (probe) return fail("the phase probe runs in the wgmma kernels only");
    if (e->QKV16L) return fail("split-precision attention runs in the wgmma kernel (N <= %d)", ATTW_KEYS);
    if (kernel == ATT_MMA16) return launch_attention_t<16>(e, B, s);
    return launch_attention_t<8>(e, B, s);
}

// The attention-pooling head's attention (attention_pool_kernel): the probe query q [D] f32 against the k | v of B images, N = P key rows
// each -> out [B][D] f16.  kv: head-major planes [2 H][max_batch * N][64] f16 at head dim 64, row-major [B * N][2 D] at head dim 72.
int launch_attention_pool(vitb200_engine *e, const float *q, const __half *kv, __half *out, int B, cudaStream_t s)
{
    const int P = e->N, H = e->hp.num_attention_heads;
    return launch(e, head_dim(e) == ATT72_HD ? attention_pool_kernel<ATT72_HD> : attention_pool_kernel<64>, dim3(B * H), dim3(APOOL_THREADS),
                  (size_t)P * sizeof(float), s, LAUNCH_PLAIN, kv, (size_t)e->max_batch * P, q, out, P, H);
}

// D2H helpers for the debug taps
int tap_f32(float *dst, const float *src, size_t n, cudaStream_t s)
{
    if (!dst) return 0;
    CUDA_TRY(cudaStreamSynchronize(s));
    CUDA_TRY(cudaMemcpy(dst, src, n * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
}
int tap_f16(float *dst, const __half *src, size_t n, cudaStream_t s, const __half *lo = nullptr)
{
    if (!dst) return 0;
    CUDA_TRY(cudaStreamSynchronize(s));
    std::vector<__half> tmp(n);
    CUDA_TRY(cudaMemcpy(tmp.data(), src, n * sizeof(__half), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i) dst[i] = __half2float(tmp[i]);
    if (lo) // split-precision tensor: value = hi + lo
    {
        CUDA_TRY(cudaMemcpy(tmp.data(), lo, n * sizeof(__half), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n; ++i) dst[i] += __half2float(tmp[i]);
    }
    return 0;
}

// debug tap of e4m3 rows with per-row scales (the FP8 engine's LayerNorm outputs): q * scale in f32
int tap_e4m3(float *dst, const uint8_t *q, const float *scale, size_t rows, size_t cols, cudaStream_t s)
{
    if (!dst) return 0;
    CUDA_TRY(cudaStreamSynchronize(s));
    std::vector<uint8_t> tq(rows * cols);
    std::vector<float> ts(rows);
    CUDA_TRY(cudaMemcpy(tq.data(), q, tq.size(), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(ts.data(), scale, rows * sizeof(float), cudaMemcpyDeviceToHost));
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c)
        {
            const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)tq[r * cols + c], __NV_E4M3);
            dst[r * cols + c] = host_f16_to_f32(h.x) * ts[r];
        }
    return 0;
}

// debug tap of the q | k | v activations in the reference's [tokens][3 D] order (the device buffers are head-major, [3 H][rows][64], at
// head dim 64, and already in that order at head dim 80)
int tap_qkv(vitb200_engine *e, float *dst, int T, cudaStream_t s)
{
    if (!dst) return 0;
    const int D = e->hp.hidden_size, H = e->hp.num_attention_heads;
    if (head_dim(e) != 64) return tap_f16(dst, e->QKV16, (size_t)T * 3 * D, s, e->QKV16L);
    const size_t plane_rows = (size_t)e->max_batch * e->N, n = (size_t)3 * H * plane_rows * 64;
    std::vector<float> tmp(n);
    if (tap_f16(tmp.data(), e->QKV16, n, s, e->QKV16L)) return 1;
    for (int t = 0; t < T; ++t)
        for (int pl = 0; pl < 3 * H; ++pl)
            memcpy(dst + (size_t)t * 3 * D + (size_t)pl * 64, tmp.data() + ((size_t)pl * plane_rows + t) * 64, 64 * sizeof(float));
    return 0;
}

// The embedding stage of the image schedule (vit.cpp:772-797): afterwards the residual stream X holds the input of block 0
int run_embed(vitb200_engine *e, const float *d_images, int B, cudaStream_t s, const vitb200_taps *taps)
{
    const int D = e->hp.hidden_size, N = e->N, T = B * N;
    __half *PA = e->PA;
    // patch embedding (vit.cpp:772-797): the f16 patch matrix PA (im2col of a stride == kernel conv is a pure permutation,
    // ggml.c:11528-11608) is either already there (d_images == NULL: the u8 path's preprocess kernel wrote it) or written by
    // patchify (one warp per patch, coalesced); the TMA-fed GEMM adds conv bias + pos_embed and writes token rows.
    const bool patches_ready = d_images == nullptr;
    {
        // the epilogue writes patch p of an image to row 1 + p and adds position row 1 + p: with R prefix rows (class token and
        // registers) both bases move by R - 1 rows, so patch p lands in row R + p with position row R + p -- one row up without a
        // class token (SigLIP), R = 1 + reg_tokens rows down otherwise
        const int R = prefix_rows(e->arch);
        GemmParams p{};
        p.M = B * e->NP; p.N = D; p.K = e->KPp; p.bias = e->patch.b; p.out = e->X + (ptrdiff_t)(R - 1) * D; p.ldo = D;
        p.pos = e->pos + (ptrdiff_t)(R - 1) * D; p.np = e->NP; p.ntok = N;
        ProfScope ps(e, PK_PATCH, 2.0 * p.M * p.N * e->KP, s);
        if (!patches_ready && launch_patchify(e, d_images, PA, B, s)) return 1;
        if (R > 0 && launch(e, cls_rows_kernel, dim3((B * R * D + 255) / 256), dim3(256), 0, s, LAUNCH_PLAIN, e->X, e->cls, e->pos, B, R, N, D))
            return 1;
        if (launch_gemm(e, EPI_PATCH_F32, e->tmA_P, e->patch.tm, p, s)) return 1;
    }
    if (e->arch.pre_norm)
    {
        // CLIP's ln_pre (timm norm_pre) on every token row, back into the stream every TMA map points at
        ProfScope ps(e, PK_LN, 0.0, s);
        if (launch_layernorm_inplace(e, e->X, e->npre_w, e->npre_b, T, s)) return 1;
    }
    if (taps && tap_f32(taps->embed, e->X, (size_t)T * D, s)) return 1;
    return 0;
}

// Blocks first .. last-1 (vit.cpp:802-901) on the residual stream X of B images or sequences, in place
int run_blocks(vitb200_engine *e, int B, int first, int last, cudaStream_t s, const vitb200_taps *taps)
{
    const int D = e->hp.hidden_size, N = e->N, T = B * N;
    for (int il = first; il < last; ++il)
    {
        const Layer &L = e->layers[il];
        const bool tap = taps && taps->layer == il;
        {
            ProfScope ps(e, PK_LN, 0.0, s);
            if (e->fp8)
            {
                if (launch_layernorm(e, e->X, (size_t)D, L.n1w, L.n1b, (__nv_fp8_e4m3 *)e->A8, T, s, 0, 0, e->SA)) return 1;
                if (tap && tap_e4m3(taps->ln1, e->A8, e->SA, (size_t)T, (size_t)D, s)) return 1;
            }
            else
            {
                if (launch_layernorm(e, e->X, (size_t)D, L.n1w, L.n1b, e->A16, T, s)) return 1; // vit.cpp:808-812
                if (tap && tap_f16(taps->ln1, e->A16, (size_t)T * D, s)) return 1;
            }
        }
        {
            GemmParams p{};
            // head dim 64: the head-major planes the attention's TMA maps read; head dim 80: row-major [T][3 D]
            p.M = T; p.N = 3 * D; p.K = D; p.bias = L.qkv.b; p.out = e->QKV16; p.out2 = e->QKV16L; p.ldo = 3 * D;
            p.headmajor = head_dim(e) == 64; p.plane_rows = (size_t)e->max_batch * N;
            p.a_scale = e->SA; p.w_scale = L.qkv.w_scale;
            ProfScope ps(e, PK_QKV, 2.0 * p.M * p.N * p.K, s);
            if (launch_gemm(e, e->QKV16L ? EPI_BIAS_F16_HILO : EPI_BIAS_F16, e->fp8 ? e->tmA8 : e->tmA_D, L.qkv.tm, p, s, e->fp8)) return 1; // vit.cpp:820-821
        }
        if (tap && tap_qkv(e, taps->qkv, T, s)) return 1;
        {
            ProfScope ps(e, PK_ATTN, 4.0 * B * e->hp.num_attention_heads * (double)N * N * head_dim(e), s);
            if (launch_attention(e, B, s)) return 1; // vit.cpp:826-866
        }
        if (tap && tap_f16(taps->attn, e->A16, (size_t)T * D, s)) return 1;
        {
            GemmParams p{};
            p.M = T; p.N = D; p.K = D; p.bias = L.proj.b; p.out = e->X; p.ldo = D; p.resid = e->X; p.gamma = L.ls1;
            ProfScope ps(e, PK_PROJ, 2.0 * p.M * p.N * p.K, s);
            if (launch_gemm(e, resid_epilogue(e), e->tmA_D, L.proj.tm, p, s)) return 1; // proj + residual, vit.cpp:868-873
        }
        if (tap && tap_f32(taps->x1, e->X, (size_t)T * D, s)) return 1;
        {
            ProfScope ps(e, PK_LN, 0.0, s);
            if (e->fp8 ? launch_layernorm(e, e->X, (size_t)D, L.n2w, L.n2b, (__nv_fp8_e4m3 *)e->A8, T, s, 0, 0, e->SA)
                       : launch_layernorm(e, e->X, (size_t)D, L.n2w, L.n2b, e->A16, T, s)) return 1; // vit.cpp:881-885
        }
        if (tap && (e->fp8 ? tap_e4m3(taps->ln2, e->A8, e->SA, (size_t)T, (size_t)D, s) : tap_f16(taps->ln2, e->A16, (size_t)T * D, s))) return 1;
        {
            GemmParams p{};
            // SwiGLU: N = the interleaved 2 round_up(F, 64) rows of fc1, F columns stored
            p.M = T; p.N = L.fc1.n_out; p.K = D; p.bias = L.fc1.b; p.out = e->H16; p.ldo = e->F; p.F = e->F;
            p.a_scale = e->SA; p.w_scale = L.fc1.w_scale;
            ProfScope ps(e, PK_FC1, 2.0 * p.M * (e->arch.activation == 4 ? 2 * e->F : e->F) * p.K, s);
            if (launch_gemm(e, fc1_epilogue(e), e->fp8 ? e->tmA8 : e->tmA_D, L.fc1.tm, p, s, e->fp8)) return 1; // vit.cpp:889-893
        }
        if (tap && tap_f16(taps->h, e->H16, (size_t)T * e->F, s)) return 1;
        {
            GemmParams p{};
            p.M = T; p.N = D; p.K = e->F; p.bias = L.fc2.b; p.out = e->X; p.ldo = D; p.resid = e->X; p.gamma = L.ls2;
            ProfScope ps(e, PK_FC2, 2.0 * p.M * p.N * p.K, s);
            if (launch_gemm(e, resid_epilogue(e), e->tmA_H, L.fc2.tm, p, s)) return 1; // fc2 + residual, vit.cpp:896-900
        }
        if (tap && tap_f32(taps->x2, e->X, (size_t)T * D, s)) return 1;
    }
    return 0;
}

// The encoder part of the fixed kernel schedule: embeddings, then blocks 0 .. layers-1; afterwards the residual stream X holds the
// encoder's output at that depth.
int run_encoder(vitb200_engine *e, const float *d_images, int B, int layers, cudaStream_t s, const vitb200_taps *taps)
{
    return run_embed(e, d_images, B, s, taps) || run_blocks(e, B, 0, layers, s, taps);
}

// per-row width of probs and logits: the zero-shot head's classes while one is set, else the model's
int num_outputs(const vitb200_engine *e) { return e->zs_C ? e->zs_C : e->hp.num_classes; }

int check_batch(const vitb200_engine *e, int batch)
{
    if (batch < 1 || batch > e->max_batch) return fail("batch %d out of range (1..%d)", batch, e->max_batch);
    return 0;
}

int check_k(const vitb200_engine *e, int k)
{
    if (k < 0 || k > e->max_k) return fail("k %d out of range (0..%d)", k, e->max_k);
    return 0;
}

// Soft-max + top-k of `rows` logits rows of pitch ldl >= C: the working row in dynamic shared memory up to kSoftmaxSmemMax, beyond it
// in e->d_sm_scratch ([rows][C] floats).  sigmoid: the zero-shot head's mode 1 (per-class sigmoid, top-k by logit)
int launch_softmax_topk(vitb200_engine *e, const float *lg, int ldl, int rows, int C, float *d_probs, int32_t *d_topk_idx, float *d_topk_val,
                        int k, cudaStream_t s, bool sigmoid = false)
{
    const size_t row_bytes = (size_t)C * sizeof(float);
    float *scratch = row_bytes > kSoftmaxSmemMax ? e->d_sm_scratch : nullptr;
    if (row_bytes > kSoftmaxSmemMax && !scratch) return fail("soft-max: %d classes need a global working row and none is allocated", C);
    return launch(e, sigmoid ? softmax_topk_kernel<true> : softmax_topk_kernel<false>, dim3(rows), dim3(256), scratch ? 0 : row_bytes, s,
                  LAUNCH_PLAIN, lg, ldl, d_probs, d_topk_idx, d_topk_val, C, k, scratch);
}

// After the head GEMM has written the R rows lg (pitch ldl, num_classes columns): the zero-shot head's scores into d_logits (dense
// [R][zs_C]) or, when the caller takes none, into ZS_S, then its soft-max or sigmoid and top-k over the zs_C classes.  One launch more
// than the schedule without a head (the head's scores replace the 2-D copy of the logits).
int run_zero_shot(vitb200_engine *e, const float *lg, int ldl, int R, float *d_probs, float *d_logits, int32_t *d_topk_idx, float *d_topk_val,
                  int k, cudaStream_t s)
{
    const int Z = e->zs_C;
    float *z = d_logits ? d_logits : e->ZS_S;
    if (launch(e, zero_shot_kernel, dim3((unsigned)((R + ZS_TILE - 1) / ZS_TILE), (unsigned)((Z + ZS_TILE - 1) / ZS_TILE)), dim3(ZS_THREADS), 0, s,
               LAUNCH_PLAIN, lg, ldl, (const float *)e->ZS_T, z, Z, R, e->hp.num_classes, Z, e->zs_s, e->zs_b))
        return 1;
    if (d_probs || (k > 0 && (d_topk_idx || d_topk_val)))
        return launch_softmax_topk(e, z, Z, R, Z, d_probs, d_topk_idx, d_topk_val, k, s, e->zs_mode == 1);
    return 0;
}

// SigLIP's attention-pooling head (vitb200_arch.pool = 2, HF SiglipMultiheadAttentionPoolingHead) on the residual stream X of B images
// at its current depth: POOL32 [B][D] f32 = h + fc2(act(fc1(LN_head(h)))), h = out_proj(the probe's attention over post_layernorm(X)).
// f16 operands and f32 accumulation in both engines.  Launches: LN, k | v GEMM, attention, out_proj, LN, fc1, fc2.
int run_map_head(vitb200_engine *e, int B, cudaStream_t s)
{
    const int D = e->hp.hidden_size, T = B * e->N;
    {
        ProfScope ps(e, PK_LN, 0.0, s);
        if (launch_layernorm(e, e->X, (size_t)D, e->norm_w, e->norm_b, e->A16, T, s)) return 1; // post_layernorm, every token row
    }
    {
        // k | v of every row into QKV16 as the qkv GEMM lays out k and v: the head-major planes 0 .. 2 H - 1 at head dim 64, row-major
        // [T][2 D] at head dim 72
        GemmParams kv{};
        kv.M = T; kv.N = 2 * D; kv.K = D; kv.bias = e->pool_kv.b; kv.out = e->QKV16; kv.ldo = 2 * D; kv.headmajor = head_dim(e) == 64;
        kv.plane_rows = (size_t)e->max_batch * e->N;
        GemmParams o{};
        o.M = B; o.N = D; o.K = D; o.bias = e->pool_proj.b; o.out = e->POOL32; o.ldo = D;
        ProfScope ps(e, PK_POOL, 2.0 * kv.M * kv.N * kv.K + 4.0 * T * D + 2.0 * B * D * D, s);
        if (launch_gemm(e, EPI_BIAS_F16, e->tmA_D, e->pool_kv.tm, kv, s) || launch_attention_pool(e, e->pool_q, e->QKV16, e->CLS16, B, s) ||
            launch_gemm(e, EPI_BIAS_F32, e->tmA_C, e->pool_proj.tm, o, s))
            return 1;
    }
    {
        ProfScope ps(e, PK_LN, 0.0, s);
        if (launch_layernorm_rows<true>(e, e->POOL32, (size_t)D, e->pool_nw, e->pool_nb, e->A16, B, s, 0, 0)) return 1;
    }
    // the head's MLP has the blocks' width F (4 D but for So400m-shaped towers)
    GemmParams f1{};
    f1.M = B; f1.N = e->F; f1.K = D; f1.bias = e->pool_fc1.b; f1.out = e->H16; f1.ldo = e->F;
    GemmParams f2{};
    f2.M = B; f2.N = D; f2.K = e->F; f2.bias = e->pool_fc2.b; f2.out = e->POOL32; f2.ldo = D; f2.resid = e->POOL32;
    ProfScope ps(e, PK_POOL, 2.0 * B * 2.0 * e->F * D, s);
    return launch_gemm(e, fc1_epilogue(e), e->tmA_D, e->pool_fc1.tm, f1, s) || launch_gemm(e, EPI_BIAS_RESID_F32, e->tmA_H, e->pool_fc2.tm, f2, s);
}

// The fixed kernel schedule == reference vit_encode_image (vit.cpp:718-941), batched over images.
int run_forward(vitb200_engine *e, const float *d_images, int B, float *d_probs, float *d_logits, int32_t *d_topk_idx,
                float *d_topk_val, int k, cudaStream_t s, const vitb200_taps *taps)
{
    if (check_batch(e, B) || check_k(e, k)) return 1;
    if (!d_images && taps) return fail("debug taps need the f32 image path");
    const int D = e->hp.hidden_size, N = e->N, T = B * N, C = e->hp.num_classes;
    if (run_encoder(e, d_images, B, e->hp.num_hidden_layers, s, taps)) return 1;
    if (taps && tap_f32(taps->x_final, e->X, (size_t)T * D, s)) return 1;

    // pool (token 0; the first 25 tokens for ViTSTR, vitstr.cpp:864-883) + final LN + head + soft-max + top-k
    // (vit.cpp:910-933, 1047-1057); one row of the head GEMM / one soft-max per pooled token.  DINOv2 (arch.pool = 1): one row of
    // [LN(token 0) || mean of LN(patches)] per image; SigLIP: the attention-pooling head's row rounded to f16 (pool = 2) or the mean of
    // LN(rows) (pool = 3)
    const int TH = e->head_tokens, R = B * TH;
    if (e->arch.pool == 2)
    {
        if (run_map_head(e, B, s)) return 1;
        ProfScope ps(e, PK_POOL, 0.0, s);
        if (launch_layernorm_rows<false>(e, e->POOL32, (size_t)D, nullptr, nullptr, e->CLS16, B, s, 0, 0)) return 1;
    }
    else if (e->arch.pool ? launch_pool<true>(e, e->CLS16, B, s)
                          : launch_layernorm(e, e->X, (size_t)D, e->norm_w, e->norm_b, e->CLS16, R, s, TH, (size_t)N * D))
        return 1;
    if (taps && tap_f16(taps->final_ln, e->CLS16, (size_t)R * e->KH, s)) return 1;
    // internal logits rows have pitch Cp (num_classes padded to 4; the padded W rows are TMA zero fill, the padded bias is 0);
    // a caller's dense [rows][num_classes] buffer is written directly when the two coincide, else through a 2-D copy
    const int Cp = e->Cp;
    float *lg = (d_logits && Cp == C && !e->zs_C) ? d_logits : e->d_logits;
    {
        GemmParams p{};
        p.M = R; p.N = Cp; p.K = e->KH; p.bias = e->head.b; p.out = lg; p.ldo = Cp;
        ProfScope ps(e, PK_HEAD, 2.0 * p.M * C * p.K, s);
        if (launch_gemm(e, EPI_BIAS_F32, e->tmA_C, e->head.tm, p, s)) return 1;
    }
    if (e->zs_C) return run_zero_shot(e, lg, Cp, R, d_probs, d_logits, d_topk_idx, d_topk_val, k, s);
    if (d_logits && lg != d_logits)
        CUDA_TRY(cudaMemcpy2DAsync(d_logits, (size_t)C * 4, lg, (size_t)Cp * 4, (size_t)C * 4, (size_t)R, cudaMemcpyDeviceToDevice, s));
    if ((d_probs || (k > 0 && (d_topk_idx || d_topk_val))) && launch_softmax_topk(e, lg, Cp, R, C, d_probs, d_topk_idx, d_topk_val, k, s)) return 1;
    return 0;
}

// run((OutT *)dst, std::integral_constant<bool, NORM>) for a features output: dtype 0 f32, 1 f16, 2 bf16, normalised or not
template <class Run>
int with_features_type(int dtype, bool norm, void *dst, Run run)
{
    auto typed = [&](auto *y) { return norm ? run(y, std::true_type()) : run(y, std::false_type()); };
    if (dtype == 0) return typed((float *)dst);
    if (dtype == 1) return typed((__half *)dst);
    if (dtype == 2) return typed((__nv_bfloat16 *)dst);
    return fail("features: dtype %d unknown", dtype);
}

// Encoder features (vitb200_features*): the encoder up to block req->layers, then the requested rows of the residual stream -- all T
// token rows into d_tokens, the head_tokens pooled rows of every image into d_prelogits -- normalised with the final LayerNorm or not,
// as f32 / f16 / bf16.  Device destinations; either may be NULL.  An un-normalised f32 output is a copy, every other one a kernel.
// The requested rows of the residual stream X into dst, as req asks for them: rows_per_group of every group of N rows, normalised with the
// final LayerNorm or not, as f32 / f16 / bf16.  An un-normalised f32 output is a copy, every other one a kernel.  dst NULL: nothing.
int emit_rows(vitb200_engine *e, const vitb200_features_req *req, void *dst, int rows, int rows_per_group, cudaStream_t s)
{
    const int D = e->hp.hidden_size, N = e->N;
    if (!dst) return 0;
    return with_features_type(req->dtype, req->norm, dst, [&](auto *y, auto norm) -> int {
        if constexpr (norm() || !std::is_same<decltype(y), float *>::value)
        {
            ProfScope ps(e, PK_LN, 0.0, s);
            return launch_layernorm_rows<norm()>(e, e->X, (size_t)D, norm() ? e->norm_w : nullptr, norm() ? e->norm_b : nullptr, y, rows, s,
                                                 rows_per_group, (size_t)N * D);
        }
        // [B][rows_per_group][D] out of [B][N][D]: one 2-D copy (the token rows are a single plain copy)
        const size_t w = (size_t)rows_per_group * D * sizeof(float);
        CUDA_TRY(cudaMemcpy2DAsync(dst, w, e->X, (size_t)N * D * sizeof(float), w, (size_t)rows / rows_per_group, cudaMemcpyDeviceToDevice, s));
        return 0;
    });
}

int run_features(vitb200_engine *e, const float *d_images, int B, const vitb200_features_req *req, void *d_tokens, void *d_prelogits, cudaStream_t s)
{
    const int D = e->hp.hidden_size, N = e->N, TH = e->head_tokens;
    if (run_encoder(e, d_images, B, req->layers, s, nullptr)) return 1;
    auto emit = [&](void *dst, int rows, int rows_per_group) { return emit_rows(e, req, dst, rows, rows_per_group, s); };
    if (d_prelogits && e->arch.pool == 2)
    {
        // SigLIP's attention-pooling head on the final LayerNorm of the rows at this depth (norm = 1, check_features), before the
        // token rows are emitted: the host path stages those in H16, where the head's fc1 writes
        if (run_map_head(e, B, s)) return 1;
        {
            ProfScope ps(e, PK_POOL, 0.0, s);
            if (with_features_type(req->dtype, false, d_prelogits, [&](auto *y, auto) -> int {
                    if constexpr (std::is_same<decltype(y), float *>::value)
                        CUDA_TRY(cudaMemcpyAsync(d_prelogits, e->POOL32, (size_t)B * D * sizeof(float), cudaMemcpyDeviceToDevice, s));
                    else
                        return launch_layernorm_rows<false>(e, e->POOL32, (size_t)D, nullptr, nullptr, y, B, s, 0, 0);
                    return 0;
                }))
                return 1;
        }
        return emit(d_tokens, B * N, N);
    }
    if (emit(d_tokens, B * N, N)) return 1;
    if (d_prelogits && e->arch.pool)
    {
        // DINOv2: [token 0 || mean of the patch rows] per image, through the final LayerNorm or not; SigLIP (pool = 3): the mean alone
        ProfScope ps(e, PK_LN, 0.0, s);
        return with_features_type(req->dtype, req->norm, d_prelogits, [&](auto *y, auto norm) { return launch_pool<norm()>(e, y, B, s); });
    }
    return emit(d_prelogits, B * TH, TH);
}

// `run` (one kernel schedule, no taps) through a cached CUDA graph: the first call with a given argument set runs eagerly (also sets
// the kernels' function attributes), the second captures + instantiates, later ones replay.  Profiling always runs eagerly.
template <typename Run>
int run_graphed(vitb200_engine *e, const GraphKey &key, cudaStream_t s, Run run)
{
    // Graph replay pays off where the ~90 launches are a visible fraction of the step (small batches); at B = 256 every kernel
    // runs >= 80 us and eager launches stay ahead of the GPU (measured: no gain), so large batches launch eagerly.
    if (!e->use_graph || e->profile || (long long)key.batch * e->N > 8192) return run();
    vitb200_engine::GraphEntry *g = nullptr;
    for (auto &x : e->graphs)
        if (x.key == key) { g = &x; break; }
    if (!g)
    {
        if (e->graphs.size() >= 16) { if (e->graphs.front().exec) cudaGraphExecDestroy(e->graphs.front().exec); e->graphs.erase(e->graphs.begin()); }
        e->graphs.push_back({key, 0, 0, nullptr});
        g = &e->graphs.back();
    }
    if (g->state == 0)
    {
        if (run()) return 1;
        g->state = 1;
        return 0;
    }
    if (g->state == 1)
    {
        cudaGraph_t graph = nullptr;
        const int before = e->launches;
        CUDA_TRY(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        const int rc = run();
        cudaError_t ce = cudaStreamEndCapture(s, &graph);
        // the captured kernels did not run: the graph launch below, or the eager fallback, counts them
        g->launches = e->launches - before;
        e->launches = before;
        if (rc != 0 || ce != cudaSuccess || !graph)
        {
            if (graph) cudaGraphDestroy(graph);
            (void)cudaGetLastError();
            g->state = 0;
            e->use_graph = false; // fall back to eager launches (same kernels, same results)
            return run();
        }
        ce = cudaGraphInstantiate(&g->exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ce != cudaSuccess) { g->exec = nullptr; g->state = 0; e->use_graph = false; return fail("cudaGraphInstantiate failed: %s", cudaGetErrorString(ce)); }
        g->state = 2;
    }
    CUDA_TRY(cudaGraphLaunch(g->exec, s));
    e->launches += g->launches;
    return 0;
}

int run_forward_graphed(vitb200_engine *e, const float *d_images, int B, float *d_probs, float *d_logits, int32_t *d_topk_idx,
                        float *d_topk_val, int k, cudaStream_t s)
{
    const GraphKey key{d_images, B, d_probs, d_logits, d_topk_idx, d_topk_val, k, -1, 0, 0, nullptr, nullptr};
    return run_graphed(e, key, s, [&] { return run_forward(e, d_images, B, d_probs, d_logits, d_topk_idx, d_topk_val, k, s, nullptr); });
}

int run_features_graphed(vitb200_engine *e, const float *d_images, int B, const vitb200_features_req *req, void *d_tokens, void *d_prelogits,
                         cudaStream_t s)
{
    const GraphKey key{d_images, B, nullptr, nullptr, nullptr, nullptr, 0, req->layers, req->norm, req->dtype, d_tokens, d_prelogits};
    return run_graphed(e, key, s, [&] { return run_features(e, d_images, B, req, d_tokens, d_prelogits, s); });
}

// The text schedule (vitb200_encode_text*): the token rows, blocks 0 .. L-1 with the token rows emitted after block req->layers (the blocks
// past it only when embeds are wanted), then each sequence's pooled row through the final LayerNorm and the head.  Device destinations;
// either may be NULL (req is read only with d_tokens).
int run_text(vitb200_engine *e, const int32_t *d_ids, int B, float *d_embeds, const vitb200_features_req *req, void *d_tokens, cudaStream_t s)
{
    const int D = e->hp.hidden_size, N = e->N, L = e->hp.num_hidden_layers, E = e->hp.num_classes;
    {
        ProfScope ps(e, PK_PATCH, 0.0, s);
        if (launch(e, token_embed_kernel, dim3((unsigned)N, (unsigned)B), dim3(TOKEN_EMBED_THREADS), 0, s, LAUNCH_PLAIN, d_ids, e->tok, e->pos,
                   e->X, N, D, e->V))
            return 1;
    }
    const int at = d_tokens ? req->layers : L;
    if (run_blocks(e, B, 0, at, s, nullptr) || (d_tokens && emit_rows(e, req, d_tokens, B * N, N, s))) return 1;
    if (!d_embeds) return 0;
    if (run_blocks(e, B, at, L, s, nullptr)) return 1;
    {
        ProfScope ps(e, PK_LN, 0.0, s);
        if (launch_rows_kernel(e, [](auto V) { return text_pool_kernel<V()>; }, dim3((unsigned)((B + TEXT_POOL_WARPS - 1) / TEXT_POOL_WARPS)),
                               dim3(TEXT_POOL_WARPS * 32), 0, s, e->X, d_ids, B, N, e->text_arch.pool, e->text_arch.eos_token_id, e->norm_w, e->norm_b,
                               e->CLS16, D, e->hp.eps))
            return 1;
    }
    // rows of pitch Cp (E padded to 4) unless the caller's dense rows coincide, as the image head's logits
    float *lg = e->Cp == E ? d_embeds : e->d_logits;
    GemmParams p{};
    p.M = B; p.N = e->Cp; p.K = D; p.bias = e->head.b; p.out = lg; p.ldo = e->Cp;
    {
        ProfScope ps(e, PK_HEAD, 2.0 * B * E * D, s);
        if (launch_gemm(e, EPI_BIAS_F32, e->tmA_C, e->head.tm, p, s)) return 1;
    }
    if (lg != d_embeds)
        CUDA_TRY(cudaMemcpy2DAsync(d_embeds, (size_t)E * 4, lg, (size_t)e->Cp * 4, (size_t)E * 4, (size_t)B, cudaMemcpyDeviceToDevice, s));
    return 0;
}

int run_text_graphed(vitb200_engine *e, const int32_t *d_ids, int B, float *d_embeds, const vitb200_features_req *req, void *d_tokens, cudaStream_t s)
{
    const GraphKey key{d_ids, B, nullptr, d_embeds, nullptr, nullptr, 0, d_tokens ? req->layers : -1, d_tokens ? req->norm : 0,
                       d_tokens ? req->dtype : 0, d_tokens, nullptr};
    return run_graphed(e, key, s, [&] { return run_text(e, d_ids, B, d_embeds, req, d_tokens, s); });
}

// The refusal of an image entry point on a text engine
int image_only(const vitb200_engine *e, const char *fn)
{
    if (e && e->text) return fail("%s: this is a text engine (vitb200_create_text); it takes token ids through vitb200_encode_text", fn);
    return 0;
}

// Argument checks of the two vitb200_encode_text entry points, before anything is enqueued
int check_text(const vitb200_engine *e, const void *ids, int batch, const void *embeds, const vitb200_features_req *req, const void *tokens)
{
    if (!e || !ids) return fail("vitb200_encode_text: null argument");
    if (!e->text) return fail("vitb200_encode_text: this is an image engine; the text entry points need a text tower (vitb200_create_text)");
    if (!embeds && !tokens) return fail("vitb200_encode_text: both outputs are NULL");
    if (tokens)
    {
        if (!req) return fail("vitb200_encode_text: tokens need a vitb200_features_req");
        if (req->layers < 0 || req->layers > e->hp.num_hidden_layers)
            return fail("vitb200_encode_text: layers %d out of range (0..%d)", req->layers, e->hp.num_hidden_layers);
        if (req->norm != 0 && req->norm != 1) return fail("vitb200_encode_text: norm must be 0 or 1 (got %d)", req->norm);
        if (req->dtype < 0 || req->dtype > 2) return fail("vitb200_encode_text: dtype %d unknown (0 f32, 1 f16, 2 bf16)", req->dtype);
    }
    return check_batch(e, batch);
}

// Argument checks of the three vitb200_features entry points, before anything is enqueued
int check_features(const vitb200_engine *e, const void *images, int batch, const vitb200_features_req *req, const void *tokens, const void *prelogits)
{
    if (!e || !images || !req) return fail("vitb200_features: null argument");
    if (image_only(e, "vitb200_features")) return 1;
    if (req->layers < 0 || req->layers > e->hp.num_hidden_layers)
        return fail("vitb200_features: layers %d out of range (0..%d)", req->layers, e->hp.num_hidden_layers);
    if (req->norm != 0 && req->norm != 1) return fail("vitb200_features: norm must be 0 or 1 (got %d)", req->norm);
    if (req->dtype < 0 || req->dtype > 2) return fail("vitb200_features: dtype %d unknown (0 f32, 1 f16, 2 bf16)", req->dtype);
    if (!tokens && !prelogits) return fail("vitb200_features: both outputs are NULL");
    if (prelogits && e->arch.pool == 2 && !req->norm)
        return fail("vitb200_features: the attention-pooling head (vitb200_arch.pool = 2) reads the final LayerNorm's rows: prelogits need norm = 1");
    return check_batch(e, batch);
}

size_t features_elem_bytes(const vitb200_features_req *req) { return req->dtype == 0 ? 4 : 2; }

// Selects `device` for the calling thread and requires an sm_90 part: the device check of vitb200_create and of every test hook
int open_device(int device, cudaDeviceProp &prop)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail("no CUDA device: the vit.cpp_b200 forward path has no CPU fallback");
    if (device < 0 || device >= ndev) return fail("device %d out of range (%d devices)", device, ndev);
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail("device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    return 0;
}

// An engine that vitb200_destroy frees unless it is released: a half-built one, or a test hook's scratch engine
struct EngineDeleter
{
    void operator()(vitb200_engine *e) const { vitb200_destroy(e); }
};
using EnginePtr = std::unique_ptr<vitb200_engine, EngineDeleter>;

// SigLIP's attention-pooling head (vitb200_arch.pool = 2), timm AttentionPoolLatent names; 'kv' rows are k then v
constexpr int kPoolTensorCount = 13;
const char *const kPoolTensors[kPoolTensorCount] = {
    "attn_pool.latent", "attn_pool.q.weight", "attn_pool.q.bias", "attn_pool.kv.weight", "attn_pool.kv.bias", "attn_pool.proj.weight",
    "attn_pool.proj.bias", "attn_pool.norm.weight", "attn_pool.norm.bias", "attn_pool.mlp.fc1.weight", "attn_pool.mlp.fc1.bias",
    "attn_pool.mlp.fc2.weight", "attn_pool.mlp.fc2.bias"};

// The values of a weight tensor as stored (f32, f16, bf16 or a ggml block format), widened to f64
int host_values(const vitb200_tensor *x, const std::string &name, std::vector<double> &out)
{
    const size_t cnt = (size_t)nelem(x);
    out.resize(cnt);
    if (x->type == 0) for (size_t i = 0; i < cnt; ++i) out[i] = ((const float *)x->data)[i];
    else if (x->type == 1) for (size_t i = 0; i < cnt; ++i) out[i] = host_f16_to_f32(((const uint16_t *)x->data)[i]);
    else if (x->type == 30)
        for (size_t i = 0; i < cnt; ++i)
        {
            const uint32_t u = (uint32_t)((const uint16_t *)x->data)[i] << 16;
            float f;
            memcpy(&f, &u, 4);
            out[i] = f;
        }
    else if (quant_block_bytes(x->type) && cnt % 32 == 0)
    {
        float y[32];
        for (size_t b = 0; b < cnt / 32; ++b)
        {
            dequant_block(x->type, (const uint8_t *)x->data + b * quant_block_bytes(x->type), y);
            for (int i = 0; i < 32; ++i) out[b * 32 + i] = y[i];
        }
    }
    else return fail("tensor '%s': weight type %d is not supported", name.c_str(), x->type);
    return 0;
}

// The attention-pooling head's query is the same for every image: latent Wq^T + bq, computed once here in f64 from the stored values
// ('attn_pool.latent' [1, 1, D] and 'attn_pool.q.bias' [D] f32, 'attn_pool.q.weight' [D][D]) and kept in f32
int upload_probe_query(vitb200_engine *e, const vitb200_tensor *t, int n, int D)
{
    const vitb200_tensor *lat = find_tensor(t, n, "attn_pool.latent"), *w = find_tensor(t, n, "attn_pool.q.weight"), *b = find_tensor(t, n, "attn_pool.q.bias");
    if (!lat || !w || !b) return fail("missing tensor 'attn_pool.latent', 'attn_pool.q.weight' or 'attn_pool.q.bias'");
    if (lat->type != 0 || b->type != 0) return fail("tensors 'attn_pool.latent' and 'attn_pool.q.bias' must be f32");
    if (check_shape(lat, "attn_pool.latent", D, 1, 1, 1) || check_shape(b, "attn_pool.q.bias", D, 1, 1, 1) ||
        check_shape(w, "attn_pool.q.weight", D, D, 1, 1))
        return 1;
    std::vector<double> wv;
    if (host_values(w, "attn_pool.q.weight", wv)) return 1;
    const float *l = (const float *)lat->data, *bq = (const float *)b->data;
    std::vector<float> q(D);
    for (int i = 0; i < D; ++i)
    {
        double acc = 0.0;
        for (int k = 0; k < D; ++k) acc += (double)l[k] * wv[(size_t)i * D + k];
        q[i] = (float)(acc + (double)bq[i]);
    }
    if (dev_alloc(e, &e->pool_q, (size_t)D)) return 1;
    CUDA_TRY(cudaMemcpy(e->pool_q, q.data(), (size_t)D * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

// The weights of every block ('blocks.{i}.*': LayerNorms, qkv, proj, fc1, fc2 and, with layer_scale, the LayerScale gammas) and the final
// LayerNorm ('norm.*'), as e->hp, e->F and e->fp8 describe them; swiglu: fc1 is SwiGLU's [2 F][D]
int upload_blocks(vitb200_engine *e, const vitb200_tensor *t, int n, bool swiglu, bool layer_scale)
{
    const int D = e->hp.hidden_size, F = e->F;
    const bool fp8 = e->fp8;
    e->layers.resize(e->hp.num_hidden_layers);
    for (int i = 0; i < e->hp.num_hidden_layers; ++i)
    {
        Layer &L = e->layers[i];
        const std::string p = "blocks." + std::to_string(i) + ".";
        if (upload_f32(e, t, n, p + "norm1.weight", D, 1, 1, 1, &L.n1w) || upload_f32(e, t, n, p + "norm1.bias", D, 1, 1, 1, &L.n1b) ||
            upload_f32(e, t, n, p + "norm2.weight", D, 1, 1, 1, &L.n2w) || upload_f32(e, t, n, p + "norm2.bias", D, 1, 1, 1, &L.n2b))
            return 1;
        if (upload_linear(e, t, n, p + "attn.qkv.weight", p + "attn.qkv.bias", 3 * D, D, D, &L.qkv, 0, fp8) ||
            upload_linear(e, t, n, p + "attn.proj.weight", p + "attn.proj.bias", D, D, D, &L.proj) ||
            upload_linear(e, t, n, p + "mlp.fc1.weight", p + "mlp.fc1.bias", swiglu ? 2 * F : F, D, D, &L.fc1, 0, fp8, swiglu) ||
            upload_linear(e, t, n, p + "mlp.fc2.weight", p + "mlp.fc2.bias", D, F, F, &L.fc2))
            return 1;
        if (layer_scale && (upload_f32(e, t, n, p + "ls1.gamma", D, 1, 1, 1, &L.ls1) || upload_f32(e, t, n, p + "ls2.gamma", D, 1, 1, 1, &L.ls2)))
            return 1;
    }
    return upload_f32(e, t, n, "norm.weight", D, 1, 1, 1, &e->norm_w) || upload_f32(e, t, n, "norm.bias", D, 1, 1, 1, &e->norm_b);
}

// The MLP's hidden width F from block 0's fc1 ([2 F][D] with SwiGLU's gate, [F][D] otherwise): F % 8 == 0 and 8 <= F <= 8 D, and every
// block's fc1 and fc2 ([D][F]) must agree with it.  `what` names the setting that reads F from the weights in the messages.
int mlp_width(const vitb200_tensor *t, int n, int D, int layers, bool swiglu, const char *what, int &F)
{
    const vitb200_tensor *w1 = find_tensor(t, n, "blocks.0.mlp.fc1.weight");
    if (!w1) return fail("missing tensor 'blocks.0.mlp.fc1.weight'");
    const int64_t rows = dim_of(w1, 1), f = swiglu ? rows / 2 : rows;
    if (swiglu && rows % 2) return fail("%s needs an even row count 2 F in 'blocks.0.mlp.fc1.weight', got %lld", what, (long long)rows);
    if (f % 8) return fail("%s: F = %lld is not a multiple of 8", what, (long long)f);
    if (f < 8 || f > 8 * (int64_t)D) return fail("%s: F = %lld out of range (8..%d = 8 D)", what, (long long)f, 8 * D);
    F = (int)f;
    for (int i = 0; i < layers; ++i)
    {
        const std::string p = "blocks." + std::to_string(i) + ".mlp.";
        const vitb200_tensor *a = find_tensor(t, n, p + "fc1.weight"), *b = find_tensor(t, n, p + "fc2.weight");
        if ((a && dim_of(a, 1) != (swiglu ? 2 : 1) * f) || (b && dim_of(b, 0) != f))
            return fail("%s: block %d's mlp.fc1 [%lld][%lld] or mlp.fc2 [%lld][%lld] disagrees with F = %d (fc1 [%sF][D], fc2 [D][F])", what, i,
                        a ? (long long)dim_of(a, 1) : 0ll, a ? (long long)dim_of(a, 0) : 0ll, b ? (long long)dim_of(b, 1) : 0ll,
                        b ? (long long)dim_of(b, 0) : 0ll, F, swiglu ? "2 " : "");
    }
    return 0;
}

// The FP8 engine's e4m3 rows: LayerNorms 1 and 2 write D bytes per token, which the qkv and fc1 GEMMs read through TMA with a
// 16-byte row stride
int fail_fp8_width(int D)
{
    return fail("FP8 engine: hidden size %d not supported (a multiple of 16: the e4m3 activation rows of D bytes are read in 16-byte "
                "strides; head dim 72 needs an even head count)", D);
}

// Builds an engine; *out receives it only when everything succeeded.  labels: the class names of a model file.
int create_impl(const vitb200_hparams *hp, const vitb200_arch *arch, const vitb200_tensor *t, int n, int device, int max_batch, int head_tokens,
                bool fp8, vitb200_engine **out, const std::map<int, std::string> *labels = nullptr)
{
    if (!hp || !t || !out) return fail("vitb200_create: null argument");
    *out = nullptr;
    // hyper-parameter sanity first (no division by a field a corrupt file may have zeroed; no device needed to reject them)
    if (hp->hidden_size < 64 || hp->hidden_size > 8192 || hp->num_hidden_layers < 1 || hp->num_hidden_layers > 4096 ||
        hp->num_attention_heads < 1 || hp->num_attention_heads > 128 || hp->num_classes < 1 || hp->num_classes > (1 << 20) ||
        hp->patch_size < 1 || hp->patch_size > 64 || hp->img_size < hp->patch_size || hp->img_size > 4096 || n < 1)
        return fail("invalid hyper-parameters (hidden %d, layers %d, heads %d, classes %d, patch %d, img %d)", hp->hidden_size,
                    hp->num_hidden_layers, hp->num_attention_heads, hp->num_classes, hp->patch_size, hp->img_size);
    const vitb200_arch ar = arch ? *arch : vitb200_arch{};
    if (ar.pre_norm != 0 && ar.pre_norm != 1) return fail("vitb200_arch.pre_norm = %d out of range (0 none, 1 LayerNorm 'norm_pre')", ar.pre_norm);
    if (ar.activation < 0 || ar.activation > 4)
        return fail("vitb200_arch.activation = %d out of range (0 gelu_tanh, 1 gelu_erf, 2 quick_gelu, 3 gelu_pytorch_tanh, 4 swiglu)", ar.activation);
    if (ar.layer_scale != 0 && ar.layer_scale != 1)
        return fail("vitb200_arch.layer_scale = %d out of range (0 none, 1 LayerScale 'blocks.{i}.ls1.gamma' / 'ls2.gamma')", ar.layer_scale);
    if (ar.reg_tokens < 0 || ar.reg_tokens > VB_MAX_REG_TOKENS)
        return fail("vitb200_arch.reg_tokens = %d out of range (0..%d register tokens)", ar.reg_tokens, VB_MAX_REG_TOKENS);
    if (ar.pool < 0 || ar.pool > 3) return fail("vitb200_arch.pool = %d out of range (0 token, 1 cls_patch_mean, 2 map, 3 mean)", ar.pool);
    if (ar.activation == 3 && ar.pool < 2)
        return fail("vitb200_arch.activation = 3 out of range for pool %d: gelu_pytorch_tanh is the SigLIP towers' activation (pools 2 map and "
                    "3 mean)", ar.pool);
    if (ar.activation == 4 && ar.pool >= 2)
        return fail("vitb200_arch.activation = 4 out of range for pool %d: swiglu is DINOv2's MLP (pools 0 token and 1 cls_patch_mean)", ar.pool);
    if (ar.pool >= 2)
    {
        // SigLIP: the token rows are the patch rows alone
        if (find_tensor(t, n, "cls_token"))
            return fail("vitb200_arch.pool = %d out of range for a model with a class token: pools 2 (map) and 3 (mean) read patch rows only, "
                        "and the tensor 'cls_token' is present", ar.pool);
        if (ar.reg_tokens > 0) return fail("vitb200_arch.pool = %d needs reg_tokens = 0 (got %d): its token rows are the patch rows only", ar.pool, ar.reg_tokens);
        // the floor grid G = img_size / patch_size: a size the patch does not divide drops the last pixel rows and columns (HF's valid conv)
        const int64_t np = (int64_t)(hp->img_size / hp->patch_size) * (hp->img_size / hp->patch_size);
        const vitb200_tensor *pe = find_tensor(t, n, "pos_embed");
        if (pe && dim_of(pe, 1) != np)
            return fail("vitb200_arch.pool = %d needs 'pos_embed' with the %lld patch rows only (no class token), got %lld rows", ar.pool,
                        (long long)np, (long long)dim_of(pe, 1));
    }
    for (int i = 0; ar.pool == 2 && i < kPoolTensorCount; ++i)
        if (!find_tensor(t, n, kPoolTensors[i])) return fail("vitb200_arch.pool = 2 needs the attention-pooling head's tensor '%s'", kPoolTensors[i]);
    if (ar.pre_norm && (!find_tensor(t, n, "norm_pre.weight") || !find_tensor(t, n, "norm_pre.bias")))
        return fail("vitb200_arch.pre_norm = 1 needs the tensors 'norm_pre.weight' and 'norm_pre.bias'");
    for (int i = 0; ar.layer_scale && i < hp->num_hidden_layers; ++i)
        for (const char *g : {"ls1", "ls2"})
        {
            const std::string name = "blocks." + std::to_string(i) + "." + g + ".gamma";
            if (!find_tensor(t, n, name)) return fail("vitb200_arch.layer_scale = 1 needs the tensor '%s'", name.c_str());
        }
    if (ar.reg_tokens > 0 && !find_tensor(t, n, "reg_token"))
        return fail("vitb200_arch.reg_tokens = %d needs the tensor 'reg_token'", ar.reg_tokens);
    // the MLP's hidden width: 4 D, or F from the weights for SwiGLU and the SigLIP towers (So400m: 4304), checked by mlp_width
    int F = 4 * hp->hidden_size;
    if (ar.activation == 4)
    {
        if (mlp_width(t, n, hp->hidden_size, hp->num_hidden_layers, true, "vitb200_arch.activation = 4 (swiglu)", F)) return 1;
    }
    else if (ar.pool >= 2)
    {
        const std::string what = "vitb200_arch.pool = " + std::to_string(ar.pool);
        if (mlp_width(t, n, hp->hidden_size, hp->num_hidden_layers, false, what.c_str(), F)) return 1;
        // the attention-pooling head's MLP has the blocks' width
        const vitb200_tensor *a = find_tensor(t, n, "attn_pool.mlp.fc1.weight"), *b = find_tensor(t, n, "attn_pool.mlp.fc2.weight");
        if ((a && dim_of(a, 1) != F) || (b && dim_of(b, 0) != F))
            return fail("%s: the attention-pooling head's %s [%lld][%lld] disagrees with the blocks' F = %d (fc1 [F][D], fc2 [D][F])", what.c_str(),
                        a && dim_of(a, 1) != F ? "'attn_pool.mlp.fc1.weight'" : "'attn_pool.mlp.fc2.weight'",
                        a && dim_of(a, 1) != F ? (long long)dim_of(a, 1) : (long long)dim_of(b, 1),
                        a && dim_of(a, 1) != F ? (long long)dim_of(a, 0) : (long long)dim_of(b, 0), F);
    }
    if (ar.pool && head_tokens != 1) return fail("vitb200_arch.pool = %d needs head_tokens = 1 (got %d)", ar.pool, head_tokens);
    {
        // the head's K: the pooled row it reads is D wide, or 2 D with the class-plus-patch-mean pool
        const vitb200_tensor *hw = find_tensor(t, n, "head.weight");
        const int64_t k = (ar.pool == 1 ? 2 : 1) * (int64_t)hp->hidden_size;
        if (hw && dim_of(hw, 0) != k)
            return fail("vitb200_arch.pool = %d needs 'head.weight' with K = %lld (%s), got [%lld, %lld]", ar.pool, (long long)k,
                        ar.pool == 1 ? "2 D: class token || patch mean" : "D", (long long)dim_of(hw, 0), (long long)dim_of(hw, 1));
    }
    // input channels from the patch kernel [P, P, C, D] (vit.cpp:515; C = 1 in vitstr.cpp:482)
    const vitb200_tensor *pw = find_tensor(t, n, "patch_embed.proj.weight");
    const int64_t per_c = (int64_t)hp->hidden_size * hp->patch_size * hp->patch_size;
    if (!pw || nelem(pw) % per_c != 0 || (nelem(pw) / per_c != 1 && nelem(pw) / per_c != 3))
        return fail("tensor 'patch_embed.proj.weight' is missing or is not a 1- or 3-channel %dx%d kernel", hp->patch_size, hp->patch_size);
    const int in_chans = (int)(nelem(pw) / per_c);
    // shapes no kernel is built for: rejected here, where the caller can act on it, rather than by every forward call
    const int hd = hp->hidden_size / hp->num_attention_heads;
    if (hp->hidden_size % hp->num_attention_heads != 0 || (hd != 64 && hd != ATT80_HD && (hd != ATT72_HD || ar.pool < 2)))
        return fail("head dim %d not supported (64 or 80; 72 with pools 2 map and 3 mean, the SigLIP towers)", hd);
    if (hd == ATT80_HD && ar.pool == 2)
        return fail("vitb200_arch.pool = 2 (map) not supported at head dim 80 (the attention-pooling head's kernel is 64 or 72 columns wide)");
    if (fp8 && hp->hidden_size % 16 != 0) return fail_fp8_width(hp->hidden_size);
    if (hp->img_size % hp->patch_size != 0 && ar.pool < 2)
        return fail("img_size %d not a multiple of patch_size %d (only the SigLIP pools 2 and 3 take the floor grid)", hp->img_size, hp->patch_size);
    if (hp->img_size % hp->patch_size != 0 && patchify_reads_16b(hp->patch_size) && hp->img_size % 4 != 0)
        return fail("img_size %d not supported with patch_size %d: a floor grid needs img_size %% 4 == 0 at this patch size (16-byte loads of "
                    "each pixel row)", hp->img_size, hp->patch_size);
    if (!patchify_supports(hp->patch_size, in_chans))
        return fail("patch size %d not supported for %d-channel input (%s)", hp->patch_size, in_chans, patchify_sizes(in_chans));
    if (hp->hidden_size > LN_MAX_HIDDEN) return fail("hidden size %d not supported (max %d)", hp->hidden_size, LN_MAX_HIDDEN);
    const int n_tokens = (hp->img_size / hp->patch_size) * (hp->img_size / hp->patch_size) + prefix_rows(ar);
    if (n_tokens > max_tokens(hd))
        return fail("%d tokens not supported (max %d at head dim %d: K and V of one attention head must fit in shared memory)", n_tokens,
                    max_tokens(hd), hd);
    cudaDeviceProp prop;
    if (open_device(device, prop)) return 1;
    if (max_batch < 1) return fail("max_batch must be >= 1");
    if (check_unique_names(t, n)) return 1;
    if (head_tokens < 1 || head_tokens > n_tokens) return fail("head_tokens %d out of range (1..%d)", head_tokens, n_tokens);

    EnginePtr owner(new vitb200_engine());
    vitb200_engine *e = owner.get();
    e->hp = *hp;
    e->arch = ar;
    if (e->hp.eps <= 0.f) e->hp.eps = 1e-6f;
    e->device = device;
    e->max_batch = max_batch;
    e->fp8 = fp8;
    e->num_sms = prop.multiProcessorCount;
    const int D = hp->hidden_size, P = hp->patch_size;
    e->G = hp->img_size / P;
    e->NP = e->G * e->G;
    e->N = e->NP + prefix_rows(ar);
    e->F = F;
    e->C = in_chans;
    e->head_tokens = head_tokens;
    e->KH = (ar.pool == 1 ? 2 : 1) * hp->hidden_size;
    e->Cp = (hp->num_classes + 3) / 4 * 4;
    e->KP = e->C * P * P;
    e->KPp = (e->KP + 63) / 64 * 64;
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) return fail("cudaStreamCreate failed");

    // ---- weights (names: reference vit.cpp:518-579)
    // the prefix rows [cls_token; reg_token] as one array, the cls_rows_kernel's source (none with SigLIP's pools)
    if (prefix_rows(ar) > 0 && upload_f32(e, t, n, "cls_token", D, 1, 1, 1, &e->cls, (int64_t)(1 + ar.reg_tokens) * D)) return 1;
    if (ar.reg_tokens > 0)
    {
        float *reg = nullptr;
        if (upload_f32(e, t, n, "reg_token", D, ar.reg_tokens, 1, 1, &reg)) return 1;
        CUDA_TRY(cudaMemcpy(e->cls + D, reg, (size_t)ar.reg_tokens * D * sizeof(float), cudaMemcpyDeviceToDevice));
    }
    if (upload_f32(e, t, n, "pos_embed", D, e->N, 1, 1, &e->pos)) return 1;
    if (upload_linear(e, t, n, "patch_embed.proj.weight", "patch_embed.proj.bias", D, e->KP, e->KPp, &e->patch, P)) return 1;
    if (ar.pre_norm && (upload_f32(e, t, n, "norm_pre.weight", D, 1, 1, 1, &e->npre_w) || upload_f32(e, t, n, "norm_pre.bias", D, 1, 1, 1, &e->npre_b)))
        return 1;
    if (upload_blocks(e, t, n, ar.activation == 4, ar.layer_scale != 0)) return 1;
    if (upload_linear(e, t, n, "head.weight", "head.bias", hp->num_classes, e->KH, e->KH, &e->head)) return 1;
    if (ar.pool == 2 &&
        (upload_linear(e, t, n, "attn_pool.kv.weight", "attn_pool.kv.bias", 2 * D, D, D, &e->pool_kv) ||
         upload_linear(e, t, n, "attn_pool.proj.weight", "attn_pool.proj.bias", D, D, D, &e->pool_proj) ||
         upload_f32(e, t, n, "attn_pool.norm.weight", D, 1, 1, 1, &e->pool_nw) || upload_f32(e, t, n, "attn_pool.norm.bias", D, 1, 1, 1, &e->pool_nb) ||
         upload_linear(e, t, n, "attn_pool.mlp.fc1.weight", "attn_pool.mlp.fc1.bias", F, D, D, &e->pool_fc1) ||
         upload_linear(e, t, n, "attn_pool.mlp.fc2.weight", "attn_pool.mlp.fc2.bias", D, F, F, &e->pool_fc2) ||
         upload_probe_query(e, t, n, D) || dev_alloc(e, &e->POOL32, (size_t)max_batch * D)))
        return 1;

    // ---- activation arena
    const size_t B = (size_t)max_batch, T = B * e->N;
    const size_t R = B * (size_t)e->head_tokens;                        // classifier rows: pooled tokens of all images
    // the MLP hidden buffer, which the features calls also use to stage T x D f32 tokens and R pooled f32 rows (features_to_host)
    const size_t h16 = std::max(T * F, 2 * T * D + 2 * R * e->KH);
    // The patch matrix [B*NP][KPp] aliases the MLP hidden buffer (dead while the patch GEMM runs) when it fits and
    // has no K padding; otherwise it gets its own buffer whose zeroed padding columns are never written again.
    const size_t pa_elems = B * e->NP * e->KPp;
    const bool pa_alias = (e->KPp == e->KP) && pa_elems <= h16;
    const size_t img_elems = (size_t)e->C * hp->img_size * hp->img_size; // per image
    if (dev_alloc(e, &e->X, T * D) || dev_alloc(e, &e->A16, T * D) || dev_alloc(e, &e->QKV16, T * 3 * D) || dev_alloc(e, &e->H16, h16) ||
        dev_alloc(e, &e->CLS16, R * e->KH) || dev_alloc(e, &e->d_logits, R * e->Cp))
        return 1;
    // soft-max working row: dynamic shared memory up to the per-CTA limit, global scratch beyond it
    if ((size_t)hp->num_classes * sizeof(float) > kSoftmaxSmemMax && dev_alloc(e, &e->d_sm_scratch, R * hp->num_classes)) return 1;
    e->out_cols = hp->num_classes;
    e->sm_cols = e->d_sm_scratch ? hp->num_classes : 0;
    for (Slot &sl : e->slot)
    {
        if (dev_alloc(e, &sl.img, B * img_elems) || dev_alloc(e, &sl.probs, R * hp->num_classes) || dev_alloc(e, &sl.logits, R * hp->num_classes) ||
            dev_alloc(e, &sl.topk_idx, R * e->max_k) || dev_alloc(e, &sl.topk_val, R * e->max_k))
            return 1;
        if (e->C == 1 && e->head_tokens >= 2 &&
            (dev_alloc(e, &sl.chars, B * (e->head_tokens - 1)) || dev_alloc(e, &sl.len, B) || dev_alloc(e, &sl.score, B)))
            return 1;
        if (cudaEventCreateWithFlags(&sl.ev_h2d, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming) != cudaSuccess)
            return fail("cudaEventCreate failed");
    }
    if (cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking) != cudaSuccess) return fail("cudaStreamCreate failed");
    if (pa_alias) e->PA = e->H16;
    else
    {
        if (dev_alloc(e, &e->PA, pa_elems)) return 1;
        if (cudaMemset(e->PA, 0, pa_elems * sizeof(__half)) != cudaSuccess) return fail("cudaMemset failed");
    }
    // the GEMMs' A operands [rows][cols], dense rows: box = one k-block (128 B) x GEMM_A_BOX_ROWS rows
    auto a_map = [&](CUtensorMap *m, const void *ptr, cuuint64_t rows, cuuint64_t cols, bool e4m3 = false) {
        return e4m3 ? make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, ptr, {cols, rows}, {cols}, {2 * GEMM_BK, GEMM_A_BOX_ROWS})
                    : make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ptr, {cols, rows}, {2 * cols}, {GEMM_BK, GEMM_A_BOX_ROWS});
    };
    if (a_map(&e->tmA_D, e->A16, T, D) || a_map(&e->tmA_H, e->H16, T, (cuuint64_t)F) || a_map(&e->tmA_P, e->PA, B * e->NP, e->KPp) ||
        a_map(&e->tmA_C, e->CLS16, R, e->KH))
        return 1;
    if (fp8 && (dev_alloc(e, &e->A8, T * D) || dev_alloc(e, &e->SA, T) || a_map(&e->tmA8, e->A8, T, D, true))) return 1;
    // split-precision q, k, v (reference: f32 operands, vit.cpp:848,858) wherever hi + lo K and V fit next to each other in shared
    // memory (N <= 224), i.e. wherever the wgmma attention runs, or the head-dim-80 kernel in its split form (which reads the row-major
    // buffers directly: no TMA maps)
    if (e->N <= ATTW_KEYS && (dev_alloc(e, &e->QKV16L, T * 3 * D) || (hd == 64 && make_attention_maps(e)))) return 1;
    if (cudaDeviceSynchronize() != cudaSuccess) return fail("device sync after upload failed");
    if (labels) e->labels = *labels;
    *out = owner.release();
    return 0;
}

template <typename T>
int upload(vitb200_engine *e, T **d, const void *src, size_t count);

// Builds a text engine (vitb200_create_text); *out receives it only when everything succeeded.  The blocks, the final LayerNorm and the
// head are the image engine's; the token table and the position rows replace the patch embedding, and N = context <= 224, so the qkv GEMM
// always writes hi + lo for the split-precision attention.
int create_text_impl(const vitb200_hparams *hp, const vitb200_text_arch *ta, const vitb200_tensor *t, int n, int device, int max_batch, bool fp8,
                     vitb200_engine **out)
{
    if (!hp || !ta || !t || !out) return fail("vitb200_create_text: null argument");
    *out = nullptr;
    if (hp->hidden_size < 64 || hp->hidden_size > 8192 || hp->num_hidden_layers < 1 || hp->num_hidden_layers > 4096 ||
        hp->num_attention_heads < 1 || hp->num_attention_heads > 128 || hp->num_classes < 1 || hp->num_classes > (1 << 20) || n < 1)
        return fail("invalid hyper-parameters (hidden %d, layers %d, heads %d, projection %d)", hp->hidden_size, hp->num_hidden_layers,
                    hp->num_attention_heads, hp->num_classes);
    if (hp->patch_size != 0 || hp->img_size != 0)
        return fail("vitb200_create_text: patch_size and img_size must be 0 for a text tower (got %d and %d)", hp->patch_size, hp->img_size);
    const vitb200_text_arch a = *ta;
    if (a.context < 1 || a.context > ATTW_KEYS)
        return fail("vitb200_text_arch.context = %d out of range (1..%d tokens: the keys of the split-precision attention)", a.context, ATTW_KEYS);
    if (a.causal != 0 && a.causal != 1) return fail("vitb200_text_arch.causal = %d out of range (0 bidirectional, 1 causal)", a.causal);
    if (a.pool < 0 || a.pool > 2) return fail("vitb200_text_arch.pool = %d out of range (0 eos, 1 eos_argmax, 2 last)", a.pool);
    if (a.activation < 0 || a.activation > 3)
        return fail("vitb200_text_arch.activation = %d out of range (0 gelu_tanh, 1 gelu_erf, 2 quick_gelu, 3 gelu_pytorch_tanh; swiglu is "
                    "not a text tower's MLP)", a.activation);
    const int D = hp->hidden_size;
    // head dim 72 (SigLIP So400m) runs the row-major attention kernel, which has no causal mask
    const int hd = D / hp->num_attention_heads;
    if (D % hp->num_attention_heads != 0 || (hd != 64 && (hd != ATT72_HD || a.causal)))
        return fail("head dim %d not supported (64; 72 with causal = 0, the SigLIP text towers)", hd);
    if (fp8 && D % 16 != 0) return fail_fp8_width(D);
    if (D > LN_MAX_HIDDEN) return fail("hidden size %d not supported (max %d)", D, LN_MAX_HIDDEN);
    const vitb200_tensor *te = find_tensor(t, n, "token_embd.weight"), *pe = find_tensor(t, n, "pos_embed");
    if (!te) return fail("missing tensor 'token_embd.weight'");
    const int64_t V = dim_of(te, 1);
    if (dim_of(te, 0) != D || V < 1 || V > (1 << 30) || dim_of(te, 2) != 1 || dim_of(te, 3) != 1)
        return fail("tensor 'token_embd.weight' must be [V][%d] with 1 <= V <= 2^30, got [%lld, %lld, %lld, %lld] (ggml order)", D,
                    (long long)dim_of(te, 0), (long long)dim_of(te, 1), (long long)dim_of(te, 2), (long long)dim_of(te, 3));
    if (pe && dim_of(pe, 1) != a.context)
        return fail("vitb200_text_arch.context = %d, but 'pos_embed' has %lld rows", a.context, (long long)dim_of(pe, 1));
    // the MLP's width: F from the weights for the SigLIP (bidirectional) towers, 4 D for CLIP's
    int F = 4 * D;
    if (!a.causal && mlp_width(t, n, D, hp->num_hidden_layers, false, "vitb200_text_arch.causal = 0", F)) return 1;
    cudaDeviceProp prop;
    if (open_device(device, prop)) return 1;
    if (max_batch < 1) return fail("max_batch must be >= 1");
    if (check_unique_names(t, n)) return 1;

    EnginePtr owner(new vitb200_engine());
    vitb200_engine *e = owner.get();
    e->hp = *hp;
    if (e->hp.eps <= 0.f) e->hp.eps = 1e-6f;
    e->text = true;
    e->text_arch = a;
    e->arch.activation = a.activation; // the fc1 epilogue (fc1_epilogue)
    e->device = device;
    e->max_batch = max_batch;
    e->fp8 = fp8;
    e->num_sms = prop.multiProcessorCount;
    e->N = a.context;
    e->F = F;
    e->C = 0;
    e->KH = D;
    e->V = (int)V;
    e->Cp = (hp->num_classes + 3) / 4 * 4;
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) return fail("cudaStreamCreate failed");
    {
        // the token table in f16, whatever its file format (as upload_linear converts a weight)
        std::vector<double> v;
        if (host_values(te, "token_embd.weight", v)) return 1;
        std::vector<uint16_t> h(v.size());
        for (size_t i = 0; i < v.size(); ++i) h[i] = host_f32_to_f16((float)v[i]);
        if (upload(e, &e->tok, h.data(), h.size())) return 1;
    }
    if (upload_f32(e, t, n, "pos_embed", D, e->N, 1, 1, &e->pos) || upload_blocks(e, t, n, false, false) ||
        upload_linear(e, t, n, "head.weight", "head.bias", hp->num_classes, D, D, &e->head))
        return 1;

    const size_t B = (size_t)max_batch, T = B * e->N;
    if (dev_alloc(e, &e->X, T * D) || dev_alloc(e, &e->A16, T * D) || dev_alloc(e, &e->QKV16, T * 3 * D) || dev_alloc(e, &e->QKV16L, T * 3 * D) ||
        dev_alloc(e, &e->H16, T * e->F) || dev_alloc(e, &e->CLS16, B * D) || dev_alloc(e, &e->d_logits, B * e->Cp) ||
        dev_alloc(e, &e->TOKS, T * D * sizeof(float)))
        return 1;
    for (Slot &sl : e->slot)
    {
        if (dev_alloc(e, &sl.ids, T) || dev_alloc(e, &sl.logits, B * hp->num_classes)) return 1;
        if (cudaEventCreateWithFlags(&sl.ev_h2d, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming) != cudaSuccess)
            return fail("cudaEventCreate failed");
    }
    if (cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking) != cudaSuccess) return fail("cudaStreamCreate failed");
    auto a_map = [&](CUtensorMap *m, const void *ptr, cuuint64_t rows, cuuint64_t cols, bool e4m3 = false) {
        return e4m3 ? make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, ptr, {cols, rows}, {cols}, {2 * GEMM_BK, GEMM_A_BOX_ROWS})
                    : make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, ptr, {cols, rows}, {2 * cols}, {GEMM_BK, GEMM_A_BOX_ROWS});
    };
    if (a_map(&e->tmA_D, e->A16, T, D) || a_map(&e->tmA_H, e->H16, T, (cuuint64_t)e->F) || a_map(&e->tmA_C, e->CLS16, B, D) ||
        (hd == 64 && make_attention_maps(e)))
        return 1;
    if (fp8 && (dev_alloc(e, &e->A8, T * D) || dev_alloc(e, &e->SA, T) || a_map(&e->tmA8, e->A8, T, D, true))) return 1;
    if (cudaDeviceSynchronize() != cudaSuccess) return fail("device sync after upload failed");
    *out = owner.release();
    return 0;
}

// The test hooks' harness: each hook opens the device into a scratch engine with a non-blocking stream of its own, allocates with
// dev_alloc (vitb200_destroy frees it with the engine) and checks every copy.
int scratch_engine(int device, EnginePtr &e)
{
    cudaDeviceProp prop;
    if (open_device(device, prop)) return 1;
    e.reset(new vitb200_engine());
    e->device = device;
    e->num_sms = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) return fail("stream creation failed");
    return 0;
}

// host -> a new device buffer of `count` elements
template <typename T>
int upload(vitb200_engine *e, T **d, const void *src, size_t count)
{
    if (dev_alloc(e, d, count)) return 1;
    CUDA_TRY(cudaMemcpy(*d, src, count * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
}

// Runs a test hook's kernels on the scratch engine's stream and waits for them; `what` names them in the error.  cudaMemcpy from
// pageable memory may return before the DMA has landed, and the kernels run on a NON-BLOCKING stream (no implicit ordering with the
// legacy stream the uploads used): the device is synchronised before the launch.
template <class Launch>
int run_scratch(vitb200_engine *e, const char *what, Launch launch)
{
    if (cudaDeviceSynchronize() != cudaSuccess) return fail("device sync after upload failed");
    if (launch()) return 1;
    const cudaError_t err = cudaStreamSynchronize(e->stream);
    if (err != cudaSuccess)
    {
        (void)cudaGetLastError();
        return fail("%s failed: %s", what, cudaGetErrorString(err));
    }
    return 0;
}

// Stand-alone run of the block LayerNorm as the engine launches it (persistent bulk-copy kernel for hidden sizes that are a multiple of 128
// and >= 8 rows, the row-per-warp kernel otherwise): x [rows][D] f32 -> y [rows][D] (f16 results widened to f32).
// OutT = __nv_fp8_e4m3: the FP8 engine's LayerNorm 1 / 2, y e4m3 and y_scale the row scales.  Both outputs are poisoned with 0xFF
// first, so an element the kernel never writes reads back as NaN.
template <typename OutT>
int test_layernorm_impl(int device, int rows, int D, const float *x, const float *w, const float *b, float eps, OutT **y,
                        float **y_scale, EnginePtr &owner)
{
    if (scratch_engine(device, owner)) return 1;
    vitb200_engine *e = owner.get();
    e->hp.hidden_size = D; e->hp.eps = eps;
    float *dx = nullptr, *dw = nullptr, *db = nullptr;
    if (upload(e, &dx, x, (size_t)rows * D) || upload(e, &dw, w, D) || upload(e, &db, b, D) || dev_alloc(e, y, (size_t)rows * D)) return 1;
    CUDA_TRY(cudaMemset(*y, 0xFF, (size_t)rows * D * sizeof(OutT)));
    if (y_scale)
    {
        if (dev_alloc(e, y_scale, rows)) return 1;
        CUDA_TRY(cudaMemset(*y_scale, 0xFF, (size_t)rows * sizeof(float)));
    }
    return run_scratch(e, "LayerNorm kernel",
                       [&] { return launch_layernorm(e, dx, (size_t)D, dw, db, *y, rows, e->stream, 0, 0, y_scale ? *y_scale : nullptr); });
}

// The GEMM test hooks' one body: the GEMM alone on a scratch engine, as the engine launches it, with A [M][K] and W [N][K] f16 bits or
// (GEMM_OP_E4M3) e4m3 bytes.  SwiGLU takes W and bias in HF's order, interleaves them as the engine uploads them and stores [M][N / 2].
// plane_rows > 0: the f16 output is head-major, [N / 64][plane_rows][64] as the qkv and pool k | v GEMMs write it, both buffers filled
// with 0xFFFF first (rows M .. plane_rows - 1 of every plane keep it), and hi_bits / lo_bits receive the raw planes instead of `out`.
template <int OP, typename T>
int test_gemm_run(int device, int M, int N, int K, int epilogue, const T *A, const T *W, const float *bias, const float *a_scale,
                  float w_scale, const float *gamma, const float *resid, float *out, size_t plane_rows = 0, uint16_t *hi_bits = nullptr,
                  uint16_t *lo_bits = nullptr)
{
    const GemmEpiDesc d = gemm_epi(epilogue);
    if (d.swiglu && (N < 16 || N % 16 != 0)) return fail("SwiGLU: N = 2 F with F a multiple of 8 (got N = %d)", N);
    EnginePtr owner;
    if (scratch_engine(device, owner)) return 1;
    vitb200_engine *e = owner.get();
    const int F = N / 2, Nw = d.swiglu ? swiglu_rows(F) : N, No = d.swiglu ? F : N; // SwiGLU: Nw rows computed, No stored
    std::vector<T> wi;
    std::vector<float> bi;
    if (d.swiglu) { wi = swiglu_interleave(W, F, (size_t)K); bi = swiglu_interleave(bias, F, 1); W = wi.data(); bias = bi.data(); }
    const size_t MN = plane_rows ? plane_rows * No : (size_t)M * No;
    T *dA = nullptr, *dW = nullptr;
    __half *hi = nullptr, *lo = nullptr;
    float *dB = nullptr, *dS = nullptr, *dG = nullptr, *o32 = nullptr;
    if (upload(e, &dA, A, (size_t)M * K) || upload(e, &dW, W, (size_t)Nw * K) || upload(e, &dB, bias, Nw)) return 1;
    if ((a_scale && upload(e, &dS, a_scale, M)) || (gamma && upload(e, &dG, gamma, N))) return 1;
    if (d.f16 && (dev_alloc(e, &hi, MN) || (d.hilo && dev_alloc(e, &lo, MN)))) return 1;
    if (plane_rows)
    {
        CUDA_TRY(cudaMemset(hi, 0xFF, MN * sizeof(__half)));
        if (lo) CUDA_TRY(cudaMemset(lo, 0xFF, MN * sizeof(__half)));
    }
    // the residual epilogues work in place on the f32 stream, like the engine uses them (X += ...)
    if (!d.f16 && (d.resid ? upload(e, &o32, resid, MN) : dev_alloc(e, &o32, MN))) return 1;
    constexpr bool e4m3 = OP == GEMM_OP_E4M3;
    constexpr CUtensorMapDataType type = e4m3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    constexpr cuuint32_t kb = e4m3 ? 2 * GEMM_BK : GEMM_BK; // one k-block of 128 B
    const cuuint64_t Mu = (cuuint64_t)M, Nu = (cuuint64_t)Nw, Ku = (cuuint64_t)K;
    CUtensorMap tA, tB;
    if (make_tmap(&tA, type, dA, {Ku, Mu}, {sizeof(T) * Ku}, {kb, GEMM_A_BOX_ROWS}) || make_tmap(&tB, type, dW, {Ku, Nu}, {sizeof(T) * Ku}, {kb, GEMM_BN}))
        return 1;
    GemmParams p{};
    p.M = M; p.N = Nw; p.K = K; p.bias = dB; p.out = d.f16 ? (void *)hi : (void *)o32; p.out2 = lo; p.ldo = No; p.resid = o32; p.gamma = dG;
    p.a_scale = dS; p.w_scale = w_scale; p.F = F; p.headmajor = plane_rows > 0; p.plane_rows = plane_rows;
    if (run_scratch(e, e4m3 ? "e4m3 GEMM kernel" : "GEMM kernel", [&] { return launch_gemm(e, epilogue, tA, tB, p, e->stream, e4m3); })) return 1;
    if (plane_rows)
    {
        CUDA_TRY(cudaMemcpy(hi_bits, hi, MN * sizeof(__half), cudaMemcpyDeviceToHost));
        if (lo) CUDA_TRY(cudaMemcpy(lo_bits, lo, MN * sizeof(__half), cudaMemcpyDeviceToHost));
        return 0;
    }
    // split-precision result: hi + lo (exact in f32: the two parts do not overlap); the other f16 epilogues' hi alone, so that a -0 stays -0
    return d.f16 ? tap_f16(out, hi, MN, e->stream, lo) : tap_f32(out, o32, MN, e->stream);
}

// "0, 1, ...": the epilogue ids that `accepts`, for a hook's refusal
std::string gemm_epi_list(bool (*accepts)(int))
{
    std::string s;
    for (int epi = 0; epi < GEMM_EPI_END; ++epi)
        if (gemm_epi(epi).valid && accepts(epi)) s += (s.empty() ? "" : ", ") + std::to_string(epi);
    return s;
}

// One call of the host pipeline, once its arguments are checked: begin_submit picks its slot and starts the call's launch count; end_submit
// marks the slot's last use (everything enqueued on the compute stream so far) and counts the call
Slot &begin_submit(vitb200_engine *e)
{
    e->launches = 0;
    return e->slot[e->submits & 1];
}

int end_submit(vitb200_engine *e, Slot &sl)
{
    CUDA_TRY(cudaEventRecord(sl.ev_done, e->stream));
    e->submits++;
    return 0;
}

// The classifier forward of one pipelined call into slot sl, then the copies of the requested outputs to the caller's host buffers.
// d_images: sl.img, or NULL when the u8 preprocess has written the patch matrix.
int classify_to_host(vitb200_engine *e, const Slot &sl, const float *d_images, int batch, float *probs, float *logits, int32_t *topk_idx,
                     float *topk_prob, int k, const vitb200_taps *taps)
{
    cudaStream_t s = e->stream;
    const bool want_topk = k > 0 && (topk_idx || topk_prob);
    float *dp = (probs || want_topk) ? sl.probs : nullptr;
    int32_t *di = want_topk ? sl.topk_idx : nullptr;
    float *dv = want_topk ? sl.topk_val : nullptr;
    const int kk = want_topk ? k : 0;
    if (taps ? run_forward(e, d_images, batch, dp, sl.logits, di, dv, kk, s, taps) : run_forward_graphed(e, d_images, batch, dp, sl.logits, di, dv, kk, s))
        return 1;
    const size_t rows = (size_t)batch * e->head_tokens, C = (size_t)num_outputs(e); // classifier rows returned
    if (probs) CUDA_TRY(cudaMemcpyAsync(probs, sl.probs, rows * C * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (logits) CUDA_TRY(cudaMemcpyAsync(logits, sl.logits, rows * C * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (want_topk && topk_idx) CUDA_TRY(cudaMemcpyAsync(topk_idx, sl.topk_idx, rows * k * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (want_topk && topk_prob) CUDA_TRY(cudaMemcpyAsync(topk_prob, sl.topk_val, rows * k * sizeof(float), cudaMemcpyDeviceToHost, s));
    return 0;
}

} // namespace

extern "C" {

const char *vitb200_last_error(void) { return g_err.c_str(); }

int vitb200_create(const vitb200_hparams *hp, const vitb200_tensor *t, int n, int device, int max_batch, vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_impl(hp, nullptr, t, n, device, max_batch, 1, false, out); });
}

int vitb200_create_ex(const vitb200_hparams *hp, const vitb200_tensor *t, int n, int device, int max_batch, int head_tokens,
                      vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_impl(hp, nullptr, t, n, device, max_batch, head_tokens, false, out); });
}

int vitb200_create_fp8(const vitb200_hparams *hp, const vitb200_tensor *t, int n, int device, int max_batch, int head_tokens,
                       vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_impl(hp, nullptr, t, n, device, max_batch, head_tokens, true, out); });
}

int vitb200_create_arch(const vitb200_hparams *hp, const vitb200_arch *arch, const vitb200_tensor *t, int n, int device, int max_batch,
                        int head_tokens, int fp8, vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_impl(hp, arch, t, n, device, max_batch, head_tokens, fp8 != 0, out); });
}

int vitb200_create_text(const vitb200_hparams *hp, const vitb200_text_arch *ta, const vitb200_tensor *t, int n, int device, int max_batch,
                        int fp8, vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_text_impl(hp, ta, t, n, device, max_batch, fp8 != 0, out); });
}

int vitb200_get_text_arch(const vitb200_engine *e, vitb200_text_arch *out)
{
    return guarded(__func__, [&] {
        if (!e || !out) return fail("null argument");
        if (!e->text) return fail("vitb200_get_text_arch: this is an image engine");
        *out = e->text_arch;
        return 0;
    });
}

int vitb200_get_arch(const vitb200_engine *e, vitb200_arch *out)
{
    return guarded(__func__, [&] {
        if (!e || !out) return fail("null argument");
        if (image_only(e, __func__)) return 1;
        *out = e->arch;
        return 0;
    });
}

// vitb200_set_image_proc's checks for a model of C input channels and input size S, shared with the GGUF loader (which runs them before
// it creates the engine); each refusal names the field
static int check_image_proc(int C, int S, const vitb200_image_proc &p)
{
    if (C != 3) return fail("image_proc: this model takes %d-channel input; Hugging Face's image processors are for RGB models", C);
    if (p.resample != 2 && p.resample != 3) return fail("image_proc.resample = %d: 2 (BILINEAR) or 3 (BICUBIC) only", p.resample);
    if (p.shortest_edge < 0) return fail("image_proc.shortest_edge = %d: must not be negative", p.shortest_edge);
    if (p.shortest_edge == 0 && (p.height <= 0 || p.width <= 0))
        return fail("image_proc.height / width = %d x %d: must be positive when shortest_edge is 0", p.height, p.width);
    if (p.crop_height < 0 || p.crop_width < 0 || (p.crop_height == 0) != (p.crop_width == 0))
        return fail("image_proc.crop_height / crop_width = %d x %d: both positive, or both 0 (no crop)", p.crop_height, p.crop_width);
    const bool crop = p.crop_height > 0;
    if (p.shortest_edge > 0 && !crop)
        return fail("image_proc.shortest_edge = %d without crop_height / crop_width: the output size would depend on the image", p.shortest_edge);
    const int rh = p.shortest_edge > 0 ? p.shortest_edge : p.height, rw = p.shortest_edge > 0 ? p.shortest_edge : p.width;
    if (crop && (p.crop_height > rh || p.crop_width > rw))
        return fail("image_proc.crop_height / crop_width = %d x %d: larger than the resize target %d x %d (padding is not supported)", p.crop_height,
                    p.crop_width, rh, rw);
    const int fh = crop ? p.crop_height : p.height, fw = crop ? p.crop_width : p.width;
    if (fh != S || fw != S)
        return fail("image_proc: the final size %d x %d (%s) is not the model's img_size %d x %d", fh, fw, crop ? "crop_height x crop_width" : "height x width", S, S);
    if (!std::isfinite(p.rescale_factor) || !(p.rescale_factor > 0.0)) return fail("image_proc.rescale_factor = %g: must be finite and positive", p.rescale_factor);
    for (int c = 0; c < 3; ++c)
    {
        if (!std::isfinite(p.mean[c])) return fail("image_proc.mean[%d] = %g: must be finite", c, (double)p.mean[c]);
        if (!std::isfinite(p.std[c]) || p.std[c] == 0.0f) return fail("image_proc.std[%d] = %g: must be finite and non-zero", c, (double)p.std[c]);
    }
    return 0;
}

static int set_image_proc(vitb200_engine *e, const vitb200_image_proc *p)
{
    if (!e) return fail("null argument");
    if (image_only(e, "vitb200_set_image_proc")) return 1;
    if (p && check_image_proc(e->C, e->hp.img_size, *p)) return 1;
    e->has_proc = p != nullptr;
    e->proc = p ? *p : vitb200_image_proc{};
    return 0;
}

int vitb200_set_image_proc(vitb200_engine *e, const vitb200_image_proc *p)
{
    return guarded(__func__, [&] { return set_image_proc(e, p); });
}

int vitb200_get_image_proc(const vitb200_engine *e, vitb200_image_proc *out)
{
    return guarded(__func__, [&] {
        if (!e || !out) return fail("null argument");
        if (image_only(e, __func__)) return 1;
        *out = e->proc;
        return 0;
    });
}

// vitb200_set_zero_shot's checks on a head for an engine whose head rows are E wide, shared with vitb200_test_zero_shot; each refusal
// names the field or the row.  On success T holds the unit class rows (normalised in f64, stored f32), s = f32(exp(logit_scale)) (the
// exponential in f64) and b = logit_bias, 0 for NaN.
static int prepare_zero_shot(const vitb200_zero_shot &z, int E, std::vector<float> &T, float &s, float &b)
{
    if (z.n_classes < 1 || z.n_classes > (1 << 20)) return fail("zero_shot.n_classes = %d out of range (1..%d)", z.n_classes, 1 << 20);
    if (!z.class_embeds) return fail("zero_shot.class_embeds is NULL");
    if (z.mode != 0 && z.mode != 1) return fail("zero_shot.mode = %d: 0 (soft-max, CLIP) or 1 (sigmoid, SigLIP)", z.mode);
    if (!std::isfinite(z.logit_scale)) return fail("zero_shot.logit_scale = %g: must be finite", (double)z.logit_scale);
    const float sc = (float)std::exp((double)z.logit_scale);
    if (!std::isfinite(sc)) return fail("zero_shot.logit_scale = %g: exp(logit_scale) overflows f32", (double)z.logit_scale);
    if (std::isinf(z.logit_bias)) return fail("zero_shot.logit_bias = %g: must be finite, or NaN for none", (double)z.logit_bias);
    T.resize((size_t)z.n_classes * E);
    for (int c = 0; c < z.n_classes; ++c)
    {
        const float *row = z.class_embeds + (size_t)c * E;
        double ss = 0.0;
        for (int k = 0; k < E; ++k)
        {
            if (!std::isfinite(row[k])) return fail("zero_shot.class_embeds[%d][%d] = %g: must be finite", c, k, (double)row[k]);
            ss += (double)row[k] * row[k];
        }
        if (ss == 0.0) return fail("zero_shot.class_embeds row %d has zero norm", c);
        const double norm = std::sqrt(ss);
        for (int k = 0; k < E; ++k) T[(size_t)c * E + k] = (float)(row[k] / norm);
    }
    s = sc;
    b = std::isnan(z.logit_bias) ? 0.f : z.logit_bias;
    return 0;
}

static int set_zero_shot(vitb200_engine *e, const vitb200_zero_shot *z)
{
    if (!e) return fail("null argument");
    if (image_only(e, "vitb200_set_zero_shot")) return 1;
    if (e->C != 3) return fail("vitb200_set_zero_shot: this model takes %d-channel input; a zero-shot head is for RGB image towers", e->C);
    if (e->head_tokens > 1)
        return fail("vitb200_set_zero_shot: head_tokens is %d (ViTSTR); a zero-shot head scores one row per image", e->head_tokens);
    std::vector<float> T;
    float s = 0.f, b = 0.f;
    if (z && prepare_zero_shot(*z, e->hp.num_classes, T, s, b)) return 1;
    CUDA_TRY(cudaSetDevice(e->device));
    // work already enqueued (on any stream: vitb200_forward_device may run on the caller's) can still read the buffers replaced below
    CUDA_TRY(cudaDeviceSynchronize());
    // a captured graph holds the schedule and the buffer addresses of its capture
    for (auto &g : e->graphs)
        if (g.exec) cudaGraphExecDestroy(g.exec);
    e->graphs.clear();
    e->zs_C = 0;
    dev_free(e, &e->ZS_T);
    dev_free(e, &e->ZS_S);
    if (!z) return 0;
    const size_t R = (size_t)e->max_batch * e->head_tokens, Z = (size_t)z->n_classes;
    if (upload(e, &e->ZS_T, T.data(), T.size()) || dev_alloc(e, &e->ZS_S, R * Z)) return 1;
    if ((int)Z > e->out_cols)
    {
        for (Slot &sl : e->slot)
        {
            dev_free(e, &sl.probs);
            dev_free(e, &sl.logits);
            if (dev_alloc(e, &sl.probs, R * Z) || dev_alloc(e, &sl.logits, R * Z)) return 1;
        }
        e->out_cols = (int)Z;
    }
    if (Z * sizeof(float) > kSoftmaxSmemMax && (int)Z > e->sm_cols)
    {
        dev_free(e, &e->d_sm_scratch);
        if (dev_alloc(e, &e->d_sm_scratch, R * Z)) return 1;
        e->sm_cols = (int)Z;
    }
    e->zs_s = s;
    e->zs_b = b;
    e->zs_mode = z->mode;
    e->zs_logit_scale = z->logit_scale;
    e->zs_logit_bias = z->logit_bias;
    e->zs_C = (int)Z;
    return 0;
}

int vitb200_set_zero_shot(vitb200_engine *e, const vitb200_zero_shot *z)
{
    return guarded(__func__, [&] { return set_zero_shot(e, z); });
}

int vitb200_get_zero_shot(const vitb200_engine *e, int32_t *n_classes, float *logit_scale, float *logit_bias, int32_t *mode)
{
    return guarded(__func__, [&] {
        if (!e) return fail("null argument");
        if (image_only(e, __func__)) return 1;
        if (n_classes) *n_classes = e->zs_C;
        if (logit_scale) *logit_scale = e->zs_C ? e->zs_logit_scale : 0.f;
        if (logit_bias) *logit_bias = e->zs_C ? e->zs_logit_bias : 0.f;
        if (mode) *mode = e->zs_C ? e->zs_mode : 0;
        return 0;
    });
}

int vitb200_num_outputs(const vitb200_engine *e) { return e ? num_outputs(e) : 0; }

void vitb200_destroy(vitb200_engine *e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    for (void *p : e->allocs) cudaFree(p);
    for (auto &g : e->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    for (Slot &sl : e->slot)
    {
        if (sl.d_u8) cudaFree(sl.d_u8);
        if (sl.h_u8) cudaFreeHost(sl.h_u8);
        if (sl.d_proc) cudaFree(sl.d_proc);
        if (sl.ev_h2d) cudaEventDestroy(sl.ev_h2d);
        if (sl.ev_done) cudaEventDestroy(sl.ev_done);
    }
    for (auto &r : e->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    for (auto ev : e->event_pool) cudaEventDestroy(ev);
    if (e->stream) cudaStreamDestroy(e->stream);
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    delete e;
}

int vitb200_get_hparams(const vitb200_engine *e, vitb200_hparams *out)
{
    return guarded(__func__, [&] {
        if (!e || !out) return fail("null argument");
        *out = e->hp;
        return 0;
    });
}

const char *vitb200_label(const vitb200_engine *e, int class_id)
{
    if (!e) return nullptr;
    auto it = e->labels.find(class_id);
    return it == e->labels.end() ? nullptr : it->second.c_str();
}

int vitb200_last_launch_count(const vitb200_engine *e) { return e ? e->launches : 0; }
int vitb200_in_chans(const vitb200_engine *e) { return e ? e->C : 0; }
int vitb200_head_tokens(const vitb200_engine *e) { return e ? e->head_tokens : 0; }
int vitb200_fp8(const vitb200_engine *e) { return e && e->fp8 ? 1 : 0; }
int vitb200_mlp_dim(const vitb200_engine *e) { return e ? e->F : 0; }

int vitb200_profile_enable(vitb200_engine *e, int on)
{
    return guarded(__func__, [&]() -> int {
        if (!e) return fail("null argument");
        CUDA_TRY(cudaSetDevice(e->device));
        CUDA_TRY(cudaDeviceSynchronize());
        for (auto &r : e->prof) { e->event_pool.push_back(r.a); e->event_pool.push_back(r.b); }
        e->prof.clear();
        e->profile = on != 0;
        return 0;
    });
}

int vitb200_profile_read(vitb200_engine *e, int kind, double *ms_total, int *launches, double *flops_per_launch)
{
    return guarded(__func__, [&]() -> int {
        if (!e || !ms_total || !launches || !flops_per_launch) return fail("null argument");
        if (kind < 0 || kind >= PK_COUNT) return fail("profile kind %d out of range", kind);
        CUDA_TRY(cudaSetDevice(e->device));
        CUDA_TRY(cudaDeviceSynchronize());
        double ms = 0.0, fl = 0.0;
        int n = 0;
        for (auto &r : e->prof)
        {
            if (r.kind != kind) continue;
            float t = 0.f;
            CUDA_TRY(cudaEventElapsedTime(&t, r.a, r.b));
            ms += t; fl = r.flops; ++n;
        }
        *ms_total = ms; *launches = n; *flops_per_launch = fl;
        return 0;
    });
}

// causal: the wgmma kernel with CLIP's causal mask, as a causal text engine launches it.  probe: launch the wgmma kernel's phase probe
// and copy its records (grid x ATT_PROBE_PROBLEMS x ATT_PROBE_FIELDS) there, the grid size to *grid
static int test_attention_impl(int device, int kernel, int B, int N, int H, const uint16_t *qkv, const uint16_t *qkv_lo, float *out,
                               bool causal = false, unsigned long long *probe = nullptr, int *grid = nullptr)
{
    if (!qkv || !out || B < 1 || N < 1 || H < 1) return fail("bad argument");
    EnginePtr owner;
    if (scratch_engine(device, owner)) return 1;
    vitb200_engine *e = owner.get();
    e->N = N; e->hp.hidden_size = H * 64; e->hp.num_attention_heads = H; e->max_batch = B;
    e->text = causal; e->text_arch.causal = causal ? 1 : 0;
    const int D = H * 64;
    const uint64_t T = (uint64_t)B * N;
    // the kernels read the HEAD-MAJOR layout the qkv GEMM writes ([3 H][T][64]); the caller hands over the reference's [T][3 D]
    std::vector<uint16_t> hm((size_t)T * 3 * D);
    auto to_head_major = [&](const uint16_t *src) {
        for (uint64_t t = 0; t < T; ++t)
            for (int pl = 0; pl < 3 * H; ++pl)
                memcpy(&hm[((size_t)pl * T + t) * 64], src + (size_t)t * 3 * D + (size_t)pl * 64, 128);
    };
    to_head_major(qkv);
    if (upload(e, &e->QKV16, hm.data(), hm.size()) || dev_alloc(e, &e->A16, (size_t)T * D)) return 1;
    CUDA_TRY(cudaMemset(e->A16, 0xFF, T * D * sizeof(__half))); // an output the kernel never writes reads back as NaN
    const bool wgmma = kernel == ATT_WGMMA || kernel == ATT_WGMMA_HEAD;
    if (kernel < ATT_AUTO || kernel > ATT_WGMMA_HEAD || kernel == ATT_MMA80) return fail("attention kernel %d unknown", kernel);
    if (wgmma && N > ATTW_KEYS) return fail("wgmma attention needs N <= %d", ATTW_KEYS);
    if (kernel == ATT_MMA16 && (N <= 128 || N > ATT_MAX_KEYS_16)) return fail("16-warp attention needs 128 < N <= %d", ATT_MAX_KEYS_16);
    if (wgmma || (kernel == ATT_AUTO && N <= ATTW_KEYS))
    {
        // the wgmma kernel always runs on split-precision operands: without lo halves it reads zero lo planes (dev_alloc zero-fills
        // them), whose products add exact zeros
        if (qkv_lo) to_head_major(qkv_lo);
        if (qkv_lo ? upload(e, &e->QKV16L, hm.data(), hm.size()) : dev_alloc(e, &e->QKV16L, hm.size())) return 1;
        if (make_attention_maps(e)) return 1;
    }
    unsigned long long *d_probe = nullptr;
    const int n_cta = kernel == ATT_WGMMA && N <= ATTP_KEYS ? std::min(B * H, e->num_sms) : B * H;
    const size_t n_probe = (size_t)n_cta * ATT_PROBE_PROBLEMS * ATT_PROBE_FIELDS;
    if (probe)
    {
        if (dev_alloc(e, &d_probe, n_probe)) return 1;
        CUDA_TRY(cudaMemcpyToSymbol(g_attn_probe, &d_probe, sizeof(d_probe)));
    }
    if (run_scratch(e, "attention kernel", [&] { return launch_attention(e, B, e->stream, kernel, probe != nullptr); })) return 1;
    if (probe)
    {
        CUDA_TRY(cudaStreamSynchronize(e->stream));
        CUDA_TRY(cudaMemcpy(probe, d_probe, n_probe * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        *grid = n_cta;
    }
    return tap_f16(out, e->A16, (size_t)T * D, e->stream);
}

int vitb200_test_attention_phases(int device, int kernel, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo,
                                  unsigned long long *rec, int *grid)
{
    return guarded(__func__, [&] {
        if (!qkv_lo || !rec || !grid) return fail("bad argument");
        if (kernel != ATT_WGMMA && kernel != ATT_WGMMA_HEAD) return fail("the phase probe runs in the wgmma kernels (2 or 5), not %d", kernel);
        std::vector<float> out((size_t)B * N * H * 64);
        return test_attention_impl(device, kernel, B, N, H, qkv_hi, qkv_lo, out.data(), false, rec, grid);
    });
}

int vitb200_test_attention(int device, int kernel, int B, int N, int H, const uint16_t *qkv, float *out)
{
    return guarded(__func__, [&] { return test_attention_impl(device, kernel, B, N, H, qkv, nullptr, out); });
}

int vitb200_test_attention_hilo(int device, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out)
{
    return guarded(__func__, [&] {
        if (!qkv_lo) return fail("bad argument");
        return test_attention_impl(device, ATT_WGMMA, B, N, H, qkv_hi, qkv_lo, out);
    });
}

int vitb200_test_attention_hilo_causal(int device, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out)
{
    return guarded(__func__, [&] {
        if (!qkv_lo) return fail("bad argument");
        return test_attention_impl(device, ATT_WGMMA, B, N, H, qkv_hi, qkv_lo, out, true);
    });
}

// The row-major attention kernel at head dim hd (80 or 72) on the caller's [T][3 D] hi (and lo) buffers
int test_attention_rowmajor(int device, int kernel, int B, int N, int H, int hd, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out)
{
    if (!qkv_hi || !out || B < 1 || N < 1 || H < 1 || H > 128) return fail("bad argument");
    if (kernel != ATT_AUTO && (hd != ATT80_HD || kernel != ATT_MMA80)) return fail("attention kernel %d does not run head dim %d", kernel, hd);
    if (N > max_tokens(hd)) return fail("%d tokens not supported (max %d at head dim %d)", N, max_tokens(hd), hd);
    if (qkv_lo && N > ATTW_KEYS) return fail("split-precision head-dim-%d attention needs N <= %d (got %d)", hd, ATTW_KEYS, N);
    EnginePtr owner;
    if (scratch_engine(device, owner)) return 1;
    vitb200_engine *e = owner.get();
    e->N = N; e->hp.hidden_size = H * hd; e->hp.num_attention_heads = H; e->max_batch = B;
    const size_t T = (size_t)B * N, D = (size_t)H * hd;
    // the row-major [T][3 D] buffer the qkv GEMM writes at this head dim, as given; lo halves (the split form) when passed
    if (upload(e, &e->QKV16, qkv_hi, T * 3 * D) || (qkv_lo && upload(e, &e->QKV16L, qkv_lo, T * 3 * D)) || dev_alloc(e, &e->A16, T * D))
        return 1;
    CUDA_TRY(cudaMemset(e->A16, 0xFF, T * D * sizeof(__half))); // an output the kernel never writes reads back as NaN
    if (run_scratch(e, "attention kernel", [&] { return launch_attention(e, B, e->stream, kernel); })) return 1;
    return tap_f16(out, e->A16, T * D, e->stream);
}

int vitb200_test_attention_hd(int device, int kernel, int B, int N, int H, int hd, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out)
{
    return guarded(__func__, [&]() -> int {
        if (hd == 64)
        {
            if (qkv_lo && ((kernel != ATT_AUTO && kernel != ATT_WGMMA && kernel != ATT_WGMMA_HEAD) || N > ATTW_KEYS))
                return fail("split-precision operands run in the wgmma kernel (N <= %d)", ATTW_KEYS);
            return test_attention_impl(device, kernel, B, N, H, qkv_hi, qkv_lo, out);
        }
        if (hd != ATT80_HD) return fail("head dim %d not supported (64 or 80)", hd);
        return test_attention_rowmajor(device, kernel, B, N, H, hd, qkv_hi, qkv_lo, out);
    });
}

int vitb200_test_attention_hd72(int device, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out)
{
    return guarded(__func__, [&]() -> int { return test_attention_rowmajor(device, ATT_AUTO, B, N, H, ATT72_HD, qkv_hi, qkv_lo, out); });
}

// The attention-pool kernel at head dim hd on the caller's q [D] and k | v rows [B * P][2 D] (head-major planes built from them at 64)
int test_attention_pool(int device, int B, int P, int H, int hd, const float *q, const uint16_t *kv, float *out)
{
    if (!q || !kv || !out || B < 1 || P < 1 || P > max_tokens(hd) || H < 1 || H > 128) return fail("bad argument");
    EnginePtr owner;
    if (scratch_engine(device, owner)) return 1;
    vitb200_engine *e = owner.get();
    e->N = P; e->max_batch = B; e->hp.num_attention_heads = H; e->hp.hidden_size = H * hd;
    const size_t T = (size_t)B * P, D = (size_t)H * hd;
    std::vector<uint16_t> hm(kv, kv + T * 2 * D);
    // head dim 64: the head-major planes the k | v GEMM writes ([2 H][T][64]) from the caller's [T][2 D] rows
    for (size_t r = 0; hd == 64 && r < T; ++r)
        for (int pl = 0; pl < 2 * H; ++pl) memcpy(&hm[((size_t)pl * T + r) * 64], kv + r * 2 * D + (size_t)pl * 64, 128);
    float *dq = nullptr;
    __half *dkv = nullptr, *dout = nullptr;
    if (upload(e, &dq, q, D) || upload(e, &dkv, hm.data(), hm.size()) || dev_alloc(e, &dout, (size_t)B * D)) return 1;
    CUDA_TRY(cudaMemset(dout, 0xFF, (size_t)B * D * sizeof(__half))); // an output the kernel never writes reads back as NaN
    if (run_scratch(e, "attention-pool kernel", [&] { return launch_attention_pool(e, dq, dkv, dout, B, e->stream); })) return 1;
    return tap_f16(out, dout, (size_t)B * D, e->stream);
}

int vitb200_test_attention_pool(int device, int B, int P, int H, const float *q, const uint16_t *kv, float *out)
{
    return guarded(__func__, [&]() -> int { return test_attention_pool(device, B, P, H, 64, q, kv, out); });
}

int vitb200_test_attention_pool_hd72(int device, int B, int P, int H, const float *q, const uint16_t *kv, float *out)
{
    return guarded(__func__, [&]() -> int { return test_attention_pool(device, B, P, H, ATT72_HD, q, kv, out); });
}

int vitb200_test_softmax_topk(int device, int rows, int C, int k, const float *logits, float *probs, int32_t *topk_idx, float *topk_val)
{
    return guarded(__func__, [&]() -> int {
        if (!logits || !probs || rows < 1 || C < 1 || C > (1 << 20)) return fail("bad argument");
        if (k > 0 && (!topk_idx || !topk_val)) return fail("null argument");
        EnginePtr owner;
        if (scratch_engine(device, owner)) return 1;
        vitb200_engine *e = owner.get();
        e->max_k = 16;
        if (check_k(e, k)) return 1;
        // rows of pitch Cp, as the head GEMM leaves them; the padding columns hold NaN, which the kernel must never read
        const int Cp = (C + 3) / 4 * 4;
        std::vector<float> padded((size_t)rows * Cp, std::nanf(""));
        for (int r = 0; r < rows; ++r) memcpy(&padded[(size_t)r * Cp], logits + (size_t)r * C, (size_t)C * sizeof(float));
        float *dl = nullptr, *dp = nullptr, *dv = nullptr;
        int32_t *di = nullptr;
        if (upload(e, &dl, padded.data(), padded.size()) || dev_alloc(e, &dp, (size_t)rows * C) || dev_alloc(e, &di, (size_t)rows * k + 1) ||
            dev_alloc(e, &dv, (size_t)rows * k + 1))
            return 1;
        // outputs poisoned with 0x7f bytes (3.4e38, index 2139062143): an entry the kernel never writes cannot pass for a result
        CUDA_TRY(cudaMemset(dp, 0x7f, (size_t)rows * C * sizeof(float)));
        CUDA_TRY(cudaMemset(di, 0x7f, ((size_t)rows * k + 1) * sizeof(int32_t)));
        CUDA_TRY(cudaMemset(dv, 0x7f, ((size_t)rows * k + 1) * sizeof(float)));
        if ((size_t)C * sizeof(float) > kSoftmaxSmemMax && dev_alloc(e, &e->d_sm_scratch, (size_t)rows * C)) return 1;
        if (run_scratch(e, "soft-max kernel", [&] { return launch_softmax_topk(e, dl, Cp, rows, C, dp, k ? di : nullptr, k ? dv : nullptr, k, e->stream); }))
            return 1;
        CUDA_TRY(cudaMemcpy(probs, dp, (size_t)rows * C * sizeof(float), cudaMemcpyDeviceToHost));
        if (k > 0)
        {
            CUDA_TRY(cudaMemcpy(topk_idx, di, (size_t)rows * k * sizeof(int32_t), cudaMemcpyDeviceToHost));
            CUDA_TRY(cudaMemcpy(topk_val, dv, (size_t)rows * k * sizeof(float), cudaMemcpyDeviceToHost));
        }
        return 0;
    });
}

int vitb200_test_zero_shot(int device, int rows, int E, int C, const float *x, const float *T, float logit_scale, float logit_bias, int mode, int k,
                           float *probs, float *logits, int32_t *topk_idx, float *topk_val)
{
    return guarded(__func__, [&]() -> int {
        if (!x || !T || !probs || !logits || rows < 1 || E < 1 || E > (1 << 20)) return fail("bad argument");
        if (k > 0 && (!topk_idx || !topk_val)) return fail("null argument");
        std::vector<float> Tn;
        float s = 0.f, b = 0.f;
        if (prepare_zero_shot(vitb200_zero_shot{T, C, logit_scale, logit_bias, mode}, E, Tn, s, b)) return 1;
        EnginePtr owner;
        if (scratch_engine(device, owner)) return 1;
        vitb200_engine *e = owner.get();
        e->max_k = 16;
        if (check_k(e, k)) return 1;
        e->hp.num_classes = E;
        e->zs_C = C; e->zs_s = s; e->zs_b = b; e->zs_mode = mode;
        // head rows of pitch round_up(E, 4), as the head GEMM leaves them; the padding columns hold NaN, which the kernel must never read
        const int Ep = (E + 3) / 4 * 4;
        std::vector<float> padded((size_t)rows * Ep, std::nanf(""));
        for (int r = 0; r < rows; ++r) memcpy(&padded[(size_t)r * Ep], x + (size_t)r * E, (size_t)E * sizeof(float));
        float *dx = nullptr, *dp = nullptr, *dl = nullptr, *dv = nullptr;
        int32_t *di = nullptr;
        const size_t RC = (size_t)rows * C;
        if (upload(e, &dx, padded.data(), padded.size()) || upload(e, &e->ZS_T, Tn.data(), Tn.size()) || dev_alloc(e, &dp, RC) ||
            dev_alloc(e, &dl, RC) || dev_alloc(e, &di, (size_t)rows * k + 1) || dev_alloc(e, &dv, (size_t)rows * k + 1))
            return 1;
        // outputs poisoned with 0x7f bytes (3.4e38, index 2139062143): an entry the kernels never write cannot pass for a result
        CUDA_TRY(cudaMemset(dp, 0x7f, RC * sizeof(float)));
        CUDA_TRY(cudaMemset(dl, 0x7f, RC * sizeof(float)));
        CUDA_TRY(cudaMemset(di, 0x7f, ((size_t)rows * k + 1) * sizeof(int32_t)));
        CUDA_TRY(cudaMemset(dv, 0x7f, ((size_t)rows * k + 1) * sizeof(float)));
        if ((size_t)C * sizeof(float) > kSoftmaxSmemMax && dev_alloc(e, &e->d_sm_scratch, RC)) return 1;
        if (run_scratch(e, "zero-shot kernels", [&] { return run_zero_shot(e, dx, Ep, rows, dp, dl, k ? di : nullptr, k ? dv : nullptr, k, e->stream); }))
            return 1;
        CUDA_TRY(cudaMemcpy(probs, dp, RC * sizeof(float), cudaMemcpyDeviceToHost));
        CUDA_TRY(cudaMemcpy(logits, dl, RC * sizeof(float), cudaMemcpyDeviceToHost));
        if (k > 0)
        {
            CUDA_TRY(cudaMemcpy(topk_idx, di, (size_t)rows * k * sizeof(int32_t), cudaMemcpyDeviceToHost));
            CUDA_TRY(cudaMemcpy(topk_val, dv, (size_t)rows * k * sizeof(float), cudaMemcpyDeviceToHost));
        }
        return 0;
    });
}

int vitb200_test_dequant(int type, const void *blocks, int64_t n_blocks, uint16_t *out_f16)
{
    return guarded(__func__, [&] {
        const size_t bs = quant_block_bytes(type);
        if (!bs) return fail("type %d is not a supported block format", type);
        if (!blocks || !out_f16 || n_blocks < 0) return fail("null argument");
        float y[32];
        for (int64_t b = 0; b < n_blocks; ++b)
        {
            dequant_block(type, (const uint8_t *)blocks + (size_t)b * bs, y);
            for (int i = 0; i < 32; ++i) out_f16[b * 32 + i] = host_f32_to_f16(y[i]);
        }
        return 0;
    });
}

void *vitb200_stream(vitb200_engine *e) { return e ? (void *)e->stream : nullptr; }

int vitb200_forward_device(vitb200_engine *e, const float *d_images, int batch, float *d_probs, float *d_logits,
                           int32_t *d_topk_idx, float *d_topk_prob, int k, void *stream)
{
    return guarded(__func__, [&]() -> int {
        if (!e || !d_images) return fail("null argument");
        if (image_only(e, __func__)) return 1;
        CUDA_TRY(cudaSetDevice(e->device));
        if (check_batch(e, batch) || check_k(e, k)) return 1;
        e->launches = 0;
        return run_forward_graphed(e, d_images, batch, d_probs, d_logits, d_topk_idx, d_topk_prob, k, stream ? (cudaStream_t)stream : e->stream);
    });
}

int vitb200_features_device(vitb200_engine *e, const float *d_images, int batch, const vitb200_features_req *req, void *d_tokens,
                            void *d_prelogits, void *stream)
{
    return guarded(__func__, [&]() -> int {
        if (check_features(e, d_images, batch, req, d_tokens, d_prelogits)) return 1;
        if (((uintptr_t)d_tokens | (uintptr_t)d_prelogits) % 16 != 0) return fail("vitb200_features_device: output buffers must be 16-byte aligned");
        CUDA_TRY(cudaSetDevice(e->device));
        e->launches = 0;
        return run_features_graphed(e, d_images, batch, req, d_tokens, d_prelogits, stream ? (cudaStream_t)stream : e->stream);
    });
}

// Host images -> this call's input slot on the copy stream, once the slot's previous call has consumed it; the compute stream waits
// for the copy.  The device is waited on, not the host: only device memory is overwritten.
static int stage_images(vitb200_engine *e, const Slot &sl, const float *images, int batch)
{
    cudaStream_t cs = e->copy_stream;
    const size_t img_elems = (size_t)e->C * e->hp.img_size * e->hp.img_size;
    if (e->submits >= 2) CUDA_TRY(cudaStreamWaitEvent(cs, sl.ev_done, 0)); // slot's previous forward has consumed its inputs/outputs
    CUDA_TRY(cudaMemcpyAsync(sl.img, images, (size_t)batch * img_elems * sizeof(float), cudaMemcpyHostToDevice, cs));
    CUDA_TRY(cudaEventRecord(sl.ev_h2d, cs));
    CUDA_TRY(cudaStreamWaitEvent(e->stream, sl.ev_h2d, 0));
    return 0;
}

// Encoder features to HOST buffers, enqueued on the compute stream: kernel outputs are staged in H16 (the MLP hidden buffer, dead
// after the last block's fc2: T x 4D f16 holds T x D f32 tokens plus the pooled f32 rows), then copied back; an un-normalised f32
// output is copied straight out of the residual stream.
static int features_to_host(vitb200_engine *e, const float *d_images, int batch, const vitb200_features_req *req, void *tokens, void *prelogits)
{
    const size_t D = e->hp.hidden_size, N = e->N, TH = e->head_tokens, esz = features_elem_bytes(req);
    // pooled rows per image: head_tokens rows of D, or one row of 2 D with arch.pool = 1 (always a kernel's output)
    const size_t tok_bytes = (size_t)batch * N * D * esz, pre_bytes = (size_t)batch * TH * e->KH * esz;
    cudaStream_t s = e->stream;
    const bool copy = !req->norm && req->dtype == 0, pre_copy = copy && !e->arch.pool;
    uint8_t *stage = reinterpret_cast<uint8_t *>(e->H16);
    void *d_tok = tokens && !copy ? stage : nullptr;
    void *d_pre = prelogits && !pre_copy ? stage + tok_bytes : nullptr;
    if (run_features_graphed(e, d_images, batch, req, d_tok, d_pre, s)) return 1;
    if (tokens) CUDA_TRY(cudaMemcpyAsync(tokens, copy ? (const void *)e->X : d_tok, tok_bytes, cudaMemcpyDeviceToHost, s));
    if (prelogits && pre_copy)
        CUDA_TRY(cudaMemcpy2DAsync(prelogits, TH * D * 4, e->X, N * D * 4, TH * D * 4, (size_t)batch, cudaMemcpyDeviceToHost, s));
    else if (prelogits)
        CUDA_TRY(cudaMemcpyAsync(prelogits, d_pre, pre_bytes, cudaMemcpyDeviceToHost, s));
    return 0;
}

// Enqueue one batched forward with HOST buffers.  The H2D of this call runs on the copy stream and may overlap the kernels of the
// previous call (other slot); kernels + D2H run on the compute stream in call order.
static int forward_enqueue(vitb200_engine *e, const float *images, int batch, float *probs, float *logits, int32_t *topk_idx,
                           float *topk_prob, int k, const vitb200_taps *taps)
{
    if (!e || !images) return fail("null argument");
    if (image_only(e, "vitb200_forward")) return 1;
    if (check_batch(e, batch) || check_k(e, k)) return 1; // before anything is enqueued
    CUDA_TRY(cudaSetDevice(e->device));
    Slot &sl = begin_submit(e);
    if (stage_images(e, sl, images, batch) || classify_to_host(e, sl, sl.img, batch, probs, logits, topk_idx, topk_prob, k, taps)) return 1;
    return end_submit(e, sl);
}

int vitb200_forward_async(vitb200_engine *e, const float *images, int batch, float *probs, float *logits, int32_t *topk_idx,
                          float *topk_prob, int k)
{
    return guarded(__func__, [&] { return forward_enqueue(e, images, batch, probs, logits, topk_idx, topk_prob, k, nullptr); });
}

int vitb200_sync(vitb200_engine *e)
{
    return guarded(__func__, [&]() -> int {
        if (!e) return fail("null argument");
        CUDA_TRY(cudaSetDevice(e->device));
        CUDA_TRY(cudaStreamSynchronize(e->copy_stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
        return 0;
    });
}

static int forward_host(vitb200_engine *e, const float *images, int batch, float *probs, float *logits, int32_t *topk_idx,
                        float *topk_prob, int k, const vitb200_taps *taps)
{
    if (forward_enqueue(e, images, batch, probs, logits, topk_idx, topk_prob, k, taps)) return 1;
    return vitb200_sync(e);
}

// Data-parallel forward over several engines (one per GPU, weights replicated) driven from ONE host thread: image b goes to
// engine floor(b * n / batch)-style contiguous shards, every shard is enqueued with the non-blocking pipeline entry point, then
// all engines are synchronised.  No collective: shards are independent (SURVEY.md 8e).
static int forward_sharded_impl(vitb200_engine *const *engines, int n_engines, const float *images, int batch, float *probs, float *logits,
                                int32_t *topk_idx, float *topk_prob, int k, bool sync)
{
    if (!engines || n_engines < 1 || !images) return fail("null argument");
    const vitb200_engine *e0 = engines[0];
    if (!e0) return fail("null engine");
    if (check_k(e0, k)) return 1;
    {
        // validate every shard before the first one is enqueued
        const int base0 = batch / n_engines, rem0 = batch % n_engines;
        for (int g = 0; g < n_engines; ++g)
        {
            const int cnt = base0 + (g < rem0 ? 1 : 0);
            if (cnt == 0) continue;
            if (!engines[g]) return fail("null engine %d", g);
            if (cnt > engines[g]->max_batch) return fail("shard %d: batch %d out of range (1..%d)", g, cnt, engines[g]->max_batch);
        }
    }
    const size_t img_elems = (size_t)e0->C * e0->hp.img_size * e0->hp.img_size;
    const size_t C = (size_t)num_outputs(e0) * e0->head_tokens; // output floats per image
    const size_t kk = (size_t)k * e0->head_tokens;                 // top-k entries per image
    const int base = batch / n_engines, rem = batch % n_engines;
    int begin = 0;
    for (int g = 0; g < n_engines; ++g)
    {
        const int cnt = base + (g < rem ? 1 : 0);
        if (cnt == 0) continue;
        if (!engines[g]) return fail("null engine %d", g);
        if (engines[g]->hp.img_size != e0->hp.img_size || engines[g]->hp.num_classes != e0->hp.num_classes || engines[g]->head_tokens != e0->head_tokens ||
            engines[g]->C != e0->C)
            return fail("engine %d holds a different model", g);
        if (num_outputs(engines[g]) != num_outputs(e0))
            return fail("engine %d returns %d outputs per row and engine 0 returns %d (set the same zero-shot head on every engine)", g,
                        num_outputs(engines[g]), num_outputs(e0));
        if (vitb200_forward_async(engines[g], images + (size_t)begin * img_elems, cnt, probs ? probs + (size_t)begin * C : nullptr,
                                  logits ? logits + (size_t)begin * C : nullptr, topk_idx ? topk_idx + (size_t)begin * kk : nullptr,
                                  topk_prob ? topk_prob + (size_t)begin * kk : nullptr, k))
        {
            // shards already enqueued are copying into the caller's buffers: drain them before reporting the failure
            const std::string first = g_err;
            for (int h = 0; h < g; ++h)
                if (engines[h]) (void)vitb200_sync(engines[h]);
            g_err = first;
            return 1;
        }
        begin += cnt;
    }
    if (!sync) return 0;
    int rc = 0;
    for (int g = 0; g < n_engines; ++g)
        if (engines[g] && vitb200_sync(engines[g])) rc = 1;
    return rc;
}

int vitb200_forward_sharded(vitb200_engine *const *engines, int n_engines, const float *images, int batch, float *probs, float *logits,
                            int32_t *topk_idx, float *topk_prob, int k)
{
    return guarded(__func__, [&] { return forward_sharded_impl(engines, n_engines, images, batch, probs, logits, topk_idx, topk_prob, k, true); });
}

// Pipelined form: every shard goes through its engine's two-slot vitb200_forward_async pipeline and the call returns; the host
// thread can enqueue the next global batch (other host buffers) while this one runs.  vitb200_sync_all() waits for everything.
int vitb200_forward_sharded_async(vitb200_engine *const *engines, int n_engines, const float *images, int batch, float *probs,
                                  float *logits, int32_t *topk_idx, float *topk_prob, int k)
{
    return guarded(__func__, [&] { return forward_sharded_impl(engines, n_engines, images, batch, probs, logits, topk_idx, topk_prob, k, false); });
}

int vitb200_sync_all(vitb200_engine *const *engines, int n_engines)
{
    return guarded(__func__, [&] {
        if (!engines || n_engines < 1) return fail("null argument");
        int rc = 0;
        for (int g = 0; g < n_engines; ++g)
            if (engines[g] && vitb200_sync(engines[g])) rc = 1;
        return rc;
    });
}

int vitb200_forward(vitb200_engine *e, const float *images, int batch, float *probs, float *logits, int32_t *topk_idx,
                    float *topk_prob, int k)
{
    return guarded(__func__, [&] { return forward_host(e, images, batch, probs, logits, topk_idx, topk_prob, k, nullptr); });
}

int vitb200_forward_debug(vitb200_engine *e, const float *images, int batch, float *probs, float *logits, const vitb200_taps *taps)
{
    return guarded(__func__, [&] { return forward_host(e, images, batch, probs, logits, nullptr, nullptr, 0, taps); });
}

int vitb200_features(vitb200_engine *e, const float *images, int batch, const vitb200_features_req *req, void *tokens, void *prelogits)
{
    return guarded(__func__, [&]() -> int {
        if (check_features(e, images, batch, req, tokens, prelogits)) return 1;
        CUDA_TRY(cudaSetDevice(e->device));
        Slot &sl = begin_submit(e);
        if (stage_images(e, sl, images, batch) || features_to_host(e, sl.img, batch, req, tokens, prelogits) || end_submit(e, sl)) return 1;
        return vitb200_sync(e);
    });
}

// vit_image_preprocess (reference vit.cpp:289-305) for a batch of u8 RGB images of arbitrary sizes, on the GPU, followed by the
// forward pass: the "images" of vitb200_forward never exist on the host, and (unless images_f32_out asks for them) not in HBM
// either -- the preprocess kernel writes the f16 patch matrix the patch-embedding GEMM reads.  Pipelined like
// vitb200_forward_async: the caller's images are packed into this slot's pinned staging buffer, ONE host-to-device copy on the copy
// stream overlaps the previous call's kernels, nothing synchronises on entry and nothing is allocated once the staging buffers
// have grown to the largest batch seen.
// stage_u8 packs the images into slot sl and makes the compute stream wait for their copy (sl.d_u8 holds the pixels, then the
// PreImage table at table_off); it waits on the host, because it overwrites pinned host memory the slot's previous copy may still be
// reading.  preprocess_u8 adds the RGB kernel up to the patch matrix (and the optional f32 read-back).  The caller has checked the
// images (check_u8_images, or the recognition's own check).
static int check_u8_images(const uint8_t *const *images, const int *nx, const int *ny, int batch)
{
    for (int b = 0; b < batch; ++b)
        if (!images[b] || nx[b] < 1 || ny[b] < 1) return fail("image %d: bad pointer or size", b);
    return 0;
}

// extra / extra_bytes: a second per-call table (the image processor's ProcGeom rows), copied after the PreImage table at
// table_off + batch * sizeof(PreImage) in the same host-to-device copy
static int stage_u8(vitb200_engine *e, Slot &sl, const uint8_t *const *images, const int *nx, const int *ny, int batch, size_t &table_off,
                    const void *extra = nullptr, size_t extra_bytes = 0)
{
    size_t total = 0;
    for (int b = 0; b < batch; ++b) total += ((size_t)nx[b] * ny[b] * 3 + 255) / 256 * 256;
    table_off = total;
    total += (size_t)batch * sizeof(PreImage) + extra_bytes;
    CUDA_TRY(cudaSetDevice(e->device));
    cudaStream_t s = e->stream, cs = e->copy_stream;
    // this slot's previous call (two submissions ago) must have consumed its staging buffer before the host overwrites it
    if (e->submits >= 2) CUDA_TRY(cudaEventSynchronize(sl.ev_done));
    if (total > sl.u8_cap)
    {
        const size_t cap = total + total / 4;
        if (sl.h_u8) cudaFreeHost(sl.h_u8);
        if (sl.d_u8) cudaFree(sl.d_u8);
        sl.h_u8 = nullptr; sl.d_u8 = nullptr; sl.u8_cap = 0;
        CUDA_TRY(cudaHostAlloc((void **)&sl.h_u8, cap, cudaHostAllocDefault));
        CUDA_TRY(cudaMalloc((void **)&sl.d_u8, cap));
        sl.u8_cap = cap;
    }
    PreImage *table = reinterpret_cast<PreImage *>(sl.h_u8 + table_off);
    size_t off = 0;
    for (int b = 0; b < batch; ++b)
    {
        const size_t n = (size_t)nx[b] * ny[b] * 3;
        memcpy(sl.h_u8 + off, images[b], n);
        table[b].offset = off; table[b].nx = nx[b]; table[b].ny = ny[b];
        off += (n + 255) / 256 * 256;
    }
    if (extra_bytes) memcpy(sl.h_u8 + table_off + (size_t)batch * sizeof(PreImage), extra, extra_bytes);
    CUDA_TRY(cudaMemcpyAsync(sl.d_u8, sl.h_u8, total, cudaMemcpyHostToDevice, cs));
    CUDA_TRY(cudaEventRecord(sl.ev_h2d, cs));
    CUDA_TRY(cudaStreamWaitEvent(s, sl.ev_h2d, 0));
    return 0;
}

// Pillow's precompute_coeffs along one axis of a resize in -> out, on the host: the tap-table width ksize = ceil(support) * 2 + 1 (1 when
// the axis keeps its size), and the source range [first, end) of output index xx, in the device's operation order (pil_coeffs)
static double pil_ksize(int64_t in, int64_t out, int resample)
{
    if (in == out) return 1.0;
    const double scale = (double)in / (double)out;
    return std::ceil((resample == 2 ? 1.0 : 2.0) * (scale < 1.0 ? 1.0 : scale)) * 2.0 + 1.0;
}

static void pil_range(int64_t in, int64_t out, int64_t xx, int resample, int64_t &first, int64_t &end)
{
    if (in == out) { first = xx; end = xx + 1; return; }
    const double scale = (double)in / (double)out;
    const double support = (resample == 2 ? 1.0 : 2.0) * (scale < 1.0 ? 1.0 : scale);
    const double center = ((double)xx + 0.5) * scale;
    const double lo = center - support + 0.5, hi = center + support + 0.5;
    first = std::max<int64_t>((int64_t)lo, 0);
    end = std::min<int64_t>((int64_t)hi, in);
}

// The geometry of the image processor's two passes for a batch of checked images, worked out on the host in 64-bit integers before
// anything is enqueued, so that a 1 x 5000 photo (resized to 224 x 1120000) costs what its crop costs
static int plan_proc(vitb200_engine *e, const int *nx, const int *ny, int batch)
{
    const vitb200_image_proc &p = e->proc;
    const int S = e->hp.img_size;
    const size_t smem_max = 227 * 1024; // the opt-in shared memory of one H100 CTA
    ProcPlan &plan = e->proc_plan;
    plan.geo.resize((size_t)batch);
    double kh = 1.0, kv = 1.0;
    plan.max_rows = 1;
    plan.tmp_total = 0;
    for (int b = 0; b < batch; ++b)
    {
        const int64_t w = nx[b], h = ny[b];
        int64_t ow = p.width, oh = p.height;
        if (p.shortest_edge > 0)
        {
            const int64_t sh = std::min(w, h), lg = std::max(w, h);
            const int64_t nl = (int64_t)((double)(p.shortest_edge * lg) / (double)sh);
            ow = w <= h ? p.shortest_edge : nl;
            oh = w <= h ? nl : p.shortest_edge;
        }
        if (ow > (1 << 30) || oh > (1 << 30))
            return fail("image %d (%dx%d): resized to %lld x %lld pixels, more than 2^30 along one side", b, nx[b], ny[b], (long long)ow, (long long)oh);
        const int64_t ch = p.crop_height ? p.crop_height : oh, cw = p.crop_width ? p.crop_width : ow;
        const int64_t top = (oh - ch) / 2, left = (ow - cw) / 2;
        int64_t y0, y1, unused;
        pil_range(h, oh, top, p.resample, y0, unused);
        pil_range(h, oh, top + S - 1, p.resample, unused, y1);
        const double kx = pil_ksize(w, ow, p.resample), ky = pil_ksize(h, oh, p.resample);
        if ((kx + 2.0) * IMG_PROC_H_COLS * sizeof(int) > smem_max || (ky + 2.0) * IMG_PROC_V_ROWS * sizeof(int) > smem_max)
            return fail("image %d (%dx%d): resizing it to %lld x %lld pixels needs more taps than fit in shared memory", b, nx[b], ny[b],
                        (long long)ow, (long long)oh);
        kh = std::max(kh, kx);
        kv = std::max(kv, ky);
        ProcGeom &g = plan.geo[(size_t)b];
        g.tmp = plan.tmp_total;
        g.ow = (int)ow; g.oh = (int)oh; g.left = (int)left; g.top = (int)top; g.y0 = (int)y0; g.rows = (int)(y1 - y0);
        plan.max_rows = std::max(plan.max_rows, g.rows);
        plan.tmp_total += ((size_t)g.rows * S * 3 + 255) / 256 * 256;
    }
    plan.kh = (int)kh;
    plan.kv = (int)kv;
    return 0;
}

// The u8 entry points' checks: the images, and with an image processor the bilinear flag and the batch's geometry (plan_proc)
static int check_u8_call(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear)
{
    if (check_u8_images(images, nx, ny, batch)) return 1;
    if (!e->has_proc) return 0;
    if (bilinear) return fail("bilinear = %d: the engine's image processor fixes the resample (vitb200_set_image_proc)", bilinear);
    return plan_proc(e, nx, ny, batch);
}

// The image processor's two passes (image_proc_h_kernel, image_proc_v_kernel) as plan_proc laid them out
static int preprocess_proc(vitb200_engine *e, Slot &sl, const uint8_t *const *images, const int *nx, const int *ny, int batch,
                           float *images_f32_out)
{
    const vitb200_image_proc &p = e->proc;
    const ProcPlan &plan = e->proc_plan;
    const int S = e->hp.img_size;
    size_t table_off = 0;
    if (stage_u8(e, sl, images, nx, ny, batch, table_off, plan.geo.data(), plan.geo.size() * sizeof(ProcGeom))) return 1;
    if (plan.tmp_total > sl.proc_cap)
    {
        const size_t cap = plan.tmp_total + plan.tmp_total / 4;
        if (sl.d_proc) cudaFree(sl.d_proc);
        sl.d_proc = nullptr; sl.proc_cap = 0;
        CUDA_TRY(cudaMalloc((void **)&sl.d_proc, cap));
        sl.proc_cap = cap;
    }
    const PreImage *d_imgs = reinterpret_cast<const PreImage *>(sl.d_u8 + table_off);
    const ProcGeom *d_geo = reinterpret_cast<const ProcGeom *>(sl.d_u8 + table_off + (size_t)batch * sizeof(PreImage));
    cudaStream_t s = e->stream;
    float *d_f32 = images_f32_out ? sl.img : nullptr;
    const ProcNorm nm{p.rescale_factor, {p.mean[0], p.mean[1], p.mean[2]}, {p.std[0], p.std[1], p.std[2]}};
    const int KH = plan.kh, KV = plan.kv, max_rows = plan.max_rows;
    if (launch(e, image_proc_h_kernel, dim3((unsigned)((S + IMG_PROC_H_COLS - 1) / IMG_PROC_H_COLS),
                                            (unsigned)((max_rows + IMG_PROC_H_ROWS - 1) / IMG_PROC_H_ROWS), (unsigned)batch),
               dim3(256), (size_t)(KH + 2) * IMG_PROC_H_COLS * sizeof(int), s, LAUNCH_PLAIN, sl.d_u8, d_imgs, d_geo, sl.d_proc, S,
               (int)p.resample, KH) ||
        launch(e, image_proc_v_kernel, dim3((unsigned)((S + IMG_PROC_V_ROWS - 1) / IMG_PROC_V_ROWS), (unsigned)batch), dim3(256),
               (size_t)(KV + 2) * IMG_PROC_V_ROWS * sizeof(int), s, LAUNCH_PDL, (const uint8_t *)sl.d_proc, d_imgs, d_geo, d_f32, S,
               (int)p.resample, KV, nm, e->PA, e->hp.patch_size, e->KPp))
        return 1;
    if (images_f32_out) CUDA_TRY(cudaMemcpyAsync(images_f32_out, d_f32, (size_t)batch * 3 * S * S * sizeof(float), cudaMemcpyDeviceToHost, s));
    return 0;
}

static int preprocess_u8(vitb200_engine *e, Slot &sl, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                         float *images_f32_out)
{
    if (e->has_proc) return preprocess_proc(e, sl, images, nx, ny, batch, images_f32_out);
    size_t table_off = 0;
    if (stage_u8(e, sl, images, nx, ny, batch, table_off)) return 1;
    cudaStream_t s = e->stream;
    const int S = e->hp.img_size;
    float *d_f32 = images_f32_out ? sl.img : nullptr;
    if (launch(e, preprocess_kernel, dim3((unsigned)((S * S + 255) / 256), (unsigned)batch), dim3(256), 0, s, LAUNCH_PLAIN, sl.d_u8,
               reinterpret_cast<const PreImage *>(sl.d_u8 + table_off), d_f32, S, bilinear ? 1 : 0, e->PA, e->hp.patch_size, e->KPp))
        return 1;
    const size_t img_elems = (size_t)3 * S * S;
    if (images_f32_out) CUDA_TRY(cudaMemcpyAsync(images_f32_out, d_f32, (size_t)batch * img_elems * sizeof(float), cudaMemcpyDeviceToHost, s));
    return 0;
}

static int forward_u8_enqueue(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                              float *images_f32_out, float *probs, float *logits, int32_t *topk_idx, float *topk_prob, int k)
{
    if (!e || !images || !nx || !ny) return fail("null argument");
    if (image_only(e, "vitb200_forward_u8")) return 1;
    if (e->C != 3) return fail("vitb200_forward_u8 implements vit_image_preprocess (RGB, vit.cpp:289-305); this model takes %d-channel input", e->C);
    if (check_batch(e, batch) || check_k(e, k) || check_u8_call(e, images, nx, ny, batch, bilinear)) return 1;
    Slot &sl = begin_submit(e);
    if (preprocess_u8(e, sl, images, nx, ny, batch, bilinear, images_f32_out)) return 1;
    if ((probs || logits || (k > 0 && (topk_idx || topk_prob))) && classify_to_host(e, sl, nullptr, batch, probs, logits, topk_idx, topk_prob, k, nullptr))
        return 1;
    return end_submit(e, sl);
}

int vitb200_forward_u8_async(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                             float *probs, float *logits, int32_t *topk_idx, float *topk_prob, int k)
{
    return guarded(__func__, [&] { return forward_u8_enqueue(e, images, nx, ny, batch, bilinear, nullptr, probs, logits, topk_idx, topk_prob, k); });
}

int vitb200_forward_u8(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                       float *images_f32_out, float *probs, float *logits, int32_t *topk_idx, float *topk_prob, int k)
{
    return guarded(__func__, [&] {
        if (forward_u8_enqueue(e, images, nx, ny, batch, bilinear, images_f32_out, probs, logits, topk_idx, topk_prob, k)) return 1;
        return vitb200_sync(e);
    });
}

int vitb200_features_u8(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                        const vitb200_features_req *req, void *tokens, void *prelogits)
{
    return guarded(__func__, [&] {
        if (check_features(e, images, batch, req, tokens, prelogits)) return 1;
        if (!nx || !ny) return fail("vitb200_features_u8: null argument");
        if (e->C != 3) return fail("vitb200_features_u8 implements vit_image_preprocess (RGB, vit.cpp:289-305); this model takes %d-channel input", e->C);
        if (check_u8_call(e, images, nx, ny, batch, bilinear)) return 1;
        Slot &sl = begin_submit(e);
        if (preprocess_u8(e, sl, images, nx, ny, batch, bilinear, nullptr) || features_to_host(e, nullptr, batch, req, tokens, prelogits) ||
            end_submit(e, sl))
            return 1;
        return vitb200_sync(e);
    });
}

// Text recognition with the ViTSTR extension (reference extensions/vitstr.cpp): its grayscale preprocess (vitstr.cpp:128-201) writes
// the 1-channel patch matrix, the forward pass leaves the top-1 class and probability of every head token in the slot, and its greedy
// decode (vitstr.cpp:1020-1054) turns token rows 1 .. head_tokens-1 into class ids, a length and a score -- all on the device, in the
// same two-slot pipeline as vitb200_forward_async / vitb200_forward_u8_async.  Every argument is checked before anything is enqueued.
static int recognize_enqueue(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, float *images_f32_out,
                             int32_t *chars, int32_t *lengths, double *scores, float *probs)
{
    if (!e || !images || !nx || !ny) return fail("vitb200_recognize_u8: null argument");
    if (image_only(e, "vitb200_recognize_u8")) return 1;
    if (e->C != 1)
        return fail("vitb200_recognize_u8 implements the ViTSTR grayscale preprocess (1-channel, vitstr.cpp:128-201); this model takes "
                    "%d-channel input", e->C);
    if (e->head_tokens < 2) return fail("vitb200_recognize_u8: head_tokens is %d; the greedy decode reads token rows 1 .. head_tokens-1", e->head_tokens);
    if (e->hp.patch_size != 16 && e->hp.patch_size != 8) return fail("1-channel input: patch size %d not supported (8, 16)", e->hp.patch_size);
    if (check_batch(e, batch)) return 1;
    for (int b = 0; b < batch; ++b)
    {
        if (!images[b]) return fail("vitb200_recognize_u8: null argument (image %d)", b);
        if (nx[b] < 2 || ny[b] < 2) return fail("image %d is %dx%d pixels; the grayscale resize needs at least 2x2", b, nx[b], ny[b]);
    }
    Slot &sl = begin_submit(e);
    size_t table_off = 0;
    if (stage_u8(e, sl, images, nx, ny, batch, table_off)) return 1;
    cudaStream_t s = e->stream;
    const int S = e->hp.img_size, TH = e->head_tokens, C = e->hp.num_classes;
    float *d_f32 = images_f32_out ? sl.img : nullptr;
    if (launch(e, preprocess_gray_kernel, dim3((unsigned)((S * S + 255) / 256), (unsigned)batch), dim3(256), 0, s, LAUNCH_PLAIN, sl.d_u8,
               reinterpret_cast<const PreImage *>(sl.d_u8 + table_off), d_f32, S, e->PA, e->hp.patch_size, e->KPp))
        return 1;
    if (images_f32_out) CUDA_TRY(cudaMemcpyAsync(images_f32_out, d_f32, (size_t)batch * S * S * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (chars || lengths || scores || probs)
    {
        // patches ready (d_images = NULL); top-1 of every head token into the slot; probabilities only when asked for
        if (run_forward_graphed(e, nullptr, batch, probs ? sl.probs : nullptr, nullptr, sl.topk_idx, sl.topk_val, 1, s) ||
            launch(e, vitstr_decode_kernel, dim3((batch + 127) / 128), dim3(128), 0, s, LAUNCH_PLAIN, sl.topk_idx, sl.topk_val, batch, TH, sl.chars,
                   sl.len, sl.score))
            return 1;
        if (chars) CUDA_TRY(cudaMemcpyAsync(chars, sl.chars, (size_t)batch * (TH - 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        if (lengths) CUDA_TRY(cudaMemcpyAsync(lengths, sl.len, (size_t)batch * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        if (scores) CUDA_TRY(cudaMemcpyAsync(scores, sl.score, (size_t)batch * sizeof(double), cudaMemcpyDeviceToHost, s));
        if (probs) CUDA_TRY(cudaMemcpyAsync(probs, sl.probs, (size_t)batch * TH * C * sizeof(float), cudaMemcpyDeviceToHost, s));
    }
    return end_submit(e, sl);
}

int vitb200_recognize_u8_async(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int32_t *chars,
                               int32_t *lengths, double *scores, float *probs)
{
    return guarded(__func__, [&] { return recognize_enqueue(e, images, nx, ny, batch, nullptr, chars, lengths, scores, probs); });
}

int vitb200_recognize_u8(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, float *images_f32_out,
                         int32_t *chars, int32_t *lengths, double *scores, float *probs)
{
    return guarded(__func__, [&] {
        if (recognize_enqueue(e, images, nx, ny, batch, images_f32_out, chars, lengths, scores, probs)) return 1;
        return vitb200_sync(e);
    });
}

int vitb200_encode_text(vitb200_engine *e, const int32_t *ids, int batch, float *embeds, const vitb200_features_req *req, void *tokens)
{
    return guarded(__func__, [&]() -> int {
        if (check_text(e, ids, batch, embeds, req, tokens)) return 1;
        const int N = e->N, D = e->hp.hidden_size;
        for (int b = 0; b < batch; ++b)
            for (int t = 0; t < N; ++t)
                if (ids[(size_t)b * N + t] < 0 || ids[(size_t)b * N + t] >= e->V)
                    return fail("vitb200_encode_text: sequence %d, position %d: id %d out of range (0..%d)", b, t, ids[(size_t)b * N + t], e->V - 1);
        CUDA_TRY(cudaSetDevice(e->device));
        Slot &sl = begin_submit(e);
        cudaStream_t s = e->stream, cs = e->copy_stream;
        // the ids into this call's slot once its previous call has consumed them; the token rows are staged in TOKS (written mid-schedule)
        if (e->submits >= 2) CUDA_TRY(cudaStreamWaitEvent(cs, sl.ev_done, 0));
        CUDA_TRY(cudaMemcpyAsync(sl.ids, ids, (size_t)batch * N * sizeof(int32_t), cudaMemcpyHostToDevice, cs));
        CUDA_TRY(cudaEventRecord(sl.ev_h2d, cs));
        CUDA_TRY(cudaStreamWaitEvent(s, sl.ev_h2d, 0));
        if (run_text_graphed(e, sl.ids, batch, embeds ? sl.logits : nullptr, req, tokens ? e->TOKS : nullptr, s)) return 1;
        if (embeds) CUDA_TRY(cudaMemcpyAsync(embeds, sl.logits, (size_t)batch * e->hp.num_classes * sizeof(float), cudaMemcpyDeviceToHost, s));
        if (tokens)
            CUDA_TRY(cudaMemcpyAsync(tokens, e->TOKS, (size_t)batch * N * D * features_elem_bytes(req), cudaMemcpyDeviceToHost, s));
        if (end_submit(e, sl)) return 1;
        return vitb200_sync(e);
    });
}

int vitb200_encode_text_device(vitb200_engine *e, const int32_t *d_ids, int batch, float *d_embeds, const vitb200_features_req *req,
                               void *d_tokens, void *stream)
{
    return guarded(__func__, [&]() -> int {
        if (check_text(e, d_ids, batch, d_embeds, req, d_tokens)) return 1;
        if (((uintptr_t)d_embeds | (uintptr_t)d_tokens) % 16 != 0) return fail("vitb200_encode_text_device: output buffers must be 16-byte aligned");
        CUDA_TRY(cudaSetDevice(e->device));
        e->launches = 0;
        return run_text_graphed(e, d_ids, batch, d_embeds, req, d_tokens, stream ? (cudaStream_t)stream : e->stream);
    });
}

// vitb200_test_gemm and vitb200_test_gemm_layer_scale: gamma is the LayerScale epilogue's [N] (NULL for every other epilogue)
static int test_gemm_f16(int device, int M, int N, int K, int epilogue, const uint16_t *A, const uint16_t *W, const float *bias,
                         const float *gamma, const float *resid, float *out)
{
    if (!A || !W || !bias || !out) return fail("null argument");
    // the patch-embedding epilogue needs the position table and token geometry, which this hook does not take: every other runs here
    if (!gemm_epi(epilogue).valid || epilogue == EPI_PATCH_F32)
        return fail("GEMM epilogue %d not supported (%s; %d through vitb200_test_gemm_layer_scale)", epilogue,
                    gemm_epi_list([](int epi) { return epi != EPI_PATCH_F32 && epi != EPI_BIAS_SCALE_RESID_F32; }).c_str(), EPI_BIAS_SCALE_RESID_F32);
    if (K % 8 != 0) return fail("K must be a multiple of 8");
    if (gemm_epi(epilogue).resid && !resid) return fail("resid required");
    if ((epilogue == EPI_BIAS_SCALE_RESID_F32) != (gamma != nullptr))
        return fail("gamma goes with the LayerScale epilogue %d only (vitb200_test_gemm_layer_scale)", EPI_BIAS_SCALE_RESID_F32);
    return test_gemm_run<GEMM_OP_F16>(device, M, N, K, epilogue, A, W, bias, nullptr, 0.f, gamma, resid, out);
}

int vitb200_test_gemm(int device, int M, int N, int K, int epilogue, const uint16_t *A, const uint16_t *W, const float *bias,
                      const float *resid, float *out)
{
    return guarded(__func__, [&] { return test_gemm_f16(device, M, N, K, epilogue, A, W, bias, nullptr, resid, out); });
}

int vitb200_test_gemm_layer_scale(int device, int M, int N, int K, const uint16_t *A, const uint16_t *W, const float *bias,
                                  const float *gamma, const float *resid, float *out)
{
    return guarded(__func__, [&]() -> int {
        if (!gamma || !resid) return fail("null argument");
        return test_gemm_f16(device, M, N, K, EPI_BIAS_SCALE_RESID_F32, A, W, bias, gamma, resid, out);
    });
}

int vitb200_test_layernorm(int device, int rows, int D, const float *x, const float *w, const float *b, float eps, float *y)
{
    return guarded(__func__, [&] {
        if (!x || !w || !b || !y || rows < 1 || D < 4 || D % 4 != 0 || D > LN_MAX_HIDDEN) return fail("bad argument");
        EnginePtr owner;
        __half *dy = nullptr;
        if (test_layernorm_impl(device, rows, D, x, w, b, eps, &dy, nullptr, owner)) return 1;
        return tap_f16(y, dy, (size_t)rows * D, owner->stream);
    });
}

int vitb200_test_quantize_fp8(const uint16_t *w_f16, int64_t n, uint8_t *q, float *scale)
{
    return guarded(__func__, [&] {
        if (!w_f16 || !q || !scale || n < 1) return fail("bad argument");
        *scale = quantize_e4m3(w_f16, (size_t)n, q);
        return 0;
    });
}

// Stand-alone run of the e4m3 GEMM as the FP8 engine launches it (qkv and fc1): A [M][K] and W [N][K] e4m3 bytes, a_scale [M], w_scale.
int vitb200_test_gemm_fp8(int device, int M, int N, int K, int epilogue, const uint8_t *A, const float *a_scale, const uint8_t *W,
                          float w_scale, const float *bias, float *out)
{
    return guarded(__func__, [&]() -> int {
        if (!A || !a_scale || !W || !bias || !out) return fail("null argument");
        if (M < 1 || N < 4 || K < 16 || K % 16 != 0) return fail("bad shape (M >= 1, N >= 4, K >= 16 and K %% 16 == 0)");
        if (!gemm_epi(epilogue).e4m3)
            return fail("e4m3 GEMM epilogue %d not supported (%s)", epilogue, gemm_epi_list([](int epi) { return gemm_epi(epi).e4m3; }).c_str());
        return test_gemm_run<GEMM_OP_E4M3>(device, M, N, K, epilogue, A, W, bias, a_scale, w_scale, nullptr, nullptr, out);
    });
}

// The qkv and pool k | v GEMMs as the engine runs them at head dim 64: the output in head-major planes, f16 or e4m3 operands
int vitb200_test_gemm_planes(int device, int M, int N, int K, int epilogue, int64_t plane_rows, int e4m3, const void *A, const float *a_scale,
                             const void *W, float w_scale, const float *bias, uint16_t *hi, uint16_t *lo)
{
    return guarded(__func__, [&]() -> int {
        if (!A || !W || !bias || !hi) return fail("null argument");
        if (epilogue != EPI_BIAS_F16 && epilogue != EPI_BIAS_F16_HILO)
            return fail("head-major GEMM epilogue %d not supported (%d, %d: the qkv and k | v GEMMs)", epilogue, EPI_BIAS_F16, EPI_BIAS_F16_HILO);
        if ((epilogue == EPI_BIAS_F16_HILO) != (lo != nullptr)) return fail("lo goes with epilogue %d, and only with it", EPI_BIAS_F16_HILO);
        if (e4m3 != 0 && e4m3 != 1) return fail("e4m3 = %d out of range (0 f16 operands, 1 e4m3)", e4m3);
        if (e4m3 != (a_scale != nullptr)) return fail("a_scale goes with e4m3 operands, and only with them");
        const int kmul = e4m3 ? 16 : 8; // 16-byte operand rows
        if (M < 1 || K < kmul || K % kmul != 0 || N < 64 || N % 64 != 0)
            return fail("bad shape (M >= 1, N a multiple of 64, K a multiple of %d; got M = %d, N = %d, K = %d)", kmul, M, N, K);
        if (plane_rows < M || plane_rows > INT32_MAX) return fail("plane_rows = %lld out of range (M = %d .. 2^31 - 1)", (long long)plane_rows, M);
        if (e4m3)
            return test_gemm_run<GEMM_OP_E4M3>(device, M, N, K, epilogue, (const uint8_t *)A, (const uint8_t *)W, bias, a_scale, w_scale,
                                               nullptr, nullptr, nullptr, (size_t)plane_rows, hi, lo);
        return test_gemm_run<GEMM_OP_F16>(device, M, N, K, epilogue, (const uint16_t *)A, (const uint16_t *)W, bias, nullptr, 0.f, nullptr,
                                          nullptr, nullptr, (size_t)plane_rows, hi, lo);
    });
}

// The FP8 engine's LayerNorm 1 / 2 alone, launched as vitb200_test_layernorm launches the f16 one: q [rows][D] e4m3 bytes, sa [rows].
int vitb200_test_layernorm_fp8(int device, int rows, int D, const float *x, const float *w, const float *b, float eps, uint8_t *q, float *sa)
{
    return guarded(__func__, [&]() -> int {
        if (!x || !w || !b || !q || !sa || rows < 1 || D < 4 || D % 16 != 0 || D > LN_MAX_HIDDEN) return fail("bad argument");
        EnginePtr owner;
        __nv_fp8_e4m3 *dq = nullptr;
        float *ds = nullptr;
        if (test_layernorm_impl(device, rows, D, x, w, b, eps, &dq, &ds, owner)) return 1;
        CUDA_TRY(cudaMemcpy(q, dq, (size_t)rows * D, cudaMemcpyDeviceToHost));
        return tap_f32(sa, ds, rows, owner->stream);
    });
}

// q8_0 linear layer on the integer tensor cores (gemm_q8_wgmma.cuh; prototype for BASELINE.json configs[4]): x [M][K] f32 is
// quantised on the device exactly as the reference quantises activation rows, w is a q8_0 tensor in the model-file layout
// ([N][K/32] blocks of {f16 d; int8 q[32]}, ggml-quants.h:42-46).  Outputs: y [M][N] f32, and (optional) the quantised activations
// xq [M][K] int8, xd [M][K/32] f32.  iters > 0 additionally times `iters` back-to-back GEMM launches (CUDA events) into *ms_per_launch.
int vitb200_test_gemm_q8(int device, int M, int N, int K, const float *x, const void *w_q8_0, const float *bias, float *y,
                         int8_t *xq, float *xd, int iters, float *ms_per_launch)
{
    return guarded(__func__, [&]() -> int {
        if (!x || !w_q8_0 || !bias || !y || M < 1 || N < 1 || K < 1) return fail("bad argument");
        if (K % Q8_BK != 0) return fail("K must be a multiple of %d", Q8_BK);
        if (N % 4 != 0) return fail("N must be a multiple of 4");
        EnginePtr owner;
        if (scratch_engine(device, owner)) return 1;
        vitb200_engine *e = owner.get();
        cudaStream_t s = e->stream;
        const int KB = K / 32;
        // repack the 34-byte blocks: int8 plane [N][K] + transposed scale plane [K/32][N]
        std::vector<int8_t> wq((size_t)N * K);
        std::vector<float> wdT((size_t)KB * N);
        const uint8_t *blk = (const uint8_t *)w_q8_0;
        for (int n = 0; n < N; ++n)
            for (int b = 0; b < KB; ++b)
            {
                const uint8_t *src = blk + ((size_t)n * KB + b) * 34;
                uint16_t du;
                memcpy(&du, src, 2);
                wdT[(size_t)b * N + n] = host_f16_to_f32(du);
                memcpy(&wq[(size_t)n * K + (size_t)b * 32], src + 2, 32);
            }
        float *dX = nullptr, *dAd = nullptr, *dWd = nullptr, *dB = nullptr, *dY = nullptr;
        int8_t *dAq = nullptr, *dWq = nullptr;
        if (upload(e, &dX, x, (size_t)M * K) || dev_alloc(e, &dAq, (size_t)M * K) || dev_alloc(e, &dAd, (size_t)M * KB) ||
            upload(e, &dWq, wq.data(), wq.size()) || upload(e, &dWd, wdT.data(), wdT.size()) || upload(e, &dB, bias, N) ||
            dev_alloc(e, &dY, (size_t)M * N))
            return 1;
        CUtensorMap tA, tW, tAd, tWd;
        const cuuint64_t Mu = (cuuint64_t)M, Nu = (cuuint64_t)N, Ku = (cuuint64_t)K, KBu = (cuuint64_t)KB;
        if (make_tmap(&tA, CU_TENSOR_MAP_DATA_TYPE_UINT8, dAq, {Ku, Mu}, {Ku}, {Q8_BK, Q8_BM}) ||
            make_tmap(&tW, CU_TENSOR_MAP_DATA_TYPE_UINT8, dWq, {Ku, Nu}, {Ku}, {Q8_BK, Q8_BN}) ||
            make_tmap(&tAd, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dAd, {KBu, Mu}, {4 * KBu}, {4, Q8_BM}, CU_TENSOR_MAP_SWIZZLE_NONE) ||
            make_tmap(&tWd, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dWd, {Nu, KBu}, {4 * Nu}, {Q8_BN, 4}, CU_TENSOR_MAP_SWIZZLE_NONE))
            return 1;
        Q8GemmParams p{};
        p.M = M; p.N = N; p.K = K; p.bias = dB; p.out = dY; p.ldo = N;
        const int grid = ((M + Q8_BM - 1) / Q8_BM) * ((N + Q8_BN - 1) / Q8_BN); // one CTA per tile
        auto gemm = [&] { return launch(e, gemm_q8_wgmma_kernel, dim3(grid), dim3(Q8_THREADS), Q8_SMEM_BYTES, s, LAUNCH_PLAIN, tA, tW, tAd, tWd, p); };
        auto run = [&] {
            const long long n_blocks = (long long)M * KB;
            const int qthreads = 256;
            const long long qgrid = (n_blocks * 8 + qthreads - 1) / qthreads;
            if (launch(e, quantize_q8_0_kernel, dim3((unsigned)qgrid), dim3(qthreads), 0, s, LAUNCH_PLAIN, dX, dAq, dAd, n_blocks)) return 1;
            return gemm();
        };
        if (run_scratch(e, "q8_0 GEMM kernel", run) || tap_f32(y, dY, (size_t)M * N, s)) return 1;
        if (xq) CUDA_TRY(cudaMemcpy(xq, dAq, (size_t)M * K, cudaMemcpyDeviceToHost));
        if (xd) CUDA_TRY(cudaMemcpy(xd, dAd, (size_t)M * KB * 4, cudaMemcpyDeviceToHost));
        if (iters > 0 && ms_per_launch)
        {
            // the engine's event pool is destroyed with it
            cudaEvent_t t0 = nullptr, t1 = nullptr;
            CUDA_TRY(cudaEventCreate(&t0));
            e->event_pool.push_back(t0);
            CUDA_TRY(cudaEventCreate(&t1));
            e->event_pool.push_back(t1);
            auto timed = [&]() -> int {
                CUDA_TRY(cudaEventRecord(t0, s));
                for (int i = 0; i < iters; ++i)
                    if (gemm()) return 1;
                CUDA_TRY(cudaEventRecord(t1, s));
                return 0;
            };
            if (run_scratch(e, "q8_0 GEMM kernel", timed)) return 1;
            float ms = 0.f;
            CUDA_TRY(cudaEventElapsedTime(&ms, t0, t1));
            *ms_per_launch = ms / (float)iters;
        }
        return 0;
    });
}

} // extern "C"

// ------------------------------------------------------------------------------------------------
// Legacy-ggml model file reader (the format reference vit_model_load parses, vit.cpp:308-712; written by
// convert-pth-to-ggml.py:105-158).  Validation mirrors the reference: magic, known tensor names, element
// counts; failures return non-zero with a message, never abort.

static int create_from_file(const char *path, int device, int max_batch, int head_tokens, bool fp8, vitb200_engine **out)
{
    if (!path || !out) return fail("null argument");
    *out = nullptr;
    std::ifstream fin(path, std::ios::binary);
    if (!fin) return fail("failed to open '%s'", path);
    fin.seekg(0, std::ios::end);
    const std::streamoff fend = fin.tellg();
    // a directory or an unseekable stream reports -1; model files beyond 64 GiB are not something this loader stages in host memory
    if (!fin || fend < 0) return fail("failed to read '%s' (not a regular file)", path);
    if ((unsigned long long)fend > (64ull << 30)) return fail("model file '%s' is too large (%lld bytes)", path, (long long)fend);
    const size_t fsize = (size_t)fend;
    fin.seekg(0);
    std::vector<char> buf(fsize);
    fin.read(buf.data(), (std::streamsize)fsize);
    if (!fin) return fail("failed to read '%s'", path);
    // a true GGUF container (SURVEY.md 8(f) rank 3) or the legacy-ggml file the reference itself reads; both parsers live in
    // gguf_file.hpp (plain host C++, fuzzed under ASan/UBSan by tests/cpp/gguf_fuzz.cpp) and fill the same structure
    GgufModel g;
    const bool is_gguf = fsize >= 4 && memcmp(buf.data(), "GGUF", 4) == 0;
    if (is_gguf)
    {
        if (!parse_gguf(buf.data(), fsize, g)) return fail("invalid GGUF file '%s': %s", path, g.error.c_str());
    }
    else if (!parse_legacy_ggml(buf.data(), fsize, g))
        return fail("invalid model file '%s' (%s)", path, g.error.c_str());
    vitb200_hparams hp{};
    auto i32 = [](int64_t v) { return (int32_t)(v < -1 ? -1 : (v > (1 << 30) ? (1 << 30) : v)); }; // out-of-range values stay out of range
    hp.hidden_size = i32(g.hidden_size); hp.num_hidden_layers = i32(g.num_hidden_layers);
    hp.num_attention_heads = i32(g.num_attention_heads); hp.num_classes = i32(g.num_classes);
    hp.patch_size = i32(g.patch_size); hp.img_size = i32(g.img_size); hp.ftype = i32(g.ftype); hp.eps = g.eps;
    if (hp.num_hidden_layers < 1 || hp.num_hidden_layers > 4096) return fail("invalid model file '%s' (num_hidden_layers %d)", path, hp.num_hidden_layers);
    auto tensor_list = [&](std::vector<vitb200_tensor> &ts) {
        ts.resize(g.tensors.size());
        for (size_t i = 0; i < g.tensors.size(); ++i)
        {
            ts[i].name = g.tensors[i].name.c_str();
            ts[i].data = buf.data() + g.tensors[i].offset;
            ts[i].type = g.tensors[i].type;
            ts[i].n_dims = g.tensors[i].n_dims;
            for (int j = 0; j < 4; ++j) ts[i].ne[j] = g.tensors[i].ne[j];
        }
    };
    if (g.text)
    {
        // a CLIP or SigLIP text tower: token_embd, pos_embed, the blocks, norm and head
        if (head_tokens != 1) return fail("'%s' is a text tower: head_tokens must be 1 (got %d)", path, head_tokens);
        if (g.text_causal != 0 && g.text_causal != 1) return fail("invalid model file '%s' (vit.text.causal %lld)", path, (long long)g.text_causal);
        const vitb200_text_arch ta{i32(g.text_context), (int32_t)g.text_causal, g.text_pool, i32(g.text_eos), g.activation, g.logit_scale, g.logit_bias};
        const int expected = 12 * hp.num_hidden_layers + 6;
        if ((int)g.tensors.size() != expected) return fail("model file has %d tensors, but %d tensors were expected", (int)g.tensors.size(), expected);
        std::vector<vitb200_tensor> ts;
        tensor_list(ts);
        return create_text_impl(&hp, &ta, ts.data(), (int)ts.size(), device, max_batch, fp8, out);
    }
    if (g.pre_norm != 0 && g.pre_norm != 1) return fail("invalid model file '%s' (vit.pre_norm %lld)", path, (long long)g.pre_norm);
    if (g.layer_scale != 0 && g.layer_scale != 1) return fail("invalid model file '%s' (vit.layer_scale %lld)", path, (long long)g.layer_scale);
    if (g.reg_tokens < 0 || g.reg_tokens > VB_MAX_REG_TOKENS)
        return fail("invalid model file '%s' (vit.reg_tokens %lld, 0..%d)", path, (long long)g.reg_tokens, VB_MAX_REG_TOKENS);
    const vitb200_arch arch{(int32_t)g.pre_norm, g.activation, (int32_t)g.layer_scale, (int32_t)g.reg_tokens, g.pool};
    // vit.cpp:697, plus norm_pre.weight / .bias, the ls1 / ls2 gammas of every block and reg_token; SigLIP's pools have no cls_token,
    // and the attention-pooling head has 13 tensors of its own
    const int expected = 4 + 12 * hp.num_hidden_layers + 4 + 2 * arch.pre_norm + 2 * hp.num_hidden_layers * arch.layer_scale + (arch.reg_tokens > 0) -
                         (arch.pool >= 2) + (arch.pool == 2 ? kPoolTensorCount : 0);
    if ((int)g.tensors.size() != expected) return fail("model file has %d tensors, but %d tensors were expected", (int)g.tensors.size(), expected);
    std::vector<vitb200_tensor> ts;
    tensor_list(ts);
    const vitb200_image_proc proc{i32(g.ip_shortest_edge), i32(g.ip_height), i32(g.ip_width), i32(g.ip_crop_height), i32(g.ip_crop_width),
                                  i32(g.ip_resample), g.ip_rescale_factor, {g.ip_mean[0], g.ip_mean[1], g.ip_mean[2]},
                                  {g.ip_std[0], g.ip_std[1], g.ip_std[2]}};
    if (g.has_image_proc)
    {
        // the input channels as create_impl takes them, from the patch kernel [P, P, C, D] (a file without one fails there)
        const vitb200_tensor *pw = find_tensor(ts.data(), (int)ts.size(), "patch_embed.proj.weight");
        if (check_image_proc(pw ? (int)dim_of(pw, 2) : 3, hp.img_size, proc))
            return fail("invalid model file '%s' (vit.%s)", path, std::string(g_err).c_str());
    }
    if (create_impl(&hp, &arch, ts.data(), (int)ts.size(), device, max_batch, head_tokens, fp8, out, &g.labels)) return 1;
    return g.has_image_proc ? set_image_proc(*out, &proc) : 0;
}

extern "C" int vitb200_create_from_file(const char *path, int device, int max_batch, vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_from_file(path, device, max_batch, 1, false, out); });
}

extern "C" int vitb200_create_from_file_ex(const char *path, int device, int max_batch, int head_tokens, vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_from_file(path, device, max_batch, head_tokens, false, out); });
}

extern "C" int vitb200_create_from_file_fp8(const char *path, int device, int max_batch, int head_tokens, vitb200_engine **out)
{
    return guarded(__func__, [&] { return create_from_file(path, device, max_batch, head_tokens, true, out); });
}
