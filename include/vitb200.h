/* vitb200.h -- C ABI of the Hopper-native (sm_90a) ViT forward path (drop-in boundary for staghado/vit.cpp).
 *
 * The reference exposes the forward path as C++ free functions in vit.h:
 *     bool vit_model_load(const std::string&, vit_model&)                       (reference vit.h:120, vit.cpp:308-712)
 *     int  vit_predict(const vit_model&, vit_state&, const image_f32,
 *                      const vit_params&, std::vector<std::pair<float,int>>&)   (reference vit.h:122, vit.cpp:1004-1075)
 * There is no plugin registry; the seam is the vit_predict function boundary (SURVEY.md 8b).  The entry points
 * below are what a binding at that seam needs: plain pointers and sizes, no C++ or torch types.  INTEGRATION.md
 * shows the vit.h-side shim (vit_predict re-implemented on top of this header) and the ctypes binding.
 *
 * Conventions (same as the reference, SURVEY.md 8b "Error convention"): functions return 0 on success and a
 * non-zero code on failure; a message is retrievable with vitb200_last_error(); nothing throws or aborts.
 * An engine is bound to ONE CUDA device and is thread-compatible (not thread-safe), like vit_state.
 */
#ifndef VITB200_H
#define VITB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vitb200_engine vitb200_engine;

/* Mirrors the POD part of vit_hparams (reference vit.h:20-37). */
typedef struct vitb200_hparams
{
    int32_t hidden_size;
    int32_t num_hidden_layers;
    int32_t num_attention_heads;
    int32_t num_classes;
    int32_t patch_size;
    int32_t img_size;
    int32_t ftype; /* the model file's ftype (reference vit.cpp:385-414): 0 f32, 1 f16, 2 q4_0, 3 q4_1, 6 q5_0, 7 q5_1, 8 q8_0.
                    * Informational: what counts is each tensor's own `type`.  f16 is the native path; every other format the
                    * reference loader accepts is converted to f16 once at upload (DESIGN.md section 3) */
    float eps;     /* layer-norm epsilon, 1e-6 in the reference (vit.h:29) */
} vitb200_hparams;

/* One host tensor, as found in vit_model::tensors (reference vit.h:88, names at vit.cpp:518-579).
 * `type` uses ggml's type ids for the formats the loader accepts: 0 = F32, 1 = F16, 2 = Q4_0, 3 = Q4_1, 6 = Q5_0, 7 = Q5_1,
 * 8 = Q8_0 (block layouts ggml-quants.h:11-47), plus 30 = BF16 for GGUF containers.  `ne` is ggml order (ne[0] fastest); entries
 * at index >= n_dims are ignored (treated as 1).  Shapes are checked against the reference's declarations (vit.cpp:510-574) and
 * names must be unique. */
typedef struct vitb200_tensor
{
    const char *name;
    const void *data;
    int32_t type;
    int32_t n_dims;
    int64_t ne[4];
} vitb200_tensor;

/* Create an engine from weights that already live in host memory (this is what a vit.h-side shim calls with
 * the contents of vit_model::tensors).  Weights are repacked and uploaded once; the host arena is not retained.
 * max_batch bounds the batch accepted by vitb200_forward*.  Replaces, per model, what the reference re-does per
 * image in vit_predict (graph build x2, ggml_allocr, thread pool; vit.cpp:1009-1036).
 * Accepted shapes (every create function; anything else fails here, with a message naming the limit, not in the first forward):
 *   head dim 64 or 80 (hidden_size = 64 or 80 * num_attention_heads), hidden_size <= 2048 (the widest LayerNorm row a warp holds);
 *   head dim 72 (SigLIP So400m) with the SigLIP pools 2 and 3 only (vitb200_create_arch) and in SigLIP text towers;
 *   head dim 80 (ViT-H/14) without the attention-pooling head (vitb200_arch.pool = 2, whose kernel is 64 or 72 columns wide);
 *   patch_size 8, 14, 16 or 32 for 3-channel input, 8 or 16 for 1-channel input, dividing img_size (with pools 2 and 3 it need not: the
 *   grid is then G = floor(img_size / patch_size), as HF's valid-padding conv takes it; with patch size 8, 16 or 32, whose patch
 *   embedding reads pixel rows in 16-byte loads, such an img_size must then be a multiple of 4);
 *   at most 896 tokens at head dim 64, 800 at head dim 72 and 640 at head dim 80, G^2 + 1 (K and V of one attention head in 227 KB of
 *   shared memory);
 *   FP8 engines (vitb200_create_fp8, fp8 = 1 of vitb200_create_arch and vitb200_create_text): hidden_size a multiple of 16 (the e4m3
 *   activation rows are read in 16-byte strides), so head dim 72 with an even head count. */
int vitb200_create(const vitb200_hparams *hp, const vitb200_tensor *tensors, int n_tensors, int device, int max_batch,
                   vitb200_engine **out);

/* Same, reading the legacy-ggml model file the reference's vit_model_load parses (vit.cpp:308-712), or a true GGUF v2/v3
 * container with the same tensors (vit.cpp_b200/csrc/gguf_file.hpp). */
int vitb200_create_from_file(const char *path, int device, int max_batch, vitb200_engine **out);

/* The ViTSTR extension of the reference (extensions/vitstr.cpp): the same encoder on a 1-channel image -- the channel count
 * is taken from the patch kernel's shape [P, P, C, D] (vitstr.cpp:482; C = 3 in vit.cpp:515) -- whose classifier reads the
 * first `head_tokens` tokens of every image instead of token 0 (vitstr.cpp:864-903: 25 tokens -> LayerNorm -> head ->
 * soft-max per token).  head_tokens = 1 is vitb200_create / vitb200_create_from_file.  With head_tokens = n every per-image
 * output of vitb200_forward* becomes n consecutive rows: probs/logits float32[batch][n][num_classes], top-k [batch][n][k];
 * images are float32[batch][img][img][C]. */
int vitb200_create_ex(const vitb200_hparams *hp, const vitb200_tensor *tensors, int n_tensors, int device, int max_batch,
                      int head_tokens, vitb200_engine **out);
int vitb200_create_from_file_ex(const char *path, int device, int max_batch, int head_tokens, vitb200_engine **out);
/* FP8 engine: the same arguments and the same entry points (forward in every form, u8, features, recognition, sharded), with the
 * qkv and fc1 linear layers of every block on the e4m3 tensor cores.  Numerics (everything not listed is the f16 engine's):
 *   weights     attn.qkv.weight and mlp.fc1.weight, taken as the f16 values the f16 engine would store (any file format), get one f32
 *               scale per tensor, sw = amax / 448 (1 when amax = 0), and are stored only as qw = e4m3_rn_satfinite(w * (448 / amax)).
 *   activations LayerNorms 1 and 2 quantise each token row of their f32 output y (the values the f16 engine rounds to f16) with its
 *               own scale: sa = amax / 448 over the row (1 when amax = 0), q = e4m3_rn_satfinite(y * (448 / amax)).
 *   GEMM        x[m][n] = acc * (sa[m] * sw) + bias[n], acc = sum_k q[m][k] qw[n][k] accumulated by the tensor cores in f32 (on Hopper
 *               an e4m3 MMA adds its products with fewer than f32's mantissa bits); then the f16 engine's epilogue on x (qkv: hi + lo
 *               split for the attention; fc1: f16, GELU, f16).
 * proj, fc2, the patch embedding, attention, the final LayerNorm and the head are unchanged.  The ln1 / ln2 debug taps return q * sa.
 * The accuracy cost against the reference is stated in README.md. */
int vitb200_create_fp8(const vitb200_hparams *hp, const vitb200_tensor *tensors, int n_tensors, int device, int max_batch,
                       int head_tokens, vitb200_engine **out);
int vitb200_create_from_file_fp8(const char *path, int device, int max_batch, int head_tokens, vitb200_engine **out);
/* ---- architecture variants: CLIP image towers (no reference counterpart) ------------------------------------------------------
 * The reference's ViT is timm's VisionTransformer with tanh GELU and no pre-norm.  CLIP towers (OpenAI and LAION CLIP, LLaVA's vision
 * encoder, timm's vit_*_clip_* models) add a LayerNorm on the embeddings and use another MLP activation. */
typedef struct vitb200_arch
{
    int32_t pre_norm;   /* 0: none (the reference).  1: LayerNorm 'norm_pre.weight' / 'norm_pre.bias' [D] (HF CLIP's pre_layrnorm, timm's
                         *    norm_pre) on every token row of the embeddings (cls included), written back to the f32 residual stream, before
                         *    block 0.  Same arithmetic and eps as the block LayerNorms, f32 out. */
    int32_t activation; /* MLP activation after fc1: 0 GELU, tanh form, through ggml's f16 table (the reference, unchanged); 1 GELU, erf form,
                         * 0.5 x (1 + erf(x / sqrt 2)); 2 QuickGELU, x / (1 + exp(-1.702 x)); 3 GELU, tanh form as PyTorch's
                         * gelu(approximate='tanh') ('gelu_pytorch_tanh'), 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))), with pools 2 and 3
                         * only (SigLIP); 4 SwiGLU ('swiglu', DINOv2 ViT-g, pools 0 and 1 only): 'mlp.fc1.weight' is [2 F][D] and
                         * 'mlp.fc1.bias' [2 F] in HF's order (x1 rows 0 .. F-1, then the x2 rows), 'mlp.fc2.weight' [D][F], and
                         * h = f16(silu(x1) * x2), silu(x) = x / (1 + exp(-x)); F is read from block 0's fc1, every block must agree,
                         * F % 8 == 0 and 8 <= F <= 8 D.  Forms 1 to 4 take x = acc + bias (FP8 engine: acc (sa sw) + bias) in f32, without
                         * rounding it to f16 first, and store f16(act(x)). */
    /* DINOv2 (HF Dinov2Model / Dinov2WithRegistersModel and their ForImageClassification heads).  Zero is the behaviour above. */
    int32_t layer_scale; /* 0 or 1.  1: x = x + f32(f32(acc + bias) * gamma[n]) after proj ('blocks.{i}.ls1.gamma' [D]) and fc2
                          * ('blocks.{i}.ls2.gamma' [D]), gamma kept in f32 (HF's LayerScale order; not folded into the f16 weights). */
    int32_t reg_tokens;  /* R = 0..16 register tokens ('reg_token' [1, R, D]).  Token rows per image are [cls, reg_1..R, patch_1..P],
                          * N = P + 1 + R; 'pos_embed' is [1, N, D] with the R register rows after the class row (zero for DINOv2). */
    int32_t pool;        /* 0: the head reads the first head_tokens rows (the reference).  1: the head reads one row of 2 D per image,
                          * LN(token 0) || mean over the P patch rows of LN(patch) (registers excluded, LN = the final LayerNorm):
                          * DINOv2's classifier input.  'head.weight' is then [C][2 D] and head_tokens must be 1.
                          * SigLIP (HF SiglipVisionModel, SiglipForImageClassification): pools 2 and 3 have NO class token -- the token rows
                          * are [patch_1..P], N = P, 'pos_embed' is [1, P, D], there is no 'cls_token', reg_tokens = 0, head_tokens = 1.
                          * 2 'map': the attention-pooling head (HF SiglipMultiheadAttentionPoolingHead, timm AttentionPoolLatent): one learned
                          *   probe 'attn_pool.latent' [1, 1, D], q = latent Wq^T + bq ('attn_pool.q.*', computed once at load in f64, kept
                          *   in f32), attends per head over k | v = LN(rows) Wkv^T + bkv ('attn_pool.kv.*' [2 D, D], rows k then v; LN = the
                          *   final LayerNorm) with softmax(q k / sqrt(hd)) in f32 (1 / 8 at head dim 64, f32(1 / sqrtf(72)) at 72); h =
                          *   out_proj ('attn_pool.proj.*'); pooled = h + fc2(act(fc1(LN_head(h)))) ('attn_pool.norm.*', 'attn_pool.mlp.fc1.*'
                          *   [F, D], 'attn_pool.mlp.fc2.*' [D, F], F the blocks' MLP width), f32.  The head reads
                          *   f16(pooled): HF's pooler_output.  f16 operands and f32 accumulation in the f16 and FP8 engines alike.
                          * 3 'mean': the head reads the mean over all P rows of LN(row): SiglipForImageClassification's classifier input.
                          * With pools 2 and 3 the MLP width F is read from block 0's 'mlp.fc1.weight' [F][D] (So400m: 4304) with SwiGLU's checks,
                          * img_size need not be a multiple of patch_size (So400m at 384 px: a 27 x 27 grid, P = 729; at patch size 8, 16 or 32
                          * it must then be a multiple of 4), and images still arrive
                          * img_size x img_size: the pixels past G patch_size in each direction are read by no patch. */
} vitb200_arch;
/* vitb200_create_ex (fp8 = 0) or vitb200_create_fp8 (fp8 = 1) for a model of architecture `arch` (NULL = all zero, the reference).
 * Fields out of range, activation = 3 with pool 0 or 1, activation = 4 with pool 2 or 3, activation = 4 with an odd fc1 row count, an
 * F that is not a multiple of 8 or outside 8..8 D, or a block whose fc1 or fc2 disagrees with F, pre_norm = 1 without both norm_pre tensors, layer_scale = 1 without every
 * ls1 / ls2 gamma, reg_tokens > 0 without 'reg_token', pool > 0 with head_tokens > 1, pool 2 or 3 with a 'cls_token' tensor, with
 * reg_tokens > 0 or with a 'pos_embed' of other than P rows, pool 2 without one of its 13 'attn_pool.*' tensors, and a head whose K is
 * not D (pools 0, 2, 3) or 2 D (pool 1) fail here before the device is touched, and so do an 'attn_pool.mlp.fc1' / 'fc2' whose width is not
 * the blocks' F and N above the head dim's token limit (896, 800 at 72, 640 at 80), registers included.  Every entry
 * point works on such an engine; the u8 entry points keep vit.cpp's preprocessing unless an image processor is set
 * (vitb200_set_image_proc: Hugging Face's CLIP, SigLIP and DINOv2 preprocessing).  The launch count of one forward is 3 + 7 L + 3 for pools 0 and 1, plus 1 with the
 * pre-norm (the pool of pool = 1 replaces the head rows' LayerNorm); 2 + 7 L + 3 for pool 3 (no class-row kernel); 2 + 7 L + 10 for
 * pool 2 (the head adds LN, k | v GEMM, attention, out_proj, LN, fc1, fc2 and the f16 rounding of its row); each plus 1 (the similarity
 * kernel) while a zero-shot head is set (vitb200_set_zero_shot).
 * A GGUF file selects the architecture with the keys vit.pre_norm (bool or integer), vit.activation ("gelu_tanh", "gelu_erf",
 * "quick_gelu", "gelu_pytorch_tanh", "swiglu"; any other string fails the load), vit.layer_scale (bool or integer), vit.reg_tokens (integer) and
 * vit.pool ("token", "cls_patch_mean", "map" or "mean"; any other string fails the load), and then holds 2 more tensors with the
 * pre-norm, 2 L more with LayerScale and 1 more with registers, 1 fewer (no 'cls_token') with pools 2 and 3 and 13 more with pool 2;
 * a file without these keys is the reference's architecture, and legacy-ggml files never carry them. */
int vitb200_create_arch(const vitb200_hparams *hp, const vitb200_arch *arch, const vitb200_tensor *tensors, int n_tensors, int device,
                        int max_batch, int head_tokens, int fp8, vitb200_engine **out);
int vitb200_get_arch(const vitb200_engine *e, vitb200_arch *out);
int vitb200_fp8(const vitb200_engine *e);         /* 1 for an FP8 engine, else 0 */
int vitb200_in_chans(const vitb200_engine *e);    /* 3, or 1 for a ViTSTR model */
int vitb200_head_tokens(const vitb200_engine *e); /* classifier rows per image */
int vitb200_mlp_dim(const vitb200_engine *e);     /* the MLP's hidden width: F with activation 4 (SwiGLU), pools 2 and 3 and SigLIP text
                                                   * towers, else 4 D */

void vitb200_destroy(vitb200_engine *e);

int vitb200_get_hparams(const vitb200_engine *e, vitb200_hparams *out);

/* id2label entry of the model file (vit.cpp:356-371); NULL if absent or created from tensors. */
const char *vitb200_label(const vitb200_engine *e, int class_id);

/* Batched vit_predict with HOST buffers (host->device copy of the images and device->host copy of the results
 * are part of the call).  images: float32[batch][img][img][3], the image_f32 layout (vit.h:98-103).
 * Any output pointer may be NULL.  probs/logits: float32[batch][num_classes]; probs are the reference's
 * soft-maxed `state.prediction` (vit.cpp:931-933), logits the pre-softmax node (vit.cpp:928).
 * topk_idx/topk_prob: [batch][k], probabilities descending (the head of the reference's sorted
 * `predictions`, vit.cpp:1047-1057), the lowest class id first among equal probabilities.  Entries r >= num_classes (k > num_classes)
 * are (-1, 0); so is every entry of a row whose probabilities are NaN (a NaN or +Inf logit), so an id is always -1 or in
 * [0, num_classes).
 * Images are independent: an image's outputs (here, and in every forward, features and recognition call) depend only on that image,
 * whatever its batch mates or the images of earlier calls held -- NaN and Inf pixels, or pixels that overflow f16, included. */
int vitb200_forward(vitb200_engine *e, const float *images, int batch, float *probs, float *logits, int32_t *topk_idx,
                    float *topk_prob, int k);

/* Pipelined form of vitb200_forward: returns as soon as the work is enqueued; the host->device copy of call i+1 overlaps the
 * kernels of call i (two input/output slots).  Host buffers (pinned memory for real overlap) must stay valid, and outputs
 * must not be read, until vitb200_sync() returns.  vitb200_forward == vitb200_forward_async + vitb200_sync. */
int vitb200_forward_async(vitb200_engine *e, const float *images, int batch, float *probs, float *logits,
                          int32_t *topk_idx, float *topk_prob, int k);
int vitb200_sync(vitb200_engine *e);

/* Data-parallel vitb200_forward over n_engines engines (one per GPU of the box, same model, weights replicated) from one host
 * thread: contiguous image shards, no collective (images are independent units).  batch may exceed one engine's max_batch
 * as long as every shard fits. */
int vitb200_forward_sharded(vitb200_engine *const *engines, int n_engines, const float *images, int batch, float *probs, float *logits,
                            int32_t *topk_idx, float *topk_prob, int k);
/* Pipelined form: returns once every shard is enqueued on its engine's two-slot pipeline (vitb200_forward_async), so the same host
 * thread can submit the next global batch while this one runs; buffers must stay valid until vitb200_sync_all() (== vitb200_sync
 * on every engine) returns.  vitb200_forward_sharded == this + vitb200_sync_all. */
int vitb200_forward_sharded_async(vitb200_engine *const *engines, int n_engines, const float *images, int batch, float *probs,
                                  float *logits, int32_t *topk_idx, float *topk_prob, int k);
int vitb200_sync_all(vitb200_engine *const *engines, int n_engines);

/* vit_image_preprocess + vit_predict fused on the GPU (reference vit.h:119, vit.cpp:130-305 + vit.cpp:1004): `images[b]` is the
 * interleaved RGB u8 image the reference's load_image_from_file produces (image_u8::data, vit.h:91-96), nx[b] x ny[b]
 * pixels, any size.  bilinear = 0 selects the reference's default bicubic path (hparams.interpolation, vit.h:30).  The resize,
 * the round-to-u8 and the mean/std normalisation run on the device and feed the forward pass directly; images_f32_out
 * (optional, host, [batch][img][img][3]) returns the pre-processed image_f32 batch.  probs/logits/top-k as vitb200_forward;
 * all of them NULL = preprocess only. */
int vitb200_forward_u8(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                       float *images_f32_out, float *probs, float *logits, int32_t *topk_idx, float *topk_prob, int k);

/* Pipelined form (vitb200_forward_u8 == this + vitb200_sync, plus the optional f32 read-back): the images are packed into a pinned
 * staging buffer inside the call (so `images` may be reused as soon as it returns), ONE host-to-device copy per batch overlaps the
 * previous call's kernels, the pre-processed pixels go straight into the f16 patch matrix of the patch-embedding GEMM, and nothing
 * synchronises or allocates in steady state.  Output buffers must stay valid until vitb200_sync().  Shares its two pipeline slots
 * with vitb200_forward_async. */
int vitb200_forward_u8_async(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                             float *probs, float *logits, int32_t *topk_idx, float *topk_prob, int k);

/* ---- Hugging Face image processors (no reference counterpart) ------------------------------------------------------------------
 * CLIP, SigLIP and DINOv2 towers were trained on pixels prepared by Hugging Face's image processors (CLIPImageProcessor,
 * SiglipImageProcessor, BitImageProcessor), not by vit_image_preprocess.  With an image processor set, every RGB u8 entry point
 * (vitb200_forward_u8, vitb200_forward_u8_async, vitb200_features_u8, images_f32_out included) prepares its images as the PIL backend
 * of those processors does, bit for bit: Pillow's Image.resize (8-bit ImagingResample, anti-aliased when it downscales), HF's centre
 * crop, x = f32(f64(v) * rescale_factor), y = (x - mean_c) / std_c in f32.  images_f32_out then holds HF's pixel_values, in HWC order.
 * The resize and the crop run in two kernels, a horizontal pass into a per-slot scratch and a vertical pass that writes the patch
 * matrix, so a processor call launches one kernel more than vit_image_preprocess (vitb200_forward_u8 without outputs: 2).
 * The processor is read on the host when a call is enqueued; changing it between asynchronous calls is safe.  bilinear != 0 is
 * refused while one is set (the processor fixes the resample). */
typedef struct vitb200_image_proc
{
    int32_t shortest_edge;           /* > 0: resize so the short side is this and the long side int(shortest_edge * long / short) (HF's
                                      * get_resize_output_image_size, default_to_square = False); 0: resize to height x width */
    int32_t height, width;           /* the resize target when shortest_edge == 0 */
    int32_t crop_height, crop_width; /* HF's centre crop after the resize: top = (h - crop_h) / 2, left = (w - crop_w) / 2; 0 = none */
    int32_t resample;                /* Pillow's ids, as preprocessor_config.json stores them: 2 BILINEAR, 3 BICUBIC */
    double rescale_factor;           /* x = f32(f64(v) * rescale_factor) (1.0 when the config's do_rescale is false) */
    float mean[3], std[3];           /* y = (x - mean_c) / std_c in f32 (0 and 1 when do_normalize is false) */
} vitb200_image_proc;
/* Set (p != NULL) or clear (p == NULL: back to vit_image_preprocess) the engine's image processor.  Refused, naming the field, before
 * anything changes: a 1-channel (ViTSTR) engine; resample other than 2 or 3; a negative or missing size (shortest_edge 0 with height or
 * width <= 0, or one crop extent 0 and the other not); shortest_edge without a crop (the output shape would depend on the image); a crop
 * larger than the resize target (HF would pad); a final size other than img_size x img_size; a non-finite or non-positive
 * rescale_factor; a non-finite mean; a zero or non-finite std.  A call is refused when an image's taps along one axis do not fit in
 * shared memory: a bicubic downscale by more than 453, or a bilinear one by more than 906, along one axis.
 * A GGUF file carries a processor in the optional keys vit.image_proc.shortest_edge, .height, .width, .crop_height, .crop_width,
 * .resample (integers), .rescale_factor (float64), .image_mean and .image_std (arrays of 3 float32); the loader sets it through the
 * same checks.  A file without them, and every legacy-ggml file, has none. */
int vitb200_set_image_proc(vitb200_engine *e, const vitb200_image_proc *p);
int vitb200_get_image_proc(const vitb200_engine *e, vitb200_image_proc *out); /* 0; *out all zero when none is set */

/* ---- zero-shot heads: CLIP and SigLIP (no reference counterpart) --------------------------------------------------------------
 * Zero-shot classification against text embeddings, on the GPU: Hugging Face's logits_per_image.  With a head set, each image's head
 * output x (the f32 row of num_classes = E values, the projection width, that the logits are without a head) becomes C class scores
 *     logit[c] = s * (x . t_c) / ||x|| + b
 * t_c = row c of class_embeds normalised once at set time (in f64, stored f32), s = f32(exp(logit_scale)) (logit_scale as HF stores it:
 * vitb200_text_arch.logit_scale), b = logit_bias, or 0 when it is NaN.  mode 0: probs = the soft-max over the C scores with the reference's
 * f16-exp semantics (CLIP), exactly as vitb200_forward's soft-max; mode 1: probs = 1 / (1 + exp(-logit)) per class (SigLIP), and the top-k
 * ranks the scores, not the probabilities (which round to 1.0f above about 17), and returns the probability of each entry.  Top-k rules
 * are vitb200_forward's: the lowest class id first on ties, (-1, 0) past C and for a row with a NaN score.
 * The class matrix is [C][E] f32, any rows: usually text embeddings (vitb200_encode_text), or the mean of several prompt templates per
 * class.  The scores are f32 FFMA dot products with the image norm computed in the same kernel, each summed in a fixed order, so an
 * image's scores depend only on that image.  A forward with a head launches one kernel more than without (the similarity kernel). */
typedef struct vitb200_zero_shot
{
    const float *class_embeds; /* [n_classes][num_classes] f32, row-major; copied (normalised) by the setter */
    int32_t n_classes;         /* C, 1 .. 2^20 */
    float logit_scale;         /* the log of the scale, as HF stores it */
    float logit_bias;          /* added to every score (SigLIP); NaN for none (CLIP) */
    int32_t mode;              /* 0 soft-max (CLIP), 1 sigmoid (SigLIP) */
} vitb200_zero_shot;
/* Set (z != NULL) or clear (z == NULL) the engine's zero-shot head.  While one is set, every entry point that returns probs, logits or
 * top-k returns them over the C classes: vitb200_forward, _async, _device, _debug, vitb200_forward_u8, _u8_async, and
 * vitb200_forward_sharded, _sharded_async (which refuse engines whose output widths differ, naming the engine); logits are the scores
 * above.  Features calls and recognition are unchanged, and with no head every call behaves as before.
 * Refused, naming the field or the row, before anything changes: a text engine; a 1-channel engine or head_tokens > 1 (ViTSTR); C < 1 or
 * C > 2^20; a NULL class_embeds; a non-finite value or a row of zero norm in class_embeds; a non-finite logit_scale, or one whose exp
 * overflows f32; a logit_bias of +-Inf; a mode other than 0 or 1.
 * The setter waits for all work enqueued on the engine's device (its buffers are replaced) and drops the engine's cached CUDA graphs (a
 * replayed graph would run the schedule and the buffers of its capture); the next small-batch calls run eagerly and capture again.  It
 * sizes the per-slot probs and logits, the internal scores and the soft-max scratch for C classes; no forward call allocates. */
int vitb200_set_zero_shot(vitb200_engine *e, const vitb200_zero_shot *z);
/* The head as set (any pointer may be NULL): *n_classes = 0 (and the rest 0) when none is set. */
int vitb200_get_zero_shot(const vitb200_engine *e, int32_t *n_classes, float *logit_scale, float *logit_bias, int32_t *mode);
/* Per-row width of probs and logits: C while a zero-shot head is set, else num_classes. */
int vitb200_num_outputs(const vitb200_engine *e);

/* Text recognition with a ViTSTR model (1-channel, head_tokens >= 2; reference extensions/vitstr.cpp), image to text on the GPU:
 * the extension's vit_image_preprocess (vitstr.cpp:128-201: grayscale in double, its own bilinear resize to img^2 with no half-pixel
 * offset, (v / 255 - 0.5) * 2), the forward pass, and its greedy decode (vitstr.cpp:1020-1054: the arg-max of token rows
 * 1 .. head_tokens-1, lowest class id among equal maxima, stopping at the first row whose arg-max is class 1 = [s]).
 * `images[b]` is interleaved RGB u8, nx[b] x ny[b] pixels with nx, ny >= 2, as the extension's load_image_from_file produces
 * (vitstr.cpp:107-125).  Outputs (host, any of them may be NULL; all NULL = preprocess only):
 *   images_f32_out  float32 [batch][img][img]   the pre-processed images (the extension's image_f32)
 *   chars           int32   [batch][head_tokens - 1]  decoded class ids, -1 past the end of the string (id2label gives the text)
 *   lengths         int32   [batch]             characters before [s] (head_tokens - 1 if it never wins)
 *   scores          double  [batch]             the extension's `conf`: the product of the emitted maxima, in token order; 1 if empty
 *   probs           float32 [batch][head_tokens][num_classes]  as vitb200_forward returns them for this model
 * vitb200_recognize_u8_async follows vitb200_forward_u8_async's buffer rules (images are copied inside the call; outputs must stay
 * valid until vitb200_sync()) and shares its two pipeline slots; vitb200_recognize_u8 == the async form + vitb200_sync, plus the
 * optional f32 read-back. */
int vitb200_recognize_u8(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, float *images_f32_out,
                         int32_t *chars, int32_t *lengths, double *scores, float *probs);
int vitb200_recognize_u8_async(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int32_t *chars,
                               int32_t *lengths, double *scores, float *probs);

/* Same with DEVICE buffers on the engine's device, enqueued on `stream` (a cudaStream_t; NULL = the engine's own
 * stream) without synchronising: the caller owns ordering.  This is the resident-data path bench.py times. */
int vitb200_forward_device(vitb200_engine *e, const float *d_images, int batch, float *d_probs, float *d_logits,
                           int32_t *d_topk_idx, float *d_topk_prob, int k, void *stream);

/* ---- encoder features (no reference counterpart: the reference only returns classifier outputs) -----------------------------
 * The encoder's own outputs instead of the classifier's: every token of the residual stream after any block (a multimodal model's
 * vision tower), and the pooled pre-logits rows the classifier head reads (retrieval, deduplication, linear probes). */
typedef struct vitb200_features_req
{
    int32_t layers; /* encoder blocks to run, 0..num_hidden_layers.  0 = the embeddings (patch GEMM + conv bias + cls + pos_embed,
                     * reference vit.cpp:772-797), after the pre-norm when the model has one (vitb200_arch): the input of block 0, which
                     * is Hugging Face CLIP's hidden_states[0]; num_hidden_layers = the whole encoder (vit.cpp:802-901).  Blocks past
                     * `layers` are not launched.  LLaVA's image features: layers = num_hidden_layers - 1, norm = 0, tokens 1..N-1. */
    int32_t norm;   /* 1: apply the model's final LayerNorm (norm.weight / norm.bias, vit.cpp:915-919) to every emitted row;
                     * 0: the residual stream as it stands after `layers` blocks */
    int32_t dtype;  /* 0 f32, 1 f16, 2 bf16 -- the 16-bit forms are the f32 result rounded to nearest even */
} vitb200_features_req;

/* tokens:    [batch][N][D], every token, cls first, then the R register tokens, then the patches (N = (img/patch)^2 + 1 + R,
 *            Hugging Face's last_hidden_state / hidden_states[i] order); with vitb200_arch.pool 2 or 3 (SigLIP), [batch][P][D], the
 *            patch rows only (P = (img/patch)^2, HF's last_hidden_state / hidden_states[i]).  May be NULL
 * prelogits: [batch][head_tokens][D], the rows the classifier head reads (token 0, vit.cpp:910; the first 25 for ViTSTR,
 *            vitstr.cpp:864-883); with vitb200_arch.pool = 1, [batch][1][2 D]: token 0 || the mean of the patch rows, each row
 *            through the final LayerNorm first when norm == 1; with pool = 2, [batch][1][D]: the attention-pooling head run on the
 *            final LayerNorm of the rows at depth `layers` (HF's pooler_output at layers == num_hidden_layers; needs norm == 1); with
 *            pool = 3, [batch][1][D]: the mean of the rows, through the final LayerNorm first when norm == 1.  May be NULL.  At
 *            layers == num_hidden_layers with norm == 1 this is the head's input before its f16 rounding.  At least one of the two must be
 *            non-NULL.
 * vitb200_features: HOST buffers, blocking, like vitb200_forward (images as there).
 * vitb200_features_device: DEVICE buffers (16-byte aligned) enqueued on `stream` without synchronising, like vitb200_forward_device.
 * vitb200_features_u8: u8 RGB images pre-processed on the GPU, like vitb200_forward_u8 (RGB models only); host outputs, blocking.
 * Small batches replay a cached CUDA graph per argument set, as the classification calls do. */
int vitb200_features(vitb200_engine *e, const float *images, int batch, const vitb200_features_req *req, void *tokens, void *prelogits);
int vitb200_features_device(vitb200_engine *e, const float *d_images, int batch, const vitb200_features_req *req, void *d_tokens,
                            void *d_prelogits, void *stream);
int vitb200_features_u8(vitb200_engine *e, const uint8_t *const *images, const int *nx, const int *ny, int batch, int bilinear,
                        const vitb200_features_req *req, void *tokens, void *prelogits);

/* ---- text towers: CLIP and SigLIP (no reference counterpart) --------------------------------------------------------------------
 * The text half of CLIP (HF CLIPTextModel, CLIPTextModelWithProjection, the text tower of CLIPModel) and SigLIP (SiglipTextModel, the text
 * tower of SiglipModel): the same pre-LN blocks as the image towers, fed with token ids.  Tokenisation is the caller's job (Hugging Face
 * tokenizers): its vocabulary files, normalisation and BPE merges are host-side string work that each model family defines its own way,
 * and the ids are all the GPU needs.
 * hp: hidden_size, num_hidden_layers, num_attention_heads, eps and ftype as for images; num_classes = E, the projection width (the head's
 * rows); patch_size and img_size must be 0.  Tensors: 'token_embd.weight' [V][D] (any weight format, stored f16), 'pos_embed' [1][N][D] f32,
 * 'blocks.*' as for images, 'norm.*' (the final LayerNorm), 'head.weight' [E][D] and 'head.bias' [E] (zeros for CLIP's projection; the
 * identity for CLIPTextModel).  The image checks apply (head dim 64, D <= 2048, MLP 4 D, unique names, shapes), except that a bidirectional
 * (SigLIP, causal = 0) tower may have head dim 72 (So400m) and reads its MLP width F from the weights as pools 2 and 3 do; context must equal the
 * 'pos_embed' rows and be at most 224 and V >= 1.  Anything else fails before the device is touched, naming the limit.
 * A GGUF file is a text tower when it has the key vit.text.context_length; it then carries vit.text.causal (bool or integer),
 * vit.text.pool ("eos", "eos_argmax" or "last"; any other string fails the load), vit.text.eos_token_id (integer) and optionally
 * vit.text.logit_scale / vit.text.logit_bias (float32), must not carry vit.patch_size, vit.image_size, vit.pre_norm, vit.layer_scale,
 * vit.reg_tokens, vit.pool or vit.image_proc.*, refuses unknown vit.text.* keys, and holds 12 L + 6 tensors.  vitb200_create_from_file and
 * vitb200_create_from_file_fp8 (head_tokens 1) create a text engine from it. */
typedef struct vitb200_text_arch
{
    int32_t context;      /* N tokens per sequence = 'pos_embed' rows, 1..224 */
    int32_t causal;       /* 1 CLIP's causal mask (query t sees keys 0..t), 0 bidirectional (SigLIP) */
    int32_t pool;         /* 0 "eos": the first position whose id == eos_token_id, row 0 if there is none;
                           * 1 "eos_argmax": the first position of the largest id (HF CLIP configs with eos_token_id == 2);
                           * 2 "last": row N - 1 (SigLIP) */
    int32_t eos_token_id; /* pool 0 only */
    int32_t activation;   /* 0..3 as vitb200_arch.activation; 4 (SwiGLU) is refused */
    float logit_scale, logit_bias; /* HF's parameters as stored (the scale is its log), NaN when absent; metadata, no kernel reads them */
} vitb200_text_arch;

/* fp8 as vitb200_create_arch.  An engine is either a text or an image engine: every image entry point (forward, u8, features,
 * recognition, sharded, image processor, vitb200_get_arch) fails on a text engine with a message, and the text entry points fail on an
 * image engine.  vitb200_get_hparams, vitb200_mlp_dim, vitb200_fp8, vitb200_last_launch_count and profiling work on both. */
int vitb200_create_text(const vitb200_hparams *hp, const vitb200_text_arch *ta, const vitb200_tensor *t, int n, int device, int max_batch,
                        int fp8, vitb200_engine **out);
int vitb200_get_text_arch(const vitb200_engine *e, vitb200_text_arch *out); /* non-zero on an image engine */
/* ids: int32 [batch][N], padded by the caller to the context length (under the causal mask the padding leaves CLIP's EOS row as it is;
 * SigLIP was trained on padded sequences).
 * embeds (may be NULL): f32 [batch][E], the head applied to the f16 final LayerNorm of the pooled row: HF's text_embeds, or pooler_output
 * when the head is the identity.
 * req, tokens (may be NULL together): as vitb200_features: tokens [batch][N][D] after req->layers blocks, through the final LayerNorm or
 * not, f32 / f16 / bf16 (layers = L - 1, norm = 0 is HF's hidden_states[-2], SDXL's conditioning).  Both outputs may be asked for in one
 * call: the tokens are emitted after block req->layers and the remaining blocks run; blocks past req->layers run only when embeds is
 * requested.  At least one output.
 * vitb200_encode_text: HOST buffers, blocking; an id outside [0, V) is refused before anything is enqueued, naming the sequence and the
 * position.  Small batches replay a cached CUDA graph.
 * vitb200_encode_text_device: DEVICE buffers (16-byte aligned) on `stream` (NULL = the engine's), not synchronised; a sequence holding an
 * id outside [0, V) gets NaN in every row (and so NaN outputs), its table rows are never read, and its batch mates are unaffected.
 * Sequences are independent: a sequence's outputs depend only on its own ids.
 * Launches: 1 + 7 L + 2 for embeds alone (token gather, the blocks, the pool kernel, the head GEMM); tokens add one kernel (or a copy, for
 * un-normalised f32) and skip the blocks past req->layers when embeds is NULL.  Profile kinds: the gather is kind 0, the pool kernel 7. */
int vitb200_encode_text(vitb200_engine *e, const int32_t *ids, int batch, float *embeds, const vitb200_features_req *req, void *tokens);
int vitb200_encode_text_device(vitb200_engine *e, const int32_t *d_ids, int batch, float *d_embeds, const vitb200_features_req *req,
                               void *d_tokens, void *stream);

/* Number of kernels launched by the most recent call on this engine that enqueued work: a forward, features or recognition call,
 * including one that only pre-processes images (vitb200_forward_u8 without outputs: 1, or 2 with an image processor).  A call rejected by its argument checks
 * leaves the count as it was. */
int vitb200_last_launch_count(const vitb200_engine *e);

/* Per-kernel device timing for roofline reporting: while enabled, CUDA-event pairs are recorded around every
 * launch of the tracked kernels on the stream the forward runs on.  kind: 0 patch GEMM, 1 qkv GEMM, 2 proj GEMM,
 * 3 fc1 GEMM, 4 fc2 GEMM, 5 head GEMM, 6 attention, 7 layernorm, 8 the attention-pooling head of vitb200_arch.pool = 2 (every
 * launch it makes but its two LayerNorms, which are kind 7).  profile_read synchronises the device and returns
 * the summed duration, the launch count and the algorithmic FLOPs of one launch (0 for HBM-bound kernels). */
int vitb200_profile_enable(vitb200_engine *e, int on);
int vitb200_profile_read(vitb200_engine *e, int kind, double *ms_total, int *launches, double *flops_per_launch);

/* Opaque handles for timing on the engine's stream (bench.py passes its own stream instead, normally). */
void *vitb200_stream(vitb200_engine *e);

const char *vitb200_last_error(void);

/* ---- test / debug surface (used by tests/ only) -------------------------------------------------------- */

/* Intermediates of one forward of `batch` <= max_batch images, converted to float32 on the host.
 * Any pointer may be NULL.  Shapes per image (N = tokens, D = hidden): see oracle/vit_oracle.c vo_taps. */
typedef struct vitb200_taps
{
    int32_t layer;
    float *embed;    /* [batch][N][D]  the input of block 0 (after the pre-norm, if any) */
    float *ln1;      /* [batch][N][D]  */
    float *qkv;      /* [batch][N][3D] */
    float *attn;     /* [batch][N][D]  */
    float *x1;       /* [batch][N][D]  */
    float *ln2;      /* [batch][N][D]  */
    float *h;        /* [batch][N][F]  the MLP's hidden activations, F = vitb200_mlp_dim */
    float *x2;       /* [batch][N][D]  */
    float *final_ln; /* [batch][D]     the head's f16 input ([batch][2 D] with vitb200_arch.pool = 1; the pooled row with pool 2, 3) */
    float *x_final;  /* [batch][N][D]  */
} vitb200_taps;

int vitb200_forward_debug(vitb200_engine *e, const float *images, int batch, float *probs, float *logits,
                          const vitb200_taps *taps);

/* Stand-alone run of the wgmma GEMM kernel: out[M][N] = epilogue(A[M][K] (f16 bits) x W[N][K]^T (f16 bits)).
 * epilogue: 0 bias->f16, 1 bias+gelu->f16, 2 bias+resid->f32, 4 bias->f32, 6 bias->split precision (hi = f16(x), lo = f16(x - hi);
 * `out` receives hi + lo), 7 bias+gelu_erf->f16, 8 bias+quick_gelu->f16, 10 bias+gelu_pytorch_tanh->f16 (vitb200_arch.activation 1, 2
 * and 3), 11 SwiGLU->f16 (activation 4: W [N][K] and bias [N] in HF's order, N = 2 F, F % 8 == 0; out [M][N / 2] = f16(silu(x1) x2)).
 * out is float32[M][N] on the host (f16 results widened).  resid may be NULL unless epilogue == 2.  Any other epilogue is refused
 * before the device is touched (3, the patch embedding, needs the position table; 9 runs through vitb200_test_gemm_layer_scale). */
int vitb200_test_gemm(int device, int M, int N, int K, int epilogue, const uint16_t *A, const uint16_t *W,
                      const float *bias, const float *resid, float *out);

/* The same with the LayerScale residual epilogue (vitb200_arch.layer_scale, proj and fc2): out float32 [M][N] =
 * f32(f32(acc + bias[n]) * gamma[n]) + resid[m][n], computed in place on a copy of resid as the engine does.  K % 8 == 0, N % 4 == 0. */
int vitb200_test_gemm_layer_scale(int device, int M, int N, int K, const uint16_t *A, const uint16_t *W, const float *bias,
                                  const float *gamma, const float *resid, float *out);

/* Stand-alone run of the block LayerNorm kernel the forward schedule uses (reference ggml_norm + ggml_mul + ggml_add, vit.cpp:808-812,
 * ggml.c:8959-9008): x float32 [rows][D] -> y float32 [rows][D] holding the f16 results (the next GEMM's A operand) widened. */
int vitb200_test_layernorm(int device, int rows, int D, const float *x, const float *w, const float *b, float eps, float *y);

/* Host-only: the FP8 engine's upload-time quantisation of one weight tensor (vitb200_create_fp8): n f16 values (bits) -> n e4m3
 * bytes q and the tensor's scale *scale.  Needs no GPU. */
int vitb200_test_quantize_fp8(const uint16_t *w_f16, int64_t n, uint8_t *q, float *scale);

/* Stand-alone run of the e4m3 GEMM the FP8 engine uses for qkv and fc1: A [M][K] and W [N][K] e4m3 bytes, a_scale float32 [M] (one per
 * A row), w_scale, bias [N]; out float32 [M][N] = the epilogue's f16 result widened (epilogue 0 bias->f16, 1 bias+gelu->f16,
 * 6 split precision: hi + lo, 7 bias+gelu_erf->f16, 8 bias+quick_gelu->f16, 10 bias+gelu_pytorch_tanh->f16, 11 SwiGLU
 * as vitb200_test_gemm takes it, out [M][N / 2]) of x = acc * (a_scale[m] * w_scale) + bias[n].  K % 16 == 0. */
int vitb200_test_gemm_fp8(int device, int M, int N, int K, int epilogue, const uint8_t *A, const float *a_scale, const uint8_t *W,
                          float w_scale, const float *bias, float *out);

/* Stand-alone run of the qkv and pool k | v GEMMs as the engine runs them at head dim 64: the output in head-major planes, every 64
 * output columns one plane of plane_rows rows, uint16 f16 bits hi [N / 64][plane_rows][64] (and lo, the same shape, for epilogue 6).
 * epilogue: 0 bias->f16, 6 split precision (hi = f16(x), lo = f16(x - hi)); lo is given exactly with 6.  e4m3 = 0: A [M][K] and
 * W [N][K] f16 bits, a_scale NULL, K % 8 == 0; e4m3 = 1: e4m3 bytes with a_scale float32 [M] and w_scale as vitb200_test_gemm_fp8 takes
 * them, K % 16 == 0.  N % 64 == 0, plane_rows >= M.  Both outputs are filled with 0xFFFF first: rows M .. plane_rows - 1 of every plane
 * must keep it.  Shapes and epilogues outside these are refused before the device is touched. */
int vitb200_test_gemm_planes(int device, int M, int N, int K, int epilogue, int64_t plane_rows, int e4m3, const void *A, const float *a_scale,
                             const void *W, float w_scale, const float *bias, uint16_t *hi, uint16_t *lo);

/* The FP8 engine's LayerNorm 1 / 2 alone, the kernel chosen as vitb200_test_layernorm chooses it: x float32 [rows][D] -> q e4m3 bytes
 * [rows][D] and the row scales sa float32 [rows].  D % 16 == 0. */
int vitb200_test_layernorm_fp8(int device, int rows, int D, const float *x, const float *w, const float *b, float eps, uint8_t *q, float *sa);

/* Prototype of the reference's q8_0 x q8_0 linear layer on the INTEGER tensor cores (wgmma s8, one K = 32 MMA per
 * q8_0 block; csrc/gemm_q8_wgmma.cuh).  Replaces, for one layer, quantize_row_q8_0 (reference ggml-quants.c:702-790: the f32
 * activation rows x [M][K] are quantised on the device, bit for bit as the reference does) + ggml_vec_dot_q8_0_q8_0
 * (ggml-quants.c:3521+) + the bias add.  w_q8_0 is the tensor as stored in a q8_0 model file: [N][K/32] blocks of {f16 d; int8 q[32]}
 * (ggml-quants.h:42-46).  y = float32 [M][N]; xq (int8 [M][K]) and xd (float32 [M][K/32]) optionally receive the quantised
 * activations; with iters > 0 *ms_per_launch receives the CUDA-event time of one GEMM launch averaged over `iters` launches.
 * K % 128 == 0, N % 4 == 0.  Not part of the forward schedule (it is slower than the f16 tensor-core path, DESIGN.md section 3). */
int vitb200_test_gemm_q8(int device, int M, int N, int K, const float *x, const void *w_q8_0, const float *bias, float *y,
                         int8_t *xq, float *xd, int iters, float *ms_per_launch);

/* Stand-alone run of one attention kernel (head dim 64) over a fused QKV buffer: qkv = f16 bits [B*N][3*H*64] (what the qkv
 * GEMM leaves behind, reference vit.cpp:826-846), out = float32 [B*N][H*64] (the merged heads before proj, vit.cpp:860-866).
 * kernel: 0 = the engine's choice for N, 1 = two-pass mma.sync with 8 warps (any N), 2 = wgmma with TMA-staged operands (N <= 224:
 * the persistent kernel up to 200 tokens, one CTA per (image, head) beyond, as the engine picks them), 3 = two-pass mma.sync with 16
 * warps (128 < N <= 640), 5 = the one-CTA-per-(image, head) wgmma kernel at any N <= 224.  The wgmma kernels always run on
 * split-precision operands; here their lo halves are zero, so they compute with the f16 values of qkv as given. */
int vitb200_test_attention(int device, int kernel, int B, int N, int H, const uint16_t *qkv, float *out);

/* The wgmma attention kernel (N <= 224) on split-precision operands, the way the engine runs it: every q, k, v value is
 * the sum of two f16 numbers, qkv_hi + qkv_lo (what the qkv GEMM's hi-lo epilogue leaves behind: hi = f16(x), lo = f16(x - hi)), so
 * the f16 tensor cores reproduce the reference's f32-operand attention mat-muls (vit.cpp:848,858).  Both halves are taken as given:
 * lo need not be the residue of hi, so a test can place an operand in one half alone.  The same holds for the split form of
 * vitb200_test_attention_hd and vitb200_test_attention_hd72 below. */
int vitb200_test_attention_hilo(int device, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out);
/* The same with CLIP's causal mask (vitb200_text_arch.causal): query row t attends to keys 0 .. t of its sequence. */
int vitb200_test_attention_hilo_causal(int device, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out);
/* vitb200_test_attention_hilo through kernel 2 or 5 of vitb200_test_attention with the kernel's phase probe on: per CTA and per problem
 * it takes (the first 64), 9 %globaltimer stamps in ns -- the K V load issued, then for each of the two computing warpgroups: waiting
 * for its first q tile's operands, operands landed, S done, P V done (0 where a warpgroup had no tile).  rec receives
 * grid x 64 x 9 stamps and must hold B*H x 64 x 9; *grid receives the grid size.  For tools/attention_phases.py. */
int vitb200_test_attention_phases(int device, int kernel, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo,
                                  unsigned long long *rec, int *grid);
/* Stand-alone run of the attention kernel of head dim hd (64 or 80) over a row-major QKV buffer: qkv_hi = f16 bits [B*N][3*H*hd],
 * out = float32 [B*N][H*hd].  hd 80 runs the head-dim-80 kernel (kernel 0 = the engine's choice, or 4; 1 <= N <= 640, the
 * engine's limit): on split-precision operands qkv_hi + qkv_lo when qkv_lo is given (N <= 224, as the engine runs it there), on the
 * f16 values of qkv_hi when qkv_lo is NULL (as the engine runs it above 224 tokens).  hd 64 runs vitb200_test_attention's kernels, with
 * the lo halves when qkv_lo is given (kernel 0, 2 or 5). */
int vitb200_test_attention_hd(int device, int kernel, int B, int N, int H, int hd, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out);
/* The same for head dim 72 (SigLIP So400m), which vitb200_test_attention_hd refuses: qkv_hi = f16 bits [B*N][3*H*72], out = float32
 * [B*N][H*72], 1 <= N <= 800; split precision with qkv_lo (N <= 224), the f16 values of qkv_hi without it. */
int vitb200_test_attention_hd72(int device, int B, int N, int H, const uint16_t *qkv_hi, const uint16_t *qkv_lo, float *out);

/* Stand-alone run of the attention-pooling head's attention kernel (vitb200_arch.pool = 2) through the engine's launcher: one query
 * q float32 [H*64] (the probe's, scaled by 1/8 inside) per head against the P key rows of each image; kv = f16 bits [B*P][2*H*64], every
 * row k then v (what the k | v GEMM computes), out = float32 [B][H*64] = the f16 result sum_j softmax_j(q_h k_j / 8) v_j, widened.
 * 1 <= P <= 896. */
int vitb200_test_attention_pool(int device, int B, int P, int H, const float *q, const uint16_t *kv, float *out);
/* The same at head dim 72: q float32 [H*72] (scaled by f32(1 / sqrtf(72)) inside), kv = f16 bits [B*P][2*H*72], every row k then v, as
 * the engine's k | v GEMM leaves it for this head dim, out = float32 [B][H*72].  1 <= P <= 800. */
int vitb200_test_attention_pool_hd72(int device, int B, int P, int H, const float *q, const uint16_t *kv, float *out);

/* Stand-alone run of the classifier's soft-max + top-k kernel, launched as the forward launches it (the working row in shared memory
 * up to 227 KB of classes, in global scratch beyond): logits float32 [rows][C] (dense) are copied into rows of pitch round_up(C, 4),
 * as the head GEMM leaves them, with NaN in the padding columns; probs float32 [rows][C], topk_idx int32 / topk_val float32 [rows][k]
 * on the host (may be NULL when k == 0).  0 <= k <= 16; top-k entries as vitb200_forward returns them. */
int vitb200_test_softmax_topk(int device, int rows, int C, int k, const float *logits, float *probs, int32_t *topk_idx, float *topk_val);

/* Stand-alone run of the zero-shot head's kernels (vitb200_set_zero_shot), launched as the forward launches them: x float32 [rows][E] (the
 * head's rows, copied into rows of pitch round_up(E, 4) with NaN in the padding columns), T float32 [C][E] raw class rows (normalised and
 * checked as the setter does), logit_scale / logit_bias / mode as in vitb200_zero_shot.  Outputs on the host: logits float32 [rows][C] (the
 * scores), probs float32 [rows][C], topk_idx int32 / topk_val float32 [rows][k] (may be NULL when k == 0); 0 <= k <= 16. */
int vitb200_test_zero_shot(int device, int rows, int E, int C, const float *x, const float *T, float logit_scale, float logit_bias, int mode, int k,
                           float *probs, float *logits, int32_t *topk_idx, float *topk_val);

/* Host-only: the upload-time weight conversion of one quantised tensor, `n_blocks` ggml blocks of 32 weights
 * (type = ggml_type / file ftype: 2 q4_0, 3 q4_1, 6 q5_0, 7 q5_1, 8 q8_0; ggml-quants.h:11-47) -> f16 bits, exactly what
 * vitb200_create stores on the device.  Needs no GPU.  Follows dequantize_row_q* (ggml-quants.c:1074-1185). */
int vitb200_test_dequant(int type, const void *blocks, int64_t n_blocks, uint16_t *out_f16);

#ifdef __cplusplus
}
#endif
#endif /* VITB200_H */
