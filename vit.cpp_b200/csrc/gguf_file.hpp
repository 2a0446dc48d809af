// gguf_file.hpp -- reader for a true GGUF (v2/v3) container holding a ViT (host code, no CUDA).
//
// The reference's ".gguf" files are the legacy ggml format (magic "ggml", reference vit.cpp:320-328); real GGUF exists in its ggml
// tree (ggml/docs/gguf.md, gguf_init_from_file ggml.c:18017) but vit.cpp never calls it and defines no ViT key names.  This
// reader is the SURVEY.md 8(f) rank-3 extension: same tensors (timm names, ggml dimension order ne[0] = fastest), same types
// (+ BF16, ggml type 30 in current ggml, which gives bf16 checkpoints a container), hyper-parameters as metadata:
//     general.architecture = "vit"                         general.alignment (default 32)          general.file_type (optional)
//     vit.hidden_size, vit.num_hidden_layers, vit.num_attention_heads, vit.num_classes, vit.patch_size, vit.image_size  (integers)
//     vit.layer_norm_eps (float32, default 1e-6)           vit.id2label (array of strings, index = class id; optional)
//     vit.pre_norm (bool or integer, default 0: 1 = a LayerNorm 'norm_pre' before block 0, as in CLIP towers)
//     vit.activation (string, default "gelu_tanh"; "gelu_erf", "quick_gelu", "gelu_pytorch_tanh" or "swiglu": the MLP activation)
//     vit.layer_scale (bool or integer, default 0: 1 = LayerScale gammas 'blocks.{i}.ls1.gamma' / 'ls2.gamma', as in DINOv2)
//     vit.reg_tokens (integer, default 0: register tokens 'reg_token' after the class token)
//     vit.pool (string, default "token"; "cls_patch_mean": the head reads the class token || the mean of the patch tokens; "map" or
//              "mean": SigLIP, no class token, the head reads the attention-pooling head's output or the mean of the tokens)
//     vit.image_proc.shortest_edge, .height, .width, .crop_height, .crop_width, .resample (integers), .rescale_factor (float64),
//     vit.image_proc.image_mean, .image_std (arrays of 3 float32): Hugging Face's image preprocessing (vitb200_image_proc), optional
//     vit.text.context_length (integer): the file is a CLIP or SigLIP text tower (vitb200_text_arch), with vit.text.causal (bool or
//              integer), vit.text.pool ("eos", "eos_argmax" or "last"), vit.text.eos_token_id (integer) and optionally
//              vit.text.logit_scale / vit.text.logit_bias (float32); it carries no image key (patch_size, image_size, pre_norm, layer_scale,
//              reg_tokens, pool, image_proc.*), and no other vit.text.* key
// Layout (gguf.md): header {magic "GGUF", u32 version, u64 n_tensors, u64 n_kv}, n_kv x {string key, u32 type, value},
// n_tensors x {string name, u32 n_dims, u64 ne[n_dims], u32 type, u64 offset}, padding to the alignment, tensor data (offsets
// relative to the start of the data section).  Strings are {u64 length, bytes}.
#pragma once
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace vitb200 {

struct GgufTensor
{
    std::string name;
    int32_t type = 0, n_dims = 0;
    int64_t ne[4] = {1, 1, 1, 1};
    size_t offset = 0, nbytes = 0; // offset from the start of the file
};

struct GgufModel
{
    int64_t hidden_size = 0, num_hidden_layers = 0, num_attention_heads = 0, num_classes = 0, patch_size = 0, img_size = 0, ftype = 1;
    float eps = 1e-6f;
    int64_t pre_norm = 0; // vit.pre_norm (vitb200_arch.pre_norm; the loader checks the range)
    int32_t activation = 0; // vit.activation: 0 gelu_tanh, 1 gelu_erf, 2 quick_gelu, 3 gelu_pytorch_tanh, 4 swiglu (vitb200_arch.activation)
    int64_t layer_scale = 0, reg_tokens = 0; // vit.layer_scale, vit.reg_tokens (vitb200_arch; the loader checks the ranges)
    int32_t pool = 0;       // vit.pool: 0 token, 1 cls_patch_mean, 2 map, 3 mean (vitb200_arch.pool)
    // vit.image_proc.* (vitb200_image_proc; the loader checks the values): has_image_proc once any of the keys is present.  A missing
    // key keeps a value the checks refuse (resample 0, rescale_factor 0, a mean or std without 3 values)
    bool has_image_proc = false;
    int64_t ip_shortest_edge = 0, ip_height = 0, ip_width = 0, ip_crop_height = 0, ip_crop_width = 0, ip_resample = 0;
    double ip_rescale_factor = 0.0;
    float ip_mean[3] = {0, 0, 0}, ip_std[3] = {0, 0, 0};
    // vit.text.* (vitb200_text_arch; the loader checks the values): text once vit.text.context_length is present.  image_key: the first
    // image-only key seen, which a text file must not have
    bool text = false;
    int64_t text_context = 0, text_causal = 0, text_eos = 0;
    int32_t text_pool = 0;
    float logit_scale = __builtin_nanf(""), logit_bias = __builtin_nanf("");
    std::string image_key;
    std::map<int, std::string> labels;
    std::vector<GgufTensor> tensors;
    std::string error;
};

constexpr uint32_t GGUF_MAGIC_LE = 0x46554747u; // "GGUF"

// bytes of n elements of a ggml tensor type; 0 = unsupported type or a row that is not a whole number of blocks
inline size_t gguf_type_bytes(int type, int64_t n, int64_t ne0)
{
    switch (type)
    {
    case 0: return (size_t)n * 4;   // F32
    case 1: return (size_t)n * 2;   // F16
    case 30: return (size_t)n * 2;  // BF16
    case 2: return ne0 % 32 ? 0 : (size_t)n / 32 * 18; // Q4_0
    case 3: return ne0 % 32 ? 0 : (size_t)n / 32 * 20; // Q4_1
    case 6: return ne0 % 32 ? 0 : (size_t)n / 32 * 22; // Q5_0
    case 7: return ne0 % 32 ? 0 : (size_t)n / 32 * 24; // Q5_1
    case 8: return ne0 % 32 ? 0 : (size_t)n / 32 * 34; // Q8_0
    default: return 0;
    }
}

inline bool parse_gguf(const char *buf, size_t size, GgufModel &m)
{
    size_t off = 0;
    auto fail = [&](const std::string &why) { m.error = why; return false; };
    auto rd = [&](void *dst, size_t n) { if (off + n > size) return false; memcpy(dst, buf + off, n); off += n; return true; };
    auto rd_str = [&](std::string &s) {
        uint64_t len = 0;
        if (!rd(&len, 8) || len > size - off) return false;
        s.assign(buf + off, (size_t)len);
        off += (size_t)len;
        return true;
    };
    uint32_t magic = 0, version = 0;
    uint64_t n_tensors = 0, n_kv = 0;
    if (!rd(&magic, 4) || magic != GGUF_MAGIC_LE) return fail("not a GGUF file");
    if (!rd(&version, 4) || (version != 2 && version != 3)) return fail("unsupported GGUF version " + std::to_string(version));
    if (!rd(&n_tensors, 8) || !rd(&n_kv, 8) || n_tensors > (1u << 20) || n_kv > (1u << 20)) return fail("corrupt GGUF header");

    static const size_t scalar_size[13] = {1, 1, 2, 2, 4, 4, 4, 1, 0, 0, 8, 8, 8};
    uint64_t alignment = 32;
    std::string arch;
    for (uint64_t i = 0; i < n_kv; ++i)
    {
        std::string key;
        uint32_t vt = 0;
        if (!rd_str(key) || !rd(&vt, 4) || vt > 12) return fail("corrupt GGUF metadata");
        if (vt == 8) // string
        {
            std::string v;
            if (!rd_str(v)) return fail("truncated GGUF string value");
            if (key == "general.architecture") arch = v;
            else if (key == "vit.text.pool")
            {
                if (v == "eos") m.text_pool = 0;
                else if (v == "eos_argmax") m.text_pool = 1;
                else if (v == "last") m.text_pool = 2;
                else return fail("unknown vit.text.pool '" + v + "' (eos, eos_argmax or last)");
            }
            else if (key.compare(0, 9, "vit.text.") == 0) return fail("unknown key " + key + " (or not a string)");
            else if (key == "vit.activation")
            {
                if (v == "gelu_tanh") m.activation = 0;
                else if (v == "gelu_erf") m.activation = 1;
                else if (v == "quick_gelu") m.activation = 2;
                else if (v == "gelu_pytorch_tanh") m.activation = 3;
                else if (v == "swiglu") m.activation = 4;
                else return fail("unknown vit.activation '" + v + "' (gelu_tanh, gelu_erf, quick_gelu, gelu_pytorch_tanh or swiglu)");
            }
            else if (key == "vit.pool")
            {
                if (m.image_key.empty()) m.image_key = key;
                if (v == "token") m.pool = 0;
                else if (v == "cls_patch_mean") m.pool = 1;
                else if (v == "map") m.pool = 2;
                else if (v == "mean") m.pool = 3;
                else return fail("unknown vit.pool '" + v + "' (token, cls_patch_mean, map or mean)");
            }
        }
        else if (vt == 9) // array
        {
            uint32_t et = 0;
            uint64_t cnt = 0;
            if (!rd(&et, 4) || !rd(&cnt, 8) || et > 12 || et == 9) return fail("corrupt GGUF array");
            float *f3 = key == "vit.image_proc.image_mean" ? m.ip_mean : key == "vit.image_proc.image_std" ? m.ip_std : nullptr;
            if (f3)
            {
                if (et != 6 || cnt != 3) return fail(key + " must be an array of 3 float32");
                if (!rd(f3, 12)) return fail("truncated GGUF array");
                m.has_image_proc = true;
                if (m.image_key.empty()) m.image_key = key;
                continue;
            }
            if (key.compare(0, 15, "vit.image_proc.") == 0 || key.compare(0, 9, "vit.text.") == 0) return fail("unknown key " + key);
            for (uint64_t j = 0; j < cnt; ++j)
            {
                if (et == 8)
                {
                    std::string v;
                    if (!rd_str(v)) return fail("truncated GGUF string array");
                    if (key == "vit.id2label") m.labels[(int)j] = v;
                }
                else
                {
                    if (off + scalar_size[et] > size) return fail("truncated GGUF array");
                    off += scalar_size[et];
                }
            }
        }
        else
        {
            unsigned char raw[8] = {0};
            if (!rd(raw, scalar_size[vt])) return fail("truncated GGUF value");
            int64_t iv = 0;
            double fv = 0.0;
            switch (vt)
            {
            case 0: iv = *(uint8_t *)raw; break;
            case 1: iv = *(int8_t *)raw; break;
            case 2: { uint16_t x; memcpy(&x, raw, 2); iv = x; break; }
            case 3: { int16_t x; memcpy(&x, raw, 2); iv = x; break; }
            case 4: { uint32_t x; memcpy(&x, raw, 4); iv = x; break; }
            case 5: { int32_t x; memcpy(&x, raw, 4); iv = x; break; }
            case 6: { float x; memcpy(&x, raw, 4); fv = x; iv = (int64_t)x; break; }
            case 7: iv = raw[0] != 0; break;
            case 10: { uint64_t x; memcpy(&x, raw, 8); iv = (int64_t)x; break; }
            case 11: memcpy(&iv, raw, 8); break;
            case 12: memcpy(&fv, raw, 8); iv = (int64_t)fv; break;
            }
            if (vt != 6 && vt != 12) fv = (double)iv;
            const bool image_only = key == "vit.patch_size" || key == "vit.image_size" || key == "vit.img_size" || key == "vit.pre_norm" ||
                                    key == "vit.layer_scale" || key == "vit.reg_tokens" || key.compare(0, 15, "vit.image_proc.") == 0;
            if (image_only && m.image_key.empty()) m.image_key = key;
            if (key == "general.alignment") alignment = (uint64_t)iv;
            else if (key == "general.file_type") m.ftype = iv;
            else if (key == "vit.hidden_size") m.hidden_size = iv;
            else if (key == "vit.num_hidden_layers" || key == "vit.block_count") m.num_hidden_layers = iv;
            else if (key == "vit.num_attention_heads") m.num_attention_heads = iv;
            else if (key == "vit.num_classes") m.num_classes = iv;
            else if (key == "vit.patch_size") m.patch_size = iv;
            else if (key == "vit.image_size" || key == "vit.img_size") m.img_size = iv;
            else if (key == "vit.layer_norm_eps") m.eps = (float)fv;
            else if (key == "vit.pre_norm") m.pre_norm = iv;
            else if (key == "vit.layer_scale") m.layer_scale = iv;
            else if (key == "vit.reg_tokens") m.reg_tokens = iv;
            else if (key.compare(0, 9, "vit.text.") == 0)
            {
                const std::string f = key.substr(9);
                if (f == "context_length") { m.text_context = iv; m.text = true; }
                else if (f == "causal") m.text_causal = iv;
                else if (f == "eos_token_id") m.text_eos = iv;
                else if ((f == "logit_scale" || f == "logit_bias") && vt == 6) (f == "logit_scale" ? m.logit_scale : m.logit_bias) = (float)fv;
                else if (f == "logit_scale" || f == "logit_bias") return fail(key + " must be float32");
                else return fail("unknown key " + key);
            }
            else if (key.compare(0, 15, "vit.image_proc.") == 0)
            {
                const std::string f = key.substr(15);
                int64_t *dst = f == "shortest_edge" ? &m.ip_shortest_edge : f == "height" ? &m.ip_height : f == "width" ? &m.ip_width
                             : f == "crop_height" ? &m.ip_crop_height : f == "crop_width" ? &m.ip_crop_width : f == "resample" ? &m.ip_resample
                             : nullptr;
                if (dst) *dst = iv;
                else if (f == "rescale_factor") m.ip_rescale_factor = fv;
                else return fail("unknown key " + key);
                m.has_image_proc = true;
            }
        }
    }
    if (!arch.empty() && arch != "vit") return fail("GGUF architecture is '" + arch + "', expected 'vit'");
    if (alignment < 8 || alignment % 8 != 0 || alignment > (1u << 20)) return fail("bad general.alignment");
    if (m.text && !m.image_key.empty()) return fail("a text tower (vit.text.context_length) must not carry the image key " + m.image_key);
    if (m.hidden_size <= 0 || m.num_hidden_layers <= 0 || m.num_attention_heads <= 0 || m.num_classes <= 0 ||
        (!m.text && (m.patch_size <= 0 || m.img_size <= 0)))
        return fail("GGUF file lacks the vit.* hyper-parameter keys");

    m.tensors.resize((size_t)n_tensors);
    for (auto &t : m.tensors)
    {
        uint32_t nd = 0, type = 0;
        uint64_t rel = 0;
        if (!rd_str(t.name) || !rd(&nd, 4) || nd < 1 || nd > 4) return fail("corrupt GGUF tensor info");
        int64_t n = 1;
        for (uint32_t d = 0; d < nd; ++d)
        {
            uint64_t e = 0;
            if (!rd(&e, 8) || e < 1 || e > (1ull << 40)) return fail("corrupt GGUF tensor dims");
            t.ne[d] = (int64_t)e;
            if (n > (int64_t)(1ull << 40) / (int64_t)e) return fail("corrupt GGUF tensor dims (too many elements)");
            n *= (int64_t)e;
        }
        if (!rd(&type, 4) || !rd(&rel, 8)) return fail("corrupt GGUF tensor info");
        t.n_dims = (int32_t)nd;
        t.type = (int32_t)type;
        t.nbytes = gguf_type_bytes(t.type, n, t.ne[0]);
        if (t.nbytes == 0) return fail("tensor '" + t.name + "': unsupported ggml type " + std::to_string(type));
        if (rel % alignment != 0) return fail("tensor '" + t.name + "': data offset is not aligned");
        t.offset = (size_t)rel; // made absolute below
    }
    const size_t data0 = off + (alignment - off % alignment) % alignment;
    for (auto &t : m.tensors)
    {
        t.offset += data0;
        if (t.offset + t.nbytes > size) return fail("tensor '" + t.name + "' has wrong size in model file");
    }
    return true;
}

// ------------------------------------------------------------------------------------------------
// Legacy-ggml model file (the format reference vit_model_load parses, vit.cpp:308-712; written by convert-pth-to-ggml.py:105-158):
//   int32 magic 0x67676d6c ("ggml", ggml.h:211), 7 x int32 hparams (hidden, layers, heads, classes, patch, img, ftype; vit.cpp:335-341),
//   int32 n_labels, n x {int32 id, int32 len, bytes} (vit.cpp:356-371), then per tensor {int32 n_dims, int32 name_len, int32 type,
//   n_dims x int32 ne, name, raw data} (vit.cpp:590-695).  Validation mirrors the reference (magic, known types, sizes); the tensor
//   inventory and shapes are checked against the hyper-parameters by vitb200_create.  Fills the same GgufModel.
inline bool parse_legacy_ggml(const char *buf, size_t size, GgufModel &m)
{
    size_t off = 0;
    auto fail = [&](const std::string &why) { m.error = why; return false; };
    auto rd32 = [&](int32_t &v) { if (off + 4 > size) return false; memcpy(&v, buf + off, 4); off += 4; return true; };
    int32_t magic = 0;
    if (!rd32(magic) || (uint32_t)magic != 0x67676d6cu) return fail("bad magic");
    int32_t hp[7] = {0};
    for (int i = 0; i < 7; ++i)
        if (!rd32(hp[i])) return fail("truncated header");
    m.hidden_size = hp[0]; m.num_hidden_layers = hp[1]; m.num_attention_heads = hp[2]; m.num_classes = hp[3];
    m.patch_size = hp[4]; m.img_size = hp[5];
    m.ftype = hp[6] % 1000; // GGML_QNT_VERSION_FACTOR, vit.cpp:343-354
    m.eps = 1e-6f;
    int32_t n_labels = 0;
    if (!rd32(n_labels) || n_labels < 0) return fail("truncated label table");
    for (int i = 0; i < n_labels; ++i)
    {
        int32_t key = 0, len = 0;
        if (!rd32(key) || !rd32(len) || len < 0 || (size_t)len > size - off) return fail("truncated label table");
        m.labels[key] = std::string(buf + off, (size_t)len);
        off += (size_t)len;
    }
    while (off < size)
    {
        GgufTensor t;
        int32_t len = 0;
        if (!rd32(t.n_dims) || !rd32(len) || !rd32(t.type)) return fail("truncated tensor record");
        if (t.n_dims < 1 || t.n_dims > 4 || len < 0) return fail("corrupt tensor record");
        int64_t n = 1;
        for (int i = 0; i < t.n_dims; ++i)
        {
            int32_t d = 0;
            if (!rd32(d) || d < 1) return fail("corrupt tensor dims");
            t.ne[i] = d;
            if (n > (int64_t)(1ull << 40) / d) return fail("corrupt tensor dims (too many elements)");
            n *= d;
        }
        if ((size_t)len > size - off) return fail("truncated tensor name");
        t.name.assign(buf + off, (size_t)len);
        off += (size_t)len;
        if (t.type == 30) return fail("unknown ftype 30 in model file (tensor '" + t.name + "')"); // BF16 exists in GGUF containers only
        t.nbytes = gguf_type_bytes(t.type, n, t.ne[0]); // vit.cpp:645-678
        if (t.nbytes == 0)
            return fail(t.type == 0 || t.type == 1 || t.type == 2 || t.type == 3 || t.type == 6 || t.type == 7 || t.type == 8
                            ? "tensor '" + t.name + "': quantised rows must be a multiple of 32"
                            : "unknown ftype " + std::to_string(t.type) + " in model file (tensor '" + t.name + "')");
        if (t.nbytes > size - off) return fail("tensor '" + t.name + "' has wrong size in model file");
        t.offset = off;
        off += t.nbytes;
        m.tensors.push_back(t);
    }
    return true;
}

} // namespace vitb200
