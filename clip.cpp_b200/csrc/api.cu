// api.cu -- the C ABI of libclip_b200.so (include/clip_b200.h): loader, static kernel schedule of both towers,
// host<->device plumbing.  No graph, no dispatch: each encode call issues a fixed sequence of kernel launches on
// one stream.  There is NO CPU path -- if CUDA is unavailable clip_model_load fails loudly.
#include <chrono>
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <numeric>
#include <thread>

#include "common.cuh"
#include "gguf.hpp"
#include "kernels.h"
#include "model.h"
#include "wpack.h"

using namespace cb;

namespace {

thread_local std::string g_err;
void set_err(const std::string& s) { g_err = s; fprintf(stderr, "clip_b200: %s\n", s.c_str()); }

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            set_err(std::string(#call) + " failed: " + cudaGetErrorString(e_));                    \
            return false;                                                                          \
        }                                                                                          \
    } while (0)

uint16_t f32_to_bf16(float f) {
    uint32_t x;
    memcpy(&x, &f, 4);
    if ((x & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((x >> 16) | 0x40u);
    x += 0x7FFFu + ((x >> 16) & 1u);
    return (uint16_t)(x >> 16);
}

template <class T>
bool dev_alloc(clip_ctx* c, T** p, size_t count) {
    void* d = nullptr;
    const size_t bytes = std::max<size_t>(count * sizeof(T), 256);
    cudaError_t e = cudaMalloc(&d, bytes);
    if (e != cudaSuccess) { set_err(std::string("cudaMalloc(") + std::to_string(bytes) + ") failed: " + cudaGetErrorString(e)); return false; }
    c->allocs.push_back(d);
    *p = (T*)d;
    return true;
}
template <class T>
bool upload(clip_ctx* c, T** p, const void* host, size_t bytes) {
    uint8_t* d = nullptr;
    if (!dev_alloc(c, &d, bytes)) return false;
    CK(cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice));
    *p = (T*)d;
    return true;
}

// ---- profiling hooks (CUDA events on the launch stream) -------------------------------------------------
cudaEvent_t get_event(clip_ctx* c) {
    if (!c->ev_pool.empty()) { cudaEvent_t e = c->ev_pool.back(); c->ev_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}
struct Scope {
    clip_ctx* c; cudaEvent_t e0 = nullptr; int kind;
    Scope(clip_ctx* c_, int kind_) : c(c_), kind(kind_) {
        c->launches++;
        if (c->profile) { e0 = get_event(c); cudaEventRecord(e0, c->stream); }
    }
    ~Scope() {
        if (!c->profile) return;
        cudaEvent_t e1 = get_event(c);
        cudaEventRecord(e1, c->stream);
        c->prof.push_back({kind, e0, e1});
        if (c->prof.size() > 65536) {        // nobody drains the records: recycle the older half instead of growing without bound
            for (size_t i = 0; i < 32768; i++) { c->ev_pool.push_back(c->prof[i].e0); c->ev_pool.push_back(c->prof[i].e1); }
            c->prof.erase(c->prof.begin(), c->prof.begin() + 32768);
        }
    }
};
enum { K_GEMM = 0, K_ATTN = 1, K_LN = 2, K_OTHER = 3, K_TOKEN_ROWS = 4, K_POS_RESAMPLE = 5, K_ATTN_PROBS = 6, K_KNN16 = 7, K_KNN_I8 = 8, K_KNN_B1 = 9, K_RESCORE = 10, K_IVF_SCAN = 11,
       K_IVF_LAYOUT = 12, K_ADC = 13, K_PQ = 14 };

// ---- tensor lookup helpers ---------------------------------------------------------------------------------
const GgufTensor* need(const GgufFile& g, const std::string& name) {
    const GgufTensor* t = g.tensor(name);
    if (!t) set_err("unable to find tensor " + name);
    return t;
}
bool kv_u32(const GgufFile& g, const std::string& k, int32_t& out) {
    const GgufKV* kv = g.find(k);
    if (!kv) { set_err("key " + k + " not found in file"); return false; }
    out = (int32_t)kv->u;
    return true;
}
bool kv_f32(const GgufFile& g, const std::string& k, float& out) {
    const GgufKV* kv = g.find(k);
    if (!kv) { set_err("key " + k + " not found in file"); return false; }
    out = (float)kv->f;
    return true;
}
bool kv_bool(const GgufFile& g, const std::string& k, bool& out) {
    const GgufKV* kv = g.find(k);
    if (!kv) { set_err("key " + k + " not found in file"); return false; }
    out = kv->u != 0;
    return true;
}

// fp32 vector/table on the device, dequantised exactly as ggml_get_rows / the f32 ops would see it
bool upload_f32(clip_ctx* c, const GgufFile& g, const std::string& name, float** out, int64_t expect_elems) {
    const GgufTensor* t = need(g, name);
    if (!t) return false;
    if ((int64_t)t->nelements() != expect_elems) { set_err("tensor " + name + " has unexpected size"); return false; }
    std::vector<float> h((size_t)expect_elems);
    const int64_t k = (int64_t)t->ne[0], rows = expect_elems / k;
    const size_t rb = (size_t)(k / (int64_t)ggml_type_block_elems(t->type)) * ggml_type_block_bytes(t->type);
    for (int64_t r = 0; r < rows; r++)
        if (!dequant_row((int)t->type, t->data + (size_t)r * rb, h.data() + r * k, k)) { set_err("cannot dequantise " + name); return false; }
    return upload(c, out, h.data(), h.size() * 4);
}

// Columns of a tower's fused QKV activations: Q | K | V, each heads x qkv_head_cols(head_dim) (head_dim 104 pads each head to 112).
int qkv_width(const Tower& tw) { return 3 * tw.heads * qkv_head_cols(tw.hidden / tw.heads); }

// GEMM weight from one or more row-concatenated tensors (fused QKV).  kpad > 0 zero-pads K (patch embedding).  head_dim > 0 pads
// the rows (and bias) of every part to qkv_head_cols(head_dim) per head of head_dim rows, with zero rows (pad_head_rows).
bool make_linear(clip_ctx* c, const GgufFile& g, const std::vector<std::string>& wn, const std::vector<std::string>& bn, Linear& L,
                 int kpad = 0, int head_dim = 0) {
    std::vector<const GgufTensor*> ts;
    for (auto& n : wn) { const GgufTensor* t = need(g, n); if (!t) return false; ts.push_back(t); }
    const uint32_t type = ts[0]->type;
    int64_t K = 1;
    for (uint32_t d = 0; d + 1 < std::max(ts[0]->n_dims, 2u); d++) K *= (int64_t)ts[0]->ne[d];   // 4-D conv weight: K = P*P*3
    const int dhp = head_dim > 0 ? qkv_head_cols(head_dim) : 0;
    const bool pad = dhp > head_dim;
    int64_t N = 0;
    std::vector<std::vector<uint8_t>> padded(ts.size());
    std::vector<const uint8_t*> src(ts.size());       // each part's rows, padded if asked
    std::vector<int64_t> part_rows(ts.size());
    for (size_t i = 0; i < ts.size(); i++) {
        const GgufTensor* t = ts[i];
        if (t->type != type || (int64_t)(t->nelements() / (t->ne[ts[0]->n_dims - 1])) != K) { set_err("inconsistent fused weight " + wn[0]); return false; }
        const int64_t rows = (int64_t)t->ne[t->n_dims - 1];
        src[i] = t->data; part_rows[i] = rows;
        if (pad) {
            const size_t rb = t->nbytes / (size_t)rows;
            padded[i].resize((size_t)(rows / head_dim) * dhp * rb);
            if (!pad_head_rows(t->data, rb, rows, head_dim, dhp, padded[i].data())) { set_err("weight " + wn[i] + " is not a whole number of heads"); return false; }
            src[i] = padded[i].data(); part_rows[i] = rows / head_dim * dhp;
        }
        N += part_rows[i];
    }
    const int64_t Kp = kpad > 0 ? kpad : K;
    if (N % GEMM_BM || Kp % GEMM_BK) { set_err("weight " + wn[0] + ": shape [" + std::to_string(N) + "," + std::to_string(Kp) + "] is not tileable (N%128, K%64)"); return false; }
    L.N = (int)N; L.K = (int)Kp;
    if (type == 0 || type == 1) {
        L.qtype = QT_F16;
        std::vector<uint16_t> h((size_t)N * Kp, 0);
        int64_t r0 = 0;
        for (size_t i = 0; i < ts.size(); i++) {
            const int64_t rows = part_rows[i];
            for (int64_t r = 0; r < rows; r++) {
                uint16_t* dst = h.data() + (size_t)(r0 + r) * Kp;
                if (type == 1) memcpy(dst, src[i] + (size_t)r * K * 2, (size_t)K * 2);
                else { const float* s = (const float*)(src[i]) + (size_t)r * K; for (int64_t k = 0; k < K; k++) dst[k] = f32_to_f16(s[k]); }
            }
            r0 += rows;
        }
        if (!upload(c, &L.d_w, h.data(), h.size() * 2)) return false;
        if (!make_tma_2d_16bit(&L.w_map, L.d_w, (uint64_t)N, (uint64_t)Kp, (uint64_t)Kp, GEMM_BM)) { set_err("cuTensorMapEncodeTiled failed for " + wn[0]); return false; }
        L.d_raw = L.d_w;
    } else {
        if (kpad > 0) { set_err("quantized weights cannot be K-padded: " + wn[0]); return false; }
        L.qtype = (int)type;
        const size_t chunk = wpack_chunk_bytes((int)type), bb = wpack_ggml_block_bytes((int)type);
        if (!chunk) { set_err("unsupported weight type in " + wn[0]); return false; }
        std::vector<uint8_t> packed(wpack_total_bytes((int)type, N, K));
        int64_t r0 = 0;
        for (size_t i = 0; i < ts.size(); i++) {
            const int64_t rows = part_rows[i];
            if (rows % GEMM_BM) { set_err("fused part of " + wn[0] + " is not a multiple of 128 rows"); return false; }
            if (!wpack_repack((int)type, src[i], rows, K, packed.data() + (size_t)(r0 / GEMM_BM) * (K / GEMM_BK) * chunk)) { set_err("re-tiling failed for " + wn[0]); return false; }
            r0 += rows;
        }
        if (!upload(c, &L.d_w, packed.data(), packed.size())) return false;
        if (c->debug_naive) {
            std::vector<uint8_t> raw((size_t)N * (K / 32) * bb);
            size_t o = 0;
            for (size_t i = 0; i < ts.size(); i++) {
                const size_t nb = (size_t)part_rows[i] * (K / 32) * bb;
                memcpy(raw.data() + o, src[i], nb);
                o += nb;
            }
            if (!upload(c, &L.d_raw, raw.data(), raw.size())) return false;
        }
    }
    if (!bn.empty()) {
        std::vector<float> hb;
        for (auto& n : bn) {
            const GgufTensor* t = need(g, n);
            if (!t) return false;
            if (t->type != 0) { set_err("bias " + n + " must be f32"); return false; }
            const int64_t ne = (int64_t)t->nelements();
            if (pad) {
                std::vector<float> pb((size_t)(ne / head_dim) * dhp);
                if (!pad_head_rows(t->data, 4, ne, head_dim, dhp, reinterpret_cast<uint8_t*>(pb.data()))) { set_err("bias " + n + " is not a whole number of heads"); return false; }
                hb.insert(hb.end(), pb.begin(), pb.end());
            } else {
                const float* p = (const float*)t->data;
                hb.insert(hb.end(), p, p + ne);
            }
        }
        if ((int64_t)hb.size() != N) { set_err("bias size mismatch for " + wn[0]); return false; }
        if (!upload(c, &L.d_bias, hb.data(), hb.size() * 4)) return false;
    }
    return true;
}

bool load_blocks(clip_ctx* c, const GgufFile& g, const char* p, Tower& tw) {
    tw.L.resize(tw.layers);
    for (int il = 0; il < tw.layers; il++) {
        const std::string b = std::string(p) + ".blk." + std::to_string(il) + ".";
        Layer& l = tw.L[il];
        if (!make_linear(c, g, {b + "attn_q.weight", b + "attn_k.weight", b + "attn_v.weight"},
                         {b + "attn_q.bias", b + "attn_k.bias", b + "attn_v.bias"}, l.qkv, 0, tw.hidden / tw.heads)) return false;
        if (!make_linear(c, g, {b + "attn_out.weight"}, {b + "attn_out.bias"}, l.out)) return false;
        if (!make_linear(c, g, {b + "ffn_down.weight"}, {b + "ffn_down.bias"}, l.fc1)) return false;   // HF fc1: h -> f
        if (!make_linear(c, g, {b + "ffn_up.weight"}, {b + "ffn_up.bias"}, l.fc2)) return false;       // HF fc2: f -> h
        if (l.qkv.N != qkv_width(tw) || l.qkv.K != tw.hidden || l.out.N != tw.hidden || l.out.K != tw.hidden ||
            l.fc1.N != tw.ff || l.fc1.K != tw.hidden || l.fc2.N != tw.hidden || l.fc2.K != tw.ff) { set_err("layer shape mismatch in " + b); return false; }
        if (!upload_f32(c, g, b + "ln1.weight", &l.ln1_g, tw.hidden) || !upload_f32(c, g, b + "ln1.bias", &l.ln1_b, tw.hidden) ||
            !upload_f32(c, g, b + "ln2.weight", &l.ln2_g, tw.hidden) || !upload_f32(c, g, b + "ln2.bias", &l.ln2_b, tw.hidden)) return false;
    }
    return true;
}

bool check_geometry(const clip_ctx* c, const char* what, const Tower& t) {
    if (t.hidden <= 0 || t.ff <= 0 || t.heads <= 0 || t.layers < 0 || t.layers > 1024 || t.proj <= 0 || !(t.eps >= 0.f)) { set_err(std::string(what) + ": non-positive hyper-parameter in the file"); return false; }
    const std::string hh = " (hidden " + std::to_string(t.hidden) + ", heads " + std::to_string(t.heads) + ")";
    const int dh = t.heads > 0 && t.hidden % t.heads == 0 ? t.hidden / t.heads : 0;
    if (dh != 64 && dh != 80 && dh != 104) { set_err(std::string(what) + ": head_dim must be 64 or 80 (ViT-B/L/H) or 104 (ViT-bigG/14)" + hh); return false; }
    if (!c->attn_tc && t.hidden / t.heads != 64) { set_err(std::string(what) + ": the legacy attention kernel (CLIP_B200_ATTN=legacy) supports head_dim 64 only" + hh); return false; }
    if (t.hidden > 2048) { set_err(std::string(what) + ": hidden size > 2048 is not supported by the register-resident LayerNorm"); return false; }
    if (t.hidden % 128 || t.ff % 128 || t.proj % 128) { set_err(std::string(what) + ": hidden/ff/projection sizes must be multiples of 128"); return false; }
    return true;
}

bool any_f16_gemm(const Tower& t) {
    if (!t.present) return false;
    bool f = t.proj_w.qtype == QT_F16;
    for (auto& l : t.L) f = f || l.qkv.qtype == QT_F16 || l.out.qtype == QT_F16 || l.fc1.qtype == QT_F16 || l.fc2.qtype == QT_F16;
    return f;
}

// ---- workspaces ----------------------------------------------------------------------------------------------
bool ensure_ws(clip_ctx* c, Tower& tw, int items, int T, bool vision) {
    Workspace& w = tw.ws;
    if (w.cap_items >= items && w.T == T) return true;
    if (w.cap_items) { set_err("workspace re-sizing is not supported after the first encode"); return false; }
    const int h = tw.hidden;
    // Row counts are ints, and every GEMM of a pass addresses its output (and the patch GEMM its input) with 32-bit element offsets
    // (gemm_launch): refuse a micro_batch past either limit here, before anything is allocated, so the context stays usable.
    const size_t rows = (size_t)items * (size_t)T;
    const size_t widest = std::max({(size_t)qkv_width(tw), (size_t)tw.ff, (size_t)tw.proj, vision ? (size_t)tw.kpad : (size_t)0});
    if (rows > (size_t)INT_MAX || rows * widest >= ((size_t)1 << 32)) {
        const size_t limit = std::min((size_t)INT_MAX / T, (((size_t)1 << 32) - 1) / (widest * T));
        set_err(std::string(vision ? "vision" : "text") + " micro_batch " + std::to_string(items) + " is too large: " + std::to_string(rows) +
                " rows of " + std::to_string(T) + " per " + (vision ? "image" : "sequence") + " x " + std::to_string(widest) +
                " columns exceed 32-bit offsets; the limit is " + std::to_string(limit) + " (clip_b200_set_micro_batch)");
        return false;
    }
    w.cap_items = items; w.T = T; w.cap_rows = (int)rows;
    if (!dev_alloc(c, &w.x, rows * h) || !dev_alloc(c, &w.a, rows * h) || !dev_alloc(c, &w.qkv, rows * qkv_width(tw)) ||
        !dev_alloc(c, &w.g, rows * tw.ff) || !dev_alloc(c, &w.sel16, (size_t)items * h) || !dev_alloc(c, &w.sel32, (size_t)items * h) ||
        !dev_alloc(c, &w.proj32, (size_t)items * tw.proj)) return false;
    bool ok = make_tma_2d_16bit(&w.map_a, w.a, rows, h, h, GEMM_BN) && make_tma_2d_16bit(&w.map_g, w.g, rows, tw.ff, tw.ff, GEMM_BN) &&
              make_tma_2d_16bit(&w.map_sel, w.sel16, items, h, h, GEMM_BN);
    if (vision) {
        const size_t per = (size_t)tw.image_size * tw.image_size * 3;
        if (!dev_alloc(c, &w.pixels[0], items * per) || !dev_alloc(c, &w.pixels[1], items * per) ||
            !dev_alloc(c, &w.patches, (size_t)items * tw.n_patches * tw.kpad) || !dev_alloc(c, &w.patch32, (size_t)items * tw.n_patches * h)) return false;
        ok = ok && make_tma_2d_16bit(&w.map_patches, w.patches, (uint64_t)items * tw.n_patches, tw.kpad, tw.kpad, GEMM_BN);
    } else {
        if (!dev_alloc(c, &w.ids, rows) || !dev_alloc(c, &w.last, (size_t)items)) return false;
    }
    if (!ok) { set_err("cuTensorMapEncodeTiled failed for a workspace buffer"); return false; }
    return true;
}

bool run_linear(clip_ctx* c, const Linear& L, const TmaMap* xmap, const void* xptr, bool x_bf16, int M, void* out, int ldo, int epi,
                int out_bf16, int scale_cols = 0, float scale = 1.f) {
    Scope s(c, K_GEMM);
    if (c->debug_naive) {
        launch_naive_gemm(xptr, x_bf16, L.d_raw, L.qtype, L.d_bias, out, M, L.N, L.K, ldo, epi, out_bf16, scale_cols, scale, c->stream);
        CK(cudaGetLastError());
        return true;
    }
    GemmArgs a;
    a.x_map = xmap; a.w_map = &L.w_map; a.w_packed = L.d_w; a.qtype = L.qtype; a.operand_bf16 = x_bf16;
    a.bias = L.d_bias; a.out = out; a.M = M; a.N = L.N; a.K = L.K; a.ldo = ldo; a.epi = epi; a.out_bf16 = out_bf16;
    a.scale_cols = scale_cols; a.scale = scale;
    CK(gemm_launch(a, c->stream, c->num_sms, nullptr));
    return true;
}

// A packed pass (the image *_mixed and text *_packed calls): nseq sequences of different lengths packed back to back in `rows`
// rows; d_seq is K3's varlen table on the device (launch_attention_tc_varlen), groups its 64-row groups per head; causal: the text
// tower's mask.
struct Packed {
    int rows = 0, nseq = 0, groups = 0;
    const int* d_seq = nullptr;
    bool causal = false;
};

// The per-layer schedule shared by both towers (clip.cpp:1064-1143 text, 1342-1423 vision): blocks first .. end-1 on ws.x (a
// multi-layer tokens call resumes where its previous stop left x).  pk: a packed pass instead of nseq x T rows.
bool run_blocks(clip_ctx* c, Tower& tw, int nseq, int T, bool causal, int first, int end, const Packed* pk = nullptr) {
    // The residual stream x stays fp32 (as in the reference).  The branch GEMMs (out-proj, FC2) add their result INTO x themselves
    // (EPI_REDADD32): LayerNorm then only reads x and writes its 16-bit output.
    Workspace& w = tw.ws;
    const int M = pk ? pk->rows : nseq * T, h = tw.hidden;
    const int bf = c->operand_bf16 ? 1 : 0;
    const int dh = h / tw.heads;                      // 64, 80 or 104 (check_geometry)
    const float qscale = 1.0f / sqrtf((float)dh);     // clip.cpp:1082, 1363: the real head_dim, not the padded one
    const int qw = qkv_width(tw);
    for (int il = first; il < end; il++) {
        const Layer& l = tw.L[il];
        { Scope s(c, K_LN); launch_layernorm(w.x, h, M, h, tw.eps, l.ln1_g, l.ln1_b, nullptr, w.a, bf, c->stream); }
        if (!run_linear(c, l.qkv, &w.map_a, w.a, bf, M, w.qkv, qw, EPI_STORE16, bf, qw / 3, qscale)) return false;
        if (pk) { Scope s(c, K_ATTN); CK(launch_attention_tc_varlen(w.qkv, w.a, pk->rows, pk->nseq, pk->d_seq, pk->groups, tw.heads, dh, pk->causal ? 1 : 0, bf, c->stream)); }
        else if (c->attn_tc) { Scope s(c, K_ATTN); CK(launch_attention_tc(w.qkv, w.a, nseq, T, tw.heads, dh, causal ? 1 : 0, bf, c->stream)); }
        else { Scope s(c, K_ATTN); launch_attention(w.qkv, w.a, nseq, T, tw.heads, causal ? 1 : 0, bf, c->stream); }
        if (!run_linear(c, l.out, &w.map_a, w.a, bf, M, w.x, h, EPI_REDADD32, 0)) return false;
        { Scope s(c, K_LN); launch_layernorm(w.x, h, M, h, tw.eps, l.ln2_g, l.ln2_b, nullptr, w.a, bf, c->stream); }
        if (!run_linear(c, l.fc1, &w.map_a, w.a, bf, M, w.g, tw.ff, c->use_gelu ? EPI_GELU16 : EPI_QGELU16, bf)) return false;
        if (!run_linear(c, l.fc2, &w.map_g, w.g, bf, M, w.x, h, EPI_REDADD32, 0)) return false;
    }
    CK(cudaGetLastError());
    return true;
}

// ---- packed passes: what the image *_mixed and text *_packed forms share ------------------------------------------------------
// Pass boundaries of a packed call whose item i has T[i] rows: each pass is the longest prefix of the remaining items that
// fits(rows, items, t) admits (the pass's rows and items so far, the next item's rows), and holds at least one item.
template <class F>
std::vector<size_t> pack_passes(const std::vector<int>& T, F fits) {
    std::vector<size_t> b{0};
    size_t rows = 0, k = 0;
    for (size_t i = 0; i < T.size(); i++) {
        if (k && !fits(rows, k, T[i])) {
            b.push_back(i);
            rows = k = 0;
        }
        rows += (size_t)T[i]; k++;
    }
    b.push_back(T.size());
    return b;
}

// K3's varlen table for the pass holding items i0 .. i1 - 1 (T[i] rows each) into seq [2 (i1 - i0 + 1)]: off (each item's first row,
// then the pass's rows), then grp (prefix sums of the items' 64-row groups).  Returns the pass's rows.
int varlen_table(const std::vector<int>& T, size_t i0, size_t i1, int* seq) {
    const size_t nb = i1 - i0;
    int* off = seq;
    int* grp = seq + nb + 1;
    off[0] = grp[0] = 0;
    for (size_t j = 0; j < nb; j++) {
        off[j + 1] = off[j] + T[i0 + j];
        grp[j + 1] = grp[j] + (T[i0 + j] + 63) / 64;
    }
    return off[nb];
}

// The pooled tail of a packed pass: rows d_rows[0 .. nb) of ws.x (device, absolute rows) -> post-LN -> projection -> (L2 norm) ->
// d_out [nb, proj], in chunks of at most cap_items rows (what the sel / proj buffers hold).  Every step works row by row, so the
// chunks change no bits, and the fp32 gather keeps the bits the unpacked forms' LayerNorm reads.
bool pooled_rows_tail(clip_ctx* c, Tower& tw, int nb, const int* d_rows, float* d_out, bool normalize) {
    Workspace& w = tw.ws;
    const int h = tw.hidden, bf = c->operand_bf16 ? 1 : 0;
    for (int j0 = 0; j0 < nb; j0 += w.cap_items) {
        const int k = std::min(w.cap_items, nb - j0);
        { Scope s(c, K_OTHER); launch_gather_rows(w.x, w.sel32, k, h, 0, d_rows + j0, nullptr, bf, c->stream); }
        { Scope s(c, K_LN); launch_layernorm(w.sel32, h, k, h, tw.eps, tw.post_g, tw.post_b, nullptr, w.sel16, bf, c->stream); }
        if (!run_linear(c, tw.proj_w, &w.map_sel, w.sel16, bf, k, w.proj32, tw.proj, EPI_STORE32, 0)) return false;
        { Scope s(c, K_OTHER); launch_l2norm(w.proj32, d_out + (size_t)j0 * tw.proj, k, tw.proj, normalize ? 1 : 0, c->stream); }
    }
    CK(cudaGetLastError());
    return true;
}

// The image size of one vision call: H x W pixels, T = (H/P)(W/P) + 1 rows per image, the position table of that grid ([T, h]).
// The model's own size is H = W = image_size with the loaded table; the *_hw entry points pass others (plan_call).
struct VisCall {
    int H = 0, W = 0, T = 0;
    const float* pos = nullptr;
    size_t per() const { return (size_t)H * W * 3; }     // floats of one NHWC image
};
VisCall native_call(const Tower& tw) {
    VisCall v;
    v.H = v.W = tw.image_size; v.T = tw.T; v.pos = tw.pos;
    return v;
}

// Vision embedding of nb images resident at d_pixels (NHWC f32): ws.x = pre_ln(class | patch embedding + position), the input of block 0.
bool vision_embed(clip_ctx* c, const float* d_pixels, int nb, const VisCall& v) {
    Tower& tw = c->vis;
    Workspace& w = tw.ws;
    const int h = tw.hidden;
    { Scope s(c, K_OTHER); launch_im2col(d_pixels, nb, v.H, v.W, tw.patch, tw.kpad, w.patches, c->stream); }
    // patch embedding = stride-P conv = GEMM over fp16 patches, fp16 weights, fp32 out, no bias (clip.cpp:1309)
    if (!run_linear(c, tw.patch_w, &w.map_patches, w.patches, false, nb * (v.T - 1), w.patch32, h, EPI_STORE32, 0)) return false;
    { Scope s(c, K_OTHER); launch_assemble_preln(w.patch32, tw.class_embd, v.pos, nb, v.T, h, tw.eps, tw.pre_g, tw.pre_b, w.x, c->stream); }
    return true;
}

// Vision tower on nb images already resident at d_pixels (NHWC f32); writes d_out [nb, proj].
bool vision_forward(clip_ctx* c, const float* d_pixels, int nb, const VisCall& v, float* d_out, bool normalize) {
    Tower& tw = c->vis;
    Workspace& w = tw.ws;
    const int h = tw.hidden, bf = c->operand_bf16 ? 1 : 0;
    if (!vision_embed(c, d_pixels, nb, v)) return false;
    if (!run_blocks(c, tw, nb, v.T, false, 0, tw.layers)) return false;
    // CLS rows -> post-LN -> projection -> (L2 norm)   (clip.cpp:1426-1455)
    { Scope s(c, K_LN); launch_layernorm(w.x, (size_t)v.T * h, nb, h, tw.eps, tw.post_g, tw.post_b, nullptr, w.sel16, bf, c->stream); }
    if (!run_linear(c, tw.proj_w, &w.map_sel, w.sel16, bf, nb, w.proj32, tw.proj, EPI_STORE32, 0)) return false;
    { Scope s(c, K_OTHER); launch_l2norm(w.proj32, d_out, nb, tw.proj, normalize ? 1 : 0, c->stream); }
    CK(cudaGetLastError());
    return true;
}

// Text tower on nb sequences padded to T tokens; ws.ids / ws.last already filled.
bool text_forward(clip_ctx* c, int nb, int T, float* d_out, bool normalize) {
    Tower& tw = c->txt;
    Workspace& w = tw.ws;
    const int h = tw.hidden, bf = c->operand_bf16 ? 1 : 0;
    { Scope s(c, K_OTHER); launch_text_embed(w.ids, tw.tok, tw.pos, nb, T, h, tw.n_vocab, w.x, c->stream); }
    if (!run_blocks(c, tw, nb, T, true, 0, tw.layers)) return false;
    // final LN is row-wise, so LN(select(EOT)) == select(LN(all)) (clip.cpp:1146-1155)
    { Scope s(c, K_OTHER); launch_gather_rows(w.x, w.sel32, nb, h, T, w.last, nullptr, bf, c->stream); }
    { Scope s(c, K_LN); launch_layernorm(w.sel32, h, nb, h, tw.eps, tw.post_g, tw.post_b, nullptr, w.sel16, bf, c->stream); }
    if (!run_linear(c, tw.proj_w, &w.map_sel, w.sel16, bf, nb, w.proj32, tw.proj, EPI_STORE32, 0)) return false;
    { Scope s(c, K_OTHER); launch_l2norm(w.proj32, d_out, nb, tw.proj, normalize ? 1 : 0, c->stream); }
    CK(cudaGetLastError());
    return true;
}

// ---- per-token hidden states (clip_b200_image_tokens / clip_b200_text_tokens) ----------------------------------------------------
// What a tokens call asks for, checked and resolved: how many blocks to run, which rows of each item, how wide.
struct TokenReq {
    int blocks = 0, skip = 0, width = 0, esize = 4, flags = 0, out_type = 0;
    int attn = 0;              // ATTENTION entry: 1 full maps, 2 the CLS row only (K9 instead of the rows of x)
};

// One entry of a tokens call on a tower that is present.
bool token_request(const clip_ctx* c, bool vision, int layer, int flags, int out_type, TokenReq& q, const char* who) {
    const Tower& tw = vision ? c->vis : c->txt;
    const int nl = tw.layers;
    if (layer < -(nl + 1) || layer > nl) {
        set_err(std::string(who) + ": layer " + std::to_string(layer) + " is outside [" + std::to_string(-(nl + 1)) + ", " + std::to_string(nl) + "]");
        return false;
    }
    if (flags & ~(CLIP_B200_TOKENS_POST_LN | CLIP_B200_TOKENS_PROJECT | CLIP_B200_TOKENS_NORMALIZE | CLIP_B200_TOKENS_NO_CLS |
                  CLIP_B200_TOKENS_ATTENTION | CLIP_B200_TOKENS_ATTENTION_CLS)) { set_err(std::string(who) + ": unknown flag bits"); return false; }
    if (flags & (CLIP_B200_TOKENS_ATTENTION | CLIP_B200_TOKENS_ATTENTION_CLS)) {
        if (!(flags & CLIP_B200_TOKENS_ATTENTION)) { set_err(std::string(who) + ": CLIP_B200_TOKENS_ATTENTION_CLS needs CLIP_B200_TOKENS_ATTENTION"); return false; }
        if (flags & (CLIP_B200_TOKENS_POST_LN | CLIP_B200_TOKENS_PROJECT | CLIP_B200_TOKENS_NORMALIZE | CLIP_B200_TOKENS_NO_CLS)) {
            set_err(std::string(who) + ": CLIP_B200_TOKENS_ATTENTION cannot be combined with POST_LN, PROJECT, NORMALIZE or NO_CLS");
            return false;
        }
        if ((flags & CLIP_B200_TOKENS_ATTENTION_CLS) && !vision) { set_err(std::string(who) + ": CLIP_B200_TOKENS_ATTENTION_CLS is for the vision tower only"); return false; }
        if (layer == 0 || layer == -(nl + 1)) {
            set_err(std::string(who) + ": CLIP_B200_TOKENS_ATTENTION needs layer >= 1 (or -n_layer .. -1): layer " + std::to_string(layer) + " is before the first block");
            return false;
        }
    }
    if ((flags & CLIP_B200_TOKENS_NO_CLS) && !vision) { set_err(std::string(who) + ": CLIP_B200_TOKENS_NO_CLS is for the vision tower only"); return false; }
    if ((flags & CLIP_B200_TOKENS_NORMALIZE) && !(flags & CLIP_B200_TOKENS_PROJECT)) { set_err(std::string(who) + ": CLIP_B200_TOKENS_NORMALIZE needs CLIP_B200_TOKENS_PROJECT"); return false; }
    if (out_type != CLIP_B200_OUT_F32 && out_type != CLIP_B200_OUT_F16 && out_type != CLIP_B200_OUT_BF16) { set_err(std::string(who) + ": unknown out_type " + std::to_string(out_type)); return false; }
    // PROJECT keeps the projected rows in the qkv and g buffers, free once the blocks have run (every CLIP geometry: d <= h, ff = 4h)
    if ((flags & CLIP_B200_TOKENS_PROJECT) && (2 * (size_t)tw.proj > 3 * (size_t)tw.hidden || 2 * (size_t)tw.proj > (size_t)tw.ff)) {
        set_err(std::string(who) + ": CLIP_B200_TOKENS_PROJECT needs projection_dim <= 1.5 hidden_size and <= feed_forward_length / 2");
        return false;
    }
    q.blocks = layer < 0 ? nl + 1 + layer : layer;
    q.skip = (flags & CLIP_B200_TOKENS_NO_CLS) ? 1 : 0;
    q.width = (flags & CLIP_B200_TOKENS_PROJECT) ? tw.proj : tw.hidden;
    q.esize = out_type == CLIP_B200_OUT_F32 ? 4 : 2;
    q.flags = flags; q.out_type = out_type;
    if (flags & CLIP_B200_TOKENS_ATTENTION) q.attn = (flags & CLIP_B200_TOKENS_ATTENTION_CLS) ? 2 : 1;
    return true;
}

// one item's rows (or attention maps) of entry q in the output of a call of T rows per item
size_t item_bytes(const TokenReq& q, const Tower& tw, int T) {
    if (q.attn) return (size_t)tw.heads * (q.attn == 2 ? 1 : T) * T * q.esize;
    return (size_t)(T - q.skip) * q.width * q.esize;
}

// After the blocks: the requested rows of ws.x for nb items of T rows -> dst (device), item-major, item_bytes per item.
// PROJECT runs today's pooled tail on every row -- K2 post_ln into the 16-bit operand type, K1 projection (fp32), l2norm -- so the
// CLS / EOT rows come out bit-identical to clip_image_batch_encode / clip_text_batch_encode; K7 then picks and converts the rows.
// An ATTENTION entry runs K9 on ws.qkv, which still holds the last block's Q | K | V (token_stops emits it before any PROJECT tail).
bool token_rows_tail(clip_ctx* c, Tower& tw, int nb, int T, const TokenReq& q, void* dst) {
    Workspace& w = tw.ws;
    const int h = tw.hidden, M = nb * T, bf = c->operand_bf16 ? 1 : 0;
    const bool ln = q.flags & (CLIP_B200_TOKENS_POST_LN | CLIP_B200_TOKENS_PROJECT);
    if (q.attn) {
        Scope s(c, K_ATTN_PROBS);
        CK(launch_attention_probs(w.qkv, dst, q.out_type, nb, T, tw.heads, h / tw.heads, &tw == &c->txt ? 1 : 0, q.attn == 2 ? 1 : 0, bf, c->stream));
    } else if (!(q.flags & CLIP_B200_TOKENS_PROJECT)) {
        Scope s(c, K_TOKEN_ROWS);
        launch_token_rows(w.x, h, nb, T, q.skip, h, ln ? tw.post_g : nullptr, tw.post_b, tw.eps, q.out_type, dst, c->stream);
    } else {
        float* p32 = reinterpret_cast<float*>(w.qkv);     // [M, proj] fp32 in the [M, 3h] 16-bit buffer
        float* n32 = reinterpret_cast<float*>(w.g);       // [M, proj] fp32 in the [M, ff] 16-bit buffer
        { Scope s(c, K_LN); launch_layernorm(w.x, h, M, h, tw.eps, tw.post_g, tw.post_b, nullptr, w.a, bf, c->stream); }
        if (!run_linear(c, tw.proj_w, &w.map_a, w.a, bf, M, p32, tw.proj, EPI_STORE32, 0)) return false;
        if (q.flags & CLIP_B200_TOKENS_NORMALIZE) { Scope s(c, K_OTHER); launch_l2norm(p32, n32, M, tw.proj, 1, c->stream); p32 = n32; }
        { Scope s(c, K_TOKEN_ROWS); launch_token_rows(p32, tw.proj, nb, T, q.skip, tw.proj, nullptr, nullptr, 0.f, q.out_type, dst, c->stream); }
    }
    CK(cudaGetLastError());
    return true;
}

// The entries of one tokens call (one for the single-layer calls), for nb items whose embedding is in ws.x: the blocks run once, up
// to the deepest entry, each run resuming where the previous stop left x; after each block count some entry asks for, emit(j) writes
// entry j's rows (token_rows_tail) while x holds that layer.  Between stops x is live, and so is qkv until the stop's ATTENTION
// entries have run: the last block's QKV GEMM wrote it and nothing after K3 in a block writes it.  So at one stop the ATTENTION
// entries come first, and only then may a PROJECT tail use a, qkv and g as scratch.
template <class Emit>
bool token_stops(clip_ctx* c, Tower& tw, int nb, int T, bool causal, const std::vector<TokenReq>& qs, Emit emit) {
    std::vector<int> order(qs.size());
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        return qs[a].blocks != qs[b].blocks ? qs[a].blocks < qs[b].blocks : (qs[a].attn != 0) > (qs[b].attn != 0);
    });
    int done = 0;
    for (int j : order) {
        if (qs[j].blocks > done) {
            if (!run_blocks(c, tw, nb, T, causal, done, qs[j].blocks)) return false;
            done = qs[j].blocks;
        }
        if (!emit(j)) return false;
    }
    return true;
}

// Layer-major output of a tokens call of T rows per item: entry j's slab of n items starts at n * (item_bytes of the entries before
// it); the shard of items lo .. of a devices-mode GPU starts lo * item_bytes_j into each slab.  The slab after an ATTENTION slab
// starts at the next multiple of 16 bytes: attention items are H x R x T elements, often an odd count, and K7's vector stores need
// the alignment.
std::vector<char*> slab_bases(const std::vector<TokenReq>& qs, const Tower& tw, int T, char* out, size_t n, size_t lo) {
    std::vector<char*> b;
    size_t off = 0;
    for (const TokenReq& q : qs) {
        const size_t ib = item_bytes(q, tw, T);
        b.push_back(out + off + lo * ib);
        off += n * ib;
        if (q.attn) off = (off + 15) / 16 * 16;
    }
    return b;
}

// memcpy split over up to nt host threads
void parallel_copy(char* dst, const char* src, size_t bytes, int nt) {
    const size_t part = (bytes + nt - 1) / nt;
    if (nt <= 1 || bytes < ((size_t)4 << 20)) { memcpy(dst, src, bytes); return; }
    std::vector<std::thread> th;
    for (size_t o = 0; o < bytes; o += part) th.emplace_back([=]() { memcpy(dst + o, src + o, std::min(part, bytes - o)); });
    for (auto& t : th) t.join();
}

template <class T>
bool ensure_buf(clip_ctx* c, T** buf, size_t* cap, size_t count);
bool host_ptr_is_pinned(const void* p);

// Host forms: rows leave the device through a two-slot ring (c->d_ring) instead of holding the launch stream on PCIe.  K7 fills slot
// s on the launch stream; the copy stream takes it to the host once K7 is done (ev_ring_rows[s]), so the D2H of one stop runs under
// the blocks of the next, and the tail into slot s first waits for that slot's previous D2H (ev_ring_free[s]).  A pinned `out`
// receives the D2H directly.  A pageable one cannot take an async D2H, so the rows land in a pinned bounce slot (c->h_ring) that host
// threads drain into `out` before that slot is copied into again (encode_pass's arena for host images, the other way round).
// Caller holds c->mu and has set the device.
struct RowRing {
    clip_ctx* c;
    bool pinned = true;
    size_t slot = 0;            // bytes per slot: one micro-batch of the widest entry
    unsigned k = 0;             // stops so far; stop k uses slot k & 1
    int nt = 1;
    char* pend[2] = {nullptr, nullptr};
    size_t pend_bytes[2] = {0, 0};

    bool init(size_t slot_bytes, const void* out) {
        slot = (slot_bytes + 255) / 256 * 256;
        pinned = host_ptr_is_pinned(out);
        nt = std::max(1, std::min(16, (int)std::thread::hardware_concurrency()));
        if (!ensure_buf(c, &c->d_ring, &c->d_ring_cap, 2 * slot)) return false;
        if (!pinned && c->h_ring_cap < 2 * slot) {
            if (c->h_ring) { cudaFreeHost(c->h_ring); c->h_ring = nullptr; c->h_ring_cap = 0; }
            CK(cudaMallocHost((void**)&c->h_ring, 2 * slot));
            c->h_ring_cap = 2 * slot;
        }
        return true;
    }
    // rows of entry q for nb items -> dst (host)
    bool put(Tower& tw, int nb, int T, const TokenReq& q, char* dst) {
        const int s = (int)(k++ & 1);
        char* d = c->d_ring + s * slot;
        CK(cudaStreamWaitEvent(c->stream, c->ev_ring_free[s], 0));
        if (!token_rows_tail(c, tw, nb, T, q, d)) return false;
        CK(cudaEventRecord(c->ev_ring_rows[s], c->stream));
        if (!drain(s)) return false;
        const size_t bytes = (size_t)nb * item_bytes(q, tw, T);
        CK(cudaStreamWaitEvent(c->copy_stream, c->ev_ring_rows[s], 0));
        CK(cudaMemcpyAsync(pinned ? dst : c->h_ring + s * slot, d, bytes, cudaMemcpyDeviceToHost, c->copy_stream));
        CK(cudaEventRecord(c->ev_ring_free[s], c->copy_stream));
        if (!pinned) { pend[s] = dst; pend_bytes[s] = bytes; }
        return true;
    }
    // bounce slot s -> its destination, once its D2H has landed
    bool drain(int s) {
        if (!pend[s]) return true;
        CK(cudaEventSynchronize(c->ev_ring_free[s]));
        parallel_copy(pend[s], c->h_ring + s * slot, pend_bytes[s], nt);
        pend[s] = nullptr;
        return true;
    }
    // the launch stream waits for the last D2Hs, so the call's end event (and its synchronisation) covers them
    bool close() {
        for (int s = 0; s < 2; s++) CK(cudaStreamWaitEvent(c->stream, c->ev_ring_free[s], 0));
        return true;
    }
    bool drain_all() { return drain((int)(k & 1)) && drain((int)((k + 1) & 1)); }     // the older slot first
};

void dev_free(clip_ctx* c, void* p) {
    if (!p) return;
    auto it = std::find(c->allocs.begin(), c->allocs.end(), p);
    if (it != c->allocs.end()) c->allocs.erase(it);
    cudaFree(p);
}
// grow-only device buffer; the outgrown one is released once the stream has drained (nothing may still read it)
template <class T>
bool ensure_buf(clip_ctx* c, T** buf, size_t* cap, size_t count) {
    if (*cap >= count) return true;
    const size_t want = std::max(count, *cap + *cap / 2);
    T* p = nullptr;
    if (!dev_alloc(c, &p, want)) return false;
    if (*buf) { cudaStreamSynchronize(c->stream); dev_free(c, *buf); }
    *buf = p; *cap = want;
    return true;
}
bool ensure_out(clip_ctx* c, size_t floats) { return ensure_buf(c, &c->d_out, &c->d_out_cap, floats); }

int default_micro_batch(int T) {   // 33 token tiles = 132/4: every N/128 that is a multiple of 4 fills whole waves of the H100's SMs
    // Fewer, longer launches: each launch pays a drain/fill gap of a few microseconds.  9 x 33 tiles of 256 rows = 295 ViT-L/14 images
    // = 1.7 GB of workspace.
    int waves = 9;
    if (const char* e = getenv("CLIP_B200_TOKEN_TILES_X33")) waves = std::max(1, atoi(e));
    const int mb = 33 * waves * GEMM_BN / T;
    return mb < 1 ? 1 : mb;
}

void chunking(size_t n, int mb, size_t& n_chunks, size_t& chunk) {
    n_chunks = (n + mb - 1) / mb;
    chunk = (n + n_chunks - 1) / n_chunks;
}

// Chunk boundaries for inputs that still have to cross PCIe: the host->device copy of the FIRST micro-batch cannot hide under any
// kernel, so it is made small (a quarter of a micro-batch); the rest is split into balanced micro-batches as usual.
std::vector<size_t> host_chunk_bounds(size_t n, int mb) {
    std::vector<size_t> b{0};
    if (n <= (size_t)mb) { b.push_back(n); return b; }
    const size_t head = std::max<size_t>(1, (size_t)mb / 4);
    b.push_back(head);
    size_t n_chunks, chunk;
    chunking(n - head, mb, n_chunks, chunk);
    for (size_t i0 = head; i0 < n; i0 += chunk) b.push_back(std::min(n, i0 + chunk));
    return b;
}

bool sync_and_time(clip_ctx* c) {
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_err(std::string("kernel execution failed: ") + cudaGetErrorString(e)); return false; }
    cudaEventElapsedTime(&c->last_ms, c->ev_t0, c->ev_t1);
    return true;
}

// H x W = 0 x 0 or (image_size x image_size): T, the position table and the images per pass of the model's own size
// (micro_batch).  Another size (already checked by check_hw_size): T = (H/P)(W/P) + 1, the table resampled to that grid (K8, cached
// for the last size), and as many images per pass as fit every workspace buffer.  The workspace itself is always sized for
// micro_batch images of the native T, at the first call of the context whatever its size, so a native call after a *_hw one finds
// it as it would have.  Caller holds c->mu and has set the device.
bool plan_call(clip_ctx* c, int H, int W, VisCall& v, int& mb, const char* who) {
    Tower& tw = c->vis;
    if (!ensure_ws(c, tw, tw.micro_batch, tw.T, true)) return false;
    if (H == 0 || (H == tw.image_size && W == tw.image_size)) {
        v = native_call(tw);
        mb = tw.micro_batch;
        return true;
    }
    const int g = tw.image_size / tw.patch, gh = H / tw.patch, gw = W / tw.patch, h = tw.hidden;
    v.H = H; v.W = W; v.T = gh * gw + 1;
    // rows of x / a / qkv / g, the sel / proj rows, and the patch rows of patches / patch32 (the pixel buffers hold exactly P*P*3
    // floats per patch row, so they fit whenever the patch rows do)
    const Workspace& w = tw.ws;
    const size_t fit = std::min({(size_t)w.cap_rows / v.T, (size_t)w.cap_items, (size_t)w.cap_items * tw.n_patches / (v.T - 1)});
    if (fit < 1) {
        set_err(std::string(who) + ": one " + std::to_string(H) + " x " + std::to_string(W) + " image needs " + std::to_string(v.T) +
                " rows, more than the workspace holds (" + std::to_string(w.cap_rows) + "); raise clip_b200_set_micro_batch before the first encode");
        return false;
    }
    mb = (int)fit;
    if (c->pos_gh != gh || c->pos_gw != gw) {
        c->pos_gh = c->pos_gw = 0;
        if (!ensure_buf(c, &c->pos_hw, &c->pos_hw_cap, (size_t)v.T * h)) return false;
        CK(cudaMemcpyAsync(c->pos_hw, tw.pos, (size_t)h * 4, cudaMemcpyDeviceToDevice, c->stream));     // the CLS row as it is
        { Scope s(c, K_POS_RESAMPLE); launch_pos_resample(tw.pos + h, g, h, gh, gw, c->pos_hw + h, c->stream); }
        CK(cudaGetLastError());
        c->pos_gh = gh; c->pos_gw = gw;
    }
    v.pos = c->pos_hw;
    return true;
}

// a *_hw size: positive multiples of patch_size, at most 4096 on each side
bool check_hw_size(const clip_ctx* c, int H, int W, const char* who) {
    const int P = c->vis.patch;
    if (H <= 0 || W <= 0 || H % P || W % P || H > 4096 || W > 4096) {
        set_err(std::string(who) + ": height and width must be positive multiples of patch_size (" + std::to_string(P) + ") and at most 4096, not " +
                std::to_string(H) + " x " + std::to_string(W));
        return false;
    }
    return true;
}

// ---- devices mode helper: f(replica, r, lo, hi) on one host thread per GPU, contiguous balanced shards of n items --------------
template <class F>
bool for_each_replica(clip_ctx* c, size_t n, F f) {
    const int w = (int)c->replicas.size();
    std::vector<std::string> errs((size_t)w);
    std::vector<char> ok((size_t)w, 1);
    std::vector<std::thread> th;
    for (int r = 0; r < w; r++) {
        size_t lo, hi;
        shard_bounds(n, r, w, lo, hi);
        th.emplace_back([&, r, lo, hi]() {
            g_err.clear();
            ok[r] = f(c->replicas[r], r, lo, hi) ? 1 : 0;
            if (!ok[r]) errs[r] = g_err;
        });
    }
    for (auto& t : th) t.join();
    cudaSetDevice(c->device);
    for (int r = 0; r < w; r++)
        if (!ok[r]) { set_err("device " + std::to_string(c->replicas[r]->device) + ": " + errs[r]); return false; }
    return true;
}

bool ranks_mode(const clip_ctx* c) { return c->replicas.size() <= 1 && c->dist.comm && c->dist.world > 1; }

// ranks mode: every rank encodes ITS n_local items and ends with ALL world * n_local embeddings, rank-major.  The last kernel of
// the tower (K5 l2norm) writes straight into this rank's slot of the gather buffer; the all-gather runs in place on the launch stream.
bool gather_in_place(clip_ctx* c, float* d_all, size_t n_local, int d) {
    if (!ranks_mode(c)) return true;
    std::string e;
    const size_t bytes = n_local * (size_t)d * 4;
    if (!dist_all_gather(c->dist, (const char*)d_all + (size_t)c->dist.rank * bytes, d_all, bytes, c->stream, e)) { set_err(e); return false; }
    return true;
}

bool host_ptr_is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

}  // namespace

// =====================================================================================================================
// C ABI
// =====================================================================================================================
extern "C" {

const char* clip_b200_last_error(void) { return g_err.c_str(); }
const char* clip_b200_version(void) { return "clip_b200 0.1 (sm_90a; wgmma fused-dequant GEMM)"; }

// one replica of the model on `device` (weights, at most about 5 GB for ViT-bigG/14 in f16: replicated, never sharded -- SURVEY.md section 8e)
static clip_ctx* load_on_device(const GgufFile& g, int device, const int verbosity) {
    {
        std::unique_ptr<clip_ctx, void (*)(clip_ctx*)> guard(new clip_ctx, [](clip_ctx* p) { clip_free(p); });
        clip_ctx* c = guard.get();
        c->device = device;
        if (cudaSetDevice(c->device) != cudaSuccess) { set_err("cudaSetDevice failed"); return nullptr; }
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, c->device) != cudaSuccess) { set_err("cudaGetDeviceProperties failed"); return nullptr; }
        if (prop.major != 9 || prop.minor != 0) { set_err(std::string("device '") + prop.name + "' is not sm_90: this library only contains sm_90a code"); return nullptr; }
        c->num_sms = prop.multiProcessorCount;
        c->debug_naive = getenv("CLIP_B200_DEBUG_NAIVE") && atoi(getenv("CLIP_B200_DEBUG_NAIVE")) != 0;
        c->profile = getenv("CLIP_B200_PROFILE") && atoi(getenv("CLIP_B200_PROFILE")) != 0;
        if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { set_err("cudaStreamCreate failed"); return nullptr; }
        for (int i = 0; i < 2; i++) {
            cudaEventCreateWithFlags(&c->ev_copied[i], cudaEventDisableTiming);
            cudaEventCreateWithFlags(&c->ev_consumed[i], cudaEventDisableTiming);
            cudaEventCreateWithFlags(&c->ev_ring_rows[i], cudaEventDisableTiming);
            cudaEventCreateWithFlags(&c->ev_ring_free[i], cudaEventDisableTiming);
        }
        cudaEventCreate(&c->ev_t0);
        cudaEventCreate(&c->ev_t1);
        if (gemm_init() != cudaSuccess || attention_tc_init() != cudaSuccess) { set_err("cudaFuncSetAttribute(max dynamic smem) failed"); return nullptr; }
        if (const char* at = getenv("CLIP_B200_ATTN")) c->attn_tc = strcmp(at, "legacy") != 0;

        if (!kv_bool(g, "clip.has_text_encoder", c->has_text) || !kv_bool(g, "clip.has_vision_encoder", c->has_vision) ||
            !kv_bool(g, "clip.use_gelu", c->use_gelu)) return nullptr;
        if (verbosity >= 1) {
            const GgufKV* nm = g.find("general.name");
            const GgufKV* ds = g.find("general.description");
            const GgufKV* ft = g.find("general.file_type");
            if (nm) printf("%s: model name:   %s\n", "clip_model_load", nm->s.c_str());
            if (ds) printf("%s: description:  %s\n", "clip_model_load", ds->s.c_str());
            printf("%s: GGUF version: %u\n", "clip_model_load", g.version);
            printf("%s: alignment:    %zu\n", "clip_model_load", g.alignment);
            printf("%s: n_tensors:    %zu\n", "clip_model_load", g.tensors.size());
            printf("%s: n_kv:         %zu\n", "clip_model_load", g.kvs.size());
            if (ft) printf("%s: ftype:        %d\n", "clip_model_load", (int)ft->u);
            printf("%s: text_encoder:   %d\n%s: vision_encoder: %d\n", "clip_model_load", c->has_text, "clip_model_load", c->has_vision);
            printf("%s: device:       %d (%s, %d SMs)\n", "clip_model_load", c->device, prop.name, c->num_sms);
        }

        if (c->has_text) {
            Tower& t = c->txt;
            auto& hp = c->thp;
            if (!kv_u32(g, "clip.text.embedding_length", hp.hidden_size) || !kv_u32(g, "clip.text.attention.head_count", hp.n_head) ||
                !kv_u32(g, "clip.text.feed_forward_length", hp.n_intermediate) || !kv_u32(g, "clip.text.block_count", hp.n_layer) ||
                !kv_u32(g, "clip.text.context_length", hp.num_positions) || !kv_u32(g, "clip.text.projection_dim", hp.projection_dim) ||
                !kv_f32(g, "clip.text.attention.layer_norm_epsilon", hp.eps)) return nullptr;
            const GgufKV* tk = g.find("tokenizer.ggml.tokens");
            if (!tk || tk->type != GT_ARR || tk->arr_type != GT_STR) { set_err("key tokenizer.ggml.tokens not found in file"); return nullptr; }
            hp.n_vocab = (int32_t)tk->strs.size();
            for (int32_t i = 0; i < hp.n_vocab; i++) c->vocab.token_to_id[tk->strs[i]] = i;
            c->vocab.n = hp.n_vocab;
            t.present = true; t.hidden = hp.hidden_size; t.ff = hp.n_intermediate; t.heads = hp.n_head; t.layers = hp.n_layer;
            t.proj = hp.projection_dim; t.eps = hp.eps; t.n_vocab = hp.n_vocab; t.n_ctx = hp.num_positions;
            if (t.n_ctx <= 0 || t.n_ctx > 4096 || t.n_vocab <= 0) { set_err("text tower: bad context_length / vocabulary size"); return nullptr; }
            if (!check_geometry(c, "text tower", t)) return nullptr;
            if (!upload_f32(c, g, "t.token_embd.weight", &t.tok, (int64_t)t.n_vocab * t.hidden) ||
                !upload_f32(c, g, "t.position_embd.weight", &t.pos, (int64_t)t.n_ctx * t.hidden) ||
                !upload_f32(c, g, "t.post_ln.weight", &t.post_g, t.hidden) || !upload_f32(c, g, "t.post_ln.bias", &t.post_b, t.hidden)) return nullptr;
            if (!make_linear(c, g, {"text_projection.weight"}, {}, t.proj_w)) return nullptr;
            if (!load_blocks(c, g, "t", t)) return nullptr;
            t.micro_batch = default_micro_batch(t.n_ctx);
            if (verbosity >= 2)
                printf("\n%s: text model hparams\nn_vocab            %d\nnum_positions      %d\nt_hidden_size      %d\nt_n_intermediate   %d\nt_projection_dim   %d\nt_n_head           %d\nt_n_layer          %d\n",
                       "clip_model_load", hp.n_vocab, hp.num_positions, hp.hidden_size, hp.n_intermediate, hp.projection_dim, hp.n_head, hp.n_layer);
        }
        if (c->has_vision) {
            Tower& t = c->vis;
            auto& hp = c->vhp;
            if (!kv_u32(g, "clip.vision.embedding_length", hp.hidden_size) || !kv_u32(g, "clip.vision.attention.head_count", hp.n_head) ||
                !kv_u32(g, "clip.vision.feed_forward_length", hp.n_intermediate) || !kv_u32(g, "clip.vision.block_count", hp.n_layer) ||
                !kv_u32(g, "clip.vision.image_size", hp.image_size) || !kv_u32(g, "clip.vision.patch_size", hp.patch_size) ||
                !kv_u32(g, "clip.vision.projection_dim", hp.projection_dim) || !kv_f32(g, "clip.vision.attention.layer_norm_epsilon", hp.eps)) return nullptr;
            const GgufKV* km = g.find("clip.vision.image_mean");
            const GgufKV* ks = g.find("clip.vision.image_std");
            if (!km || !ks || km->type != GT_ARR || ks->type != GT_ARR || km->arr_type != GT_F32 || ks->arr_type != GT_F32 || km->arr_n < 3 || ks->arr_n < 3) {
                set_err("key clip.vision.image_mean / image_std not found in file"); return nullptr;
            }
            memcpy(c->image_mean, km->raw + 12, 12);
            memcpy(c->image_std, ks->raw + 12, 12);
            t.present = true; t.hidden = hp.hidden_size; t.ff = hp.n_intermediate; t.heads = hp.n_head; t.layers = hp.n_layer;
            t.proj = hp.projection_dim; t.eps = hp.eps; t.image_size = hp.image_size; t.patch = hp.patch_size;
            if (t.patch <= 0 || t.image_size <= 0 || t.image_size > 4096 || t.image_size % t.patch) { set_err("image_size must be a positive multiple of patch_size"); return nullptr; }
            t.n_patches = (t.image_size / t.patch) * (t.image_size / t.patch);
            t.T = t.n_patches + 1;
            t.kpad = (3 * t.patch * t.patch + GEMM_BK - 1) / GEMM_BK * GEMM_BK;
            if (!check_geometry(c, "vision tower", t)) return nullptr;
            if (!make_linear(c, g, {"v.patch_embd.weight"}, {}, t.patch_w, t.kpad)) return nullptr;
            if (t.patch_w.N != t.hidden) { set_err("v.patch_embd.weight shape mismatch"); return nullptr; }
            if (!upload_f32(c, g, "v.class_embd", &t.class_embd, t.hidden) ||
                !upload_f32(c, g, "v.position_embd.weight", &t.pos, (int64_t)t.T * t.hidden) ||
                !upload_f32(c, g, "v.pre_ln.weight", &t.pre_g, t.hidden) || !upload_f32(c, g, "v.pre_ln.bias", &t.pre_b, t.hidden) ||
                !upload_f32(c, g, "v.post_ln.weight", &t.post_g, t.hidden) || !upload_f32(c, g, "v.post_ln.bias", &t.post_b, t.hidden)) return nullptr;
            if (!make_linear(c, g, {"visual_projection.weight"}, {}, t.proj_w)) return nullptr;
            if (!load_blocks(c, g, "v", t)) return nullptr;
            t.micro_batch = default_micro_batch(t.T);
            if (verbosity >= 2)
                printf("\n%s: vision model hparams\nimage_size         %d\npatch_size         %d\nv_hidden_size      %d\nv_n_intermediate   %d\nv_projection_dim   %d\nv_n_head           %d\nv_n_layer          %d\n",
                       "clip_model_load", hp.image_size, hp.patch_size, hp.hidden_size, hp.n_intermediate, hp.projection_dim, hp.n_head, hp.n_layer);
        }
        // 16-bit operand type of the towers: fp16 when any tower GEMM weight is stored unquantized (the reference rounds
        // those activations to fp16 too, ggml.c:11333-11349); bf16 for fully quantized towers unless overridden.
        const bool f16w = any_f16_gemm(c->vis) || any_f16_gemm(c->txt);
        c->operand_bf16 = !f16w;
        if (const char* op = getenv("CLIP_B200_OPERAND")) {
            if (!strcmp(op, "f16")) c->operand_bf16 = false;
            else if (!strcmp(op, "bf16") && !f16w) c->operand_bf16 = true;
        }
        if (verbosity >= 1) printf("%s: operand type: %s%s\n", "clip_model_load", c->operand_bf16 ? "bf16" : "fp16", c->debug_naive ? "  [DEBUG naive GEMM]" : "");
        if (cudaDeviceSynchronize() != cudaSuccess) { set_err("upload failed"); return nullptr; }
        return guard.release();
    }
}

// CLIP_B200_DEVICES = "all" | "0,1,2,..." -> devices mode (several GPUs behind ONE context); otherwise CLIP_B200_DEVICE (default 0),
// or LOCAL_RANK when CLIP_B200_DIST=env asks the context to join the launcher's ranks (torchrun / mpirun style environment).
static bool parse_devices(int ndev, std::vector<int>& out) {
    out.clear();
    const char* dl = getenv("CLIP_B200_DEVICES");
    if (dl && *dl) {
        if (!strcmp(dl, "all")) { for (int i = 0; i < ndev; i++) out.push_back(i); return true; }
        const char* p = dl;
        while (*p) {
            char* e = nullptr;
            const long v = strtol(p, &e, 10);
            if (e == p || v < 0 || v >= ndev) { set_err(std::string("CLIP_B200_DEVICES: bad device list '") + dl + "'"); return false; }
            if (std::find(out.begin(), out.end(), (int)v) != out.end()) { set_err("CLIP_B200_DEVICES: duplicate device"); return false; }
            out.push_back((int)v);
            p = (*e == ',') ? e + 1 : e;
            if (*e && *e != ',') { set_err(std::string("CLIP_B200_DEVICES: bad device list '") + dl + "'"); return false; }
        }
        if (out.empty()) { set_err("CLIP_B200_DEVICES: empty device list"); return false; }
        return true;
    }
    const char* dist_env = getenv("CLIP_B200_DIST");
    const char* dv = getenv("CLIP_B200_DEVICE");
    int d = dv ? atoi(dv) : 0;
    if (!dv && dist_env && !strcmp(dist_env, "env") && getenv("LOCAL_RANK")) d = atoi(getenv("LOCAL_RANK"));
    if (d < 0 || d >= ndev) { set_err("CLIP_B200_DEVICE out of range"); return false; }
    out.push_back(d);
    return true;
}

struct clip_ctx* clip_model_load(const char* fname, const int verbosity) {
    try {
        g_err.clear();
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device: libclip_b200 has no CPU path"); return nullptr; }
        GgufFile g;
        std::string err;
        if (!g.parse(fname, err)) { set_err(err); return nullptr; }
        std::vector<int> devs;
        if (!parse_devices(ndev, devs)) return nullptr;
        std::unique_ptr<clip_ctx, void (*)(clip_ctx*)> leader(load_on_device(g, devs[0], verbosity), [](clip_ctx* p) { clip_free(p); });
        if (!leader) return nullptr;
        if (devs.size() > 1) {
            // devices mode: one replica + one NCCL communicator per GPU, all owned by the leader context
            leader->replicas.push_back(leader.get());
            for (size_t i = 1; i < devs.size(); i++) {
                clip_ctx* r = load_on_device(g, devs[i], 0);
                if (!r) return nullptr;
                r->is_replica = true;
                leader->replicas.push_back(r);
            }
            std::vector<DistComm> comms(devs.size());
            std::string derr;
            if (!dist_init_all(comms.data(), devs.data(), (int)devs.size(), derr)) { set_err("devices mode: " + derr); return nullptr; }
            for (size_t i = 0; i < devs.size(); i++) leader->replicas[i]->dist = comms[i];
            if (verbosity >= 1) printf("%s: devices mode: %zu GPUs, NCCL %d\n", __func__, devs.size(), dist_nccl_version());
            cudaSetDevice(leader->device);
        } else if (const char* de = getenv("CLIP_B200_DIST")) {
            if (!strcmp(de, "env") && getenv("RANK") && getenv("WORLD_SIZE") && atoi(getenv("WORLD_SIZE")) > 1) {
                if (!clip_b200_dist_init(leader.get(), atoi(getenv("RANK")), atoi(getenv("WORLD_SIZE")), nullptr)) return nullptr;
            }
        }
        return leader.release();
    } catch (const std::exception& e) {
        set_err(std::string("clip_model_load: ") + e.what());
        return nullptr;
    }
}

void clip_free(struct clip_ctx* c) {
    if (!c) return;
    for (size_t i = 1; i < c->replicas.size(); i++) { c->replicas[i]->is_replica = false; clip_free(c->replicas[i]); }
    c->replicas.clear();
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    dist_destroy(c->dist);
    preprocess_release(c);
    for (void* p : c->allocs) cudaFree(p);
    for (int i = 0; i < 2; i++) if (c->h_stage[i]) cudaFreeHost(c->h_stage[i]);
    if (c->h_ring) cudaFreeHost(c->h_ring);
    for (auto& p : c->prof) { cudaEventDestroy(p.e0); cudaEventDestroy(p.e1); }
    for (auto e : c->ev_pool) cudaEventDestroy(e);
    for (int i = 0; i < 2; i++) { if (c->ev_copied[i]) cudaEventDestroy(c->ev_copied[i]); if (c->ev_consumed[i]) cudaEventDestroy(c->ev_consumed[i]); }
    for (int i = 0; i < 2; i++) { if (c->ev_ring_rows[i]) cudaEventDestroy(c->ev_ring_rows[i]); if (c->ev_ring_free[i]) cudaEventDestroy(c->ev_ring_free[i]); }
    for (int i = 0; i < 4; i++) if (c->marks[i]) cudaEventDestroy(c->marks[i]);
    if (c->ev_t0) cudaEventDestroy(c->ev_t0);
    if (c->ev_t1) cudaEventDestroy(c->ev_t1);
    if (c->stream) cudaStreamDestroy(c->stream);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    delete c;
}

struct clip_text_hparams* clip_get_text_hparams(struct clip_ctx* ctx) { return &ctx->thp; }
struct clip_vision_hparams* clip_get_vision_hparams(struct clip_ctx* ctx) { return &ctx->vhp; }

bool clip_tokenize(const struct clip_ctx* ctx, const char* text, struct clip_tokens* tokens) {
    if (!ctx || !ctx->has_text) { printf("This GGUF file seems to have no text encoder\n"); return false; }
    try {
        std::vector<int32_t> v = tokenize(ctx->vocab, text);
        tokens->size = v.size();
        tokens->data = new clip_vocab_id[v.size()];
        std::copy(v.begin(), v.end(), tokens->data);
        return true;
    } catch (...) { return false; }
}

struct clip_image_u8* clip_image_u8_make() { return new clip_image_u8(); }
struct clip_image_f32* clip_image_f32_make() { return new clip_image_f32(); }
void clip_image_u8_clean(struct clip_image_u8* img) { if (img && img->data) { delete[] img->data; img->data = nullptr; } }
void clip_image_f32_clean(struct clip_image_f32* res) { if (res && res->data) { delete[] res->data; res->data = nullptr; } }
void clip_image_u8_free(struct clip_image_u8* img) { clip_image_u8_clean(img); delete img; }
void clip_image_f32_free(struct clip_image_f32* res) { clip_image_f32_clean(res); delete res; }

bool clip_image_load_from_file(const char* fname, struct clip_image_u8* img) {
    std::vector<uint8_t> rgb;
    int nx = 0, ny = 0;
    if (!load_image_file(fname, rgb, nx, ny)) {
        set_err(std::string("clip_image_load_from_file: cannot decode '") + fname + "': supported formats are JPEG (Huffman baseline / progressive, 8-bit), PNG, "
                "BMP (uncompressed), GIF (first frame) and binary PGM / PPM; TGA / PSD / HDR / PIC and arithmetic-coded or 12-bit JPEG are not decoded by this library -- convert first");
        return false;
    }
    img->nx = nx; img->ny = ny; img->size = rgb.size();
    img->data = new uint8_t[rgb.size()];
    memcpy(img->data, rgb.data(), rgb.size());
    return true;
}

bool clip_image_preprocess(const struct clip_ctx* ctx, const struct clip_image_u8* img, struct clip_image_f32* res) {
    if (!ctx || !ctx->has_vision) { printf("This gguf file seems to have no vision encoder\n"); return false; }
    const int S = ctx->vhp.image_size;
    res->nx = S; res->ny = S; res->size = (size_t)3 * S * S;
    res->data = new float[res->size]();
    if (!preprocess_image(img->data, img->nx, img->ny, S, ctx->image_mean, ctx->image_std, res->data)) {
        delete[] res->data; res->data = nullptr;
        return false;
    }
    return true;
}

void clip_image_batch_preprocess(const struct clip_ctx* ctx, const int n_threads, const struct clip_image_u8_batch* in,
                                 struct clip_image_f32_batch* out) {
    // CLIP_B200_PREPROCESS=device: the same call runs K6a/K6b on the GPU (bit-identical results, new[]-owned buffers as below); a
    // failure is reported and leaves the outputs empty -- no silent detour through the host loop
    const char* where = getenv("CLIP_B200_PREPROCESS");
    if (where && strcmp(where, "device") == 0 && in->size > 0) {
        if (!clip_b200_image_batch_preprocess_device(ctx, in, out)) {
            fprintf(stderr, "clip_image_batch_preprocess (device): %s\n", clip_b200_last_error());
            for (size_t i = 0; i < in->size; i++) { out->data[i].data = nullptr; out->data[i].size = 0; }
        }
        return;
    }
    out->size = in->size;
    const size_t n = in->size;
    int nt = std::max(1, std::min<int>(n_threads, (int)n));
    if (nt == 1) { for (size_t i = 0; i < n; i++) clip_image_preprocess(ctx, &in->data[i], &out->data[i]); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nt; t++)
        th.emplace_back([=]() { for (size_t i = t; i < n; i += nt) clip_image_preprocess(ctx, &in->data[i], &out->data[i]); });
    for (auto& t : th) t.join();
}

// ---- pooled embeddings: the clip_*_encode* forms and the u8 forms ----------------------------------------------------------------
static bool check_images(clip_ctx* c, const clip_image_f32* imgs, size_t n, const char* who) {
    for (size_t i = 0; i < n; i++)
        if (imgs[i].nx != c->vis.image_size || imgs[i].ny != c->vis.image_size || !imgs[i].data) { set_err(std::string(who) + ": every image must be image_size x image_size"); return false; }
    return true;
}

// host *_hw forms: the size is the images' own (ny rows of nx pixels), the same for every image of the call
static bool check_images_hw(clip_ctx* c, const clip_image_f32* imgs, size_t n, int& H, int& W, const char* who) {
    H = imgs[0].ny; W = imgs[0].nx;
    for (size_t i = 0; i < n; i++) {
        if (!imgs[i].data) { set_err(std::string(who) + ": image " + std::to_string(i) + " has no pixels"); return false; }
        if (imgs[i].ny != H || imgs[i].nx != W) {
            set_err(std::string(who) + ": every image of one call must have the same size (height x width: image 0 is " + std::to_string(H) + " x " +
                    std::to_string(W) + ", image " + std::to_string(i) + " is " + std::to_string(imgs[i].ny) + " x " + std::to_string(imgs[i].nx) + ")");
            return false;
        }
    }
    return check_hw_size(c, H, W, who);
}

// host token sequences: none empty, none longer than context_length
static bool check_tokens(const clip_ctx* c, const clip_tokens* seqs, size_t n, const char* who) {
    size_t T = 0;
    for (size_t i = 0; i < n; i++) {
        if (seqs[i].size == 0 || !seqs[i].data) { set_err(std::string(who) + ": empty token sequence"); return false; }
        T = std::max(T, seqs[i].size);
    }
    if (T > (size_t)c->txt.n_ctx) { set_err(std::string(who) + ": token sequence longer than context_length (" + std::to_string(c->txt.n_ctx) + ")"); return false; }
    return true;
}

// checked host token sequences -> padded id matrix + EOT row indices.  Padding to a multiple of 8 tokens is causally invisible to the
// EOT row.
static void pack_tokens(const clip_ctx* c, const clip_tokens* seqs, size_t n, std::vector<int32_t>& ids, std::vector<int32_t>& last, int& T_out) {
    size_t T = 0;
    for (size_t i = 0; i < n; i++) T = std::max(T, seqs[i].size);
    T = std::min<size_t>((T + 7) / 8 * 8, (size_t)c->txt.n_ctx);
    ids.assign(n * T, 0);
    last.resize(n);
    for (size_t i = 0; i < n; i++) {
        memcpy(ids.data() + i * T, seqs[i].data, seqs[i].size * 4);
        last[i] = (int32_t)seqs[i].size - 1;     // the reference selects row N-1 (clip.cpp:1154-1155)
    }
    T_out = (int)T;
}

// What one pooled call reads, as its public form received it.  Each form fills one and calls encode_call, so every form checks its
// arguments in the same order (include/clip_b200.h) and runs the same pass driver.
struct EncodeCall {
    enum Input { F32_IMAGES, U8_IMAGES, DEVICE_PIXELS, TOKENS, DEVICE_IDS };
    const char* who;                              // the public name, for messages
    Input input;
    const void* in = nullptr;                     // host: clip_image_f32 / clip_image_u8 / clip_tokens [n]; device: NHWC f32 pixels or ids [n, seq_len]
    const int32_t* d_lens = nullptr;              // DEVICE_IDS: true lengths [n] (NULL: all seq_len)
    size_t n = 0;
    bool hw = false;                              // any patch-multiple size, H x W given (device) or the images' own (host)
    int H = 0, W = 0, seq_len = 0;
    int n_threads = 4;                            // host threads that gather pageable f32 images into the pinned arena
    bool normalize = true;
    float* vec = nullptr;                         // host output [n, proj]
    float* d_vec = nullptr;                       // device output [n, proj]; an *_all form's is [world * n, proj]
    clip_image_f32_batch* pixels = nullptr;       // the preprocessed u8 images, copied back to the host instead of any forward
    bool all = false;                             // an *_all form: in ranks mode, every rank's embeddings out
    bool reference = false;                       // a form of the reference's clip.h: prints the reference's line for a missing tower
    bool vision() const { return input <= DEVICE_PIXELS; }
    void batch(const clip_image_f32_batch* b) { if (b) { in = b->data; n = b->size; } }     // a NULL batch is an empty one
    void batch(const clip_image_u8_batch* b) { if (b) { in = b->data; n = b->size; } }
};

// One GPU, items lo .. hi of a checked call: their embeddings into d_vec (device; NULL: the context's own buffer when vec is set, and no
// forward at all when it is not), then into vec (host) unless it is NULL; sync: synchronise the launch stream and time the call.  Only
// staging a micro-batch differs by input kind.  Host f32 pixels travel on the copy stream, double-buffered against the kernels of the
// previous micro-batch.  Pinned / registered caller buffers are copied directly; PAGEABLE ones (what clip_image_preprocess returns:
// new float[]) are first gathered into a pinned arena by host threads, in sub-batches so the H2D of sub-batch k overlaps the memcpy of
// k+1 -- a pageable cudaMemcpyAsync would be staged synchronously by the driver, one 602 KB image at a time.
static bool encode_pass(clip_ctx* c, const EncodeCall& a, size_t lo, size_t hi, float* vec, float* d_vec, bool sync) {
    Tower& tw = a.vision() ? c->vis : c->txt;
    const size_t n = hi - lo;
    // ids / last are pageable vectors: the async copies below return only after the driver has staged them, so they may go out of
    // scope when this function returns even with sync == false
    std::vector<int32_t> ids, last;
    int T = a.seq_len;
    if (a.input == EncodeCall::TOKENS) pack_tokens(c, (const clip_tokens*)a.in + lo, n, ids, last, T);
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    VisCall v;
    int mb = tw.micro_batch;
    // the padded text length is fixed per context so that one workspace serves every call
    if (a.vision() ? !plan_call(c, a.H, a.W, v, mb, a.who) : !ensure_ws(c, tw, tw.micro_batch, tw.n_ctx, false)) return false;
    if (!d_vec && vec) {
        if (!ensure_out(c, n * tw.proj)) return false;
        d_vec = c->d_out;
    }
    std::vector<size_t> bounds{0};
    if (a.input == EncodeCall::F32_IMAGES) {
        bounds = host_chunk_bounds(n, mb);
    } else {
        size_t n_chunks, chunk;
        chunking(n, mb, n_chunks, chunk);
        for (size_t i0 = 0; i0 < n; i0 += chunk) bounds.push_back(std::min(n, i0 + chunk));
    }
    const size_t per = v.per();
    const clip_image_f32* imgs = a.input == EncodeCall::F32_IMAGES ? (const clip_image_f32*)a.in + lo : nullptr;
    bool pinned = true;
    int nt = 1;
    if (imgs) {
        for (size_t i = 0; i < n && pinned; i++) pinned = host_ptr_is_pinned(imgs[i].data);
        if (!pinned && c->h_stage_cap < (size_t)mb * per) {
            for (int b = 0; b < 2; b++) {
                if (c->h_stage[b]) { cudaFreeHost(c->h_stage[b]); c->h_stage[b] = nullptr; }
                CK(cudaMallocHost((void**)&c->h_stage[b], (size_t)mb * per * 4));
            }
            c->h_stage_cap = (size_t)mb * per;
        }
        nt = std::max(1, std::min({std::max(a.n_threads, 4), 16, (int)std::thread::hardware_concurrency()}));
    }
    std::vector<float> h_pixels(a.pixels ? n * per : 0);
    CK(cudaEventRecord(c->ev_t0, c->stream));
    for (size_t ci = 0; ci + 1 < bounds.size(); ci++) {
        const size_t i0 = bounds[ci];
        const int nb = (int)(bounds[ci + 1] - i0), b = (int)(ci & 1);
        const float* px = tw.ws.pixels[b];
        if (a.input == EncodeCall::F32_IMAGES) {
            if (ci >= 2) CK(cudaStreamWaitEvent(c->copy_stream, c->ev_consumed[b], 0));
            if (pinned) {
                for (int j = 0; j < nb; j++)
                    CK(cudaMemcpyAsync(tw.ws.pixels[b] + (size_t)j * per, imgs[i0 + j].data, per * 4, cudaMemcpyHostToDevice, c->copy_stream));
            } else {
                if (ci >= 2) CK(cudaEventSynchronize(c->ev_copied[b]));      // the arena's previous H2D has left the host buffer
                const int sub = 32;
                for (int j0 = 0; j0 < nb; j0 += sub) {
                    const int ns = std::min(sub, nb - j0);
                    float* dst = c->h_stage[b] + (size_t)j0 * per;
                    const clip_image_f32* src = imgs + i0 + j0;
                    const int t_use = std::min(nt, ns);
                    if (t_use <= 1) { for (int j = 0; j < ns; j++) memcpy(dst + (size_t)j * per, src[j].data, per * 4); }
                    else {
                        std::vector<std::thread> th;
                        for (int t = 0; t < t_use; t++)
                            th.emplace_back([=]() { for (int j = t; j < ns; j += t_use) memcpy(dst + (size_t)j * per, src[j].data, per * 4); });
                        for (auto& t : th) t.join();
                    }
                    CK(cudaMemcpyAsync(tw.ws.pixels[b] + (size_t)j0 * per, dst, (size_t)ns * per * 4, cudaMemcpyHostToDevice, c->copy_stream));
                }
            }
            CK(cudaEventRecord(c->ev_copied[b], c->copy_stream));
            CK(cudaStreamWaitEvent(c->stream, c->ev_copied[b], 0));
        } else if (a.input == EncodeCall::U8_IMAGES) {
            if (ci >= 2) CK(cudaEventSynchronize(c->ev_consumed[b]));      // arena b is rewritten on the host below
            std::string err;
            if (!preprocess_device(c, (const clip_image_u8*)a.in + lo + i0, nb, b, tw.ws.pixels[b], c->copy_stream, c->ev_copied[b], c->stream, err)) {
                set_err(std::string(a.who) + ": " + err);
                return false;
            }
            if (a.pixels) CK(cudaMemcpyAsync(h_pixels.data() + i0 * per, tw.ws.pixels[b], (size_t)nb * per * 4, cudaMemcpyDeviceToHost, c->stream));
        } else if (a.input == EncodeCall::DEVICE_PIXELS) {
            px = (const float*)a.in + (lo + i0) * per;
        } else if (a.input == EncodeCall::TOKENS) {
            CK(cudaMemcpyAsync(tw.ws.ids, ids.data() + i0 * T, (size_t)nb * T * 4, cudaMemcpyHostToDevice, c->stream));
            CK(cudaMemcpyAsync(tw.ws.last, last.data() + i0, (size_t)nb * 4, cudaMemcpyHostToDevice, c->stream));
        } else {
            // lengths stay on the device: a tiny kernel turns them into EOT-row indices (clamped to [1, seq_len])
            CK(cudaMemcpyAsync(tw.ws.ids, (const int32_t*)a.in + (lo + i0) * T, (size_t)nb * T * 4, cudaMemcpyDeviceToDevice, c->stream));
            launch_fill_last(a.d_lens ? a.d_lens + lo + i0 : nullptr, tw.ws.last, nb, T, c->stream);
        }
        if (d_vec && !(a.vision() ? vision_forward(c, px, nb, v, d_vec + i0 * tw.proj, a.normalize)
                                  : text_forward(c, nb, T, d_vec + i0 * tw.proj, a.normalize))) return false;
        if (a.input == EncodeCall::F32_IMAGES || a.input == EncodeCall::U8_IMAGES) CK(cudaEventRecord(c->ev_consumed[b], c->stream));
    }
    CK(cudaEventRecord(c->ev_t1, c->stream));
    if (vec) CK(cudaMemcpyAsync(vec, d_vec, n * tw.proj * 4, cudaMemcpyDeviceToHost, c->stream));
    if (sync && !sync_and_time(c)) return false;
    if (a.pixels)
        for (size_t i = 0; i < n; i++) {        // same ownership convention as clip_image_preprocess: data is new[]-allocated here
            clip_image_f32& o = a.pixels->data[lo + i];
            o.nx = v.W; o.ny = v.H; o.size = per;
            o.data = new float[per];
            memcpy(o.data, h_pixels.data() + i * per, per * 4);
        }
    return true;
}

// Devices mode shards a text call only from this many sequences per GPU: a sequence is a fraction of an image's work (77 rows against
// 257 for ViT-L/14, on a smaller tower), so a GPU needs more of them before its share outweighs the fixed cost of its host thread,
// launches and synchronise.
const size_t TEXT_SHARD_MIN = 8;

// Every pooled form: the arguments checked in one order, the first fault refused (include/clip_b200.h), then the pass.  Devices mode
// shards the forms with a host output over the GPUs, each GPU copying its slice into vec; an *_all form encodes this rank's items into
// its slot of the gather buffer and all-gathers every rank's (outside ranks mode the device forms run the same steps without the
// exchange, and the host forms are the plain ones).
static bool encode_call(const clip_ctx* cctx, EncodeCall a) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    const std::string who = a.who;
    if (a.reference && !(c && (a.vision() ? c->has_vision : c->has_text))) {
        printf(a.vision() ? "This gguf file seems to have no vision encoder\n" : "This GGUF file seems to have no text encoder\n");
        return false;
    }
    if (!c) { set_err(who + ": null context"); return false; }
    const Tower& tw = a.vision() ? c->vis : c->txt;
    if (!tw.present) { set_err(who + ": this model has no " + (a.vision() ? "vision" : "text") + " encoder"); return false; }
    const bool device = a.input == EncodeCall::DEVICE_PIXELS || a.input == EncodeCall::DEVICE_IDS;
    if (a.hw && device && !check_hw_size(c, a.H, a.W, a.who)) return false;
    const bool ranks = a.all && ranks_mode(c);
    if (a.pixels) a.pixels->size = a.n;
    if (a.n == 0) {
        if (!ranks) return true;
        set_err(who + ": every rank must pass the same, non-zero number of " + (a.vision() ? "images" : "sequences"));
        return false;
    }
    if (a.input == EncodeCall::DEVICE_IDS && (a.seq_len < 1 || a.seq_len > tw.n_ctx)) { set_err(who + ": seq_len must be in [1, context_length]"); return false; }
    if (!a.in || !(a.vec || a.d_vec || a.pixels)) {
        set_err(who + (device ? ": null device pointer" : a.in ? ": null output" : ": null input"));
        return false;
    }
    if (a.input == EncodeCall::F32_IMAGES) {
        const clip_image_f32* imgs = (const clip_image_f32*)a.in;
        if (!(a.hw ? check_images_hw(c, imgs, a.n, a.H, a.W, a.who) : check_images(c, imgs, a.n, a.who))) return false;
    }
    if (a.input == EncodeCall::TOKENS && !check_tokens(c, (const clip_tokens*)a.in, a.n, a.who)) return false;
    const int d = tw.proj;
    if (a.all && (device || ranks)) {
        const int w = ranks ? c->dist.world : 1, rank = ranks ? c->dist.rank : 0;
        float* all = a.d_vec;
        if (!all) {
            std::lock_guard<std::mutex> lk(c->mu);
            CK(cudaSetDevice(c->device));
            if (!ensure_out(c, (size_t)w * a.n * d)) return false;
            all = c->d_out;
        }
        if (!encode_pass(c, a, 0, a.n, nullptr, all + (size_t)rank * a.n * d, false)) return false;
        std::lock_guard<std::mutex> lk(c->mu);
        if (!gather_in_place(c, all, a.n, d)) return false;
        CK(cudaEventRecord(c->ev_t1, c->stream));
        if (a.vec) CK(cudaMemcpyAsync(a.vec, all, (size_t)w * a.n * d * 4, cudaMemcpyDeviceToHost, c->stream));
        return sync_and_time(c);
    }
    if (a.vec && c->replicas.size() > 1 && a.n >= (a.vision() ? 1 : TEXT_SHARD_MIN) * c->replicas.size())
        return for_each_replica(c, a.n, [&](clip_ctx* r, int, size_t lo, size_t hi) { return hi == lo || encode_pass(r, a, lo, hi, a.vec + lo * d, nullptr, true); });
    return encode_pass(c, a, 0, a.n, a.vec, a.d_vec, true);
}

bool clip_b200_image_batch_encode_u8(const struct clip_ctx* cctx, const struct clip_image_u8_batch* imgs, float* vec, const bool normalize) {
    EncodeCall a{"clip_b200_image_batch_encode_u8", EncodeCall::U8_IMAGES};
    a.batch(imgs); a.normalize = normalize; a.vec = vec;
    return encode_call(cctx, a);
}

bool clip_b200_image_batch_preprocess_device(const struct clip_ctx* cctx, const struct clip_image_u8_batch* in, struct clip_image_f32_batch* out) {
    EncodeCall a{"clip_b200_image_batch_preprocess_device", EncodeCall::U8_IMAGES};
    a.batch(in); a.pixels = out;
    return encode_call(cctx, a);
}

bool clip_b200_image_encode_device(const struct clip_ctx* cctx, const void* d_pixels, size_t n, void* d_vec, bool normalize) {
    EncodeCall a{"clip_b200_image_encode_device", EncodeCall::DEVICE_PIXELS};
    a.in = d_pixels; a.n = n; a.normalize = normalize; a.d_vec = (float*)d_vec;
    return encode_call(cctx, a);
}

bool clip_b200_image_encode_device_hw(const struct clip_ctx* cctx, const void* d_pixels, size_t n, int height, int width, void* d_vec,
                                      bool normalize) {
    EncodeCall a{"clip_b200_image_encode_device_hw", EncodeCall::DEVICE_PIXELS};
    a.in = d_pixels; a.n = n; a.hw = true; a.H = height; a.W = width; a.normalize = normalize; a.d_vec = (float*)d_vec;
    return encode_call(cctx, a);
}

bool clip_image_batch_encode(const struct clip_ctx* cctx, const int n_threads, const struct clip_image_f32_batch* imgs, float* vec,
                             const bool normalize) {
    EncodeCall a{"clip_image_batch_encode", EncodeCall::F32_IMAGES};
    a.batch(imgs); a.n_threads = n_threads; a.normalize = normalize; a.vec = vec; a.reference = true;
    return encode_call(cctx, a);
}

bool clip_b200_image_batch_encode_hw(const struct clip_ctx* cctx, const struct clip_image_f32_batch* imgs, float* vec, bool normalize) {
    EncodeCall a{"clip_b200_image_batch_encode_hw", EncodeCall::F32_IMAGES};
    a.batch(imgs); a.hw = true; a.normalize = normalize; a.vec = vec;
    return encode_call(cctx, a);
}

bool clip_image_encode(const struct clip_ctx* ctx, const int n_threads, struct clip_image_f32* img, float* vec, const bool normalize) {
    clip_image_f32_batch b;
    b.data = img; b.size = 1;
    return clip_image_batch_encode(ctx, n_threads, &b, vec, normalize);
}

bool clip_text_batch_encode(const struct clip_ctx* cctx, const int n_threads, const struct clip_tokens* seqs, const size_t n, float* vec,
                            const bool normalize) {
    (void)n_threads;
    EncodeCall a{"clip_text_batch_encode", EncodeCall::TOKENS};
    a.in = seqs; a.n = n; a.normalize = normalize; a.vec = vec; a.reference = true;
    return encode_call(cctx, a);
}

bool clip_text_encode(const struct clip_ctx* ctx, const int n_threads, const struct clip_tokens* tokens, float* vec, const bool normalize) {
    return clip_text_batch_encode(ctx, n_threads, tokens, 1, vec, normalize);
}

bool clip_b200_text_encode_device(const struct clip_ctx* cctx, const void* d_ids, const void* d_lens, size_t n, int seq_len, void* d_vec,
                                  bool normalize) {
    EncodeCall a{"clip_b200_text_encode_device", EncodeCall::DEVICE_IDS};
    a.in = d_ids; a.d_lens = (const int32_t*)d_lens; a.n = n; a.seq_len = seq_len; a.normalize = normalize; a.d_vec = (float*)d_vec;
    return encode_call(cctx, a);
}

// ---- per-token hidden states: the ten clip_b200_*_tokens* forms -------------------------------------------------------------------
// What one tokens call reads, as its public form received it.  Each form fills one and calls tokens_call, so every form checks its
// arguments in the same order (include/clip_b200.h) and runs the same pass driver.
struct TokensCall {
    const char* who;                              // the public name, for messages
    bool vision, host;                            // the tower; inputs and out in host memory (else device memory)
    bool hw = false;                              // vision: any patch-multiple size, H x W given (device) or the images' own (host)
    const clip_image_f32_batch* imgs = nullptr;   // vision, host: the images, n = imgs->size
    const void* in = nullptr;                     // vision, device: NHWC f32 pixels; text: ids [n, seq_len]
    size_t n = 0;
    int H = 0, W = 0, seq_len = 0;
    const int* layers = nullptr;                  // n_layers entries; a single-layer form passes its one (layer, flags)
    const int* flags = nullptr;                   // NULL: 0 for every entry
    int n_layers = 1;
    bool list = false;                            // a *_layers form: n_layers and layers are checked, messages name the entry
    int out_type = 0;
    void* out = nullptr;
};

// One GPU, items lo .. hi of a checked call.  Per micro-batch: stage its inputs (host images go up one copy per image on the launch
// stream into ws.pixels[0], device pixels are read in place, ids are copied into ws.ids), embed them, then token_stops; each entry's
// rows go to its slab (bases[j] = item lo in slab j), through the RowRing for host memory, so the whole output is never held on the
// device.
static bool tokens_pass(clip_ctx* c, const TokensCall& a, const std::vector<TokenReq>& qs, size_t lo, size_t hi) {
    Tower& tw = a.vision ? c->vis : c->txt;
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    VisCall v;
    int mb = tw.micro_batch, T = a.seq_len;
    if (a.vision) {
        if (!plan_call(c, a.H, a.W, v, mb, a.who)) return false;
        T = v.T;
    } else if (!ensure_ws(c, tw, tw.micro_batch, tw.n_ctx, false)) {
        return false;
    }
    const size_t n = hi - lo;
    size_t n_chunks, chunk;
    chunking(n, mb, n_chunks, chunk);
    const std::vector<char*> bases = slab_bases(qs, tw, T, (char*)a.out, a.n, lo);
    RowRing ring{c};
    if (a.host) {
        size_t widest = 0;
        for (const TokenReq& q : qs) widest = std::max(widest, item_bytes(q, tw, T));
        if (!ring.init(chunk * widest, bases[0])) return false;
    }
    const size_t per = v.per();
    CK(cudaEventRecord(c->ev_t0, c->stream));
    for (size_t i0 = 0; i0 < n; i0 += chunk) {
        const int nb = (int)std::min(chunk, n - i0);
        const size_t i = lo + i0;     // the call's index of the micro-batch's first item
        if (a.vision && a.host) {
            for (int j = 0; j < nb; j++)
                CK(cudaMemcpyAsync(tw.ws.pixels[0] + (size_t)j * per, a.imgs->data[i + j].data, per * 4, cudaMemcpyHostToDevice, c->stream));
            if (!vision_embed(c, tw.ws.pixels[0], nb, v)) return false;
        } else if (a.vision) {
            if (!vision_embed(c, (const float*)a.in + i * per, nb, v)) return false;
        } else {
            CK(cudaMemcpyAsync(tw.ws.ids, (const int32_t*)a.in + i * T, (size_t)nb * T * 4,
                               a.host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream));
            { Scope s(c, K_OTHER); launch_text_embed(tw.ws.ids, tw.tok, tw.pos, nb, T, tw.hidden, tw.n_vocab, tw.ws.x, c->stream); }
        }
        auto emit = [&](int j) {
            char* dst = bases[j] + i0 * item_bytes(qs[j], tw, T);
            return a.host ? ring.put(tw, nb, T, qs[j], dst) : token_rows_tail(c, tw, nb, T, qs[j], dst);
        };
        if (!token_stops(c, tw, nb, T, !a.vision, qs, emit)) return false;
    }
    if (a.host && !ring.close()) return false;
    CK(cudaEventRecord(c->ev_t1, c->stream));
    return sync_and_time(c) && ring.drain_all();
}

// Every tokens form: the arguments checked in one order, the first fault refused (include/clip_b200.h), then the pass; devices mode
// shards the host forms' items over the GPUs, each writing its items into every slab.
static bool tokens_call(const clip_ctx* cctx, TokensCall a) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    const std::string who = a.who;
    if (!c) { set_err(who + ": null context"); return false; }
    const Tower& tw = a.vision ? c->vis : c->txt;
    if (!tw.present) { set_err(who + ": this model has no " + (a.vision ? "vision" : "text") + " encoder"); return false; }
    if (a.hw && !a.host && !check_hw_size(c, a.H, a.W, a.who)) return false;
    if (a.list && (a.n_layers < 1 || a.n_layers > CLIP_B200_TOKENS_MAX_LAYERS)) {
        set_err(who + ": n_layers must be in [1, " + std::to_string(CLIP_B200_TOKENS_MAX_LAYERS) + "], not " + std::to_string(a.n_layers));
        return false;
    }
    if (!a.layers) { set_err(who + ": null layers"); return false; }
    std::vector<TokenReq> qs((size_t)a.n_layers);
    for (int j = 0; j < a.n_layers; j++) {
        const std::string w = a.list ? who + ": entry " + std::to_string(j) : who;
        if (!token_request(c, a.vision, a.layers[j], a.flags ? a.flags[j] : 0, a.out_type, qs[j], w.c_str())) return false;
    }
    if (a.imgs) a.n = a.imgs->size;
    if (a.n == 0) return true;
    if (!a.vision && (a.seq_len < 1 || a.seq_len > tw.n_ctx)) { set_err(who + ": seq_len must be in [1, context_length]"); return false; }
    if (!a.out || (!a.in && !a.imgs)) {
        set_err(who + (!a.host ? ": null device pointer" : a.vision ? ": null output" : ": null pointer"));
        return false;
    }
    if (a.imgs && !a.hw && !check_images(c, a.imgs->data, a.n, a.who)) return false;
    if (a.imgs && a.hw && !check_images_hw(c, a.imgs->data, a.n, a.H, a.W, a.who)) return false;
    if (a.host && c->replicas.size() > 1 && a.n >= c->replicas.size())
        return for_each_replica(c, a.n, [&](clip_ctx* r, int, size_t lo, size_t hi) { return hi == lo || tokens_pass(r, a, qs, lo, hi); });
    return tokens_pass(c, a, qs, 0, a.n);
}

bool clip_b200_image_tokens(const struct clip_ctx* cctx, const struct clip_image_f32_batch* imgs, int layer, int flags, int out_type, void* out) {
    TokensCall a{"clip_b200_image_tokens", true, true};
    a.imgs = imgs;
    a.layers = &layer; a.flags = &flags; a.out_type = out_type; a.out = out;
    return tokens_call(cctx, a);
}

bool clip_b200_image_tokens_device(const struct clip_ctx* cctx, const void* d_pixels, size_t n, int layer, int flags, int out_type, void* d_out) {
    TokensCall a{"clip_b200_image_tokens_device", true, false};
    a.in = d_pixels; a.n = n;
    a.layers = &layer; a.flags = &flags; a.out_type = out_type; a.out = d_out;
    return tokens_call(cctx, a);
}

bool clip_b200_image_tokens_hw(const struct clip_ctx* cctx, const struct clip_image_f32_batch* imgs, int layer, int flags, int out_type, void* out) {
    TokensCall a{"clip_b200_image_tokens_hw", true, true, true};
    a.imgs = imgs;
    a.layers = &layer; a.flags = &flags; a.out_type = out_type; a.out = out;
    return tokens_call(cctx, a);
}

bool clip_b200_image_tokens_device_hw(const struct clip_ctx* cctx, const void* d_pixels, size_t n, int height, int width, int layer, int flags,
                                      int out_type, void* d_out) {
    TokensCall a{"clip_b200_image_tokens_device_hw", true, false, true};
    a.in = d_pixels; a.n = n; a.H = height; a.W = width;
    a.layers = &layer; a.flags = &flags; a.out_type = out_type; a.out = d_out;
    return tokens_call(cctx, a);
}

bool clip_b200_text_tokens(const struct clip_ctx* cctx, const int32_t* ids, size_t n, int seq_len, int layer, int flags, int out_type, void* out) {
    TokensCall a{"clip_b200_text_tokens", false, true};
    a.in = ids; a.n = n; a.seq_len = seq_len;
    a.layers = &layer; a.flags = &flags; a.out_type = out_type; a.out = out;
    return tokens_call(cctx, a);
}

bool clip_b200_text_tokens_device(const struct clip_ctx* cctx, const void* d_ids, size_t n, int seq_len, int layer, int flags, int out_type,
                                  void* d_out) {
    TokensCall a{"clip_b200_text_tokens_device", false, false};
    a.in = d_ids; a.n = n; a.seq_len = seq_len;
    a.layers = &layer; a.flags = &flags; a.out_type = out_type; a.out = d_out;
    return tokens_call(cctx, a);
}

// ---- images of different sizes in one call: the four clip_b200_*_mixed forms ----------------------------------------------------
// What one mixed call reads, as its public form received it.
struct MixedCall {
    const char* who;                              // the public name, for messages
    bool tokens, host;                            // per-token rows (else pooled); host images and output (else device)
    const clip_image_f32_batch* imgs = nullptr;   // host: the images, each of its own ny x nx
    const void* in = nullptr;                     // device: the NHWC f32 images back to back
    const int *heights = nullptr, *widths = nullptr;
    size_t n = 0;
    int layer = 0, flags = 0, out_type = 0;       // tokens
    void* out = nullptr;                          // tokens: the ragged rows (host or device)
    float* vec = nullptr;                         // pooled, host
    float* d_vec = nullptr;                       // pooled, device
    bool normalize = true;
    int H(size_t i) const { return host ? imgs->data[i].ny : heights[i]; }
    int W(size_t i) const { return host ? imgs->data[i].nx : widths[i]; }
};

// check_hw_size for image i of a mixed call: the message names the image
static bool check_mixed_size(const clip_ctx* c, size_t i, int H, int W, const char* who) {
    const std::string w = std::string(who) + ": image " + std::to_string(i);
    return check_hw_size(c, H, W, w.c_str());
}

// Rows of entry q for the images of a packed pass (T[i] rows each, `rows` in all) -> dst, item-major and ragged.  Without NO_CLS the
// packed rows are already that layout, so the tail is token_rows_tail's on one item of `rows` rows.  With NO_CLS, K7 runs once per
// image on that image's rows (after the same LN / projection / l2norm over all rows with PROJECT), as it runs on an image alone.
static bool mixed_rows_tail(clip_ctx* c, Tower& tw, const std::vector<int>& T, int rows, const TokenReq& q, char* dst) {
    if (!q.skip) return token_rows_tail(c, tw, 1, rows, q, dst);
    Workspace& w = tw.ws;
    const int h = tw.hidden, bf = c->operand_bf16 ? 1 : 0;
    const float* src = w.x;
    int width = h;
    const float* gamma = (q.flags & CLIP_B200_TOKENS_POST_LN) ? tw.post_g : nullptr;
    if (q.flags & CLIP_B200_TOKENS_PROJECT) {
        float* p32 = reinterpret_cast<float*>(w.qkv);     // as token_rows_tail lays them out
        float* n32 = reinterpret_cast<float*>(w.g);
        { Scope s(c, K_LN); launch_layernorm(w.x, h, rows, h, tw.eps, tw.post_g, tw.post_b, nullptr, w.a, bf, c->stream); }
        if (!run_linear(c, tw.proj_w, &w.map_a, w.a, bf, rows, p32, tw.proj, EPI_STORE32, 0)) return false;
        if (q.flags & CLIP_B200_TOKENS_NORMALIZE) { Scope s(c, K_OTHER); launch_l2norm(p32, n32, rows, tw.proj, 1, c->stream); p32 = n32; }
        src = p32; width = tw.proj; gamma = nullptr;
    }
    Scope s(c, K_TOKEN_ROWS);
    size_t r0 = 0;
    for (int t : T) {
        launch_token_rows(src + r0 * width, width, 1, t, 1, width, gamma, tw.post_b, tw.eps, q.out_type, dst, c->stream);
        r0 += (size_t)t;
        dst += (size_t)(t - 1) * width * q.esize;
    }
    CK(cudaGetLastError());
    return true;
}

// One GPU, images lo .. hi of a checked mixed call.  Position tables for every grid first, then passes of the longest prefix of the
// remaining images that fits every workspace buffer, each one forward pass over its rows packed back to back.
static bool mixed_pass(clip_ctx* c, const MixedCall& a, const TokenReq& q, size_t lo, size_t hi) {
    Tower& tw = c->vis;
    Workspace& w = tw.ws;
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (!ensure_ws(c, tw, tw.micro_batch, tw.T, true)) return false;
    const int P = tw.patch, h = tw.hidden, g = tw.image_size / P;
    const size_t n = hi - lo;
    std::vector<int> T(n);
    for (size_t i = 0; i < n; i++) {
        const int H = a.H(lo + i), W = a.W(lo + i);
        T[i] = (H / P) * (W / P) + 1;
        if (T[i] > w.cap_rows || (size_t)(T[i] - 1) > (size_t)w.cap_items * tw.n_patches) {
            set_err(std::string(a.who) + ": image " + std::to_string(lo + i) + ": one " + std::to_string(H) + " x " + std::to_string(W) +
                    " image needs " + std::to_string(T[i]) + " rows, more than the workspace holds (" + std::to_string(w.cap_rows) +
                    "); raise clip_b200_set_micro_batch before the first encode");
            return false;
        }
    }
    // one position table per grid: the loaded one at the model's own grid, the others resampled (K8) into one arena
    std::map<std::pair<int, int>, size_t> table;
    size_t floats = 0;
    for (size_t i = 0; i < n; i++) {
        const std::pair<int, int> gg(a.H(lo + i) / P, a.W(lo + i) / P);
        if (gg != std::make_pair(g, g) && !table.count(gg)) { table[gg] = floats; floats += (size_t)T[i] * h; }
    }
    if (floats && !ensure_buf(c, &c->pos_mixed, &c->pos_mixed_cap, floats)) return false;
    for (const auto& e : table) {
        float* dst = c->pos_mixed + e.second;
        CK(cudaMemcpyAsync(dst, tw.pos, (size_t)h * 4, cudaMemcpyDeviceToDevice, c->stream));     // the CLS row as it is
        { Scope s(c, K_POS_RESAMPLE); launch_pos_resample(tw.pos + h, g, h, e.first.first, e.first.second, dst + h, c->stream); }
    }
    CK(cudaGetLastError());
    // passes: total rows <= cap_rows, patch rows (one fewer per image) <= cap_items * n_patches, images <= cap_items (plan_call's limits)
    const std::vector<size_t> bounds = pack_passes(T, [&](size_t rows, size_t k, int t) {
        return rows + t <= (size_t)w.cap_rows && rows - k + t - 1 <= (size_t)w.cap_items * tw.n_patches && k + 1 <= (size_t)w.cap_items;
    });
    size_t most = 0;
    for (size_t b = 0; b + 1 < bounds.size(); b++) most = std::max(most, bounds[b + 1] - bounds[b]);
    const size_t desc_bytes = (most * sizeof(MixedImage) + 2 * (most + 1) * sizeof(int) + 255) / 256 * 256;
    if (!ensure_buf(c, &c->d_mixed, &c->d_mixed_cap, desc_bytes)) return false;
    // where image lo + i starts: its pixels (floats from the call's first image) and its output (bytes from the call's out)
    std::vector<size_t> px0(n + 1, 0), out0(n + 1, 0);
    size_t px_lo = 0, out_lo = 0;
    for (size_t i = 0; i < lo; i++) {
        px_lo += (size_t)a.H(i) * a.W(i) * 3;
        out_lo += (size_t)((a.H(i) / P) * (a.W(i) / P) + 1 - q.skip) * q.width * q.esize;
    }
    px0[0] = px_lo; out0[0] = out_lo;
    for (size_t i = 0; i < n; i++) {
        px0[i + 1] = px0[i] + (size_t)a.H(lo + i) * a.W(lo + i) * 3;
        out0[i + 1] = out0[i] + (size_t)(T[i] - q.skip) * q.width * q.esize;
    }
    float* d_vec = a.d_vec;
    if (!a.tokens && !d_vec) {
        if (!ensure_out(c, n * tw.proj)) return false;
        d_vec = c->d_out;
    }
    char* stage = nullptr;     // host tokens: one pass's rows on the device, then copied out
    if (a.tokens && a.host) {
        size_t widest = 0;
        for (size_t b = 0; b + 1 < bounds.size(); b++) widest = std::max(widest, out0[bounds[b + 1]] - out0[bounds[b]]);
        if (!ensure_buf(c, &c->d_ring, &c->d_ring_cap, widest)) return false;
        stage = c->d_ring;
    }
    std::vector<char> blob(desc_bytes);
    CK(cudaEventRecord(c->ev_t0, c->stream));
    for (size_t b = 0; b + 1 < bounds.size(); b++) {
        const size_t i0 = bounds[b], i1 = bounds[b + 1];
        const int nb = (int)(i1 - i0);
        MixedImage* im = reinterpret_cast<MixedImage*>(blob.data());
        int* off = reinterpret_cast<int*>(blob.data() + nb * sizeof(MixedImage));
        const int* grp = off + nb + 1;
        const int rows = varlen_table(T, i0, i1, off), prows = rows - nb;
        for (int j = 0; j < nb; j++) {
            const size_t i = i0 + j;
            const int gh = a.H(lo + i) / P, gw = a.W(lo + i) / P;
            const auto it = table.find(std::make_pair(gh, gw));
            im[j].px = (long long)(px0[i] - px0[i0]);
            im[j].pos = it == table.end() ? tw.pos : c->pos_mixed + it->second;
            im[j].row = off[j]; im[j].prow = off[j] - j; im[j].gh = gh; im[j].gw = gw;
        }
        const MixedImage* d_im = reinterpret_cast<const MixedImage*>(c->d_mixed);
        const int* d_seq = reinterpret_cast<const int*>(c->d_mixed + nb * sizeof(MixedImage));
        CK(cudaMemcpyAsync(c->d_mixed, blob.data(), nb * sizeof(MixedImage) + 2 * (nb + 1) * sizeof(int), cudaMemcpyHostToDevice, c->stream));
        const float* px;
        if (a.host) {
            for (int j = 0; j < nb; j++)
                CK(cudaMemcpyAsync(w.pixels[0] + im[j].px, a.imgs->data[lo + i0 + j].data, (px0[i0 + j + 1] - px0[i0 + j]) * 4, cudaMemcpyHostToDevice, c->stream));
            px = w.pixels[0];
        } else {
            px = (const float*)a.in + px0[i0];
        }
        { Scope s(c, K_OTHER); launch_im2col_mixed(px, d_im, nb, prows, P, tw.kpad, w.patches, c->stream); }
        if (!run_linear(c, tw.patch_w, &w.map_patches, w.patches, false, prows, w.patch32, h, EPI_STORE32, 0)) return false;
        { Scope s(c, K_OTHER); launch_assemble_mixed(w.patch32, tw.class_embd, d_im, nb, rows, h, tw.eps, tw.pre_g, tw.pre_b, w.x, c->stream); }
        const Packed pk{rows, nb, grp[nb], d_seq};
        if (a.tokens) {
            if (!run_blocks(c, tw, nb, 0, false, 0, q.blocks, &pk)) return false;
            char* dst = a.host ? stage : (char*)a.out + out0[i0];
            if (!mixed_rows_tail(c, tw, std::vector<int>(T.begin() + i0, T.begin() + i1), rows, q, dst)) return false;
            if (a.host) CK(cudaMemcpyAsync((char*)a.out + out0[i0], stage, out0[i1] - out0[i0], cudaMemcpyDeviceToHost, c->stream));
        } else {
            if (!run_blocks(c, tw, nb, 0, false, 0, tw.layers, &pk)) return false;
            // the CLS rows (off[j]); a pass holds at most cap_items images, so this is one chunk
            if (!pooled_rows_tail(c, tw, nb, d_seq, d_vec + i0 * tw.proj, a.normalize)) return false;
        }
    }
    CK(cudaEventRecord(c->ev_t1, c->stream));
    if (!a.tokens && a.vec) CK(cudaMemcpyAsync(a.vec + lo * tw.proj, d_vec, n * tw.proj * 4, cudaMemcpyDeviceToHost, c->stream));
    return sync_and_time(c);
}

// Every mixed form: the arguments checked in one order, the first fault refused (include/clip_b200.h), then the passes; devices mode
// shards the host forms' images over the GPUs as clip_image_batch_encode does.
static bool mixed_call(const clip_ctx* cctx, MixedCall a) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    const std::string who = a.who;
    if (!c) { set_err(who + ": null context"); return false; }
    if (!c->vis.present) { set_err(who + ": this model has no vision encoder"); return false; }
    if (!a.host && a.heights && a.widths)
        for (size_t i = 0; i < a.n; i++)
            if (!check_mixed_size(c, i, a.heights[i], a.widths[i], a.who)) return false;
    if (a.host) a.n = a.imgs ? a.imgs->size : 0;     // a NULL batch is an empty one
    if (a.n == 0) return true;
    if (a.host) {
        if (!a.imgs->data) { set_err(who + ": null input"); return false; }
        if (!(a.tokens ? a.out : a.vec)) { set_err(who + ": null output"); return false; }
        for (size_t i = 0; i < a.n; i++) {
            if (!a.imgs->data[i].data) { set_err(who + ": image " + std::to_string(i) + " has no pixels"); return false; }
            if (!check_mixed_size(c, i, a.imgs->data[i].ny, a.imgs->data[i].nx, a.who)) return false;
        }
    } else {
        if (!a.in || !(a.tokens ? a.out : a.d_vec)) { set_err(who + ": null device pointer"); return false; }
        if (!a.heights || !a.widths) { set_err(who + ": null heights or widths"); return false; }
    }
    TokenReq q;
    if (a.tokens) {
        if (!token_request(c, true, a.layer, a.flags, a.out_type, q, a.who)) return false;
        if (q.attn) { set_err(who + ": CLIP_B200_TOKENS_ATTENTION is not supported at mixed sizes"); return false; }
    }
    if (a.host && c->replicas.size() > 1 && a.n >= c->replicas.size())
        return for_each_replica(c, a.n, [&](clip_ctx* r, int, size_t lo, size_t hi) { return hi == lo || mixed_pass(r, a, q, lo, hi); });
    return mixed_pass(c, a, q, 0, a.n);
}

bool clip_b200_image_batch_encode_mixed(const struct clip_ctx* cctx, const struct clip_image_f32_batch* imgs, float* vec, bool normalize) {
    MixedCall a{"clip_b200_image_batch_encode_mixed", false, true};
    a.imgs = imgs; a.vec = vec; a.normalize = normalize;
    return mixed_call(cctx, a);
}

bool clip_b200_image_encode_device_mixed(const struct clip_ctx* cctx, const void* d_pixels, size_t n, const int* heights, const int* widths,
                                         void* d_vec, bool normalize) {
    MixedCall a{"clip_b200_image_encode_device_mixed", false, false};
    a.in = d_pixels; a.n = n; a.heights = heights; a.widths = widths; a.d_vec = (float*)d_vec; a.normalize = normalize;
    return mixed_call(cctx, a);
}

bool clip_b200_image_tokens_mixed(const struct clip_ctx* cctx, const struct clip_image_f32_batch* imgs, int layer, int flags, int out_type,
                                  void* out) {
    MixedCall a{"clip_b200_image_tokens_mixed", true, true};
    a.imgs = imgs; a.layer = layer; a.flags = flags; a.out_type = out_type; a.out = out;
    return mixed_call(cctx, a);
}

bool clip_b200_image_tokens_device_mixed(const struct clip_ctx* cctx, const void* d_pixels, size_t n, const int* heights, const int* widths,
                                         int layer, int flags, int out_type, void* d_out) {
    MixedCall a{"clip_b200_image_tokens_device_mixed", true, false};
    a.in = d_pixels; a.n = n; a.heights = heights; a.widths = widths; a.layer = layer; a.flags = flags; a.out_type = out_type; a.out = d_out;
    return mixed_call(cctx, a);
}

// ---- token sequences of different lengths in one call: the four clip_b200_text_*_packed forms ----------------------------------
// What one packed text call reads, as its public form received it.
struct PackedTextCall {
    const char* who;                              // the public name, for messages
    bool tokens, host;                            // per-token rows (else pooled); host ids and output (else device)
    const clip_tokens* seqs = nullptr;            // host pooled: the sequences
    const int32_t* ids = nullptr;                 // the other forms: the sequences back to back (host or device)
    const int* lens = nullptr;                    // with ids: host, n entries
    size_t n = 0;
    int layer = 0, flags = 0, out_type = 0;       // tokens
    void* out = nullptr;                          // tokens: the ragged rows (host or device)
    float* vec = nullptr;                         // pooled, host
    float* d_vec = nullptr;                       // pooled, device
    bool normalize = true;
    int len(size_t i) const { return seqs ? (int)seqs[i].size : lens[i]; }
};

// One GPU, sequences lo .. hi of a checked packed call: passes of the longest prefix of the remaining sequences whose rows fit the
// workspace (micro_batch x context_length rows), each one forward pass over its rows packed back to back.  Per pass, one upload of
// K3's varlen table (whose off[] also places each row's position) and the EOT rows, the ids (read in place on the device, staged
// into ws.ids from the host), one embedding, the blocks, then the tail.  Only the staging, the embedding and the pooled rows differ
// from mixed_pass; the planner, the table, the blocks and the tails are the ones it runs.
static bool text_packed_pass(clip_ctx* c, const PackedTextCall& a, const TokenReq& q, size_t lo, size_t hi) {
    Tower& tw = c->txt;
    Workspace& w = tw.ws;
    const size_t n = hi - lo;
    std::vector<int> T(n);
    std::vector<size_t> id0(n + 1, 0), out0(n + 1, 0);     // sequence lo + i's first id and first output byte, from sequence lo's
    for (size_t i = 0; i < n; i++) {
        T[i] = a.len(lo + i);
        id0[i + 1] = id0[i] + (size_t)T[i];
        out0[i + 1] = out0[i] + (size_t)T[i] * q.width * q.esize;
    }
    size_t id_lo = 0;
    for (size_t i = 0; i < lo; i++) id_lo += (size_t)a.len(i);
    // host sequences: gathered into one pageable array, so that a pass's ids go up in one copy
    std::vector<int32_t> gathered;
    if (a.seqs) {
        gathered.resize(id0[n]);
        for (size_t i = 0; i < n; i++) memcpy(gathered.data() + id0[i], a.seqs[lo + i].data, (size_t)T[i] * 4);
    }
    const int32_t* ids = a.seqs ? gathered.data() : a.ids + id_lo;
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (!ensure_ws(c, tw, tw.micro_batch, tw.n_ctx, false)) return false;
    // every sequence fits a pass alone: its length is at most context_length
    const std::vector<size_t> bounds = pack_passes(T, [&](size_t rows, size_t, int t) { return rows + t <= (size_t)w.cap_rows; });
    size_t most = 0;
    for (size_t b = 0; b + 1 < bounds.size(); b++) most = std::max(most, bounds[b + 1] - bounds[b]);
    // one pass's descriptors: K3's varlen table [2 (nb + 1)], then the EOT rows [nb]
    std::vector<int> blob(3 * most + 2);
    if (!ensure_buf(c, &c->d_mixed, &c->d_mixed_cap, blob.size() * sizeof(int))) return false;
    float* d_vec = a.d_vec;
    if (!a.tokens && !d_vec) {
        if (!ensure_out(c, n * tw.proj)) return false;
        d_vec = c->d_out;
    }
    char* stage = nullptr;     // host tokens: one pass's rows on the device, then copied out
    if (a.tokens && a.host) {
        size_t widest = 0;
        for (size_t b = 0; b + 1 < bounds.size(); b++) widest = std::max(widest, out0[bounds[b + 1]] - out0[bounds[b]]);
        if (!ensure_buf(c, &c->d_ring, &c->d_ring_cap, widest)) return false;
        stage = c->d_ring;
    }
    const size_t out_lo = id_lo * q.width * q.esize;
    CK(cudaEventRecord(c->ev_t0, c->stream));
    for (size_t b = 0; b + 1 < bounds.size(); b++) {
        const size_t i0 = bounds[b], i1 = bounds[b + 1];
        const int nb = (int)(i1 - i0);
        int* off = blob.data();
        const int rows = varlen_table(T, i0, i1, off);
        int* eot = off + 2 * (nb + 1);
        for (int j = 0; j < nb; j++) eot[j] = off[j + 1] - 1;     // the reference selects row N-1 (clip.cpp:1154-1155)
        const int* d_seq = reinterpret_cast<const int*>(c->d_mixed);
        CK(cudaMemcpyAsync(c->d_mixed, blob.data(), (size_t)(3 * nb + 2) * sizeof(int), cudaMemcpyHostToDevice, c->stream));
        const int32_t* d_ids = ids + id0[i0];
        if (a.host) {
            CK(cudaMemcpyAsync(w.ids, d_ids, (size_t)rows * 4, cudaMemcpyHostToDevice, c->stream));
            d_ids = w.ids;
        }
        { Scope s(c, K_OTHER); launch_text_embed_packed(d_ids, tw.tok, tw.pos, d_seq, nb, rows, tw.hidden, tw.n_vocab, w.x, c->stream); }
        const Packed pk{rows, nb, off[2 * nb + 1], d_seq, true};
        if (!run_blocks(c, tw, nb, 0, true, 0, a.tokens ? q.blocks : tw.layers, &pk)) return false;
        if (a.tokens) {
            // text has no NO_CLS: the packed rows are already the ragged item-major layout
            char* dst = a.host ? stage : (char*)a.out + out_lo + out0[i0];
            if (!token_rows_tail(c, tw, 1, rows, q, dst)) return false;
            if (a.host) CK(cudaMemcpyAsync((char*)a.out + out_lo + out0[i0], stage, out0[i1] - out0[i0], cudaMemcpyDeviceToHost, c->stream));
        } else if (!pooled_rows_tail(c, tw, nb, d_seq + 2 * (nb + 1), d_vec + i0 * tw.proj, a.normalize)) {
            return false;
        }
    }
    CK(cudaEventRecord(c->ev_t1, c->stream));
    if (!a.tokens && a.vec) CK(cudaMemcpyAsync(a.vec + lo * tw.proj, d_vec, n * tw.proj * 4, cudaMemcpyDeviceToHost, c->stream));
    return sync_and_time(c);
}

// Every packed text form: the arguments checked in one order, the first fault refused (include/clip_b200.h), then the passes;
// devices mode shards the host forms' sequences over the GPUs as clip_text_batch_encode does.
static bool text_packed_call(const clip_ctx* cctx, PackedTextCall a) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    const std::string who = a.who;
    if (!c) { set_err(who + ": null context"); return false; }
    const Tower& tw = c->txt;
    if (!tw.present) { set_err(who + ": this model has no text encoder"); return false; }
    if (tw.hidden != 64 * tw.heads) {
        set_err(who + ": packed sequences need a text tower of head_dim 64, not " + std::to_string(tw.hidden / tw.heads) + " (hidden " +
                std::to_string(tw.hidden) + ", heads " + std::to_string(tw.heads) + ")");
        return false;
    }
    if (a.n == 0) return true;
    if (!(a.seqs || a.ids)) { set_err(who + ": null input"); return false; }
    if (!a.seqs && !a.lens) { set_err(who + ": null lens"); return false; }
    if (!(a.tokens ? a.out : a.host ? (void*)a.vec : (void*)a.d_vec)) { set_err(who + ": null output"); return false; }
    for (size_t i = 0; i < a.n; i++) {
        if (a.seqs && !a.seqs[i].data) { set_err(who + ": sequence " + std::to_string(i) + " has no tokens"); return false; }
        const long long L = a.seqs ? (long long)std::min<size_t>(a.seqs[i].size, (size_t)INT_MAX) : (long long)a.lens[i];
        if (L < 1 || L > tw.n_ctx) {
            set_err(who + ": sequence " + std::to_string(i) + " has length " + std::to_string(L) + ", outside [1, context_length (" +
                    std::to_string(tw.n_ctx) + ")]");
            return false;
        }
    }
    TokenReq q;
    if (a.tokens) {
        if (!token_request(c, false, a.layer, a.flags, a.out_type, q, a.who)) return false;
        if (q.attn) { set_err(who + ": CLIP_B200_TOKENS_ATTENTION is not supported at packed lengths"); return false; }
    }
    if (a.host && c->replicas.size() > 1 && a.n >= TEXT_SHARD_MIN * c->replicas.size())
        return for_each_replica(c, a.n, [&](clip_ctx* r, int, size_t lo, size_t hi) { return hi == lo || text_packed_pass(r, a, q, lo, hi); });
    return text_packed_pass(c, a, q, 0, a.n);
}

bool clip_b200_text_batch_encode_packed(const struct clip_ctx* cctx, const struct clip_tokens* seqs, size_t n, float* vec, bool normalize) {
    PackedTextCall a{"clip_b200_text_batch_encode_packed", false, true};
    a.seqs = seqs; a.n = n; a.vec = vec; a.normalize = normalize;
    return text_packed_call(cctx, a);
}

bool clip_b200_text_encode_device_packed(const struct clip_ctx* cctx, const void* d_ids, size_t n, const int* lens, void* d_vec, bool normalize) {
    PackedTextCall a{"clip_b200_text_encode_device_packed", false, false};
    a.ids = (const int32_t*)d_ids; a.n = n; a.lens = lens; a.d_vec = (float*)d_vec; a.normalize = normalize;
    return text_packed_call(cctx, a);
}

bool clip_b200_text_tokens_packed(const struct clip_ctx* cctx, const int32_t* ids, size_t n, const int* lens, int layer, int flags, int out_type,
                                  void* out) {
    PackedTextCall a{"clip_b200_text_tokens_packed", true, true};
    a.ids = ids; a.n = n; a.lens = lens; a.layer = layer; a.flags = flags; a.out_type = out_type; a.out = out;
    return text_packed_call(cctx, a);
}

bool clip_b200_text_tokens_device_packed(const struct clip_ctx* cctx, const void* d_ids, size_t n, const int* lens, int layer, int flags,
                                         int out_type, void* d_out) {
    PackedTextCall a{"clip_b200_text_tokens_device_packed", true, false};
    a.ids = (const int32_t*)d_ids; a.n = n; a.lens = lens; a.layer = layer; a.flags = flags; a.out_type = out_type; a.out = d_out;
    return text_packed_call(cctx, a);
}

// ---- several layers from one forward pass (clip_b200_*_tokens_layers) ------------------------------------------------------------
bool clip_b200_image_tokens_layers(const struct clip_ctx* cctx, const struct clip_image_f32_batch* imgs, const int* layers, const int* flags,
                                   int n_layers, int out_type, void* out) {
    TokensCall a{"clip_b200_image_tokens_layers", true, true, true};
    a.imgs = imgs;
    a.layers = layers; a.flags = flags; a.n_layers = n_layers; a.list = true; a.out_type = out_type; a.out = out;
    return tokens_call(cctx, a);
}

bool clip_b200_image_tokens_layers_device(const struct clip_ctx* cctx, const void* d_pixels, size_t n, int height, int width, const int* layers,
                                          const int* flags, int n_layers, int out_type, void* d_out) {
    TokensCall a{"clip_b200_image_tokens_layers_device", true, false, true};
    a.in = d_pixels; a.n = n; a.H = height; a.W = width;
    a.layers = layers; a.flags = flags; a.n_layers = n_layers; a.list = true; a.out_type = out_type; a.out = d_out;
    return tokens_call(cctx, a);
}

bool clip_b200_text_tokens_layers(const struct clip_ctx* cctx, const int32_t* ids, size_t n, int seq_len, const int* layers, const int* flags,
                                  int n_layers, int out_type, void* out) {
    TokensCall a{"clip_b200_text_tokens_layers", false, true};
    a.in = ids; a.n = n; a.seq_len = seq_len;
    a.layers = layers; a.flags = flags; a.n_layers = n_layers; a.list = true; a.out_type = out_type; a.out = out;
    return tokens_call(cctx, a);
}

bool clip_b200_text_tokens_layers_device(const struct clip_ctx* cctx, const void* d_ids, size_t n, int seq_len, const int* layers, const int* flags,
                                         int n_layers, int out_type, void* d_out) {
    TokensCall a{"clip_b200_text_tokens_layers_device", false, false};
    a.in = d_ids; a.n = n; a.seq_len = seq_len;
    a.layers = layers; a.flags = flags; a.n_layers = n_layers; a.list = true; a.out_type = out_type; a.out = d_out;
    return tokens_call(cctx, a);
}

float clip_similarity_score(const float* vec1, const float* vec2, const int vec_dim) {
    float dot = 0.0f;
    for (int i = 0; i < vec_dim; i++) dot += vec1[i] * vec2[i];
    return dot;
}

bool softmax_with_sorting(float* arr, const int length, float* sorted_scores, int* indices) {
    if (length <= 0) return false;
    double sum = 0.0;
    for (int i = 0; i < length; i++) { arr[i] = (float)(exp(arr[i]) + 1e-9); sum += arr[i]; }
    std::vector<int> idx(length);
    for (int i = 0; i < length; i++) { arr[i] = (float)(arr[i] / sum); idx[i] = i; }
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return arr[a] > arr[b]; });
    for (int i = 0; i < length; i++) { sorted_scores[i] = arr[idx[i]]; indices[i] = idx[i]; }
    return true;
}

bool clip_compare_text_and_image(const struct clip_ctx* ctx, const int n_threads, const char* text, const struct clip_image_u8* image,
                                 float* score) {
    if (!ctx || !(ctx->has_text && ctx->has_vision)) { printf("clip_compare_text_and_image function can only be used with two-tower models\n"); return false; }
    const int d = ctx->vhp.projection_dim;
    std::vector<float> iv(d), tv(d);
    clip_tokens tk{nullptr, 0};
    if (!clip_tokenize(ctx, text, &tk)) return false;
    const bool ok_t = clip_text_encode(ctx, n_threads, &tk, tv.data(), true);
    delete[] tk.data;
    if (!ok_t) return false;
    clip_image_f32 res{0, 0, nullptr, 0};
    if (!clip_image_preprocess(ctx, image, &res)) return false;
    const bool ok_i = clip_image_encode(ctx, n_threads, &res, iv.data(), true);
    clip_image_f32_clean(&res);
    if (!ok_i) return false;
    *score = clip_similarity_score(iv.data(), tv.data(), d);
    return true;
}

bool clip_zero_shot_label_image(struct clip_ctx* ctx, const int n_threads, const struct clip_image_u8* input_img, const char** labels,
                                const size_t n_labels, float* scores, int* indices) {
    if (!ctx || !(ctx->has_text && ctx->has_vision)) { printf("clip_zero_shot_label_image function can only be used with two-tower models\n"); return false; }
    const int d = ctx->vhp.projection_dim;
    clip_image_f32 res{0, 0, nullptr, 0};
    if (!clip_image_preprocess(ctx, input_img, &res)) return false;
    std::vector<float> iv(d);
    const bool ok_i = clip_image_encode(ctx, n_threads, &res, iv.data(), false);
    clip_image_f32_clean(&res);
    if (!ok_i) return false;
    std::vector<clip_tokens> tks(n_labels);
    for (size_t i = 0; i < n_labels; i++) if (!clip_tokenize(ctx, labels[i], &tks[i])) return false;
    std::vector<float> tv(n_labels * d), sims(n_labels);
    const bool ok_t = clip_text_batch_encode(ctx, n_threads, tks.data(), n_labels, tv.data(), false);
    for (auto& t : tks) delete[] t.data;
    if (!ok_t) return false;
    for (size_t i = 0; i < n_labels; i++) sims[i] = clip_similarity_score(iv.data(), tv.data() + i * d, d);
    return softmax_with_sorting(sims.data(), (int)n_labels, scores, indices);
}

// =====================================================================================================================
// Scoring on the device (search.cu): similarity matrix -> [softmax_with_sorting arithmetic] -> top-k, results to the host
// =====================================================================================================================
// Merge stages over d_cand_v/i[0] [rows, cand_ld]: nsl sorted runs of kk candidates (value, index) compete again until one run of kk
// is left.  Returns the buffer (0 or 1) that holds each row's best kk, best first.
static int merge_candidates(clip_ctx* c, int rows, size_t cand_ld, size_t nsl, int kk) {
    const int SL = topk_slice();
    int cur = 0;
    size_t cur_n = cand_ld;
    while (cur_n > (size_t)SL || (cur_n > (size_t)kk && nsl > 1)) {      // merge stages: candidates of all slices compete again
        const size_t nslices = (cur_n + SL - 1) / SL;
        { Scope s(c, K_OTHER); launch_topk_stage(c->d_cand_v[cur], c->d_cand_i[cur], cand_ld, rows, (int)cur_n, 0, kk, c->d_cand_v[cur ^ 1], c->d_cand_i[cur ^ 1], cand_ld, 0, c->stream); }
        cur ^= 1;
        cur_n = nslices * (size_t)kk;
        if (nslices == 1) break;
    }
    return cur;
}

// grow the four candidate buffers to `count` entries each
static bool ensure_cand(clip_ctx* c, size_t count) {
    size_t cap0 = c->d_cand_cap, cap1 = c->d_cand_cap, cap2 = c->d_cand_cap, cap3 = c->d_cand_cap;
    if (!ensure_buf(c, &c->d_cand_v[0], &cap0, count) || !ensure_buf(c, &c->d_cand_v[1], &cap1, count) ||
        !ensure_buf(c, &c->d_cand_i[0], &cap2, count) || !ensure_buf(c, &c->d_cand_i[1], &cap3, count)) return false;
    c->d_cand_cap = std::min(std::min(cap0, cap1), std::min(cap2, cap3));
    return true;
}

// What one call of the search family reads, as its public form received it: the five searches, the rescore and the three row forms
// that make their databases.  Each form fills one and calls search_call, so every form checks its arguments in the same order
// (include/clip_b200.h), and the searches run the same pass driver.
struct SearchCall {
    enum Kind { SCORE, KNN16, KNN_I8, KNN_B1, RESCORE, ROWS16, ROWS_I8, ROWS_B1, IVF_TRAIN, IVF_BUILD, IVF_SEARCH, PQ_TRAIN, PQ_ENCODE,
                PQ_BUILD, PQ_SEARCH };
    const char* who;                              // the public name, for messages
    Kind kind;
    const void* q = nullptr;                      // queries [nq, dim]; a row form: its f32 source rows [nq, dim]
    const void* db = nullptr;                     // database rows [ndb, dim]; a row form: the rows it writes [nq, dim]
    const void* xs = nullptr;                     // KNN_I8: database row scales [ndb]; ROWS_I8: the scales it writes [nq];
                                                  // ROWS_B1: the centre [dim] or NULL
    const void* qs = nullptr;                     // KNN_I8: query scales [nq]
    size_t nq = 0, ndb = 0;                       // a row form: nq = n
    int dim = 0;                                  // SCORE: the model's projection_dim, set by search_call
    int type = 0;                                 // KNN16, RESCORE: in_type; ROWS16: out_type
    const int* cand = nullptr;                    // RESCORE: host candidates [nq, n_cand]
    int n_cand = 0;
    int top_k = 0;                                // SCORE: <= 0 or > ndb means all ndb; KNN: [1, 1024], > ndb means ndb;
                                                  // RESCORE: [1, n_cand], padded past the valid candidates
    bool softmax = false;                         // SCORE: rank p = (exp(s) + 1e-9) / sum over the row instead of s
    float* scores = nullptr;                      // host outputs [nq, that top_k]
    int* indices = nullptr;
    // IVF_*: q holds the training rows, the database rows or the queries, nq their count; db is the list-ordered rows [ndb, dim]
    // (IVF_BUILD writes them, with ndb = nq)
    const void* cent = nullptr;                   // centroids [n_lists, dim] (IVF_TRAIN writes them)
    int* offsets = nullptr;                       // [n_lists + 1] and [ndb]: IVF_BUILD writes them, IVF_SEARCH reads them
    int* ids = nullptr;
    int n_lists = 0;
    int iters = 0;                                // IVF_TRAIN: n_iter; IVF_SEARCH: nprobe
    // PQ_*: q holds the training rows, the rows to encode, the codes to lay out (PQ_BUILD) or the queries; db the codes that PQ_ENCODE
    // and PQ_BUILD write and PQ_SEARCH reads; cent, offsets, ids, n_lists and iters as IVF_*
    const void* books = nullptr;                  // codebooks f32 [m, 256, dim / m] (PQ_TRAIN writes them)
    int m = 0;                                    // subspaces
    int* lists = nullptr;                         // [nq]: PQ_ENCODE writes them, PQ_BUILD reads them
    bool ivf() const { return kind >= IVF_TRAIN && kind <= IVF_SEARCH; }
    bool pq() const { return kind >= PQ_TRAIN; }
    bool search() const { return kind <= RESCORE; }
    bool knn() const { return kind == KNN16 || kind == KNN_I8 || kind == KNN_B1; }
};

// The pass driver of the searches and the rescore, for a checked call with nq, ndb > 0.  Per block of QB queries: the candidates into
// d_cand_v/i[0] [rows, cand_ld] as `runs` sorted runs of kk, merge_candidates, the best k per row to the host, a synchronise.  Only
// making the candidates differs: SCORE runs column chunks of CH rows through similarity [, softmax_with_sorting's p, clip.cpp:1591-1622]
// and a top-k stage (a ranking above 1024 over more than one slice is made on the host instead); K10 and K11 are one launch per 32768
// queries, the merge grid's row limit; K12 is one launch per block of queries whose candidates (copied from the host) fit 2^22 ints,
// writing one sorted run of top_k.  Caller holds c->mu and has set the device.
static bool search_locked(clip_ctx* c, const SearchCall& a) {
    const size_t nq = a.nq, ndb = a.ndb;
    const bool rescore = a.kind == SearchCall::RESCORE;
    const int k = rescore ? a.top_k : a.top_k <= 0 || (size_t)a.top_k > ndb ? (int)ndb : a.top_k;
    const int SL = topk_slice(), kk = std::min(k, SL);
    const bool knn = a.knn(), i8 = a.kind == SearchCall::KNN_I8, b1 = a.kind == SearchCall::KNN_B1;
    size_t QB = 32768, CH = ndb, nsl = 0;
    bool device_select = true;
    int sms = 0;
    if (knn) {
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    } else if (rescore) {
        QB = std::min<size_t>(32768, ((size_t)1 << 22) / a.n_cand);
        if (!ensure_buf(c, &c->d_rcand, &c->d_rcand_cap, std::min(QB, nq) * a.n_cand) || !ensure_cand(c, std::min(QB, nq) * k)) return false;
    } else {
        const size_t budget = (size_t)32 << 20;                           // floats of similarity scratch per pass (128 MB)
        CH = std::min(ndb, std::max<size_t>(budget / std::min<size_t>(nq, 256), (size_t)SL));
        // whole rows: the normalisation needs them, and so does the host ranking taken when top_k > 1024 (a ranking per chunk would
        // keep only the last chunk's best, numbered within that chunk)
        if (a.softmax || k > 1024) CH = ndb;
        QB = std::max<size_t>(1, std::min<size_t>({nq, budget / CH + 1, (size_t)32768}));
        for (size_t c0 = 0; c0 < ndb; c0 += CH) nsl += (std::min(CH, ndb - c0) + SL - 1) / SL;
        device_select = nsl == 1 || k <= 1024;                            // each stage must shrink the candidate set
        if (!ensure_buf(c, &c->d_logits, &c->d_logits_cap, QB * CH)) return false;
        if (device_select && !ensure_cand(c, QB * nsl * kk)) return false;
    }
    std::vector<float> hrow;
    std::vector<int> hidx;
    for (size_t r0 = 0; r0 < nq; r0 += QB) {
        const int rows = (int)std::min(QB, nq - r0);
        size_t runs = nsl, cand_ld = nsl * kk;
        if (rescore) {
            runs = 1;
            cand_ld = k;
            CK(cudaMemcpyAsync(c->d_rcand, a.cand + r0 * a.n_cand, (size_t)rows * a.n_cand * 4, cudaMemcpyHostToDevice, c->stream));
            const size_t q_row = (size_t)a.dim * (a.type == CLIP_B200_OUT_F32 ? 4 : 2);
            Scope s(c, K_RESCORE);
            const cudaError_t e = launch_rescore(a.type, (const uint8_t*)a.q + r0 * q_row, rows, a.db, (int)ndb, a.dim, c->d_rcand, a.n_cand, k,
                                                 c->d_cand_v[0], c->d_cand_i[0], cand_ld, c->stream);
            if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        } else if (b1) {
            const KnnPlan pl = knn_b1_plan(rows, (int)ndb, k, sms);
            runs = pl.parts;
            cand_ld = (size_t)pl.parts * k;
            if (!ensure_buf(c, &c->d_knn, &c->d_knn_cap, 2 * pl.buf_entries) || !ensure_cand(c, (size_t)rows * cand_ld)) return false;
            Scope s(c, K_KNN_B1);
            const cudaError_t e = launch_knn_b1((const uint8_t*)a.q + r0 * (a.dim / 8), rows, a.db, (int)ndb, a.dim, k, pl, c->d_knn,
                                                c->d_cand_v[0], c->d_cand_i[0], cand_ld, c->stream);
            if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        } else if (knn) {
            const KnnPlan pl = knn_plan(rows, (int)ndb, k, sms);
            runs = pl.parts;
            cand_ld = (size_t)pl.parts * k;
            if (!ensure_buf(c, &c->d_knn, &c->d_knn_cap, 2 * pl.buf_entries) || !ensure_cand(c, (size_t)rows * cand_ld)) return false;
            const KOp op = i8 ? KOp::S8 : a.type == CLIP_B200_OUT_BF16 ? KOp::BF16 : KOp::F16;
            const size_t q_row = i8 ? a.dim : 2 * (size_t)a.dim;               // bytes per query row
            Scope s(c, i8 ? K_KNN_I8 : K_KNN16);
            const cudaError_t e = launch_knn(op, (const uint8_t*)a.q + r0 * q_row, i8 ? (const float*)a.qs + r0 : nullptr, rows, a.db,
                                             (const float*)a.xs, (int)ndb, a.dim, k, pl, c->d_knn, c->d_cand_v[0], c->d_cand_i[0], cand_ld,
                                             c->stream);
            if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        } else {
            const float* q = (const float*)a.q + r0 * a.dim;
            size_t sl0 = 0;
            for (size_t c0 = 0; c0 < ndb; c0 += CH) {
                const int cols = (int)std::min(CH, ndb - c0);
                { Scope s(c, K_OTHER); launch_similarity(q, (const float*)a.db + c0 * a.dim, c->d_logits, rows, cols, a.dim, CH, c->stream); }
                if (a.softmax) { Scope s(c, K_OTHER); launch_softmax_ref(c->d_logits, rows, cols, CH, c->stream); }
                if (device_select) {
                    Scope s(c, K_OTHER);
                    launch_topk_stage(c->d_logits, nullptr, CH, rows, cols, (int)c0, kk, c->d_cand_v[0], c->d_cand_i[0], cand_ld, (int)(sl0 * kk), c->stream);
                    sl0 += ((size_t)cols + SL - 1) / SL;
                } else {
                    // full ranking of rows longer than one sort slice (top_k > 1024): ranked on the host, as the reference does.  cols
                    // is the whole row (CH = ndb above) and k <= ndb.  NaN becomes -FLT_MAX as in topk_stage_kernel: it ranks last, ties
                    // by index, and the comparator stays a strict weak order.
                    hrow.resize((size_t)rows * cols);
                    CK(cudaMemcpy2DAsync(hrow.data(), (size_t)cols * 4, c->d_logits, CH * 4, (size_t)cols * 4, rows, cudaMemcpyDeviceToHost, c->stream));
                    CK(cudaStreamSynchronize(c->stream));
                    for (float& v : hrow) if (v != v) v = -FLT_MAX;
                    hidx.resize(cols);
                    for (int i = 0; i < rows; i++) {
                        const float* r = hrow.data() + (size_t)i * cols;
                        std::iota(hidx.begin(), hidx.end(), 0);
                        std::partial_sort(hidx.begin(), hidx.begin() + k, hidx.end(), [&](int x, int y) { return r[x] > r[y] || (r[x] == r[y] && x < y); });
                        for (int j = 0; j < k; j++) { a.scores[(r0 + i) * k + j] = r[hidx[j]]; a.indices[(r0 + i) * k + j] = hidx[j]; }
                    }
                }
            }
            if (!device_select) continue;
        }
        const int cur = merge_candidates(c, rows, cand_ld, runs, kk);
        CK(cudaMemcpy2DAsync(a.scores + r0 * k, (size_t)k * 4, c->d_cand_v[cur], cand_ld * 4, (size_t)k * 4, rows, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpy2DAsync(a.indices + r0 * k, (size_t)k * 4, c->d_cand_i[cur], cand_ld * 4, (size_t)k * 4, rows, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    }
    CK(cudaGetLastError());
    return true;
}

// ---- the inverted-file index (clip_b200_ivf_*) ---------------------------------------------------------------------------------------
// Carve the IVF arena into pieces of the given byte sizes, each 256-byte aligned, growing it first if it is too small.
static bool ivf_arena(clip_ctx* c, std::initializer_list<size_t> sizes, std::initializer_list<void**> out) {
    size_t total = 0;
    for (size_t b : sizes) total += (b + 255) / 256 * 256;
    if (!ensure_buf(c, &c->d_ivf, &c->d_ivf_cap, std::max<size_t>(total, 256))) return false;
    size_t o = 0;
    auto it = out.begin();
    for (size_t b : sizes) { **it++ = c->d_ivf + o; o += (b + 255) / 256 * 256; }
    return true;
}

// The list of each of the n rows x [n, dim]: K10 with top_k = 1 over the centroids, kept on the device through the merge, one
// index per row to the host.  Blocks of 32768 rows, the merge grid's row limit.
static bool ivf_assign(clip_ctx* c, const SearchCall& a, const void* x, size_t n, std::vector<int>& list) {
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    const KOp op = a.type == CLIP_B200_OUT_BF16 ? KOp::BF16 : KOp::F16;
    list.resize(n);
    for (size_t r0 = 0; r0 < n; r0 += 32768) {
        const int rows = (int)std::min<size_t>(32768, n - r0);
        const KnnPlan pl = knn_plan(rows, a.n_lists, 1, sms);
        if (!ensure_buf(c, &c->d_knn, &c->d_knn_cap, 2 * pl.buf_entries) || !ensure_cand(c, (size_t)rows * pl.parts)) return false;
        {
            Scope s(c, K_KNN16);
            const cudaError_t e = launch_knn(op, (const uint8_t*)x + r0 * a.dim * 2, nullptr, rows, a.cent, nullptr, a.n_lists, a.dim, 1, pl,
                                             c->d_knn, c->d_cand_v[0], c->d_cand_i[0], pl.parts, c->stream);
            if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        }
        const int cur = merge_candidates(c, rows, pl.parts, pl.parts, 1);
        CK(cudaMemcpy2DAsync(list.data() + r0, 4, c->d_cand_i[cur], (size_t)pl.parts * 4, 4, rows, cudaMemcpyDeviceToHost, c->stream));
    }
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

// The layout of an assignment: a counting sort, stable by row index.  off [n_lists + 1], ids [n].
static void ivf_layout(const std::vector<int>& list, int n_lists, std::vector<int>& off, std::vector<int>& ids) {
    off.assign(n_lists + 1, 0);
    for (int l : list) off[l + 1]++;
    for (int l = 0; l < n_lists; l++) off[l + 1] += off[l];
    std::vector<int> pos(off.begin(), off.end() - 1);
    ids.resize(list.size());
    for (size_t i = 0; i < list.size(); i++) ids[pos[list[i]]++] = (int)i;
}

// k-means: initial centroids gathered from rows floor(i n / n_lists), then per iteration an assignment, its layout and the update
// kernels (fp64 sums over chunks of IVF_CHUNK members, combined in chunk order).
constexpr int IVF_CHUNK = 512;
static bool ivf_train_locked(clip_ctx* c, const SearchCall& a) {
    const size_t n = a.nq;
    const int L = a.n_lists;
    void* cent = const_cast<void*>(a.cent);
    std::vector<int> list, off, ids, chunk_begin(L + 1);
    std::vector<int2> chunks;
    ids.resize(L);
    for (int i = 0; i < L; i++) ids[i] = (int)((size_t)i * n / L);
    {
        int* d_init = nullptr;
        if (!ivf_arena(c, {(size_t)L * 4}, {(void**)&d_init})) return false;
        CK(cudaMemcpyAsync(d_init, ids.data(), (size_t)L * 4, cudaMemcpyHostToDevice, c->stream));
        Scope s(c, K_IVF_LAYOUT);
        launch_gather_rows16(a.q, d_init, L, a.dim, cent, c->stream);
    }
    for (int it = 0; it < a.iters; it++) {
        if (!ivf_assign(c, a, a.q, n, list)) return false;
        ivf_layout(list, L, off, ids);
        chunks.clear();
        for (int l = 0; l < L; l++) {
            for (int b = off[l]; b < off[l + 1]; b += IVF_CHUNK) chunks.push_back(make_int2(b, std::min(b + IVF_CHUNK, off[l + 1])));
            chunk_begin[l + 1] = (int)chunks.size();
        }
        int *d_ids = nullptr, *d_off = nullptr, *d_cb = nullptr;
        int2* d_ch = nullptr;
        double* d_part = nullptr;
        if (!ivf_arena(c, {n * 4, (size_t)(L + 1) * 4, (size_t)(L + 1) * 4, chunks.size() * 8, chunks.size() * a.dim * 8},
                       {(void**)&d_ids, (void**)&d_off, (void**)&d_cb, (void**)&d_ch, (void**)&d_part})) return false;
        CK(cudaMemcpyAsync(d_ids, ids.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_off, off.data(), (size_t)(L + 1) * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_cb, chunk_begin.data(), (size_t)(L + 1) * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_ch, chunks.data(), chunks.size() * 8, cudaMemcpyHostToDevice, c->stream));
        Scope s(c, K_IVF_LAYOUT);
        launch_ivf_update(a.type == CLIP_B200_OUT_BF16, a.q, a.dim, d_ids, d_ch, (int)chunks.size(), d_cb, d_off, L, d_part, cent, c->stream);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

static bool ivf_build_locked(clip_ctx* c, const SearchCall& a) {
    std::vector<int> list, off, ids;
    if (!ivf_assign(c, a, a.q, a.nq, list)) return false;
    ivf_layout(list, a.n_lists, off, ids);
    CK(cudaMemcpyAsync(a.offsets, off.data(), off.size() * 4, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(a.ids, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, c->stream));
    {
        Scope s(c, K_IVF_LAYOUT);
        launch_gather_rows16(a.q, a.ids, a.nq, a.dim, const_cast<void*>(a.db), c->stream);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

// One query block of an IVF search as its plan hands it to the form's scan: queries r0 .. r0 + rows - 1, P (query, probed list)
// pairs grouped by list, each with its query row in the block (d_pq) and its coarse score (d_ps), the work units of query tile
// 8 nt, each pair's run slot, and the form's own piece of the arena (`extra`).
struct IvfBlock {
    size_t r0;
    int rows, P, nt, nunits;
    const int* d_pq;
    const float* d_ps;
    const IvfUnit* d_units;
    const size_t* d_slot;
    void* extra;
};

// The plan both IVF searches run, per block of QB queries: the probes (K10 top-nprobe over the centroids, their ids and scores to
// the host), the host plan of the fine scan's work units (include/clip_b200.h, clip_b200_ivf_search_16), the candidate pre-fill, the
// form's scan (extra_bytes(P, rows) bytes of its own arena piece), the merge, the padding.  A unit holds at most 8 nt_max pairs:
// K10 scores a unit's pairs together in its MMA, so up to 128; K13 scores them one after another, so a unit of np pairs costs np
// times its rows, and 8 pairs a unit keep the plan's work estimate, and with it the units' balance, true to that cost.
extern "C++" {
template <class Extra, class Scan>
static bool ivf_search_plan(clip_ctx* c, const SearchCall& a, const std::vector<int>& off, size_t QB, int nt_max, Extra extra_bytes,
                            Scan scan) {
    const int L = a.n_lists, np = std::min(a.iters, L), w = (int)std::min<size_t>(a.top_k, a.ndb), KB = knn_tile_rows();
    const bool bf = a.type == CLIP_B200_OUT_BF16;
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    std::vector<int> probes, cnt(L), pstart(L + 1), fill(L), pair_q, runs;
    std::vector<float> pscore, pair_s;
    std::vector<size_t> slot;
    std::vector<IvfUnit> units;
    for (size_t r0 = 0; r0 < a.nq; r0 += QB) {
        const int rows = (int)std::min(QB, a.nq - r0);
        const uint8_t* q = (const uint8_t*)a.q + r0 * a.dim * 2;
        // coarse: the best np lists of each query, best first, with their scores
        const KnnPlan pl = knn_plan(rows, L, np, sms);
        if (!ensure_buf(c, &c->d_knn, &c->d_knn_cap, 2 * pl.buf_entries) || !ensure_cand(c, (size_t)rows * pl.parts * np)) return false;
        {
            Scope s(c, K_KNN16);
            const cudaError_t e = launch_knn(bf ? KOp::BF16 : KOp::F16, q, nullptr, rows, a.cent, nullptr, L, a.dim, np, pl, c->d_knn,
                                             c->d_cand_v[0], c->d_cand_i[0], (size_t)pl.parts * np, c->stream);
            if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        }
        const int pc = merge_candidates(c, rows, (size_t)pl.parts * np, pl.parts, np);
        probes.resize((size_t)rows * np);
        pscore.resize((size_t)rows * np);
        CK(cudaMemcpy2DAsync(probes.data(), (size_t)np * 4, c->d_cand_i[pc], (size_t)pl.parts * np * 4, (size_t)np * 4, rows,
                             cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpy2DAsync(pscore.data(), (size_t)np * 4, c->d_cand_v[pc], (size_t)pl.parts * np * 4, (size_t)np * 4, rows,
                             cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        // the plan: pairs (query, probed non-empty list) grouped by list, stable by query
        std::fill(cnt.begin(), cnt.end(), 0);
        for (int l : probes) if (off[l + 1] > off[l]) cnt[l]++;
        int lists = 0;
        for (int l = 0; l < L; l++) { pstart[l + 1] = pstart[l] + cnt[l]; lists += cnt[l] > 0; }
        const int P = pstart[L];
        pair_q.resize(P);
        pair_s.resize(P);
        std::copy(pstart.begin(), pstart.end() - 1, fill.begin());
        for (int r = 0; r < rows; r++)
            for (int j = 0; j < np; j++) {
                const size_t e = (size_t)r * np + j;
                const int l = probes[e];
                if (off[l + 1] > off[l]) { pair_s[fill[l]] = pscore[e]; pair_q[fill[l]++] = r; }
            }
        // query tile: the least 8 nt >= the mean pairs per probed list (at most 128); row ranges of R rows so that about 4 units per SM
        const int mean = lists ? (P + lists - 1) / lists : 1;
        int nt = 1;
        while (8 * nt < std::min(mean, 128) && nt < nt_max) nt <<= 1;
        const int N = 8 * nt;
        size_t work = 0;
        for (int l = 0; l < L; l++) work += (size_t)((cnt[l] + N - 1) / N) * (off[l + 1] - off[l]);
        const size_t per = (work + 4 * (size_t)sms - 1) / (4 * (size_t)sms);
        const int R = (int)std::min<size_t>((size_t)1 << 30, std::max<size_t>(KB, (per + KB - 1) / KB * KB));
        units.clear();
        for (int l = 0; l < L; l++)
            for (int j = 0; j < cnt[l]; j += N)
                for (int b = off[l], r = 0; b < off[l + 1]; b += R, r++)
                    units.push_back(IvfUnit{pstart[l] + j, std::min(N, cnt[l] - j), b, (int)std::min<int64_t>((int64_t)b + R, off[l + 1]), r});
        // run slots: query r's runs in probe order, one per row range of each probed list
        runs.assign(rows, 0);
        int runs_max = 1;
        for (int r = 0; r < rows; r++) {
            for (int j = 0; j < np; j++) { const int l = probes[(size_t)r * np + j]; runs[r] += (off[l + 1] - off[l] + R - 1) / R; }
            runs_max = std::max(runs_max, runs[r]);
        }
        const size_t cand_ld = (size_t)runs_max * w;
        slot.resize(P);
        std::copy(pstart.begin(), pstart.end() - 1, fill.begin());
        for (int r = 0; r < rows; r++)
            for (int j = 0, run = 0; j < np; j++) {
                const int l = probes[(size_t)r * np + j], nr = (off[l + 1] - off[l] + R - 1) / R;
                if (nr) slot[fill[l]++] = (size_t)r * cand_ld + (size_t)run * w;
                run += nr;
            }
        int* d_pq = nullptr;
        float* d_ps = nullptr;
        IvfUnit* d_units = nullptr;
        size_t* d_slot = nullptr;
        void* extra = nullptr;
        if (!ivf_arena(c, {(size_t)P * 4, (size_t)P * 4, units.size() * sizeof(IvfUnit), (size_t)P * 8, extra_bytes(P, rows)},
                       {(void**)&d_pq, (void**)&d_ps, (void**)&d_units, (void**)&d_slot, &extra})) return false;
        if (!ensure_cand(c, (size_t)rows * cand_ld)) return false;
        CK(cudaMemcpyAsync(d_pq, pair_q.data(), (size_t)P * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_ps, pair_s.data(), (size_t)P * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_units, units.data(), units.size() * sizeof(IvfUnit), cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_slot, slot.data(), (size_t)P * 8, cudaMemcpyHostToDevice, c->stream));
        {
            Scope s(c, K_OTHER);
            launch_fill_cand(c->d_cand_v[0], c->d_cand_i[0], (size_t)rows * cand_ld, c->stream);
        }
        if (!scan(IvfBlock{r0, rows, P, nt, (int)units.size(), d_pq, d_ps, d_units, d_slot, extra})) return false;
        const int cur = merge_candidates(c, rows, cand_ld, runs_max, w);
        float* os = a.scores + r0 * w;
        int* oi = a.indices + r0 * w;
        CK(cudaMemcpy2DAsync(os, (size_t)w * 4, c->d_cand_v[cur], cand_ld * 4, (size_t)w * 4, rows, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpy2DAsync(oi, (size_t)w * 4, c->d_cand_i[cur], cand_ld * 4, (size_t)w * 4, rows, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        for (size_t e = 0; e < (size_t)rows * w; e++)
            if (oi[e] == 0x7fffffff) { oi[e] = -1; os[e] = -INFINITY; }
    }
    CK(cudaGetLastError());
    return true;
}
}  // extern "C++"

// IVF search over 16-bit rows: the pairs' query rows gathered, K10's IVF instance.
static bool ivf_search_locked(clip_ctx* c, const SearchCall& a, const std::vector<int>& off) {
    const int np = std::min(a.iters, a.n_lists), w = (int)std::min<size_t>(a.top_k, a.ndb), KB = knn_tile_rows();
    const bool bf = a.type == CLIP_B200_OUT_BF16;
    const size_t QB = std::min<size_t>(32768, std::max<size_t>(1, ((size_t)1 << 24) / ((size_t)(w + 2 * KB) * np)));
    return ivf_search_plan(c, a, off, QB, 16, [&](int P, int) { return (size_t)P * a.dim * 2; }, [&](const IvfBlock& b) {
        const size_t buf = (size_t)b.nunits * 8 * b.nt * (size_t)(w + 2 * KB);
        if (!ensure_buf(c, &c->d_knn, &c->d_knn_cap, 2 * buf)) return false;
        {
            Scope s(c, K_OTHER);
            launch_gather_rows16((const uint8_t*)a.q + b.r0 * a.dim * 2, b.d_pq, b.P, a.dim, b.extra, c->stream);
        }
        Scope s(c, K_IVF_SCAN);
        const cudaError_t e = launch_knn_ivf(bf, b.extra, b.P, a.db, (int)a.ndb, a.dim, w, b.nt, b.d_units, b.nunits, b.d_slot, a.ids,
                                             c->d_knn, c->d_cand_v[0], c->d_cand_i[0], c->stream);
        if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        return true;
    });
}

// ---- IVF with product-quantised residuals (clip_b200_ivfpq_*) -----------------------------------------------------------------
// IVF-PQ search: each query's lookup tables, then K13 over the stored codes.  The query block also bounds the tables, Q * m KiB.
static bool pq_search_locked(clip_ctx* c, const SearchCall& a, const std::vector<int>& off) {
    const int np = std::min(a.iters, a.n_lists), w = (int)std::min<size_t>(a.top_k, a.ndb), KB = knn_tile_rows();
    const bool bf = a.type == CLIP_B200_OUT_BF16;
    const size_t QB = std::min<size_t>({32768, std::max<size_t>(1, ((size_t)1 << 24) / ((size_t)(w + 2 * KB) * np)), ((size_t)1 << 18) / a.m});
    return ivf_search_plan(c, a, off, QB, 1, [&](int, int rows) { return (size_t)rows * a.m * 1024; }, [&](const IvfBlock& b) {
        if (!ensure_buf(c, &c->d_knn, &c->d_knn_cap, 2 * (size_t)b.nunits * adc_cap(w))) return false;
        float* tables = (float*)b.extra;
        cudaError_t e;
        {
            Scope s(c, K_PQ);
            e = launch_pq_tables(bf, (const uint8_t*)a.q + b.r0 * a.dim * 2, b.rows, a.dim, a.m, (const float*)a.books, tables, c->stream);
        }
        if (e == cudaSuccess) {
            Scope s(c, K_ADC);
            e = launch_adc(a.db, (int)a.ndb, a.m, tables, b.d_ps, b.d_pq, w, b.d_units, b.nunits, b.d_slot, a.ids, c->d_knn,
                           c->d_cand_v[0], c->d_cand_i[0], c->stream);
        }
        if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        return true;
    });
}

// Codebook k-means: the lists of the training rows (the build's assignment), the initial codewords, then per iteration the codes
// of every residual, their layout per subspace (rows grouped by code, stable by row, on the host) and the update kernels (fp64
// sums over chunks of IVF_CHUNK members, combined in chunk order).  The arena is carved once, at the most chunks a layout can have.
static bool pq_train_locked(clip_ctx* c, const SearchCall& a) {
    const size_t n = a.nq;
    const int m = a.m, dsub = a.dim / m, NB = m * 256;
    const bool bf = a.type == CLIP_B200_OUT_BF16;
    std::vector<int> list;
    if (!ivf_assign(c, a, a.q, n, list)) return false;
    const size_t nch_max = (size_t)m * (n / IVF_CHUNK + 256);
    int *d_lists = nullptr, *d_ids = nullptr, *d_cb = nullptr, *d_cnt = nullptr;
    uint8_t* d_codes = nullptr;
    longlong2* d_ch = nullptr;
    double* d_part = nullptr;
    if (!ivf_arena(c, {n * 4, n * m, n * m * 4, (size_t)(NB + 1) * 4, (size_t)NB * 4, nch_max * 16, nch_max * dsub * 8},
                   {(void**)&d_lists, (void**)&d_codes, (void**)&d_ids, (void**)&d_cb, (void**)&d_cnt, (void**)&d_ch, (void**)&d_part})) return false;
    CK(cudaMemcpyAsync(d_lists, list.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
    float* books = (float*)const_cast<void*>(a.books);
    {
        Scope s(c, K_PQ);
        launch_pq_init(bf, a.q, n, a.dim, m, d_lists, a.cent, books, c->stream);
    }
    std::vector<uint8_t> codes(n * m);
    std::vector<int> ids(n * m), cnt(NB), pos(NB), chunk_begin(NB + 1);
    std::vector<longlong2> chunks;
    for (int it = 0; it < a.iters; it++) {
        {
            Scope s(c, K_PQ);
            const cudaError_t e = launch_pq_encode(bf, a.q, n, a.dim, m, d_lists, a.cent, books, d_codes, c->stream);
            if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
        }
        CK(cudaMemcpyAsync(codes.data(), d_codes, n * m, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        std::fill(cnt.begin(), cnt.end(), 0);
        for (size_t r = 0; r < n; r++)
            for (int s = 0; s < m; s++) cnt[s * 256 + codes[r * m + s]]++;
        chunks.clear();
        for (int s = 0; s < m; s++)
            for (int k = 0, p = 0; k < 256; k++) {
                const int bk = s * 256 + k;
                pos[bk] = p;
                for (int b = p; b < p + cnt[bk]; b += IVF_CHUNK)
                    chunks.push_back(make_longlong2((long long)s * n + b, (long long)s * n + std::min(b + IVF_CHUNK, p + cnt[bk])));
                chunk_begin[bk + 1] = (int)chunks.size();
                p += cnt[bk];
            }
        for (size_t r = 0; r < n; r++)
            for (int s = 0; s < m; s++) { const int bk = s * 256 + codes[r * m + s]; ids[(size_t)s * n + pos[bk]++] = (int)r; }
        CK(cudaMemcpyAsync(d_ids, ids.data(), n * m * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_cb, chunk_begin.data(), (size_t)(NB + 1) * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_cnt, cnt.data(), (size_t)NB * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_ch, chunks.data(), chunks.size() * 16, cudaMemcpyHostToDevice, c->stream));
        Scope s(c, K_PQ);
        launch_pq_update(bf, a.q, n, a.dim, m, d_lists, a.cent, d_ids, d_ch, (int)chunks.size(), d_cb, d_cnt, d_part, books, c->stream);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

static bool pq_encode_locked(clip_ctx* c, const SearchCall& a) {
    std::vector<int> list;
    if (!ivf_assign(c, a, a.q, a.nq, list)) return false;
    CK(cudaMemcpyAsync(a.lists, list.data(), a.nq * 4, cudaMemcpyHostToDevice, c->stream));
    {
        Scope s(c, K_PQ);
        const cudaError_t e = launch_pq_encode(a.type == CLIP_B200_OUT_BF16, a.q, a.nq, a.dim, a.m, a.lists, a.cent, (const float*)a.books,
                                               const_cast<void*>(a.db), c->stream);
        if (e != cudaSuccess) { set_err(std::string(a.who) + ": launch: " + cudaGetErrorString(e)); return false; }
    }
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

// The build reads the lists first and refuses a value outside [0, n_lists) before it writes anything.
static bool pq_build_locked(clip_ctx* c, const SearchCall& a) {
    std::vector<int> list(a.nq), off, ids;
    CK(cudaMemcpy(list.data(), a.lists, a.nq * 4, cudaMemcpyDeviceToHost));
    for (int l : list)
        if (l < 0 || l >= a.n_lists) { set_err(std::string(a.who) + ": d_lists values must be in [0, n_lists)"); return false; }
    ivf_layout(list, a.n_lists, off, ids);
    CK(cudaMemcpyAsync(a.offsets, off.data(), off.size() * 4, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(a.ids, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, c->stream));
    {
        Scope s(c, K_IVF_LAYOUT);
        launch_gather_rows16(a.q, a.ids, a.nq, a.m / 2, const_cast<void*>(a.db), c->stream);       // a code row is m / 2 16-bit columns
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

// Reads d_offsets and refuses an index whose offsets do not run non-decreasing from 0 to n_db (the IVF searches' check).
static bool ivf_offsets(clip_ctx* c, const SearchCall& a, std::vector<int>& off) {
    off.resize(a.n_lists + 1);
    CK(cudaMemcpy(off.data(), a.offsets, off.size() * 4, cudaMemcpyDeviceToHost));
    bool ok = off[0] == 0 && (size_t)off[a.n_lists] == a.ndb;
    for (int l = 0; ok && l < a.n_lists; l++) ok = off[l + 1] >= off[l];
    if (!ok) set_err(std::string(a.who) + ": d_offsets must run non-decreasing from 0 to n_db");
    return ok;
}

// The IVF-PQ forms past the counts: empty calls, pointers, then the locked work.
static bool pq_call(clip_ctx* c, SearchCall& a) {
    const std::string who = a.who;
    const SearchCall::Kind kind = a.kind;
    if ((kind == SearchCall::PQ_SEARCH && (a.nq == 0 || a.ndb == 0)) || (kind == SearchCall::PQ_ENCODE && a.nq == 0)) return true;
    const bool empty_build = kind == SearchCall::PQ_BUILD && a.nq == 0;
    // 16-byte aligned: rows, queries, centroids, codebooks and codes; 4-byte aligned: lists, offsets and ids
    std::vector<const void*> p16, p4;
    if (kind == SearchCall::PQ_BUILD) {
        if (!empty_build) p16 = {a.q, a.db};
        p4 = empty_build ? std::vector<const void*>{a.offsets} : std::vector<const void*>{a.lists, a.offsets, a.ids};
    } else {
        p16 = {a.q, a.cent, a.books};
        if (kind != SearchCall::PQ_TRAIN) p16.push_back(a.db);
        if (kind == SearchCall::PQ_ENCODE) p4 = {a.lists};
        if (kind == SearchCall::PQ_SEARCH) p4 = {a.offsets, a.ids};
    }
    for (const void* p : p16)
        if (!p || (uintptr_t)p % 16) { set_err(who + ": null or not 16-byte aligned device pointer"); return false; }
    for (const void* p : p4)
        if (!p || (uintptr_t)p % 4) { set_err(who + ": null or not 4-byte aligned d_lists, d_offsets or d_ids"); return false; }
    if (kind == SearchCall::PQ_SEARCH && (!a.scores || !a.indices)) { set_err(who + ": null output"); return false; }
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (empty_build) {
        CK(cudaMemsetAsync(a.offsets, 0, (size_t)(a.n_lists + 1) * 4, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        return true;
    }
    if (kind == SearchCall::PQ_TRAIN) return pq_train_locked(c, a);
    if (kind == SearchCall::PQ_ENCODE) return pq_encode_locked(c, a);
    if (kind == SearchCall::PQ_BUILD) return pq_build_locked(c, a);
    std::vector<int> off;
    return ivf_offsets(c, a, off) && pq_search_locked(c, a, off);
}

// The IVF forms past the counts: empty calls, pointers, then the locked work.  IVF_SEARCH reads d_offsets first and refuses an index
// whose offsets do not run non-decreasing from 0 to n_db, so a malformed index cannot send the scan out of d_rows.
static bool ivf_call(clip_ctx* c, SearchCall& a) {
    const std::string who = a.who;
    const SearchCall::Kind kind = a.kind;
    if (kind == SearchCall::IVF_TRAIN && a.nq < (size_t)a.n_lists) { set_err(who + ": n_train must be at least n_lists"); return false; }
    if (kind == SearchCall::IVF_SEARCH && (a.nq == 0 || a.ndb == 0)) return true;
    const bool empty_build = kind == SearchCall::IVF_BUILD && a.nq == 0;
    // 16-byte aligned: the rows and centroids (TMA, 16-byte loads); 4-byte aligned: offsets and ids
    const void* p16[3] = {a.q, a.cent, a.db};
    const int n16 = empty_build ? 0 : kind == SearchCall::IVF_TRAIN ? 2 : 3;
    for (int i = 0; i < n16; i++)
        if (!p16[i] || (uintptr_t)p16[i] % 16) { set_err(who + ": null or not 16-byte aligned device pointer"); return false; }
    const int* p4[2] = {a.offsets, a.ids};
    const int n4 = kind == SearchCall::IVF_TRAIN ? 0 : empty_build ? 1 : 2;
    for (int i = 0; i < n4; i++)
        if (!p4[i] || (uintptr_t)p4[i] % 4) { set_err(who + ": null or not 4-byte aligned d_offsets or d_ids"); return false; }
    if (kind == SearchCall::IVF_SEARCH && (!a.scores || !a.indices)) { set_err(who + ": null output"); return false; }
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (empty_build) {
        CK(cudaMemsetAsync(a.offsets, 0, (size_t)(a.n_lists + 1) * 4, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        return true;
    }
    if (kind == SearchCall::IVF_TRAIN) return ivf_train_locked(c, a);
    if (kind == SearchCall::IVF_BUILD) return ivf_build_locked(c, a);
    std::vector<int> off;
    return ivf_offsets(c, a, off) && ivf_search_locked(c, a, off);
}

// Every form of the family: the arguments checked in one order, the first fault refused (include/clip_b200.h), then the search pass or
// the row kernel.
static bool search_call(const clip_ctx* cctx, SearchCall a) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    const std::string who = a.who;
    const SearchCall::Kind kind = a.kind;
    if (!c) { set_err(who + ": null context"); return false; }
    const bool typed = a.ivf() || (a.pq() && kind != SearchCall::PQ_BUILD);      // the IVF forms that read 16-bit rows
    if ((kind == SearchCall::KNN16 || kind == SearchCall::ROWS16 || typed) && a.type != CLIP_B200_OUT_F16 && a.type != CLIP_B200_OUT_BF16) {
        set_err(who + (kind == SearchCall::ROWS16 ? ": out_type" : ": in_type") + " must be CLIP_B200_OUT_F16 or CLIP_B200_OUT_BF16");
        return false;
    }
    if (kind == SearchCall::RESCORE && a.type != CLIP_B200_OUT_F32 && a.type != CLIP_B200_OUT_F16 && a.type != CLIP_B200_OUT_BF16) {
        set_err(who + ": in_type must be CLIP_B200_OUT_F32, CLIP_B200_OUT_F16 or CLIP_B200_OUT_BF16");
        return false;
    }
    const int step = kind == SearchCall::KNN16 || kind == SearchCall::RESCORE || typed ? 8 : kind == SearchCall::ROWS16 ? 4
                   : kind == SearchCall::KNN_B1 || kind == SearchCall::ROWS_B1 ? 128 : 16;     // SCORE's dim is the model's
    if (kind != SearchCall::SCORE && kind != SearchCall::PQ_BUILD && (a.dim < step || a.dim > 2048 || a.dim % step)) {
        set_err(who + ": dim must be a multiple of " + std::to_string(step) + " in [" + std::to_string(step) + ", 2048]");
        return false;
    }
    if (kind == SearchCall::RESCORE) {
        if (a.n_cand < 1 || a.n_cand > 2048) { set_err(who + ": n_cand must be in [1, 2048]"); return false; }
        if (a.top_k < 1 || a.top_k > a.n_cand) { set_err(who + ": top_k must be in [1, n_cand]"); return false; }
    }
    // m: whole 16-byte words of codes per row (the build's copy is launch_gather_rows16 on m / 2 16-bit columns), dividing dim
    if (a.pq() && (a.m < 16 || a.m > 256 || a.m % 16 || (kind != SearchCall::PQ_BUILD && a.dim % a.m))) {
        set_err(who + (kind == SearchCall::PQ_BUILD ? ": m must be a multiple of 16 in [16, 256]" : ": m must be a multiple of 16 in [16, 256] that divides dim"));
        return false;
    }
    const bool train = kind == SearchCall::IVF_TRAIN || kind == SearchCall::PQ_TRAIN, isearch = kind == SearchCall::IVF_SEARCH || kind == SearchCall::PQ_SEARCH;
    if ((a.ivf() || a.pq()) && (a.n_lists < 1 || a.n_lists > 65536)) { set_err(who + ": n_lists must be in [1, 65536]"); return false; }
    if (train && (a.iters < 1 || a.iters > 1000)) { set_err(who + ": n_iter must be in [1, 1000]"); return false; }
    if (isearch && (a.iters < 1 || a.iters > 1024)) { set_err(who + ": nprobe must be in [1, 1024]"); return false; }
    if ((a.knn() || isearch) && (a.top_k < 1 || a.top_k > 1024)) { set_err(who + ": top_k must be in [1, 1024]"); return false; }
    if (a.nq > 0x7fffffffull || a.ndb > 0x7fffffffull) {
        set_err(who + (a.search() || isearch ? ": n_queries and n_db must be below 2^31"
                       : train ? ": n_train must be below 2^31" : kind == SearchCall::IVF_BUILD || kind == SearchCall::PQ_BUILD ? ": n_db must be below 2^31"
                       : ": n must be below 2^31"));
        return false;
    }
    if (kind == SearchCall::PQ_TRAIN && a.nq < 256) { set_err(who + ": n_train must be at least 256"); return false; }
    if (a.ivf()) return ivf_call(c, a);
    if (a.pq()) return pq_call(c, a);
    if (a.nq == 0 || (a.search() && a.ndb == 0)) return true;
    // the device pointers the kind reads or writes: q and db, then the int8 forms' scales or ROWS_B1's optional centre.  K10, K11, K12
    // and the row kernels load and store 16 bytes at a time; the fp32 kernels read single floats.
    const void* ptr[4] = {a.q, a.db, a.xs, a.qs};
    const int n_ptr = kind == SearchCall::KNN_I8 ? 4 : kind == SearchCall::ROWS_I8 || kind == SearchCall::ROWS_B1 ? 3 : 2;
    for (int i = 0; i < n_ptr; i++)
        if ((!ptr[i] && !(kind == SearchCall::ROWS_B1 && i == 2)) || (kind != SearchCall::SCORE && (uintptr_t)ptr[i] % 16)) {
            set_err(who + (kind == SearchCall::SCORE ? ": null device pointer" : ": null or not 16-byte aligned device pointer"));
            return false;
        }
    if (kind == SearchCall::RESCORE && !a.cand) { set_err(who + ": null cand"); return false; }
    if (a.search() && (!a.scores || !a.indices)) { set_err(who + ": null output"); return false; }
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (kind == SearchCall::SCORE) a.dim = c->has_vision ? c->vhp.projection_dim : c->thp.projection_dim;
    if (a.search()) return search_locked(c, a);
    if (kind == SearchCall::ROWS16) {
        // K7 with one row per item, no CLS skip and no LayerNorm: an RNE copy.  Its offsets are size_t, so n * dim may pass 2^32.
        Scope s(c, K_TOKEN_ROWS);
        launch_token_rows((const float*)a.q, (size_t)a.dim, (int)a.nq, 1, 0, a.dim, nullptr, nullptr, 0.f, a.type, const_cast<void*>(a.db), c->stream);
    } else if (kind == SearchCall::ROWS_I8) {
        Scope s(c, K_OTHER);
        launch_rows_to_int8((const float*)a.q, (int)a.nq, a.dim, const_cast<void*>(a.db), (float*)const_cast<void*>(a.xs), c->stream);
    } else {
        Scope s(c, K_OTHER);
        launch_rows_to_binary((const float*)a.q, (int)a.nq, a.dim, (const float*)a.xs, const_cast<void*>(a.db), c->stream);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

bool clip_b200_zero_shot_batch(const struct clip_ctx* cctx, const void* d_img, size_t n_img, const void* d_txt, size_t n_txt, float* scores,
                               int* indices, int top_k) {
    SearchCall a{"clip_b200_zero_shot_batch", SearchCall::SCORE};
    a.q = d_img; a.nq = n_img; a.db = d_txt; a.ndb = n_txt; a.top_k = top_k; a.softmax = true; a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

bool clip_b200_topk_search(const struct clip_ctx* cctx, const void* d_queries, size_t n_queries, const void* d_db, size_t n_db, int top_k,
                           float* scores, int* indices) {
    SearchCall a{"clip_b200_topk_search", SearchCall::SCORE};
    a.q = d_queries; a.nq = n_queries; a.db = d_db; a.ndb = n_db; a.top_k = top_k; a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

bool clip_b200_rows_to_16bit(const struct clip_ctx* cctx, const void* d_src, size_t n, int dim, int out_type, void* d_dst) {
    SearchCall a{"clip_b200_rows_to_16bit", SearchCall::ROWS16};
    a.q = d_src; a.nq = n; a.dim = dim; a.type = out_type; a.db = d_dst;
    return search_call(cctx, a);
}

bool clip_b200_topk_search_16(const struct clip_ctx* cctx, const void* d_queries, size_t n_queries, const void* d_db, size_t n_db, int dim,
                              int in_type, int top_k, float* scores, int* indices) {
    SearchCall a{"clip_b200_topk_search_16", SearchCall::KNN16};
    a.q = d_queries; a.nq = n_queries; a.db = d_db; a.ndb = n_db; a.dim = dim; a.type = in_type; a.top_k = top_k;
    a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

bool clip_b200_rows_to_int8(const struct clip_ctx* cctx, const void* d_src, size_t n, int dim, void* d_codes, void* d_scales) {
    SearchCall a{"clip_b200_rows_to_int8", SearchCall::ROWS_I8};
    a.q = d_src; a.nq = n; a.dim = dim; a.db = d_codes; a.xs = d_scales;
    return search_call(cctx, a);
}

bool clip_b200_topk_search_i8(const struct clip_ctx* cctx, const void* d_q_codes, const void* d_q_scales, size_t n_queries,
                              const void* d_db_codes, const void* d_db_scales, size_t n_db, int dim, int top_k, float* scores, int* indices) {
    SearchCall a{"clip_b200_topk_search_i8", SearchCall::KNN_I8};
    a.q = d_q_codes; a.qs = d_q_scales; a.nq = n_queries; a.db = d_db_codes; a.xs = d_db_scales; a.ndb = n_db; a.dim = dim;
    a.top_k = top_k; a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

bool clip_b200_rows_to_binary(const struct clip_ctx* cctx, const void* d_src, size_t n, int dim, const void* d_center, void* d_bits) {
    SearchCall a{"clip_b200_rows_to_binary", SearchCall::ROWS_B1};
    a.q = d_src; a.nq = n; a.dim = dim; a.xs = d_center; a.db = d_bits;
    return search_call(cctx, a);
}

bool clip_b200_topk_search_b1(const struct clip_ctx* cctx, const void* d_q_bits, size_t n_queries, const void* d_db_bits, size_t n_db,
                              int dim, int top_k, float* scores, int* indices) {
    SearchCall a{"clip_b200_topk_search_b1", SearchCall::KNN_B1};
    a.q = d_q_bits; a.nq = n_queries; a.db = d_db_bits; a.ndb = n_db; a.dim = dim; a.top_k = top_k; a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

bool clip_b200_topk_rescore(const struct clip_ctx* cctx, const void* d_queries, size_t n_queries, const void* d_db, size_t n_db, int dim,
                            int in_type, const int* cand, int n_cand, int top_k, float* scores, int* indices) {
    SearchCall a{"clip_b200_topk_rescore", SearchCall::RESCORE};
    a.q = d_queries; a.nq = n_queries; a.db = d_db; a.ndb = n_db; a.dim = dim; a.type = in_type; a.cand = cand; a.n_cand = n_cand;
    a.top_k = top_k; a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

bool clip_b200_ivf_train_16(const struct clip_ctx* cctx, const void* d_train, size_t n_train, int dim, int in_type, int n_lists, int n_iter,
                            void* d_centroids) {
    SearchCall a{"clip_b200_ivf_train_16", SearchCall::IVF_TRAIN};
    a.q = d_train; a.nq = n_train; a.dim = dim; a.type = in_type; a.n_lists = n_lists; a.iters = n_iter; a.cent = d_centroids;
    return search_call(cctx, a);
}

bool clip_b200_ivf_build_16(const struct clip_ctx* cctx, const void* d_db, size_t n_db, int dim, int in_type, const void* d_centroids,
                            int n_lists, int* d_offsets, int* d_ids, void* d_rows) {
    SearchCall a{"clip_b200_ivf_build_16", SearchCall::IVF_BUILD};
    a.q = d_db; a.nq = n_db; a.dim = dim; a.type = in_type; a.cent = d_centroids; a.n_lists = n_lists; a.offsets = d_offsets; a.ids = d_ids;
    a.db = d_rows;
    return search_call(cctx, a);
}

bool clip_b200_ivf_search_16(const struct clip_ctx* cctx, const void* d_queries, size_t n_queries, int dim, int in_type, const void* d_centroids,
                             int n_lists, const int* d_offsets, const int* d_ids, const void* d_rows, size_t n_db, int nprobe, int top_k,
                             float* scores, int* indices) {
    SearchCall a{"clip_b200_ivf_search_16", SearchCall::IVF_SEARCH};
    a.q = d_queries; a.nq = n_queries; a.dim = dim; a.type = in_type; a.cent = d_centroids; a.n_lists = n_lists;
    a.offsets = const_cast<int*>(d_offsets); a.ids = const_cast<int*>(d_ids); a.db = d_rows; a.ndb = n_db; a.iters = nprobe; a.top_k = top_k;
    a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

bool clip_b200_ivfpq_train_16(const struct clip_ctx* cctx, const void* d_train, size_t n_train, int dim, int in_type, const void* d_centroids,
                              int n_lists, int m, int n_iter, void* d_codebooks) {
    SearchCall a{"clip_b200_ivfpq_train_16", SearchCall::PQ_TRAIN};
    a.q = d_train; a.nq = n_train; a.dim = dim; a.type = in_type; a.cent = d_centroids; a.n_lists = n_lists; a.m = m; a.iters = n_iter;
    a.books = d_codebooks;
    return search_call(cctx, a);
}

bool clip_b200_ivfpq_encode_16(const struct clip_ctx* cctx, const void* d_rows, size_t n, int dim, int in_type, const void* d_centroids,
                               int n_lists, const void* d_codebooks, int m, int* d_lists, void* d_codes) {
    SearchCall a{"clip_b200_ivfpq_encode_16", SearchCall::PQ_ENCODE};
    a.q = d_rows; a.nq = n; a.dim = dim; a.type = in_type; a.cent = d_centroids; a.n_lists = n_lists; a.books = d_codebooks; a.m = m;
    a.lists = d_lists; a.db = d_codes;
    return search_call(cctx, a);
}

bool clip_b200_ivfpq_build(const struct clip_ctx* cctx, const int* d_lists, const void* d_codes, size_t n_db, int n_lists, int m,
                           int* d_offsets, int* d_ids, void* d_codes_out) {
    SearchCall a{"clip_b200_ivfpq_build", SearchCall::PQ_BUILD};
    a.lists = const_cast<int*>(d_lists); a.q = d_codes; a.nq = n_db; a.n_lists = n_lists; a.m = m; a.offsets = d_offsets; a.ids = d_ids;
    a.db = d_codes_out;
    return search_call(cctx, a);
}

bool clip_b200_ivfpq_search_16(const struct clip_ctx* cctx, const void* d_queries, size_t n_queries, int dim, int in_type,
                               const void* d_centroids, int n_lists, const void* d_codebooks, int m, const int* d_offsets, const int* d_ids,
                               const void* d_codes, size_t n_db, int nprobe, int top_k, float* scores, int* indices) {
    SearchCall a{"clip_b200_ivfpq_search_16", SearchCall::PQ_SEARCH};
    a.q = d_queries; a.nq = n_queries; a.dim = dim; a.type = in_type; a.cent = d_centroids; a.n_lists = n_lists; a.books = d_codebooks;
    a.m = m; a.offsets = const_cast<int*>(d_offsets); a.ids = const_cast<int*>(d_ids); a.db = d_codes; a.ndb = n_db; a.iters = nprobe;
    a.top_k = top_k; a.scores = scores; a.indices = indices;
    return search_call(cctx, a);
}

// =====================================================================================================================
// Multi-GPU inside the library (dist.h).  ranks mode: one process per GPU joined by clip_b200_dist_init; devices mode: one
// process, CLIP_B200_DEVICES at clip_model_load.  The ONLY exchange of the path is one NCCL all-gather of final embeddings.
// =====================================================================================================================
bool clip_b200_dist_unique_id(void* out128) {
    std::string e;
    if (!dist_unique_id(out128, e)) { set_err(e); return false; }
    return true;
}

bool clip_b200_dist_init_with_id(struct clip_ctx* c, int rank, int world, const void* id128) {
    if (!c || !id128) { set_err("clip_b200_dist_init: null argument"); return false; }
    if (c->replicas.size() > 1) { set_err("clip_b200_dist_init: this context is already in devices mode (CLIP_B200_DEVICES)"); return false; }
    if (c->dist.comm) { set_err("clip_b200_dist_init: already initialised"); return false; }
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    std::string e;
    if (!dist_init_rank(c->dist, rank, world, id128, e)) { set_err(e); return false; }
    return true;
}

bool clip_b200_dist_init(struct clip_ctx* c, int rank, int world, const char* rendezvous) {
    if (!c) { set_err("clip_b200_dist_init: null context"); return false; }
    if (world == 1) return true;
    unsigned char id[128];
    std::string e;
    if (!dist_rendezvous_id(rank, world, rendezvous, id, e)) { set_err(e); return false; }
    const bool ok = clip_b200_dist_init_with_id(c, rank, world, id);
    dist_rendezvous_done(rank);
    return ok;
}

int clip_b200_dist_rank(const struct clip_ctx* c) { return c ? c->dist.rank : 0; }
int clip_b200_dist_world(const struct clip_ctx* c) { return c ? (c->replicas.size() > 1 ? 1 : c->dist.world) : 1; }
int clip_b200_device_count(const struct clip_ctx* c) { return c ? std::max<int>(1, (int)c->replicas.size()) : 0; }
int clip_b200_nccl_version(void) { return dist_nccl_version(); }
int clip_b200_cuda_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }

static bool ensure_scalars(clip_ctx* c) {
    if (c->d_scalars) return true;
    return dev_alloc(c, &c->d_scalars, 16);
}

bool clip_b200_dist_all_gather(const struct clip_ctx* cctx, const void* d_send, void* d_recv, size_t bytes_per_rank) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    if (!c) return false;
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (!ranks_mode(c)) {
        if (d_send != d_recv) CK(cudaMemcpyAsync(d_recv, d_send, bytes_per_rank, cudaMemcpyDeviceToDevice, c->stream));
    } else {
        std::string e;
        if (!dist_all_gather(c->dist, d_send, d_recv, bytes_per_rank, c->stream, e)) { set_err(e); return false; }
    }
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

bool clip_b200_dist_max_f64(const struct clip_ctx* cctx, double* vals, int n) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    if (!c || n < 0 || n > 16) { set_err("clip_b200_dist_max_f64: n must be in [0, 16]"); return false; }
    if (!ranks_mode(c) || n == 0) return true;
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (!ensure_scalars(c)) return false;
    CK(cudaMemcpyAsync(c->d_scalars, vals, (size_t)n * 8, cudaMemcpyHostToDevice, c->stream));
    std::string e;
    if (!dist_all_reduce_max_f64(c->dist, c->d_scalars, (size_t)n, c->stream, e)) { set_err(e); return false; }
    CK(cudaMemcpyAsync(vals, c->d_scalars, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return true;
}

bool clip_b200_dist_barrier(const struct clip_ctx* cctx) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    if (!c) return false;
    if (ranks_mode(c)) { double v = 0.0; if (!clip_b200_dist_max_f64(c, &v, 1)) return false; }
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    return true;
}

bool clip_b200_image_encode_device_all(const struct clip_ctx* cctx, const void* d_pixels, size_t n_local, void* d_vec_all, bool normalize) {
    EncodeCall a{"clip_b200_image_encode_device_all", EncodeCall::DEVICE_PIXELS};
    a.in = d_pixels; a.n = n_local; a.normalize = normalize; a.d_vec = (float*)d_vec_all; a.all = true;
    return encode_call(cctx, a);
}

bool clip_b200_image_batch_encode_all(const struct clip_ctx* cctx, const int n_threads, const struct clip_image_f32_batch* imgs, float* vec_all,
                                      const bool normalize) {
    EncodeCall a{"clip_b200_image_batch_encode_all", EncodeCall::F32_IMAGES};
    a.batch(imgs); a.n_threads = n_threads; a.normalize = normalize; a.vec = vec_all; a.all = true;
    return encode_call(cctx, a);
}

bool clip_b200_text_batch_encode_all(const struct clip_ctx* cctx, const int n_threads, const struct clip_tokens* seqs, const size_t n, float* vec_all,
                                     const bool normalize) {
    (void)n_threads;
    EncodeCall a{"clip_b200_text_batch_encode_all", EncodeCall::TOKENS};
    a.in = seqs; a.n = n; a.normalize = normalize; a.vec = vec_all; a.all = true;
    return encode_call(cctx, a);
}

bool clip_b200_text_encode_device_all(const struct clip_ctx* cctx, const void* d_ids, const void* d_lens, size_t n_local, int seq_len,
                                      void* d_vec_all, bool normalize) {
    EncodeCall a{"clip_b200_text_encode_device_all", EncodeCall::DEVICE_IDS};
    a.in = d_ids; a.d_lens = (const int32_t*)d_lens; a.n = n_local; a.seq_len = seq_len; a.normalize = normalize; a.d_vec = (float*)d_vec_all;
    a.all = true;
    return encode_call(cctx, a);
}

// Batched zero-shot labelling (BASELINE.json configs[4]; per image the arithmetic of clip_zero_shot_label_image, clip.cpp:1624-1659):
//   single GPU   : n images x n_labels labels
//   devices mode : images AND labels are sharded over the GPUs, the label embeddings are all-gathered (NCCL), every GPU scores its images
//   ranks mode   : the caller passes THIS rank's images and THIS rank's label shard (same count on every rank); label j of rank r has
//                  global index r * n_labels + j; scores / indices cover this rank's images against all world * n_labels labels
// scores / indices: [n images, top_k], best first.  The embeddings never leave the GPUs.
bool clip_b200_zero_shot_images(const struct clip_ctx* cctx, const int n_threads, const struct clip_image_f32_batch* imgs,
                                const struct clip_tokens* labels, const size_t n_labels, const bool normalize, int top_k, float* scores,
                                int* indices) {
    clip_ctx* c = const_cast<clip_ctx*>(cctx);
    const char* who = "clip_b200_zero_shot_images";
    if (!c || !(c->has_text && c->has_vision)) { set_err("clip_b200_zero_shot_images needs a two-tower model"); return false; }
    const size_t n = imgs ? imgs->size : 0;
    if (n == 0 || n_labels == 0) return n == 0;
    if (!check_images(c, imgs->data, n, who) || !check_tokens(c, labels, n_labels, who)) return false;
    EncodeCall ai{who, EncodeCall::F32_IMAGES}, at{who, EncodeCall::TOKENS};
    ai.batch(imgs); ai.n_threads = n_threads; ai.normalize = normalize;
    at.in = labels; at.n = n_labels; at.normalize = normalize;
    const int d = c->vis.proj;
    // the last phase on context r (caller holds r->mu and has set its device): its nq images against ndb labels, into the output
    // rows from lo on
    const auto score = [&](clip_ctx* r, size_t nq, size_t ndb, size_t lo) {
        SearchCall s{who, SearchCall::SCORE};
        s.q = r->d_emb[0]; s.nq = nq; s.db = r->d_emb[1]; s.ndb = ndb; s.dim = d; s.top_k = top_k; s.softmax = true;
        s.scores = scores + lo * top_k; s.indices = indices + lo * top_k;
        return search_locked(r, s);
    };
    if (c->replicas.size() > 1) {
        const int w = (int)c->replicas.size();
        const size_t per = (n_labels + w - 1) / w, tot = (size_t)w * per;      // equal slots; only the last ones may be partly empty
        if (top_k <= 0 || (size_t)top_k > n_labels) top_k = (int)n_labels;
        // phase 1: every GPU encodes its image shard and its label shard (slot r of its own gather buffer)
        if (!for_each_replica(c, n, [&](clip_ctx* r, int ri, size_t lo, size_t hi) {
                {
                    std::lock_guard<std::mutex> lk(r->mu);
                    CK(cudaSetDevice(r->device));
                    if (!ensure_buf(r, &r->d_emb[0], &r->d_emb_cap[0], std::max<size_t>(hi - lo, 1) * d) || !ensure_buf(r, &r->d_emb[1], &r->d_emb_cap[1], tot * d)) return false;
                    CK(cudaMemsetAsync(r->d_emb[1], 0, tot * d * 4, r->stream));
                }
                if (hi > lo && !encode_pass(r, ai, lo, hi, nullptr, r->d_emb[0], false)) return false;
                const size_t l0 = std::min(n_labels, (size_t)ri * per), l1 = std::min(n_labels, l0 + per);
                if (l1 > l0 && !encode_pass(r, at, l0, l1, nullptr, r->d_emb[1] + (size_t)ri * per * d, false)) return false;
                return true;
            })) return false;
        // phase 2: ONE all-gather of the label embeddings, in place on every GPU (group call: one thread drives all communicators)
        std::string e;
        if (!dist_group_start(e)) { set_err(e); return false; }
        for (int ri = 0; ri < w; ri++) {
            clip_ctx* r = c->replicas[ri];
            cudaSetDevice(r->device);
            if (!dist_all_gather(r->dist, r->d_emb[1] + (size_t)ri * per * d, r->d_emb[1], per * d * 4, r->stream, e)) { dist_group_end(e); set_err(e); return false; }
        }
        if (!dist_group_end(e)) { set_err(e); return false; }
        cudaSetDevice(c->device);
        // phase 3: every GPU ranks the labels for its images and copies its slice of the result to the caller
        return for_each_replica(c, n, [&](clip_ctx* r, int, size_t lo, size_t hi) {
            if (hi == lo) return true;
            std::lock_guard<std::mutex> lk(r->mu);
            CK(cudaSetDevice(r->device));
            return score(r, hi - lo, n_labels, lo);
        });
    }
    const int w = ranks_mode(c) ? c->dist.world : 1, rank = ranks_mode(c) ? c->dist.rank : 0;
    const size_t n_all = (size_t)w * n_labels;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        CK(cudaSetDevice(c->device));
        if (!ensure_buf(c, &c->d_emb[0], &c->d_emb_cap[0], n * d) || !ensure_buf(c, &c->d_emb[1], &c->d_emb_cap[1], n_all * d)) return false;
    }
    if (!encode_pass(c, ai, 0, n, nullptr, c->d_emb[0], false)) return false;
    if (!encode_pass(c, at, 0, n_labels, nullptr, c->d_emb[1] + (size_t)rank * n_labels * d, false)) return false;
    std::lock_guard<std::mutex> lk(c->mu);
    CK(cudaSetDevice(c->device));
    if (!gather_in_place(c, c->d_emb[1], n_labels, d)) return false;
    return score(c, n, n_all, 0);
}

bool clip_model_quantize(const char* fname_inp, const char* fname_out, const int itype) {
    try {
        std::string err;
        if (!quantize_file(fname_inp, fname_out, itype, err)) { set_err("clip_model_quantize: " + err); return false; }
        return true;
    } catch (const std::exception& e) { set_err(std::string("clip_model_quantize: ") + e.what()); return false; }
}

// ---- helpers ---------------------------------------------------------------------------------------------------
void* clip_b200_device_malloc(const struct clip_ctx* c, size_t bytes) {
    if (c) cudaSetDevice(c->device);
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { set_err("cudaMalloc failed"); return nullptr; }
    return p;
}
void clip_b200_device_free(const struct clip_ctx* c, void* p) { if (c) cudaSetDevice(c->device); cudaFree(p); }
void* clip_b200_host_malloc(size_t bytes) { void* p = nullptr; if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr; return p; }
void clip_b200_host_free(void* p) { cudaFreeHost(p); }
// Returns once the bytes are on the device.  A plain cudaMemcpy from pageable memory may return while its last DMA is still in
// flight, and the context's streams are non-blocking (not ordered after the legacy default stream), so the next launch could read
// the buffer's tail before it lands.  The copy therefore goes on the context's stream, which every later launch is ordered after.
bool clip_b200_memcpy_h2d(const struct clip_ctx* c, void* d, const void* h, size_t bytes) {
    if (!c) {
        CK(cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice));
        CK(cudaDeviceSynchronize());
        return true;
    }
    CK(cudaSetDevice(c->device));
    CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return true;
}
bool clip_b200_memcpy_d2h(const struct clip_ctx* c, void* h, const void* d, size_t bytes) {
    if (c) cudaSetDevice(c->device);
    CK(cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost));
    return true;
}
bool clip_b200_synchronize(const struct clip_ctx* c) { if (c) cudaSetDevice(c->device); CK(cudaDeviceSynchronize()); return true; }
void* clip_b200_get_stream(const struct clip_ctx* c) { return c ? (void*)c->stream : nullptr; }
void clip_b200_set_micro_batch(const struct clip_ctx* cc, int images, int sequences) {
    clip_ctx* c = const_cast<clip_ctx*>(cc);
    if (!c) return;
    if (images > 0 && c->has_vision && c->vis.ws.cap_items == 0) c->vis.micro_batch = images;
    if (sequences > 0 && c->has_text && c->txt.ws.cap_items == 0) c->txt.micro_batch = sequences;
}
// CUDA-event stopwatch on the launch stream (slots 0..3) so that callers can time a region on the device; the events belong to
// the context (= to its device)
bool clip_b200_mark(const struct clip_ctx* cc, int slot) {
    clip_ctx* c = const_cast<clip_ctx*>(cc);
    if (!c || slot < 0 || slot > 3) return false;
    CK(cudaSetDevice(c->device));
    if (!c->marks[slot]) CK(cudaEventCreate(&c->marks[slot]));
    CK(cudaEventRecord(c->marks[slot], c->stream));
    return true;
}
float clip_b200_mark_elapsed_ms(const struct clip_ctx* c, int a, int b) {
    if (!c || a < 0 || a > 3 || b < 0 || b > 3 || !c->marks[a] || !c->marks[b]) return -1.f;
    cudaSetDevice(c->device);
    if (cudaEventSynchronize(c->marks[b]) != cudaSuccess) return -1.f;
    float ms = -1.f;
    cudaEventElapsedTime(&ms, c->marks[a], c->marks[b]);
    return ms;
}
uint64_t clip_b200_kernel_launches(const struct clip_ctx* c) { return c ? c->launches : 0; }
float clip_b200_last_device_ms(const struct clip_ctx* c) { return c ? c->last_ms : 0.f; }
float clip_b200_kernel_ms(const struct clip_ctx* cc, int kind, uint64_t* count) {
    clip_ctx* c = const_cast<clip_ctx*>(cc);
    if (!c) return 0.f;
    std::lock_guard<std::mutex> lk(c->mu);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    float total = 0.f;
    uint64_t n = 0;
    std::vector<ProfEvent> keep;
    for (auto& p : c->prof) {
        if (p.kind == kind) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, p.e0, p.e1);
            total += ms; n++;
            c->ev_pool.push_back(p.e0); c->ev_pool.push_back(p.e1);
        } else keep.push_back(p);
    }
    c->prof.swap(keep);
    if (count) *count = n;
    return total;
}

int clip_b200_debug_gemm_scaled(int qtype, int operand_bf16, int M, int N, int K, int epi, int use_naive, float scale, const float* x,
                                const void* w_rows, const float* bias, const float* resid_in, float* y_out, float* ms) {
    g_err.clear();
    if (gemm_init() != cudaSuccess) { set_err("gemm_init failed"); return 1; }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, dev);
    const bool out32 = (epi == EPI_STORE32 || epi == EPI_REDADD32);
    int eff_q = qtype;
    std::vector<uint16_t> x16((size_t)M * K);
    for (size_t i = 0; i < x16.size(); i++) x16[i] = operand_bf16 ? f32_to_bf16(x[i]) : f32_to_f16(x[i]);
    std::vector<uint8_t> wdev;
    std::vector<uint16_t> wf16;
    size_t raw_bytes;
    if (qtype == 0 || qtype == 1) {
        eff_q = QT_F16;
        wf16.resize((size_t)N * K);
        if (qtype == 1) memcpy(wf16.data(), w_rows, wf16.size() * 2);
        else for (size_t i = 0; i < wf16.size(); i++) wf16[i] = f32_to_f16(((const float*)w_rows)[i]);
        raw_bytes = wf16.size() * 2;
    } else {
        raw_bytes = (size_t)N * (K / 32) * wpack_ggml_block_bytes(qtype);
        wdev.resize(wpack_total_bytes(qtype, N, K));
        if (!wpack_repack(qtype, (const uint8_t*)w_rows, N, K, wdev.data())) { set_err("repack failed"); return 2; }
    }
    void *d_x = nullptr, *d_w = nullptr, *d_raw = nullptr, *d_out = nullptr;
    float* d_bias = nullptr;
    const size_t out_bytes = (size_t)M * N * (out32 ? 4 : 2);
    // one token tile of guard rows past row M, filled with 0xFF: the GEMM must leave them untouched
    const size_t guard_bytes = (size_t)GEMM_BN * N * (out32 ? 4 : 2);
    int rc = 0;
    cudaStream_t st = nullptr;
    cudaEvent_t e0, e1;
    cudaStreamCreate(&st); cudaEventCreate(&e0); cudaEventCreate(&e1);
    auto fail = [&](const char* m, cudaError_t e) { set_err(std::string(m) + ": " + cudaGetErrorString(e)); rc = 3; };
    cudaError_t e;
    do {
        if ((e = cudaMalloc(&d_x, x16.size() * 2)) != cudaSuccess) { fail("malloc x", e); break; }
        if ((e = cudaMalloc(&d_out, out_bytes + guard_bytes)) != cudaSuccess) { fail("malloc out", e); break; }
        cudaMemset((uint8_t*)d_out + out_bytes, 0xFF, guard_bytes);
        if ((e = cudaMalloc(&d_raw, raw_bytes)) != cudaSuccess) { fail("malloc raw", e); break; }
        cudaMemcpy(d_x, x16.data(), x16.size() * 2, cudaMemcpyHostToDevice);
        cudaMemcpy(d_raw, eff_q == QT_F16 ? (const void*)wf16.data() : w_rows, raw_bytes, cudaMemcpyHostToDevice);
        if (eff_q == QT_F16) d_w = d_raw;
        else { if ((e = cudaMalloc(&d_w, wdev.size())) != cudaSuccess) { fail("malloc w", e); break; } cudaMemcpy(d_w, wdev.data(), wdev.size(), cudaMemcpyHostToDevice); }
        if (bias) { cudaMalloc(&d_bias, (size_t)N * 4); cudaMemcpy(d_bias, bias, (size_t)N * 4, cudaMemcpyHostToDevice); }
        if (epi == EPI_REDADD32 && resid_in) cudaMemcpy(d_out, resid_in, out_bytes, cudaMemcpyHostToDevice);
        else cudaMemset(d_out, 0, out_bytes);
        TmaMap xm, wm;
        memset(&wm, 0, sizeof(wm));
        if (!make_tma_2d_16bit(&xm, d_x, M, K, K, GEMM_BN)) { set_err("tensor map X failed"); rc = 4; break; }
        if (eff_q == QT_F16 && !make_tma_2d_16bit(&wm, d_w, N, K, K, GEMM_BM)) { set_err("tensor map W failed"); rc = 4; break; }
        cudaEventRecord(e0, st);
        if (use_naive) {
            launch_naive_gemm(d_x, operand_bf16, d_raw, eff_q, d_bias, d_out, M, N, K, N, epi, operand_bf16, N / 2, scale, st);
            e = cudaGetLastError();
        } else {
            GemmArgs a;
            a.x_map = &xm; a.w_map = &wm; a.w_packed = (const uint8_t*)d_w; a.qtype = eff_q; a.operand_bf16 = operand_bf16 != 0;
            a.bias = d_bias; a.out = d_out; a.M = M; a.N = N; a.K = K; a.ldo = N; a.epi = epi; a.out_bf16 = operand_bf16;
            a.scale_cols = N / 2; a.scale = scale;
            e = gemm_launch(a, st, prop.multiProcessorCount, nullptr);
        }
        cudaEventRecord(e1, st);
        if (e != cudaSuccess) { fail("launch", e); break; }
        if ((e = cudaStreamSynchronize(st)) != cudaSuccess) { fail("kernel", e); break; }
        if (ms) cudaEventElapsedTime(ms, e0, e1);
        std::vector<uint8_t> guard(guard_bytes);
        cudaMemcpy(guard.data(), (uint8_t*)d_out + out_bytes, guard_bytes, cudaMemcpyDeviceToHost);
        if (std::any_of(guard.begin(), guard.end(), [](uint8_t b) { return b != 0xFF; })) { set_err("GEMM wrote past row M"); rc = 5; break; }
        if (out32) cudaMemcpy(y_out, d_out, out_bytes, cudaMemcpyDeviceToHost);
        else {
            std::vector<uint16_t> o16((size_t)M * N);
            cudaMemcpy(o16.data(), d_out, out_bytes, cudaMemcpyDeviceToHost);
            for (size_t i = 0; i < o16.size(); i++) {
                if (operand_bf16) { uint32_t b = (uint32_t)o16[i] << 16; memcpy(&y_out[i], &b, 4); }
                else y_out[i] = f16_to_f32(o16[i]);
            }
        }
    } while (0);
    cudaFree(d_x); cudaFree(d_out); cudaFree(d_raw); if (d_w && d_w != d_raw) cudaFree(d_w); cudaFree(d_bias);
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaStreamDestroy(st);
    return rc;
}

int clip_b200_debug_gemm(int qtype, int operand_bf16, int M, int N, int K, int epi, int use_naive, const float* x, const void* w_rows,
                         const float* bias, const float* resid_in, float* y_out, float* ms) {
    return clip_b200_debug_gemm_scaled(qtype, operand_bf16, M, N, K, epi, use_naive, 0.125f, x, w_rows, bias, resid_in, y_out, ms);
}


// The hooks' qkv [rows, 3*H*dh] (fp32) as the model's 16-bit QKV activations: rounded to the operand type, and each head padded to
// qkv_head_cols(dh) columns with zeros, as the loader's padded QKV projection leaves them.
static std::vector<uint16_t> qkv_to16_padded(const float* qkv, size_t rows, int H, int dh, int bf16) {
    const int dhp = qkv_head_cols(dh);
    const size_t parts = (size_t)3 * H, src_cols = parts * dh, cols = parts * dhp;
    std::vector<uint16_t> h16(rows * cols, 0);
    for (size_t r = 0; r < rows; r++)
        for (size_t ph = 0; ph < parts; ph++)
            for (int d = 0; d < dh; d++) {
                const float v = qkv[r * src_cols + ph * dh + d];
                h16[r * cols + ph * dhp + d] = bf16 ? f32_to_bf16(v) : f32_to_f16(v);
            }
    return h16;
}

// TEST HOOK: one attention launch on device 0.  qkv: fp32 host [nseq*T, 3*H*dh] (columns Q | K | V, the Q columns already scaled),
// rounded to the operand type on the way in (and padded as qkv_to16_padded does); out: fp32 host [nseq*T, H*dh].  use_legacy=1 runs
// the mma.sync flash kernel (dh 64).
int clip_b200_debug_attention_hd(int operand_bf16, int nseq, int T, int H, int head_dim, int causal, int use_legacy, const float* qkv,
                                 float* out, float* ms) {
    g_err.clear();
    if (head_dim != 64 && head_dim != 80 && head_dim != 104) { set_err("attention: head_dim must be 64 or 80 (ViT-B/L/H) or 104 (ViT-bigG/14)"); return 2; }
    if (use_legacy && head_dim != 64) { set_err("attention: the legacy kernel supports head_dim 64 only"); return 2; }
    if (attention_tc_init() != cudaSuccess) { set_err("attention_tc_init failed"); return 1; }
    const size_t rows = (size_t)nseq * T, hid = (size_t)H * head_dim, qcols = (size_t)3 * H * qkv_head_cols(head_dim);
    const std::vector<uint16_t> h16 = qkv_to16_padded(qkv, rows, H, head_dim, operand_bf16);
    uint16_t *d_qkv = nullptr, *d_out = nullptr;
    cudaStream_t st = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    int rc = 0;
    do {
        cudaError_t e;
        // one 128-row box of padding past the last sequence
        if ((e = cudaMalloc(&d_qkv, (rows + 128) * qcols * 2)) != cudaSuccess || (e = cudaMalloc(&d_out, rows * hid * 2)) != cudaSuccess) { set_err(std::string("cudaMalloc: ") + cudaGetErrorString(e)); rc = 3; break; }
        // the padding is POISONED (0xFFFF = NaN in fp16 and bf16): rows past the last sequence are stale memory in the model path
        // (ensure_ws never initialises the workspace tail), and no output may depend on them
        cudaMemset(d_qkv, 0xff, (rows + 128) * qcols * 2);
        cudaMemset(d_out, 0xff, rows * hid * 2);
        cudaMemcpy(d_qkv, h16.data(), h16.size() * 2, cudaMemcpyHostToDevice);
        cudaStreamCreate(&st); cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int rep = 0; rep < (ms ? 3 : 1); rep++) {
            cudaEventRecord(e0, st);
            if (use_legacy) { launch_attention(d_qkv, d_out, nseq, T, H, causal, operand_bf16, st); e = cudaGetLastError(); }
            else e = launch_attention_tc(d_qkv, d_out, nseq, T, H, head_dim, causal, operand_bf16, st);
            cudaEventRecord(e1, st);
            if (e != cudaSuccess) break;
            if ((e = cudaStreamSynchronize(st)) != cudaSuccess) break;
        }
        if (e != cudaSuccess) { set_err(std::string("attention: ") + cudaGetErrorString(e)); rc = 5; break; }
        if (ms) cudaEventElapsedTime(ms, e0, e1);
        std::vector<uint16_t> o16(rows * hid);
        cudaMemcpy(o16.data(), d_out, o16.size() * 2, cudaMemcpyDeviceToHost);
        for (size_t i = 0; i < o16.size(); i++) {
            if (operand_bf16) { uint32_t b = (uint32_t)o16[i] << 16; memcpy(&out[i], &b, 4); }
            else out[i] = f16_to_f32(o16[i]);
        }
    } while (0);
    cudaFree(d_qkv); cudaFree(d_out);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (st) cudaStreamDestroy(st);
    return rc;
}

int clip_b200_debug_attention(int operand_bf16, int nseq, int T, int H, int causal, int use_legacy, const float* qkv, float* out, float* ms) {
    return clip_b200_debug_attention_hd(operand_bf16, nseq, T, H, 64, causal, use_legacy, qkv, out, ms);
}

}  // extern "C"

namespace {
// Device buffers and a private stream on device 0 for the row-kernel test hooks; everything is released when it goes out of scope.
struct HookScratch {
    std::vector<void*> bufs;
    cudaStream_t st = nullptr;
    bool ok = true;
    HookScratch() {
        cudaError_t e = cudaSetDevice(0);
        if (e == cudaSuccess) e = cudaStreamCreate(&st);
        if (e != cudaSuccess) { set_err(std::string("hook setup: ") + cudaGetErrorString(e)); ok = false; }
    }
    ~HookScratch() {
        for (void* p : bufs) cudaFree(p);
        if (st) cudaStreamDestroy(st);
    }
    // `bytes` of device memory, every byte set to `fill` (0xff poisons: NaN in fp32, fp16 and bf16), then `src` copied to its start
    void* alloc(size_t bytes, int fill, const void* src = nullptr, size_t src_bytes = 0) {
        if (!ok) return nullptr;
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, std::max<size_t>(bytes, 256));
        if (e == cudaSuccess) bufs.push_back(d);
        if (e == cudaSuccess) e = cudaMemset(d, fill, std::max<size_t>(bytes, 256));
        if (e == cudaSuccess && src && src_bytes) e = cudaMemcpy(d, src, src_bytes, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { set_err(std::string("hook alloc: ") + cudaGetErrorString(e)); ok = false; return nullptr; }
        return d;
    }
    // the launch's own error, then the kernel's
    bool finish(const char* what) {
        if (!ok) return false;
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_err(std::string(what) + ": " + cudaGetErrorString(e)); ok = false; }
        return ok;
    }
    bool copy_back(void* dst, const void* src, size_t bytes) {
        if (!ok) return false;
        cudaError_t e = cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { set_err(std::string("hook copy back: ") + cudaGetErrorString(e)); ok = false; }
        return ok;
    }
};

std::vector<uint16_t> to16(const float* x, size_t n, int bf16) {
    std::vector<uint16_t> o(n);
    for (size_t i = 0; i < n; i++) o[i] = bf16 ? f32_to_bf16(x[i]) : f32_to_f16(x[i]);
    return o;
}
void from16(const uint16_t* x, size_t n, int bf16, float* out) {
    for (size_t i = 0; i < n; i++) {
        if (bf16) { uint32_t b = (uint32_t)x[i] << 16; memcpy(&out[i], &b, 4); }
        else out[i] = f16_to_f32(x[i]);
    }
}
}  // namespace

extern "C" {

// TEST HOOK: K3's varlen instance on device 0.  nseq sequences of lens[s] rows packed back to back: qkv fp32 host [sum lens, 3*H*dh]
// (laid out, rounded and padded as for clip_b200_debug_attention_hd), out fp32 host [sum lens, H*dh].  The qkv rows past the last
// sequence and one 128-row block of guard rows after the output are poisoned (0xFF); a guard row written is an error (rc 6).
static int debug_attention_varlen(const char* who, int operand_bf16, int nseq, const int* lens, int H, int head_dim, int causal,
                                  const float* qkv, float* out) {
    g_err.clear();
    const std::string w = who;
    if (causal && head_dim != 64) { set_err(w + ": head_dim must be 64"); return 2; }
    if (head_dim != 64 && head_dim != 80 && head_dim != 104) { set_err(w + ": head_dim must be 64, 80 or 104"); return 2; }
    if (nseq <= 0 || H <= 0 || !lens) { set_err(w + ": bad shape"); return 2; }
    std::vector<int> seq(2 * ((size_t)nseq + 1), 0);
    int* off = seq.data();
    int* grp = off + nseq + 1;
    for (int i = 0; i < nseq; i++) {
        if (lens[i] <= 0) { set_err(w + ": every length must be positive"); return 2; }
        off[i + 1] = off[i] + lens[i];
        grp[i + 1] = grp[i] + (lens[i] + 63) / 64;
    }
    if (attention_tc_init() != cudaSuccess) { set_err("attention_tc_init failed"); return 1; }
    const size_t rows = (size_t)off[nseq], hid = (size_t)H * head_dim, qcols = (size_t)3 * H * qkv_head_cols(head_dim), guard = 128 * hid;
    const std::vector<uint16_t> h16 = qkv_to16_padded(qkv, rows, H, head_dim, operand_bf16);
    HookScratch s;
    uint16_t* d_qkv = (uint16_t*)s.alloc((rows + 128) * qcols * 2, 0xff, h16.data(), h16.size() * 2);
    uint16_t* d_out = (uint16_t*)s.alloc((rows * hid + guard) * 2, 0xff);
    int* d_seq = (int*)s.alloc(seq.size() * 4, 0, seq.data(), seq.size() * 4);
    if (!s.ok) return 3;
    const cudaError_t e = launch_attention_tc_varlen(d_qkv, d_out, (int)rows, nseq, d_seq, grp[nseq], H, head_dim, causal, operand_bf16, s.st);
    if (e != cudaSuccess) { set_err(w + ": " + cudaGetErrorString(e)); return 5; }
    if (!s.finish(who)) return 5;
    std::vector<uint16_t> o16(rows * hid + guard);
    if (!s.copy_back(o16.data(), d_out, o16.size() * 2)) return 6;
    if (std::any_of(o16.begin() + rows * hid, o16.end(), [](uint16_t b) { return b != 0xffff; })) { set_err(w + ": a guard row was written"); return 6; }
    from16(o16.data(), rows * hid, operand_bf16, out);
    return 0;
}

int clip_b200_debug_attention_mixed(int operand_bf16, int nseq, const int* lens, int H, int head_dim, const float* qkv, float* out) {
    return debug_attention_varlen("attention_mixed", operand_bf16, nseq, lens, H, head_dim, 0, qkv, out);
}

// TEST HOOK: the same with the causal mask (the text tower's packed passes), head_dim 64 only
int clip_b200_debug_attention_mixed_causal(int operand_bf16, int nseq, const int* lens, int H, int head_dim, const float* qkv, float* out) {
    return debug_attention_varlen("attention_mixed_causal", operand_bf16, nseq, lens, H, head_dim, 1, qkv, out);
}

int clip_b200_debug_layernorm(int rows, int h, size_t in_stride, float eps, const float* x, const float* gamma, const float* beta,
                              const float* delta, int operand_bf16, float* y_out, float* x_out) {
    g_err.clear();
    if (rows <= 0 || h <= 0 || h % 4 || h > 2048 || in_stride < (size_t)h || in_stride % 4) { set_err("debug_layernorm: bad shape"); return 1; }
    HookScratch s;
    const size_t span = ((size_t)rows - 1) * in_stride + h, hb = (size_t)h * 4;
    float* d_x = (float*)s.alloc(span * 4, 0xff);
    uint16_t* d_delta = nullptr;
    if (delta) {
        const std::vector<uint16_t> d16 = to16(delta, (size_t)rows * h, operand_bf16);
        d_delta = (uint16_t*)s.alloc(span * 2, 0xff);
        if (s.ok && cudaMemcpy2D(d_delta, in_stride * 2, d16.data(), (size_t)h * 2, (size_t)h * 2, rows, cudaMemcpyHostToDevice) != cudaSuccess) {
            set_err("debug_layernorm: upload delta");
            return 3;
        }
    }
    float* d_g = (float*)s.alloc(hb, 0, gamma, hb);
    float* d_b = (float*)s.alloc(hb, 0, beta, hb);
    uint16_t* d_y = (uint16_t*)s.alloc((size_t)rows * h * 2, 0xff);
    if (s.ok && cudaMemcpy2D(d_x, in_stride * 4, x, hb, hb, rows, cudaMemcpyHostToDevice) != cudaSuccess) { set_err("debug_layernorm: upload"); return 3; }
    if (!s.ok) return 3;
    launch_layernorm(d_x, in_stride, rows, h, eps, d_g, d_b, d_delta, d_y, operand_bf16, s.st);
    if (!s.finish("layernorm")) return 5;
    std::vector<uint16_t> y16((size_t)rows * h);
    if (!s.copy_back(y16.data(), d_y, y16.size() * 2)) return 6;
    from16(y16.data(), y16.size(), operand_bf16, y_out);
    if (x_out && cudaMemcpy2D(x_out, hb, d_x, in_stride * 4, hb, rows, cudaMemcpyDeviceToHost) != cudaSuccess) { set_err("debug_layernorm: copy back x"); return 6; }
    return 0;
}

int clip_b200_debug_assemble_preln(const float* patch, const float* class_embd, const float* pos, int B, int T, int h, float eps,
                                   const float* gamma, const float* beta, float* x_out) {
    g_err.clear();
    if (B <= 0 || T < 2 || h <= 0 || h % 4) { set_err("debug_assemble_preln: bad shape"); return 1; }
    HookScratch s;
    const size_t hb = (size_t)h * 4, np = (size_t)B * (T - 1);
    float* d_patch = (float*)s.alloc(np * hb, 0, patch, np * hb);
    float* d_cls = (float*)s.alloc(hb, 0, class_embd, hb);
    float* d_pos = (float*)s.alloc((size_t)T * hb, 0, pos, (size_t)T * hb);
    float* d_g = (float*)s.alloc(hb, 0, gamma, hb);
    float* d_b = (float*)s.alloc(hb, 0, beta, hb);
    float* d_x = (float*)s.alloc((size_t)B * T * hb, 0xff);
    if (!s.ok) return 3;
    launch_assemble_preln(d_patch, d_cls, d_pos, B, T, h, eps, d_g, d_b, d_x, s.st);
    if (!s.finish("assemble_preln")) return 5;
    return s.copy_back(x_out, d_x, (size_t)B * T * hb) ? 0 : 6;
}

int clip_b200_debug_im2col(const float* pixels, int B, int S, int P, int kpad, float* out) {
    g_err.clear();
    if (B <= 0 || P <= 0 || S % P || kpad < 3 * P * P) { set_err("debug_im2col: bad shape"); return 1; }
    HookScratch s;
    const size_t pb = (size_t)B * S * S * 3 * 4, n = (size_t)B * (S / P) * (S / P) * kpad;
    float* d_px = (float*)s.alloc(pb, 0, pixels, pb);
    uint16_t* d_out = (uint16_t*)s.alloc(n * 2, 0xff);
    if (!s.ok) return 3;
    launch_im2col(d_px, B, S, S, P, kpad, d_out, s.st);
    if (!s.finish("im2col")) return 5;
    std::vector<uint16_t> o16(n);
    if (!s.copy_back(o16.data(), d_out, n * 2)) return 6;
    from16(o16.data(), n, 0, out);
    return 0;
}

int clip_b200_debug_im2col_hw(const float* pixels, int B, int H, int W, int P, int kpad, float* out) {
    g_err.clear();
    if (B <= 0 || P <= 0 || H <= 0 || W <= 0 || H % P || W % P || kpad < 3 * P * P) { set_err("debug_im2col_hw: bad shape"); return 1; }
    HookScratch s;
    const size_t pb = (size_t)B * H * W * 3 * 4, n = (size_t)B * (H / P) * (W / P) * kpad;
    float* d_px = (float*)s.alloc(pb, 0, pixels, pb);
    uint16_t* d_out = (uint16_t*)s.alloc(n * 2, 0xff);
    if (!s.ok) return 3;
    launch_im2col(d_px, B, H, W, P, kpad, d_out, s.st);
    if (!s.finish("im2col")) return 5;
    std::vector<uint16_t> o16(n);
    if (!s.copy_back(o16.data(), d_out, n * 2)) return 6;
    from16(o16.data(), n, 0, out);
    return 0;
}

int clip_b200_debug_pos_resample(const float* table, int g, int h, int gh, int gw, float* out) {
    g_err.clear();
    if (g <= 0 || h <= 0 || gh <= 0 || gw <= 0) { set_err("debug_pos_resample: bad shape"); return 1; }
    HookScratch s;
    const size_t tb = (size_t)g * g * h * 4, ob = (size_t)gh * gw * h * 4;
    float* d_t = (float*)s.alloc(tb, 0, table, tb);
    float* d_out = (float*)s.alloc(ob, 0xff);
    if (!s.ok) return 3;
    launch_pos_resample(d_t, g, h, gh, gw, d_out, s.st);
    if (!s.finish("pos_resample")) return 5;
    return s.copy_back(out, d_out, ob) ? 0 : 6;
}

int clip_b200_debug_text_embed(const int32_t* ids, const float* tok, const float* pos, int nseq, int T, int h, int n_vocab, float* x_out) {
    g_err.clear();
    if (nseq <= 0 || T <= 0 || h <= 0 || h % 4 || n_vocab <= 0) { set_err("debug_text_embed: bad shape"); return 1; }
    HookScratch s;
    const size_t hb = (size_t)h * 4, rows = (size_t)nseq * T;
    int32_t* d_ids = (int32_t*)s.alloc(rows * 4, 0, ids, rows * 4);
    float* d_tok = (float*)s.alloc((size_t)n_vocab * hb, 0, tok, (size_t)n_vocab * hb);
    float* d_pos = (float*)s.alloc((size_t)T * hb, 0, pos, (size_t)T * hb);
    float* d_x = (float*)s.alloc(rows * hb, 0xff);
    if (!s.ok) return 3;
    launch_text_embed(d_ids, d_tok, d_pos, nseq, T, h, n_vocab, d_x, s.st);
    if (!s.finish("text_embed")) return 5;
    return s.copy_back(x_out, d_x, rows * hb) ? 0 : 6;
}

int clip_b200_debug_gather_rows(const float* src, int src_rows, int rows, int h, int stride_rows, const int32_t* offs,
                                const float* delta, int operand_bf16, float* out) {
    g_err.clear();
    if (src_rows <= 0 || rows <= 0 || h <= 0 || h % 4) { set_err("debug_gather_rows: bad shape"); return 1; }
    for (int r = 0; r < rows; r++) {
        const long long i = (long long)r * stride_rows + (offs ? offs[r] : 0);
        if (i < 0 || i >= src_rows) { set_err("debug_gather_rows: row index out of range"); return 1; }
    }
    HookScratch s;
    const size_t hb = (size_t)h * 4, sn = (size_t)src_rows * h;
    float* d_src = (float*)s.alloc(sn * 4, 0, src, sn * 4);
    int32_t* d_offs = offs ? (int32_t*)s.alloc((size_t)rows * 4, 0, offs, (size_t)rows * 4) : nullptr;
    uint16_t* d_delta = nullptr;
    if (delta) {
        const std::vector<uint16_t> d16 = to16(delta, sn, operand_bf16);
        d_delta = (uint16_t*)s.alloc(sn * 2, 0, d16.data(), sn * 2);
    }
    float* d_out = (float*)s.alloc((size_t)rows * hb, 0xff);
    if (!s.ok) return 3;
    launch_gather_rows(d_src, d_out, rows, h, stride_rows, d_offs, d_delta, operand_bf16, s.st);
    if (!s.finish("gather_rows")) return 5;
    return s.copy_back(out, d_out, (size_t)rows * hb) ? 0 : 6;
}

int clip_b200_debug_l2norm(const float* v, int rows, int d, int normalize, float* out) {
    g_err.clear();
    if (rows <= 0 || d <= 0) { set_err("debug_l2norm: bad shape"); return 1; }
    HookScratch s;
    const size_t n = (size_t)rows * d * 4;
    float* d_v = (float*)s.alloc(n, 0, v, n);
    float* d_out = (float*)s.alloc(n, 0xff);
    if (!s.ok) return 3;
    launch_l2norm(d_v, d_out, rows, d, normalize, s.st);
    if (!s.finish("l2norm")) return 5;
    return s.copy_back(out, d_out, n) ? 0 : 6;
}

int clip_b200_debug_fill_last(const int32_t* lens, int n, int seq_len, int32_t* last) {
    g_err.clear();
    if (n <= 0 || seq_len <= 0) { set_err("debug_fill_last: bad shape"); return 1; }
    HookScratch s;
    int32_t* d_lens = lens ? (int32_t*)s.alloc((size_t)n * 4, 0, lens, (size_t)n * 4) : nullptr;
    int32_t* d_last = (int32_t*)s.alloc((size_t)n * 4, 0xff);
    if (!s.ok) return 3;
    launch_fill_last(d_lens, d_last, n, seq_len, s.st);
    if (!s.finish("fill_last")) return 5;
    return s.copy_back(last, d_last, (size_t)n * 4) ? 0 : 6;
}

int clip_b200_debug_token_rows(int n, int T, int h, size_t in_stride, int no_cls, float eps, const float* x, const float* gamma,
                               const float* beta, int out_type, void* out) {
    g_err.clear();
    const int skip = no_cls ? 1 : 0;
    if (n <= 0 || T <= skip || h <= 0 || h % 4 || h > 2048 || in_stride < (size_t)h || in_stride % 4 || out_type < 0 || out_type > 2) {
        set_err("debug_token_rows: bad shape");
        return 1;
    }
    HookScratch s;
    const size_t rows = (size_t)n * T, hb = (size_t)h * 4, span = (rows - 1) * in_stride + h;
    const size_t out_bytes = (size_t)n * (T - skip) * h * (out_type == 0 ? 4 : 2);
    float* d_x = (float*)s.alloc(span * 4, 0xff);
    float* d_g = gamma ? (float*)s.alloc(hb, 0, gamma, hb) : nullptr;
    float* d_b = gamma ? (float*)s.alloc(hb, 0, beta, hb) : nullptr;
    void* d_out = s.alloc(out_bytes, 0xff);
    if (s.ok && cudaMemcpy2D(d_x, in_stride * 4, x, hb, hb, rows, cudaMemcpyHostToDevice) != cudaSuccess) { set_err("debug_token_rows: upload"); return 3; }
    if (!s.ok) return 3;
    launch_token_rows(d_x, in_stride, n, T, skip, h, d_g, d_b, eps, out_type, d_out, s.st);
    if (!s.finish("token_rows")) return 5;
    return s.copy_back(out, d_out, out_bytes) ? 0 : 6;
}

// K9 on qkv (fp32 host [nseq*T, 3*H*head_dim], rounded to the operand type and padded on the way in; one 128-row box of poisoned
// rows follows the last sequence, as in clip_b200_debug_attention_hd).  Poisoned guard bytes follow the output.
int clip_b200_debug_attention_probs(int operand_bf16, int nseq, int T, int H, int head_dim, int causal, int cls_row, int out_type,
                                    const float* qkv, void* out) {
    g_err.clear();
    if ((head_dim != 64 && head_dim != 80 && head_dim != 104) || nseq <= 0 || T <= 0 || H <= 0 || out_type < 0 || out_type > 2 || !qkv || !out) {
        set_err("debug_attention_probs: bad arguments (head_dim 64 or 80, or 104; positive sizes, out_type 0..2)");
        return 2;
    }
    HookScratch s;
    if (s.ok && attention_tc_init() != cudaSuccess) { set_err("attention_tc_init failed"); return 1; }
    const size_t rows = (size_t)nseq * T, cols = (size_t)3 * H * qkv_head_cols(head_dim), guard = 4096;
    const size_t out_bytes = (size_t)nseq * H * (cls_row ? 1 : T) * T * (out_type == 0 ? 4 : 2);
    const std::vector<uint16_t> q16 = qkv_to16_padded(qkv, rows, H, head_dim, operand_bf16);
    void* d_qkv = s.alloc((rows + 128) * cols * 2, 0xff, q16.data(), q16.size() * 2);
    uint8_t* d_out = (uint8_t*)s.alloc(out_bytes + guard, 0xff);
    if (!s.ok) return 3;
    const cudaError_t e = launch_attention_probs(d_qkv, d_out, out_type, nseq, T, H, head_dim, causal ? 1 : 0, cls_row ? 1 : 0, operand_bf16 ? 1 : 0, s.st);
    if (e != cudaSuccess) { set_err(std::string("attention_probs launch: ") + cudaGetErrorString(e)); return 4; }
    if (!s.finish("attention_probs")) return 4;
    std::vector<uint8_t> g(guard);
    if (!s.copy_back(g.data(), d_out + out_bytes, guard)) return 6;
    if (std::any_of(g.begin(), g.end(), [](uint8_t b) { return b != 0xFF; })) { set_err("attention_probs wrote past the output"); return 5; }
    return s.copy_back(out, d_out, out_bytes) ? 0 : 6;
}


// ---- CPU-only test hooks (no context / GPU needed) ----------------------------------------------------------
// The loader's QKV row padding (pad_head_rows) on one fused part or the whole Q | K | V: src holds 3*H*dh rows of a [*, K] weight of
// ggml type qtype (0 f32, 1 f16, or a block type; qtype 0 with K = 1 is a bias), out receives 3*H*dhp rows.  dhp must be
// qkv_head_cols(dh) or any other value >= dh.
int clip_b200_debug_pad_qkv(int qtype, int H, int dh, int dhp, int K, const void* src, void* out) {
    g_err.clear();
    const size_t bb = qtype == 0 ? 4 : qtype == 1 ? 2 : wpack_ggml_block_bytes(qtype), be = qtype <= 1 ? 1 : 32;
    if (H <= 0 || dh <= 0 || dhp < dh || K <= 0 || !bb || K % be || !src || !out) { set_err("debug_pad_qkv: bad arguments"); return 1; }
    const size_t rb = (size_t)K / be * bb;
    return pad_head_rows((const uint8_t*)src, rb, (int64_t)3 * H * dh, dh, dhp, (uint8_t*)out) ? 0 : 1;
}

// ranks-mode rendezvous of the NCCL unique id (dist.cpp) without a GPU: rank 0 publishes, the others read the same 128 bytes
int clip_b200_debug_rendezvous(int rank, int world, const char* path, void* out128) {
    std::string e;
    if (!dist_rendezvous_id(rank, world, path, out128, e)) { set_err(e); return 1; }
    return 0;
}
void clip_b200_debug_shard_bounds(size_t n, int r, int w, size_t* lo, size_t* hi) { shard_bounds(n, r, w, *lo, *hi); }
int clip_b200_debug_repack_roundtrip(int qtype, const void* rows, int N, int K) {
    const size_t raw = (size_t)N * (K / 32) * wpack_ggml_block_bytes(qtype);
    std::vector<uint8_t> packed(wpack_total_bytes(qtype, N, K)), back(raw);
    if (!wpack_repack(qtype, (const uint8_t*)rows, N, K, packed.data())) return 1;
    if (!wpack_unpack(qtype, packed.data(), N, K, back.data())) return 2;
    return memcmp(back.data(), rows, raw) == 0 ? 0 : 3;
}
int clip_b200_debug_tokenize(const char* gguf_path, const char* text, int32_t* out, int cap) {
    GgufFile g;
    std::string err;
    if (!g.parse(gguf_path, err)) { set_err(err); return -1; }
    const GgufKV* tk = g.find("tokenizer.ggml.tokens");
    if (!tk) { set_err("no vocabulary"); return -1; }
    Vocab v;
    for (size_t i = 0; i < tk->strs.size(); i++) v.token_to_id[tk->strs[i]] = (int32_t)i;
    std::vector<int32_t> ids = tokenize(v, text);
    for (size_t i = 0; i < ids.size() && (int)i < cap; i++) out[i] = ids[i];
    return (int)ids.size();
}
int clip_b200_debug_preprocess(const uint8_t* rgb, int nx, int ny, int out_size, const float* mean, const float* stdv, float* out) {
    return preprocess_image(rgb, nx, ny, out_size, mean, stdv, out) ? 0 : 1;
}

// ---- ggml/ggml.h shim symbols (include/ggml/ggml.h) ---------------------------------------------------------
static std::chrono::steady_clock::time_point g_t0 = std::chrono::steady_clock::now();
void ggml_time_init(void) { g_t0 = std::chrono::steady_clock::now(); }
int64_t ggml_time_us(void) { return std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - g_t0).count(); }
int64_t ggml_time_ms(void) { return ggml_time_us() / 1000; }

}  // extern "C"
