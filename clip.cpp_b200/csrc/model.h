// model.h -- device-resident model, workspaces and the static kernel schedule of the two towers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <string>
#include <vector>

#include "../../include/clip_b200.h"
#include "dist.h"
#include "gemm.h"
#include "host_ops.h"

namespace cb {

struct Linear {              // one GEMM weight, [N features, K]
    int qtype = 1;           // QT_F16 or a quantized type (f32 files are rounded to f16 at load)
    int N = 0, K = 0;
    uint8_t* d_w = nullptr;  // packed blocks (wpack.h) or fp16 [N, K]
    TmaMap w_map;            // QT_F16 only
    float* d_bias = nullptr;
    uint8_t* d_raw = nullptr;   // ggml-format rows, only uploaded when CLIP_B200_DEBUG_NAIVE=1
};

struct Layer {
    float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
    Linear qkv, out, fc1, fc2;
};

struct Workspace {
    int cap_items = 0, T = 0, cap_rows = 0;
    float* x = nullptr;          // residual stream fp32 [rows, h]
    uint16_t* a = nullptr;       // LN output / attention output 16-bit [rows, h]
    uint16_t* qkv = nullptr;     // [rows, 3h]
    uint16_t* g = nullptr;       // [rows, ff]
    uint16_t* sel16 = nullptr;   // CLS / EOT rows after post-LN [items, h]
    float* sel32 = nullptr;      // gathered EOT rows fp32 [items, h] (text)
    float* proj32 = nullptr;     // [items, d]
    // vision only
    float* pixels[2] = {nullptr, nullptr};   // staging for host inputs [items, S, S, 3]
    uint16_t* patches = nullptr;             // fp16 [items*Np, kpad]
    float* patch32 = nullptr;                // [items*Np, h]
    // text only
    int32_t* ids = nullptr;
    int32_t* last = nullptr;     // index of the EOT row per sequence (len - 1)
    TmaMap map_a, map_g, map_patches, map_sel;
};

struct Tower {
    bool present = false;
    int hidden = 0, ff = 0, heads = 0, layers = 0, proj = 0;
    float eps = 1e-5f;
    std::vector<Layer> L;
    float *post_g = nullptr, *post_b = nullptr;
    Linear proj_w;
    // vision
    int image_size = 0, patch = 0, n_patches = 0, T = 0, kpad = 0;
    Linear patch_w;
    float *class_embd = nullptr, *pos = nullptr, *pre_g = nullptr, *pre_b = nullptr;
    // text
    int n_vocab = 0, n_ctx = 0;
    float* tok = nullptr;
    Workspace ws;
    int micro_batch = 0;
};

struct ProfEvent { int kind; cudaEvent_t e0, e1; };

struct PreArena {                // staging of the device-side preprocess (preprocess.cu), one per pixel staging buffer
    uint8_t* h = nullptr;        // pinned: descriptors, tap tables, raw u8 pixels of one micro-batch
    uint8_t* d = nullptr;        // device copy of the blob
    size_t cap = 0, last_bytes = 0;
    float* d_tmp = nullptr;      // horizontally resized rows
    size_t tmp_cap = 0;          // in floats
};

}  // namespace cb

struct clip_ctx {
    bool has_text = false, has_vision = false, use_gelu = false;
    clip_text_hparams thp{};
    clip_vision_hparams vhp{};
    float image_mean[3] = {0, 0, 0}, image_std[3] = {1, 1, 1};
    cb::Vocab vocab;
    cb::Tower vis, txt;
    bool operand_bf16 = false;   // 16-bit activation / unpacked-weight type of the towers
    int device = 0, num_sms = 132;
    cudaStream_t stream = nullptr, copy_stream = nullptr;
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_consumed[2] = {nullptr, nullptr}, ev_t0 = nullptr, ev_t1 = nullptr;
    std::vector<void*> allocs;   // every device allocation, freed in clip_free
    float* d_out = nullptr;      // result staging [n, d]
    size_t d_out_cap = 0;
    bool debug_naive = false, profile = false, attn_tc = true;
    uint64_t launches = 0;
    float last_ms = 0.f;
    std::vector<cb::ProfEvent> prof;
    std::vector<cudaEvent_t> ev_pool;
    cb::PreArena pre[2];
    std::mutex mu;
    cudaEvent_t marks[4] = {nullptr, nullptr, nullptr, nullptr};   // clip_b200_mark stopwatch slots (per context = per device)
    // pinned staging for PAGEABLE caller buffers (clip_image_preprocess hands out new float[]): filled by host threads, one async
    // H2D per micro-batch -- pageable cudaMemcpyAsync would be staged synchronously by the driver, image by image
    float* h_stage[2] = {nullptr, nullptr};
    size_t h_stage_cap = 0;                 // floats per buffer
    // host *_tokens calls: the two-slot ring their rows leave the device through (RowRing in api.cu), grow-only; h_ring is the
    // pinned bounce for pageable caller buffers.  ev_ring_rows[s]: K7 has filled slot s; ev_ring_free[s]: its D2H has finished.
    char* d_ring = nullptr; size_t d_ring_cap = 0;
    char* h_ring = nullptr; size_t h_ring_cap = 0;
    cudaEvent_t ev_ring_rows[2] = {nullptr, nullptr}, ev_ring_free[2] = {nullptr, nullptr};
    // scoring scratch (search.cu), grow-only
    float* d_logits = nullptr; size_t d_logits_cap = 0;
    float* d_cand_v[2] = {nullptr, nullptr}; int* d_cand_i[2] = {nullptr, nullptr}; size_t d_cand_cap = 0;
    uint32_t* d_knn = nullptr; size_t d_knn_cap = 0;    // clip_b200_topk_search_16: K10's per-CTA candidate buffers, 2 words per entry
    int* d_rcand = nullptr; size_t d_rcand_cap = 0;     // clip_b200_topk_rescore: the candidates of one block of queries
    uint8_t* d_ivf = nullptr; size_t d_ivf_cap = 0;     // the clip_b200_ivf_* calls: host-planned tables and their scratch
    float* d_emb[2] = {nullptr, nullptr}; size_t d_emb_cap[2] = {0, 0};     // image / text embeddings kept on the device (zero-shot)
    // the last position table resampled for a non-native image size (*_hw calls): CLS row + gh*gw patch rows [T, h], grow-only
    float* pos_hw = nullptr; size_t pos_hw_cap = 0;
    int pos_gh = 0, pos_gw = 0;
    // the *_mixed calls: the position tables of every non-native grid of one call, back to back, and one pass's descriptors
    // (MixedImage, then K3's varlen table), both grow-only
    float* pos_mixed = nullptr; size_t pos_mixed_cap = 0;
    char* d_mixed = nullptr; size_t d_mixed_cap = 0;
    double* d_scalars = nullptr;            // 16 doubles for the tiny all-reduces (barrier, max over ranks)
    // ---- multi-GPU (dist.h) ------------------------------------------------------------------------------------------
    cb::DistComm dist;                      // this replica's NCCL communicator (ranks mode or devices mode); world == 1: none
    std::vector<clip_ctx*> replicas;        // devices mode, on the leader only: every replica, this context first
    bool is_replica = false;                // owned by a leader: never handed to the caller
};
