// kernels.h -- host launchers of the non-GEMM kernels (kernels.cu, attention.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cb {

// K2 LayerNorm: y16[r, :] = ((x[r*in_stride ...] - mean) * rstd) * gamma + beta   (reference: ggml.c:10796-10845,
// affine clip.cpp:1071-1074).  x fp32, row r starts at x + r*in_stride.  One warp per row.
// If delta16 != NULL the kernel first applies a pending residual branch: x[r,:] += delta16[r,:] (written back in fp32); the model
// schedule passes NULL (round 2: the GEMM epilogues add into x).
void launch_layernorm(float* x, size_t in_stride, int rows, int h, float eps, const float* gamma, const float* beta,
                      const void* delta16, void* y16, int bf16, cudaStream_t st);

// K7 token rows: for each of n items, rows skip .. T-1 of x (item i's row t at x + (i*T + t)*in_stride) -> out [n*(T-skip), h],
// contiguous, as out_type (0 fp32, 1 fp16, 2 bf16; round to nearest even).  gamma != NULL applies LayerNorm (gamma, beta, eps) first,
// with K2's arithmetic: the 16-bit output of the operand type equals launch_layernorm's bit for bit.  h % 4 == 0, h <= 2048.
void launch_token_rows(const float* x, size_t in_stride, int n, int T, int skip, int h, const float* gamma, const float* beta, float eps,
                       int out_type, void* out, cudaStream_t st);

// K0a im2col for the stride-P patch conv: pixels NHWC f32 [B,H,W,3] -> fp16 [B*Np, kpad], Np = (H/P)(W/P) patches in row-major
// grid order, k = c*P*P + ky*P + kx, zero padded to kpad (reference conv_2d im2col, ggml.c:13595-13631; pixel -> fp16 rounding
// ggml.c:13623).  The model's own size passes H = W = image_size.
void launch_im2col(const float* pixels, int B, int H, int W, int P, int kpad, void* patches16, cudaStream_t st);

// K8 position-table resample (HF interpolate_pos_encoding): table fp32 [g*g, h] (the patch rows of a g x g grid) -> out fp32
// [gh*gw, h], torch's upsample_bicubic2d (A = -0.75, align_corners = False, taps clamped to the edge) evaluated in fp64 without
// contraction, horizontal pass first, rounded once to fp32.  Torch evaluates the same formula in fp32, so the two agree within
// the rounding of torch's fp32 coordinates, weights and sums (tests/test_pos_resample.py), not bit for bit.
void launch_pos_resample(const float* table, int g, int h, int gh, int gw, float* out, cudaStream_t st);

// K4v assemble + pre-LN: x[b,t,:] = LN( (t==0 ? class_embd : patch[b*Np+t-1,:]) + pos[t,:] ) * g + b  -> fp32
// (clip.cpp:1315-1339)
void launch_assemble_preln(const float* patch, const float* class_embd, const float* pos, int B, int T, int h, float eps,
                           const float* gamma, const float* beta, float* x, cudaStream_t st);

// One image of a mixed-size pass (the clip_b200_*_mixed calls): its rows are packed back to back with no padding.
struct MixedImage {
    long long px;          // its first pixel float, from the pass's pixel base (NHWC f32, gh*P x gw*P x 3)
    const float* pos;      // its position table [gh*gw + 1, h]
    int row, prow;         // its first token row (CLS) and first patch row in the pass
    int gh, gw;            // its patch grid
};
// K0a and K4v over the n images of a mixed-size pass (im: device descriptors in row order): patches [prows, kpad] and x [rows, h]
// hold each image's rows at its own offsets, bit for bit what launch_im2col / launch_assemble_preln write for that image alone.
void launch_im2col_mixed(const float* pixels, const MixedImage* im, int n, int prows, int P, int kpad, void* patches16, cudaStream_t st);
void launch_assemble_mixed(const float* patch, const float* class_embd, const MixedImage* im, int n, int rows, int h, float eps,
                           const float* gamma, const float* beta, float* x, cudaStream_t st);

// K4t text embed: x[s*T+t,:] = tok[ids[s*T+t],:] + pos[t,:]   (clip.cpp:1059-1061), tables fp32 (dequantised at load)
void launch_text_embed(const int32_t* ids, const float* tok, const float* pos, int nseq, int T, int h, int n_vocab, float* x,
                       cudaStream_t st);
// K4t over the nseq sequences of a packed pass (the *_packed text calls): row r of sequence s = rows off[s] .. off[s + 1] - 1 (off:
// device, nseq + 1 entries, off[nseq] = rows) is tok[ids[r]] + pos[r - off[s]], bit for bit what launch_text_embed writes for s alone
void launch_text_embed_packed(const int32_t* ids, const float* tok, const float* pos, const int* off, int nseq, int rows, int h, int n_vocab,
                              float* x, cudaStream_t st);

// K3 attention: softmax(Q K^T [causal]) V per (sequence, head); qkv 16-bit [nseq*T, 3*H*dh] (Q pre-scaled by 1/sqrt(dh)),
// out 16-bit [nseq*T, H*dh].  (clip.cpp:1100-1108, 1382-1388)
// launch_attention: warp-level mma.sync kernel (attention.cu), head_dim 64 only, kept as the cross-check of the wgmma kernel
// (CLIP_B200_ATTN=legacy).
void launch_attention(const void* qkv16, void* out16, int nseq, int T, int H, int causal, int bf16, cudaStream_t st);

// Columns a head of head_dim dh takes in the fused QKV matrix: dh, except 104 (ViT-bigG/14), which the loader pads to 112 with 8
// exactly-zero columns per head so that the attention kernels' pieces (64 + 32 + 16 columns) never reach into the next head.
constexpr int qkv_head_cols(int dh) { return dh == 104 ? 112 : dh; }

// K3 on wgmma (attention_tc.cu): head_dim dh = 64, 80 or 104 (anything else: cudaErrorInvalidValue), a persistent grid over
// 64-row query groups, online softmax over 128-key blocks (64-key at 104), any T.  qkv16 is [nseq*T, 3*H*qkv_head_cols(dh)]; out
// stays [nseq*T, H*dh].  The Q / K / V boxes come from per-launch 3-D TMA views [sequence][token][column] of qkv16 (zero fill past
// each sequence's T tokens).
cudaError_t attention_tc_init();
cudaError_t launch_attention_tc(const void* qkv16, void* out16, int nseq, int T, int H, int dh, int causal, int bf16, cudaStream_t st);
// K3 on nseq packed sequences of different lengths: qkv16 [rows, 3*H*qkv_head_cols(dh)], out16 [rows, H*dh], sequence s = rows
// off[s] .. off[s + 1] - 1.  d_seq (device): off [nseq + 1] (off[0] = 0, off[nseq] = rows), then grp [nseq + 1], the prefix sums of
// ceil(len_s / 64); groups = grp[nseq].  causal (the text tower): head_dim 64 only.  Each sequence's rows equal, bit for bit, a
// launch_attention_tc of that sequence alone with the same causal.
cudaError_t launch_attention_tc_varlen(const void* qkv16, void* out16, int rows, int nseq, const int* d_seq, int groups, int H, int dh, int causal,
                                      int bf16, cudaStream_t st);

// K9 attention probabilities (attention_tc.cu): the softmax(Q K^T [causal]) K3 computes internally, from the same qkv16, written out:
// out [nseq, H, R, T] of elem_type (0 fp32, 1 fp16, 2 bf16: RNE of the fp32 value), R = T, or 1 with cls_only (query row 0 alone).
// Masked keys are +0.  Any T, head_dim 64, 80 or 104 (qkv16 laid out as for K3); out needs only the element type's alignment.
cudaError_t launch_attention_probs(const void* qkv16, void* out, int elem_type, int nseq, int T, int H, int dh, int causal, int cls_only,
                                   int bf16, cudaStream_t st);

// K5 head tail: out[r,:] = normalize ? v / sqrt(sum v^2) : v    (clip.cpp:1163-1166, 1448-1455)
void launch_l2norm(const float* v, float* out, int rows, int d, int normalize, cudaStream_t st);

// gather rows: dst[r,:] = src[idx(r),:] where idx(r) = r*stride_rows + offs[r] (offs may be null -> 0)
void launch_gather_rows(const float* src, float* dst, int rows, int h, int stride_rows, const int32_t* offs, const void* delta16,
                        int bf16, cudaStream_t st);   // dst = src[idx] (+ delta16[idx])

// text: last[i] = clamp(lens ? lens[i] : seq_len, 1, seq_len) - 1  (index of the EOT row, clip.cpp:1154-1155), on the device
void launch_fill_last(const int32_t* lens, int32_t* last, int n, int seq_len, cudaStream_t st);

// ---- scoring (search.cu) ----------------------------------------------------------------------------------------------
// S[i, j] = <a_i, b_j> fp32, one sequential fmaf chain per element (clip_similarity_score, clip.cpp:1525-1532); row stride lds
void launch_similarity(const float* a, const float* b, float* s, int na, int nb, int d, size_t lds, cudaStream_t st);
// in place p = (exp(s) + 1e-9) / sum with softmax_with_sorting's rounding points (clip.cpp:1599-1607)
void launch_softmax_ref(float* logits, int rows, int cols, size_t ld, cudaStream_t st);
// one top-k stage: every slice of topk_slice() candidates of a row is sorted (value desc, index asc) and its best kk are written to
// out[row, out_off + slice * kk ...]; in_idx == nullptr: candidate j has index idx_base + j
int topk_slice();
void launch_topk_stage(const float* vals, const int* in_idx, size_t ld, int rows, int n, int idx_base, int kk, float* out_v, int* out_i,
                       size_t out_ld, int out_off, cudaStream_t st);

// K10 nearest-neighbour search (search.cu): q [nq, dim] x db [ndb, dim] of operand kind op, 16-byte aligned, dim <= 2048.
//   F16, BF16  dim % 8 == 0; qs and xs are unused (NULL)
//   S8         int8 codes with f32 scales qs [nq] and xs [ndb], also 16-byte aligned, dim % 16 == 0;
//              score = fp32(fp32(float(exact int32 dot) * qs) * xs)
// Writes each query's best kk (<= 1024) per database partition, sorted, to out[query, partition * kk ...] (row stride out_ld >=
// parts * kk); padding entries are (-inf, INT_MAX).  The plan fixes the query tile (8 nt queries), the partitions and the scratch
// `buf` of buf_entries (value, index) pairs the launch needs.
enum class KOp { F16, BF16, S8, F16_IVF, BF16_IVF };      // the IVF instances: launch_knn_ivf only
struct KnnPlan {
    int nt, parts, rows_per_part, grid, cap;
    size_t buf_entries;
};
KnnPlan knn_plan(int nq, int ndb, int kk, int sms);
cudaError_t launch_knn(KOp op, const void* q, const float* qs, int nq, const void* db, const float* xs, int ndb, int dim, int kk,
                       const KnnPlan& pl, void* buf, float* out_v, int* out_i, size_t out_ld, cudaStream_t st);
// K10's IVF instances (kernel class 11): CTA u runs unit units[u], pairs p0 .. p0 + np - 1 (rows of pq [npairs, dim], the gathered
// query of each (query, probed list) pair) against stored rows row_begin .. row_end - 1 of rows [ndb, dim], all in one list.  Pair
// p's best kk of the unit go, sorted, to out[slot[p] + range * kk ...] with each row's original index ids[stored position]; padding
// is (-inf, INT_MAX).  Query tile 8 nt; scratch `buf` of nunits * 8 nt * (kk + 256) (value, index) pairs.
struct IvfUnit { int p0, np, row_begin, row_end, range; };
cudaError_t launch_knn_ivf(bool bf, const void* pq, int npairs, const void* rows, int ndb, int dim, int kk, int nt, const IvfUnit* units,
                           int nunits, const size_t* slot, const int* ids, void* buf, float* out_v, int* out_i, cudaStream_t st);
int knn_tile_rows();                                                    // K10's KB: rows per tile
// dst[p] = src[idx[p]], p < n, rows of dim 16-bit elements (dim % 8 == 0), 16-byte aligned; 64-bit offsets
void launch_gather_rows16(const void* src, const int* idx, size_t n, int dim, void* dst, cudaStream_t st);
// (v, i)[0 .. n) = (-inf, INT_MAX): the candidate matrix's unused runs
void launch_fill_cand(float* v, int* i, size_t n, cudaStream_t st);
// one k-means update (clip_b200_ivf_train_16's rule): x [n, dim] 16-bit (bf: bf16) in list order through ids; chunks[c] = (begin, end)
// positions in ids, chunk_begin[l] .. chunk_begin[l + 1] - 1 the chunks of list l, offsets [n_lists + 1]; part [nchunks, dim] fp64
// scratch.  Rewrites cent [n_lists, dim] in place, keeping the centroid of an empty list or of a zero mean.
void launch_ivf_update(bool bf, const void* x, int dim, const int* ids, const int2* chunks, int nchunks, const int* chunk_begin,
                       const int* offsets, int n_lists, double* part, void* cent, cudaStream_t st);
// IVF-PQ (clip_b200_ivfpq_*'s rule, clip_b200.h).  x and cent are 16-bit (bf: bf16) [n, dim] and [n_lists, dim]; lists [n] the list
// of each row; books f32 [m, 256, dim / m]; codes uint8 [n, m], 16-byte aligned.  64-bit offsets throughout.
// codes of each row's residual x - cent[list] (kernel class 14)
cudaError_t launch_pq_encode(bool bf, const void* x, size_t n, int dim, int m, const int* lists, const void* cent, const float* books,
                             void* codes, cudaStream_t st);
// initial codebooks: codeword i of every subspace from the residual of row floor(i n / 256), n >= 256
void launch_pq_init(bool bf, const void* x, size_t n, int dim, int m, const int* lists, const void* cent, float* books, cudaStream_t st);
// one codebook update: ids [m][n] the rows of each subspace grouped by code (stable), chunks[c] = positions [begin, end) in that flat
// array, chunk_begin [m * 256 + 1] the chunks of codeword s * 256 + k, count [m * 256] its members, part [nchunks, dim / m] fp64
// scratch.  Rewrites each non-empty codeword with the fp64 mean of its members' residuals, rounded once to f32.
void launch_pq_update(bool bf, const void* x, size_t n, int dim, int m, const int* lists, const void* cent, const int* ids,
                      const longlong2* chunks, int nchunks, const int* chunk_begin, const int* count, double* part, float* books,
                      cudaStream_t st);
// lookup tables [nq, m, 256] f32 of queries q [nq, dim] 16-bit (kernel class 14)
cudaError_t launch_pq_tables(bool bf, const void* q, int nq, int dim, int m, const float* books, float* tables, cudaStream_t st);
// K13, the ADC scan (kernel class 13): CTA u runs unit units[u] of K10's IVF plan over stored codes [ndb, m].  Pair p (query
// pair_q[p], coarse score pscore[p]) scores a row v = pscore[p] + T[s][code_s] for s in order, T = tables[pair_q[p]]; its best kk of
// the unit go to out as launch_knn_ivf writes them.  Scratch `buf` of nunits * adc_cap(kk) (value, index) pairs.
size_t adc_cap(int kk);
cudaError_t launch_adc(const void* codes, int ndb, int m, const float* tables, const float* pscore, const int* pair_q, int kk,
                       const IvfUnit* units, int nunits, const size_t* slot, const int* ids, void* buf, float* out_v, int* out_i,
                       cudaStream_t st);
// Q8 quantiser: x [n, dim] f32 -> codes [n, dim] int8 and scales [n] f32 by the rule of clip_b200_rows_to_int8 (clip_b200.h).
// dim % 16 == 0, dim <= 2048, 16-byte aligned pointers; 64-bit offsets, so n * dim may pass 2^32.
void launch_rows_to_int8(const float* x, int n, int dim, void* codes, float* scales, cudaStream_t st);

// K11 Hamming top-k (search.cu): q [nq, dim / 8] and db [ndb, dim / 8] bytes of sign bits (clip_b200_rows_to_binary), 16-byte
// aligned, dim % 128 == 0, dim <= 2048; score = dim - 2 popc(q ^ x), exact.  Output as launch_knn's; the plan is knn_plan's on one or
// two CTAs an SM (knn_b1_plan).
KnnPlan knn_b1_plan(int nq, int ndb, int kk, int sms);
cudaError_t launch_knn_b1(const void* q, int nq, const void* db, int ndb, int dim, int kk, const KnnPlan& pl, void* buf, float* out_v,
                          int* out_i, size_t out_ld, cudaStream_t st);
// K12 rescore (search.cu): per query, the distinct candidates of cand [nq, n_cand] (device) in [0, ndb), scored by one fmaf chain over
// q [nq, dim] x db [ndb, dim] of type (0 f32, 1 f16, 2 bf16), 16-byte aligned, dim % 8 == 0, dim <= 2048, n_cand <= 2048; the best
// kk (<= n_cand) to out [nq, out_ld], sorted, padded with (-inf, -1).
cudaError_t launch_rescore(int type, const void* q, int nq, const void* db, int ndb, int dim, const int* cand, int n_cand, int kk,
                           float* out_v, int* out_i, size_t out_ld, cudaStream_t st);
// B1 quantiser: x [n, dim] f32 (center [dim] f32 or NULL) -> bits [n, dim / 8], bit i = x_i > center_i, LSB first; dim % 128 == 0,
// dim <= 2048, 16-byte aligned; 64-bit offsets.
void launch_rows_to_binary(const float* x, int n, int dim, const float* center, void* bits, cudaStream_t st);

}  // namespace cb
struct clip_ctx;
struct clip_image_u8;
#include <string>
namespace cb {
// N1 device-side preprocess (preprocess.cu): raw u8 images -> [nb, S, S, 3] fp32 crops, bit-identical to host_ops.cpp: preprocess_image
bool preprocess_device(clip_ctx* c, const clip_image_u8* imgs, int nb, int buf, float* d_pixels, cudaStream_t copy_st, cudaEvent_t copied,
                       cudaStream_t st, std::string& err);
void preprocess_release(clip_ctx* c);

// DEBUG ONLY (tests / CLIP_B200_DEBUG_NAIVE=1): scalar GEMM straight from ggml-format rows on the device.
void launch_naive_gemm(const void* x16, int x_bf16, const void* w_ggml, int qtype, const float* bias, void* out, int M, int N,
                       int K, int ldo, int epi, int out_bf16, int scale_cols, float scale, cudaStream_t st);

}  // namespace cb
