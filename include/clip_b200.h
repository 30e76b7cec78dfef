/*
 * clip_b200.h -- C ABI of libclip_b200.so, the H100-native drop-in for monatis/clip.cpp's encode path.
 *
 * PART 1 re-declares, symbol for symbol and struct for struct, the reference's public interface
 * (reference: /root/reference/clip.h:8-113, 22 extern "C" functions + 8 POD structs) so that the reference's
 * own callers -- examples/main.cpp, zsl.cpp, extract.cpp, simple.c, tests/benchmark.cpp, the ctypes binding in
 * examples/python_bindings/clip_cpp/clip.py -- link against this library unchanged.  Each declaration cites the
 * reference definition it replaces.  Differences in behaviour are limited to error handling: where the reference
 * throws a C++ exception through the C ABI, calls exit(1) or aborts (clip.cpp:85-115, 289-292, 1293), this
 * library returns false / NULL and records a message retrievable with clip_b200_last_error().
 *
 * PART 2 declares the additive entry points the reference lacks (batched text, device-resident buffers,
 * batched zero-shot scoring, measurement hooks).  Nothing in part 2 changes the meaning of part 1.
 *
 * Plain pointers and sizes only; no CUDA, torch or C++ types appear in any signature.
 */
#ifndef CLIP_B200_H
#define CLIP_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* =====================================================================================================
 * PART 1 -- the reference interface (clip.h)
 * ===================================================================================================== */

struct clip_ctx; /* opaque; clip.h:8 (definition clip.cpp:240-253) */

/* clip.h:14-23 -- text tower hyper-parameters, filled from GGUF KV (clip.cpp:464-477) */
struct clip_text_hparams {
    int32_t n_vocab;
    int32_t num_positions;
    int32_t hidden_size;
    int32_t n_intermediate;
    int32_t projection_dim;
    int32_t n_head;
    int32_t n_layer;
    float eps;
};

/* clip.h:25-34 -- vision tower hyper-parameters (clip.cpp:524-535) */
struct clip_vision_hparams {
    int32_t image_size;
    int32_t patch_size;
    int32_t hidden_size;
    int32_t n_intermediate;
    int32_t projection_dim;
    int32_t n_head;
    int32_t n_layer;
    float eps;
};

/* clip.h:36-40 -- token id sequence; `data` is allocated by clip_tokenize with new[] (clip.cpp:675) */
typedef int32_t clip_vocab_id;
struct clip_tokens {
    clip_vocab_id * data;
    size_t size;
};

/* clip.h:50-56 -- RGB uint8 image, interleaved */
struct clip_image_u8 {
    int nx;
    int ny;
    uint8_t * data;
    size_t size;
};

/* clip.h:58-64 -- RGB float32 image, NHWC (RGBRGB...), already mean/std normalised */
struct clip_image_f32 {
    int nx;
    int ny;
    float * data;
    size_t size;
};

/* clip.h:66-74 */
struct clip_image_u8_batch {
    struct clip_image_u8 * data;
    size_t size;
};
struct clip_image_f32_batch {
    struct clip_image_f32 * data;
    size_t size;
};

/* clip.h:42, clip.cpp:334-596.  Parses the GGUF file, uploads the weights to HBM (re-tiled for TMA) and returns a
 * context bound to one GPU (env CLIP_B200_DEVICE, default 0).  NULL on any failure -- missing key/tensor, unsupported
 * geometry, no CUDA device -- with the reason in clip_b200_last_error(); never throws, exits or falls back to a CPU. */
struct clip_ctx * clip_model_load(const char * fname, const int verbosity);

/* clip.h:44, clip.cpp:1010-1014 */
void clip_free(struct clip_ctx * ctx);

/* clip.h:46-47, clip.cpp:1846-1847 -- pointers into the context */
struct clip_text_hparams * clip_get_text_hparams(struct clip_ctx * ctx);
struct clip_vision_hparams * clip_get_vision_hparams(struct clip_ctx * ctx);

/* clip.h:76, clip.cpp:598-679 -- host side; same word split + greedy longest-match as the reference */
bool clip_tokenize(const struct clip_ctx * ctx, const char * text, struct clip_tokens * tokens);

/* clip.h:78-85, clip.cpp:681-707 */
struct clip_image_u8 * clip_image_u8_make();
struct clip_image_f32 * clip_image_f32_make();
void clip_image_u8_clean(struct clip_image_u8 * img);
void clip_image_f32_clean(struct clip_image_f32 * res);
void clip_image_u8_free(struct clip_image_u8 * img);
void clip_image_f32_free(struct clip_image_f32 * res);

/* clip.h:87, clip.cpp:709-726 -- the reference decodes with stb_image; this library has its own decoders for JPEG (Huffman baseline and
 * progressive, 8-bit, grey / YCbCr / RGB / CMYK / YCCK, any integer sampling ratio, restart intervals), PNG (every colour type and bit
 * depth, plain or Adam7-interlaced), BMP (palettes, 16 / 24 / 32 bits, no RLE), GIF (first frame) and binary PGM / PPM.  Each returns the same 3-channel
 * pixels as stb_image, byte for byte (JPEG included: the inverse DCT, chroma up-sampling and colour conversion follow stb_image's
 * integer arithmetic; tests/golden/jpeg).  TGA / PSD / HDR / PIC and arithmetic-coded or 12-bit JPEG return false with an explicit
 * message in clip_b200_last_error. */
bool clip_image_load_from_file(const char * fname, struct clip_image_u8 * img);

/* clip.h:88, clip.cpp:797-927 -- host side PIL-style bicubic resize + centre crop + normalise */
bool clip_image_preprocess(const struct clip_ctx * ctx, const struct clip_image_u8 * img, struct clip_image_f32 * res);

/* clip.h:90-91, clip.cpp:1016-1233 -- one token sequence (<= context_length) -> vec[projection_dim] */
bool clip_text_encode(const struct clip_ctx * ctx, const int n_threads, const struct clip_tokens * tokens, float * vec,
                      const bool normalize);
/* clip.h:92-93, clip.cpp:1235-1245 */
bool clip_image_encode(const struct clip_ctx * ctx, const int n_threads, struct clip_image_f32 * img, float * vec,
                       const bool normalize);

/* clip.h:95-96, clip.cpp:963-1008 -- host threads = min(n_threads, n images) */
void clip_image_batch_preprocess(const struct clip_ctx * ctx, const int n_threads,
                                 const struct clip_image_u8_batch * img_inputs, struct clip_image_f32_batch * imgs_resized);

/* clip.h:97-98, clip.cpp:1247-1523 -- THE HOT PATH.  vec receives imgs->size * projection_dim floats, image-major.
 * Semantics: B independent single-image encodes (the reference's own batched conv path is wrong for ViT-L/14,
 * SURVEY.md section 8c).  n_threads is accepted and ignored by the GPU forward. */
bool clip_image_batch_encode(const struct clip_ctx * ctx, const int n_threads, const struct clip_image_f32_batch * imgs,
                             float * vec, const bool normalize);

/* clip.h:102-103, clip.cpp:1534-1571 */
bool clip_compare_text_and_image(const struct clip_ctx * ctx, const int n_threads, const char * text,
                                 const struct clip_image_u8 * image, float * score);
/* clip.h:104, clip.cpp:1525-1532 */
float clip_similarity_score(const float * vec1, const float * vec2, const int vec_dim);
/* clip.h:105, clip.cpp:1591-1622 -- p_i = (exp(s_i) + 1e-9) / sum, sorted descending */
bool softmax_with_sorting(float * arr, const int length, float * sorted_scores, int * indices);
/* clip.h:106-107, clip.cpp:1624-1659 */
bool clip_zero_shot_label_image(struct clip_ctx * ctx, const int n_threads, const struct clip_image_u8 * input_img,
                                const char ** labels, const size_t n_labels, float * scores, int * indices);

/* clip.h:109, clip.cpp:1661-1844 -- f32/f16 GGUF -> q4_0(2) q4_1(3) q5_0(6) q5_1(7) q8_0(8); output is byte-identical
 * to the reference's (tests/test_host_side.py) */
bool clip_model_quantize(const char * fname_inp, const char * fname_out, const int itype);

/* =====================================================================================================
 * PART 2 -- additive entry points of this library (not in the reference)
 * ===================================================================================================== */

/* n independent clip_text_encode calls in one launch sequence; seqs may be ragged (each <= context_length).
 * vec receives n * projection_dim floats.  (SURVEY.md section 8b "needed extension") */
bool clip_text_batch_encode(const struct clip_ctx * ctx, const int n_threads, const struct clip_tokens * seqs,
                            const size_t n, float * vec, const bool normalize);

/* Device-resident variants: inputs/outputs are DEVICE pointers on the context's GPU (obtained from
 * clip_b200_device_malloc or any CUDA allocator in the same process).  No host<->device copy is made.
 *   d_pixels : n * image_size*image_size*3 floats, NHWC per image;  d_vec : n * projection_dim floats
 *   d_ids    : n * seq_len int32 (padded), d_lens : n int32 true lengths (NULL = all seq_len) */
bool clip_b200_image_encode_device(const struct clip_ctx * ctx, const void * d_pixels, size_t n, void * d_vec,
                                   bool normalize);
bool clip_b200_text_encode_device(const struct clip_ctx * ctx, const void * d_ids, const void * d_lens, size_t n,
                                  int seq_len, void * d_vec, bool normalize);

/* Every pooled form -- clip_image_batch_encode and clip_text_batch_encode (and clip_image_encode / clip_text_encode through them), the
 * two above, the *_hw, *_all and u8 forms and clip_b200_image_batch_preprocess_device -- checks its arguments in one order and
 * reports the first fault: 1. a null context; 2. the tower; 3. height x width of clip_b200_image_encode_device_hw; 4. n == 0 (a NULL
 * batch is an empty one) returns true here, except in the *_all forms in ranks mode, which refuse it; 5. seq_len in [1,
 * context_length] of the device text forms; 6. null input or output pointers; 7. the host inputs: image_size x image_size images (one
 * patch-multiple size for clip_b200_image_batch_encode_hw), token sequences neither empty nor longer than context_length.  Messages
 * start with the form's name, except for 1 and 2 in the reference's four forms, which print the reference's line to stdout and leave
 * clip_b200_last_error as it was.  Devices mode checks a call once, before it shards it. */

/* Per-token hidden states of either tower (HF output_hidden_states, open_clip forward_intermediates): every row of the residual
 * stream after a chosen layer, for vision-language front ends (LLaVA reads the patch rows of the penultimate layer) and diffusion
 * text conditioning (Stable Diffusion reads all 77 rows, post_ln applied).
 *   layer    HF hidden_states numbering: 0 = the input of block 0 (vision: the pre_ln output; text: token + position embeddings),
 *            i = the output of block i (1 .. n_layer), negative counts from the end (-1 = the last block, -2 = the penultimate one).
 *            Only the blocks up to `layer` run.  Outside [-(n_layer + 1), n_layer]: refused.
 *   flags    CLIP_B200_TOKENS_* below, or 0 for the raw residual rows.
 *   out      item-major, row-major: vision [n, T or T - 1, width] with T = (image_size / patch_size)^2 + 1, CLS first; text
 *            [n, seq_len, width].  width = hidden_size, or projection_dim with PROJECT.  Elements of out_type, rounded to nearest even.
 * With PROJECT the CLS row of an image (row 0) and the EOT row of a sequence (row len - 1) equal clip_image_batch_encode /
 * clip_text_batch_encode's embedding bit for bit (normalize = whether NORMALIZE is set).  Text ids are padded by the caller (any pad id
 * of the caller's model; causal attention keeps the rows before the padding independent of it).
 * Refused with a message in clip_b200_last_error(): a bad layer, unknown flag bits or out_type, NO_CLS on text, NORMALIZE without
 * PROJECT, a model without the tower.  n == 0 returns true.
 * Every tokens form (these four, the *_hw and the *_tokens_layers forms below) checks its arguments in one order and reports the
 * first fault: 1. a null context; 2. the tower; 3. height x width where they are arguments (the device *_hw and *_layers forms);
 * 4. the request: n_layers, NULL layers, then each entry in order; 5. n == 0 returns true here; 6. seq_len in [1, context_length];
 * 7. null input or output pointers; 8. the host images: image_size x image_size for clip_b200_image_tokens, one patch-multiple size
 * for the host *_hw and *_layers forms.
 * Host variants: devices mode (CLIP_B200_DEVICES) shards the batch like clip_image_batch_encode, each GPU copying its slice into out;
 * each micro-batch's rows are copied straight into out (the whole output is never held on the device).  Device variants: pointers on
 * the context's GPU, d_out 16-byte aligned (any cudaMalloc pointer is). */
enum { CLIP_B200_OUT_F32 = 0, CLIP_B200_OUT_F16 = 1, CLIP_B200_OUT_BF16 = 2 };
#define CLIP_B200_TOKENS_POST_LN    1  /* the tower's final LayerNorm (post_ln) on every returned row               */
#define CLIP_B200_TOKENS_PROJECT    2  /* post_ln + projection: rows of projection_dim instead of hidden_size        */
#define CLIP_B200_TOKENS_NORMALIZE  4  /* with PROJECT: L2-normalise each row (as normalize=true does)               */
#define CLIP_B200_TOKENS_NO_CLS     8  /* vision only: patch tokens, T-1 rows per image                               */
/* bit 16 is deliberately left unassigned (tests use it as an unknown flag); new flags take bits above 64 */
#define CLIP_B200_TOKENS_ATTENTION      32  /* the softmax probabilities of block `layer` instead of its residual rows        */
#define CLIP_B200_TOKENS_ATTENTION_CLS  64  /* with ATTENTION, vision only: query row 0 (CLS) only                            */
/* ATTENTION entries (HF output_attentions): `layer` l >= 1, or negative (-1 = the last block), returns the attention of the l-th
 * block, HF's attentions[l - 1]; only blocks 0 .. l - 1 run.  Layer 0 and -(n_layer + 1) are refused (no block has run).
 *   out      per item [H, R, T] row-major (item-major [n, H, R, T], HF's layout), R = T, or 1 with ATTENTION_CLS; elements of
 *            out_type, rounded to nearest even.  Text rows use the causal mask: entries above the diagonal are exactly +0.  Padding is
 *            the caller's, as for hidden states: the rows before a sequence's padding do not depend on it.
 *   flags    ATTENTION cannot be combined with POST_LN, PROJECT, NORMALIZE or NO_CLS; ATTENTION_CLS needs ATTENTION and is refused on
 *            text.
 * Numerics: the scores are those of the attention kernel -- Q already scaled by 1/sqrt(head_dim) and rounded to the 16-bit operand
 * type, K 16-bit, products accumulated in fp32 -- and the softmax runs in fp32 with ex2: p = ex2(s log2e - m log2e) * (1 / l), m the
 * row max, l the sum of ex2(s log2e - m log2e) accumulated block by block as the attention kernel accumulates it.  16-bit outputs are
 * the RNE of that fp32 value.  Not bit-identical to the P the attention kernel multiplies V with: that one is rescaled online and
 * rounded to 16 bits (tests/_attention_probs_bound.py derives the element-wise bound against an fp64 softmax of the same operands).
 * Memory: full maps are large (ViT-L/14 at 224: 16 x 257 x 257 elements per image and layer, 2.1 MB in f16); the host forms stage
 * one micro-batch of the widest entry twice on the device (see *_tokens_layers). */
bool clip_b200_image_tokens(const struct clip_ctx * ctx, const struct clip_image_f32_batch * imgs, int layer, int flags, int out_type,
                            void * out);
bool clip_b200_image_tokens_device(const struct clip_ctx * ctx, const void * d_pixels, size_t n, int layer, int flags, int out_type,
                                   void * d_out);
bool clip_b200_text_tokens(const struct clip_ctx * ctx, const int32_t * ids, size_t n, int seq_len, int layer, int flags, int out_type,
                           void * out);
bool clip_b200_text_tokens_device(const struct clip_ctx * ctx, const void * d_ids, size_t n, int seq_len, int layer, int flags,
                                  int out_type, void * d_out);

/* Vision tower at height x width pixels (both positive multiples of patch_size, <= 4096; rectangular allowed) -- HF
 * CLIPVisionModel(..., interpolate_pos_encoding=True).  The patch grid is gh x gw = height/P x width/P, T = gh*gw + 1.  Patch rows of
 * the position table are resampled to gh x gw as HF's interpolate_pos_encoding does (bicubic, A = -0.75, align_corners = False);
 * the CLS row is unchanged.  The resample is evaluated in fp64 and rounded once to fp32, where torch evaluates it in fp32: the table
 * agrees with HF's to within the fp32 rounding of torch's source coordinates, weights and sums (up to ~25 ulps of the table's
 * largest entry in tests/test_pos_resample.py), not bit for bit.  At height = width = image_size no resampling happens and every result equals
 * the existing entry point's bit for bit.
 *   pixels   NHWC f32 [n, height, width, 3], already normalised, as for the entry points above.
 *   d_vec    [n, projection_dim];  token rows [n, T or T - 1, width], patch rows in row-major grid order (y, then x), as HF's
 *            flatten(2) gives them.  layer, flags and out_type are those of clip_b200_image_tokens, with the same refusals.
 * The workspace is sized as for the model's own size (micro_batch images of the native T, clip_b200_set_micro_batch); a call at
 * another size runs as many images per pass as fit it.  The context keeps the last resampled table, so a call at a new size costs
 * one resample launch.  Refused with a message in clip_b200_last_error(): a size that is not a positive multiple of patch_size or
 * is above 4096, mixed sizes in one host call, a model without a vision tower, a size too large for even one image to fit the
 * workspace.  n == 0 returns true.  Host forms: the size is the images' own (ny rows of nx pixels), every image of one call must
 * have the same size; devices mode (CLIP_B200_DEVICES) shards the batch as clip_image_batch_encode does. */
bool clip_b200_image_encode_device_hw(const struct clip_ctx * ctx, const void * d_pixels, size_t n, int height, int width,
                                      void * d_vec, bool normalize);
bool clip_b200_image_tokens_device_hw(const struct clip_ctx * ctx, const void * d_pixels, size_t n, int height, int width,
                                      int layer, int flags, int out_type, void * d_out);
bool clip_b200_image_batch_encode_hw(const struct clip_ctx * ctx, const struct clip_image_f32_batch * imgs, float * vec,
                                     bool normalize);
bool clip_b200_image_tokens_hw(const struct clip_ctx * ctx, const struct clip_image_f32_batch * imgs, int layer, int flags,
                               int out_type, void * out);

/* Images of different sizes in one call (photos at their own aspect ratio, document pages): the *_hw entry points above with a
 * height x width per image.  The images' rows are packed back to back into one forward pass, attention runs per image over packed
 * sequences of different lengths, and each image gets the position table of its own grid.
 *   sizes    every *_hw rule applies per image: positive multiples of patch_size, at most 4096.  Host forms read each image's size
 *            from its ny / nx; device forms take heights[i] / widths[i], host arrays of n entries, and d_pixels holds the NHWC f32
 *            images back to back (image i starts at float 3 * sum_{j<i} H_j W_j).  Images of one size, and images at image_size (the
 *            loaded table, no resample), are valid calls.
 *   vec      [n, projection_dim], as in the other pooled forms.
 *   out      ragged, item-major: item i is T_i - skip rows of width elements, T_i = (H_i/P)(W_i/P) + 1, skip = 1 with NO_CLS, width =
 *            hidden_size or projection_dim; it starts at byte sum_{j<i} (T_j - skip) * width * element size (16-byte aligned, as every
 *            CLIP width is a multiple of 8).  layer, flags and out_type are those of clip_b200_image_tokens; the ATTENTION flags are
 *            refused.
 * Item i's outputs equal, byte for byte, those of image i passed alone to clip_b200_image_encode_device_hw /
 * clip_b200_image_tokens_device_hw with the same arguments, whatever the other images, their order and how the call is split into
 * passes: no value of one image reaches another image's outputs, and an image holding NaN or Inf leaves the others' bits unchanged.
 * A pass holds the longest prefix of the remaining images that fits the workspace (sized for micro_batch images of the native size,
 * as for the *_hw forms): its rows, patch rows and image count.
 * Arguments are checked in this order, the first fault refused with a message in clip_b200_last_error(): 1. a null context; 2. the
 * vision tower; 3. device forms: each image's size (the message names the first bad image; skipped while heights or widths is NULL);
 * 4. n == 0 (a NULL batch is an empty one) returns true; 5. null pointers: host input and output, device pixels and output, then
 * heights and widths; 6. host forms: each image's pixels and size; 7. tokens: the request, as clip_b200_image_tokens_hw refuses it,
 * then ATTENTION; 8. an image whose rows alone exceed the workspace (the *_hw message, with the image's index).
 * Host forms: devices mode (CLIP_B200_DEVICES) shards the images as clip_image_batch_encode does (by count); each pass's rows are
 * copied to the host before the next pass runs. */
bool clip_b200_image_batch_encode_mixed(const struct clip_ctx * ctx, const struct clip_image_f32_batch * imgs, float * vec, bool normalize);
bool clip_b200_image_encode_device_mixed(const struct clip_ctx * ctx, const void * d_pixels, size_t n, const int * heights,
                                         const int * widths, void * d_vec, bool normalize);
bool clip_b200_image_tokens_mixed(const struct clip_ctx * ctx, const struct clip_image_f32_batch * imgs, int layer, int flags,
                                  int out_type, void * out);
bool clip_b200_image_tokens_device_mixed(const struct clip_ctx * ctx, const void * d_pixels, size_t n, const int * heights,
                                         const int * widths, int layer, int flags, int out_type, void * d_out);

/* Token sequences of different lengths in one call, with no padding: clip_text_batch_encode, clip_b200_text_encode_device and
 * clip_b200_text_tokens[_device] with every sequence at its own length.  The sequences' rows are packed back to back into one forward
 * pass (every GEMM and LayerNorm runs on the real rows only) and causal attention runs per sequence over packed sequences of
 * different lengths.  The unpadded forms above still accept ragged lengths; they pad every sequence to the longest of the call.
 *   ids      ids / d_ids: int32, the sequences back to back; sequence i starts at element sum_{j<i} lens[j].  lens: a HOST array of n
 *            lengths.  clip_b200_text_batch_encode_packed takes clip_tokens as clip_text_batch_encode does.
 *   vec      vec / d_vec [n, projection_dim]: the EOT row of each sequence (row len - 1, as the reference selects it).
 *   out      ragged, item-major: item i is lens[i] rows of width elements (hidden_size, or projection_dim with PROJECT); it starts at
 *            byte sum_{j<i} lens[j] * width * element size (16-byte aligned, as every CLIP width is a multiple of 8).  layer, flags
 *            and out_type are those of clip_b200_text_tokens, with the same refusals; the ATTENTION flags are refused.
 * Item i's outputs equal, byte for byte, sequence i passed alone to clip_b200_text_encode_device / clip_b200_text_tokens_device at
 * seq_len = lens[i], and clip_text_batch_encode's row i for the same sequences, whatever the other sequences, their order and how the
 * call is split into passes: a sequence holding ids that lead to NaN or Inf leaves the others' bits unchanged.
 * A pass holds the longest prefix of the remaining sequences whose rows fit the workspace (micro_batch x context_length rows,
 * clip_b200_set_micro_batch), so short sequences take proportionally more per pass.
 * Text towers of head_dim 64 only (every CLIP text tower: ViT-B, L, H/14 and bigG/14); others are refused.
 * Arguments are checked in this order, the first fault refused with a message in clip_b200_last_error() that starts with the
 * form's name: 1. a null context; 2. the text tower; 3. a text head_dim other than 64; 4. n == 0 returns true; 5. null pointers:
 * input, lens, then output; 6. each sequence's length in [1, context_length] (the message names the first bad sequence; a
 * clip_tokens with NULL data or size 0 fails here); 7. tokens forms: the request, as clip_b200_text_tokens refuses it, then ATTENTION.
 * Host forms: devices mode (CLIP_B200_DEVICES) shards the sequences by count as clip_text_batch_encode does; each pass's rows are
 * copied to the host before the next pass runs. */
bool clip_b200_text_batch_encode_packed(const struct clip_ctx * ctx, const struct clip_tokens * seqs, size_t n, float * vec,
                                        bool normalize);
bool clip_b200_text_encode_device_packed(const struct clip_ctx * ctx, const void * d_ids, size_t n, const int * lens, void * d_vec,
                                         bool normalize);
bool clip_b200_text_tokens_packed(const struct clip_ctx * ctx, const int32_t * ids, size_t n, const int * lens, int layer, int flags,
                                  int out_type, void * out);
bool clip_b200_text_tokens_device_packed(const struct clip_ctx * ctx, const void * d_ids, size_t n, const int * lens, int layer,
                                         int flags, int out_type, void * d_out);

/* Several layers' token rows from ONE forward pass of a tower (HF output_hidden_states returns all n_layer + 1; multi-layer VLM
 * connectors read 3 or 4 vision layers; SDXL reads layer -2 raw and the projected EOT row of layer -1 of the same text pass).
 *   layers[j], flags[j]  entry j: a layer and CLIP_B200_TOKENS_* flags exactly as `layer` / `flags` of the single-layer calls above.
 *            Any order, duplicates allowed.  flags == NULL: 0 for every entry.  Only blocks 0 .. deepest - 1 run, each once.
 *   n_layers 1 .. CLIP_B200_TOKENS_MAX_LAYERS;  out_type applies to every entry.
 *   out      layer-major: entry j is one slab of n * item_bytes_j bytes at offset n * (item_bytes_0 + ... + item_bytes_{j-1}), laid
 *            out as the single-layer call lays out its whole output (item_bytes_j = rows x width x element size of that entry;
 *            H x R x T x element size for an ATTENTION entry).  After an ATTENTION slab the next slab starts at the next multiple of
 *            16 bytes (from out), so that the vector stores of the slab after an odd-sized attention slab stay aligned; only
 *            attention slabs are padded, and a list without ATTENTION entries is laid out as above, byte for byte.
 * Slab j equals, byte for byte, the single-layer call with (layers[j], flags[j], out_type) on the same inputs: the same kernels run
 * on the same residual stream.  Image size: the host form takes it from the images, as clip_b200_image_tokens_hw does (at
 * image_size x image_size that is the native path); the device form takes height x width (image_size x image_size: native).  Every
 * *_hw rule applies.  Refused with a message in clip_b200_last_error(): n_layers outside [1, CLIP_B200_TOKENS_MAX_LAYERS], NULL
 * layers or output, any entry the single-layer call would refuse (the message names the entry's index), a bad image size or mixed
 * sizes in one host call, a model without the tower.  n == 0 returns true.
 * Host forms: rows leave the device through a two-slot staging ring on a copy stream, so one layer's device-to-host copy runs under
 * the next layer's blocks; a pinned `out` (clip_b200_host_malloc) receives them directly, a pageable one through a pinned bounce
 * buffer (two micro-batches of the widest entry, grow-only).  Devices mode (CLIP_B200_DEVICES) shards the items as the single-layer
 * host forms do, each GPU writing its items into every slab.  Device forms: pointers on the context's GPU, d_out 16-byte aligned. */
#define CLIP_B200_TOKENS_MAX_LAYERS 4096
bool clip_b200_image_tokens_layers(const struct clip_ctx * ctx, const struct clip_image_f32_batch * imgs,
                                   const int * layers, const int * flags, int n_layers, int out_type, void * out);
bool clip_b200_image_tokens_layers_device(const struct clip_ctx * ctx, const void * d_pixels, size_t n, int height, int width,
                                          const int * layers, const int * flags, int n_layers, int out_type, void * d_out);
bool clip_b200_text_tokens_layers(const struct clip_ctx * ctx, const int32_t * ids, size_t n, int seq_len,
                                  const int * layers, const int * flags, int n_layers, int out_type, void * out);
bool clip_b200_text_tokens_layers_device(const struct clip_ctx * ctx, const void * d_ids, size_t n, int seq_len,
                                         const int * layers, const int * flags, int n_layers, int out_type, void * d_out);

/* Batched zero-shot scoring on the device (clip.cpp:1624-1659 semantics per image): d_img_vec [n_img, d], d_txt_vec [n_txt, d]
 * -> host scores/indices [n_img, top_k], best first; similarity matrix, softmax and top-k selection all run on the GPU.
 * Ranking (here and in clip_b200_topk_search): top_k <= 0 or top_k > n_txt means all n_txt, and row i of the output starts at
 * i * (that clamped top_k).  Equal scores are ordered by lower index first.  A NaN score ranks last and is reported as -FLT_MAX.
 * Refusals (here and in clip_b200_topk_search), with a message in clip_b200_last_error that starts with the function's name, in
 * this order: null context; a count (n_img / n_queries or n_txt / n_db) >= 2^31; then, when there is work (a count of 0 returns
 * true and writes nothing), a null device pointer (no alignment is required) and null outputs.  These two forms used to check
 * less, and differ from earlier versions in four ways:
 * - a null context sets a message (it returned false without one);
 * - the 2^31 message starts with the function's name (it started with "scoring:");
 * - a null device pointer or null output is refused when there is work (the call used to fault on the device or fail later);
 * - a call with one count 0 and the other >= 2^31 is refused (it returned true), the order of every search form. */
bool clip_b200_zero_shot_batch(const struct clip_ctx * ctx, const void * d_img_vec, size_t n_img, const void * d_txt_vec,
                               size_t n_txt, float * scores, int * indices, int top_k);

/* Nearest-neighbour search on the device (stands in for USearch in examples/image-search/search.cpp:114-158): raw dot products
 * (cosine similarity for normalised embeddings) of n_queries x n_db device-resident vectors, best top_k per query to the host.
 * Each score is one sequential fmaf chain over the d features.  top_k <= 0 or top_k > n_db means all n_db, and row i of the output
 * starts at i * (that clamped top_k).  Equal scores are ordered by lower index first.  A NaN score ranks last and is reported as
 * -FLT_MAX.  Refusals: those of clip_b200_zero_shot_batch, in the same order. */
bool clip_b200_topk_search(const struct clip_ctx * ctx, const void * d_queries, size_t n_queries, const void * d_db, size_t n_db,
                           int top_k, float * scores, int * indices);

/* f32 rows -> f16 / bf16 rows (round to nearest even), device to device: how pooled embeddings (or token rows) become a 16-bit
 * database or query set for clip_b200_topk_search_16.  d_src [n, dim] f32 and d_dst [n, dim] of out_type (CLIP_B200_OUT_F16 or
 * CLIP_B200_OUT_BF16), row-major, on the context's GPU, 16-byte aligned; dim a multiple of 4 in [4, 2048]; n < 2^31 (n * dim may
 * exceed 2^32).  n == 0 returns true.  Returns once the rows are written.  Its time is kernel class 4. */
bool clip_b200_rows_to_16bit(const struct clip_ctx * ctx, const void * d_src, size_t n, int dim, int out_type, void * d_dst);

/* Nearest-neighbour search over a 16-bit database on the tensor cores (kernel K10), the opt-in companion of clip_b200_topk_search
 * for databases stored in 16 bits.  No score matrix is written: each CTA keeps its own top_k while it scores.
 * - Inputs: in_type is CLIP_B200_OUT_F16 or CLIP_B200_OUT_BF16.  d_queries [n_queries, dim] and d_db [n_db, dim] are row-major, of
 *   that type, on the context's GPU, 16-byte aligned.  dim is a multiple of 8 in [8, 2048]; it is an argument, not the model's
 *   projection_dim (patch-token features can be searched too), and the model's towers are not used.
 * - Scores: the dot product of the 16-bit query and row; the products are exact in fp32 and accumulated in fp32 on the tensor
 *   cores, in k16 steps.  Each score lies within (2 * ceil(dim / 16) + 4) * 2^-24 * sum_i |q_i x_i| of the exact value.  A score
 *   depends only on the query and the row: it has the same bits on every call, whatever n_db, top_k or the row's position.
 * - Ranking: the best top_k of all n_db scores, score descending, then lower index first, host [n_queries, top_k], row i at
 *   i * top_k.  A NaN score ranks last and is reported as -FLT_MAX.
 * - top_k must be in [1, 1024]; a value above n_db means n_db.  Unlike clip_b200_topk_search there is no "all rows" ranking
 *   on the host: top_k <= 0 or > 1024 is refused.
 * - Refusals, with a message in clip_b200_last_error, in this order: null context; in_type; dim; top_k; n_queries or n_db >= 2^31;
 *   then, when there is work (n_queries == 0 or n_db == 0 returns true and writes nothing), null or misaligned device pointers
 *   and null outputs.
 * - Runs on the context's first GPU (in devices mode too); the database is not sharded.
 * - Workspace, grow-only, on the context: per launch of up to 32768 queries (Q of them), with the plan's query tile N = the least
 *   power of two >= min(Q, 128), at least 8, P partitions and G CTAs (G <= max(#SMs, Q / 128 rounded up), P * ceil(Q / N) = G):
 *   G * N * (top_k + 256) * 8 bytes of per-CTA candidates, plus 4 * Q * P * top_k * 4 bytes of merge buffers (shared with
 *   clip_b200_topk_search). */
bool clip_b200_topk_search_16(const struct clip_ctx * ctx, const void * d_queries, size_t n_queries, const void * d_db, size_t n_db,
                              int dim, int in_type, int top_k, float * scores, int * indices);

/* f32 rows -> scalar-quantised int8 rows (one signed byte per feature and one f32 scale per row, as FAISS SQ8 and USearch i8),
 * device to device: how a database or query set is made for clip_b200_topk_search_i8.  It takes dim + 4 bytes a row.
 * - d_src [n, dim] f32, d_codes [n, dim] int8, d_scales [n] f32, row-major, on the context's GPU, 16-byte aligned.  dim is a
 *   multiple of 16 in [16, 2048]; n < 2^31 (n * dim may exceed 2^32).
 * - The rule, per row, exactly: m = max_i |x_i|; s = m / 127 in f32, rounded to nearest; c_i = clamp(rint(x_i / s), -127, 127), the
 *   division IEEE and correctly rounded, rint rounding half to even, nothing flushed to zero (the clamp matters when s is
 *   subnormal).  A row whose s is 0 (all zeros, or m / 127 underflows) gets s = 0 and all-zero codes.  A row holding any NaN or
 *   +-Inf gets s = NaN and all-zero codes.  No code is -128.
 * - Refusals, with a message in clip_b200_last_error, in this order: null context; dim; n >= 2^31; then, when n > 0 (n == 0
 *   returns true), null or misaligned pointers.  Returns once the rows are written.  Its time is kernel class 3. */
bool clip_b200_rows_to_int8(const struct clip_ctx * ctx, const void * d_src, size_t n, int dim, void * d_codes, void * d_scales);

/* Nearest-neighbour search over an int8 database (clip_b200_rows_to_int8's form) on the tensor cores: K10's s8 instance, the same
 * kernel, plan and ranking as clip_b200_topk_search_16, reading half the bytes per row.
 * - Inputs: query codes [n_queries, dim] and scales [n_queries], database codes [n_db, dim] and scales [n_db], as
 *   clip_b200_rows_to_int8 writes them, on the context's GPU, 16-byte aligned.  dim is a multiple of 16 in [16, 2048].
 * - Scores, exactly: acc = the int32 dot product of the codes (exact: |acc| <= 127^2 * 2048 < 2^31), then
 *   score = fp32(fp32(float_rn(acc) * s_q) * s_x), both products rounded to nearest, in this order, not contracted.  A score
 *   depends only on the query's and the row's codes and scales.  Against the exact dot product of the f32 rows q and x that
 *   were quantised, a finite score lies within
 *       |score - q.x| <= sum_i (|q_i| d_x + |x_i| d_q + d_q d_x) + 2^-22 |score| + 2^-149 (1 + s_x),
 *   where d = s (1/2 + 2^-16) is how far a code times its scale can lie from the value (half a step, widened by the rounding of
 *   x_i / s), or m - 127 s if that is larger, which happens only for subnormal s.  With normal scales that is about
 *   sum_i (|q_i| s_x + |x_i| s_q) / 2 + dim s_q s_x / 4 + a few ulps of |score| (derived in tests/_search_i8.py).
 * - Ranking: the best top_k of all n_db scores, score descending, then lower index first, host [n_queries, top_k], row i at
 *   i * top_k.  A NaN score (a non-finite row or query) ranks last and is reported as -FLT_MAX.
 * - top_k must be in [1, 1024]; a value above n_db means n_db.
 * - Refusals, with a message in clip_b200_last_error, in this order: null context; dim; top_k; n_queries or n_db >= 2^31; then,
 *   when there is work (n_queries == 0 or n_db == 0 returns true and writes nothing), null or misaligned device pointers and
 *   null outputs.
 * - Runs on the context's first GPU (in devices mode too); the database is not sharded.  Queries go in launches of up to 32768.
 * - Workspace: clip_b200_topk_search_16's formula, in the same grow-only buffers.  Its kernel time is kernel class 8. */
bool clip_b200_topk_search_i8(const struct clip_ctx * ctx, const void * d_q_codes, const void * d_q_scales, size_t n_queries,
                              const void * d_db_codes, const void * d_db_scales, size_t n_db, int dim, int top_k,
                              float * scores, int * indices);

/* f32 rows -> binary rows (one sign bit per feature, as USearch b1 and FAISS binary indexes store them), device to device: how a
 * database or query set is made for clip_b200_topk_search_b1.  A 768-d row takes 96 bytes.
 * - d_src [n, dim] f32, d_center [dim] f32 or NULL (all zeros), d_bits [n, dim / 8] uint8, row-major, on the context's GPU,
 *   16-byte aligned.  dim is a multiple of 128 in [128, 2048], so a row is whole 16-byte words; n < 2^31 (n * dim may exceed 2^32).
 * - The rule, exactly: bit i is 1 iff x_i > c_i, an IEEE compare with nothing flushed to zero: a NaN gives 0, so does -0 against 0,
 *   and a subnormal above 0 gives 1.  Feature i goes to byte i / 8, bit i % 8, least significant bit first
 *   (numpy.packbits(bits, axis=1, bitorder="little")).
 * - The centre: CLIP embeddings share a common mean direction, so the signs of raw coordinates spend bits on it.  Passing the
 *   database's mean (of a sample) as d_center is the usual fix.
 * - Refusals, with a message in clip_b200_last_error, in this order: null context; dim; n >= 2^31; then, when n > 0 (n == 0
 *   returns true), null or misaligned d_src / d_bits, or a misaligned non-NULL d_center.  Returns once the rows are written.  Its
 *   time is kernel class 3. */
bool clip_b200_rows_to_binary(const struct clip_ctx * ctx, const void * d_src, size_t n, int dim, const void * d_center,
                              void * d_bits);

/* Nearest-neighbour search over a binary database (clip_b200_rows_to_binary's form) on the tensor cores (kernel K11): K10's plan,
 * candidate buffers and merge, with 1-bit tensor-core products (mma m16n8k256 b1, AND + popcount).
 * - Inputs: d_q_bits [n_queries, dim / 8] and d_db_bits [n_db, dim / 8], as clip_b200_rows_to_binary writes them, on the context's
 *   GPU, 16-byte aligned.  dim is a multiple of 128 in [128, 2048].
 * - Scores, exactly: s = dim - 2 popcount(q XOR x), the dot product of the +-1 vectors (bit 1 is +1): an integer in [-dim, dim],
 *   returned as an exact float.  No NaN can occur.  A score depends only on the query's and the row's bits.
 * - Ranking: the best top_k of all n_db scores, score descending, then lower index first, host [n_queries, top_k], row i at
 *   i * top_k.  Scores take at most dim + 1 values, so ties are common; the index order settles them.
 * - top_k must be in [1, 1024]; a value above n_db means n_db.
 * - Refusals, with a message in clip_b200_last_error, in this order: null context; dim; top_k; n_queries or n_db >= 2^31; then,
 *   when there is work (n_queries == 0 or n_db == 0 returns true and writes nothing), null or misaligned device pointers and
 *   null outputs.
 * - Runs on the context's first GPU (in devices mode too); the database is not sharded.  Queries go in launches of up to 32768.
 * - Workspace: clip_b200_topk_search_16's formula, in the same grow-only buffers, except that with a query tile below 64 the plan
 *   takes G <= 2 x #SMs CTAs.  Its kernel time is kernel class 9. */
bool clip_b200_topk_search_b1(const struct clip_ctx * ctx, const void * d_q_bits, size_t n_queries, const void * d_db_bits,
                              size_t n_db, int dim, int top_k, float * scores, int * indices);

/* Exact rescoring of a shortlist (kernel K12), as FAISS IndexRefine and "binary + rescore" pipelines do it: per query, the
 * candidates a cheaper search returned are scored again against full-precision rows and the best top_k kept.
 * - Inputs: in_type is CLIP_B200_OUT_F32, CLIP_B200_OUT_F16 or CLIP_B200_OUT_BF16, for both d_queries [n_queries, dim] and d_db
 *   [n_db, dim], row-major, on the context's GPU, 16-byte aligned.  dim is a multiple of 8 in [8, 2048].  cand is HOST memory
 *   [n_queries, n_cand] int32, for example exactly what a search form wrote into its indices.  n_cand is in [1, 2048].
 * - Scores, exactly: one sequential fmaf chain from +0 over features 0 .. dim - 1; 16-bit values are widened to f32 first (exact).
 *   In F32 this is clip_b200_topk_search's chain, so every score has the same bits as that search's score for the pair.  With
 *   16-bit rows each product is exact in f32 and only the sums round.  A NaN score ranks last among the valid candidates and is
 *   reported as -FLT_MAX.
 * - Candidates are a set: entries outside [0, n_db) (-1, INT_MAX, ...) are skipped and a duplicate counts once.  The best top_k
 *   (top_k in [1, n_cand]) of the distinct valid candidates go to host [n_queries, top_k], score descending, then lower index
 *   first; if fewer remain, the rest of the row is (-INFINITY, -1).
 * - Refusals, with a message in clip_b200_last_error, in this order: null context; in_type; dim; n_cand; top_k; n_queries or n_db
 *   >= 2^31; then, when there is work (n_queries == 0 or n_db == 0 returns true and writes nothing), null or misaligned device
 *   pointers, null cand, null outputs.
 * - Runs on the context's first GPU.  Workspace, grow-only: a device copy of the candidates of up to min(32768, 2^22 / n_cand)
 *   queries at a time, and the merge buffers of clip_b200_topk_search.  Its kernel time is kernel class 10. */
bool clip_b200_topk_rescore(const struct clip_ctx * ctx, const void * d_queries, size_t n_queries, const void * d_db, size_t n_db,
                            int dim, int in_type, const int * cand, int n_cand, int top_k, float * scores, int * indices);

/* ---- inverted-file index over a 16-bit database (FAISS IndexIVFFlat, spherical k-means) -------------------------------------
 * k-means splits the database into n_lists lists; each row is stored with its list; a query scores the centroids and scans only
 * its nprobe best lists.  At n_lists = 4096 and nprobe = 32 a query reads under 1 % of the rows.  The caller owns the index, four
 * device buffers: centroids [n_lists, dim] of in_type, offsets [n_lists + 1] int32, ids [n_db] int32, rows [n_db, dim] of in_type.
 * - Limits: in_type is CLIP_B200_OUT_F16 or CLIP_B200_OUT_BF16; dim is a multiple of 8 in [8, 2048]; n_lists in [1, 65536];
 *   top_k in [1, 1024]; nprobe in [1, 1024], a value above n_lists meaning n_lists; n_iter in [1, 1000]; counts below 2^31.
 *   Device pointers are 16-byte aligned, except d_offsets and d_ids, which need 4 bytes.  All three run on the context's first
 *   GPU (in devices mode too).
 * - Assignment: a row's list is its best centroid under clip_b200_topk_search_16's score and ranking (score descending, then the
 *   lower list index), i.e. clip_b200_topk_search_16(row, centroids, top_k = 1).  Train and build assign alike.
 * - Refusals, each with a message in clip_b200_last_error that starts with the function's name, in this order: null context;
 *   in_type; dim; n_lists; n_iter / nprobe; top_k; a count >= 2^31 (train: then n_train < n_lists); then, when there is work,
 *   null or misaligned device pointers, then null outputs.
 * - Kernel time: the assignments and the probes are kernel class 7 (K10), the fine scan class 11, the k-means update and the
 *   build's row gather class 12. */

/* k-means (Lloyd, spherical) on the tensor cores: n_lists unit-norm centroids of in_type [n_lists, dim] to d_centroids.
 * 1. The initial centroids are the training rows at indices floor(i * n_train / n_lists), so n_train >= n_lists is required (a
 *    caller who wants a random start shuffles the training set).
 * 2. Each of the n_iter iterations assigns every training row, then replaces the centroid c of each non-empty list by the mean m
 *    of its members, L2-normalised: m_j = (fp64 sum of the members' values, exact when widened) / count in fp64, and
 *    c_j = rne_16(m_j / sqrt(sum_j m_j^2)), in fp64, rounded once to in_type.  The sums run in a fixed order (members in row
 *    order, in chunks of 512 whose sums are added in chunk order; the squares by a fixed tree), so a call gives the same bits
 *    every time.  An empty list, and a list whose mean is exactly zero, keep their previous centroid.
 * Workspace, grow-only: about n_train * 4 + (n_train / 512 + n_lists) * dim * 8 bytes, plus the K10 buffers of
 * clip_b200_topk_search_16 at top_k = 1. */
bool clip_b200_ivf_train_16(const struct clip_ctx * ctx, const void * d_train, size_t n_train, int dim, int in_type,
                            int n_lists, int n_iter, void * d_centroids);

/* Assign every row of d_db [n_db, dim] to its list and lay the database out list by list: d_offsets[l] .. d_offsets[l + 1] - 1 are
 * the stored positions of list l, lists in list order, rows within a list in increasing original index; d_ids[p] is the original
 * index at stored position p and d_rows[p] that row, byte for byte.  n_db == 0 writes n_lists + 1 zeros to d_offsets and nothing
 * else.  Offsets of the copy are 64-bit, so n_db * dim * 2 may pass 2^32. */
bool clip_b200_ivf_build_16(const struct clip_ctx * ctx, const void * d_db, size_t n_db, int dim, int in_type,
                            const void * d_centroids, int n_lists, int * d_offsets, int * d_ids, void * d_rows);

/* Probe the nprobe best lists of each query and return its best top_k rows, by original row index, to host [n_queries, w],
 * w = min(top_k, n_db), row i at i * w.
 * - The probes of query q are the best nprobe lists of clip_b200_topk_search_16(q, centroids, nprobe).  The result is the best w
 *   rows of the union of the probed lists in clip_b200_topk_search_16's ranking: score descending, then the lower ORIGINAL index.
 *   Each score has the bits clip_b200_topk_search_16 gives the pair (query, row): a score does not depend on the query's place in
 *   a query tile nor on the tile's width.  A NaN score ranks last and is reported as -FLT_MAX.  When the probed lists hold fewer
 *   than w rows, the rest of the row is (-INFINITY, -1), as clip_b200_topk_rescore pads.
 * - Consequence: with nprobe >= n_lists the output equals clip_b200_topk_search_16 over the original database, byte for byte.
 * - Before any device work d_offsets is read and must run non-decreasing from 0 to n_db; a malformed index is refused with a
 *   message.  d_ids is only copied to the output, never dereferenced.  n_queries == 0 or n_db == 0 returns true and writes
 *   nothing.
 * - The fine scan is K10 run from a table of work units (list, up to N of its (query, list) pairs, a range of up to R of its
 *   rows): N = 8 nt, the least power of two >= the mean pairs per probed list (8 to 128); R, a multiple of 128, so that the
 *   units come to about 4 per SM.  Queries go in blocks of Q = min(32768, max(1, 2^24 / ((w + 256) * min(nprobe, n_lists))))
 *   queries, P = Q * min(nprobe, n_lists) pairs at most.
 * - Workspace, grow-only, per block: the K10 buffers of the probes (clip_b200_topk_search_16's formula at top_k = nprobe), then
 *   U * N * (w + 256) * 8 bytes of per-unit candidates for U units (U * N < 3 P + 8 * lists probed + 512 * #SMs), P * (dim * 2 + 16)
 *   bytes of gathered queries and tables, and 4 * Q * runs * w * 4 bytes of merge buffers, runs = the most row ranges one query
 *   probes. */
bool clip_b200_ivf_search_16(const struct clip_ctx * ctx, const void * d_queries, size_t n_queries, int dim, int in_type,
                             const void * d_centroids, int n_lists, const int * d_offsets, const int * d_ids,
                             const void * d_rows, size_t n_db, int nprobe, int top_k, float * scores, int * indices);

/* ---- inverted-file index with product-quantised residuals (FAISS IndexIVFPQ, by residual, 8-bit codes) ----------------------
 * The lists of clip_b200_ivf_*, but each row is stored as m one-byte codes of its residual against its list's centroid: m bytes a
 * row instead of dim * 2, so 10^8 768-d rows take 9.6 GB of codes at m = 96.  The residual's dim features are split into m
 * subspaces of dsub = dim / m features, and each subspace has its own 256 codewords.  The caller owns the index: centroids
 * [n_lists, dim] of in_type (from clip_b200_ivf_train_16, for example), codebooks f32 [m, 256, dsub], and from the build offsets
 * [n_lists + 1] int32, ids [n_db] int32 and codes uint8 [n_db, m].  Encode and build are separate calls, so a database larger than
 * device memory is encoded in chunks of rows; only its codes and lists need to be resident at build time.
 * - Limits: in_type, dim, n_lists, nprobe, n_iter and top_k as clip_b200_ivf_*.  m is a multiple of 16 in [16, 256] that divides
 *   dim, so a code row is whole 16-byte words.  Training needs n_train >= 256.  Counts below 2^31; offsets into the codes are 64-bit,
 *   so n_db * m may pass 2^32.  Device pointers are 16-byte aligned, except d_lists, d_offsets and d_ids, which need 4 bytes.  All
 *   four run on the context's first GPU.
 * - The rule; every step is exact, so a restatement in numpy reproduces every output bit for bit (tests/_search_ivfpq.py):
 *   1. A row's list is its best centroid under clip_b200_ivf_build_16's rule: clip_b200_topk_search_16(row, centroids, 1).
 *   2. Its residual r_j = x_j - c_j in fp32, rounded to nearest, both values widened exactly from in_type.
 *   3. The distance of r to codeword b of subspace s: t = r_j - b_j in fp32, d = fmaf(t, t, d), over the subspace's features in
 *      order, from +0.  A NaN distance counts as +inf.
 *   4. The code of subspace s is the codeword with the least distance, the lower index on ties.  So a row holding NaN or +-Inf
 *      gets code 0 in every subspace it touches.
 * - Refusals, each with a message in clip_b200_last_error that starts with the function's name, in the order of the steps that
 *   apply to the form: null context; in_type; dim; m; n_lists; n_iter / nprobe; top_k; a count >= 2^31 (train: then n_train < 256);
 *   then, when there is work, null or misaligned device pointers, then null outputs.
 * - Kernel time: the assignments and the probes are kernel class 7 (K10), the ADC scan class 13, the lookup tables, the codebook
 *   k-means and the encoding class 14, the build's code gather class 12. */

/* Codebook k-means (Lloyd, Euclidean) over the residuals of d_train [n_train, dim] -> d_codebooks f32 [m, 256, dsub].
 * 1. Every training row is assigned to its list (rule 1) and its residual taken (rule 2).
 * 2. The initial codeword i of every subspace is the residual of training row floor(i * n_train / 256).
 * 3. Each of the n_iter iterations assigns every residual in every subspace (rules 3 and 4), then replaces each non-empty codeword
 *    by the fp64 mean of its members' residuals, rounded once to fp32.  The members are summed in row order, in chunks of 512 whose
 *    sums are added in chunk order, as clip_b200_ivf_train_16 sums, so a call gives the same bits every time.  An empty codeword
 *    keeps its value.  There is no normalisation.
 * Workspace, grow-only: about n_train * (5 m + 4) + (n_train / 512 + 256) * dim * 8 bytes, plus the K10 buffers of
 * clip_b200_topk_search_16 at top_k = 1; the host holds n_train * 5 m bytes. */
bool clip_b200_ivfpq_train_16(const struct clip_ctx * ctx, const void * d_train, size_t n_train, int dim, int in_type,
                              const void * d_centroids, int n_lists, int m, int n_iter, void * d_codebooks);

/* Encode d_rows [n, dim]: each row's list (rule 1) to d_lists [n] int32 and its codes (rules 2-4) to d_codes uint8 [n, m].  Chunks
 * of a database encoded by separate calls give the bytes one call gives.  n == 0 returns true and writes nothing. */
bool clip_b200_ivfpq_encode_16(const struct clip_ctx * ctx, const void * d_rows, size_t n, int dim, int in_type,
                               const void * d_centroids, int n_lists, const void * d_codebooks, int m,
                               int * d_lists, void * d_codes);

/* Lay encoded rows out list by list: d_offsets and d_ids are the stable layout by original index that clip_b200_ivf_build_16 writes
 * for the same lists, and stored position p of d_codes_out [n_db, m] holds the codes of row d_ids[p], byte for byte.  d_lists is
 * read first: a value outside [0, n_lists) is refused before anything is written.  n_db == 0 writes n_lists + 1 zeros to d_offsets
 * and nothing else. */
bool clip_b200_ivfpq_build(const struct clip_ctx * ctx, const int * d_lists, const void * d_codes, size_t n_db, int n_lists, int m,
                           int * d_offsets, int * d_ids, void * d_codes_out);

/* Probe the nprobe best lists of each query and return its best top_k stored rows, by original row index, to host [n_queries, w],
 * w = min(top_k, n_db), row i at i * w.
 * - The probes and their coarse scores s_c are exactly what clip_b200_topk_search_16(q, centroids, nprobe) returns, NaN read as
 *   -FLT_MAX included.
 * - The lookup table of a query: T[s][k] = the fmaf chain over subspace s's features j of q_j * b_kj, from +0, in order, with q
 *   widened exactly.  A stored row with codes c in list l scores v = s_c, then v = v + T[s][c_s] in fp32 for s = 0 .. m - 1 in
 *   order.  For inner product this is FAISS's by-residual IVFPQ score <q, c_l> + <q, r^>; the table depends on the query alone.
 * - Ranking, padding and d_offsets' check are clip_b200_ivf_search_16's: score descending, then the lower original index; a NaN
 *   score ranks last and is reported as -FLT_MAX; (-INFINITY, -1) past the probed rows; a malformed d_offsets is refused before
 *   any device work.  n_queries == 0 or n_db == 0 returns true and writes nothing.
 * - The scan (K13) runs clip_b200_ivf_search_16's work units with at most N = 8 pairs a unit (K13 scores a unit's pairs one after
 *   another, so a unit costs its pairs times its rows), 256 threads over rows, one pair at a time, with the pair's table in shared
 *   memory in slices of up to 128 subspaces.  Queries go in blocks of
 *   Q = min(32768, max(1, 2^24 / ((w + 256) * min(nprobe, n_lists))), 2^18 / m), so the tables of a block, Q * m KiB, stay within
 *   256 MiB.
 * - Workspace, grow-only, per block: the K10 buffers of the probes, Q * m KiB of tables, U * (w + 384) * 8 bytes of per-unit
 *   candidates for U units (U < 3 P + lists probed + 512 * #SMs, P = Q * min(nprobe, n_lists) pairs at most), P * 16 + U * 20 bytes
 *   of plan, and 4 * Q * runs * w * 4 bytes of merge buffers, runs = the most row ranges one query probes. */
bool clip_b200_ivfpq_search_16(const struct clip_ctx * ctx, const void * d_queries, size_t n_queries, int dim, int in_type,
                               const void * d_centroids, int n_lists, const void * d_codebooks, int m,
                               const int * d_offsets, const int * d_ids, const void * d_codes, size_t n_db,
                               int nprobe, int top_k, float * scores, int * indices);

/* Batched zero-shot labelling, the batch form of clip_zero_shot_label_image (clip.h:106-107, clip.cpp:1624-1659): n images x
 * n_labels token sequences -> scores / indices [n, top_k], best first (p = (exp(s)+1e-9)/sum over ALL labels, clip.cpp:1591-1622).
 * normalize = false reproduces the reference (un-normalised embeddings).  Works in every multi-GPU mode (see below): in devices
 * mode images and labels are sharded over the GPUs and the label embeddings all-gathered; in ranks mode the caller passes this
 * rank's images and this rank's label shard (same count on every rank; global label index = rank * n_labels + j). */
bool clip_b200_zero_shot_images(const struct clip_ctx * ctx, const int n_threads, const struct clip_image_f32_batch * imgs,
                                const struct clip_tokens * labels, const size_t n_labels, const bool normalize, int top_k,
                                float * scores, int * indices);

/* ---- multi-GPU inside the library (csrc/dist.h; the reference's analogue is ggml-cuda.cu:404-407, 5934-5957) -----------------
 * devices mode: set CLIP_B200_DEVICES=0,1,...|all before clip_model_load: ONE context drives a replica per GPU (NCCL communicators
 *   from ncclCommInitAll); clip_image_batch_encode / clip_text_batch_encode / clip_b200_zero_shot_images shard their batch
 *   contiguously and each GPU copies its slice of the result into the caller's buffer.
 * ranks mode:   one process per GPU (torchrun, mpirun, ...): clip_b200_dist_init joins an NCCL communicator (ncclCommInitRank);
 *   rendezvous = NULL takes the 128-byte unique id from a file named after MASTER_PORT and the launcher's pid (single node), or
 *   exchange clip_b200_dist_unique_id's output yourself and call clip_b200_dist_init_with_id.  CLIP_B200_DIST=env makes
 *   clip_model_load do this from RANK / WORLD_SIZE / LOCAL_RANK.  The *_all entry points encode this rank's items and return the
 *   embeddings of ALL ranks, rank-major (one in-place ncclAllGather on the launch stream; every rank must pass the same count).
 * libnccl.so.2 is dlopen'ed on first use; no torch, no MPI. */
bool clip_b200_dist_unique_id(void * out128);
bool clip_b200_dist_init_with_id(struct clip_ctx * ctx, int rank, int world, const void * id128);
bool clip_b200_dist_init(struct clip_ctx * ctx, int rank, int world, const char * rendezvous);
int  clip_b200_dist_rank(const struct clip_ctx * ctx);
int  clip_b200_dist_world(const struct clip_ctx * ctx);
int  clip_b200_device_count(const struct clip_ctx * ctx);           /* GPUs behind this context (devices mode), else 1 */
int  clip_b200_nccl_version(void);                                  /* 0 when libnccl cannot be loaded */
int  clip_b200_cuda_device_count(void);                             /* visible CUDA devices (0 without a driver) */
bool clip_b200_dist_barrier(const struct clip_ctx * ctx);           /* all ranks + device synchronize */
bool clip_b200_dist_max_f64(const struct clip_ctx * ctx, double * vals, int n);   /* element-wise max over ranks, n <= 16 */
bool clip_b200_dist_all_gather(const struct clip_ctx * ctx, const void * d_send, void * d_recv, size_t bytes_per_rank);
bool clip_b200_image_encode_device_all(const struct clip_ctx * ctx, const void * d_pixels, size_t n_local, void * d_vec_all,
                                       bool normalize);
bool clip_b200_text_encode_device_all(const struct clip_ctx * ctx, const void * d_ids, const void * d_lens, size_t n_local,
                                      int seq_len, void * d_vec_all, bool normalize);
bool clip_b200_image_batch_encode_all(const struct clip_ctx * ctx, const int n_threads, const struct clip_image_f32_batch * imgs,
                                      float * vec_all, const bool normalize);
bool clip_b200_text_batch_encode_all(const struct clip_ctx * ctx, const int n_threads, const struct clip_tokens * seqs,
                                     const size_t n, float * vec_all, const bool normalize);

/* memory + stream helpers so that a plain C caller needs no CUDA headers.  clip_b200_memcpy_h2d returns once the bytes are on the
 * device, so the context's next call reads all of them, pageable source or not. */
void * clip_b200_device_malloc(const struct clip_ctx * ctx, size_t bytes);
void   clip_b200_device_free(const struct clip_ctx * ctx, void * p);
void * clip_b200_host_malloc(size_t bytes);            /* pinned */
void   clip_b200_host_free(void * p);
bool   clip_b200_memcpy_h2d(const struct clip_ctx * ctx, void * d_dst, const void * h_src, size_t bytes);
bool   clip_b200_memcpy_d2h(const struct clip_ctx * ctx, void * h_dst, const void * d_src, size_t bytes);
bool   clip_b200_synchronize(const struct clip_ctx * ctx);
void * clip_b200_get_stream(const struct clip_ctx * ctx);          /* the cudaStream_t every kernel is launched on */

/* images (vision) / sequences (text) processed per pass through the layer stack; 0 keeps the current value.  Workspaces are sized
 * once, at the first encode of a tower: a call after that is ignored for that tower.  A pass must fit 32-bit element offsets:
 * micro_batch x T rows (T = the native token count, or context_length for text) times the widest activation of the tower (3 x
 * hidden, ff, projection_dim, and for vision the padded patch width) must stay below 2^32, e.g. at most 4 080 ViT-L/14 images.
 * A larger value is accepted here but the first encode of that tower is refused with a message naming micro_batch and the limit,
 * before anything is allocated; a smaller value set after that refusal takes effect. */
void   clip_b200_set_micro_batch(const struct clip_ctx * ctx, int images, int sequences);

/* measurement hooks */
uint64_t clip_b200_kernel_launches(const struct clip_ctx * ctx);   /* kernels launched by this context so far */
float    clip_b200_last_device_ms(const struct clip_ctx * ctx);    /* CUDA-event time of the last encode's kernels */
/* per-kernel-class CUDA-event time accumulated since the last call with the same kind (0 GEMM, 1 attention,
 * 2 layernorm, 3 other, 4 the token-row kernel of the *_tokens calls, 5 the position-table resample of the *_hw calls, 6 the
 * attention-probability kernel of ATTENTION entries, 7 the 16-bit search kernel of clip_b200_topk_search_16, 8 the int8 search
 * kernel of clip_b200_topk_search_i8, 9 the binary search kernel of clip_b200_topk_search_b1, 10 the rescore kernel of
 * clip_b200_topk_rescore, 11 the fine scan of clip_b200_ivf_search_16, 12 the k-means update of clip_b200_ivf_train_16 and the row
 * gather of clip_b200_ivf_build_16 and clip_b200_ivfpq_build, 13 the ADC scan of clip_b200_ivfpq_search_16, 14 its lookup tables,
 * the codebook k-means of clip_b200_ivfpq_train_16 and the encoding of clip_b200_ivfpq_encode_16); *count
 * receives the number of launches.  Enabled by env CLIP_B200_PROFILE=1. */
float    clip_b200_kernel_ms(const struct clip_ctx * ctx, int kind, uint64_t * count);
/* CUDA-event stopwatch on the launch stream: mark(slot 0..3), then elapsed(a, b) in ms (-1 on error) */
bool     clip_b200_mark(const struct clip_ctx * ctx, int slot);
float    clip_b200_mark_elapsed_ms(const struct clip_ctx * ctx, int a, int b);
const char * clip_b200_last_error(void);
const char * clip_b200_version(void);

/* TEST HOOK: run one fused-dequant GEMM  Y[M,N] = X[M,K] . W[N,K]^T (+bias) on device 0.
 * w_rows: ggml-format rows of type qtype; x: fp32 host [M,K] (rounded to the operand type on the way in);
 * y_out: fp32 host [M,N].  use_naive=1 runs the scalar debug kernel instead.  EPI_STORE16 scales the first N/2 features by 0.125
 * (the Q scale of head_dim 64).  Returns 0 on success, 5 if the GEMM wrote into the poisoned guard rows that follow row M of its
 * output buffer. */
int clip_b200_debug_gemm(int qtype, int operand_bf16, int M, int N, int K, int epi, int use_naive, const float * x,
                         const void * w_rows, const float * bias, const float * resid_in, float * y_out, float * ms);
/* the same with the Q scale as an argument: EPI_STORE16 writes (acc + bias) * scale on the first N/2 features, as the fused QKV
 * GEMM does with 1/sqrt(head_dim) (1/sqrt(80) for head_dim 80 is not a power of two) */
int clip_b200_debug_gemm_scaled(int qtype, int operand_bf16, int M, int N, int K, int epi, int use_naive, float scale,
                                const float * x, const void * w_rows, const float * bias, const float * resid_in, float * y_out,
                                float * ms);

/* N1 (SURVEY.md section 8f) -- clip_image_batch_preprocess (clip.h:98, clip.cpp:963-1008) on the device, fused with the encode:
 * raw u8 RGB images of any size are uploaded (3 B/pixel), resized (PIL-style antialiased bicubic, a = -0.5), centre-cropped and
 * normalised on the GPU -- bit-identical to clip_image_preprocess -- and encoded like clip_image_batch_encode (clip.h:104). */
bool clip_b200_image_batch_encode_u8(const struct clip_ctx * ctx, const struct clip_image_u8_batch * imgs, float * vec, const bool normalize);
/* the device preprocess alone, results copied back into new[]-allocated clip_image_f32 buffers exactly like
 * clip_image_batch_preprocess fills them (clip.cpp:985-1007) */
bool clip_b200_image_batch_preprocess_device(const struct clip_ctx * ctx, const struct clip_image_u8_batch * in,
                                             struct clip_image_f32_batch * out);

/* TEST HOOK: one attention launch (clip.cpp:1082-1108 / 1363-1388 semantics: softmax(Q K^T [+ causal mask]) V per head, head_dim 64).
 * qkv: fp32 host [nseq*T, 3*H*64], columns Q | K | V with the 1/sqrt(64) scale already applied to Q; out: fp32 host [nseq*T, H*64].
 * use_legacy=1 runs the warp-level mma.sync kernel instead of the wgmma one.  ms (optional): device time of the last of 3 launches. */
int clip_b200_debug_attention(int operand_bf16, int nseq, int T, int H, int causal, int use_legacy, const float * qkv, float * out,
                              float * ms);
/* The same for head_dim 64, 80 or 104: qkv [nseq*T, 3*H*head_dim], the 1/sqrt(head_dim) scale already applied to Q; out
 * [nseq*T, H*head_dim].  At head_dim 104 the hook lays qkv out on the device as the loader lays out the QKV activations, each head
 * padded to 112 columns with zeros.  Returns 2 with a message for any other head_dim, and for use_legacy=1 with head_dim 80 or 104
 * (the legacy kernel is head_dim 64 only). */
int clip_b200_debug_attention_hd(int operand_bf16, int nseq, int T, int H, int head_dim, int causal, int use_legacy, const float * qkv,
                                 float * out, float * ms);
/* The variable-length instance behind the *_mixed calls: nseq non-causal sequences of lens[s] rows packed back to back, qkv
 * [sum lens, 3*H*head_dim] and out [sum lens, H*head_dim], laid out and padded as for clip_b200_debug_attention_hd.  The qkv rows past
 * the last sequence and 128 guard rows after the output are poisoned (0xFF).  Returns 2 for bad arguments, 5 for a launch or kernel
 * error, 6 if a guard row was written. */
int clip_b200_debug_attention_mixed(int operand_bf16, int nseq, const int * lens, int H, int head_dim, const float * qkv, float * out);
/* The same with the causal mask (the instance behind the text *_packed calls): head_dim 64 only, anything else returns 2. */
int clip_b200_debug_attention_mixed_causal(int operand_bf16, int nseq, const int * lens, int H, int head_dim, const float * qkv,
                                           float * out);
/* The attention probabilities of the same qkv (the kernel behind CLIP_B200_TOKENS_ATTENTION): out [nseq, H, R, T] with R = T, or 1
 * with cls_row (query row 0 only), of out_type (0 fp32, 1 fp16, 2 bf16: raw 16-bit values, not widened).  Runs on device 0.  Returns
 * 2 for bad arguments (head_dim other than 64 / 80 / 104, a non-positive size, an unknown out_type), 5 if the kernel wrote into the
 * poisoned guard bytes that follow the output. */
int clip_b200_debug_attention_probs(int operand_bf16, int nseq, int T, int H, int head_dim, int causal, int cls_row, int out_type,
                                    const float * qkv, void * out);

/* TEST HOOKS for the row kernels (csrc/kernels.cu): each runs one launcher on a private stream on device 0 and returns 0 on
 * success (clip_b200_last_error says why not).  Host buffers are fp32 / int32; 16-bit inputs are rounded to the operand type
 * (operand_bf16) on the way in and 16-bit outputs come back widened to fp32.  Device outputs start poisoned (all bits set).
 *
 * LayerNorm over rows x h of x (host [rows, h], placed on the device at row stride in_stride >= h with the gaps poisoned);
 * delta (host [rows, h] or NULL) selects the form that first adds the 16-bit residual branch into x.  y_out [rows, h];
 * x_out [rows, h] (optional): x after the kernel. */
int clip_b200_debug_layernorm(int rows, int h, size_t in_stride, float eps, const float * x, const float * gamma, const float * beta,
                              const float * delta, int operand_bf16, float * y_out, float * x_out);
/* pre-LN assembly: patch [B*(T-1), h], class_embd [h], pos [T, h] -> x_out [B*T, h] fp32 */
int clip_b200_debug_assemble_preln(const float * patch, const float * class_embd, const float * pos, int B, int T, int h, float eps,
                                   const float * gamma, const float * beta, float * x_out);
/* im2col: NHWC pixels [B, S, S, 3] -> fp16 patches [B*(S/P)^2, kpad] (widened to fp32 in out) */
int clip_b200_debug_im2col(const float * pixels, int B, int S, int P, int kpad, float * out);
/* the same for rectangles: [B, H, W, 3] -> [B*(H/P)*(W/P), kpad], patches in row-major grid order */
int clip_b200_debug_im2col_hw(const float * pixels, int B, int H, int W, int P, int kpad, float * out);
/* position-table resample (K8): table [g*g, h] (patch rows only) -> out [gh*gw, h], as the *_hw entry points resample */
int clip_b200_debug_pos_resample(const float * table, int g, int h, int gh, int gw, float * out);
/* text embedding: ids [nseq*T] (clamped to [0, n_vocab)), tok [n_vocab, h], pos [T, h] -> x_out [nseq*T, h] */
int clip_b200_debug_text_embed(const int32_t * ids, const float * tok, const float * pos, int nseq, int T, int h, int n_vocab,
                               float * x_out);
/* row gather: out[r] = src[r*stride_rows + offs[r]] (+ delta[same row]); src and delta (optional) [src_rows, h], offs optional */
int clip_b200_debug_gather_rows(const float * src, int src_rows, int rows, int h, int stride_rows, const int32_t * offs,
                                const float * delta, int operand_bf16, float * out);
/* L2 norm of each row of v [rows, d] (normalize = 0: plain copy) */
int clip_b200_debug_l2norm(const float * v, int rows, int d, int normalize, float * out);
/* EOT row index per sequence: last[i] = clamp(lens ? lens[i] : seq_len, 1, seq_len) - 1 */
int clip_b200_debug_fill_last(const int32_t * lens, int n, int seq_len, int32_t * last);
/* token rows (K7): x host [n*T, h] placed at row stride in_stride (gaps poisoned); out receives rows 1 .. T-1 (no_cls) or 0 .. T-1
 * of each item, [n, T or T-1, h], as out_type (0 fp32, 1 fp16, 2 bf16: raw 16-bit values, not widened); gamma = NULL: no
 * LayerNorm, otherwise post_ln with gamma, beta, eps */
int clip_b200_debug_token_rows(int n, int T, int h, size_t in_stride, int no_cls, float eps, const float * x, const float * gamma,
                               const float * beta, int out_type, void * out);

/* CPU-only TEST HOOKS (no context, no GPU): lossless re-tiling check, tokenizer and preprocess without a model context */
int clip_b200_debug_repack_roundtrip(int qtype, const void * rows, int N, int K);
int clip_b200_debug_rendezvous(int rank, int world, const char * path, void * out128);     /* ranks-mode id exchange (csrc/dist.cpp) */
/* the loader's QKV padding at head_dim 104: src = 3*H*dh rows of a [*, K] weight of ggml type qtype (0 f32, 1 f16, 2/3/6/7/8 the
 * block types; qtype 0 with K = 1 is a bias) -> out = 3*H*dhp rows, each head's dh rows followed by dhp - dh rows of zero bytes.
 * Returns 0, or 1 for bad arguments (dhp < dh, K not a whole number of blocks, an unknown type). */
int clip_b200_debug_pad_qkv(int qtype, int H, int dh, int dhp, int K, const void * src, void * out);
void clip_b200_debug_shard_bounds(size_t n, int r, int w, size_t * lo, size_t * hi);        /* devices-mode sharding rule */
int clip_b200_debug_tokenize(const char * gguf_path, const char * text, int32_t * out, int cap);
int clip_b200_debug_preprocess(const uint8_t * rgb, int nx, int ny, int out_size, const float * mean, const float * stdv,
                               float * out);

#ifdef __cplusplus
}
#endif
#endif /* CLIP_B200_H */
