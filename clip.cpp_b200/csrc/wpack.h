// wpack.h -- HBM layout of quantized GEMM weights ("re-tiled once at load", SURVEY.md section 7 step 2).
//
// ggml stores a [N, K] weight as N rows of K/32 blocks (18/20/22/24/34 B each; ggml/src/ggml.c:866-911):
// not 16-B aligned, scales interleaved with quants.  The loader re-tiles every GEMM weight so that ONE
// 1-D TMA bulk copy (cp.async.bulk, 16-B aligned, contiguous) brings the packed blocks + scales of a
// [128 features x 64 k] tile into shared memory, and each of the 256 unpack threads reads its 32-weight
// block with conflict-free 128-bit loads.  Values are preserved bit for bit (same quants, same fp16 d/m);
// only their order in memory changes.
//
// A weight [N, K] (N % 128 == 0, K % 64 == 0) becomes (N/128) x (K/64) chunks, chunk (ft, kb) at byte
// offset (ft * (K/64) + kb) * wpack_chunk_bytes(type).  Inside a chunk, unpack thread t = half*128 + r
// owns ggml block (row ft*128 + r, block index kb*2 + half):
//
//   q4_0 : qs[256][16 B]  | d [256] f16
//   q4_1 : qs[256][16 B]  | dm[256] {f16 d, f16 m}
//   q5_0 : qs[256][16 B]  | qh[256] u32 | d [256] f16
//   q5_1 : qs[256][16 B]  | qh[256] u32 | dm[256] {f16 d, f16 m}
//   q8_0 : qa[256][16 B]  | qb[256][16 B] | d[256] f16          (qa = elements 0..15, qb = 16..31, natural order)
//
// 4/5-bit: the 16-B `qs` entry is four u32 words; word j holds block elements 8j..8j+7 with element e at bit
// (e>>1)*4 + (e&1)*16, so that ((word >> 4i) & 0x000f000f) is the adjacent pair (8j+2i, 8j+2i+1) already in
// 16-bit-lane order.  q5 `qh`: 5th bit of element 8j+e at bit 4j + (e>>1) + 16*(e&1).
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace cb {

constexpr int WPACK_ROWS = 128;   // features per GEMM tile (two wgmma M = 64 warpgroups)
constexpr int WPACK_K = 64;       // k per tile (one 128-B swizzle row of 16-bit operands)

inline size_t wpack_chunk_bytes(int qtype) {
    switch (qtype) {
    case 2: return 4096 + 512;            // q4_0
    case 3: return 4096 + 1024;           // q4_1
    case 6: return 4096 + 1024 + 512;     // q5_0
    case 7: return 4096 + 1024 + 1024;    // q5_1
    case 8: return 8192 + 512;            // q8_0
    default: return 0;
    }
}
inline size_t wpack_ggml_block_bytes(int qtype) {
    switch (qtype) {
    case 2: return 18;
    case 3: return 20;
    case 6: return 22;
    case 7: return 24;
    case 8: return 34;
    default: return 0;
    }
}
inline size_t wpack_total_bytes(int qtype, int64_t N, int64_t K) {
    return (size_t)(N / WPACK_ROWS) * (size_t)(K / WPACK_K) * wpack_chunk_bytes(qtype);
}

// Host-side re-tiling of one ggml quantized weight [N, K] (row-major blocks) into `dst`.
// Returns false if the shape cannot be tiled.
bool wpack_repack(int qtype, const uint8_t* src, int64_t N, int64_t K, uint8_t* dst);

// Row padding of the fused QKV projection (kernels.h: qkv_head_cols): `rows` rows of `row_bytes` bytes, in groups of dh rows (one
// head of Q, K or V), become groups of dhp rows: the dh source rows, then dhp - dh rows of zero bytes.  All-zero bytes are an exact
// zero in f32, f16 and every ggml block type (d = m = 0), so the padded output features of the GEMM are exact zeros.  Returns false
// unless rows % dh == 0 and dhp >= dh.
bool pad_head_rows(const uint8_t* src, size_t row_bytes, int64_t rows, int dh, int dhp, uint8_t* dst);

// Inverse (used by the unit tests to prove the re-tiling is lossless).
bool wpack_unpack(int qtype, const uint8_t* packed, int64_t N, int64_t K, uint8_t* dst_ggml);

}  // namespace cb
