// gemm_dq.cu -- K1: fused block-dequant GEMM on Hopper warpgroup MMA (sm_90a wgmma).
//
// Replaces ggml_compute_forward_mul_mat + vec_dot_q*_q8_* (reference: ggml/src/ggml.c:11223-11437,
// 2333-3624) for every weight GEMM of the ViT / text transformer (clip.cpp:1080-1137, 1360-1417).
//
//   Y[token, feature] = sum_k X[token, k] * W[feature, k]  (+ bias, + epilogue)
//
// computed "swap-AB": the WEIGHT tile is the wgmma A operand (M = 128 features, 64 per consumer warpgroup), the ACTIVATION tile is
// the B operand (N = 256 tokens); fp32 accumulators live in registers (128 per thread).  Persistent CTA, one per SM, 384 threads; the
// producer warpgroup hands its registers to the consumers (setmaxnreg 40 / 232):
//   warp 8      producer, one thread: per k-block ONE 1-D bulk copy of the packed 32-weight blocks + scales of the [128 x 64] weight
//               tile (wpack.h) into the Q ring, and a TMA box of the activation tile [256 tokens x 64 k] (128-B swizzle) into the X
//               ring; unquantized f16 weights come as a second TMA box [128 features x 64 k] in the same X stage instead
//   warps 0-7   two consumer warpgroups; group g owns features [64 g, 64 g + 64) of the tile.  Quantized weights never exist unpacked in
//               shared memory: every lane dequantises exactly the 16-bit pairs of its own wgmma A fragments (2 rows x 16 k per k-block)
//               from the packed chunk into registers, and the group issues 4 register-A wgmma m64n256k16 per k-block (B = activation
//               tile from shared memory), keeping one k-block of MMAs in flight while it unpacks the next.  f16 weights: both operands
//               from shared memory.  Epilogue: bias / scale / GELU computed from the accumulator registers, written in chunks into a
//               ring of swizzled staging slots in shared memory and sent out by bulk tensor stores that drain while the group runs
//               the next tile's main loop; x += acc + bias into the fp32 residual stream adds to x that TMA brought into the slot
//               (every element has exactly one owner thread: deterministic).  See epilogue_staged.
// Bytes per launch (DESIGN.md section 5): packed W once per token tile, X once per feature tile, Y once; FLOPs = 2*M*N*K.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "gemm.h"
#include "wgmma.cuh"
#include "wpack.h"

namespace cb {

namespace {

constexpr int BM = GEMM_BM, BN = GEMM_BN, BK = GEMM_BK;
constexpr int X_STAGE = BN * BK * 2;   // 32768 B
constexpr int W_STAGE = BM * BK * 2;   // 16384 B (f16 path only)
constexpr int THREADS = 384;           // 2 consumer warpgroups + 1 producer warpgroup (one thread of it issues the copies)
static_assert(X_STAGE % 1024 == 0 && W_STAGE % 1024 == 0, "swizzled stage alignment");

__host__ __device__ constexpr uint32_t chunk_bytes(int qt) {
    return qt == 2 ? 4608u : qt == 3 ? 5120u : qt == 6 ? 5632u : qt == 7 ? 6144u : qt == 8 ? 8704u : 0u;
}
constexpr uint32_t E_SLOT = 4096;   // one epilogue staging slot (epilogue_staged)
// Shared-memory plan per weight type (fits the 227 KB carve-out): X ring, packed-weight ring, epilogue staging (SE slots per consumer
// group, as many as the rings leave room for), barriers.  The producer issues Q(kb) just before it waits for X(kb)'s stage, and the
// consumers release a Q chunk a k-block before its X stage, so no more than SX + 1 Q chunks are ever in use: the Q ring is that deep.
//   q4_0  4 x 32 KB X + 5 x 4.5 KB Q + 2 x 9 x 4 KB        q5_1  4 x 32 KB X + 5 x 6 KB Q + 2 x 8 x 4 KB
//   q4_1  4 x 32 KB X + 5 x 5 KB Q + 2 x 9 x 4 KB          q8_0  4 x 32 KB X + 5 x 8.5 KB Q + 2 x 6 x 4 KB
//   q5_0  4 x 32 KB X + 5 x 5.5 KB Q + 2 x 8 x 4 KB        f16   4 x 48 KB (X + W) + 2 x 4 x 4 KB
template <int QT>
struct Cfg {
    static constexpr bool DQ = (QT != QT_F16);
    static constexpr uint32_t CHUNK = chunk_bytes(QT);
    static constexpr int SX = 4;                                       // X ring (f16: X + W per stage)
    static constexpr int SQ = DQ ? SX + 1 : 0;                         // packed-weight ring
    static constexpr uint32_t XS = DQ ? (uint32_t)X_STAGE : (uint32_t)(X_STAGE + W_STAGE);
    static constexpr uint32_t Q_OFF = SX * XS;
    static constexpr uint32_t E_OFF = (Q_OFF + SQ * CHUNK + 1023) / 1024 * 1024;   // swizzled slots: 1024-byte aligned
    static constexpr int SE = (232448 - 512 - 1024 - E_OFF) / (2 * E_SLOT);
    static constexpr uint32_t BAR_OFF = E_OFF + 2 * SE * E_SLOT;
    static constexpr uint32_t SMEM = BAR_OFF + 512 /*barriers*/ + 1024 /*align slack*/;
    static_assert(SMEM <= 232448, "shared memory plan exceeds 227 KB");
    static_assert(16 * SX + 16 * SQ + 16 * SE <= 512, "barrier area");
};

struct KParams {
    CUtensorMap tm_x;
    CUtensorMap tm_w;
    CUtensorMap tm_out;   // Y [M, N]: exactly M rows, so bulk stores clip a ragged last tile; boxes of one staging chunk
    const uint8_t* w_packed;
    const float* bias;
    int M, N, K;
    int epi, scale_cols;
    float scale;
};

// explicit .shared accesses on 32-bit shared-window addresses (generic ld/st would cost an address-space check)
CB_DEVINL uint4 lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
CB_DEVINL uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
CB_DEVINL uint16_t lds16(uint32_t a) { uint16_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a)); return v; }
// (a & MASK) | c  and  (a & MASK) ^ c  as ONE LOP3 each (nvcc splits the C expression into two when mask and c are both
// immediates: LOP3 takes a single immediate, so c is handed over in a register)
template <uint32_t MASK>
CB_DEVINL uint32_t and_or(uint32_t a, uint32_t c) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(a), "n"(MASK), "r"(c));
    return r;
}
template <uint32_t MASK>
CB_DEVINL uint32_t and_xor(uint32_t a, uint32_t c) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0x6A;" : "=r"(r) : "r"(a), "n"(MASK), "r"(c));
    return r;
}
CB_DEVINL uint32_t opaque_const(uint32_t v) {      // a constant the optimiser keeps in a register
    uint32_t r;
    asm volatile("mov.b32 %0, %1;" : "=r"(r) : "r"(v));
    return r;
}
CB_DEVINL uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}

// Unpack four 16-bit weight pairs of the 32-weight ggml block b (= half*128 + row) of a packed [128 x 64] tile (wpack.h): v[j] holds
// block elements 8j + 2t and 8j + 2t + 1 (t = lane % 4), i.e. what one lane contributes to the wgmma A fragments of the block's two
// 16-wide k steps.  Arithmetic matches dequantize_row_q* (ggml/src/ggml.c:1496-1606): (q - zero) * d  or  q * d + m, with the integer
// part exact (magic-number int->float) and ONE rounding of the product to the operand type.
template <int QT, bool BF>
CB_DEVINL void unpack_pairs(uint32_t q, int b, int t, uint32_t (&v)[4]) {
    using P = P2<BF>;
    if constexpr (QT == QT_Q8_0) {
        const uint32_t d2 = P::splat_from_f16bits(lds16(q + 8192 + 2 * b));
        const uint32_t wa = q + 16 * b + 4 * (t >> 1), wb = wa + 4096;          // qa: elements 0..15, qb: 16..31, 4 per word
        const uint32_t words[4] = {lds32(wa), lds32(wa + 8), lds32(wb), lds32(wb + 8)};
        const uint32_t sel = (t & 1) ? 0x4342u : 0x4140u;                       // bytes of elements 2t, 2t+1 -> 16-bit lanes
        const uint32_t magic = opaque_const(P::MAGIC), c4380 = opaque_const(0x43804380u);
        (void)magic; (void)c4380;
        #pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t pr = prmt(words[j] ^ 0x80808080u, 0u, sel);          // int8 -> biased 0..255
            if constexpr (!BF) {   // fp16: 1024 + s is exact, minus 1152 = signed quant
                v[j] = P::mul(P::sub(pr | P::MAGIC, 0x64806480u), d2);
            } else {               // bf16 has 7 mantissa bits: 128 + (s & 127), minus 128 or 256 by bit 7
                v[j] = P::mul(P::sub(and_or<0x007f007fu>(pr, magic), and_xor<0x00800080u>(pr, c4380)), d2);
            }
        }
    } else {
        constexpr bool Q5 = (QT == QT_Q5_0 || QT == QT_Q5_1);
        constexpr bool AFFINE = (QT == QT_Q4_1 || QT == QT_Q5_1);
        const uint4 qs = lds128(q + 16 * b);
        uint32_t hq = 0;
        uint32_t off = 4096;
        if constexpr (Q5) { hq = lds32(q + off + 4 * b); off += 1024; }
        uint32_t d2, m2 = 0;
        if constexpr (AFFINE) {
            const uint32_t dm = lds32(q + off + 4 * b);
            d2 = P::splat_from_f16bits((uint16_t)(dm & 0xffffu));
            m2 = P::splat_from_f16bits((uint16_t)(dm >> 16));
        } else {
            d2 = P::splat_from_f16bits(lds16(q + off + 2 * b));
        }
        // zero point folded into the exact integer subtraction: 8 (q4_0), 16 (q5_0), 0 (q4_1 / q5_1)
        constexpr uint32_t ZP = (QT == QT_Q4_0) ? 8u : (QT == QT_Q5_0) ? 16u : 0u;
        constexpr uint32_t C2 = P::MAGIC + (ZP | (ZP << 16));
        const uint32_t words[4] = {qs.x, qs.y, qs.z, qs.w};
        const uint32_t magic = opaque_const(P::MAGIC);
        #pragma unroll
        for (int j = 0; j < 4; j++) {
            uint32_t x = and_or<0x000f000fu>(words[j] >> (4 * t), magic);       // pair t of word j: elements 8j + 2t, 8j + 2t + 1
            if constexpr (Q5) {
                const int sh = 4 * j + t;   // 5th bits of this pair sit at bits sh and sh+16 -> move to bits 4 / 20
                const uint32_t hb = (sh >= 4) ? (hq >> (sh - 4)) : (hq << (4 - sh));
                x = and_or<0x00100010u>(hb, x);
            }
            const uint32_t qv = P::sub(x, C2);
            v[j] = AFFINE ? P::fma(qv, d2, m2) : P::mul(qv, d2);
        }
    }
}

// wgmma A fragments of one 64-deep k-block for this lane: tile rows r and r + 8, t = lane % 4.  k step s = 2 half + u covers elements
// 16u .. 16u + 15 of ggml block (row, half); a[4s + 0 / 1] = rows r / r + 8 at k 2t, 2t + 1, a[4s + 2 / 3] = the same rows at k 2t + 8, 2t + 9.
template <int QT, bool BF>
CB_DEVINL void unpack_frag(uint32_t q, int r, int t, uint32_t (&a)[16]) {
    #pragma unroll
    for (int half = 0; half < 2; half++) {
        #pragma unroll
        for (int h8 = 0; h8 < 2; h8++) {
            uint32_t v[4];
            unpack_pairs<QT, BF>(q, half * 128 + r + 8 * h8, t, v);
            #pragma unroll
            for (int u = 0; u < 2; u++) {
                a[4 * (2 * half + u) + h8] = v[2 * u];
                a[4 * (2 * half + u) + 2 + h8] = v[2 * u + 1];
            }
        }
    }
}

// register budget of the calling warpgroup (all its threads execute it): producer down, consumers up
template <int N>
CB_DEVINL void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
CB_DEVINL void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// keeps the compiler from reusing a register an in-flight wgmma may still read before the wgmma_wait that retires it
CB_DEVINL void fence_frag(uint32_t (&a)[16]) {
    #pragma unroll
    for (int i = 0; i < 16; i++) asm volatile("" : "+r"(a[i])::"memory");
}

// 16-bit epilogue value of one accumulator element.  EPI_STORE16 rounds (acc + b) to fp32 before the scale, the reference's order
// (ggml_add then ggml_scale, clip.cpp:1082, 1363): the Q scale 1/sqrt(80) of head_dim 80 is not a power of two, so a single FFMA
// with a pre-scaled bias would round differently.  For 1/sqrt(64) = 0.125 the two forms give the same bits.  The GELUs are
// common.cuh's, which the scalar debug kernel runs too.
template <int EPI>
CB_DEVINL float epi_value(float acc, float bias, float mul) {
    if constexpr (EPI == EPI_GELU16) return gelu_tanh(acc + bias);
    else if constexpr (EPI == EPI_QGELU16) return gelu_quick(acc + bias);
    else return (acc + bias) * mul;
}

// ---- epilogue staging: bulk tensor stores (and, for the residual add, loads) between the staging slots and the output matrix
CB_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
CB_DEVINL void group_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }   // the 128 threads of one group
CB_DEVINL void tma_store_2d(const void* tmap, uint32_t src_smem, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(tmap)),
                 "r"(src_smem), "r"(c0), "r"(c1)
                 : "memory");
}
CB_DEVINL void tma_prefetch_l2(const void* tmap, int c0, int c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1)
                 : "memory");
}
CB_DEVINL void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
CB_DEVINL void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }   // sources reusable
CB_DEVINL void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }                // writes complete
CB_DEVINL float lds_f32(uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a)); return v; }
CB_DEVINL void sts_f32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
// four 8x8 16-bit matrices from accumulator-layout fragments, each stored transposed: row i of matrix m (address of lane 8m + i)
// receives column i of the fragment, i.e. 8 features of one token
CB_DEVINL void stmatrix_x4_trans(uint32_t a, const uint32_t (&r)[4]) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(r[0]), "r"(r[1]), "r"(r[2]),
                 "r"(r[3])
                 : "memory");
}

// Output rectangle of one consumer group: [256 tokens x 64 features] of Y, staged through a ring of SE slots of E_SLOT bytes in
// shared memory, laid out [token][feature] with the 128-byte swizzle of the output tensor map (rows of 128 B, 16-byte piece p of row
// r at p ^ (r & 7)).  A chunk fills one slot: 32 tokens x 64 features of 16-bit values (one box), or 16 tokens x 64 features of fp32
// (two boxes of 32 features).  Chunks past the last token are skipped; the map's M rows clip the rest of a ragged tile.
constexpr int TC16 = E_SLOT / 128, TC32 = E_SLOT / 256;   // tokens per chunk
template <int EPI>
struct EpiShape {
    static constexpr bool F32 = (EPI == EPI_STORE32 || EPI == EPI_REDADD32);
    static constexpr int TC = F32 ? TC32 : TC16;
    static constexpr int CH = BN / TC;                     // chunks per tile
};
CB_DEVINL int epi_chunks(int m_left, int tc) { return min(BN / tc, (m_left + tc - 1) / tc); }

// x of the residual add: the leader thread loads chunk n of the tile (sequence number e) into its slot
template <int SE>
CB_DEVINL void load_x_chunk(const KParams& p, uint32_t ring, uint32_t full, uint32_t e, int tok0, int f0, int n) {
    const uint32_t s = e % SE, dst = ring + s * E_SLOT;
    mbar_arrive_expect_tx(full + 8 * s, E_SLOT);          // rows past M are zero-filled and still counted
    tma_load_2d(dst, &p.tm_out, f0, tok0 + n * TC32, full + 8 * s);
    tma_load_2d(dst + E_SLOT / 2, &p.tm_out, f0 + 32, tok0 + n * TC32, full + 8 * s);
}
// Residual add, from the middle of a tile's main loop: the leader loads the tile's first SE chunks of x into the group's slots (the
// previous tile's stores read them long ago) and has L2 fetch the others, which the epilogue then loads from L2.
template <int SE>
CB_DEVINL void prefetch_x(const KParams& p, uint32_t ring, uint32_t full, uint32_t e, int tok0, int f0) {
    const int nch = epi_chunks(p.M - tok0, TC32);
    bulk_wait_read<0>();
    for (int n = 0; n < nch; n++) {
        if (n < SE) {
            load_x_chunk<SE>(p, ring, full, e + n, tok0, f0, n);
        } else {
            tma_prefetch_l2(&p.tm_out, f0, tok0 + n * TC32);
            tma_prefetch_l2(&p.tm_out, f0 + 32, tok0 + n * TC32);
        }
    }
}

// Epilogue of one consumer group's [64 features x 256 tokens] accumulator (fragment layout: wgmma.cuh): this thread (warp w of the
// group) owns features 16w + lane/4 (+ 8) and tokens 8j + 2 (lane % 4) + {0, 1}.  Per chunk: the values go into the slot, every
// thread fences them to the async proxy, the group syncs and its leader thread issues the bulk store; nobody waits for the store.
// A slot is written again only after the store that read it is past its source (the leader's wait_group.read before the group
// barrier).  Residual add: the slot already holds the chunk's x (load_x_chunk: the first SE chunks during the main loop, chunk n + SE
// once the store of chunk n has read the slot); x + (acc + bias) is written back in place.  `e` numbers this group's chunks.
template <int EPI, bool BF, int SE>
CB_DEVINL void epilogue_staged(const KParams& p, const float (&acc)[BN / 2], int tok0, int f0, int w, int lane, const float (&bias)[2],
                               const float (&mul)[2], uint32_t ring, uint32_t full, uint32_t& e, bool leader, int bar_id) {
    using S = EpiShape<EPI>;
    static_assert(SE >= 2, "a staging ring needs two slots");
    const int nch = epi_chunks(p.M - tok0, S::TC);
    #pragma unroll
    for (int c = 0; c < S::CH; c++) {
        if (c >= nch) break;
        const uint32_t slot = ring + (e % SE) * E_SLOT;
        if constexpr (!S::F32) {
            const int m = lane >> 3, rr = lane & 7;
            #pragma unroll
            for (int jp = 0; jp < TC16 / 16; jp++) {
                const int j = c * (TC16 / 8) + 2 * jp;     // token groups j and j + 1: matrices (j, f), (j, f + 8), (j + 1, f), (j + 1, f + 8)
                uint32_t r[4];
                #pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int i = 4 * (j + (q >> 1)) + 2 * (q & 1), h = q & 1;
                    r[q] = (uint32_t)P2<BF>::from_float(epi_value<EPI>(acc[i], bias[h], mul[h])) |
                           ((uint32_t)P2<BF>::from_float(epi_value<EPI>(acc[i + 1], bias[h], mul[h])) << 16);
                }
                const uint32_t row = 16 * jp + 8 * (m >> 1) + rr;
                stmatrix_x4_trans(slot + row * 128 + ((uint32_t)((2 * w + (m & 1)) ^ rr) << 4), r);
            }
        } else {
            if constexpr (EPI == EPI_REDADD32) mbar_wait(full + 8 * (e % SE), (e / SE) & 1);
            #pragma unroll
            for (int jj = 0; jj < TC32 / 8; jj++) {
                #pragma unroll
                for (int q = 0; q < 4; q++) {
                    const uint32_t row = 8 * jj + 2 * (lane & 3) + (q & 1);
                    const uint32_t piece = 4 * (w & 1) + 2 * (q >> 1) + (lane >> 4);
                    const uint32_t a = slot + (w >> 1) * (E_SLOT / 2) + row * 128 + ((piece ^ (row & 7)) << 4) + 4 * ((lane >> 2) & 3);
                    const float v = acc[4 * (c * (TC32 / 8) + jj) + q] + bias[q >> 1];
                    if constexpr (EPI == EPI_REDADD32) sts_f32(a, lds_f32(a) + v);
                    else sts_f32(a, v);
                }
            }
        }
        fence_proxy_async();
        if constexpr (EPI != EPI_REDADD32) {
            if (leader) bulk_wait_read<SE - 2>();          // the store of chunk e + 1 - SE has read the slot chunk e + 1 will write
        }
        group_bar(bar_id);
        if (leader) {
            const int row = tok0 + c * S::TC;
            if constexpr (S::F32) {
                tma_store_2d(&p.tm_out, slot, f0, row);
                tma_store_2d(&p.tm_out, slot + E_SLOT / 2, f0 + 32, row);
            } else {
                tma_store_2d(&p.tm_out, slot, f0, row);
            }
            bulk_commit();
            if constexpr (EPI == EPI_REDADD32) {
                if (c >= 1 && c - 1 + SE < nch) {              // the slot of chunk c - 1 is free once its store has read it
                    bulk_wait_read<1>();
                    load_x_chunk<SE>(p, ring, full, e - 1 + SE, tok0, f0, c - 1 + SE);
                }
            }
        }
        __syncwarp();
        e++;
    }
}

template <int QT, bool BF>
__global__ void __launch_bounds__(THREADS, 1) gemm_dq_kernel(const __grid_constant__ KParams p) {
    using C = Cfg<QT>;
    constexpr bool DQ = C::DQ;
    constexpr int SX = C::SX, SQ = DQ ? C::SQ : 1, SE = C::SE;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t bars = smem_base + C::BAR_OFF;
    // barrier slots (8 B each); e_full: x of the residual add arrived in a staging slot (SE per consumer group)
    const uint32_t x_full = bars, x_empty = x_full + 8 * SX, q_full = x_empty + 8 * SX, q_empty = q_full + 8 * SQ,
                   e_full = q_empty + 8 * SQ;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < SX; i++) { mbar_init(x_full + 8 * i, 1); mbar_init(x_empty + 8 * i, 8); }   // released by each consumer warp
        for (int i = 0; i < SQ; i++) { mbar_init(q_full + 8 * i, 1); mbar_init(q_empty + 8 * i, 8); }
        for (int i = 0; i < 2 * SE; i++) mbar_init(e_full + 8 * i, 1);
        mbar_fence_init();
        tma_prefetch_desc(&p.tm_x);
        if (!DQ) tma_prefetch_desc(&p.tm_w);
        tma_prefetch_desc(&p.tm_out);
    }
    __syncthreads();
    pdl_trigger();      // the next kernel of the stream may start placing CTAs as ours retire ...
    pdl_wait();         // ... and we touch global memory only after the previous grid has completed

    // work units: [128 features x 256 tokens] tiles, feature tile fastest (CTAs running at the same time share their X tile in L2)
    const int n_ft = p.N / BM, n_tt = (p.M + BN - 1) / BN, n_tiles = n_ft * n_tt, nkb = p.K / BK;

    if (warp >= 8) {
        // ------------------------------------------------------------------ producer (one thread)
        setmaxnreg_dec<40>();
        if (warp == 8 && lane == 0) {
            uint32_t s = 0, ph = 0, qs = 0, qph = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const int ft = tile % n_ft, tt = tile / n_ft;
                for (int kb = 0; kb < nkb; kb++) {
                    if constexpr (DQ) {
                        mbar_wait(q_empty + 8 * qs, qph ^ 1);
                        mbar_arrive_expect_tx(q_full + 8 * qs, C::CHUNK);
                        bulk_load_1d(smem_base + C::Q_OFF + qs * C::CHUNK, p.w_packed + ((size_t)ft * nkb + kb) * C::CHUNK, C::CHUNK, q_full + 8 * qs);
                        if (++qs == SQ) { qs = 0; qph ^= 1; }
                    }
                    mbar_wait(x_empty + 8 * s, ph ^ 1);
                    mbar_arrive_expect_tx(x_full + 8 * s, C::XS);      // rows past M are zero-filled and still counted
                    tma_load_2d(smem_base + s * C::XS, &p.tm_x, kb * BK, tt * BN, x_full + 8 * s);
                    if constexpr (!DQ) tma_load_2d(smem_base + s * C::XS + X_STAGE, &p.tm_w, kb * BK, ft * BM, x_full + 8 * s);
                    if (++s == SX) { s = 0; ph ^= 1; }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int fr = (warp & 3) * 16 + (lane >> 2);   // accumulator row (feature in the group)
    const bool leader = (threadIdx.x & 127) == 0;   // issues this group's bulk stores and residual loads
    const uint32_t ring = smem_base + C::E_OFF + (uint32_t)wg * SE * E_SLOT, ring_full = e_full + 8 * SE * wg;
    uint32_t s = 0, ph = 0, qs = 0, qph = 0, e = 0;
    float acc[BN / 2];
    uint32_t afr0[16], afr1[16];      // A fragments of two consecutive k-blocks: one is read by in-flight MMAs while the next is unpacked
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int ft = tile % n_ft, tt = tile / n_ft;
        const int tok0 = tt * BN, f0 = ft * BM + wg * 64;
        uint32_t prev = 0;
        auto kblock = [&](uint32_t (&a)[16], uint32_t (&other)[16], int kb) {
            if constexpr (DQ) {
                mbar_wait(q_full + 8 * qs, qph);
                unpack_frag<DQ ? QT : QT_Q4_0, BF>(smem_base + C::Q_OFF + qs * C::CHUNK, wg * 64 + fr, lane & 3, a);
                __syncwarp();
                if (lane == 0) mbar_arrive(q_empty + 8 * qs);
                if (++qs == SQ) { qs = 0; qph ^= 1; }
            }
            mbar_wait(x_full + 8 * s, ph);
            const uint64_t db = wgmma_desc_sw128(smem_base + s * C::XS);
            wgmma_fence();
            if constexpr (DQ) {
                #pragma unroll
                for (int k = 0; k < BK / 16; k++) {
                    const uint32_t ak[4] = {a[4 * k], a[4 * k + 1], a[4 * k + 2], a[4 * k + 3]};
                    wgmma_rs_n256<BF>(acc, ak, db + 2 * k, (uint32_t)(kb | k));                      // B: +16 k = +32 B
                }
            } else {
                const uint64_t da = wgmma_desc_sw128(smem_base + s * C::XS + X_STAGE + (uint32_t)wg * 64u * 128u);
                #pragma unroll
                for (int k = 0; k < BK / 16; k++) wgmma_ss_n256<BF>(acc, da + 2 * k, db + 2 * k, (uint32_t)(kb | k));
            }
            wgmma_commit();
            wgmma_wait<1>();            // the MMAs of k-block kb-1 are done: release its X stage, its A fragments may be overwritten
            fence_frag(other);
            if (kb > 0) { __syncwarp(); if (lane == 0) mbar_arrive(x_empty + 8 * prev); }
            prev = s;
            if (++s == SX) { s = 0; ph ^= 1; }
            if (p.epi == EPI_REDADD32 && kb == nkb / 2) {
                if (leader) prefetch_x<SE>(p, ring, ring_full, e, tok0, f0);
                __syncwarp();
            }
        };
        int kb = 0;
        for (; kb + 1 < nkb; kb += 2) { kblock(afr0, afr1, kb); kblock(afr1, afr0, kb + 1); }
        if (kb < nkb) kblock(afr0, afr1, kb);
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        fence_frag(afr0);
        fence_frag(afr1);
        __syncwarp();
        if (lane == 0) mbar_arrive(x_empty + 8 * prev);

        const int f = f0 + fr;
        float mul[2], bias[2];
        #pragma unroll
        for (int h = 0; h < 2; h++) {
            mul[h] = (f + 8 * h < p.scale_cols) ? p.scale : 1.0f;
            bias[h] = p.bias ? p.bias[f + 8 * h] : 0.0f;
        }
#define CB_EPI(E) epilogue_staged<E, BF, SE>(p, acc, tok0, f0, warp & 3, lane, bias, mul, ring, ring_full, e, leader, 1 + wg)
        switch (p.epi) {
        case EPI_STORE16: CB_EPI(EPI_STORE16); break;
        case EPI_GELU16: CB_EPI(EPI_GELU16); break;
        case EPI_QGELU16: CB_EPI(EPI_QGELU16); break;
        case EPI_REDADD32: CB_EPI(EPI_REDADD32); break;
        default: CB_EPI(EPI_STORE32); break;
        }
#undef CB_EPI
        // the last tile's stores have written Y before the grid counts as complete (and shared memory goes away).  Inside the loop:
        // the same wait after it makes ptxas serialize the wgmmas for want of registers.
        if (leader && tile + (int)gridDim.x >= n_tiles) bulk_wait_all();
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

template <int QT, bool BF>
cudaError_t launch_t(const KParams& kp, int grid, cudaStream_t st) {
    return launch_pdl(gemm_dq_kernel<QT, BF>, (unsigned)grid, (unsigned)THREADS, Cfg<QT>::SMEM, st, 1, kp);
}
template <int QT, bool BF>
cudaError_t set_attr() {
    return cudaFuncSetAttribute(gemm_dq_kernel<QT, BF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<QT>::SMEM);
}

}  // namespace

bool make_tma_2d_16bit(TmaMap* out, const void* gptr, uint64_t rows, uint64_t cols, uint64_t row_stride_elems,
                       uint32_t box_rows) {
    static_assert(sizeof(CUtensorMap) == sizeof(TmaMap), "CUtensorMap size");
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {row_stride_elems * 2};
    const cuuint32_t box[2] = {(cuuint32_t)GEMM_BK, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(reinterpret_cast<CUtensorMap*>(out), CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(gptr), dims,
                     strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

cudaError_t gemm_init() {
    cudaError_t e;
    if ((e = set_attr<QT_F16, false>()) != cudaSuccess) return e;
#define CB_SET(QT)                                                  \
    if ((e = set_attr<QT, false>()) != cudaSuccess) return e;      \
    if ((e = set_attr<QT, true>()) != cudaSuccess) return e;
    CB_SET(QT_Q4_0) CB_SET(QT_Q4_1) CB_SET(QT_Q5_0) CB_SET(QT_Q5_1) CB_SET(QT_Q8_0)
#undef CB_SET
    return cudaSuccess;
}

cudaError_t gemm_launch(const GemmArgs& a, cudaStream_t stream, int num_sms, uint64_t* launches) {
    if (a.M <= 0) return cudaSuccess;
    if (a.N % BM || a.K % BK || !a.x_map || !a.out) return cudaErrorInvalidValue;
    if ((unsigned long long)a.M * (unsigned long long)a.ldo >= (1ull << 32)) return cudaErrorInvalidValue;   // 32-bit element offsets
    if ((a.epi == EPI_STORE16 || a.epi == EPI_GELU16 || a.epi == EPI_QGELU16) && (a.out_bf16 != 0) != a.operand_bf16) return cudaErrorInvalidValue;
    if (a.qtype == QT_F16 && (a.operand_bf16 || !a.w_map)) return cudaErrorInvalidValue;
    if (a.qtype != QT_F16 && !a.w_packed) return cudaErrorInvalidValue;
    // the output map: Y [M, N] with row stride ldo, one staging chunk per box (epilogue_staged); a bulk tensor copy needs a 16-byte
    // aligned base and row stride
    const bool out32 = (a.epi == EPI_STORE32 || a.epi == EPI_REDADD32);
    const uint64_t row_bytes = (uint64_t)a.ldo * (out32 ? 4 : 2);
    if (a.ldo < a.N || reinterpret_cast<uintptr_t>(a.out) % 16 || row_bytes % 16) return cudaErrorInvalidValue;
    EncodeTiledFn enc = get_encode();
    if (!enc) return cudaErrorInvalidValue;
    KParams kp;
    {
        const cuuint64_t dims[2] = {(cuuint64_t)a.N, (cuuint64_t)a.M};
        const cuuint64_t strides[1] = {row_bytes};
        const cuuint32_t box[2] = {out32 ? 32u : 64u, (cuuint32_t)(out32 ? TC32 : TC16)};
        const cuuint32_t estr[2] = {1, 1};
        if (enc(&kp.tm_out, out32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, a.out, dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return cudaErrorInvalidValue;
    }
    memcpy(&kp.tm_x, a.x_map, sizeof(CUtensorMap));
    if (a.w_map) memcpy(&kp.tm_w, a.w_map, sizeof(CUtensorMap));
    else memset(&kp.tm_w, 0, sizeof(CUtensorMap));
    kp.w_packed = a.w_packed;
    kp.bias = a.bias;
    kp.M = a.M; kp.N = a.N; kp.K = a.K;
    kp.epi = a.epi; kp.scale_cols = a.scale_cols; kp.scale = a.scale;
    const int n_tiles = (a.N / BM) * ((a.M + BN - 1) / BN);
    const int grid = n_tiles < num_sms ? n_tiles : num_sms;
    if (launches) ++*launches;
    switch (a.qtype) {
    case QT_F16: return launch_t<QT_F16, false>(kp, grid, stream);
#define CB_CASE(QT) case QT: return a.operand_bf16 ? launch_t<QT, true>(kp, grid, stream) : launch_t<QT, false>(kp, grid, stream);
    CB_CASE(QT_Q4_0) CB_CASE(QT_Q4_1) CB_CASE(QT_Q5_0) CB_CASE(QT_Q5_1) CB_CASE(QT_Q8_0)
#undef CB_CASE
    default: return cudaErrorInvalidValue;
    }
}

}  // namespace cb
