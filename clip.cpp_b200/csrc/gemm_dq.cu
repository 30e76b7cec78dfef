// gemm_dq.cu -- K1: fused block-dequant GEMM on Hopper warpgroup MMA (sm_90a wgmma).
//
// Replaces ggml_compute_forward_mul_mat + vec_dot_q*_q8_* (reference: ggml/src/ggml.c:11223-11437,
// 2333-3624) for every weight GEMM of the ViT / text transformer (clip.cpp:1080-1137, 1360-1417).
//
//   Y[token, feature] = sum_k X[token, k] * W[feature, k]  (+ bias, + epilogue)
//
// computed "swap-AB": the WEIGHT tile is the wgmma A operand (M = 128 features, 64 per consumer warpgroup), the ACTIVATION tile is
// the B operand (N = 192 tokens); fp32 accumulators live in registers (96 per thread).  Persistent CTA, one per SM, 384 threads; the
// producer warpgroup hands its registers to the consumers (setmaxnreg 40 / 232):
//   warp 8      producer, one thread: per k-block ONE 1-D bulk copy of the packed 32-weight blocks + scales of the [128 x 64] weight
//               tile (wpack.h) into the Q ring, and a TMA box of the activation tile [192 tokens x 64 k] (128-B swizzle) into the X
//               ring; unquantized f16 weights come as a second TMA box [128 features x 64 k] in the same X stage instead
//   warps 0-7   two consumer warpgroups; group g owns features [64 g, 64 g + 64) of the tile.  Quantized weights never exist unpacked in
//               shared memory: every lane dequantises exactly the 16-bit pairs of its own wgmma A fragments (2 rows x 16 k per k-block)
//               from the packed chunk into registers, and the group issues 4 register-A wgmma m64n192k16 per k-block (B = activation
//               tile from shared memory), keeping one k-block of MMAs in flight while it unpacks the next.  f16 weights: both operands
//               from shared memory.  Epilogue straight from the accumulator registers: bias / scale / GELU and 16-bit or fp32 stores,
//               or x += acc + bias into the fp32 residual stream (every element has exactly one owner thread: deterministic), its x
//               values read in four batches of independent loads (epilogue_regs).
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
constexpr int X_STAGE = BN * BK * 2;   // 24576 B
constexpr int W_STAGE = BM * BK * 2;   // 16384 B (f16 path only)
constexpr int THREADS = 384;           // 2 consumer warpgroups + 1 producer warpgroup (one thread of it issues the copies)
static_assert(X_STAGE % 1024 == 0 && W_STAGE % 1024 == 0, "swizzled stage alignment");

__host__ __device__ constexpr uint32_t chunk_bytes(int qt) {
    return qt == 2 ? 4608u : qt == 3 ? 5120u : qt == 6 ? 5632u : qt == 7 ? 6144u : qt == 8 ? 8704u : 0u;
}
// shared-memory plan per weight type (fits the 227 KB carve-out): X ring, packed-weight ring, barriers
template <int QT>
struct Cfg {
    static constexpr bool DQ = (QT != QT_F16);
    static constexpr uint32_t CHUNK = chunk_bytes(QT);
    static constexpr int SX = DQ ? 6 : 5;                              // X ring (f16: X + W per stage)
    static constexpr int SQ = DQ ? 8 : 0;                              // packed-weight ring
    static constexpr uint32_t XS = DQ ? (uint32_t)X_STAGE : (uint32_t)(X_STAGE + W_STAGE);
    static constexpr uint32_t Q_OFF = SX * XS;
    static constexpr uint32_t BAR_OFF = (Q_OFF + SQ * CHUNK + 127) / 128 * 128;
    static constexpr uint32_t SMEM = BAR_OFF + 256 /*barriers*/ + 1024 /*align slack*/;
    static_assert(SMEM <= 232448, "shared memory plan exceeds 227 KB");
    static_assert(16 * SX + 16 * SQ <= 256, "barrier area");
};

struct KParams {
    CUtensorMap tm_x;
    CUtensorMap tm_w;
    const uint8_t* w_packed;
    const float* bias;
    void* out;
    int M, N, K, ldo;
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
// with a pre-scaled bias would round differently.  For 1/sqrt(64) = 0.125 the two forms give the same bits.
// quick-GELU x * sigmoid(1.702 x) = h + h * tanh(0.851 x) with h = x / 2.
template <int EPI>
CB_DEVINL float epi_value(float acc, float bias, float mul) {
    if constexpr (EPI == EPI_GELU16) return gelu_tanh(acc + bias);
    else if constexpr (EPI == EPI_QGELU16) {
        const float x = acc + bias, h = 0.5f * x;
        float t;
        asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.851f * x));
        return fmaf(h, t, h);
    } else return (acc + bias) * mul;
}

// Global accesses of the epilogue, predicated on `ok` (token rows past M) inside one asm: no branch per element.  All are volatile, so
// they reach ptxas in source order: the residual loads of a batch are issued before any of its stores.
CB_DEVINL float ldg_f32_if(const float* a, bool ok) {
    float v = 0.f;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p ld.global.f32 %0, [%1];\n\t}" : "+f"(v) : "l"(a), "r"((int)ok));
    return v;
}
CB_DEVINL void stg_f32_if(float* a, float v, bool ok) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.global.f32 [%0], %1;\n\t}" ::"l"(a), "f"(v), "r"((int)ok));
}
CB_DEVINL void stg_u16_if(uint16_t* a, uint16_t v, bool ok) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.global.u16 [%0], %1;\n\t}" ::"l"(a), "h"(v), "r"((int)ok));
}

// Epilogue of one consumer group's [64 features x 192 tokens] accumulator (fragment layout: wgmma.cuh).  This thread owns features
// f and f + 8 and tokens 8j + tc + {0, 1}; element offsets are 32-bit (host checks M*ldo < 2^32).
// The residual add x += acc + bias reads its 96 x values in four batches of 24, each batch loaded completely before the first of its
// stores: four memory round trips per tile instead of a chain of 96 dependent ones (with loads and stores through one pointer the
// compiler cannot prove them disjoint, so written as x[o] += v it keeps every load behind the previous store).
template <int EPI, bool BF>
CB_DEVINL void epilogue_regs(void* out, int M, int ldo_, float (&acc)[BN / 2], int tok0, int f, int tc, const float (&bias)[2],
                             const float (&mul)[2]) {
    const int nt = min(BN, M - tok0) - tc;     // this thread's token 8j + tc + e1 is in range iff 8j + e1 < nt
    const uint32_t ldo = (uint32_t)ldo_;
    const uint32_t o0 = (uint32_t)(tok0 + tc) * ldo + (uint32_t)f;
    auto off = [&](int j, int e) { return o0 + (uint32_t)(8 * j + (e & 1)) * ldo + 8u * (uint32_t)(e >> 1); };
    if constexpr (EPI == EPI_REDADD32) {
        float* x = reinterpret_cast<float*>(out);
        constexpr int JB = 6;                  // 6 token groups = 24 elements per batch: the most that fits 168 registers without spills
        #pragma unroll
        for (int b = 0; b < BN / 8 / JB; b++) {
            float r[4 * JB];
            #pragma unroll
            for (int jj = 0; jj < JB; jj++) {
                #pragma unroll
                for (int e = 0; e < 4; e++) r[4 * jj + e] = ldg_f32_if(x + off(b * JB + jj, e), 8 * (b * JB + jj) + (e & 1) < nt);
            }
            #pragma unroll
            for (int jj = 0; jj < JB; jj++) {
                #pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int j = b * JB + jj;
                    stg_f32_if(x + off(j, e), r[4 * jj + e] + (acc[4 * j + e] + bias[e >> 1]), 8 * j + (e & 1) < nt);
                }
            }
        }
    } else {
        #pragma unroll
        for (int j = 0; j < BN / 8; j++) {
            #pragma unroll
            for (int e = 0; e < 4; e++) {
                const int h = e >> 1;
                const bool ok = 8 * j + (e & 1) < nt;
                const float a = acc[4 * j + e];
                if constexpr (EPI == EPI_STORE32) stg_f32_if(reinterpret_cast<float*>(out) + off(j, e), a + bias[h], ok);
                else stg_u16_if(reinterpret_cast<uint16_t*>(out) + off(j, e), P2<BF>::from_float(epi_value<EPI>(a, bias[h], mul[h])), ok);
            }
        }
    }
}

template <int QT, bool BF>
__global__ void __launch_bounds__(THREADS, 1) gemm_dq_kernel(const __grid_constant__ KParams p) {
    using C = Cfg<QT>;
    constexpr bool DQ = C::DQ;
    constexpr int SX = C::SX, SQ = DQ ? C::SQ : 1;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t bars = smem_base + C::BAR_OFF;
    // barrier slots (8 B each)
    const uint32_t x_full = bars, x_empty = x_full + 8 * SX, q_full = x_empty + 8 * SX, q_empty = q_full + 8 * SQ;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < SX; i++) { mbar_init(x_full + 8 * i, 1); mbar_init(x_empty + 8 * i, 8); }   // released by each consumer warp
        for (int i = 0; i < SQ; i++) { mbar_init(q_full + 8 * i, 1); mbar_init(q_empty + 8 * i, 8); }
        mbar_fence_init();
        tma_prefetch_desc(&p.tm_x);
        if (!DQ) tma_prefetch_desc(&p.tm_w);
    }
    __syncthreads();
    pdl_trigger();      // the next kernel of the stream may start placing CTAs as ours retire ...
    pdl_wait();         // ... and we touch global memory only after the previous grid has completed

    // work units: [128 features x 192 tokens] tiles, feature tile fastest (CTAs running at the same time share their X tile in L2)
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
    const int fr = (warp & 3) * 16 + (lane >> 2), tc = 2 * (lane & 3);   // accumulator row (feature in the group) and token column
    uint32_t s = 0, ph = 0, qs = 0, qph = 0;
    float acc[BN / 2];
    uint32_t afr0[16], afr1[16];      // A fragments of two consecutive k-blocks: one is read by in-flight MMAs while the next is unpacked
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int ft = tile % n_ft, tt = tile / n_ft;
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
                    wgmma_rs_n192<BF>(acc, ak, db + 2 * k, (uint32_t)(kb | k));                      // B: +16 k = +32 B
                }
            } else {
                const uint64_t da = wgmma_desc_sw128(smem_base + s * C::XS + X_STAGE + (uint32_t)wg * 64u * 128u);
                #pragma unroll
                for (int k = 0; k < BK / 16; k++) wgmma_ss_n192<BF>(acc, da + 2 * k, db + 2 * k, (uint32_t)(kb | k));
            }
            wgmma_commit();
            wgmma_wait<1>();            // the MMAs of k-block kb-1 are done: release its X stage, its A fragments may be overwritten
            fence_frag(other);
            if (kb > 0) { __syncwarp(); if (lane == 0) mbar_arrive(x_empty + 8 * prev); }
            prev = s;
            if (++s == SX) { s = 0; ph ^= 1; }
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

        const int tok0 = tt * BN, f = ft * BM + wg * 64 + fr;
        float mul[2], bias[2];
        #pragma unroll
        for (int h = 0; h < 2; h++) {
            mul[h] = (f + 8 * h < p.scale_cols) ? p.scale : 1.0f;
            bias[h] = p.bias ? p.bias[f + 8 * h] : 0.0f;
        }
        void* const out = p.out;
        switch (p.epi) {
        case EPI_STORE16: epilogue_regs<EPI_STORE16, BF>(out, p.M, p.ldo, acc, tok0, f, tc, bias, mul); break;
        case EPI_GELU16: epilogue_regs<EPI_GELU16, BF>(out, p.M, p.ldo, acc, tok0, f, tc, bias, mul); break;
        case EPI_QGELU16: epilogue_regs<EPI_QGELU16, BF>(out, p.M, p.ldo, acc, tok0, f, tc, bias, mul); break;
        case EPI_REDADD32: epilogue_regs<EPI_REDADD32, BF>(out, p.M, p.ldo, acc, tok0, f, tc, bias, mul); break;
        default: epilogue_regs<EPI_STORE32, BF>(out, p.M, p.ldo, acc, tok0, f, tc, bias, mul); break;
        }
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
    KParams kp;
    memcpy(&kp.tm_x, a.x_map, sizeof(CUtensorMap));
    if (a.w_map) memcpy(&kp.tm_w, a.w_map, sizeof(CUtensorMap));
    else memset(&kp.tm_w, 0, sizeof(CUtensorMap));
    kp.w_packed = a.w_packed;
    kp.bias = a.bias;
    kp.out = a.out;
    kp.M = a.M; kp.N = a.N; kp.K = a.K; kp.ldo = a.ldo;
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
