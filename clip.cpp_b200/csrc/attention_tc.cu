// attention_tc.cu -- K3 on Hopper tensor cores: S = Q K^T and O = P V as warpgroup MMAs (wgmma), online softmax in registers.
//
// Reference semantics: clip.cpp:1082-1108 (text, causal) / 1363-1388 (vision); soft_max ggml.c:12201-12270.
// Persistent: min(iterations, SMs) CTAs of 288 threads, 161 KB (head_dim 64), 201 KB (head_dim 80) or 225 KB (head_dim 104) of
// shared memory.  The work unit is
// a GROUP of 64 query rows, numbered in (sequence, head, group) order; iteration `it` of the launch takes groups 2it and 2it + 1, one
// per consumer warpgroup, and CTA b runs iterations b, b + grid, ...  So the CTAs running at one time cover consecutive groups, and the
// K / V blocks of a (sequence, head) are read from HBM about once and then from L2.  A group never holds a row past T; only the odd
// group at the very end leaves a warpgroup without work.
//   warp 8      producer, one thread: TMA of both groups' Q rows into a two-deep Q ring, then K and V in 128-key blocks into a two-deep
//               ring whose stages have a slot per head: when the two groups belong to two (sequence, head)s, both heads' blocks are
//               loaded.  All straight out of the fused QKV activation matrix through a 3-D view [sequence][token][column], in boxes of
//               64 rows: rows past a sequence's T tokens arrive as zeros, so padded keys can never inject another sequence's (or stale)
//               NaN / Inf into P.V, and a box wholly past the last key a group uses is not loaded.  The producer's ring positions run on
//               across iterations, so the next item's Q and first K / V blocks arrive while the consumers finish the current one.
//   warps 0-7   two consumer warpgroups, one group each.  Per key block: S[64 x W] = Q.K^T (wgmma m64nWk16, both operands from shared
//               memory; W = 128 except in the last block, where it is the least of 16, 32, 64, 128 that covers the keys left), length /
//               causal mask, online softmax (running row max and sum, quad shuffles), the probabilities re-packed IN REGISTERS as
//               16-bit A fragments, O[64 x dh] += P.V (wgmma m64n64k16 per 16 keys, A from registers, V read MN-major from the same
//               [key][dh] tile, 8 NT / 16 steps).  O / l -> 16-bit stores.
// Trimmed keys only ever contributed -inf to a row maximum and exact zeros to sums, so every output has the bits of the full-width
// computation.
// head_dim 80 (ViT-H/14): a 128-byte-swizzle box holds at most 64 sixteen-bit columns, and a wider box would reach into the next
// head (the tensor map's zero fill stops only at token and matrix ends, not at head boundaries).  So every Q / K / V box arrives
// as two pieces from two tensor maps over the same buffer: columns 0-63 (128-byte swizzle) and 64-79 (32-byte swizzle).  S takes
// one extra k16 step on the tail pieces, O one extra m64n16k16 wgmma per 16 keys into 8 more accumulators per thread.
// head_dim 104 (ViT-bigG/14): the loader pads each head of the QKV projection to 112 columns, the last 8 exactly zero
// (qkv_head_cols), and every box arrives as three pieces: columns 0-63 (128-byte swizzle), 64-95 (64-byte swizzle) and 96-111
// (32-byte swizzle).  The zero columns add exact zeros to S and give O columns that are never stored, and no piece reaches into
// the next head.  S takes 4 + 2 + 1 k16 steps, O n64 + n32 + n16 per 16 keys (56 accumulators).  A 224-byte row makes a 128-key
// K / V tile 28 KB, so this instance runs 64-key blocks in a ring of three stages (225 KB of shared memory in all).
// Any T; a causal group stops at its own diagonal.
// One kernel, two schedules (Sched, a template argument folded away per instance): FIXED takes nseq sequences of T rows through
// the 3-D view above; PACKED / PACKED_CAUSAL take sequences of different lengths stored back to back (VarLen) through a view of the
// packed rows as one sequence, find each group's sequence by a forward gallop, and have the producer warp zero the V rows a box
// brings in from past a sequence's end.
#include <cuda.h>

#include <type_traits>

#include "common.cuh"
#include "gemm.h"
#include "kernels.h"
#include "wgmma.cuh"

namespace cb {

namespace {

constexpr int AG = 64, AK = 128;                       // query rows per group, keys per block
constexpr int ABOX = 64;                               // rows per TMA box
constexpr int ATT_THREADS = 288;                       // 2 consumer warpgroups + 1 producer warp

// Shared-memory layout for one head_dim.  A head's columns arrive as up to three pieces, each a row-major block of its own: columns
// 0-63 (128-byte swizzle), at head_dim 104 columns 64-95 (64-byte swizzle), and the last 16 columns (32-byte swizzle: 64-79 at
// head_dim 80, 96-111 of the 112-column padded head at 104).  A tile of R rows is the R-row blocks of its pieces one after the
// other; a 64-row box fills a 64-row slice of each.  Two Q tiles of 128 rows (rows 0-63: the first group, 64-127: the second), then
// NST stages of two head slots [K | V], each tile KB keys.  Head_dim 104 takes 64-key blocks: its 224-byte rows would need 280 KB
// at 128 keys and two stages.
template <int DH>
struct AttnGeo {
    static_assert(DH == 64 || DH == 80 || DH == 104, "head_dim 64, 80 or 104");
    static constexpr bool MID = DH == 104, TAIL = DH != 64;
    static constexpr int DHP = qkv_head_cols(DH);                   // columns per head in the qkv matrix
    static constexpr int tail_col() { return MID ? 96 : 64; }       // first column of the 16-column tail piece
    static constexpr uint32_t ROW_BYTES = 128 + (MID ? 64 : 0) + (TAIL ? 32 : 0);
    static constexpr int KB = MID ? 64 : AK;                        // keys per K / V block
    static constexpr int NST = MID ? 3 : 2;                         // K / V ring stages
    static constexpr uint32_t MAIN = AK * 128, TILE = AK * ROW_BYTES;          // a 128-row (Q) tile: its first piece, all of it
    static constexpr uint32_t KTILE = KB * ROW_BYTES;                          // a K or V tile
    static constexpr uint32_t BOX_BYTES = ABOX * ROW_BYTES;                    // one 64-row box, every piece
    static constexpr uint32_t KV_OFF = 2 * TILE;
    static constexpr uint32_t BAR_OFF = KV_OFF + NST * 4 * KTILE;
    // offsets of the mid and tail pieces in a tile of `rows` rows
    static constexpr uint32_t mid_off(int rows) { return (uint32_t)rows * 128; }
    static constexpr uint32_t tail_off(int rows) { return (uint32_t)rows * (128 + (MID ? 64 : 0)); }
    static_assert(2 * AG == AK && 2 * ABOX == AK && MAIN % 1024 == 0 && TILE % 1024 == 0 && KTILE % 1024 == 0, "tile alignment");
};

struct AParams {
    CUtensorMap tm_qkv;     // boxes of columns 0-63 of a head
    CUtensorMap tm_tail;    // head_dim 80 / 104: boxes of the 16-column tail piece
    uint16_t* out;
    int T, H, causal;
    int ngrp;               // 64-row groups per (sequence, head)
    int ngroups, niter;     // groups in the launch, iterations (pairs of groups)
};

CB_DEVINL void tma_load_3d(uint32_t dst_smem, const void* tmap, int c0, int c1, int c2, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst_smem),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
CB_DEVINL float ex2f(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
template <bool BF>
CB_DEVINL uint32_t pack2(float lo, float hi) {
    uint32_t r;
    if constexpr (BF) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// K3's schedules.  FIXED: nseq sequences of T rows each, through the 3-D view [sequence][token][column].  PACKED: sequences of
// different lengths stored back to back (VarLen), through the same maps viewing the packed rows as one sequence; PACKED_CAUSAL: the
// same with the causal mask (the text tower's packed passes, head_dim 64 only).
enum Sched { FIXED, PACKED, PACKED_CAUSAL };

// One group of 64 query rows: its (sequence, head), first row and the end of the keys any of its rows can see
struct Group {
    int seq, head, g0, kend;
};
// A group of a packed causal sequence: its key end (min(len, g0 + 64)) and its sequence's length, which bounds the key mask and the
// row stores, apart.  A type of its own, so that the non-causal packed instances keep Group's layout and code.
struct GroupLen : Group {
    int len;
};
template <Sched S>
using GroupOf = std::conditional_t<S == PACKED_CAUSAL, GroupLen, Group>;
CB_DEVINL int seq_len(const Group& g) { return g.kend; }         // non-causal: the key end is the length
CB_DEVINL int seq_len(const GroupLen& g) { return g.len; }
CB_DEVINL Group group_of(const AParams& p, int g) {
    const int sh = g / p.ngrp;
    Group r;
    r.g0 = (g - sh * p.ngrp) * AG;
    r.head = sh % p.H;
    r.seq = sh / p.H;
    r.kend = p.causal ? min(p.T, r.g0 + AG) : p.T;
    return r;
}

// The packed schedules' sequences (launch_attention_tc_varlen): sequence s is rows [off[s], off[s + 1]) of one [row][column] view of
// the qkv matrix, and its groups are numbered from H * grp[s] (grp: prefix sums of the per-sequence group counts ceil(len / 64)).
struct VarLen {
    const int* off;
    const int* grp;
    int nseq;
};

// group_of for packed sequences.  Group::seq holds the sequence's first row (distinct for distinct sequences, so iter_of's test of a
// shared (sequence, head) holds) and kend its length; causal, kend is the group's diagonal end as group_of has it and len the
// length.  s: a sequence at or before group g's, advanced to g's.  A thread's groups only increase, so the search gallops forward from the
// last sequence found (one load when g is still in it) and ends in a binary search of the bracket.
template <Sched S>
CB_DEVINL GroupOf<S> group_var(const AParams& p, const VarLen& v, int g, int& s) {
    int lo = s, step = 1;
    while (lo + step < v.nseq && __ldg(v.grp + lo + step) * p.H <= g) { lo += step; step *= 2; }
    int hi = min(lo + step, v.nseq) - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(v.grp + mid) * p.H <= g) lo = mid;
        else hi = mid - 1;
    }
    s = lo;
    const int ng = __ldg(v.grp + lo + 1) - __ldg(v.grp + lo), local = g - __ldg(v.grp + lo) * p.H;
    GroupOf<S> r;
    r.head = local / ng;
    r.g0 = (local - r.head * ng) * AG;
    r.seq = __ldg(v.off + lo);
    r.kend = __ldg(v.off + lo + 1) - r.seq;
    if constexpr (S == PACKED_CAUSAL) {
        r.len = r.kend;
        r.kend = min(r.len, r.g0 + AG);
    }
    return r;
}

// The two groups of iteration `it` and what the K / V stages hold for them: slot 0 the first group's head (and the second's, when it
// is the same (sequence, head) or there is no second group), slot 1 the second group's head otherwise.  kend0 / kend1: the keys a
// slot must hold (0: slot unused); nkb: key blocks (of KB keys) of the iteration.
template <class Gr>
struct IterOf {
    Gr a, b;
    bool has_b, shared;
    int kend0, kend1, nkb;
};
// group g of schedule S (s: group_var's cursor)
template <Sched S>
CB_DEVINL GroupOf<S> group_at(const AParams& p, const VarLen& v, int g, int& s) {
    if constexpr (S == FIXED) return group_of(p, g);
    else return group_var<S>(p, v, g, s);
}
// s: group_var's sequence cursor (packed schedules only)
template <int KB, Sched S>
CB_DEVINL IterOf<GroupOf<S>> iter_of(const AParams& p, const VarLen& v, int it, int& s) {
    IterOf<GroupOf<S>> r;
    r.has_b = 2 * it + 1 < p.ngroups;
    r.a = group_at<S>(p, v, 2 * it, s);
    // with no second group, FIXED recomputes the first and the packed schedules copy it (each instance's code as it always was)
    r.b = S == FIXED || r.has_b ? group_at<S>(p, v, r.has_b ? 2 * it + 1 : 2 * it, s) : r.a;
    r.shared = r.a.seq == r.b.seq && r.a.head == r.b.head;
    r.kend0 = r.shared ? max(r.a.kend, r.b.kend) : r.a.kend;
    r.kend1 = r.shared ? 0 : r.b.kend;
    r.nkb = (max(r.kend0, r.kend1) + KB - 1) / KB;
    return r;
}

// 64-row boxes of key block kb (KB keys) that a slot holding keys [0, kend) needs
template <int KB>
CB_DEVINL int kv_boxes(int kend, int kb) {
    const int key0 = kb * KB;
    return key0 >= kend ? 0 : (KB == ABOX || key0 + ABOX >= kend) ? 1 : 2;
}

// Rows of the last 64-row box a slot holding keys [0, kend) loads for block kb that lie past kend (0 when kb is not the slot's last
// block).  In a packed view those rows belong to the next sequence.
template <int KB>
CB_DEVINL int kv_pad_rows(int kend, int kb) {
    const int nb = kv_boxes<KB>(kend, kb);
    return nb ? max(0, kb * KB + nb * ABOX - kend) : 0;
}

// Zero rows [r0, r1) of every piece of the KB-row tile at `tile`: each piece is row-major and its swizzle permutes 16-byte chunks
// within a row, so a row's bytes are one contiguous range of the piece whatever the swizzle.  The calling warp's 32 lanes store.
template <int DH>
CB_DEVINL void zero_tile_rows(uint32_t tile, int r0, int r1, int lane) {
    using G = AttnGeo<DH>;
    auto zero = [&](uint32_t a0, uint32_t a1) {
        for (uint32_t a = a0 + 16u * lane; a < a1; a += 512u) asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0u) : "memory");
    };
    zero(tile + r0 * 128u, tile + r1 * 128u);
    if constexpr (G::MID) zero(tile + G::mid_off(G::KB) + r0 * 64u, tile + G::mid_off(G::KB) + r1 * 64u);
    if constexpr (G::TAIL) zero(tile + G::tail_off(G::KB) + r0 * 32u, tile + G::tail_off(G::KB) + r1 * 32u);
}

// one 64-row box (every piece) into box `b` of the `rows`-row tile at `tile`; tm_mid: the head_dim 104 map of columns 64-95
template <int DH, int ROWS>
CB_DEVINL void load_box(uint32_t tile, int b, const AParams& p, const CUtensorMap& tm_mid, int col, int row, int seq, uint32_t bar) {
    using G = AttnGeo<DH>;
    tma_load_3d(tile + (uint32_t)b * (ABOX * 128), &p.tm_qkv, col, row, seq, bar);
    if constexpr (G::MID) tma_load_3d(tile + G::mid_off(ROWS) + (uint32_t)b * (ABOX * 64), &tm_mid, col + 64, row, seq, bar);
    if constexpr (G::TAIL) tma_load_3d(tile + G::tail_off(ROWS) + (uint32_t)b * (ABOX * 32), &p.tm_tail, col + G::tail_col(), row, seq, bar);
}

template <bool BF, int NT>
CB_DEVINL void wgmma_ss_nt(float (&d)[4 * NT], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (NT == 16) wgmma_ss_n128<BF>(d, da, db, accumulate);
    else if constexpr (NT == 8) wgmma_ss_n64<BF>(d, da, db, accumulate);
    else if constexpr (NT == 4) wgmma_ss_n32<BF>(d, da, db, accumulate);
    else wgmma_ss_n16<BF>(d, da, db, accumulate);
}

// One key block of one consumer warpgroup, S NT n-tiles (8 keys each) wide: keys [key0, key0 + 8 NT) of the stage at k_s / v_s.
// The same operations in the same order as the full 128-key block: the keys past 8 NT would only have been masked to -inf.
template <bool BF, int DH, int NT>
CB_DEVINL void attend_block(float (&o)[32], float (&om)[16], float (&ot)[8], float (&m_run)[2], float (&l_run)[2], uint64_t dq,
                            uint64_t dq_m, uint64_t dq_t, uint32_t k_s, uint32_t v_s, int key0, int T, int causal, int wrow0, int r0, int tc) {
    using G = AttnGeo<DH>;
    constexpr float LOG2E = 1.4426950408889634f;
    float sc[4 * NT];
    const uint64_t dk = wgmma_desc_sw128(k_s);
    wgmma_fence();
    #pragma unroll
    for (int k = 0; k < 4; k++) wgmma_ss_nt<BF, NT>(sc, dq + 2 * k, dk + 2 * k, (uint32_t)k);
    if constexpr (G::MID) {
        const uint64_t dkm = wgmma_desc_sw64(k_s + G::mid_off(G::KB));
        #pragma unroll
        for (int k = 0; k < 2; k++) wgmma_ss_nt<BF, NT>(sc, dq_m + 2 * k, dkm + 2 * k, 1u);
    }
    if constexpr (G::TAIL) wgmma_ss_nt<BF, NT>(sc, dq_t, wgmma_desc_sw32(k_s + G::tail_off(G::KB)), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    // masking is only needed in the last (ragged) key block and, for the causal text tower, on the diagonal block
    if (key0 + 8 * NT > T || (causal && key0 + 8 * NT - 1 > wrow0)) {
        #pragma unroll
        for (int j = 0; j < NT; j++) {
            #pragma unroll
            for (int e = 0; e < 4; e++) {
                const int key = key0 + 8 * j + tc + (e & 1), row = r0 + 8 * (e >> 1);
                if (key >= T || (causal && key > row)) sc[4 * j + e] = -INFINITY;
            }
        }
    }
    #pragma unroll
    for (int h = 0; h < 2; h++) {
        float mx = -INFINITY;
        #pragma unroll
        for (int j = 0; j < NT; j++) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * h], sc[4 * j + 2 * h + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        // every row (padded rows past T included: zero queries) sees at least one unmasked key per visited block
        const float m_new = fmaxf(m_run[h], mx);
        const float alpha = ex2f((m_run[h] - m_new) * LOG2E), mb = m_new * LOG2E;
        float rs = 0.f;
        #pragma unroll
        for (int j = 0; j < NT; j++) {
            const float p0 = ex2f(sc[4 * j + 2 * h] * LOG2E - mb), p1 = ex2f(sc[4 * j + 2 * h + 1] * LOG2E - mb);
            sc[4 * j + 2 * h] = p0; sc[4 * j + 2 * h + 1] = p1;
            rs += p0 + p1;
        }
        l_run[h] = l_run[h] * alpha + rs;
        m_run[h] = m_new;
        #pragma unroll
        for (int j = 0; j < 8; j++) { o[4 * j + 2 * h] *= alpha; o[4 * j + 2 * h + 1] *= alpha; }
        if constexpr (G::MID) {
            #pragma unroll
            for (int j = 0; j < 4; j++) { om[4 * j + 2 * h] *= alpha; om[4 * j + 2 * h + 1] *= alpha; }
        }
        if constexpr (G::TAIL) {
            #pragma unroll
            for (int j = 0; j < 2; j++) { ot[4 * j + 2 * h] *= alpha; ot[4 * j + 2 * h + 1] *= alpha; }
        }
    }
    // O += P.V: key step kk covers S n-tiles 2kk (A fragment registers 0, 1) and 2kk + 1 (registers 2, 3).  Keys in [kend, key0 + 8 NT)
    // have P = 0 and zero-filled V rows (they lie past T); a data-dependent skip of their steps would make ptxas serialize the chain.
    wgmma_fence();
    #pragma unroll
    for (int kk = 0; kk < NT / 2; kk++) {
        const uint32_t a[4] = {pack2<BF>(sc[8 * kk], sc[8 * kk + 1]), pack2<BF>(sc[8 * kk + 2], sc[8 * kk + 3]),
                               pack2<BF>(sc[8 * kk + 4], sc[8 * kk + 5]), pack2<BF>(sc[8 * kk + 6], sc[8 * kk + 7])};
        wgmma_rs_n64_bmn<BF>(o, a, wgmma_desc_sw128(v_s + (uint32_t)kk * 2048u), 1u);      // 16 keys = 2048 B of V
        if constexpr (G::MID) wgmma_rs_n32_bmn<BF>(om, a, wgmma_desc_sw64(v_s + G::mid_off(G::KB) + (uint32_t)kk * 1024u), 1u);   // 1024 B
        if constexpr (G::TAIL) wgmma_rs_n16_bmn<BF>(ot, a, wgmma_desc_sw32(v_s + G::tail_off(G::KB) + (uint32_t)kk * 512u), 1u);  // 512 B
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if constexpr (G::MID) wgmma_fence_regs(om);
    if constexpr (G::TAIL) wgmma_fence_regs(ot);
}

// Row r of the sequence whose Group::seq is `seq` has box coordinates (r, seq) in FIXED's 3-D view, (seq + r, 0) in the packed rows' view
template <Sched S> CB_DEVINL int box_row0(int seq) { return S == FIXED ? 0 : seq; }
template <Sched S> CB_DEVINL int box_seq(int seq) { return S == FIXED ? seq : 0; }

// K3, in either schedule.  The packed schedules count a group's rows and keys from its sequence's first row and take its length for
// T, so every key block and the width of the last one are those a FIXED launch of that sequence alone takes, and each kept row has its
// arithmetic.  Their box rows past a sequence's end hold the next sequence's rows instead of zeros: their scores are masked by
// select, their Q rows are never stored, but P.V would turn a non-finite V row into NaN (0 * Inf), so the producer warp zeroes those
// V rows once the box has landed and before the consumers may read the stage: such a stage lands on a barrier of the producer's own
// (kv_land), and the producer arrives on the stage's full barrier once the zeros are stored.
// PACKED_CAUSAL: a group's keys end at min(len, g0 + 64), as group_of has them, and attend_block masks with T = len and causal = 1,
// as a causal FIXED launch calls it.  A key end before the sequence's end is g0 + 64, a multiple of the 64-row box, so a slot's last
// box then ends exactly at its key end: box rows past a key end, the rows the producer zeroes, still occur only at a sequence's end.
// tm_mid: head_dim 104's map of columns 64-95 (unused otherwise; a parameter of its own, so AParams keeps its layout); v: the packed
// schedules' sequences (unused by FIXED).
template <bool BF, int DH, Sched S>
__global__ void __launch_bounds__(ATT_THREADS, 1) attention_tc_kernel(const __grid_constant__ AParams p, const __grid_constant__ CUtensorMap tm_mid,
                                                                      const VarLen v) {
    using G = AttnGeo<DH>;
    constexpr bool PACK = S != FIXED;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t smem_base = smem_u32(smem);
    // [i] = +8i bytes: Q tile full / empty (rings of two), K-V stage full / empty (rings of NST), then (packed) kv_land
    const uint32_t q_full = smem_base + G::BAR_OFF, q_empty = q_full + 16, kv_full = q_full + 32, kv_empty = kv_full + 8 * G::NST;
    const uint32_t kv_land = kv_empty + 8 * G::NST;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < G::NST; i++) {
            if (i < 2) { mbar_init(q_full + 8 * i, 1); mbar_init(q_empty + 8 * i, 8); }      // released by each consumer warp
            mbar_init(kv_full + 8 * i, 1); mbar_init(kv_empty + 8 * i, 8);
        }
        if constexpr (PACK) mbar_init(kv_land, 1);
        mbar_fence_init();
        tma_prefetch_desc(&p.tm_qkv);
        if constexpr (G::MID) tma_prefetch_desc(&tm_mid);
        if constexpr (G::TAIL) tma_prefetch_desc(&p.tm_tail);
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();      // qkv is read (and the output written) only after the QKV GEMM grid has completed

    const int hid = p.H * DH, qcols = p.H * G::DHP;           // output row, and Q / K / V part of a qkv row
    // Ring positions run on across iterations: the i-th iteration of this CTA uses Q tile i % 2 (its (i / 2)-th use), the n-th key
    // block of this CTA stage n % NST (its (n / NST)-th use).  A use waits for full with the use's parity and, in the producer, for the
    // release of the previous use of the slot (parity flipped: the first wait on a fresh barrier passes).
    if (warp == 8) {
        // ------------------------------------------------------------------ producer
        // FIXED: one thread.  Packed: one warp, of which lane 0 issues the loads.  A stage that holds a sequence's last block lands
        // on kv_land instead of kv_full; the whole warp waits for it, zeroes the V rows past the sequence's end and only then arrives
        // on kv_full.  nz: such stages so far.
        if (!PACK && lane != 0) return;
        uint32_t n = 0, i = 0, nz = 0;
        int sq = 0;
        for (int it = blockIdx.x; it < p.niter; it += gridDim.x, i++) {
            const auto w = iter_of<G::KB, S>(p, v, it, sq);
            const uint32_t qb = i & 1, q_s = smem_base + qb * G::TILE;
            if (lane == 0) {
                mbar_wait(q_empty + 8 * qb, ((i >> 1) & 1) ^ 1);
                mbar_arrive_expect_tx(q_full + 8 * qb, (w.has_b ? 2 : 1) * G::BOX_BYTES);
                load_box<DH, AK>(q_s, 0, p, tm_mid, w.a.head * G::DHP, box_row0<S>(w.a.seq) + w.a.g0, box_seq<S>(w.a.seq), q_full + 8 * qb);
                if (w.has_b) load_box<DH, AK>(q_s, 1, p, tm_mid, w.b.head * G::DHP, box_row0<S>(w.b.seq) + w.b.g0, box_seq<S>(w.b.seq), q_full + 8 * qb);
            }
            for (int kb = 0; kb < w.nkb; kb++, n++) {
                // the stage's slots and the barrier its loads land on, each schedule in its own order (FIXED's one thread takes
                // the slots after the wait): the instances' register allocation depends on it.  z0 / z1: V rows the warp zeroes.
                uint32_t s, bar, slot0, slot1;
                int nb0, nb1, z0 = 0, z1 = 0;
                if constexpr (!PACK) {
                    s = n % G::NST; bar = kv_full + 8 * s;
                    nb0 = kv_boxes<G::KB>(w.kend0, kb); nb1 = kv_boxes<G::KB>(w.kend1, kb);
                    mbar_wait(kv_empty + 8 * s, ((n / G::NST) & 1) ^ 1);
                    mbar_arrive_expect_tx(bar, (uint32_t)(nb0 + nb1) * 2 * G::BOX_BYTES);
                    slot0 = smem_base + G::KV_OFF + s * (4 * G::KTILE); slot1 = slot0 + 2 * G::KTILE;
                } else {
                    s = n % G::NST;
                    nb0 = kv_boxes<G::KB>(w.kend0, kb); nb1 = kv_boxes<G::KB>(w.kend1, kb);
                    slot0 = smem_base + G::KV_OFF + s * (4 * G::KTILE); slot1 = slot0 + 2 * G::KTILE;
                    z0 = kv_pad_rows<G::KB>(w.kend0, kb); z1 = kv_pad_rows<G::KB>(w.kend1, kb);
                    bar = (z0 || z1) ? kv_land : kv_full + 8 * s;
                }
                if (lane == 0) {
                    if constexpr (PACK) {
                        mbar_wait(kv_empty + 8 * s, ((n / G::NST) & 1) ^ 1);
                        mbar_arrive_expect_tx(bar, (uint32_t)(nb0 + nb1) * 2 * G::BOX_BYTES);
                    }
                    for (int b = 0; b < nb0; b++) {
                        load_box<DH, G::KB>(slot0, b, p, tm_mid, qcols + w.a.head * G::DHP, box_row0<S>(w.a.seq) + kb * G::KB + b * ABOX, box_seq<S>(w.a.seq), bar);
                        load_box<DH, G::KB>(slot0 + G::KTILE, b, p, tm_mid, 2 * qcols + w.a.head * G::DHP, box_row0<S>(w.a.seq) + kb * G::KB + b * ABOX, box_seq<S>(w.a.seq), bar);
                    }
                    for (int b = 0; b < nb1; b++) {
                        load_box<DH, G::KB>(slot1, b, p, tm_mid, qcols + w.b.head * G::DHP, box_row0<S>(w.b.seq) + kb * G::KB + b * ABOX, box_seq<S>(w.b.seq), bar);
                        load_box<DH, G::KB>(slot1 + G::KTILE, b, p, tm_mid, 2 * qcols + w.b.head * G::DHP, box_row0<S>(w.b.seq) + kb * G::KB + b * ABOX, box_seq<S>(w.b.seq), bar);
                    }
                }
                if constexpr (PACK) {
                    __syncwarp();
                    if (z0 || z1) {
                        mbar_wait(kv_land, nz++ & 1);
                        if (z0) zero_tile_rows<DH>(slot0 + G::KTILE, nb0 * ABOX - z0, nb0 * ABOX, lane);
                        if (z1) zero_tile_rows<DH>(slot1 + G::KTILE, nb1 * ABOX - z1, nb1 * ABOX, lane);
                        // the zeros (generic proxy) before the consumers' wgmma reads and the next TMA into the stage (async proxy)
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        __syncwarp();
                        if (lane == 0) mbar_arrive(kv_full + 8 * s);
                    }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers (fragment layout: wgmma.cuh)
    const int wg = warp >> 2;
    const int tc = 2 * (lane & 3);                             // this thread: columns 8j + tc + {0, 1}
    uint32_t n = 0, i = 0;
    int sq = 0;
    for (int it = blockIdx.x; it < p.niter; it += gridDim.x, i++) {
        const int sq_it = sq;                                  // at or before both groups' sequences
        const auto w = iter_of<G::KB, S>(p, v, it, sq);
        // this warpgroup's group: the same value either way, but each form gives its instances their register allocation
        GroupOf<S> g;
        if constexpr (PACK) g = (wg == 0 || !w.has_b) ? w.a : w.b;
        else g = group_of(p, min(2 * it + wg, p.ngroups - 1));
        const bool live = wg == 0 || w.has_b;                  // warpgroup-uniform: only the launch's last, odd group leaves one idle
        const uint32_t slot = (wg == 0 || w.shared) ? 0u : 1u;
        const int nkb = (g.kend + G::KB - 1) / G::KB;
        const int len = PACK ? seq_len(g) : p.T;               // the sequence's length: the key mask and the row stores
        const int wrow0 = g.g0 + (warp & 3) * 16;              // first query row of this warp
        const int r0 = wrow0 + (lane >> 2);                    // this thread: rows r0 and r0 + 8
        // o: columns 0-63, om: 64-95 (head_dim 104 only), ot: the 16-column tail (head_dim 80, 104)
        float o[32], om[16], ot[8], m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        #pragma unroll
        for (int j = 0; j < 32; j++) o[j] = 0.f;
        #pragma unroll
        for (int j = 0; j < 16; j++) om[j] = 0.f;
        #pragma unroll
        for (int j = 0; j < 8; j++) ot[j] = 0.f;
        const uint32_t qb = i & 1, q_s = smem_base + qb * G::TILE;
        mbar_wait(q_full + 8 * qb, (i >> 1) & 1);
        const uint64_t dq = wgmma_desc_sw128(q_s + (uint32_t)wg * 64u * 128u);
        const uint64_t dq_m = wgmma_desc_sw64(q_s + G::mid_off(AK) + (uint32_t)wg * 64u * 64u);
        const uint64_t dq_t = wgmma_desc_sw32(q_s + G::tail_off(AK) + (uint32_t)wg * 64u * 32u);
        for (int kb = 0; kb < w.nkb; kb++, n++) {
            const uint32_t s = n % G::NST;
            const uint32_t k_s = smem_base + G::KV_OFF + s * (4 * G::KTILE) + slot * (2 * G::KTILE), v_s = k_s + G::KTILE;
            mbar_wait(kv_full + 8 * s, (n / G::NST) & 1);
            if (live && kb < nkb) {
                const int key0 = kb * G::KB, rem = g.kend - key0, causal = PACK ? S == PACKED_CAUSAL : p.causal;
                // S at the narrowest width that covers the keys left (a 64-key block never needs 128)
                if (G::KB == 128 && rem > 64) attend_block<BF, DH, 16>(o, om, ot, m_run, l_run, dq, dq_m, dq_t, k_s, v_s, key0, len, causal, wrow0, r0, tc);
                else if (rem > 32) attend_block<BF, DH, 8>(o, om, ot, m_run, l_run, dq, dq_m, dq_t, k_s, v_s, key0, len, causal, wrow0, r0, tc);
                else if (rem > 16) attend_block<BF, DH, 4>(o, om, ot, m_run, l_run, dq, dq_m, dq_t, k_s, v_s, key0, len, causal, wrow0, r0, tc);
                else attend_block<BF, DH, 2>(o, om, ot, m_run, l_run, dq, dq_m, dq_t, k_s, v_s, key0, len, causal, wrow0, r0, tc);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(kv_empty + 8 * s);
        }
        // every S product that read this Q tile has completed (wgmma_wait<0> in attend_block)
        __syncwarp();
        if (lane == 0) mbar_arrive(q_empty + 8 * qb);
        if (!live) continue;
        // packed: the group's first row and head looked up again rather than held in registers through the key loop (the head_dim 80
        // instance has none to spare at 168, the most 288 threads can have)
        const auto ge = [&] {
            if constexpr (PACK) {
                int sq_e = sq_it;
                return group_var<S>(p, v, 2 * it + wg, sq_e);
            } else {
                return g;
            }
        }();
        #pragma unroll
        for (int h = 0; h < 2; h++) {
            float l = l_run[h];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = 1.0f / l;
            const int row = r0 + 8 * h;
            if (row < len) {
                uint16_t* orow = p.out + (PACK ? (size_t)ge.seq + row : (size_t)ge.seq * p.T + row) * hid + ge.head * DH;
                #pragma unroll
                for (int j = 0; j < 8; j++)
                    *reinterpret_cast<uint32_t*>(orow + 8 * j + tc) = pack2<BF>(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
                if constexpr (G::MID) {
                    #pragma unroll
                    for (int j = 0; j < 4; j++)
                        *reinterpret_cast<uint32_t*>(orow + 64 + 8 * j + tc) = pack2<BF>(om[4 * j + 2 * h] * inv, om[4 * j + 2 * h + 1] * inv);
                }
                if constexpr (G::TAIL) {
                    // the real tail columns only: at head_dim 104, columns 104-111 are the padding
                    #pragma unroll
                    for (int j = 0; j < (DH - G::tail_col()) / 8; j++)
                        *reinterpret_cast<uint32_t*>(orow + G::tail_col() + 8 * j + tc) = pack2<BF>(ot[4 * j + 2 * h] * inv, ot[4 * j + 2 * h + 1] * inv);
                }
            }
        }
    }
}

// an instance's shared memory: AttnGeo's tiles, its barriers (the packed schedules' kv_land too) and the slack for 1024-byte alignment
template <int DH, Sched S>
constexpr uint32_t k3_smem() { return AttnGeo<DH>::BAR_OFF + 32 + 16 * AttnGeo<DH>::NST + (S == FIXED ? 0 : 8) + 1024; }

// ---- K9: the attention probabilities themselves (the *_tokens calls' ATTENTION entries) ------------------------------------------
// softmax(Q.K^T [causal]) of one block, recomputed from the qkv matrix K3 read (Q scaled by 1/sqrt(dh) and rounded, K 16-bit) through
// the same 3-D maps, as rows of T elements.  CTA = one consumer warpgroup (warps 0-3) + one producer warp (warp 4); work unit = one
// (sequence, head, 64-row query group), in CLS mode one (sequence, head), group 0, of which only row 0 is written.
//   producer  one thread: the group's Q box, then K only (V is never loaded) in 128-key blocks into a two-deep ring, every block twice.
//   pass 1    per key block: S = Q.K^T (wgmma, K3's widths 16 / 32 / 64 / 128 and masks), running row max and sum with K3's arithmetic.
//   pass 2    the blocks again: p = ex2(s log2e - m log2e) * (1 / l) in fp32 (a 16-bit output is the RNE of that fp32 value), masked
//             keys +0.  Each [64 x <= 128] block is staged in shared memory and leaves as row segments of coalesced element stores:
//             rows are T elements long and T is mostly odd, so no store wider than one element is aligned.  The keys of a causal
//             group past its diagonal block are written as +0 without being computed.
constexpr int PROBS_THREADS = 160;
constexpr int PSTRIDE = AK + 8;          // staging row stride in elements: a warp's fragment stores of 4 rows fill 32 distinct banks

// Q: one box in a tile of QROWS rows (head_dim 104: a 64-row tile, so that two CTAs fit on an SM; 64 and 80 keep the half-used
// 128-row tile they always had); then the two K stages of 128-row tiles.
template <int DH>
struct ProbsGeo {
    using G = AttnGeo<DH>;
    static constexpr int QROWS = G::MID ? ABOX : AK;
    static constexpr uint32_t K_OFF = QROWS * G::ROW_BYTES;
    static constexpr uint32_t STAGE_OFF = K_OFF + 2 * G::TILE;        // [64][PSTRIDE] elements of up to 4 bytes
    static constexpr uint32_t BAR_OFF = STAGE_OFF + AG * PSTRIDE * 4;
    static constexpr uint32_t SMEM = BAR_OFF + 64 + 1024;
};

struct PParams {
    AParams a;              // maps, T, H, causal; ngrp = 64-row groups per (sequence, head), 1 in CLS mode
    void* out;              // [nseq, H, rows, T] of otype
    int otype, rows;        // 0 f32, 1 f16, 2 bf16;  rows = T, or 1 (CLS)
};

CB_DEVINL void probs_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }      // the consumer warpgroup only

// S of one key block, NT n-tiles wide, masked as in attend_block
template <bool BF, int DH, int NT>
CB_DEVINL void probs_scores(float (&sc)[4 * NT], uint64_t dq, uint64_t dq_m, uint64_t dq_t, uint32_t k_s, int key0, int T, int causal,
                            int wrow0, int r0, int tc) {
    using G = AttnGeo<DH>;
    const uint64_t dk = wgmma_desc_sw128(k_s);
    wgmma_fence();
    #pragma unroll
    for (int k = 0; k < 4; k++) wgmma_ss_nt<BF, NT>(sc, dq + 2 * k, dk + 2 * k, (uint32_t)k);
    if constexpr (G::MID) {
        const uint64_t dkm = wgmma_desc_sw64(k_s + G::mid_off(AK));
        #pragma unroll
        for (int k = 0; k < 2; k++) wgmma_ss_nt<BF, NT>(sc, dq_m + 2 * k, dkm + 2 * k, 1u);
    }
    if constexpr (G::TAIL) wgmma_ss_nt<BF, NT>(sc, dq_t, wgmma_desc_sw32(k_s + G::tail_off(AK)), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    if (key0 + 8 * NT > T || (causal && key0 + 8 * NT - 1 > wrow0)) {
        #pragma unroll
        for (int j = 0; j < NT; j++) {
            #pragma unroll
            for (int e = 0; e < 4; e++) {
                const int key = key0 + 8 * j + tc + (e & 1), row = r0 + 8 * (e >> 1);
                if (key >= T || (causal && key > row)) sc[4 * j + e] = -INFINITY;
            }
        }
    }
}

// pass 1: the running row max and sum over one key block, exactly as attend_block updates them
template <bool BF, int DH, int NT>
CB_DEVINL void probs_stats(float (&m_run)[2], float (&l_run)[2], uint64_t dq, uint64_t dq_m, uint64_t dq_t, uint32_t k_s, int key0, int T,
                           int causal, int wrow0, int r0, int tc) {
    constexpr float LOG2E = 1.4426950408889634f;
    float sc[4 * NT];
    probs_scores<BF, DH, NT>(sc, dq, dq_m, dq_t, k_s, key0, T, causal, wrow0, r0, tc);
    #pragma unroll
    for (int h = 0; h < 2; h++) {
        float mx = -INFINITY;
        #pragma unroll
        for (int j = 0; j < NT; j++) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * h], sc[4 * j + 2 * h + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[h], mx);
        const float alpha = ex2f((m_run[h] - m_new) * LOG2E), mb = m_new * LOG2E;
        float rs = 0.f;
        #pragma unroll
        for (int j = 0; j < NT; j++) rs += ex2f(sc[4 * j + 2 * h] * LOG2E - mb) + ex2f(sc[4 * j + 2 * h + 1] * LOG2E - mb);
        l_run[h] = l_run[h] * alpha + rs;
        m_run[h] = m_new;
    }
}

// pass 2: the probabilities of one key block into the staging buffer (row lr0 + 8h, columns 8j + tc + {0, 1}); the K stage is
// released as soon as S is in registers
template <bool BF, int DH, int NT>
CB_DEVINL void probs_block(const float (&mb)[2], const float (&inv)[2], uint64_t dq, uint64_t dq_m, uint64_t dq_t, uint32_t k_s, int key0,
                           int T, int causal, int wrow0, int r0, int tc, int lr0, uint8_t* stage, int otype, uint32_t release, int lane) {
    constexpr float LOG2E = 1.4426950408889634f;
    float sc[4 * NT];
    probs_scores<BF, DH, NT>(sc, dq, dq_m, dq_t, k_s, key0, T, causal, wrow0, r0, tc);
    __syncwarp();
    if (lane == 0) mbar_arrive(release);
    probs_bar();                                               // the previous block's stores have read the staging buffer
    #pragma unroll
    for (int h = 0; h < 2; h++) {
        const int lr = lr0 + 8 * h;
        #pragma unroll
        for (int j = 0; j < NT; j++) {
            const float p0 = ex2f(sc[4 * j + 2 * h] * LOG2E - mb[h]) * inv[h], p1 = ex2f(sc[4 * j + 2 * h + 1] * LOG2E - mb[h]) * inv[h];
            const int e = lr * PSTRIDE + 8 * j + tc;
            if (otype == 0) *reinterpret_cast<float2*>(stage + 4 * e) = make_float2(p0, p1);
            else *reinterpret_cast<uint32_t*>(stage + 2 * e) = otype == 2 ? pack2<true>(p0, p1) : pack2<false>(p0, p1);
        }
    }
    probs_bar();
}

template <bool BF, int DH>
__global__ void __launch_bounds__(PROBS_THREADS, 1) attention_probs_kernel(const __grid_constant__ PParams p, const __grid_constant__ CUtensorMap tm_mid) {
    using G = AttnGeo<DH>;
    using PG = ProbsGeo<DH>;
    constexpr float LOG2E = 1.4426950408889634f;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t smem_base = smem_u32(smem);
    // Q full, K stage full [0|1], K stage empty [0|1]
    const uint32_t q_full = smem_base + PG::BAR_OFF, kv_full = q_full + 8, kv_empty = q_full + 24;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        mbar_init(q_full, 1);
        for (int i = 0; i < 2; i++) { mbar_init(kv_full + 8 * i, 1); mbar_init(kv_empty + 8 * i, 4); }     // released by each consumer warp
        mbar_fence_init();
        tma_prefetch_desc(&p.a.tm_qkv);
        if constexpr (G::MID) tma_prefetch_desc(&tm_mid);
        if constexpr (G::TAIL) tma_prefetch_desc(&p.a.tm_tail);
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();      // qkv is read (and the output written) only after the kernels before this one have completed

    const int T = p.a.T;
    const int sh = blockIdx.x / p.a.ngrp;                     // (sequence, head)
    const int g0 = (blockIdx.x - sh * p.a.ngrp) * AG, head = sh % p.a.H, seq = sh / p.a.H;
    const int kend = p.a.causal ? min(T, g0 + AG) : T;
    const int nkb = (kend + AK - 1) / AK;
    if (warp == 4) {
        // ------------------------------------------------------------------ producer (one thread): Q, then K blocks 0 .. nkb-1 twice
        if (lane == 0) {
            mbar_arrive_expect_tx(q_full, G::BOX_BYTES);
            load_box<DH, PG::QROWS>(smem_base, 0, p.a, tm_mid, head * G::DHP, g0, seq, q_full);
            const int kcol = p.a.H * G::DHP + head * G::DHP;
            for (int n = 0; n < 2 * nkb; n++) {
                const int kb = n < nkb ? n : n - nkb, nb = kv_boxes<AK>(kend, kb);
                const uint32_t s = n & 1, bar = kv_full + 8 * s;
                mbar_wait(kv_empty + 8 * s, ((n >> 1) & 1) ^ 1);
                mbar_arrive_expect_tx(bar, (uint32_t)nb * G::BOX_BYTES);
                for (int b = 0; b < nb; b++) load_box<DH, AK>(smem_base + PG::K_OFF + s * G::TILE, b, p.a, tm_mid, kcol, kb * AK + b * ABOX, seq, bar);
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers (fragment layout: wgmma.cuh)
    const int tc = 2 * (lane & 3);
    const int lr0 = warp * 16 + (lane >> 2);                  // this thread: group rows lr0 and lr0 + 8
    const int wrow0 = g0 + warp * 16, r0 = g0 + lr0;
    mbar_wait(q_full, 0);
    const uint64_t dq = wgmma_desc_sw128(smem_base), dq_m = wgmma_desc_sw64(smem_base + G::mid_off(PG::QROWS));
    const uint64_t dq_t = wgmma_desc_sw32(smem_base + G::tail_off(PG::QROWS));
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    uint32_t n = 0;
    for (int kb = 0; kb < nkb; kb++, n++) {
        const uint32_t s = n & 1, k_s = smem_base + PG::K_OFF + s * G::TILE;
        mbar_wait(kv_full + 8 * s, (n >> 1) & 1);
        const int key0 = kb * AK, rem = kend - key0;
        if (rem > 64) probs_stats<BF, DH, 16>(m_run, l_run, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc);
        else if (rem > 32) probs_stats<BF, DH, 8>(m_run, l_run, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc);
        else if (rem > 16) probs_stats<BF, DH, 4>(m_run, l_run, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc);
        else probs_stats<BF, DH, 2>(m_run, l_run, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc);
        __syncwarp();
        if (lane == 0) mbar_arrive(kv_empty + 8 * s);
    }
    float mb[2], inv[2];
    #pragma unroll
    for (int h = 0; h < 2; h++) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[h] = 1.0f / l;
        mb[h] = m_run[h] * LOG2E;
    }

    uint8_t* stage = smem + PG::STAGE_OFF;
    const int nrows = p.rows == 1 ? 1 : min(AG, T - g0);
    const size_t obase = ((size_t)sh * p.rows + g0) * T;      // element offset of the group's first row
    for (int kb = 0; kb < nkb; kb++, n++) {
        const uint32_t s = n & 1, k_s = smem_base + PG::K_OFF + s * G::TILE, release = kv_empty + 8 * s;
        mbar_wait(kv_full + 8 * s, (n >> 1) & 1);
        const int key0 = kb * AK, rem = kend - key0;
        if (rem > 64) probs_block<BF, DH, 16>(mb, inv, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc, lr0, stage, p.otype, release, lane);
        else if (rem > 32) probs_block<BF, DH, 8>(mb, inv, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc, lr0, stage, p.otype, release, lane);
        else if (rem > 16) probs_block<BF, DH, 4>(mb, inv, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc, lr0, stage, p.otype, release, lane);
        else probs_block<BF, DH, 2>(mb, inv, dq, dq_m, dq_t, k_s, key0, T, p.a.causal, wrow0, r0, tc, lr0, stage, p.otype, release, lane);
        // columns key0 .. min(key0 + 128, kend) - 1 of every row, one warp per row
        const int cw = min(AK, rem);
        if (p.otype == 0) {
            const float* sf = reinterpret_cast<const float*>(stage);
            float* o = reinterpret_cast<float*>(p.out) + obase + key0;
            for (int r = warp; r < nrows; r += 4)
                for (int c = lane; c < cw; c += 32) o[(size_t)r * T + c] = sf[r * PSTRIDE + c];
        } else {
            const uint16_t* sh16 = reinterpret_cast<const uint16_t*>(stage);
            uint16_t* o = reinterpret_cast<uint16_t*>(p.out) + obase + key0;
            for (int r = warp; r < nrows; r += 4)
                for (int c = lane; c < cw; c += 32) o[(size_t)r * T + c] = sh16[r * PSTRIDE + c];
        }
    }
    // a causal group's keys past its diagonal block: +0
    if (kend < T) {
        for (int r = warp; r < nrows; r += 4) {
            const size_t o = obase + (size_t)r * T;
            for (int c = kend + lane; c < T; c += 32) {
                if (p.otype == 0) reinterpret_cast<float*>(p.out)[o + c] = 0.f;
                else reinterpret_cast<uint16_t*>(p.out)[o + c] = 0;
            }
        }
    }
}

typedef CUresult (*EncodeTiledFn3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [nseq][T][3*H*dhp] view of the fused QKV activations (dhp = qkv_head_cols(dh)), box = `box_cols` columns x 64 tokens x 1
// sequence (zero fill past T): 64 columns with the 128-byte swizzle, 32 with the 64-byte swizzle, or 16 with the 32-byte swizzle
bool make_qkv_map(CUtensorMap* out, const void* qkv16, int nseq, int T, int H, int dh, int box_cols, CUtensorMapSwizzle swz) {
    static EncodeTiledFn3 enc = nullptr;
    if (!enc) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return false;
        enc = reinterpret_cast<EncodeTiledFn3>(f);
    }
    const cuuint64_t cols = (cuuint64_t)3 * H * qkv_head_cols(dh);
    const cuuint64_t dims[3] = {cols, (cuuint64_t)T, (cuuint64_t)nseq};
    const cuuint64_t strides[2] = {cols * 2, cols * 2 * (cuuint64_t)T};
    const cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)ABOX, 1}, estr[3] = {1, 1, 1};
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(qkv16), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the maps of every piece of a dh-wide head (AttnGeo): tm_mid is left zero unless dh == 104
bool make_piece_maps(AParams& p, CUtensorMap& tm_mid, const void* qkv16, int nseq, int T, int H, int dh) {
    memset(&tm_mid, 0, sizeof(tm_mid));
    if (!make_qkv_map(&p.tm_qkv, qkv16, nseq, T, H, dh, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return false;
    if (dh == 104 && !make_qkv_map(&tm_mid, qkv16, nseq, T, H, dh, 32, CU_TENSOR_MAP_SWIZZLE_64B)) return false;
    return dh == 64 || make_qkv_map(&p.tm_tail, qkv16, nseq, T, H, dh, 16, CU_TENSOR_MAP_SWIZZLE_32B);
}

template <int DH, Sched S>
cudaError_t set_k3_smem() {
    const cudaError_t e = cudaFuncSetAttribute(attention_tc_kernel<true, DH, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k3_smem<DH, S>());
    return e != cudaSuccess ? e : cudaFuncSetAttribute(attention_tc_kernel<false, DH, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k3_smem<DH, S>());
}

template <int DH>
cudaError_t set_smem() {
    cudaError_t e = set_k3_smem<DH, FIXED>();
    if (e == cudaSuccess) e = set_k3_smem<DH, PACKED>();
    if constexpr (DH == 64) {
        if (e == cudaSuccess) e = set_k3_smem<DH, PACKED_CAUSAL>();
    }
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attention_probs_kernel<true, DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ProbsGeo<DH>::SMEM);
    return e != cudaSuccess ? e : cudaFuncSetAttribute(attention_probs_kernel<false, DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ProbsGeo<DH>::SMEM);
}

template <int DH, Sched S>
cudaError_t launch_dh(const AParams& p, const CUtensorMap& tm_mid, const VarLen& v, unsigned grid, int bf16, cudaStream_t st) {
    constexpr uint32_t smem = k3_smem<DH, S>();
    static_assert(smem <= 227 * 1024, "shared memory per block");
    return bf16 ? launch_pdl(attention_tc_kernel<true, DH, S>, grid, (unsigned)ATT_THREADS, smem, st, 1, p, tm_mid, v)
                : launch_pdl(attention_tc_kernel<false, DH, S>, grid, (unsigned)ATT_THREADS, smem, st, 1, p, tm_mid, v);
}

// What both K3 launchers share once p's maps, out, T, H and causal (and FIXED's ngrp) are set: the group count, the grid and the
// dispatch on dh (PACKED_CAUSAL: 64 only) and bf16
template <Sched S>
cudaError_t launch_k3(AParams& p, const CUtensorMap& tm_mid, const VarLen& v, long long ngroups, int dh, int bf16, cudaStream_t st) {
    if (ngroups > 0x7ffffffell) return cudaErrorInvalidValue;
    p.ngroups = (int)ngroups;
    p.niter = (p.ngroups + 1) / 2;
    // persistent: at most one CTA per SM (the shared memory admits no second one)
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)min(p.niter, sms);
    if constexpr (S == PACKED_CAUSAL) e = launch_dh<64, S>(p, tm_mid, v, grid, bf16, st);
    else e = dh == 104 ? launch_dh<104, S>(p, tm_mid, v, grid, bf16, st) : dh == 80 ? launch_dh<80, S>(p, tm_mid, v, grid, bf16, st)
                                                                         : launch_dh<64, S>(p, tm_mid, v, grid, bf16, st);
    return e != cudaSuccess ? e : cudaGetLastError();
}

template <int DH>
cudaError_t launch_probs_dh(const PParams& p, const CUtensorMap& tm_mid, unsigned grid, int bf16, cudaStream_t st) {
    constexpr uint32_t smem = ProbsGeo<DH>::SMEM;
    return bf16 ? launch_pdl(attention_probs_kernel<true, DH>, grid, (unsigned)PROBS_THREADS, smem, st, 1, p, tm_mid)
                : launch_pdl(attention_probs_kernel<false, DH>, grid, (unsigned)PROBS_THREADS, smem, st, 1, p, tm_mid);
}

bool supported_dh(int dh) { return dh == 64 || dh == 80 || dh == 104; }

}  // namespace

cudaError_t attention_tc_init() {
    cudaError_t e = set_smem<64>();
    if (e == cudaSuccess) e = set_smem<80>();
    return e != cudaSuccess ? e : set_smem<104>();
}

cudaError_t launch_attention_tc(const void* qkv16, void* out16, int nseq, int T, int H, int dh, int causal, int bf16, cudaStream_t st) {
    if (!supported_dh(dh)) return cudaErrorInvalidValue;
    if (nseq <= 0) return cudaSuccess;
    AParams p;
    CUtensorMap tm_mid;
    memset(&p, 0, sizeof(p));
    if (!make_piece_maps(p, tm_mid, qkv16, nseq, T, H, dh)) return cudaErrorInvalidValue;
    p.out = (uint16_t*)out16; p.T = T; p.H = H; p.causal = causal;
    p.ngrp = (T + AG - 1) / AG;
    return launch_k3<FIXED>(p, tm_mid, VarLen{}, (long long)nseq * H * p.ngrp, dh, bf16, st);
}

cudaError_t launch_attention_tc_varlen(const void* qkv16, void* out16, int rows, int nseq, const int* d_seq, int groups, int H, int dh, int causal,
                                      int bf16, cudaStream_t st) {
    if (!supported_dh(dh) || (causal && dh != 64)) return cudaErrorInvalidValue;
    if (nseq <= 0) return cudaSuccess;
    AParams p;
    CUtensorMap tm_mid;
    memset(&p, 0, sizeof(p));
    if (!make_piece_maps(p, tm_mid, qkv16, 1, rows, H, dh)) return cudaErrorInvalidValue;
    p.out = (uint16_t*)out16; p.T = rows; p.H = H; p.causal = causal;
    const VarLen v{d_seq, d_seq + nseq + 1, nseq};
    const long long ngroups = (long long)groups * H;
    return causal ? launch_k3<PACKED_CAUSAL>(p, tm_mid, v, ngroups, dh, bf16, st) : launch_k3<PACKED>(p, tm_mid, v, ngroups, dh, bf16, st);
}

cudaError_t launch_attention_probs(const void* qkv16, void* out, int elem_type, int nseq, int T, int H, int dh, int causal, int cls_only,
                                   int bf16, cudaStream_t st) {
    if (!supported_dh(dh) || elem_type < 0 || elem_type > 2) return cudaErrorInvalidValue;
    if (nseq <= 0 || T <= 0) return cudaSuccess;
    PParams p;
    CUtensorMap tm_mid;
    memset(&p, 0, sizeof(p));
    if (!make_piece_maps(p.a, tm_mid, qkv16, nseq, T, H, dh)) return cudaErrorInvalidValue;
    p.a.T = T; p.a.H = H; p.a.causal = causal;
    p.a.ngrp = cls_only ? 1 : (T + AG - 1) / AG;
    p.out = out; p.otype = elem_type; p.rows = cls_only ? 1 : T;
    const long long units = (long long)nseq * H * p.a.ngrp;
    if (units > 0x7fffffffll) return cudaErrorInvalidValue;
    const unsigned grid = (unsigned)units;
    const cudaError_t e = dh == 104 ? launch_probs_dh<104>(p, tm_mid, grid, bf16, st)
                          : dh == 80 ? launch_probs_dh<80>(p, tm_mid, grid, bf16, st) : launch_probs_dh<64>(p, tm_mid, grid, bf16, st);
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace cb
