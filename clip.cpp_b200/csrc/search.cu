// search.cu -- scoring on the device: similarity matrix, softmax_with_sorting arithmetic, top-k selection.
//
// Replaces, for batches, the host loops of clip_zero_shot_label_image (clip.cpp:1624-1659: dot products clip.cpp:1525-1532,
// softmax_with_sorting clip.cpp:1591-1622) and the nearest-neighbour lookup of examples/image-search/search.cpp:114-158 (USearch
// there; brute force here: at <= 1e7 vectors the scan is one HBM pass).  Everything is fp32 on the CUDA cores ON PURPOSE: the whole
// 4096 x 1000 x 768 zero-shot problem is 6.3 GFLOP (0.008 % of the encode that produced the embeddings) and the ranking must not
// move in the 4th digit, which bf16 tensor-core products would do.  Each dot product is ONE sequential fmaf chain over k, the same
// order the reference's scalar loop uses.
//
// K10 (knn_kernel, below) is the separate, opt-in search over a database stored in 16 bits or in int8 with a scale per row:
// tensor-core scores and a top-k kept inside the kernel, so no score matrix ever reaches memory.  It shares the candidate order and
// the merge stage with the fp32 path.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <float.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace cb {

namespace {

constexpr int ST = 64, SK = 16;      // 64 x 64 output tile per CTA, k-chunks of 16 staged through shared memory

// S[i, j] = sum_k A[i, k] * B[j, k]   (A: [na, d] queries / images, B: [nb, d] labels / database rows), row-major fp32
__global__ void __launch_bounds__(256) sim_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ S,
                                                  int na, int nb, int d, size_t lds) {
    __shared__ float sa[SK][ST + 1], sb[SK][ST + 1];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;          // 16 x 16 threads, 4 x 4 outputs each
    const int i0 = blockIdx.y * ST, j0 = blockIdx.x * ST;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < d; k0 += SK) {
        for (int e = threadIdx.x; e < ST * SK; e += 256) {
            const int r = e / SK, k = e % SK;
            sa[k][r] = (i0 + r < na && k0 + k < d) ? A[(size_t)(i0 + r) * d + k0 + k] : 0.f;
            sb[k][r] = (j0 + r < nb && k0 + k < d) ? B[(size_t)(j0 + r) * d + k0 + k] : 0.f;
        }
        __syncthreads();
        #pragma unroll
        for (int k = 0; k < SK; k++) {
            float a[4], b[4];
            #pragma unroll
            for (int u = 0; u < 4; u++) { a[u] = sa[k][ty + 16 * u]; b[u] = sb[k][tx + 16 * u]; }
            #pragma unroll
            for (int u = 0; u < 4; u++)
                #pragma unroll
                for (int v = 0; v < 4; v++) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
        }
        __syncthreads();
    }
    #pragma unroll
    for (int u = 0; u < 4; u++)
        #pragma unroll
        for (int v = 0; v < 4; v++) {
            const int i = i0 + ty + 16 * u, j = j0 + tx + 16 * v;
            if (i < na && j < nb) S[(size_t)i * lds + j] = acc[u][v];
        }
}

CB_DEVINL double warp_sum_d(double v) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// p = (exp(s) + 1e-9) / sum  -- softmax_with_sorting's arithmetic (clip.cpp:1599-1607): exp in double, the element rounded to float,
// the sum of the rounded elements in double, the quotient rounded to float; no max subtraction (as the reference).
__global__ void __launch_bounds__(256) softmax_ref_kernel(float* __restrict__ x, int rows, int cols, size_t ld) {
    __shared__ double part[8];
    const int row = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (row >= rows) return;
    float* r = x + (size_t)row * ld;
    double s = 0.0;
    for (int i = threadIdx.x; i < cols; i += 256) { const float e = (float)(exp((double)r[i]) + 1e-9); r[i] = e; s += (double)e; }
    s = warp_sum_d(s);
    if (lane == 0) part[w] = s;
    __syncthreads();
    double tot = 0.0;
    #pragma unroll
    for (int i = 0; i < 8; i++) tot += part[i];
    for (int i = threadIdx.x; i < cols; i += 256) r[i] = (float)((double)r[i] / tot);
}

// One stage of top-k: the CTA (slice s, row r) sorts its <= SL candidates (value descending, ties by ascending index: a total
// order, unlike the reference's qsort whose tie order is unspecified) with a bitonic network in shared memory and emits the
// best kk.  in_idx == nullptr: candidate j of the row has index idx_base + j.
constexpr int SL = 4096;
struct Cand { float v; int i; };
CB_DEVINL bool before(const Cand& a, const Cand& b) { return a.v > b.v || (a.v == b.v && a.i < b.i); }

CB_DEVINL void knn_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }        // K10's two consumer warpgroups

// Bitonic network over c[0, m) in shared memory, m a power of two, run by threads 0-255: best first in `before` order.  Each step
// ends with a barrier of those threads: __syncthreads(), or knn_bar() (NAMED) where K10's producer warp does not take part.
template <bool NAMED>
CB_DEVINL void bitonic_sort(Cand* c, int m) {
    for (int size = 2; size <= m; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < (m >> 1); t += 256) {
                const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;            // final order: best first
                const Cand a = c[lo], b = c[hi];
                if (before(b, a) == desc) { c[lo] = b; c[hi] = a; }
            }
            if (NAMED) knn_bar();
            else __syncthreads();
        }
}

__global__ void __launch_bounds__(256) topk_stage_kernel(const float* __restrict__ vals, const int* __restrict__ in_idx, size_t ld, int n,
                                                         int idx_base, int kk, float* __restrict__ out_v, int* __restrict__ out_i,
                                                         size_t out_ld, int out_off) {
    __shared__ Cand c[SL];
    const int row = blockIdx.y, s0 = blockIdx.x * SL;
    const float* v = vals + (size_t)row * ld;
    const int* ii = in_idx ? in_idx + (size_t)row * ld : nullptr;
    const int cnt = min(SL, n - s0);
    int m = 1;
    while (m < cnt) m <<= 1;                                   // sort only the power of two that covers this slice
    for (int e = threadIdx.x; e < m; e += 256) {
        Cand x;
        if (e < cnt) {
            const float f = v[s0 + e];
            x.v = (f != f) ? -FLT_MAX : f;                     // NaN scores rank last instead of breaking the network
            x.i = ii ? ii[s0 + e] : idx_base + s0 + e;
        } else { x.v = -INFINITY; x.i = 0x7fffffff; }
        c[e] = x;
    }
    __syncthreads();
    bitonic_sort<false>(c, m);
    const int take = min(kk, cnt);
    float* ov = out_v + (size_t)row * out_ld + out_off + (size_t)blockIdx.x * kk;
    int* oi = out_i + (size_t)row * out_ld + out_off + (size_t)blockIdx.x * kk;
    for (int e = threadIdx.x; e < kk; e += 256) {
        ov[e] = e < take ? c[e].v : -INFINITY;
        oi[e] = e < take ? c[e].i : 0x7fffffff;
    }
}

// ---- K10: nearest-neighbour search over a 16-bit or int8 database on the tensor cores --------------------------------------------
// CTA = two consumer warpgroups (warps 0-7) + one producer warp (warp 8).  Work unit = (query tile of NQ = 8 NT <= 128 queries, database
// partition of rows_per_part rows); the partition is walked in tiles of KB = 128 rows, 64 per consumer warpgroup.
//   producer  one thread: per tile and per 64-column chunk of dim, the tile's database box [128 x 64] and the query box [NQ x 64]
//             (TMA, 128-byte swizzle, zero fill past n_db / n_q / dim) into a KSTAGES-deep mbarrier ring.
//             (NQ stops at 128: nine warps put three on one SM sub-partition, which leaves 168 registers a thread, too few for
//             n256's 128 accumulators.)
//   MMA       S[64 x NQ] = X.Q^T, database rows on the M side, queries on the N side, both K-major in shared memory: k16 steps in
//             dim order, fp32 accumulators.  The last chunk's zero-filled columns past dim add exact zeros (four steps per chunk
//             always: a data-dependent step count would serialise the wgmma chain).  A score's operations do not depend on where its row lies in the tile, the
//             partition or the database, so its bits depend on the query and the row alone.
//   select    per query the CTA keeps a candidate buffer in global memory (cap = kk + 2 KB entries) and a threshold theta in shared
//             memory: the kk-th best of the buffer after its last compaction (-inf before).  A score (NaN read as -FLT_MAX) enters
//             iff it is >= theta (ties are kept: the index order is settled by the sort).  A query whose buffer passed kk + KB entries
//             is compacted after the tile (bitonic sort in shared memory, best kk kept, theta raised), so one tile never overflows it.
//   end       every query's buffer is sorted once more and its best kk (padded with (-inf, INT_MAX)) go to the candidate matrix at
//             [query, partition * kk]; launch_topk_stage's merge passes finish the ranking across partitions.
// The int8 instance (KOp::S8) keeps all of this and changes three things.  A chunk is 128 bytes of a row either way, so 128 int8
// columns instead of 64 16-bit ones, and the boxes, the swizzle and the descriptor steps are the same.  The MMA is m64nNk32 s8.s8
// with int32 accumulators: exact sums, four k32 steps per chunk.  The score step turns each sum into
// fp32(fp32(float_rn(acc) * s_q) * s_x) before the theta test: the query scales s_q are staged in shared memory once per CTA, and
// each consumer thread loads the row scales s_x of its two rows per tile from global memory, guarded, so rows at or past row_end
// never read the scale array.
constexpr int KB = 128, KC = 64, KSTAGES = 4, KSORT = 2048;      // rows per tile, 16-bit columns per chunk, ring depth, sort capacity
constexpr int KNN_THREADS = 288;
constexpr uint32_t KDB_BYTES = KB * KC * 2;

template <KOp OP, int NT>
struct KnnGeo {
    static constexpr int NQ = 8 * NT;
    static constexpr uint32_t Q_BYTES = NQ * KC * 2, STAGE = KDB_BYTES + Q_BYTES;
    static constexpr uint32_t SORT_OFF = KSTAGES * STAGE;                     // Cand[KSORT]
    static constexpr uint32_t THETA_OFF = SORT_OFF + KSORT * 8;               // float[128]
    static constexpr uint32_t CNT_OFF = THETA_OFF + 128 * 4;                  // int[128]
    static constexpr uint32_t FLAG_OFF = CNT_OFF + 128 * 4;                   // uint32[4]: queries to compact
    static constexpr uint32_t BAR_OFF = FLAG_OFF + 32;                        // full[KSTAGES], empty[KSTAGES]
    static constexpr uint32_t QS_OFF = BAR_OFF + 16 * KSTAGES;                // S8 only: float[NQ] query scales
    static constexpr uint32_t SMEM = QS_OFF + (OP == KOp::S8 ? NQ * 4 : 0) + 1024;
    static_assert(Q_BYTES % 1024 == 0 && STAGE % 1024 == 0 && SMEM <= 227 * 1024, "K10 shared memory");
};

struct KParams {
    CUtensorMap tm_db, tm_q;
    Cand* buf;                      // [grid][NQ][cap]
    float* out_v; int* out_i;       // [nq, parts * kk], row stride out_ld
    size_t out_ld;
    int nq, ndb, nchunks, rows_per_part, parts, kk, cap;
    const float *qs, *xs;           // S8 only: query scales [nq], row scales [ndb]
    const uint4 *qb, *xb;           // K11 only: query and database bits [nq, dim / 128], [ndb, dim / 128], 16-byte words
    int dim;                        // K11 only: bits per row
    const IvfUnit* units;           // IVF instances only: the work unit of each CTA,
    const size_t* slot;             //   where pair p's run of range 0 starts in the candidate matrix (range r: + r * kk),
    const int* ids;                 //   and the original index of each stored row
    const uint8_t* codes;           // K13 only: stored codes [ndb, m],
    const float* tables;            //   each query's lookup tables [nq, m, 256],
    const float* pscore;            //   each pair's coarse score [npairs],
    const int* pair_q;              //   each pair's query [npairs],
    int m;                          //   and the subspaces
};

template <KOp OP, int NT>
CB_DEVINL void knn_mma(float (&d)[4 * NT], uint64_t da, uint64_t db, uint32_t accumulate) {
    constexpr bool BF = OP == KOp::BF16 || OP == KOp::BF16_IVF;
    if constexpr (NT == 16) wgmma_ss_n128<BF>(d, da, db, accumulate);
    else if constexpr (NT == 8) wgmma_ss_n64<BF>(d, da, db, accumulate);
    else if constexpr (NT == 4) wgmma_ss_n32<BF>(d, da, db, accumulate);
    else if constexpr (NT == 2) wgmma_ss_n16<BF>(d, da, db, accumulate);
    else wgmma_ss_n8<BF>(d, da, db, accumulate);
}
template <KOp OP, int NT>
CB_DEVINL void knn_mma(int (&d)[4 * NT], uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (NT == 16) wgmma_ss_n128_s8(d, da, db, accumulate);
    else if constexpr (NT == 8) wgmma_ss_n64_s8(d, da, db, accumulate);
    else if constexpr (NT == 4) wgmma_ss_n32_s8(d, da, db, accumulate);
    else if constexpr (NT == 2) wgmma_ss_n16_s8(d, da, db, accumulate);
    else wgmma_ss_n8_s8(d, da, db, accumulate);
}

// Sort query q's n buffered candidates (256 consumer threads) and keep the best kk: back into the buffer with theta raised
// (final = false), or into the candidate matrix row `orow` (final = true).
CB_DEVINL void knn_sort_keep(Cand* sc, Cand* b, int n, int kk, bool final, float* theta, int* cnt, float* ov, int* oi) {
    const int t = threadIdx.x;
    int m = 1;
    while (m < n) m <<= 1;
    for (int e = t; e < m; e += 256) sc[e] = e < n ? b[e] : Cand{-INFINITY, 0x7fffffff};
    knn_bar();
    bitonic_sort<true>(sc, m);
    if (final) {
        for (int e = t; e < kk; e += 256) {
            const Cand x = e < n ? sc[e] : Cand{-INFINITY, 0x7fffffff};
            ov[e] = x.v; oi[e] = x.i;
        }
    } else {
        for (int e = t; e < kk; e += 256) b[e] = sc[e];
        if (t == 0) { *theta = sc[kk - 1].v; *cnt = kk; }
    }
    knn_bar();
}

// The selection steps K10 and K11 share, run by their 256 consumer threads.  knn_push: a score v of (query q, row) that passed the
// kernel's admission test against theta[q] goes into q's buffer; a query whose buffer passed kk + KB entries is flagged.
CB_DEVINL void knn_push(const KParams& p, Cand* bufq, float v, int q, int row, int* cnt, uint32_t* flags) {
    const int pos = atomicAdd(&cnt[q], 1);
    *reinterpret_cast<float2*>(bufq + (size_t)q * p.cap + pos) = make_float2(v, __int_as_float(row));
    if (pos == p.kk + KB) atomicOr(&flags[q >> 5], 1u << (q & 31));
}

// After a tile: compact every flagged query's buffer to its best kk and raise its theta.
template <int NQ>
CB_DEVINL void knn_compact(const KParams& p, Cand* sort_s, Cand* bufq, float* theta, int* cnt, uint32_t* flags) {
    knn_bar();
    uint32_t fl[(NQ + 31) / 32];
    bool any = false;
    #pragma unroll
    for (int w = 0; w < (NQ + 31) / 32; w++) { fl[w] = flags[w]; any |= fl[w] != 0; }
    knn_bar();
    if (any) {                                                 // block-uniform
        if (threadIdx.x < 4) flags[threadIdx.x] = 0;
        #pragma unroll
        for (int w = 0; w < (NQ + 31) / 32; w++)
            for (uint32_t f = fl[w]; f; f &= f - 1) {
                const int q = 32 * w + __ffs(f) - 1;
                knn_sort_keep(sort_s, bufq + (size_t)q * p.cap, cnt[q], p.kk, false, &theta[q], &cnt[q], nullptr, nullptr);
            }
    }
}

// After the partition: each of the tile's nqv queries' best kk to the candidate matrix at [q0 + q, part * kk].
CB_DEVINL void knn_finish(const KParams& p, Cand* sort_s, Cand* bufq, const int* cnt, int nqv, int q0, int part) {
    for (int q = 0; q < nqv; q++) {
        const size_t o = (size_t)(q0 + q) * p.out_ld + (size_t)part * p.kk;
        knn_sort_keep(sort_s, bufq + (size_t)q * p.cap, cnt[q], p.kk, true, nullptr, nullptr, p.out_v + o, p.out_i + o);
    }
}

// A CTA's work: queries q0 .. q0 + nqv - 1 (rows of the query map) against rows row_begin .. row_end - 1, its run written as
// partition `part`.  K10 numbers its units from the plan; the IVF instances read them from the unit table.
struct KnnWork { int q0, nqv, part, row_begin, row_end; };

template <int NQ, bool IVF>
CB_DEVINL KnnWork knn_work(const KParams& p) {
    if constexpr (IVF) {
        const IvfUnit u = p.units[blockIdx.x];
        return KnnWork{u.p0, u.np, u.range, u.row_begin, u.row_end};
    } else {
        const int qt = blockIdx.x / p.parts, part = blockIdx.x - qt * p.parts;
        const int q0 = qt * NQ, row_begin = part * p.rows_per_part;
        return KnnWork{q0, min(NQ, p.nq - q0), part, row_begin, min(p.ndb, row_begin + p.rows_per_part)};
    }
}

// The IVF instances' end: pair q0 + q's best kk go to its own run, p.slot[q0 + q] + part * kk, with each stored position that
// knn_sort_keep wrote replaced by its original index (each thread rewrites the entries it wrote itself).
CB_DEVINL void knn_finish_ivf(const KParams& p, Cand* sort_s, Cand* bufq, const int* cnt, int nqv, int q0, int part) {
    for (int q = 0; q < nqv; q++) {
        const size_t o = p.slot[q0 + q] + (size_t)part * p.kk;
        knn_sort_keep(sort_s, bufq + (size_t)q * p.cap, cnt[q], p.kk, true, nullptr, nullptr, p.out_v + o, p.out_i + o);
        for (int e = threadIdx.x; e < p.kk; e += 256) {
            const int i = p.out_i[o + e];
            if (i != 0x7fffffff) p.out_i[o + e] = p.ids[i];
        }
    }
}

template <KOp OP, int NT>
__global__ void __launch_bounds__(KNN_THREADS, 1) knn_kernel(const __grid_constant__ KParams p) {
    using G = KnnGeo<OP, NT>;
    constexpr int NQ = G::NQ;
    constexpr bool S8 = OP == KOp::S8, IVF = OP == KOp::F16_IVF || OP == KOp::BF16_IVF;
    constexpr int KCOL = S8 ? 2 * KC : KC;                         // elements in a chunk's 128 bytes
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t full = smem_base + G::BAR_OFF, empty = full + 8 * KSTAGES;
    Cand* sort_s = reinterpret_cast<Cand*>(smem + G::SORT_OFF);
    float* theta = reinterpret_cast<float*>(smem + G::THETA_OFF);
    int* cnt = reinterpret_cast<int*>(smem + G::CNT_OFF);
    uint32_t* flags = reinterpret_cast<uint32_t*>(smem + G::FLAG_OFF);
    float* qscale = reinterpret_cast<float*>(smem + G::QS_OFF);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int qt = blockIdx.x / p.parts, part = blockIdx.x - qt * p.parts;
    int q0 = qt * NQ, nqv = min(NQ, p.nq - q0);
    int row_begin = part * p.rows_per_part, row_end = min(p.ndb, row_begin + p.rows_per_part);
    if constexpr (IVF) {
        const IvfUnit u = p.units[blockIdx.x];
        q0 = u.p0; nqv = u.np; part = u.range; row_begin = u.row_begin; row_end = u.row_end;
    }
    const int ntiles = (row_end - row_begin + KB - 1) / KB;
    if (threadIdx.x == 0) {
        for (int i = 0; i < KSTAGES; i++) { mbar_init(full + 8 * i, 1); mbar_init(empty + 8 * i, 8); }
        mbar_fence_init();
        tma_prefetch_desc(&p.tm_db);
        tma_prefetch_desc(&p.tm_q);
    }
    if (threadIdx.x < 128) { theta[threadIdx.x] = -INFINITY; cnt[threadIdx.x] = 0; }
    if (threadIdx.x < 4) flags[threadIdx.x] = 0;
    if constexpr (S8)
        if (threadIdx.x < NQ) qscale[threadIdx.x] = (int)threadIdx.x < nqv ? p.qs[q0 + threadIdx.x] : 0.f;
    __syncthreads();

    if (warp == 8) {
        // ------------------------------------------------------------------ producer (one thread)
        if (lane == 0) {
            uint32_t n = 0;
            for (int t = 0; t < ntiles; t++)
                for (int c = 0; c < p.nchunks; c++, n++) {
                    const uint32_t s = n % KSTAGES, st = smem_base + s * G::STAGE;
                    mbar_wait(empty + 8 * s, ((n / KSTAGES) & 1) ^ 1);
                    mbar_arrive_expect_tx(full + 8 * s, G::STAGE);
                    tma_load_2d(st, &p.tm_db, c * KCOL, row_begin + t * KB, full + 8 * s);
                    tma_load_2d(st + KDB_BYTES, &p.tm_q, c * KCOL, q0, full + 8 * s);
                }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers (fragment layout: wgmma.cuh)
    const int wg = warp >> 2, tc = 2 * (lane & 3);
    const int rr = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // this thread: tile rows rr and rr + 8
    Cand* const bufq = p.buf + (size_t)blockIdx.x * NQ * p.cap;
    std::conditional_t<S8, int, float> d[4 * NT];
    uint32_t n = 0;
    for (int t = 0; t < ntiles; t++) {
        float xs[2] = {0.f, 0.f};                                  // S8: the scales of rows rr and rr + 8, loaded under the MMAs
        if constexpr (S8) {
            const int r = row_begin + t * KB + rr;
            if (r < row_end) xs[0] = p.xs[r];
            if (r + 8 < row_end) xs[1] = p.xs[r + 8];
        }
        uint32_t prev = 0;
        for (int c = 0; c < p.nchunks; c++, n++) {
            const uint32_t s = n % KSTAGES, st = smem_base + s * G::STAGE;
            mbar_wait(full + 8 * s, (n / KSTAGES) & 1);
            const uint64_t da = wgmma_desc_sw128(st + (uint32_t)wg * 64u * 128u), dq = wgmma_desc_sw128(st + KDB_BYTES);
            wgmma_fence();
            #pragma unroll
            for (int k = 0; k < 4; k++) knn_mma<OP, NT>(d, da + 2 * k, dq + 2 * k, (uint32_t)(c | k));
            wgmma_commit();
            if (c > 0) {                                           // the previous chunk's MMAs have read their stage
                wgmma_wait<1>();
                __syncwarp();
                if (lane == 0) mbar_arrive(empty + 8 * prev);
            }
            prev = s;
        }
        wgmma_wait<0>();
        wgmma_fence_regs(d);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + 8 * prev);

        // candidates of this tile
        const int row0 = row_begin + t * KB + rr;
        #pragma unroll
        for (int j = 0; j < NT; j++) {
            #pragma unroll
            for (int e = 0; e < 4; e++) {
                const int q = 8 * j + tc + (e & 1), row = row0 + 8 * (e >> 1);
                float v;
                if constexpr (S8) v = __fmul_rn(__fmul_rn(__int2float_rn(d[4 * j + e]), qscale[q]), xs[e >> 1]);
                else v = d[4 * j + e];
                v = v != v ? -FLT_MAX : v;
                if (q < nqv && row < row_end && v >= theta[q]) knn_push(p, bufq, v, q, row, cnt, flags);   // ties kept
            }
        }
        knn_compact<NQ>(p, sort_s, bufq, theta, cnt, flags);
    }
    if constexpr (IVF) knn_finish_ivf(p, sort_s, bufq, cnt, nqv, q0, part);
    else knn_finish(p, sort_s, bufq, cnt, nqv, q0, part);
}

// ---- K11: Hamming top-k over a binary database on the tensor cores --------------------------------------------------------------
// Same work unit, plan, candidate buffers and selection as K10 (KParams, knn_push / knn_compact / knn_finish); 256 threads, eight
// warps of 16 rows each, so a tile is the same KB = 128 rows.  No TMA: each thread loads its rows' bits straight into registers.
//   bits      a row is W = dim / 128 16-byte words, taken in blocks of four words (64 bytes, two k256 steps), blocks past the row's
//             last word zero.  Thread (g = lane / 4, t = lane % 4) holds word 4 b + t of block b of rows g and g + 8: x, y of that word
//             feed k-step 2 b as A's slots t and t + 4, z, w feed k-step 2 b + 1.  The query tile sits in shared memory in the same
//             word order, so B's registers for query n are the same two words of that query: the k order is a permutation of the
//             bits, which a sum of popcounts does not see, and zero words add nothing.
//   MMA       mma.sync m16n8k256 b1.and.popc: a = popc(q & x), exact int32.  Hopper has no b1 wgmma; .xor.popc is not one native
//             instruction on sm_90a, .and.popc is (BMMA.168256.AND.POPC).
//   score     s = dim - 2 popc(q) - 2 popc(x) + 4 a = dim - 2 popc(q ^ x), the dot product of the +-1 vectors, an exact integer
//             float; popc(x) from the thread's registers summed over its four lanes, popc(q) staged once per CTA.
//   ties      scores take at most dim + 1 values, so ties are the normal case.  Rows reach a CTA in increasing index, so once a
//             query's buffer has been compacted to its best kk, a later row with s == theta ranks after all kk of them (equal score,
//             higher index) and can never enter: after the first compaction the admission test is s > theta, exactly.  Before it
//             theta is -inf, which every (finite) score passes.  With K10's s >= theta an all-equal database would compact every tile.
constexpr int B1_THREADS = 256;

template <int NT>
struct B1Geo {
    static constexpr int NQ = 8 * NT;
    static constexpr uint32_t SORT_OFF = 0;                                   // Cand[KSORT]
    static constexpr uint32_t THETA_OFF = SORT_OFF + KSORT * 8;               // float[128]
    static constexpr uint32_t CNT_OFF = THETA_OFF + 128 * 4;                  // int[128]
    static constexpr uint32_t PQ_OFF = CNT_OFF + 128 * 4;                     // int[128]: popc of each query
    static constexpr uint32_t FLAG_OFF = PQ_OFF + 128 * 4;                    // uint32[4]
    static constexpr uint32_t Q_OFF = FLAG_OFF + 16;                          // uint4[NQ][qstride]
    // query row stride in 16-byte words: 4 per block, an odd number of blocks, so that rows g and g + 1 of one 8-thread phase of a
    // 16-byte shared load fall in different halves of the 32 banks
    __host__ __device__ static int qstride(int nblk) { return 4 * (nblk | 1); }
    static uint32_t smem(int nblk) { return Q_OFF + (uint32_t)NQ * qstride(nblk) * 16; }
};

CB_DEVINL void bmma_and_popc(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

CB_DEVINL int popc4(const uint4& v) { return __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w); }

template <int NT>
__global__ void __launch_bounds__(B1_THREADS, NT >= 8 ? 1 : 2) knn_b1_kernel(const __grid_constant__ KParams p) {
    using G = B1Geo<NT>;
    constexpr int NQ = G::NQ;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 15) & ~(uintptr_t)15);
    Cand* sort_s = reinterpret_cast<Cand*>(smem + G::SORT_OFF);
    float* theta = reinterpret_cast<float*>(smem + G::THETA_OFF);
    int* cnt = reinterpret_cast<int*>(smem + G::CNT_OFF);
    int* pq = reinterpret_cast<int*>(smem + G::PQ_OFF);
    uint32_t* flags = reinterpret_cast<uint32_t*>(smem + G::FLAG_OFF);
    uint4* sq = reinterpret_cast<uint4*>(smem + G::Q_OFF);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    const int qt = blockIdx.x / p.parts, part = blockIdx.x - qt * p.parts;
    const int q0 = qt * NQ, nqv = min(NQ, p.nq - q0);
    const int row_begin = part * p.rows_per_part, row_end = min(p.ndb, row_begin + p.rows_per_part);
    const int ntiles = (row_end - row_begin + KB - 1) / KB;
    const int W = p.dim / 128, nblk = (W + 3) / 4, qs = G::qstride(nblk);

    if (threadIdx.x < 128) { theta[threadIdx.x] = -INFINITY; cnt[threadIdx.x] = 0; }
    if (threadIdx.x < 4) flags[threadIdx.x] = 0;
    for (int e = threadIdx.x; e < NQ * qs; e += B1_THREADS) {
        const int q = e / qs, w = e - q * qs;
        sq[e] = q < nqv && w < W ? p.qb[(size_t)(q0 + q) * W + w] : make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    if (threadIdx.x < NQ) {
        int s = 0;
        for (int w = 0; w < W; w++) s += popc4(sq[threadIdx.x * qs + w]);
        pq[threadIdx.x] = s;
    }
    __syncthreads();

    Cand* const bufq = p.buf + (size_t)blockIdx.x * NQ * p.cap;
    for (int t = 0; t < ntiles; t++) {
        const int row0 = row_begin + t * KB + warp * 16 + g;           // this thread: rows row0 and row0 + 8
        uint4 a[2][4];
        #pragma unroll
        for (int h = 0; h < 2; h++)
            #pragma unroll
            for (int b = 0; b < 4; b++) {
                const int w = 4 * b + tg, r = row0 + 8 * h;
                a[h][b] = b < nblk && w < W && r < row_end ? p.xb[(size_t)r * W + w] : make_uint4(0, 0, 0, 0);
            }
        int px[2];
        #pragma unroll
        for (int h = 0; h < 2; h++) {
            px[h] = popc4(a[h][0]) + popc4(a[h][1]) + popc4(a[h][2]) + popc4(a[h][3]);
            px[h] += __shfl_xor_sync(0xffffffffu, px[h], 1);
            px[h] += __shfl_xor_sync(0xffffffffu, px[h], 2);
        }
        int d[NT][4];
        #pragma unroll
        for (int j = 0; j < NT; j++) d[j][0] = d[j][1] = d[j][2] = d[j][3] = 0;
        #pragma unroll
        for (int b = 0; b < 4; b++) {
            if (b >= nblk) break;
            #pragma unroll
            for (int j = 0; j < NT; j++) {
                const uint4 bq = sq[(8 * j + g) * qs + 4 * b + tg];
                bmma_and_popc(d[j], a[0][b].x, a[1][b].x, a[0][b].y, a[1][b].y, bq.x, bq.y);
                bmma_and_popc(d[j], a[0][b].z, a[1][b].z, a[0][b].w, a[1][b].w, bq.z, bq.w);
            }
        }
        // candidates of this tile (accumulator layout: d[j][e] is row row0 + 8 (e >> 1), query 8 j + 2 tg + (e & 1))
        #pragma unroll
        for (int j = 0; j < NT; j++) {
            #pragma unroll
            for (int e = 0; e < 4; e++) {
                const int q = 8 * j + 2 * tg + (e & 1), row = row0 + 8 * (e >> 1);
                const float v = (float)(p.dim - 2 * pq[q] - 2 * px[e >> 1] + 4 * d[j][e]);
                if (q < nqv && row < row_end && v > theta[q]) knn_push(p, bufq, v, q, row, cnt, flags);     // strict: see above
            }
        }
        knn_compact<NQ>(p, sort_s, bufq, theta, cnt, flags);
    }
    knn_finish(p, sort_s, bufq, cnt, nqv, q0, part);
}

// ---- K12: exact rescoring of a candidate list --------------------------------------------------------------------------------------
// One CTA per query: the query, widened to f32, in shared memory; the candidates sorted by index (bitonic_sort with equal values) so
// that out-of-range entries (index INT_MAX after staging) go last and duplicates sit side by side, the first of each run kept; each
// thread walks its candidates' rows with 16-byte loads, one fmaf chain per row from +0 over features 0 .. dim - 1 (sim_kernel's
// order); then the family's order and the best kk.  A dropped entry is (-inf, INT_MAX) in the sort, after every valid candidate
// (a valid -inf score has a lower index), and (-inf, -1) in the output.
constexpr int RS_MAX = 2048, RS_PER = RS_MAX / 256;

template <int T>   // element type: 0 f32, 1 f16, 2 bf16 (CLIP_B200_OUT_*)
CB_DEVINL void widen8(const uint4& u, float (&f)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    #pragma unroll
    for (int i = 0; i < 4; i++) {
        if constexpr (T == 1) {
            const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
            f[2 * i] = h.x; f[2 * i + 1] = h.y;
        } else {
            f[2 * i] = __uint_as_float(w[i] << 16); f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
}

template <int T>
__global__ void __launch_bounds__(256) rescore_kernel(const void* __restrict__ q, const void* __restrict__ db, int ndb, int dim,
                                                      const int* __restrict__ cand, int n_cand, int kk, float* __restrict__ out_v,
                                                      int* __restrict__ out_i, size_t out_ld) {
    __shared__ Cand c[RS_MAX];
    __shared__ __align__(16) float sq[2048];
    constexpr int ESZ = T == 0 ? 4 : 2, EPV = 16 / ESZ;             // element bytes, elements per 16-byte load
    const int row = blockIdx.x;
    const size_t rbytes = (size_t)dim * ESZ;
    const uint4* qr = reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(q) + row * rbytes);
    for (int e = threadIdx.x; e < dim / EPV; e += 256) {
        const uint4 u = qr[e];
        if constexpr (T == 0) *reinterpret_cast<uint4*>(sq + 4 * e) = u;
        else {
            float f[8];
            widen8<T>(u, f);
            #pragma unroll
            for (int i = 0; i < 8; i++) sq[8 * e + i] = f[i];
        }
    }
    int m = 1;
    while (m < n_cand) m <<= 1;
    const int* cr = cand + (size_t)row * n_cand;
    for (int e = threadIdx.x; e < m; e += 256) {
        const int i = e < n_cand ? cr[e] : -1;
        c[e] = Cand{0.f, i >= 0 && i < ndb ? i : 0x7fffffff};
    }
    __syncthreads();
    bitonic_sort<false>(c, m);
    Cand mine[RS_PER];
    #pragma unroll
    for (int u = 0; u < RS_PER; u++) {
        const int e = threadIdx.x + 256 * u;
        Cand x{-INFINITY, 0x7fffffff};
        if (e < m) {
            const int i = c[e].i;
            if (i != 0x7fffffff && (e == 0 || c[e - 1].i != i)) {
                const uint4* xr = reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(db) + (size_t)i * rbytes);
                float acc = 0.f;
                #pragma unroll 4
                for (int k = 0; k < dim / EPV; k++) {
                    const uint4 v = xr[k];
                    if constexpr (T == 0) {
                        acc = fmaf(sq[4 * k], __uint_as_float(v.x), acc);
                        acc = fmaf(sq[4 * k + 1], __uint_as_float(v.y), acc);
                        acc = fmaf(sq[4 * k + 2], __uint_as_float(v.z), acc);
                        acc = fmaf(sq[4 * k + 3], __uint_as_float(v.w), acc);
                    } else {
                        float f[8];
                        widen8<T>(v, f);
                        #pragma unroll
                        for (int j = 0; j < 8; j++) acc = fmaf(sq[8 * k + j], f[j], acc);
                    }
                }
                x = Cand{acc != acc ? -FLT_MAX : acc, i};
            }
        }
        mine[u] = x;
    }
    __syncthreads();
    #pragma unroll
    for (int u = 0; u < RS_PER; u++)
        if (threadIdx.x + 256 * u < m) c[threadIdx.x + 256 * u] = mine[u];
    __syncthreads();
    bitonic_sort<false>(c, m);
    for (int e = threadIdx.x; e < kk; e += 256) {
        const Cand x = e < m ? c[e] : Cand{-INFINITY, 0x7fffffff};
        out_v[(size_t)row * out_ld + e] = x.i == 0x7fffffff ? -INFINITY : x.v;
        out_i[(size_t)row * out_ld + e] = x.i == 0x7fffffff ? -1 : x.i;
    }
}

// B1 quantiser: one warp per 128 features, which is one 16-byte output word: the rows are whole words, so word w of the flat
// [n * dim / 128] array reads floats 128 w .. 128 w + 127 and centre features 128 (w % (dim / 128)) + ...  Lane l compares its
// float4 (features 4 l .. 4 l + 3) with the centre, IEEE > with nothing flushed (the build has no -ftz), four bits LSB first; eight
// lanes OR their nibbles into a 32-bit word and lane 0 stores the four words.
__global__ void __launch_bounds__(256) quant_b1_kernel(const float4* __restrict__ x, size_t nwords, int wpr, const float4* __restrict__ center,
                                                       uint4* __restrict__ bits) {
    const int lane = threadIdx.x & 31;
    const size_t step = (size_t)gridDim.x * 8;
    for (size_t w = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5); w < nwords; w += step) {
        const float4 v = x[w * 32 + lane];
        const float4 c = center ? center[(w % wpr) * 32 + lane] : make_float4(0.f, 0.f, 0.f, 0.f);
        uint32_t nib = (v.x > c.x ? 1u : 0u) | (v.y > c.y ? 2u : 0u) | (v.z > c.z ? 4u : 0u) | (v.w > c.w ? 8u : 0u);
        nib <<= 4 * (lane & 7);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 1);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 2);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 4);
        const uint32_t w1 = __shfl_sync(0xffffffffu, nib, 8), w2 = __shfl_sync(0xffffffffu, nib, 16), w3 = __shfl_sync(0xffffffffu, nib, 24);
        if (lane == 0) bits[w] = make_uint4(nib, w1, w2, w3);
    }
}

// ---- IVF layout and k-means update -----------------------------------------------------------------------------------------------
// Row gather: dst[p] = src[idx[p]], rows of w16 16-byte words, 64-bit offsets (n * dim * 2 may pass 2^32).
__global__ void __launch_bounds__(256) gather_rows16_kernel(const uint4* __restrict__ src, const int* __restrict__ idx, size_t n, int w16,
                                                            uint4* __restrict__ dst) {
    const size_t total = n * (size_t)w16, step = (size_t)gridDim.x * 256;
    for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < total; e += step) {
        const size_t r = e / w16, w = e - r * w16;
        dst[e] = src[(size_t)idx[r] * w16 + w];
    }
}

__global__ void __launch_bounds__(256) fill_cand_kernel(float* __restrict__ v, int* __restrict__ i, size_t n) {
    const size_t step = (size_t)gridDim.x * 256;
    for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < n; e += step) { v[e] = -INFINITY; i[e] = 0x7fffffff; }
}

template <bool BF>
CB_DEVINL double load16(const uint16_t* x, size_t e) {
    const uint16_t h = x[e];
    if constexpr (BF) return (double)__uint_as_float((uint32_t)h << 16);
    else return (double)__half2float(__ushort_as_half(h));
}

// k-means sums, pass 1: chunk c = (the list-ordered members ids[begin .. end - 1]) -> part[c, dim], each feature summed in fp64 over
// the chunk's members in order (one thread per feature, so the order is fixed).
template <bool BF>
__global__ void __launch_bounds__(256) ivf_chunk_sum_kernel(const uint16_t* __restrict__ x, int dim, const int* __restrict__ ids,
                                                            const int2* __restrict__ chunks, double* __restrict__ part) {
    const int2 ch = chunks[blockIdx.x];
    for (int f = threadIdx.x; f < dim; f += 256) {
        double s = 0.0;
        for (int r = ch.x; r < ch.y; r++) s += load16<BF>(x, (size_t)ids[r] * dim + f);
        part[(size_t)blockIdx.x * dim + f] = s;
    }
}

// k-means sums, pass 2, one CTA per list: m = (the list's chunk sums added in chunk order) / count, then c = rne16(m / sqrt(sum m^2)),
// in fp64, the squares summed by a fixed tree (each thread's features in order, then warps, then the eight warp sums in order).  An
// empty list, or a mean that is exactly zero, leaves the centroid as it was.
template <bool BF>
__global__ void __launch_bounds__(256) ivf_update_kernel(const double* __restrict__ part, const int* __restrict__ chunk_begin,
                                                         const int* __restrict__ offsets, int dim, uint16_t* __restrict__ cent) {
    __shared__ double mean[2048], wsum[8];
    const int l = blockIdx.x, count = offsets[l + 1] - offsets[l];
    if (count == 0) return;
    const int c0 = chunk_begin[l], c1 = chunk_begin[l + 1];
    double sq = 0.0;
    for (int f = threadIdx.x; f < dim; f += 256) {
        double s = 0.0;
        for (int c = c0; c < c1; c++) s += part[(size_t)c * dim + f];
        const double m = s / (double)count;
        mean[f] = m;
        sq += m * m;
    }
    sq = warp_sum_d(sq);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = sq;
    __syncthreads();
    double tot = 0.0;
    #pragma unroll
    for (int w = 0; w < 8; w++) tot += wsum[w];
    if (tot == 0.0) return;
    const double nrm = sqrt(tot);
    for (int f = threadIdx.x; f < dim; f += 256) {
        const double v = mean[f] / nrm;
        cent[(size_t)l * dim + f] = BF ? __bfloat16_as_ushort(__double2bfloat16(v)) : __half_as_ushort(__double2half(v));
    }
}

// ---- IVF-PQ: residual codebooks, encoding, lookup tables and the ADC scan (K13) ----------------------------------------------------
template <bool BF>
CB_DEVINL float widen16(uint16_t h) {
    if constexpr (BF) return __uint_as_float((uint32_t)h << 16);
    else return __half2float(__ushort_as_half(h));
}

// feature f of row `row`'s residual against its list's centroid: x - c in fp32, rounded to nearest, both widened exactly
template <bool BF>
CB_DEVINL float pq_residual(const uint16_t* x, const uint16_t* cent, const int* lists, size_t row, int dim, int f) {
    return __fsub_rn(widen16<BF>(x[row * dim + f]), widen16<BF>(cent[(size_t)lists[row] * dim + f]));
}

// Codes, one thread per (row, subspace s = blockIdx.y): the residual's dsub features staged feature-major in shared memory (each
// thread reads only its own column), then the 256 codewords of s in order, d = fmaf(t, t, d) with t = r_j - b_j from +0 in feature
// order; a NaN distance is +inf; the least distance wins, the lower index on ties (strict <), so all-inf gives code 0.  Every thread
// of a warp reads the same codeword element: one broadcast load.
constexpr int PQ_ENC_THREADS = 128;
template <bool BF>
__global__ void __launch_bounds__(PQ_ENC_THREADS) pq_encode_kernel(const uint16_t* __restrict__ x, size_t n, int dim, int m,
                                                                   const int* __restrict__ lists, const uint16_t* __restrict__ cent,
                                                                   const float* __restrict__ books, uint8_t* __restrict__ codes) {
    extern __shared__ float sr[];                                          // [dsub][PQ_ENC_THREADS]
    const int s = blockIdx.y, dsub = dim / m, t = threadIdx.x;
    const size_t row = (size_t)blockIdx.x * PQ_ENC_THREADS + t;
    if (row >= n) return;
    for (int j = 0; j < dsub; j++) sr[j * PQ_ENC_THREADS + t] = pq_residual<BF>(x, cent, lists, row, dim, s * dsub + j);
    const float* b = books + (size_t)s * 256 * dsub;
    float best = INFINITY;
    int bi = 0;
    for (int k = 0; k < 256; k++) {
        float d = 0.f;
        for (int j = 0; j < dsub; j++) {
            const float e = __fsub_rn(sr[j * PQ_ENC_THREADS + t], __ldg(b + k * dsub + j));
            d = fmaf(e, e, d);
        }
        if (d != d) d = INFINITY;
        if (d < best) { best = d; bi = k; }
    }
    codes[row * m + s] = (uint8_t)bi;
}

// Initial codebooks, one CTA per subspace: codeword i of s is the residual of training row floor(i n / 256).
template <bool BF>
__global__ void __launch_bounds__(256) pq_init_kernel(const uint16_t* __restrict__ x, size_t n, int dim, int m, const int* __restrict__ lists,
                                                      const uint16_t* __restrict__ cent, float* __restrict__ books) {
    const int s = blockIdx.x, dsub = dim / m;
    for (int e = threadIdx.x; e < 256 * dsub; e += 256) {
        const int i = e / dsub, j = e - i * dsub;
        books[(size_t)s * 256 * dsub + e] = pq_residual<BF>(x, cent, lists, (size_t)i * n / 256, dim, s * dsub + j);
    }
}

// Codebook k-means sums, pass 1: chunk c = positions ch.x .. ch.y - 1 of the flat member array ids [m][n] (one codeword's members
// of subspace s = ch.x / n, in row order) -> part[c, dsub], each feature's residual summed in fp64 over the chunk in order.
template <bool BF>
__global__ void __launch_bounds__(128) pq_chunk_sum_kernel(const uint16_t* __restrict__ x, size_t n, int dim, int m, const int* __restrict__ lists,
                                                           const uint16_t* __restrict__ cent, const int* __restrict__ ids,
                                                           const longlong2* __restrict__ chunks, double* __restrict__ part) {
    const longlong2 ch = chunks[blockIdx.x];
    const int dsub = dim / m, s = (int)(ch.x / (long long)n);
    for (int j = threadIdx.x; j < dsub; j += 128) {
        double acc = 0.0;
        for (long long r = ch.x; r < ch.y; r++) acc += (double)pq_residual<BF>(x, cent, lists, (size_t)ids[r], dim, s * dsub + j);
        part[(size_t)blockIdx.x * dsub + j] = acc;
    }
}

// Pass 2, one CTA per (subspace, codeword) = blockIdx.x: the chunk sums added in chunk order, over the count in fp64, rounded once
// to fp32.  An empty codeword keeps its value.
__global__ void __launch_bounds__(128) pq_update_kernel(const double* __restrict__ part, const int* __restrict__ chunk_begin,
                                                        const int* __restrict__ count, int dsub, float* __restrict__ books) {
    const int bk = blockIdx.x, cnt = count[bk];
    if (cnt == 0) return;
    for (int j = threadIdx.x; j < dsub; j += 128) {
        double acc = 0.0;
        for (int c = chunk_begin[bk]; c < chunk_begin[bk + 1]; c++) acc += part[(size_t)c * dsub + j];
        books[(size_t)bk * dsub + j] = __double2float_rn(acc / (double)cnt);
    }
}

// Lookup tables, one CTA per (subspace s = blockIdx.x, PQ_TQ queries): codebook s staged [256][dsub | 1] (an odd row stride, so
// thread k's reads of row k fall in distinct banks) and the queries' dsub features widened; thread k writes
// T[q][s][k] = fmaf chain over j of q_j * b_kj from +0, in feature order.
constexpr int PQ_TQ = 32;
template <bool BF>
__global__ void __launch_bounds__(256) pq_table_kernel(const uint16_t* __restrict__ q, int nq, int dim, int m, const float* __restrict__ books,
                                                       float* __restrict__ tables) {
    extern __shared__ float sm[];
    const int s = blockIdx.x, q0 = blockIdx.y * PQ_TQ, nqv = min(PQ_TQ, nq - q0), dsub = dim / m, ld = dsub | 1, k = threadIdx.x;
    float* sb = sm;
    float* sq = sm + 256 * ld;
    for (int e = threadIdx.x; e < 256 * dsub; e += 256) { const int i = e / dsub; sb[i * ld + e - i * dsub] = books[(size_t)s * 256 * dsub + e]; }
    for (int e = threadIdx.x; e < nqv * dsub; e += 256) {
        const int i = e / dsub;
        sq[e] = widen16<BF>(q[(size_t)(q0 + i) * dim + s * dsub + e - i * dsub]);
    }
    __syncthreads();
    for (int i = 0; i < nqv; i++) {
        float acc = 0.f;
        for (int j = 0; j < dsub; j++) acc = fmaf(sq[i * dsub + j], sb[k * ld + j], acc);
        tables[((size_t)(q0 + i) * m + s) * 256 + k] = acc;
    }
}

// ---- K13: the ADC scan over one IVF work unit ----------------------------------------------------------------------------------
// The unit table of K10's IVF instances: CTA u runs unit u, pairs p0 .. p0 + np - 1 of one list against stored rows row_begin ..
// row_end - 1.  256 threads over rows, one pair at a time:
//   table    the pair's query's table T [m][256] fp32 in shared memory, in slices of up to PQ_SLICE subspaces (128 KiB).  With one
//            slice it is staged once per pair; with more, once per slice per 256-row tile, each row's running sum carried in a
//            register from slice to slice, so the sum's order is s = 0 .. m - 1 whatever the slicing.
//   row      v = coarse score, then v += T[s][code_s] in fp32 for s in order; codes read 16 at a time (one 16-byte load).  Threads
//            over rows look up random codes, so a lookup costs as many shared-memory wavefronts as its warp has codes in one bank.
//   select   K10's steps on one query: admission v >= theta (NaN read as -FLT_MAX), knn_push / knn_compact after each 256-row
//            tile, and knn_finish_ivf's end (the pair's best kk to its run, positions mapped to original indices).  A tile adds at
//            most 256 entries to a buffer compacted past kk + KB, so cap = kk + KB + 256 <= KSORT.
constexpr int ADC_THREADS = 256, PQ_SLICE = 128;

__global__ void __launch_bounds__(ADC_THREADS, 2) adc_kernel(const __grid_constant__ KParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 15) & ~(uintptr_t)15);
    Cand* sort_s = reinterpret_cast<Cand*>(smem);
    float* theta = reinterpret_cast<float*>(smem + KSORT * 8);
    int* cnt = reinterpret_cast<int*>(smem + KSORT * 8 + 16);
    uint32_t* flags = reinterpret_cast<uint32_t*>(smem + KSORT * 8 + 32);
    float* tab = reinterpret_cast<float*>(smem + KSORT * 8 + 64);
    const IvfUnit u = p.units[blockIdx.x];
    const int m = p.m, nsl = (m + PQ_SLICE - 1) / PQ_SLICE;
    Cand* const bufq = p.buf + (size_t)blockIdx.x * p.cap;
    for (int j = 0; j < u.np; j++) {
        const int pair = u.p0 + j;
        const float4* T = reinterpret_cast<const float4*>(p.tables + (size_t)p.pair_q[pair] * m * 256);
        const float s_c = p.pscore[pair];
        if (threadIdx.x == 0) { theta[0] = -INFINITY; cnt[0] = 0; }
        if (threadIdx.x < 4) flags[threadIdx.x] = 0;
        for (int t0 = u.row_begin; t0 < u.row_end; t0 += ADC_THREADS) {
            const int row = t0 + threadIdx.x;
            float v = s_c;
            for (int sl = 0; sl < nsl; sl++) {
                const int sb = sl * PQ_SLICE, ns = min(PQ_SLICE, m - sb);
                if (nsl > 1 || t0 == u.row_begin) {                // block-uniform
                    __syncthreads();                                // every lookup of the previous slice is done
                    float4* t4 = reinterpret_cast<float4*>(tab);
                    for (int e = threadIdx.x; e < ns * 64; e += ADC_THREADS) t4[e] = T[sb * 64 + e];
                    __syncthreads();
                }
                if (row < u.row_end) {
                    const uint4* cr = reinterpret_cast<const uint4*>(p.codes + (size_t)row * m + sb);
                    for (int g = 0; g < ns / 16; g++) {
                        const uint4 w = cr[g];
                        const uint32_t wd[4] = {w.x, w.y, w.z, w.w};
                        const float* tg = tab + g * 16 * 256;
                        #pragma unroll
                        for (int b = 0; b < 16; b++) v = __fadd_rn(v, tg[b * 256 + ((wd[b >> 2] >> (8 * (b & 3))) & 0xff)]);
                    }
                }
            }
            v = v != v ? -FLT_MAX : v;
            if (row < u.row_end && v >= theta[0]) knn_push(p, bufq, v, 0, row, cnt, flags);     // ties kept
            knn_compact<1>(p, sort_s, bufq, theta, cnt, flags);
        }
        knn_finish_ivf(p, sort_s, bufq, cnt, 1, pair, u.range);
    }
}

typedef CUresult (*EncodeTiledFnK)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [rows, dim] row-major 16-bit (elem_bytes 2) or int8 (1) elements, boxes of 128 bytes (64 or 128 columns) x box_rows rows,
// 128-byte swizzle, zero fill past both ends
bool make_rows_map(CUtensorMap* out, const void* base, int rows, int dim, int box_rows, int elem_bytes) {
    static EncodeTiledFnK enc = nullptr;
    if (!enc) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return false;
        enc = reinterpret_cast<EncodeTiledFnK>(f);
    }
    const cuuint64_t dims[2] = {(cuuint64_t)dim, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)dim * elem_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), (cuuint32_t)box_rows}, estr[2] = {1, 1};
    return enc(out, elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <KOp OP, int NT>
cudaError_t knn_launch(const KParams& p, unsigned grid, cudaStream_t st) {
    constexpr uint32_t smem = KnnGeo<OP, NT>::SMEM;
    cudaError_t e = cudaFuncSetAttribute(knn_kernel<OP, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    knn_kernel<OP, NT><<<grid, KNN_THREADS, smem, st>>>(p);
    return cudaGetLastError();
}
template <KOp OP>
cudaError_t knn_launch_nt(int nt, const KParams& p, unsigned grid, cudaStream_t st) {
    switch (nt) {
        case 1: return knn_launch<OP, 1>(p, grid, st);
        case 2: return knn_launch<OP, 2>(p, grid, st);
        case 4: return knn_launch<OP, 4>(p, grid, st);
        case 8: return knn_launch<OP, 8>(p, grid, st);
        default: return knn_launch<OP, 16>(p, grid, st);
    }
}

// Q8 quantiser: one warp per row.  Lane l holds the 16-column groups l, l + 32, l + 64 and l + 96 that exist (dim % 16 == 0,
// dim <= 2048), reduces max |x| exactly (fmaxf of magnitudes) and a finiteness flag over the warp, then writes its groups' codes
// with 16-byte stores.  The arithmetic is the rule of clip_b200_rows_to_int8 (clip_b200.h): IEEE division, rint, clamp.
__global__ void __launch_bounds__(256) quant_i8_kernel(const float* __restrict__ x, int n, int dim, int8_t* __restrict__ codes,
                                                       float* __restrict__ scales) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= n) return;
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * dim);
    const int ng = dim / 16;
    float4 v[16];
    float m = 0.f;
    bool fin = true;
    #pragma unroll
    for (int g = 0; g < 4; g++) {
        const int gi = lane + 32 * g;
        if (gi < ng) {
            #pragma unroll
            for (int u = 0; u < 4; u++) {
                const float4 a = xr[4 * gi + u];
                v[4 * g + u] = a;
                m = fmaxf(m, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))));
                fin &= isfinite(a.x) && isfinite(a.y) && isfinite(a.z) && isfinite(a.w);
            }
        }
    }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    fin = __all_sync(0xffffffffu, fin);
    float s = __fdiv_rn(m, 127.f);
    if (!fin) s = __int_as_float(0x7fc00000);                      // NaN: a non-finite row's every score is NaN
    const bool zero = !fin || s == 0.f;
    if (lane == 0) scales[row] = s;
    int4* cr = reinterpret_cast<int4*>(codes + (size_t)row * dim);
    #pragma unroll
    for (int g = 0; g < 4; g++) {
        const int gi = lane + 32 * g;
        if (gi >= ng) continue;
        uint32_t w[4];
        #pragma unroll
        for (int u = 0; u < 4; u++) {
            const float e[4] = {v[4 * g + u].x, v[4 * g + u].y, v[4 * g + u].z, v[4 * g + u].w};
            uint32_t packed = 0;
            #pragma unroll
            for (int b = 0; b < 4; b++) {
                const int c = zero ? 0 : min(127, max(-127, __float2int_rn(__fdiv_rn(e[b], s))));
                packed |= (uint32_t)(c & 0xff) << (8 * b);
            }
            w[u] = packed;
        }
        cr[gi] = make_int4((int)w[0], (int)w[1], (int)w[2], (int)w[3]);
    }
}

}  // namespace

void launch_similarity(const float* a, const float* b, float* s, int na, int nb, int d, size_t lds, cudaStream_t st) {
    if (na <= 0 || nb <= 0) return;
    dim3 grid((nb + ST - 1) / ST, (na + ST - 1) / ST);
    sim_kernel<<<grid, 256, 0, st>>>(a, b, s, na, nb, d, lds);
}

void launch_softmax_ref(float* logits, int rows, int cols, size_t ld, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return;
    softmax_ref_kernel<<<rows, 256, 0, st>>>(logits, rows, cols, ld);
}

int topk_slice() { return SL; }

void launch_topk_stage(const float* vals, const int* in_idx, size_t ld, int rows, int n, int idx_base, int kk, float* out_v, int* out_i,
                       size_t out_ld, int out_off, cudaStream_t st) {
    if (rows <= 0 || n <= 0) return;
    dim3 grid((n + SL - 1) / SL, rows);
    topk_stage_kernel<<<grid, 256, 0, st>>>(vals, in_idx, ld, n, idx_base, kk, out_v, out_i, out_ld, out_off);
}

KnnPlan knn_plan(int nq, int ndb, int kk, int sms) {
    KnnPlan pl;
    const int nqc = std::min(nq, 128);
    pl.nt = 1;
    while (8 * pl.nt < nqc) pl.nt <<= 1;
    const int qtiles = (nq + 8 * pl.nt - 1) / (8 * pl.nt);
    const int max_parts = (ndb + KB - 1) / KB;
    pl.parts = std::min(std::max(1, sms / qtiles), max_parts);
    pl.rows_per_part = ((ndb + pl.parts - 1) / pl.parts + KB - 1) / KB * KB;
    pl.parts = (ndb + pl.rows_per_part - 1) / pl.rows_per_part;
    pl.grid = qtiles * pl.parts;
    pl.cap = kk + 2 * KB;
    pl.buf_entries = (size_t)pl.grid * 8 * pl.nt * pl.cap;
    return pl;
}

cudaError_t launch_knn(KOp op, const void* q, const float* qs, int nq, const void* db, const float* xs, int ndb, int dim, int kk,
                       const KnnPlan& pl, void* buf, float* out_v, int* out_i, size_t out_ld, cudaStream_t st) {
    if (nq <= 0 || ndb <= 0) return cudaSuccess;
    const int eb = op == KOp::S8 ? 1 : 2;                          // element bytes; a chunk is 128 bytes of a row either way
    KParams p;
    memset(&p, 0, sizeof(p));
    if (!make_rows_map(&p.tm_db, db, ndb, dim, KB, eb) || !make_rows_map(&p.tm_q, q, nq, dim, 8 * pl.nt, eb)) return cudaErrorInvalidValue;
    p.buf = reinterpret_cast<Cand*>(buf);
    p.out_v = out_v; p.out_i = out_i; p.out_ld = out_ld;
    p.nq = nq; p.ndb = ndb;
    p.nchunks = (dim * eb + 127) / 128;
    p.rows_per_part = pl.rows_per_part; p.parts = pl.parts; p.kk = kk; p.cap = pl.cap;
    p.qs = qs; p.xs = xs;
    switch (op) {
        case KOp::F16: return knn_launch_nt<KOp::F16>(pl.nt, p, (unsigned)pl.grid, st);
        case KOp::BF16: return knn_launch_nt<KOp::BF16>(pl.nt, p, (unsigned)pl.grid, st);
        default: return knn_launch_nt<KOp::S8>(pl.nt, p, (unsigned)pl.grid, st);
    }
}

void launch_rows_to_int8(const float* x, int n, int dim, void* codes, float* scales, cudaStream_t st) {
    if (n <= 0) return;
    quant_i8_kernel<<<(n + 7) / 8, 256, 0, st>>>(x, n, dim, reinterpret_cast<int8_t*>(codes), scales);
}

KnnPlan knn_b1_plan(int nq, int ndb, int kk, int sms) {
    const KnnPlan pl = knn_plan(nq, ndb, kk, sms);
    return pl.nt < 8 ? knn_plan(nq, ndb, kk, 2 * sms) : pl;          // below 64-query tiles K11 runs two CTAs an SM
}

template <int NT>
static cudaError_t knn_b1_launch(const KParams& p, unsigned grid, cudaStream_t st) {
    const uint32_t smem = B1Geo<NT>::smem((p.dim / 128 + 3) / 4) + 16;
    cudaError_t e = cudaFuncSetAttribute(knn_b1_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    knn_b1_kernel<NT><<<grid, B1_THREADS, smem, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_knn_b1(const void* q, int nq, const void* db, int ndb, int dim, int kk, const KnnPlan& pl, void* buf, float* out_v,
                          int* out_i, size_t out_ld, cudaStream_t st) {
    if (nq <= 0 || ndb <= 0) return cudaSuccess;
    KParams p;
    memset(&p, 0, sizeof(p));
    p.qb = reinterpret_cast<const uint4*>(q); p.xb = reinterpret_cast<const uint4*>(db); p.dim = dim;
    p.buf = reinterpret_cast<Cand*>(buf);
    p.out_v = out_v; p.out_i = out_i; p.out_ld = out_ld;
    p.nq = nq; p.ndb = ndb;
    p.rows_per_part = pl.rows_per_part; p.parts = pl.parts; p.kk = kk; p.cap = pl.cap;
    switch (pl.nt) {
        case 1: return knn_b1_launch<1>(p, (unsigned)pl.grid, st);
        case 2: return knn_b1_launch<2>(p, (unsigned)pl.grid, st);
        case 4: return knn_b1_launch<4>(p, (unsigned)pl.grid, st);
        case 8: return knn_b1_launch<8>(p, (unsigned)pl.grid, st);
        default: return knn_b1_launch<16>(p, (unsigned)pl.grid, st);
    }
}

cudaError_t launch_rescore(int type, const void* q, int nq, const void* db, int ndb, int dim, const int* cand, int n_cand, int kk,
                           float* out_v, int* out_i, size_t out_ld, cudaStream_t st) {
    if (nq <= 0) return cudaSuccess;
    switch (type) {
        case 0: rescore_kernel<0><<<nq, 256, 0, st>>>(q, db, ndb, dim, cand, n_cand, kk, out_v, out_i, out_ld); break;
        case 1: rescore_kernel<1><<<nq, 256, 0, st>>>(q, db, ndb, dim, cand, n_cand, kk, out_v, out_i, out_ld); break;
        default: rescore_kernel<2><<<nq, 256, 0, st>>>(q, db, ndb, dim, cand, n_cand, kk, out_v, out_i, out_ld); break;
    }
    return cudaGetLastError();
}

void launch_rows_to_binary(const float* x, int n, int dim, const float* center, void* bits, cudaStream_t st) {
    if (n <= 0) return;
    const size_t nwords = (size_t)n * (dim / 128);
    const unsigned grid = (unsigned)std::min<size_t>((nwords + 7) / 8, (size_t)1 << 20);
    quant_b1_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const float4*>(x), nwords, dim / 128, reinterpret_cast<const float4*>(center),
                                          reinterpret_cast<uint4*>(bits));
}

cudaError_t launch_knn_ivf(bool bf, const void* pq, int npairs, const void* rows, int ndb, int dim, int kk, int nt, const IvfUnit* units,
                           int nunits, const size_t* slot, const int* ids, void* buf, float* out_v, int* out_i, cudaStream_t st) {
    if (nunits <= 0) return cudaSuccess;
    KParams p;
    memset(&p, 0, sizeof(p));
    if (!make_rows_map(&p.tm_db, rows, ndb, dim, KB, 2) || !make_rows_map(&p.tm_q, pq, npairs, dim, 8 * nt, 2)) return cudaErrorInvalidValue;
    p.buf = reinterpret_cast<Cand*>(buf);
    p.out_v = out_v; p.out_i = out_i;
    p.nq = npairs; p.ndb = ndb;
    p.nchunks = (dim * 2 + 127) / 128;
    p.kk = kk; p.cap = kk + 2 * KB;
    p.units = units; p.slot = slot; p.ids = ids;
    return bf ? knn_launch_nt<KOp::BF16_IVF>(nt, p, (unsigned)nunits, st) : knn_launch_nt<KOp::F16_IVF>(nt, p, (unsigned)nunits, st);
}

int knn_tile_rows() { return KB; }

void launch_gather_rows16(const void* src, const int* idx, size_t n, int dim, void* dst, cudaStream_t st) {
    if (n == 0) return;
    const int w16 = dim / 8;
    const unsigned grid = (unsigned)std::min<size_t>((n * w16 + 255) / 256, (size_t)1 << 20);
    gather_rows16_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(src), idx, n, w16, reinterpret_cast<uint4*>(dst));
}

void launch_fill_cand(float* v, int* i, size_t n, cudaStream_t st) {
    if (n == 0) return;
    fill_cand_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)1 << 16), 256, 0, st>>>(v, i, n);
}

void launch_ivf_update(bool bf, const void* x, int dim, const int* ids, const int2* chunks, int nchunks, const int* chunk_begin,
                       const int* offsets, int n_lists, double* part, void* cent, cudaStream_t st) {
    if (nchunks > 0) {
        if (bf) ivf_chunk_sum_kernel<true><<<nchunks, 256, 0, st>>>((const uint16_t*)x, dim, ids, chunks, part);
        else ivf_chunk_sum_kernel<false><<<nchunks, 256, 0, st>>>((const uint16_t*)x, dim, ids, chunks, part);
    }
    if (bf) ivf_update_kernel<true><<<n_lists, 256, 0, st>>>(part, chunk_begin, offsets, dim, (uint16_t*)cent);
    else ivf_update_kernel<false><<<n_lists, 256, 0, st>>>(part, chunk_begin, offsets, dim, (uint16_t*)cent);
}

template <class K>
static cudaError_t set_smem(K k, size_t smem) {
    return smem > 48 * 1024 ? cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) : cudaSuccess;
}

cudaError_t launch_pq_encode(bool bf, const void* x, size_t n, int dim, int m, const int* lists, const void* cent, const float* books,
                             void* codes, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const dim3 grid((unsigned)((n + PQ_ENC_THREADS - 1) / PQ_ENC_THREADS), (unsigned)m);
    const size_t smem = (size_t)(dim / m) * PQ_ENC_THREADS * 4;
    cudaError_t e = bf ? set_smem(pq_encode_kernel<true>, smem) : set_smem(pq_encode_kernel<false>, smem);
    if (e != cudaSuccess) return e;
    if (bf) pq_encode_kernel<true><<<grid, PQ_ENC_THREADS, smem, st>>>((const uint16_t*)x, n, dim, m, lists, (const uint16_t*)cent, books, (uint8_t*)codes);
    else pq_encode_kernel<false><<<grid, PQ_ENC_THREADS, smem, st>>>((const uint16_t*)x, n, dim, m, lists, (const uint16_t*)cent, books, (uint8_t*)codes);
    return cudaGetLastError();
}

void launch_pq_init(bool bf, const void* x, size_t n, int dim, int m, const int* lists, const void* cent, float* books, cudaStream_t st) {
    if (bf) pq_init_kernel<true><<<m, 256, 0, st>>>((const uint16_t*)x, n, dim, m, lists, (const uint16_t*)cent, books);
    else pq_init_kernel<false><<<m, 256, 0, st>>>((const uint16_t*)x, n, dim, m, lists, (const uint16_t*)cent, books);
}

void launch_pq_update(bool bf, const void* x, size_t n, int dim, int m, const int* lists, const void* cent, const int* ids,
                      const longlong2* chunks, int nchunks, const int* chunk_begin, const int* count, double* part, float* books,
                      cudaStream_t st) {
    if (nchunks > 0) {
        if (bf) pq_chunk_sum_kernel<true><<<nchunks, 128, 0, st>>>((const uint16_t*)x, n, dim, m, lists, (const uint16_t*)cent, ids, chunks, part);
        else pq_chunk_sum_kernel<false><<<nchunks, 128, 0, st>>>((const uint16_t*)x, n, dim, m, lists, (const uint16_t*)cent, ids, chunks, part);
    }
    pq_update_kernel<<<m * 256, 128, 0, st>>>(part, chunk_begin, count, dim / m, books);
}

cudaError_t launch_pq_tables(bool bf, const void* q, int nq, int dim, int m, const float* books, float* tables, cudaStream_t st) {
    if (nq <= 0) return cudaSuccess;
    const int dsub = dim / m;
    const size_t smem = ((size_t)256 * (dsub | 1) + (size_t)PQ_TQ * dsub) * 4;
    cudaError_t e = bf ? set_smem(pq_table_kernel<true>, smem) : set_smem(pq_table_kernel<false>, smem);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)m, (unsigned)((nq + PQ_TQ - 1) / PQ_TQ));
    if (bf) pq_table_kernel<true><<<grid, 256, smem, st>>>((const uint16_t*)q, nq, dim, m, books, tables);
    else pq_table_kernel<false><<<grid, 256, smem, st>>>((const uint16_t*)q, nq, dim, m, books, tables);
    return cudaGetLastError();
}

size_t adc_cap(int kk) { return (size_t)kk + KB + ADC_THREADS; }

cudaError_t launch_adc(const void* codes, int ndb, int m, const float* tables, const float* pscore, const int* pair_q, int kk,
                       const IvfUnit* units, int nunits, const size_t* slot, const int* ids, void* buf, float* out_v, int* out_i,
                       cudaStream_t st) {
    if (nunits <= 0) return cudaSuccess;
    KParams p;
    memset(&p, 0, sizeof(p));
    p.buf = reinterpret_cast<Cand*>(buf);
    p.out_v = out_v; p.out_i = out_i;
    p.ndb = ndb; p.kk = kk; p.cap = (int)adc_cap(kk);
    p.units = units; p.slot = slot; p.ids = ids;
    p.codes = reinterpret_cast<const uint8_t*>(codes); p.tables = tables; p.pscore = pscore; p.pair_q = pair_q; p.m = m;
    const size_t smem = 16 + KSORT * 8 + 64 + (size_t)std::min(m, PQ_SLICE) * 256 * 4;
    cudaError_t e = set_smem(adc_kernel, smem);
    if (e != cudaSuccess) return e;
    adc_kernel<<<(unsigned)nunits, ADC_THREADS, smem, st>>>(p);
    return cudaGetLastError();
}

}  // namespace cb
