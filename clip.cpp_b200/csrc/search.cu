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
};

template <KOp OP, int NT>
CB_DEVINL void knn_mma(float (&d)[4 * NT], uint64_t da, uint64_t db, uint32_t accumulate) {
    constexpr bool BF = OP == KOp::BF16;
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

template <KOp OP, int NT>
__global__ void __launch_bounds__(KNN_THREADS, 1) knn_kernel(const __grid_constant__ KParams p) {
    using G = KnnGeo<OP, NT>;
    constexpr int NQ = G::NQ;
    constexpr bool S8 = OP == KOp::S8;
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
    const int qt = blockIdx.x / p.parts, part = blockIdx.x - qt * p.parts;
    const int q0 = qt * NQ, nqv = min(NQ, p.nq - q0);
    const int row_begin = part * p.rows_per_part, row_end = min(p.ndb, row_begin + p.rows_per_part);
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
                if (q < nqv && row < row_end && v >= theta[q]) {
                    const int pos = atomicAdd(&cnt[q], 1);
                    *reinterpret_cast<float2*>(bufq + (size_t)q * p.cap + pos) = make_float2(v, __int_as_float(row));
                    if (pos == p.kk + KB) atomicOr(&flags[q >> 5], 1u << (q & 31));
                }
            }
        }
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
    for (int q = 0; q < nqv; q++) {
        const size_t o = (size_t)(q0 + q) * p.out_ld + (size_t)part * p.kk;
        knn_sort_keep(sort_s, bufq + (size_t)q * p.cap, cnt[q], p.kk, true, nullptr, nullptr, p.out_v + o, p.out_i + o);
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

}  // namespace cb
