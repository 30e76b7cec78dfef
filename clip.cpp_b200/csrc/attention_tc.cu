// attention_tc.cu -- K3 on Hopper tensor cores: S = Q K^T and O = P V as warpgroup MMAs (wgmma), online softmax in registers.
//
// Reference semantics: clip.cpp:1082-1108 (text, causal) / 1363-1388 (vision); soft_max ggml.c:12201-12270.
// One CTA per (128-query tile, head, sequence), 288 threads, 81 KB (head_dim 64) or 101 KB (head_dim 80) of shared memory:
//   warp 8      producer, one thread: TMA of the Q tile [128 x dh], then K and V blocks [128 keys x dh] into a two-deep ring, all
//               straight out of the fused QKV activation matrix through a 3-D view [sequence][token][column]: rows past a sequence's
//               T tokens arrive as zeros, so padded keys can never inject another sequence's (or stale) NaN / Inf into P.V
//   warps 0-7   two consumer warpgroups, 64 query rows each.  Per key block: S[64 x 128] = Q.K^T (wgmma m64n128k16, both operands
//               from shared memory), length / causal mask, online softmax (running row max and sum, quad shuffles), the probabilities
//               re-packed IN REGISTERS as 16-bit A fragments, O[64 x dh] += P.V (wgmma m64n64k16 per 16 keys, A from registers, V read
//               MN-major from the same [key][dh] tile).  O / l -> 16-bit stores.
// head_dim 80 (ViT-H/14): a 128-byte-swizzle box holds at most 64 sixteen-bit columns, and a wider box would reach into the next
// head (the tensor map's zero fill stops only at token and matrix ends, not at head boundaries).  So every Q / K / V tile arrives
// as two pieces from two tensor maps over the same buffer: columns 0-63 (128-byte swizzle) and 64-79 (32-byte swizzle).  S takes
// one extra k16 step on the tail pieces, O one extra m64n16k16 wgmma per 16 keys into 8 more accumulators per thread.
// HBM traffic: Q read once, K and V once per query tile, O written once.  Any T; a causal tile stops at its diagonal block.
#include <cuda.h>

#include "common.cuh"
#include "gemm.h"
#include "kernels.h"
#include "wgmma.cuh"

namespace cb {

namespace {

constexpr int AQ = 128, AK = 128;
constexpr int ATT_THREADS = 288;                       // 2 consumer warpgroups + 1 producer warp

// Shared-memory layout for one head_dim: every Q, K or V tile is [128 rows x 64 columns] (128-byte swizzle), followed for
// head_dim 80 by [128 rows x 16 columns] (32-byte swizzle).  Q tile, then two stages [K | V].
template <int DH>
struct AttnGeo {
    static_assert(DH == 64 || DH == 80, "head_dim 64 or 80");
    static constexpr bool TAIL = DH == 80;
    static constexpr uint32_t MAIN = AK * 128, TILE = MAIN + (TAIL ? AK * 32 : 0);
    static constexpr uint32_t KV_OFF = TILE;
    static constexpr uint32_t BAR_OFF = KV_OFF + 4 * TILE;
    static constexpr uint32_t SMEM = BAR_OFF + 64 + 1024;
    static_assert(AQ == AK && MAIN % 1024 == 0 && TILE % 1024 == 0, "tile alignment");
};

struct AParams {
    CUtensorMap tm_qkv;     // boxes of columns 0-63 of a head
    CUtensorMap tm_tail;    // head_dim 80: boxes of columns 64-79
    uint16_t* out;
    int T, H, ntile, causal;
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
template <bool BF, int DH>
__global__ void __launch_bounds__(ATT_THREADS, 1) attention_tc_kernel(const __grid_constant__ AParams p) {
    using G = AttnGeo<DH>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t q_full = smem_base + G::BAR_OFF, kv_full = q_full + 8, kv_empty = q_full + 24;     // kv rings: [0|1] = +8 bytes

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x % p.ntile, head = (blockIdx.x / p.ntile) % p.H, seq = blockIdx.x / (p.ntile * p.H);
    if (threadIdx.x == 0) {
        mbar_init(q_full, 1);
        for (int i = 0; i < 2; i++) { mbar_init(kv_full + 8 * i, 1); mbar_init(kv_empty + 8 * i, 8); }   // released by each consumer warp
        mbar_fence_init();
        tma_prefetch_desc(&p.tm_qkv);
        if constexpr (G::TAIL) tma_prefetch_desc(&p.tm_tail);
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();      // qkv is read (and the output written) only after the QKV GEMM grid has completed

    const int hid = p.H * DH, c = head * DH, q0 = qt * AQ;
    const int kend = p.causal ? min(p.T, q0 + AQ) : p.T;      // keys any row of this tile can see
    const int nkb = (kend + AK - 1) / AK;

    if (warp == 8) {
        // ------------------------------------------------------------------ producer (one thread)
        if (lane == 0) {
            mbar_arrive_expect_tx(q_full, G::TILE);
            tma_load_3d(smem_base, &p.tm_qkv, c, q0, seq, q_full);
            if constexpr (G::TAIL) tma_load_3d(smem_base + G::MAIN, &p.tm_tail, c + 64, q0, seq, q_full);
            for (int kb = 0; kb < nkb; kb++) {
                const uint32_t s = kb & 1, k_s = smem_base + G::KV_OFF + s * (2 * G::TILE);
                mbar_wait(kv_empty + 8 * s, ((kb >> 1) & 1) ^ 1);
                mbar_arrive_expect_tx(kv_full + 8 * s, 2 * G::TILE);
                tma_load_3d(k_s, &p.tm_qkv, hid + c, kb * AK, seq, kv_full + 8 * s);
                if constexpr (G::TAIL) tma_load_3d(k_s + G::MAIN, &p.tm_tail, hid + c + 64, kb * AK, seq, kv_full + 8 * s);
                tma_load_3d(k_s + G::TILE, &p.tm_qkv, 2 * hid + c, kb * AK, seq, kv_full + 8 * s);
                if constexpr (G::TAIL) tma_load_3d(k_s + G::TILE + G::MAIN, &p.tm_tail, 2 * hid + c + 64, kb * AK, seq, kv_full + 8 * s);
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumers (fragment layout: wgmma.cuh)
    const int wg = warp >> 2;
    const int wrow0 = q0 + wg * 64 + (warp & 3) * 16;          // first query row of this warp
    const int r0 = wrow0 + (lane >> 2), tc = 2 * (lane & 3);   // this thread: rows r0 and r0 + 8, columns 8j + tc + {0, 1}
    const bool live = q0 + wg * 64 < p.T;                      // warpgroup-uniform: T = 257 leaves one of the last tile's groups idle
    const float LOG2E = 1.4426950408889634f;
    // o: columns 0-63, ot: columns 64-79 (head_dim 80 only)
    float o[32], ot[8], m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    #pragma unroll
    for (int i = 0; i < 32; i++) o[i] = 0.f;
    #pragma unroll
    for (int i = 0; i < 8; i++) ot[i] = 0.f;
    mbar_wait(q_full, 0);
    const uint64_t dq = wgmma_desc_sw128(smem_base + (uint32_t)wg * 64u * 128u);
    const uint64_t dq_t = wgmma_desc_sw32(smem_base + G::MAIN + (uint32_t)wg * 64u * 32u);
    for (int kb = 0; kb < nkb; kb++) {
        const uint32_t s = kb & 1, k_s = smem_base + G::KV_OFF + s * (2 * G::TILE), v_s = k_s + G::TILE;
        mbar_wait(kv_full + 8 * s, (kb >> 1) & 1);
        if (live) {
            float sc[64];
            const uint64_t dk = wgmma_desc_sw128(k_s);
            wgmma_fence();
            #pragma unroll
            for (int k = 0; k < 4; k++) wgmma_ss_n128<BF>(sc, dq + 2 * k, dk + 2 * k, (uint32_t)k);
            if constexpr (G::TAIL) wgmma_ss_n128<BF>(sc, dq_t, wgmma_desc_sw32(k_s + G::MAIN), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(sc);
            const int key0 = kb * AK;
            // masking is only needed in the last (ragged) key block and, for the causal text tower, on the diagonal block
            if (key0 + AK > p.T || (p.causal && key0 + AK - 1 > wrow0)) {
                #pragma unroll
                for (int j = 0; j < AK / 8; j++) {
                    #pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const int key = key0 + 8 * j + tc + (e & 1), row = r0 + 8 * (e >> 1);
                        if (key >= p.T || (p.causal && key > row)) sc[4 * j + e] = -INFINITY;
                    }
                }
            }
            #pragma unroll
            for (int h = 0; h < 2; h++) {
                float mx = -INFINITY;
                #pragma unroll
                for (int j = 0; j < AK / 8; j++) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * h], sc[4 * j + 2 * h + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                // every row (padded rows past T included: zero queries) sees at least one unmasked key per visited block
                const float m_new = fmaxf(m_run[h], mx);
                const float alpha = ex2f((m_run[h] - m_new) * LOG2E), mb = m_new * LOG2E;
                float rs = 0.f;
                #pragma unroll
                for (int j = 0; j < AK / 8; j++) {
                    const float p0 = ex2f(sc[4 * j + 2 * h] * LOG2E - mb), p1 = ex2f(sc[4 * j + 2 * h + 1] * LOG2E - mb);
                    sc[4 * j + 2 * h] = p0; sc[4 * j + 2 * h + 1] = p1;
                    rs += p0 + p1;
                }
                l_run[h] = l_run[h] * alpha + rs;
                m_run[h] = m_new;
                #pragma unroll
                for (int j = 0; j < 8; j++) { o[4 * j + 2 * h] *= alpha; o[4 * j + 2 * h + 1] *= alpha; }
                if constexpr (G::TAIL) {
                    #pragma unroll
                    for (int j = 0; j < 2; j++) { ot[4 * j + 2 * h] *= alpha; ot[4 * j + 2 * h + 1] *= alpha; }
                }
            }
            // O += P.V: key step kk covers S n-tiles 2kk (A fragment registers 0, 1) and 2kk + 1 (registers 2, 3)
            wgmma_fence();
            #pragma unroll
            for (int kk = 0; kk < AK / 16; kk++) {
                const uint32_t a[4] = {pack2<BF>(sc[8 * kk], sc[8 * kk + 1]), pack2<BF>(sc[8 * kk + 2], sc[8 * kk + 3]),
                                       pack2<BF>(sc[8 * kk + 4], sc[8 * kk + 5]), pack2<BF>(sc[8 * kk + 6], sc[8 * kk + 7])};
                wgmma_rs_n64_bmn<BF>(o, a, wgmma_desc_sw128(v_s + (uint32_t)kk * 2048u), 1u);      // 16 keys = 2048 B of V
                if constexpr (G::TAIL) wgmma_rs_n16_bmn<BF>(ot, a, wgmma_desc_sw32(v_s + G::MAIN + (uint32_t)kk * 512u), 1u);   // 512 B
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(o);
            if constexpr (G::TAIL) wgmma_fence_regs(ot);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(kv_empty + 8 * s);
    }
    if (!live) return;
    #pragma unroll
    for (int h = 0; h < 2; h++) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.0f / l;
        const int row = r0 + 8 * h;
        if (row < p.T) {
            uint16_t* orow = p.out + ((size_t)seq * p.T + row) * hid + c;
            #pragma unroll
            for (int j = 0; j < 8; j++)
                *reinterpret_cast<uint32_t*>(orow + 8 * j + tc) = pack2<BF>(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
            if constexpr (G::TAIL) {
                #pragma unroll
                for (int j = 0; j < 2; j++)
                    *reinterpret_cast<uint32_t*>(orow + 64 + 8 * j + tc) = pack2<BF>(ot[4 * j + 2 * h] * inv, ot[4 * j + 2 * h + 1] * inv);
            }
        }
    }
}

typedef CUresult (*EncodeTiledFn3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [nseq][T][3*H*dh] view of the fused QKV activations, box = `box_cols` columns x 128 tokens x 1 sequence (zero fill past T):
// 64 columns with the 128-byte swizzle, or the 16-column tail of an 80-wide head with the 32-byte swizzle
bool make_qkv_map(CUtensorMap* out, const void* qkv16, int nseq, int T, int H, int dh, int box_cols, CUtensorMapSwizzle swz) {
    static EncodeTiledFn3 enc = nullptr;
    if (!enc) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return false;
        enc = reinterpret_cast<EncodeTiledFn3>(f);
    }
    const cuuint64_t cols = (cuuint64_t)3 * H * dh;
    const cuuint64_t dims[3] = {cols, (cuuint64_t)T, (cuuint64_t)nseq};
    const cuuint64_t strides[2] = {cols * 2, cols * 2 * (cuuint64_t)T};
    const cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)AK, 1}, estr[3] = {1, 1, 1};
    return enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, const_cast<void*>(qkv16), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int DH>
cudaError_t set_smem() {
    cudaError_t e = cudaFuncSetAttribute(attention_tc_kernel<true, DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AttnGeo<DH>::SMEM);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(attention_tc_kernel<false, DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AttnGeo<DH>::SMEM);
}

template <int DH>
cudaError_t launch_dh(const AParams& p, unsigned grid, int bf16, cudaStream_t st) {
    constexpr uint32_t smem = AttnGeo<DH>::SMEM;
    return bf16 ? launch_pdl(attention_tc_kernel<true, DH>, grid, (unsigned)ATT_THREADS, smem, st, 1, p)
                : launch_pdl(attention_tc_kernel<false, DH>, grid, (unsigned)ATT_THREADS, smem, st, 1, p);
}

}  // namespace

cudaError_t attention_tc_init() {
    cudaError_t e = set_smem<64>();
    return e != cudaSuccess ? e : set_smem<80>();
}

cudaError_t launch_attention_tc(const void* qkv16, void* out16, int nseq, int T, int H, int dh, int causal, int bf16, cudaStream_t st) {
    if (dh != 64 && dh != 80) return cudaErrorInvalidValue;
    if (nseq <= 0) return cudaSuccess;
    AParams p;
    memset(&p, 0, sizeof(p));
    if (!make_qkv_map(&p.tm_qkv, qkv16, nseq, T, H, dh, 64, CU_TENSOR_MAP_SWIZZLE_128B)) return cudaErrorInvalidValue;
    if (dh == 80 && !make_qkv_map(&p.tm_tail, qkv16, nseq, T, H, dh, 16, CU_TENSOR_MAP_SWIZZLE_32B)) return cudaErrorInvalidValue;
    p.out = (uint16_t*)out16; p.T = T; p.H = H; p.causal = causal;
    p.ntile = (T + AQ - 1) / AQ;
    const long long grid = (long long)nseq * H * p.ntile;
    if (grid > 0x7fffffffll) return cudaErrorInvalidValue;
    const cudaError_t e = dh == 80 ? launch_dh<80>(p, (unsigned)grid, bf16, st) : launch_dh<64>(p, (unsigned)grid, bf16, st);
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace cb
