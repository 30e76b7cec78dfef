// attention.cu -- K3: fused scaled-dot-product attention, one pass, nothing materialised in HBM.
//
// Reference semantics (clip.cpp:1082-1108 text / 1363-1388 vision): Q is pre-scaled by 1/sqrt(dh) after the bias add,
// KQ = K.Q, causal mask for the text tower (col > row -> -inf, ggml.c:12157-12161), row softmax (ggml.c:12201-12270),
// KQV = V.KQ, heads merged back to [T, hidden].  The reference materialises a [T, T] fp32 matrix per head; here each CTA
// streams 64-key blocks of K/V through shared memory (cp.async double buffer) with an online softmax and keeps the
// running output in registers, so HBM traffic is exactly one read of Q,K,V and one write of O.
//
// Layout: qkv is the fused QKV GEMM output [tokens, 3*hidden] (Q | K | V, 16-bit), out is [tokens, hidden].
// head_dim = 64 (true for ViT-B/32, B/16, L/14, L/14-336 and their text towers).
// Tensor-core path: warp-level mma.sync m16n8k16 (fp16 or bf16 inputs, fp32 accumulate).  Attention is ~4% of the
// model FLOPs (SURVEY.md section 8d); the production path is the wgmma kernel in attention_tc.cu, this one is its cross-check.
#include "common.cuh"
#include "kernels.h"

namespace cb {

namespace {

constexpr int DH = 64;
constexpr int TQ = 64;    // queries per CTA (4 warps x 16)
constexpr int TK = 64;    // keys per smem block

CB_DEVINL void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
CB_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
CB_DEVINL void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

CB_DEVINL void ldsm_x4(uint32_t addr, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr));
}
CB_DEVINL void ldsm_x4_t(uint32_t addr, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr));
}
template <bool BF>
CB_DEVINL void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if constexpr (BF)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <bool BF>
CB_DEVINL uint32_t pack2(float lo, float hi) {      // one F2FP: two fp32 -> packed 16-bit pair (lo in the low half)
    uint32_t r;
    if constexpr (BF) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
CB_DEVINL float ex2(float x) {                       // single MUFU.EX2 (exp2f() adds denormal range fix-ups we do not need)
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// [64 rows][64 x 16-bit] tile, 16-byte chunks XOR-swizzled by (row & 7): conflict-free for cp.async and ldmatrix
CB_DEVINL uint32_t tile_off(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

CB_DEVINL void load_tile(uint32_t smem_tile, const uint16_t* g, int ld, int row0, int T, int tid) {
    #pragma unroll
    for (int i = 0; i < 4; i++) {
        const int idx = tid + i * 128, row = idx >> 3, ch = idx & 7;
        const int gr = row0 + row;
        const bool ok = gr < T;
        cp_async16(smem_tile + tile_off(row, ch), g + (size_t)(ok ? gr : 0) * ld + ch * 8, ok ? 16u : 0u);   // 0 -> zero fill
    }
}

template <bool BF>
__global__ void __launch_bounds__(128) attention_kernel(const uint16_t* __restrict__ qkv, uint16_t* __restrict__ out, int T, int H,
                                                        int causal) {
    __shared__ __align__(128) uint8_t sQ[TQ * 128];
    __shared__ __align__(128) uint8_t sK[2][TK * 128];
    __shared__ __align__(128) uint8_t sV[2][TK * 128];

    const int qt = blockIdx.x, head = blockIdx.y, seq = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int hid = H * DH, ld = 3 * hid;
    const uint16_t* base = qkv + (size_t)seq * T * ld + head * DH;
    const uint32_t q_s = smem_u32(sQ), k_s[2] = {smem_u32(sK[0]), smem_u32(sK[1])}, v_s[2] = {smem_u32(sV[0]), smem_u32(sV[1])};

    const int nkb = causal ? (qt + 1) : (T + TK - 1) / TK;
    load_tile(q_s, base, ld, qt * TQ, T, tid);
    load_tile(k_s[0], base + hid, ld, 0, T, tid);
    load_tile(v_s[0], base + 2 * hid, ld, 0, T, tid);
    cp_async_commit();

    uint32_t qf[4][4];
    float o[8][4];
    #pragma unroll
    for (int i = 0; i < 8; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const float LOG2E = 1.4426950408889634f;
    const int qrow0 = qt * TQ + warp * 16 + g;     // rows qrow0 and qrow0 + 8
    const bool warp_active = (qt * TQ + warp * 16) < T;   // warp-uniform: T = 257 leaves 3 of 4 warps idle in the last query tile

    for (int kb = 0; kb < nkb; kb++) {
        const int buf = kb & 1;
        if (kb + 1 < nkb) {
            load_tile(k_s[buf ^ 1], base + hid, ld, (kb + 1) * TK, T, tid);
            load_tile(v_s[buf ^ 1], base + 2 * hid, ld, (kb + 1) * TK, T, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (kb == 0) {
            #pragma unroll
            for (int ks = 0; ks < 4; ks++)
                ldsm_x4(q_s + tile_off(warp * 16 + (lane & 15), ks * 2 + (lane >> 4)), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
        }
        if (warp_active) {
        // keys actually present in this block (T = 257: the 5th block holds ONE key) -> only the n-tile pairs / 16-key steps that
        // contain valid keys are computed; everything beyond is masked to -inf / multiplies p = 0 anyway
        const int kvalid = min(TK, T - kb * TK);
        const int np_lim = (kvalid + 15) >> 4;            // pairs of 8-key n-tiles == 16-key PV steps
        // ---- S = Q K^T (16 x 64 per warp)
        float s[8][4];
        #pragma unroll
        for (int i = 0; i < 8; i++) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
        #pragma unroll
        for (int ks = 0; ks < 4; ks++) {
            #pragma unroll
            for (int np = 0; np < 4; np++) {
                if (np >= np_lim) break;
                uint32_t b0, b1, b2, b3;
                const int id = lane >> 3, rr = lane & 7;
                ldsm_x4(k_s[buf] + tile_off((np * 2 + (id >> 1)) * 8 + rr, ks * 2 + (id & 1)), b0, b1, b2, b3);
                mma16816<BF>(s[2 * np], qf[ks], b0, b1);
                mma16816<BF>(s[2 * np + 1], qf[ks], b2, b3);
            }
        }
        // ---- mask + online softmax (rows g and g+8 of this warp's 16)
        const int key0 = kb * TK;
        // masking is only needed in the last (ragged) key block and, for the causal text tower, on the diagonal block
        if (key0 + TK > T || (causal && key0 + TK - 1 > qt * TQ + warp * 16)) {
            #pragma unroll
            for (int nt = 0; nt < 8; nt++) {
                #pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int key = key0 + nt * 8 + 2 * t4 + (e & 1);
                    const int qr = qrow0 + ((e >> 1) ? 8 : 0);
                    if (key >= T || (causal && key > qr)) s[nt][e] = -INFINITY;
                }
            }
        }
        #pragma unroll
        for (int r = 0; r < 2; r++) {
            float mx = -INFINITY;
            #pragma unroll
            for (int nt = 0; nt < 8; nt++) mx = fmaxf(mx, fmaxf(s[nt][2 * r], s[nt][2 * r + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_run[r], mx);
            // rows past T (zero Q) and every real row see at least one unmasked key per visited block, so m_new is finite
            const float alpha = ex2((m_run[r] - m_new) * LOG2E);
            const float mb = m_new * LOG2E;
            float rs = 0.f;
            #pragma unroll
            for (int nt = 0; nt < 8; nt++) {
                const float p0 = ex2(s[nt][2 * r] * LOG2E - mb), p1 = ex2(s[nt][2 * r + 1] * LOG2E - mb);
                s[nt][2 * r] = p0; s[nt][2 * r + 1] = p1;
                rs += p0 + p1;
            }
            l_run[r] = l_run[r] * alpha + rs;
            m_run[r] = m_new;
            #pragma unroll
            for (int nt = 0; nt < 8; nt++) { o[nt][2 * r] *= alpha; o[nt][2 * r + 1] *= alpha; }
        }
        // ---- O += P V
        #pragma unroll
        for (int ks = 0; ks < 4; ks++) {
            if (ks >= np_lim) break;
            uint32_t pa[4];
            pa[0] = pack2<BF>(s[2 * ks][0], s[2 * ks][1]);
            pa[1] = pack2<BF>(s[2 * ks][2], s[2 * ks][3]);
            pa[2] = pack2<BF>(s[2 * ks + 1][0], s[2 * ks + 1][1]);
            pa[3] = pack2<BF>(s[2 * ks + 1][2], s[2 * ks + 1][3]);
            #pragma unroll
            for (int np = 0; np < 4; np++) {
                uint32_t v0, v1, v2, v3;
                const int id = lane >> 3, rr = lane & 7;
                ldsm_x4_t(v_s[buf] + tile_off(ks * 16 + (id & 1) * 8 + rr, np * 2 + (id >> 1)), v0, v1, v2, v3);
                mma16816<BF>(o[2 * np], pa, v0, v1);
                mma16816<BF>(o[2 * np + 1], pa, v2, v3);
            }
        }
        }   // warp_active
        __syncthreads();
    }

    #pragma unroll
    for (int r = 0; r < 2; r++) {
        float l = l_run[r];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.0f / l;
        const int qr = qrow0 + r * 8;
        if (qr < T) {
            uint16_t* orow = out + ((size_t)seq * T + qr) * hid + head * DH;
            #pragma unroll
            for (int nt = 0; nt < 8; nt++)
                *reinterpret_cast<uint32_t*>(orow + nt * 8 + 2 * t4) = pack2<BF>(o[nt][2 * r] * inv, o[nt][2 * r + 1] * inv);
        }
    }
}

}  // namespace

void launch_attention(const void* qkv16, void* out16, int nseq, int T, int H, int causal, int bf16, cudaStream_t st) {
    if (nseq <= 0) return;
    // gridDim.z limit is 65535: chunk over sequences
    const int hid = H * DH;
    for (int s0 = 0; s0 < nseq; s0 += 65535) {
        const int ns = (nseq - s0) < 65535 ? (nseq - s0) : 65535;
        dim3 grid((T + TQ - 1) / TQ, H, ns);
        const uint16_t* q = (const uint16_t*)qkv16 + (size_t)s0 * T * 3 * hid;
        uint16_t* o = (uint16_t*)out16 + (size_t)s0 * T * hid;
        if (bf16) attention_kernel<true><<<grid, 128, 0, st>>>(q, o, T, H, causal);
        else attention_kernel<false><<<grid, 128, 0, st>>>(q, o, T, H, causal);
    }
}

}  // namespace cb
