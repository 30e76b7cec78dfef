// kernels.cu -- the memory-bound kernels around the GEMMs: LayerNorm (K2), im2col (K0a), embedding assembly (K4),
// L2-normalise (K5), per-token output rows (K7), position-table resample (K8), plus a scalar debug GEMM (scoring lives in search.cu).  All are HBM-bound streaming kernels: one warp per
// row, 128-bit coalesced loads, warp-shuffle reductions, no shared memory.
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace cb {

namespace {

CB_DEVINL float warp_sum(float v) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
CB_DEVINL float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
CB_DEVINL float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// Two-pass LayerNorm statistics over a row produced by `load(i4)` (i4 = float4 index), as the reference does:
// mean first, then the centred sum of squares (ggml.c:10822-10840).  The row is re-read (L1/L2 hits).
template <class Load>
CB_DEVINL void row_stats(Load load, int h4, int lane, float inv_h, float eps, float& mean, float& rstd) {
    float s = 0.f;
    for (int i = lane; i < h4; i += 32) { const float4 v = load(i); s += (v.x + v.y) + (v.z + v.w); }
    mean = warp_sum(s) * inv_h;
    float q = 0.f;
    for (int i = lane; i < h4; i += 32) {
        const float4 v = load(i);
        const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    rstd = rsqrtf(warp_sum(q) * inv_h + eps);
}

// K2 LayerNorm.  One warp per row, the row lives in registers (h <= 2048): one read of x, mean and CENTRED variance as the reference
// computes them (ggml.c:10822-10840), affine, 16-bit store.  The DELTA form (x_new = x + delta written back in fp32, delta = a 16-bit
// branch output) is an earlier deferred residual add; the out-proj / FC2 epilogues now add into x themselves and the model schedule
// always passes delta = NULL -- the form stays for callers of launch_layernorm that want it.
// MAXV = float4 per lane (row width h <= 128 * MAXV): specialised so a 1024-wide row costs 32 value registers, not 64 -- the kernel is
// latency-bound on its loads (ncu: long_scoreboard), so resident warps per SM are what buys HBM bandwidth.
template <bool BF, bool DELTA, int MAXV>
__global__ void __launch_bounds__(256) layernorm_kernel(float* __restrict__ x, size_t in_stride, int rows, int h, float eps,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        const uint16_t* __restrict__ delta, uint16_t* __restrict__ y, int descending) {
    // rows are walked from the LAST to the first: the GEMM before this kernel produced x in ascending token order, so its last rows are
    // the ones still in the 126 MB L2, and the GEMM after it starts with token tile 0, i.e. with the rows written here last
    const int lin = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    const int row = descending ? rows - 1 - lin : lin;
    pdl_trigger();
    pdl_wait();
    if (lin >= rows) return;
    float* xr = x + (size_t)row * in_stride;
    const uint16_t* dr = DELTA ? delta + (size_t)row * in_stride : nullptr;
    const int h4 = h >> 2;
    float4 v[MAXV];
    float s = 0.f;
    #pragma unroll
    for (int j = 0; j < MAXV; j++) {
        const int i = lane + 32 * j;
        if (i < h4) {
            v[j] = ld4(xr + 4 * i);
            if constexpr (DELTA) {
                const uint2 d = *reinterpret_cast<const uint2*>(dr + 4 * i);
                v[j].x += P2<BF>::to_float((uint16_t)(d.x & 0xffffu)); v[j].y += P2<BF>::to_float((uint16_t)(d.x >> 16));
                v[j].z += P2<BF>::to_float((uint16_t)(d.y & 0xffffu)); v[j].w += P2<BF>::to_float((uint16_t)(d.y >> 16));
                *reinterpret_cast<float4*>(xr + 4 * i) = v[j];
            }
            s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
        }
    }
    const float mean = warp_sum(s) / (float)h;
    float q = 0.f;
    #pragma unroll
    for (int j = 0; j < MAXV; j++) {
        if (lane + 32 * j < h4) {
            const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
            q += (a * a + b * b) + (c * c + d * d);
        }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)h + eps);
    uint16_t* yr = y + (size_t)row * h;
    #pragma unroll
    for (int j = 0; j < MAXV; j++) {
        const int i = lane + 32 * j;
        if (i < h4) {
            const float4 g = ld4(gamma + 4 * i), b = ld4(beta + 4 * i);
            const float o0 = (v[j].x - mean) * rstd * g.x + b.x, o1 = (v[j].y - mean) * rstd * g.y + b.y;
            const float o2 = (v[j].z - mean) * rstd * g.z + b.z, o3 = (v[j].w - mean) * rstd * g.w + b.w;
            uint2 pk;
            pk.x = (uint32_t)P2<BF>::from_float(o0) | ((uint32_t)P2<BF>::from_float(o1) << 16);
            pk.y = (uint32_t)P2<BF>::from_float(o2) | ((uint32_t)P2<BF>::from_float(o3) << 16);
            *reinterpret_cast<uint2*>(yr + 4 * i) = pk;
        }
    }
}

// Token rows (K7): out[r, :] = the r-th requested row of x, optionally through post_ln, as the caller's type.  Output row r of item
// i = r / rows_out takes x row i * T + skip + r % rows_out (skip = 1 drops the CLS row), rows in_stride floats apart.  With LN the
// arithmetic is K2's, expression for expression (per-lane sums, warp_sum, rsqrtf, (v - mean) * rstd * g + b in fp32), so the 16-bit
// output of the operand type equals layernorm_kernel's bit for bit.  OT: 0 fp32, 1 fp16, 2 bf16, each rounded to nearest even.
template <int OT, bool LN, int MAXV>
__global__ void __launch_bounds__(256) token_rows_kernel(const float* __restrict__ x, size_t in_stride, int rows, int rows_out, int T,
                                                         int skip, int h, float eps, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, void* __restrict__ out) {
    // last row first, as K2: the GEMM before this kernel wrote x in ascending token order, so its last rows are still in L2
    const int lin = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (lin >= rows) return;
    const int r = rows - 1 - lin;
    const float* xr = x + ((size_t)(r / rows_out) * T + skip + r % rows_out) * in_stride;
    const int h4 = h >> 2;
    float4 v[MAXV];
    float s = 0.f;
    #pragma unroll
    for (int j = 0; j < MAXV; j++) {
        const int i = lane + 32 * j;
        if (i < h4) {
            v[j] = ld4(xr + 4 * i);
            s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
        }
    }
    float mean = 0.f, rstd = 1.f;
    if constexpr (LN) {
        mean = warp_sum(s) / (float)h;
        float q = 0.f;
        #pragma unroll
        for (int j = 0; j < MAXV; j++) {
            if (lane + 32 * j < h4) {
                const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
                q += (a * a + b * b) + (c * c + d * d);
            }
        }
        rstd = rsqrtf(warp_sum(q) / (float)h + eps);
    }
    #pragma unroll
    for (int j = 0; j < MAXV; j++) {
        const int i = lane + 32 * j;
        if (i < h4) {
            float4 o = v[j];
            if constexpr (LN) {
                const float4 g = ld4(gamma + 4 * i), b = ld4(beta + 4 * i);
                o.x = (v[j].x - mean) * rstd * g.x + b.x; o.y = (v[j].y - mean) * rstd * g.y + b.y;
                o.z = (v[j].z - mean) * rstd * g.z + b.z; o.w = (v[j].w - mean) * rstd * g.w + b.w;
            }
            const size_t e = (size_t)r * h + 4 * i;
            if constexpr (OT == 0) {
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + e) = o;
            } else {
                using C = P2<OT == 2>;
                uint2 pk;
                pk.x = (uint32_t)C::from_float(o.x) | ((uint32_t)C::from_float(o.y) << 16);
                pk.y = (uint32_t)C::from_float(o.z) | ((uint32_t)C::from_float(o.w) << 16);
                *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(out) + e) = pk;
            }
        }
    }
}

__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ px, int B, int H, int W, int P, int kpad,
                                                     __half* __restrict__ out) {
    const int gh = H / P, gw = W / P, np = gh * gw, K = 3 * P * P;
    const size_t total = (size_t)B * np * kpad;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(idx % kpad);
        const size_t rowi = idx / kpad;
        float v = 0.f;
        if (k < K) {
            const int p = (int)(rowi % np), b = (int)(rowi / np);
            const int py = p / gw, pxx = p % gw;
            const int c = k / (P * P), rem = k % (P * P), ky = rem / P, kx = rem % P;
            v = px[(((size_t)b * H + (py * P + ky)) * W + (pxx * P + kx)) * 3 + c];
        }
        out[idx] = __float2half_rn(v);
    }
}

// K8 bicubic weights (torch's upsample_bicubic2d, A = -0.75) of the output index o on an axis of g -> go, in fp64 with every
// operation rounded on its own (no contraction), so that a numpy restatement reproduces them bit for bit.
CB_DEVINL void cubic_taps(int o, int g, int go, int idx[4], double w[4]) {
    const double src = __dadd_rn(__dmul_rn(__ddiv_rn((double)g, (double)go), __dadd_rn((double)o, 0.5)), -0.5);   // not clamped
    const double fi = floor(src), t = __dadd_rn(src, -fi), s = __dadd_rn(1.0, -t);
    // cc1(x) = ((A+2) x - (A+3)) x x + 1,  cc2(x) = ((A x - 5A) x + 8A) x - 4A
    auto cc1 = [](double x) { return __dadd_rn(__dmul_rn(__dmul_rn(__dadd_rn(__dmul_rn(1.25, x), -2.25), x), x), 1.0); };
    auto cc2 = [](double x) { return __dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(-0.75, x), 3.75), x), -6.0), x), 3.0); };
    w[0] = cc2(__dadd_rn(t, 1.0)); w[1] = cc1(t); w[2] = cc1(s); w[3] = cc2(__dadd_rn(s, 1.0));
    const int i = (int)fi;
    #pragma unroll
    for (int k = 0; k < 4; k++) idx[k] = min(max(i - 1 + k, 0), g - 1);
}

// K8 position-table resample: out[(oy*gw + ox), c] from table [g*g, h] (row-major grid y, then x).  One thread per output element,
// c fastest, so a warp reads and writes consecutive columns; each output reads 16 table elements (L1 / L2 hits: the table is at
// most a few MB) and is written once.  Horizontal pass first per source row, then the vertical one, each a left-to-right sum.
__global__ void __launch_bounds__(256) pos_resample_kernel(const float* __restrict__ table, int g, int h, int gh, int gw,
                                                           float* __restrict__ out) {
    const size_t total = (size_t)gh * gw * h;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(e % h), o = (int)(e / h), oy = o / gw, ox = o % gw;
        int iy[4], ix[4];
        double wy[4], wx[4];
        cubic_taps(oy, g, gh, iy, wy);
        cubic_taps(ox, g, gw, ix, wx);
        double acc = 0.0;
        #pragma unroll
        for (int j = 0; j < 4; j++) {
            const float* r = table + (size_t)iy[j] * g * h + c;
            double row = __dmul_rn((double)r[(size_t)ix[0] * h], wx[0]);
            row = __dadd_rn(row, __dmul_rn((double)r[(size_t)ix[1] * h], wx[1]));
            row = __dadd_rn(row, __dmul_rn((double)r[(size_t)ix[2] * h], wx[2]));
            row = __dadd_rn(row, __dmul_rn((double)r[(size_t)ix[3] * h], wx[3]));
            acc = j == 0 ? __dmul_rn(row, wy[0]) : __dadd_rn(acc, __dmul_rn(row, wy[j]));
        }
        out[e] = __double2float_rn(acc);
    }
}

// One row of K4v for the mixed-size kernel: xr = LN(src + pr) * gamma + beta, one warp, expression for expression
// assemble_preln_kernel's (which keeps its own copy, so that its code is unchanged)
CB_DEVINL void assemble_row(const float* __restrict__ src, const float* __restrict__ pr, int h, float eps, const float* __restrict__ gamma,
                            const float* __restrict__ beta, float* __restrict__ xr, int lane) {
    const int h4 = h >> 2;
    auto load = [&](int i) { return add4(ld4(src + 4 * i), ld4(pr + 4 * i)); };
    float mean, rstd;
    row_stats(load, h4, lane, 1.0f / (float)h, eps, mean, rstd);
    for (int i = lane; i < h4; i += 32) {
        const float4 v = load(i), g = ld4(gamma + 4 * i), bb = ld4(beta + 4 * i);
        float4 o;
        o.x = (v.x - mean) * rstd * g.x + bb.x; o.y = (v.y - mean) * rstd * g.y + bb.y;
        o.z = (v.z - mean) * rstd * g.z + bb.z; o.w = (v.w - mean) * rstd * g.w + bb.w;
        *reinterpret_cast<float4*>(xr + 4 * i) = o;
    }
}

__global__ void __launch_bounds__(256) assemble_preln_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                                             const float* __restrict__ pos, int B, int T, int h, float eps,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float* __restrict__ x) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= B * T) return;
    const int b = row / T, t = row % T;
    const float* src = (t == 0) ? cls : patch + ((size_t)b * (T - 1) + (t - 1)) * h;
    const float* pr = pos + (size_t)t * h;
    const int h4 = h >> 2;
    auto load = [&](int i) { return add4(ld4(src + 4 * i), ld4(pr + 4 * i)); };
    float mean, rstd;
    row_stats(load, h4, lane, 1.0f / (float)h, eps, mean, rstd);
    float* xr = x + (size_t)row * h;
    for (int i = lane; i < h4; i += 32) {
        const float4 v = load(i), g = ld4(gamma + 4 * i), bb = ld4(beta + 4 * i);
        float4 o;
        o.x = (v.x - mean) * rstd * g.x + bb.x; o.y = (v.y - mean) * rstd * g.y + bb.y;
        o.z = (v.z - mean) * rstd * g.z + bb.z; o.w = (v.w - mean) * rstd * g.w + bb.w;
        *reinterpret_cast<float4*>(xr + 4 * i) = o;
    }
}

// The image of a mixed-size pass that holds row `r` of the counter `field` (row or prow): images are in row order, so a binary
// search of their first rows
CB_DEVINL int image_of(const MixedImage* __restrict__ im, int n, int r, int MixedImage::*field) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (im[mid].*field <= r) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// K0a over the images of a mixed-size pass: patch row r of image i (r counted from the pass's first patch row) from its own grid,
// element for element what im2col_kernel writes for that image alone.  One block per patch row at a time.
__global__ void __launch_bounds__(256) im2col_mixed_kernel(const float* __restrict__ px, const MixedImage* __restrict__ im, int n, int prows,
                                                           int P, int kpad, __half* __restrict__ out) {
    const int K = 3 * P * P;
    for (int rowi = blockIdx.x; rowi < prows; rowi += gridDim.x) {
        const MixedImage d = im[image_of(im, n, rowi, &MixedImage::prow)];
        const int p = rowi - d.prow, py = p / d.gw, pxx = p % d.gw, W = d.gw * P;
        const float* img = px + d.px;
        for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
            float v = 0.f;
            if (k < K) {
                const int c = k / (P * P), rem = k % (P * P), ky = rem / P, kx = rem % P;
                v = img[((size_t)(py * P + ky) * W + (pxx * P + kx)) * 3 + c];
            }
            out[(size_t)rowi * kpad + k] = __float2half_rn(v);
        }
    }
}

// K4v over the images of a mixed-size pass: token row `row` is row t of image i, with i's position table; assemble_row as
// assemble_preln_kernel runs it
__global__ void __launch_bounds__(256) assemble_mixed_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                                             const MixedImage* __restrict__ im, int n, int rows, int h, float eps,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float* __restrict__ x) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const MixedImage d = im[image_of(im, n, row, &MixedImage::row)];
    const int t = row - d.row;
    const float* src = (t == 0) ? cls : patch + ((size_t)d.prow + (t - 1)) * h;
    assemble_row(src, d.pos + (size_t)t * h, h, eps, gamma, beta, x + (size_t)row * h, lane);
}

__global__ void __launch_bounds__(256) text_embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ tok,
                                                         const float* __restrict__ pos, int nseq, int T, int h, int n_vocab,
                                                         float* __restrict__ x) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= nseq * T) return;
    int id = ids[row];
    id = id < 0 ? 0 : (id >= n_vocab ? n_vocab - 1 : id);
    const float* tr = tok + (size_t)id * h;
    const float* pr = pos + (size_t)(row % T) * h;
    float* xr = x + (size_t)row * h;
    for (int i = lane; i < (h >> 2); i += 32) *reinterpret_cast<float4*>(xr + 4 * i) = add4(ld4(pr + 4 * i), ld4(tr + 4 * i));
}

// text_embed_kernel over the sequences of a packed pass: row `row` is token row - off[s] of sequence s (off in row order, so a binary
// search of the first rows), with text_embed_kernel's clamp and sum
__global__ void __launch_bounds__(256) text_embed_packed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ tok,
                                                                const float* __restrict__ pos, const int* __restrict__ off, int nseq,
                                                                int rows, int h, int n_vocab, float* __restrict__ x) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    int lo = 0, hi = nseq - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= row) lo = mid;
        else hi = mid - 1;
    }
    int id = ids[row];
    id = id < 0 ? 0 : (id >= n_vocab ? n_vocab - 1 : id);
    const float* tr = tok + (size_t)id * h;
    const float* pr = pos + (size_t)(row - off[lo]) * h;
    float* xr = x + (size_t)row * h;
    for (int i = lane; i < (h >> 2); i += 32) *reinterpret_cast<float4*>(xr + 4 * i) = add4(ld4(pr + 4 * i), ld4(tr + 4 * i));
}

__global__ void __launch_bounds__(256) l2norm_kernel(const float* __restrict__ v, float* __restrict__ out, int rows, int d,
                                                     int normalize) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* vr = v + (size_t)row * d;
    float s = 0.f;
    for (int i = lane; i < d; i += 32) s += vr[i] * vr[i];
    s = warp_sum(s);
    const float inv = normalize ? 1.0f / sqrtf(s) : 1.0f;     // no epsilon, as the reference (clip.cpp:1164-1165)
    for (int i = lane; i < d; i += 32) out[(size_t)row * d + i] = vr[i] * inv;
}

template <bool BF>
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int h,
                                                          int stride_rows, const int32_t* __restrict__ offs,
                                                          const uint16_t* __restrict__ delta) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const size_t r = (size_t)row * stride_rows + (offs ? offs[row] : 0);
    const float* s = src + r * h;
    for (int i = lane; i < (h >> 2); i += 32) {
        float4 v = ld4(s + 4 * i);
        if (delta) {
            const uint2 d = *reinterpret_cast<const uint2*>(delta + r * h + 4 * i);
            v.x += P2<BF>::to_float((uint16_t)(d.x & 0xffffu)); v.y += P2<BF>::to_float((uint16_t)(d.x >> 16));
            v.z += P2<BF>::to_float((uint16_t)(d.y & 0xffffu)); v.w += P2<BF>::to_float((uint16_t)(d.y >> 16));
        }
        *reinterpret_cast<float4*>(dst + (size_t)row * h + 4 * i) = v;
    }
}

__global__ void fill_last_kernel(const int32_t* __restrict__ lens, int32_t* __restrict__ last, int n, int seq_len) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int v = lens ? lens[i] : seq_len;
    v = v < 1 ? 1 : (v > seq_len ? seq_len : v);
    last[i] = v - 1;
}

// ---- debug scalar GEMM from raw ggml rows -----------------------------------------------------------
CB_DEVINL float dq_elem(int qt, const uint8_t* row, int k) {
    if (qt == QT_F16) return __half2float(reinterpret_cast<const __half*>(row)[k]);
    const int bi = k >> 5, e = k & 31, j = e & 15, hi = e >> 4;
    const int bs = qt == 2 ? 18 : qt == 3 ? 20 : qt == 6 ? 22 : qt == 7 ? 24 : 34;
    const uint8_t* b = row + (size_t)bi * bs;
    const float d = __half2float(*reinterpret_cast<const __half*>(b));
    if (qt == 8) return (float)reinterpret_cast<const int8_t*>(b + 2)[e] * d;
    float m = 0.f;
    const uint8_t* qs;
    uint32_t qh = 0;
    if (qt == 2) qs = b + 2;
    else if (qt == 3) { m = __half2float(*reinterpret_cast<const __half*>(b + 2)); qs = b + 4; }
    else if (qt == 6) { qh = b[2] | (b[3] << 8) | (b[4] << 16) | ((uint32_t)b[5] << 24); qs = b + 6; }
    else { m = __half2float(*reinterpret_cast<const __half*>(b + 2)); qh = b[4] | (b[5] << 8) | (b[6] << 16) | ((uint32_t)b[7] << 24); qs = b + 8; }
    int q = hi ? (qs[j] >> 4) : (qs[j] & 0x0F);
    if (qt == 6 || qt == 7) q |= ((qh >> (j + 16 * hi)) & 1) << 4;
    if (qt == 2) q -= 8;
    if (qt == 6) q -= 16;
    return (float)q * d + m;
}

__global__ void naive_gemm_kernel(const uint16_t* __restrict__ x, int x_bf16, const uint8_t* __restrict__ w, int qt,
                                  const float* __restrict__ bias, void* __restrict__ out, int M, int N, int K, int ldo, int epi,
                                  int out_bf16, int scale_cols, float scale) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
    if (n >= N || m >= M) return;
    const size_t rb = qt == QT_F16 ? (size_t)K * 2 : (size_t)(K / 32) * (qt == 2 ? 18 : qt == 3 ? 20 : qt == 6 ? 22 : qt == 7 ? 24 : 34);
    const uint8_t* wr = w + (size_t)n * rb;
    float acc = 0.f;
    for (int k = 0; k < K; k++) {
        const float xv = x_bf16 ? __bfloat162float(__ushort_as_bfloat16(x[(size_t)m * K + k])) : __half2float(__ushort_as_half(x[(size_t)m * K + k]));
        float wv = dq_elem(qt, wr, k);
        wv = x_bf16 ? __bfloat162float(__float2bfloat16_rn(wv)) : __half2float(__float2half_rn(wv));
        acc += xv * wv;
    }
    float v = acc + (bias ? bias[n] : 0.f);
    const size_t o = (size_t)m * ldo + n;
    if (epi == EPI_REDADD32) reinterpret_cast<float*>(out)[o] += v;
    else if (epi == EPI_STORE32) reinterpret_cast<float*>(out)[o] = v;
    else {
        if (epi == EPI_GELU16) v = gelu_tanh(v);
        else if (epi == EPI_QGELU16) v = gelu_quick(v);
        else if (n < scale_cols) v *= scale;
        reinterpret_cast<uint16_t*>(out)[o] = out_bf16 ? P2<true>::from_float(v) : P2<false>::from_float(v);
    }
}

inline int rows_grid(int rows, int warps_per_block) { return (rows + warps_per_block - 1) / warps_per_block; }

}  // namespace

void launch_layernorm(float* x, size_t in_stride, int rows, int h, float eps, const float* gamma, const float* beta,
                      const void* delta16, void* y16, int bf16, cudaStream_t st) {
    if (rows <= 0) return;
    const int grid = rows_grid(rows, 8);
    const uint16_t* d = (const uint16_t*)delta16;
    uint16_t* y = (uint16_t*)y16;
    static const int desc = !(getenv("CLIP_B200_ORDER") && !strcmp(getenv("CLIP_B200_ORDER"), "asc"));      // A/B switch for measurements
#define CB_LN(BFV, DV, MV) (void)launch_pdl(layernorm_kernel<BFV, DV, MV>, (unsigned)grid, 256u, 0, st, 1, x, in_stride, rows, h, eps, gamma, beta, d, y, desc)
#define CB_LN_W(BFV, DV) do { if (h <= 512) CB_LN(BFV, DV, 4); else if (h <= 1024) CB_LN(BFV, DV, 8); else CB_LN(BFV, DV, 16); } while (0)
    if (bf16) { if (d) CB_LN_W(true, true); else CB_LN_W(true, false); }
    else      { if (d) CB_LN_W(false, true); else CB_LN_W(false, false); }
#undef CB_LN_W
#undef CB_LN
}

void launch_token_rows(const float* x, size_t in_stride, int n, int T, int skip, int h, const float* gamma, const float* beta, float eps,
                       int out_type, void* out, cudaStream_t st) {
    const int rows_out = T - skip, rows = n * rows_out;
    if (rows <= 0) return;
    const int grid = rows_grid(rows, 8);
#define CB_TR(OT, LN, MV) token_rows_kernel<OT, LN, MV><<<grid, 256, 0, st>>>(x, in_stride, rows, rows_out, T, skip, h, eps, gamma, beta, out)
#define CB_TR_W(OT, LN) do { if (h <= 512) CB_TR(OT, LN, 4); else if (h <= 1024) CB_TR(OT, LN, 8); else CB_TR(OT, LN, 16); } while (0)
#define CB_TR_T(LN) do { if (out_type == 0) CB_TR_W(0, LN); else if (out_type == 1) CB_TR_W(1, LN); else CB_TR_W(2, LN); } while (0)
    if (gamma) CB_TR_T(true);
    else CB_TR_T(false);
#undef CB_TR_T
#undef CB_TR_W
#undef CB_TR
}

void launch_im2col(const float* pixels, int B, int H, int W, int P, int kpad, void* patches16, cudaStream_t st) {
    const size_t total = (size_t)B * (H / P) * (W / P) * kpad;
    if (!total) return;
    size_t blocks = (total + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;      // grid-stride loop: 32 blocks per H100 SM
    im2col_kernel<<<(int)blocks, 256, 0, st>>>(pixels, B, H, W, P, kpad, (__half*)patches16);
}

void launch_pos_resample(const float* table, int g, int h, int gh, int gw, float* out, cudaStream_t st) {
    const size_t total = (size_t)gh * gw * h;
    if (!total) return;
    size_t blocks = (total + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    pos_resample_kernel<<<(int)blocks, 256, 0, st>>>(table, g, h, gh, gw, out);
}

void launch_assemble_preln(const float* patch, const float* class_embd, const float* pos, int B, int T, int h, float eps,
                           const float* gamma, const float* beta, float* x, cudaStream_t st) {
    if (B * T <= 0) return;
    assemble_preln_kernel<<<rows_grid(B * T, 8), 256, 0, st>>>(patch, class_embd, pos, B, T, h, eps, gamma, beta, x);
}

void launch_im2col_mixed(const float* pixels, const MixedImage* im, int n, int prows, int P, int kpad, void* patches16, cudaStream_t st) {
    if (n <= 0 || prows <= 0) return;
    im2col_mixed_kernel<<<std::min(prows, 132 * 16), 256, 0, st>>>(pixels, im, n, prows, P, kpad, (__half*)patches16);
}

void launch_assemble_mixed(const float* patch, const float* class_embd, const MixedImage* im, int n, int rows, int h, float eps,
                           const float* gamma, const float* beta, float* x, cudaStream_t st) {
    if (n <= 0 || rows <= 0) return;
    assemble_mixed_kernel<<<rows_grid(rows, 8), 256, 0, st>>>(patch, class_embd, im, n, rows, h, eps, gamma, beta, x);
}

void launch_text_embed(const int32_t* ids, const float* tok, const float* pos, int nseq, int T, int h, int n_vocab, float* x,
                       cudaStream_t st) {
    if (nseq * T <= 0) return;
    text_embed_kernel<<<rows_grid(nseq * T, 8), 256, 0, st>>>(ids, tok, pos, nseq, T, h, n_vocab, x);
}

void launch_text_embed_packed(const int32_t* ids, const float* tok, const float* pos, const int* off, int nseq, int rows, int h, int n_vocab,
                              float* x, cudaStream_t st) {
    if (nseq <= 0 || rows <= 0) return;
    text_embed_packed_kernel<<<rows_grid(rows, 8), 256, 0, st>>>(ids, tok, pos, off, nseq, rows, h, n_vocab, x);
}

void launch_l2norm(const float* v, float* out, int rows, int d, int normalize, cudaStream_t st) {
    if (rows <= 0) return;
    l2norm_kernel<<<rows_grid(rows, 8), 256, 0, st>>>(v, out, rows, d, normalize);
}

void launch_gather_rows(const float* src, float* dst, int rows, int h, int stride_rows, const int32_t* offs, const void* delta16,
                        int bf16, cudaStream_t st) {
    if (rows <= 0) return;
    if (bf16) gather_rows_kernel<true><<<rows_grid(rows, 8), 256, 0, st>>>(src, dst, rows, h, stride_rows, offs, (const uint16_t*)delta16);
    else gather_rows_kernel<false><<<rows_grid(rows, 8), 256, 0, st>>>(src, dst, rows, h, stride_rows, offs, (const uint16_t*)delta16);
}

void launch_fill_last(const int32_t* lens, int32_t* last, int n, int seq_len, cudaStream_t st) {
    if (n <= 0) return;
    fill_last_kernel<<<(n + 255) / 256, 256, 0, st>>>(lens, last, n, seq_len);
}

void launch_naive_gemm(const void* x16, int x_bf16, const void* w_ggml, int qtype, const float* bias, void* out, int M, int N,
                       int K, int ldo, int epi, int out_bf16, int scale_cols, float scale, cudaStream_t st) {
    if (M <= 0) return;
    dim3 grid((N + 127) / 128, M);
    naive_gemm_kernel<<<grid, 128, 0, st>>>((const uint16_t*)x16, x_bf16, (const uint8_t*)w_ggml, qtype, bias, out, M, N, K, ldo,
                                            epi, out_bf16, scale_cols, scale);
}

}  // namespace cb
