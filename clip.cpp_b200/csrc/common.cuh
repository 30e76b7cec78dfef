// common.cuh -- sm_90a PTX building blocks shared by the kernels of libclip_b200.so.
//
// Everything here is hand-written inline PTX for Hopper (TMA / mbarrier / programmatic dependent launch; the warpgroup MMA wrappers are
// in wgmma.cuh); there is no CUTLASS/CuTe dependency.
#pragma once
#include <cstdlib>

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cb {

// --------------------------------------------------------------------------------------------------
// weight storage types == ggml type ids used by clip.cpp model files (reference: ggml.h enum ggml_type,
// accepted file types clip.cpp:117-143)
// --------------------------------------------------------------------------------------------------
enum QType : int { QT_F32 = 0, QT_F16 = 1, QT_Q4_0 = 2, QT_Q4_1 = 3, QT_Q5_0 = 6, QT_Q5_1 = 7, QT_Q8_0 = 8 };

// epilogue selectors of the fused-dequant GEMM
enum Epi : int {
    EPI_STORE16 = 0,      // out16 = (acc + bias) [* scale for the first scale_cols features]
    EPI_GELU16 = 1,       // out16 = gelu_tanh(acc + bias)          (clip.use_gelu = true)
    EPI_QGELU16 = 2,      // out16 = quick_gelu(acc + bias)         (clip.use_gelu = false)
    EPI_REDADD32 = 3,     // x32 += acc + bias  (fp32 residual stream; every element has exactly one owner thread)
    EPI_STORE32 = 4,      // out32 = acc + bias
};

#define CB_DEVINL __device__ __forceinline__

// --------------------------------------------------------------------------------------------------
// shared-memory address helpers
// --------------------------------------------------------------------------------------------------
CB_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// --------------------------------------------------------------------------------------------------
// mbarrier
// --------------------------------------------------------------------------------------------------
CB_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
CB_DEVINL void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
CB_DEVINL void mbar_arrive(uint32_t bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
CB_DEVINL void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes)
                 : "memory");
}
CB_DEVINL bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
#ifdef CB_WAIT_HINT_NS     // experiment: let the hardware suspend the thread for up to this long instead of the system default
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity), "r"((uint32_t)CB_WAIT_HINT_NS)
        : "memory");
#else
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
#endif
    return ok != 0;
}
// Bounded wait: a pipeline bug must surface as a launch failure, never as a hung GPU.
#ifndef CB_WAIT_TIMEOUT_CYCLES
#define CB_WAIT_TIMEOUT_CYCLES (20ll * 1000 * 1000 * 1000)   // ~10 s at 2 GHz
#endif
CB_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > CB_WAIT_TIMEOUT_CYCLES) __trap();
    }
}

// --------------------------------------------------------------------------------------------------
// programmatic dependent launch: the hot kernels of a tower are launched with programmaticStreamSerialization, so the next
// kernel's CTAs are placed (and run their barrier / descriptor prologue) while the previous grid drains.  pdl_wait()
// blocks until the previous grid has completed and its writes are visible: NO global memory may be touched before it.
// --------------------------------------------------------------------------------------------------
CB_DEVINL void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
CB_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// --------------------------------------------------------------------------------------------------
// TMA: tiled tensor load and 1-D bulk copy, completion on an mbarrier
// --------------------------------------------------------------------------------------------------
CB_DEVINL void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
CB_DEVINL void tma_load_2d(uint32_t dst_smem, const void* tmap, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst_smem),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
CB_DEVINL void bulk_load_1d(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
                 "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
                 : "memory");
}


// --------------------------------------------------------------------------------------------------
// packed 16-bit x2 arithmetic on raw b32 registers, selected by operand type (fp16 / bf16)
// --------------------------------------------------------------------------------------------------
template <bool BF>
struct P2;
template <>
struct P2<false> {   // fp16: 0x6400 = 1024.0, one ulp = 1
    static constexpr uint32_t MAGIC = 0x64006400u;
    CB_DEVINL static uint32_t sub(uint32_t a, uint32_t b) { uint32_t r; asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
    CB_DEVINL static uint32_t mul(uint32_t a, uint32_t b) { uint32_t r; asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
    CB_DEVINL static uint32_t fma(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
    CB_DEVINL static uint32_t splat_from_f16bits(uint16_t h) { return (uint32_t)h | ((uint32_t)h << 16); }
    CB_DEVINL static uint32_t splat_const(float v) { return splat_from_f16bits(__half_as_ushort(__float2half_rn(v))); }
    CB_DEVINL static uint16_t from_float(float v) { return __half_as_ushort(__float2half_rn(v)); }
    CB_DEVINL static float to_float(uint16_t b) { return __half2float(__ushort_as_half(b)); }
};
template <>
struct P2<true> {    // bf16: 0x4300 = 128.0, one ulp = 1
    static constexpr uint32_t MAGIC = 0x43004300u;
    CB_DEVINL static uint32_t sub(uint32_t a, uint32_t b) { uint32_t r; asm("sub.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
    CB_DEVINL static uint32_t mul(uint32_t a, uint32_t b) { uint32_t r; asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
    CB_DEVINL static uint32_t fma(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm("fma.rn.bf16x2 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
    CB_DEVINL static uint32_t splat_from_f16bits(uint16_t h) {   // block scale d is stored as fp16 in the file
        const uint16_t b = __bfloat16_as_ushort(__float2bfloat16_rn(__half2float(__ushort_as_half(h))));
        return (uint32_t)b | ((uint32_t)b << 16);
    }
    CB_DEVINL static uint32_t splat_const(float v) { const uint16_t b = __bfloat16_as_ushort(__float2bfloat16_rn(v)); return (uint32_t)b | ((uint32_t)b << 16); }
    CB_DEVINL static uint16_t from_float(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
    CB_DEVINL static float to_float(uint16_t b) { return __uint_as_float((uint32_t)b << 16); }
};

// x * sigmoid(y) for a = y log2(e): x / (1 + 2^-a) when a >= 0, x 2^a / (1 + 2^a) when a < 0, so the one exponential is
// e = 2^-|a| in (0, 1] and the denominator stays in [1, 2].  Not 0.5 x (1 + tanh(y / 2)): for y < 0 that cancels, and the
// absolute error of tanh.approx (relative 2^-11 near -1) becomes a relative error of the result that grows without bound.
// ex2.approx.ftz (relative error 2^-22) computes 2^64 e, so that e down to 2^-190 stays normal: x e is then right wherever a
// 16-bit result can be normal.  1/d by rcp.approx (relative error about 2^-23): two MUFU operations per element where tanh.approx
// took one.  A reciprocal from a linear start and two Newton steps on the FMA pipe instead measured slower in K1's epilogue (DESIGN
// section 6).  a = +-inf gives x and -+0.
CB_DEVINL float mul_sigmoid_exp2(float x, float a) {
    float es, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(es) : "f"(64.0f - fabsf(a)));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(fmaf(es, 0x1p-64f, 1.0f)));
    return (a >= 0.0f ? x : (x * es) * 0x1p-64f) * r;
}
// tanh-GELU, reference formula ggml/src/ggml.c:3756-3758: 0.5 x (1 + tanh(u)) = x sigmoid(2u), u = sqrt(2/pi) x (1 + 0.044715 x^2);
// 2u log2(e) = x (C0 + C1 x^2) with C0 = 2 sqrt(2/pi) log2(e), C1 = 0.044715 C0
CB_DEVINL float gelu_tanh(float x) { return mul_sigmoid_exp2(x, x * fmaf(0.10294323958f, x * x, 2.3022081981f)); }
// quick-GELU x sigmoid(1.702 x), ggml/src/ggml.c:3783-3785; 1.702 log2(e) = 2.45546695959
CB_DEVINL float gelu_quick(float x) { return mul_sigmoid_exp2(x, 2.4554669596f * x); }


// host side: launch with the PDL attribute (and optionally as clusters of `cluster_x` CTAs)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), unsigned grid, unsigned block, size_t smem, cudaStream_t st, unsigned cluster_x,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    unsigned n = 0;
    static const bool pdl_on = !(getenv("CLIP_B200_PDL") && atoi(getenv("CLIP_B200_PDL")) == 0);   // A/B switch for measurements
    if (pdl_on) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        n++;
    }
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster_x; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
        n++;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace cb
