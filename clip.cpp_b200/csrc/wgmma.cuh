// wgmma.cuh -- warpgroup MMA (sm_90a wgmma.mma_async) wrappers used by the GEMM and attention kernels.
//
// A warpgroup (4 consecutive warps) computes D[64 x N] += A[64 x 16] . B[16 x N] with fp32 accumulators in registers.  Accumulator
// fragment of thread (warp w of the group, lane l): n-tile j (8 columns) holds rows 16w + l/4 (d[4j], d[4j+1]) and 16w + l/4 + 8
// (d[4j+2], d[4j+3]), columns 8j + 2(l%4) + {0, 1}.  Every call must sit between wgmma_fence() and wgmma_commit(); the accumulators
// may only be read after the matching wgmma_wait().
#pragma once
#include "common.cuh"

namespace cb {

CB_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
CB_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
CB_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across a wgmma_wait()
template <int R>
CB_DEVINL void wgmma_fence_regs(float (&d)[R]) {
    #pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
CB_DEVINL void wgmma_fence_regs(int (&d)[R]) {
    #pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+r"(d[i])::"memory");
}

// Shared-memory matrix descriptor of a tile stored with the 128-byte swizzle (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): rows
// of 128 B, 8-row groups 1024 B apart.  K-major operands use only the 8-row group stride; for an MN-major operand no wider than 64
// elements the other offset is never used either, so both are 1024 B.  Tile bases are 1024-B aligned; a 16-element K step inside a
// K-major tile advances the start address by 32 B, one inside an MN-major tile by 16 rows (2048 B).
CB_DEVINL uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);   // start address       [0,14)
    d |= (uint64_t)(1024 >> 4) << 16;               // leading byte offset [16,30)
    d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset  [32,46)
    d |= (uint64_t)1 << 62;                         // layout: 128-byte swizzle [62,64)
    return d;
}

// The same for a tile 16 elements wide stored with the 32-byte swizzle (CU_TENSOR_MAP_SWIZZLE_32B): rows of 32 B, 8-row groups
// 256 B apart.  A K-major operand of one 16-deep k step and an MN-major operand 16 wide both fit in one swizzle atom across, so
// only the 8-row group stride is used.  Tile bases are 256-B aligned; a 16-row step (keys of an MN-major tile) is 512 B.
CB_DEVINL uint64_t wgmma_desc_sw32(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);   // start address       [0,14)
    d |= (uint64_t)(256 >> 4) << 16;                // leading byte offset [16,30)
    d |= (uint64_t)(256 >> 4) << 32;                // stride byte offset  [32,46)
    d |= (uint64_t)3 << 62;                         // layout: 32-byte swizzle [62,64)
    return d;
}

// The same for a tile 32 elements wide stored with the 64-byte swizzle (CU_TENSOR_MAP_SWIZZLE_64B): rows of 64 B, 8-row groups
// 512 B apart.  A K-major operand steps 16 elements (32 B) inside the row, and an MN-major operand 32 wide is one swizzle atom
// across, so only the 8-row group stride is used.  Tile bases are 512-B aligned; a 16-row step (keys of an MN-major tile) is 1024 B.
CB_DEVINL uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);   // start address       [0,14)
    d |= (uint64_t)(512 >> 4) << 16;                // leading byte offset [16,30)
    d |= (uint64_t)(512 >> 4) << 32;                // stride byte offset  [32,46)
    d |= (uint64_t)2 << 62;                         // layout: 64-byte swizzle [62,64)
    return d;
}

// D[64 x 256] (+)= A[64 x 16] . B[256 x 16]^T, both operands K-major in shared memory (descriptors), fp32 accumulators
template <bool BF>
CB_DEVINL void wgmma_ss_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_SS_N256(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %130, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])  \
                 : "l"(da), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_SS_N256("bf16");
    else CB_WGMMA_SS_N256("f16");
#undef CB_WGMMA_SS_N256
}

// D[64 x 256] (+)= A[64 x 16] . B[256 x 16]^T: A from registers (the m16n8k16 A-fragment layout per warp), B K-major in shared memory
template <bool BF>
CB_DEVINL void wgmma_rs_n256(float (&d)[128], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_RSK_N256(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %133, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])  \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_RSK_N256("bf16");
    else CB_WGMMA_RSK_N256("f16");
#undef CB_WGMMA_RSK_N256
}

// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, both operands K-major in shared memory (descriptors), fp32 accumulators
template <bool BF>
CB_DEVINL void wgmma_ss_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_SS_N128(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %66, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])  \
                 : "l"(da), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_SS_N128("bf16");
    else CB_WGMMA_SS_N128("f16");
#undef CB_WGMMA_SS_N128
}

// D[64 x 64], D[64 x 32] and D[64 x 16] (+)= A[64 x 16] . B[N x 16]^T, both operands K-major in shared memory: the narrower S
// products of the attention kernel's ragged last key block
template <bool BF>
CB_DEVINL void wgmma_ss_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_SS_N64(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %34, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])  \
                 : "l"(da), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_SS_N64("bf16");
    else CB_WGMMA_SS_N64("f16");
#undef CB_WGMMA_SS_N64
}
template <bool BF>
CB_DEVINL void wgmma_ss_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_SS_N32(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %18, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])  \
                 : "l"(da), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_SS_N32("bf16");
    else CB_WGMMA_SS_N32("f16");
#undef CB_WGMMA_SS_N32
}
template <bool BF>
CB_DEVINL void wgmma_ss_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_SS_N16(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %10, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])  \
                 : "l"(da), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_SS_N16("bf16");
    else CB_WGMMA_SS_N16("f16");
#undef CB_WGMMA_SS_N16
}

// D[64 x 64] (+)= A[64 x 16] . B[16 x 64]: A from registers (the m16n8k16 A-fragment layout per warp), B MN-major in shared memory
template <bool BF>
CB_DEVINL void wgmma_rs_n64_bmn(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_RS_N64(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %37, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])  \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_RS_N64("bf16");
    else CB_WGMMA_RS_N64("f16");
#undef CB_WGMMA_RS_N64
}

// D[64 x 32] (+)= A[64 x 16] . B[16 x 32]: A from registers, B MN-major in shared memory (columns 64-95 of a 104-wide head)
template <bool BF>
CB_DEVINL void wgmma_rs_n32_bmn(float (&d)[16], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_RS_N32(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %21, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 1;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])  \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_RS_N32("bf16");
    else CB_WGMMA_RS_N32("f16");
#undef CB_WGMMA_RS_N32
}

// D[64 x 16] (+)= A[64 x 16] . B[16 x 16]: A from registers, B MN-major in shared memory (the 16-column tail of an 80- or 104-wide
// head)
template <bool BF>
CB_DEVINL void wgmma_rs_n16_bmn(float (&d)[8], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_RS_N16(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %13, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 1;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])  \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_RS_N16("bf16");
    else CB_WGMMA_RS_N16("f16");
#undef CB_WGMMA_RS_N16
}

// D[64 x 8] (+)= A[64 x 16] . B[8 x 16]^T, both operands K-major in shared memory: the one-query tile of the 16-bit search kernel
// (search.cu)
template <bool BF>
CB_DEVINL void wgmma_ss_n8(float (&d)[4], uint64_t da, uint64_t db, uint32_t accumulate) {
#define CB_WGMMA_SS_N8(TY)                                                                                 \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %6, 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32." TY "." TY " {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t}"  \
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])  \
                 : "l"(da), "l"(db), "r"(accumulate))
    if constexpr (BF) CB_WGMMA_SS_N8("bf16");
    else CB_WGMMA_SS_N8("f16");
#undef CB_WGMMA_SS_N8
}

// D[64 x N] (+)= A[64 x 32] . B[N x 32]^T for N = 128, 64, 32, 16 and 8: signed 8-bit operands, both K-major in shared memory
// (128-byte swizzle: a k32 step is 32 B, as a k16 step of 16-bit operands), int32 accumulators in the fragment layout above.  The
// integer products and sums are exact (no saturation: the int8 search keeps |D| below 2^31).  The int8 search kernel (search.cu).
CB_DEVINL void wgmma_ss_n128_s8(int (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(da), "l"(db), "r"(accumulate));
}
CB_DEVINL void wgmma_ss_n64_s8(int (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(da), "l"(db), "r"(accumulate));
}
CB_DEVINL void wgmma_ss_n32_s8(int (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(da), "l"(db), "r"(accumulate));
}
CB_DEVINL void wgmma_ss_n16_s8(int (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "l"(da), "l"(db), "r"(accumulate));
}
CB_DEVINL void wgmma_ss_n8_s8(int (&d)[4], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %6, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k32.s32.s8.s8 {%0, %1, %2, %3}, %4, %5, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "l"(da), "l"(db), "r"(accumulate));
}

}  // namespace cb
