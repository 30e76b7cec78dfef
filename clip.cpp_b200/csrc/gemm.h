// gemm.h -- host interface of the fused block-dequant wgmma GEMM (gemm_dq.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cb {

// Opaque 128-byte CUtensorMap (driver type), kept by value so it can be passed as a __grid_constant__.
struct alignas(64) TmaMap {
    unsigned char bytes[128];
};

// Tiled tensor map over a row-major 16-bit matrix [rows, cols]; box = [box_rows, 64 cols] with the
// 128-byte swizzle (64 x 2 B = one swizzle row).  Out-of-range rows read as zero.
bool make_tma_2d_16bit(TmaMap* out, const void* gptr, uint64_t rows, uint64_t cols, uint64_t row_stride_elems,
                       uint32_t box_rows);

constexpr int GEMM_BM = 128;   // features per tile (two wgmma M = 64 warpgroups)
constexpr int GEMM_BN = 256;   // tokens per tile   (wgmma N; 128 fp32 accumulator registers per thread)
constexpr int GEMM_BK = 64;

struct GemmArgs {
    // Y[M tokens, N features] (+)= X[M, K] . W[N, K]^T (+ bias[N]),  computed as D[feature, token] tiles
    const TmaMap* x_map = nullptr;   // activations X, 16-bit, box rows = GEMM_BN
    const TmaMap* w_map = nullptr;   // QT_F16 only: weights W [N, K] fp16, box rows = GEMM_BM
    const uint8_t* w_packed = nullptr;   // quantized types: re-tiled blocks (wpack.h)
    int qtype = 1;                   // cb::QType of W
    bool operand_bf16 = false;       // X (and the unpacked W) are bf16 instead of fp16; must be false for QT_F16
    const float* bias = nullptr;     // [N] or null
    void* out = nullptr;             // EPI_*16: 16-bit [M, ldo]; EPI_*32: fp32 [M, ldo]
    int M = 0, N = 0, K = 0, ldo = 0;
    int epi = 0;                     // cb::Epi
    int out_bf16 = 0;                // 16-bit stores: bf16 (1) or fp16 (0)
    int scale_cols = 0;              // features n < scale_cols are multiplied by `scale` after the bias add
    float scale = 1.0f;              //   (Q = (x.Wq + bq) / sqrt(dh): clip.cpp:1082, 1363)
};

// Launches on `stream`; returns cudaSuccess or the launch error.  `*launches` is incremented per kernel launch.
cudaError_t gemm_launch(const GemmArgs& a, cudaStream_t stream, int num_sms, uint64_t* launches);

// One-time: opt in to the large dynamic shared memory carve-outs.
cudaError_t gemm_init();

}  // namespace cb
