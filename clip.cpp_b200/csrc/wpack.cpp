// wpack.cpp -- host-side lossless re-tiling of ggml quantized weights (see wpack.h for the layout).
#include "wpack.h"

#include <string.h>

#include <thread>
#include <vector>

namespace cb {

namespace {

struct BlockView {          // decoded fields of one ggml block (values untouched)
    uint16_t d = 0, m = 0;  // fp16 bits
    uint8_t q[32];          // unsigned stored quants (4/5 bit: 0..15 / 0..31, 8 bit: raw int8 bits)
};

// ggml block -> fields.  Layouts: ggml/src/ggml.c:866-911; element j / j+16 share byte j (ggml.c:1503-1512).
void decode_block(int qt, const uint8_t* b, BlockView& v) {
    memcpy(&v.d, b, 2);
    const uint8_t* qs = nullptr;
    uint32_t qh = 0;
    switch (qt) {
    case 2: qs = b + 2; break;
    case 3: memcpy(&v.m, b + 2, 2); qs = b + 4; break;
    case 6: memcpy(&qh, b + 2, 4); qs = b + 6; break;
    case 7: memcpy(&v.m, b + 2, 2); memcpy(&qh, b + 4, 4); qs = b + 8; break;
    case 8: memcpy(v.q, b + 2, 32); return;
    }
    for (int j = 0; j < 16; j++) {
        v.q[j] = (uint8_t)((qs[j] & 0x0F) | (((qh >> j) & 1u) << 4));
        v.q[j + 16] = (uint8_t)((qs[j] >> 4) | (((qh >> (j + 16)) & 1u) << 4));
    }
}

void encode_block(int qt, const BlockView& v, uint8_t* b) {
    memcpy(b, &v.d, 2);
    uint8_t* qs = nullptr;
    switch (qt) {
    case 2: qs = b + 2; break;
    case 3: memcpy(b + 2, &v.m, 2); qs = b + 4; break;
    case 6: qs = b + 6; break;
    case 7: memcpy(b + 2, &v.m, 2); qs = b + 8; break;
    case 8: memcpy(b + 2, v.q, 32); return;
    }
    uint32_t qh = 0;
    for (int j = 0; j < 16; j++) {
        qs[j] = (uint8_t)((v.q[j] & 0x0F) | ((v.q[j + 16] & 0x0F) << 4));
        qh |= (uint32_t)((v.q[j] >> 4) & 1u) << j;
        qh |= (uint32_t)((v.q[j + 16] >> 4) & 1u) << (j + 16);
    }
    if (qt == 6) memcpy(b + 2, &qh, 4);
    if (qt == 7) memcpy(b + 4, &qh, 4);
}

inline int nib_pos(int e) { return (e >> 1) * 4 + (e & 1) * 16; }          // 4-bit field position in a word
inline int hi_pos(int j, int e) { return 4 * j + (e >> 1) + 16 * (e & 1); }  // 5th-bit position in qh word

void put_thread(int qt, uint8_t* chunk, int t, const BlockView& v) {
    if (qt == 8) {
        memcpy(chunk + 16 * t, v.q, 16);
        memcpy(chunk + 4096 + 16 * t, v.q + 16, 16);
        memcpy(chunk + 8192 + 2 * t, &v.d, 2);
        return;
    }
    uint32_t w[4] = {0, 0, 0, 0}, hq = 0;
    for (int j = 0; j < 4; j++)
        for (int e = 0; e < 8; e++) {
            const uint8_t q = v.q[8 * j + e];
            w[j] |= (uint32_t)(q & 0x0F) << nib_pos(e);
            hq |= (uint32_t)((q >> 4) & 1u) << hi_pos(j, e);
        }
    memcpy(chunk + 16 * t, w, 16);
    size_t off = 4096;
    if (qt == 6 || qt == 7) { memcpy(chunk + off + 4 * t, &hq, 4); off += 1024; }
    if (qt == 2 || qt == 6) memcpy(chunk + off + 2 * t, &v.d, 2);
    else { memcpy(chunk + off + 4 * t, &v.d, 2); memcpy(chunk + off + 4 * t + 2, &v.m, 2); }
}

void get_thread(int qt, const uint8_t* chunk, int t, BlockView& v) {
    v = BlockView();
    if (qt == 8) {
        memcpy(v.q, chunk + 16 * t, 16);
        memcpy(v.q + 16, chunk + 4096 + 16 * t, 16);
        memcpy(&v.d, chunk + 8192 + 2 * t, 2);
        return;
    }
    uint32_t w[4], hq = 0;
    memcpy(w, chunk + 16 * t, 16);
    size_t off = 4096;
    if (qt == 6 || qt == 7) { memcpy(&hq, chunk + off + 4 * t, 4); off += 1024; }
    if (qt == 2 || qt == 6) memcpy(&v.d, chunk + off + 2 * t, 2);
    else { memcpy(&v.d, chunk + off + 4 * t, 2); memcpy(&v.m, chunk + off + 4 * t + 2, 2); }
    for (int j = 0; j < 4; j++)
        for (int e = 0; e < 8; e++)
            v.q[8 * j + e] = (uint8_t)(((w[j] >> nib_pos(e)) & 0x0F) | (((hq >> hi_pos(j, e)) & 1u) << 4));
}

template <class F>
void parallel_tiles(int64_t n_ft, F&& f) {
    unsigned nt = std::thread::hardware_concurrency();
    if (nt == 0) nt = 4;
    if (nt > 16) nt = 16;
    if ((int64_t)nt > n_ft) nt = (unsigned)n_ft;
    if (nt <= 1) { for (int64_t i = 0; i < n_ft; i++) f(i); return; }
    std::vector<std::thread> th;
    for (unsigned w = 0; w < nt; w++)
        th.emplace_back([&, w]() { for (int64_t i = w; i < n_ft; i += nt) f(i); });
    for (auto& t : th) t.join();
}

}  // namespace

bool wpack_repack(int qt, const uint8_t* src, int64_t N, int64_t K, uint8_t* dst) {
    const size_t cb_ = wpack_chunk_bytes(qt), bb = wpack_ggml_block_bytes(qt);
    if (!cb_ || N % WPACK_ROWS || K % WPACK_K) return false;
    const int64_t nkb = K / WPACK_K, row_bytes = (K / 32) * (int64_t)bb;
    parallel_tiles(N / WPACK_ROWS, [&](int64_t ft) {
        for (int64_t kb = 0; kb < nkb; kb++) {
            uint8_t* chunk = dst + (ft * nkb + kb) * cb_;
            for (int t = 0; t < 256; t++) {
                const int half = t >> 7, r = t & 127;
                BlockView v;
                decode_block(qt, src + (ft * WPACK_ROWS + r) * row_bytes + (kb * 2 + half) * bb, v);
                put_thread(qt, chunk, t, v);
            }
        }
    });
    return true;
}

bool wpack_unpack(int qt, const uint8_t* packed, int64_t N, int64_t K, uint8_t* dst) {
    const size_t cb_ = wpack_chunk_bytes(qt), bb = wpack_ggml_block_bytes(qt);
    if (!cb_ || N % WPACK_ROWS || K % WPACK_K) return false;
    const int64_t nkb = K / WPACK_K, row_bytes = (K / 32) * (int64_t)bb;
    parallel_tiles(N / WPACK_ROWS, [&](int64_t ft) {
        for (int64_t kb = 0; kb < nkb; kb++) {
            const uint8_t* chunk = packed + (ft * nkb + kb) * cb_;
            for (int t = 0; t < 256; t++) {
                const int half = t >> 7, r = t & 127;
                BlockView v;
                get_thread(qt, chunk, t, v);
                encode_block(qt, v, dst + (ft * WPACK_ROWS + r) * row_bytes + (kb * 2 + half) * bb);
            }
        }
    });
    return true;
}

bool pad_head_rows(const uint8_t* src, size_t row_bytes, int64_t rows, int dh, int dhp, uint8_t* dst) {
    if (dh <= 0 || dhp < dh || rows % dh) return false;
    const size_t head = (size_t)dh * row_bytes, pad = (size_t)(dhp - dh) * row_bytes;
    for (int64_t h = 0; h < rows / dh; h++) {
        uint8_t* d = dst + (size_t)h * (head + pad);
        memcpy(d, src + (size_t)h * head, head);
        memset(d + head, 0, pad);
    }
    return true;
}

}  // namespace cb
