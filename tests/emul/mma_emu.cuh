// mma_emu.cuh -- TEST INFRASTRUCTURE ONLY: what csrc/mma.cuh means, for the SIMT emulator.
// mma: the 32 lanes' fragments meet in a per-warp table (a warp rendezvous), then each lane forms its own four outputs
// from the PTX fragment layout, accumulating the eight products in k order.  cp.async: an immediate copy.
#pragma once
#include "simt_emu.h"

namespace h3dgs {

inline uint32_t to_tf32(float x) {
    uint32_t u = __float_as_uint(x);
    if ((u & 0x7f800000u) != 0x7f800000u) { u += 0x1000u; u &= 0xffffe000u; }
    return u;
}

inline void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    static uint32_t A[32][32][4], B[32][32][2];                     // [warp][lane][register]
    const int w = simt::g_cur->warp, lane = simt::g_cur->lane;
    memcpy(A[w][lane], a, sizeof(a));
    memcpy(B[w][lane], b, sizeof(b));
    __syncwarp();
    // A[r][k] is register (r / 8) + 2 (k / 4) of lane (r % 8) * 4 + k % 4; B[k][n] is register k / 4 of lane n * 4 + k % 4;
    // the hardware reads the TF32 bits of each operand
    const int g = lane >> 2, t = lane & 3;
    for (int e = 0; e < 4; e++) {
        const int r = g + 8 * (e >> 1), n = 2 * t + (e & 1);
        float acc = d[e];
        for (int k = 0; k < 8; k++) {
            const float av = __uint_as_float(A[w][(r & 7) * 4 + (k & 3)][(r >> 3) + 2 * (k >> 2)] & 0xffffe000u);
            const float bv = __uint_as_float(B[w][n * 4 + (k & 3)][k >> 2] & 0xffffe000u);
            acc += av * bv;
        }
        d[e] = acc;
    }
    __syncwarp();
}

inline void cp_async16(void* smem_dst, const void* gmem_src, bool valid) {
    if (valid) memcpy(smem_dst, gmem_src, 16);
    else memset(smem_dst, 0, 16);
}
inline void cp_async_commit() {}
template <int N> inline void cp_async_wait() {}

}  // namespace h3dgs
