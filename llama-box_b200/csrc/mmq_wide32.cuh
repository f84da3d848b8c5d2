// mmq_wide32.cuh — what the int8 tile kernel (mmq_tc32.cu) needs to read the wide path's non-linear 4-bit formats, IQ4_NL and IQ4_XS,
// in ggml's native block layout (the layout decode and GET_ROWS read too), and the q8_K arithmetic of the IQ4_XS activation image.
//
// Everything here is `__host__ __device__`, so tests/hostsim compiles the same functions with g++ and checks them against the C oracle
// (tests/test_mmq_iq4_hostsim.py): the loads of one 128-k stage, its unpack to int8, and the q8_K quantisation of 8 elements.
//
// A stage is 128 k = 4 blocks of 32 elements, loaded as 9 aligned 8-byte words and nothing else:
//     IQ4_NL  {f16 d; u8 qs[16]} 18 B: a row of k % 256 == 0 is k / 256 x 144 B, so stage s starts 8-byte aligned at byte 72 s and
//             its 72 bytes are the 4 blocks (at 0, 18, 36, 54: only 2-byte aligned, realigned from the words by 16-bit shifts).
//             The load ends at the stage's last byte, which at the end of a row is the end of the matrix.
//     IQ4_XS  {f16 d; u16 scales_h; u8 scales_l[4]; u8 qs[128]} 136 B, 8-byte aligned: stage s is half s % 2 of super-block s / 2,
//             its 8-byte header and the 64 qs bytes of sub-blocks 4 (s % 2) .. 4 (s % 2) + 3.
// Elements are placed as Q4_0's are (low nibbles = elements 0..15, high nibbles = 16..31), so the activation image is the natural order.
#pragma once
#include "extfmt.cuh"

#if !defined(__CUDA_ARCH__)
#  include <math.h>
#endif

// 8 bytes at p (8-byte aligned) as two little-endian words
XF_HD void w32_ld64(const uint8_t * p, uint32_t & lo, uint32_t & hi) {
#if defined(__CUDA_ARCH__)
    const uint2 v = __ldg((const uint2 *)p); lo = v.x; hi = v.y;
#else
    XF_AL(p, 8); memcpy(&lo, p, 4); memcpy(&hi, p + 4, 4);
#endif
}

// bytes of {x, y} picked by the low 3 bits of each selector nibble (PRMT without the sign-replicate mode)
XF_HD uint32_t w32_perm(uint32_t x, uint32_t y, uint32_t s) {
#if defined(__CUDA_ARCH__)
    return __byte_perm(x, y, s);
#else
    const uint64_t v = (uint64_t)x | ((uint64_t)y << 32);
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
#endif
}

// 4 nibbles (one per byte, masked to 0..15) -> kvalues_iq4nl[nibble] as 4 int8: two byte permutes over the table's 16 bytes
// (-127 -104 -83 -65 | -49 -35 -22 -10 | 1 13 25 38 | 53 69 89 113) and a per-byte select on bit 3
XF_HD uint32_t w32_iq4_lut(uint32_t n) {
    const uint32_t sel = (n & 7u) | ((n >> 4) & 0x70u) | ((n >> 8) & 0x700u) | ((n >> 12) & 0x7000u);
    const uint32_t lo = w32_perm(0xBFAD9881u, 0xF6EADDCFu, sel), hi = w32_perm(0x26190D01u, 0x71594535u, sel);
    const uint32_t m = ((n >> 3) & 0x01010101u) * 0xFFu;
    return (lo & ~m) | (hi & m);
}

// stage s of a row as loaded: w[0..17] (IQ4_NL: the 72 bytes; IQ4_XS: w[0..1] the header, w[2..17] the 64 qs bytes)
template <int T> XF_HD void w32_load(const uint8_t * row, int64_t s, uint32_t (&w)[18]) {
    if (T == XF_IQ4_NL) {
        const uint8_t * p = row + s * 72;
        for (int i = 0; i < 9; i++) w32_ld64(p + 8 * i, w[2 * i], w[2 * i + 1]);
    } else {
        const uint8_t * p = row + (s >> 1) * 136;
        w32_ld64(p, w[0], w[1]);
        p += 8 + (s & 1) * 64;
        for (int i = 0; i < 8; i++) w32_ld64(p + 8 * i, w[2 + 2 * i], w[3 + 2 * i]);
    }
}

// block b (0..3) of stage s: q[i] = int8 elements 4 i .. 4 i + 3 (i < 4) / 16 + 4 (i - 4) .. (i >= 4), i.e. the block's two 16-byte
// K-chunks of the int8 A operand; returns the word the fold needs for it:
//     IQ4_NL  d_w as f16 bits
//     IQ4_XS  d_w as f16 bits | (ls - 32) << 16 (a signed 16-bit field), ls the 6-bit scale of sub-block 4 (s % 2) + b
template <int T> XF_HD uint32_t w32_unpack(const uint32_t (&w)[18], int64_t s, int b, uint32_t (&q)[8]) {
    uint32_t qw[4], sc;
    if (T == XF_IQ4_NL) {
        const int o = 18 * b + 2;                                            // byte offset of qs in the stage: 2, 20, 38, 56
        for (int i = 0; i < 4; i++) qw[i] = (o & 2) ? (w[(o >> 2) + i] >> 16) | (w[(o >> 2) + i + 1] << 16) : w[(o >> 2) + i];
        sc = (w[(18 * b) >> 2] >> (8 * ((18 * b) & 3))) & 0xffffu;
    } else {
        for (int i = 0; i < 4; i++) qw[i] = w[2 + 4 * b + i];
        const int ib = 4 * (int)(s & 1) + b;
        sc = (w[0] & 0xffffu) | ((uint32_t)(xf_iq4xs_ls((int)(w[1] >> (8 * (ib >> 1))), w[0] >> 16, ib) - 32) << 16);
    }
    for (int i = 0; i < 4; i++) { q[i] = w32_iq4_lut(qw[i] & 0x0F0F0F0Fu); q[4 + i] = w32_iq4_lut((qw[i] >> 4) & 0x0F0F0F0Fu); }
    return sc;
}

// q8_K (quantize_row_q8_K_ref) of 8 elements of a super-block whose first element of largest |x| is maxv (am = |maxv|): iscale =
// -127 / maxv, q = MIN(127, nearest_int(iscale * x)) (round to nearest even), d = 1 / iscale; 0 and d = 0 for an all-zero super-block.
// q packed as 8 int8 (lo: elements 0..3, hi: 4..7); returns d.
XF_HD float w32_q8k_quant8(const float (&v)[8], float maxv, float am, uint32_t & lo, uint32_t & hi) {
    int q[8];
    float d = 0.0f;
    if (am != 0.0f) {
#if defined(__CUDA_ARCH__)
        const float iscale = __fdiv_rn(-127.0f, maxv);
        for (int j = 0; j < 8; j++) { const int t = __float2int_rn(__fmul_rn(iscale, v[j])); q[j] = t > 127 ? 127 : t; }
        d = __fdiv_rn(1.0f, iscale);
#else
        volatile float iscale = -127.0f / maxv;
        for (int j = 0; j < 8; j++) { const int t = (int)nearbyintf(xf_mul(iscale, v[j])); q[j] = t > 127 ? 127 : t; }
        volatile float dd = 1.0f / iscale; d = dd;
#endif
    } else {
        for (int j = 0; j < 8; j++) q[j] = 0;
    }
    lo = (q[0] & 0xff) | ((q[1] & 0xff) << 8) | ((q[2] & 0xff) << 16) | ((uint32_t)(q[3] & 0xff) << 24);
    hi = (q[4] & 0xff) | ((q[5] & 0xff) << 8) | ((q[6] & 0xff) << 16) | ((uint32_t)(q[7] & 0xff) << 24);
    return d;
}
