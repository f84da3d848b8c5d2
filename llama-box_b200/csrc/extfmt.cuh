// extfmt.cuh — per-format arithmetic of the "wide" matvec / MUL_MAT_ID / quantised GET_ROWS kernels (mmvq_ext.cu):
// one 32-element sub-block of a weight row against the matching 32 int8 activations, and its de-quantisation.
//
// Covers the formats SURVEY.md §8 (f3) lists beyond the five the tuned decode kernels carry — Q4_1, Q5_1, Q2_K, Q3_K, IQ4_NL,
// IQ4_XS, MXFP4 in ggml's native block layout (ggml/src/ggml-common.h:176-300,414-428) — and, for MUL_MAT_ID / GET_ROWS on
// the types of a Q4_K_M / Q4_0 / Q8_0 MoE file, the library's own weight layout of Q4_0 / Q5_0 / Q8_0 / Q6_K (row-wise
// structure-of-arrays, b200_ops.h "repacked") and native Q4_K / Q5_K.
//
// Numerics follow the CPU oracle (ggml-cpu/quants.c generic functions, cited per format): the integer sums are the same
// integers; only the order of the f32 additions over sub-blocks differs.
//
// Everything here is `__host__ __device__` and free of CUDA-only constructs, so tests/hostsim compiles THE SAME FUNCTIONS with
// g++ and checks them against the unmodified reference on the CPU (tests/test_extfmt_hostsim.py) — the bit manipulation is
// verified without a GPU; the kernels around it (mmvq_ext.cu) only add the loops.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#  define XF_HD __host__ __device__ __forceinline__
#else
#  define XF_HD inline
#endif

// enum ggml_type values (ggml/include/ggml.h:377-418)
enum {
    XF_Q4_0 = 2, XF_Q4_1 = 3, XF_Q5_0 = 6, XF_Q5_1 = 7, XF_Q8_0 = 8, XF_Q2_K = 10, XF_Q3_K = 11, XF_Q4_K = 12, XF_Q5_K = 13, XF_Q6_K = 14,
    XF_IQ4_NL = 20, XF_IQ4_XS = 23, XF_MXFP4 = 39,
};

// activation family of a weight type (ggml-cpu/ggml-cpu.c:209-303 vec_dot_type): 0 = q8_K (256-wide), 1 = q8_0 / q8_1 (32-wide), -1 = not handled
XF_HD int xf_act_family(int t) {
    switch (t) {
        case XF_Q2_K: case XF_Q3_K: case XF_Q4_K: case XF_Q5_K: case XF_Q6_K: case XF_IQ4_XS: return 0;
        case XF_Q4_0: case XF_Q4_1: case XF_Q5_0: case XF_Q5_1: case XF_Q8_0: case XF_IQ4_NL: case XF_MXFP4: return 1;
        default: return -1;
    }
}
XF_HD int xf_block_elems(int t) { return xf_act_family(t) == 0 ? 256 : (xf_act_family(t) == 1 ? 32 : 0); }
XF_HD int xf_block_bytes(int t) {
    switch (t) {
        case XF_Q4_0: return 18;  case XF_Q4_1: return 20;  case XF_Q5_0: return 22;  case XF_Q5_1: return 24;  case XF_Q8_0: return 34;
        case XF_Q2_K: return 84;  case XF_Q3_K: return 110; case XF_Q4_K: return 144; case XF_Q5_K: return 176; case XF_Q6_K: return 210;
        case XF_IQ4_NL: return 18; case XF_IQ4_XS: return 136; case XF_MXFP4: return 17;
        default: return 0;
    }
}
// formats this file reads in the LIBRARY's row layout (b200_repack_rows) rather than ggml's
XF_HD bool xf_is_repacked(int t) { return t == XF_Q4_0 || t == XF_Q5_0 || t == XF_Q8_0 || t == XF_Q6_K; }
// the formats only the wide kernels handle (native ggml layout)
XF_HD bool xf_is_ext_only(int t) { return t == XF_Q4_1 || t == XF_Q5_1 || t == XF_Q2_K || t == XF_Q3_K || t == XF_IQ4_NL || t == XF_IQ4_XS || t == XF_MXFP4; }

// ---- scalar helpers ----------------------------------------------------------------------------------------------------
XF_HD float xf_bits2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
// IEEE half -> float, exact (same value as F16C / __half2float)
XF_HD float xf_h2f(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    const uint32_t e = (h >> 10) & 0x1f, m = h & 0x3ffu;
    if (e == 0) {
        if (m == 0) return xf_bits2f(sign);
        // subnormal half: value = m * 2^-24
        const float v = (float)m * xf_bits2f(0x33800000u);        // 2^-24
        return sign ? -v : v;
    }
    if (e == 31) return xf_bits2f(sign | 0x7f800000u | (m << 13));
    return xf_bits2f(sign | ((e + 112) << 23) | (m << 13));
}
// E8M0 -> float, halved (ggml-impl.h:451-470 ggml_e8m0_to_fp32_half)
XF_HD float xf_e8m0_half(uint8_t x) { return xf_bits2f(x < 2 ? (0x00200000u << x) : ((uint32_t)(x - 1) << 23)); }

// host builds of the test harness (tests/hostsim, -DXF_CHECK_ALIGN) count loads a GPU would trap on; x86 tolerates them silently
#if !defined(__CUDA_ARCH__) && defined(XF_CHECK_ALIGN)
extern "C" long xf_misaligned;
#  define XF_AL(p, n) do { if ((uintptr_t)(p) & ((n) - 1)) __atomic_add_fetch(&xf_misaligned, 1, __ATOMIC_RELAXED); } while (0)
#else
#  define XF_AL(p, n) do { } while (0)
#endif
XF_HD uint32_t xf_ld8x4(const uint8_t * p)  { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
XF_HD uint32_t xf_ld16(const uint8_t * p)   { XF_AL(p, 2); return *(const uint16_t *)p; }               // p 2-byte aligned
XF_HD uint32_t xf_ld16x2(const uint8_t * p) { return xf_ld16(p) | (xf_ld16(p + 2) << 16); }             // p 2-byte aligned
XF_HD uint32_t xf_ld32(const uint8_t * p)   { XF_AL(p, 4); return *(const uint32_t *)p; }               // p 4-byte aligned

// 4 x (s8 * s8) + c.  Weight bytes below 128 may be passed as they are (u8 == s8 there).
XF_HD int xf_dp4a(uint32_t a, uint32_t b, int c) {
#if defined(__CUDA_ARCH__)
    return __dp4a((int)a, (int)b, c);
#else
    for (int i = 0; i < 4; i++) c += (int)(int8_t)(a >> (8 * i)) * (int)(int8_t)(b >> (8 * i));
    return c;
#endif
}
// bit i of x (i = 0..3) -> bit `pos` of byte i
XF_HD uint32_t xf_spread4(uint32_t x, int pos) {
    return (((x & 1u)) | ((x & 2u) << 7) | ((x & 4u) << 14) | ((x & 8u) << 21)) << pos;
}
// 16-entry int8 tables as two 64-bit constants (no memory): kvalues_iq4nl / kvalues_mxfp4 (ggml-common.h:1088-1096)
XF_HD int xf_kv_iq4nl(uint32_t i) {
    // -127, -104, -83, -65, -49, -35, -22, -10, 1, 13, 25, 38, 53, 69, 89, 113
    const uint64_t lo = 0xF6EADDCFBFAD9881ull, hi = 0x7159453526190D01ull;
    return (int)(int8_t)(((i & 8) ? hi : lo) >> (8 * (i & 7)));
}
XF_HD int xf_kv_mxfp4(uint32_t i) {
    // 0, 1, 2, 3, 4, 6, 8, 12, 0, -1, -2, -3, -4, -6, -8, -12
    const uint64_t lo = 0x0C08060403020100ull, hi = 0xF4F8FAFCFDFEFF00ull;
    return (int)(int8_t)(((i & 8) ? hi : lo) >> (8 * (i & 7)));
}
template <bool MX> XF_HD uint32_t xf_lut4(uint32_t nib) {           // 4 nibbles (one per byte, already masked) -> 4 signed bytes
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t n = (nib >> (8 * i)) & 0xF;
        r |= (uint32_t)(uint8_t)(MX ? xf_kv_mxfp4(n) : xf_kv_iq4nl(n)) << (8 * i);
    }
    return r;
}
// 6-bit scale / min j (0..7) of a Q4_K / Q5_K super-block (ggml-quants.c:703-711 get_scale_min_k4)
XF_HD void xf_scale_min_k4(int j, const uint8_t * q, int * d, int * m) {
    if (j < 4) { *d = q[j] & 63; *m = q[j + 4] & 63; }
    else       { *d = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4); *m = (q[j + 4] >> 4) | ((q[j] >> 6) << 4); }
}
// signed 6-bit scale g (0..15) of a Q3_K super-block, already minus 32 (ggml-cpu/quants.c:528-533)
XF_HD int xf_q3k_scale(const uint8_t * sc12, int g) {                     // sc12 2-byte aligned
    const uint32_t a0 = xf_ld16x2(sc12), a1 = xf_ld16x2(sc12 + 4), tmp = xf_ld16x2(sc12 + 8);
    const uint32_t k1 = 0x03030303u, k2 = 0x0f0f0f0fu;
    uint32_t w;
    switch (g >> 2) {
        case 0:  w = (a0 & k2)        | (((tmp >> 0) & k1) << 4); break;
        case 1:  w = (a1 & k2)        | (((tmp >> 2) & k1) << 4); break;
        case 2:  w = ((a0 >> 4) & k2) | (((tmp >> 4) & k1) << 4); break;
        default: w = ((a1 >> 4) & k2) | (((tmp >> 6) & k1) << 4); break;
    }
    return (int)(int8_t)(w >> (8 * (g & 3))) - 32;
}

// 6-bit scale ls of sub-block ib (0..7) of an IQ4_XS super-block (ggml-quants.c dequantize_row_iq4_xs): scl holds its scales_l byte
// scales_l[ib / 2] in the low 8 bits (higher bits are ignored), sch the 16-bit scales_h (higher bits are ignored)
XF_HD int xf_iq4xs_ls(int scl, uint32_t sch, int ib) { return (int)((scl >> (4 * (ib & 1))) & 0xF) | (int)(((sch >> (2 * ib)) & 3) << 4); }

// ---- the quantised activation column a sub-block is multiplied with ------------------------------------------------------
//   family 1 (32-wide, q8_0 / q8_1 of the x86 CPU backend, ggml-cpu/arch/x86/quants.c:290-492):
//       qs[k] int8 | d[k/32] = value of the f16-rounded scale | s[k/32] = value of f16(d_unrounded * sum)  (q8_1 only) | bs[k/32] = sum of the 32 quants
//   family 0 (256-wide, q8_K, ggml-quants.c:2555-2592):
//       qs[k] int8 | d[k/256] f32 | bs[k/16] = sums of 16 quants
struct XfAct { const int8_t * qs; const float * d; const float * s; const int16_t * bs; };

// =========================================================================================================================
// xf_sub_dot<T>: contribution of sub-block u (elements [32u, 32u+32)) of a weight row to the dot product with the column.
//   row       : first byte of the weight row;  nb = blocks per row IN THE LAYOUT (k / block elems; the repacked section offsets depend on it)
// =========================================================================================================================
template <int T> XF_HD float xf_sub_dot(const uint8_t * row, int64_t nb, int64_t u, const XfAct & A);

// Q4_0, library layout [qs 16B x nb][d f16 x nb]  (ggml-cpu/quants.c:115-149: sumi = sum (nib - 8) * q8; sumf += sumi * d_x * d_y)
template <> XF_HD float xf_sub_dot<XF_Q4_0>(const uint8_t * row, int64_t nb, int64_t u, const XfAct & A) {
    const uint8_t * qs = row + u * 16;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld32(qs + 4 * i);
        sumi = xf_dp4a(w & 0x0F0F0F0Fu, a[i], sumi);
        sumi = xf_dp4a((w >> 4) & 0x0F0F0F0Fu, a[i + 4], sumi);
    }
    sumi -= 8 * (int)A.bs[u];
    return (float)sumi * (xf_h2f((uint16_t)xf_ld16(row + nb * 16 + u * 2)) * A.d[u]);
}
// Q4_1 native {d, m, qs[16]} 20 B (ggml-cpu/quants.c:152-186: (d_x*d_y)*sumi + m_x*s_y)
template <> XF_HD float xf_sub_dot<XF_Q4_1>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const uint8_t * b = row + u * 20;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    const uint32_t dm = xf_ld32(b);
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld32(b + 4 + 4 * i);
        sumi = xf_dp4a(w & 0x0F0F0F0Fu, a[i], sumi);
        sumi = xf_dp4a((w >> 4) & 0x0F0F0F0Fu, a[i + 4], sumi);
    }
    return (xf_h2f((uint16_t)(dm & 0xffff)) * A.d[u]) * (float)sumi + xf_h2f((uint16_t)(dm >> 16)) * A.s[u];
}
// Q5_0, library layout [qs 16B x nb][qh 4B x nb][d f16 x nb]  (ggml-cpu/quants.c:219-260: values - 16)
template <> XF_HD float xf_sub_dot<XF_Q5_0>(const uint8_t * row, int64_t nb, int64_t u, const XfAct & A) {
    const uint8_t * qs = row + u * 16;
    const uint32_t qh = xf_ld32(row + nb * 16 + u * 4);
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld32(qs + 4 * i);
        sumi = xf_dp4a((w & 0x0F0F0F0Fu) | xf_spread4((qh >> (4 * i)) & 0xF, 4), a[i], sumi);
        sumi = xf_dp4a(((w >> 4) & 0x0F0F0F0Fu) | xf_spread4((qh >> (16 + 4 * i)) & 0xF, 4), a[i + 4], sumi);
    }
    sumi -= 16 * (int)A.bs[u];
    return (xf_h2f((uint16_t)xf_ld16(row + nb * 20 + u * 2)) * A.d[u]) * (float)sumi;
}
// Q5_1 native {d, m, qh[4], qs[16]} 24 B (ggml-cpu/quants.c:262-303)
template <> XF_HD float xf_sub_dot<XF_Q5_1>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const uint8_t * b = row + u * 24;
    const uint32_t dm = xf_ld32(b), qh = xf_ld32(b + 4);
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld32(b + 8 + 4 * i);
        sumi = xf_dp4a((w & 0x0F0F0F0Fu) | xf_spread4((qh >> (4 * i)) & 0xF, 4), a[i], sumi);
        sumi = xf_dp4a(((w >> 4) & 0x0F0F0F0Fu) | xf_spread4((qh >> (16 + 4 * i)) & 0xF, 4), a[i + 4], sumi);
    }
    return (xf_h2f((uint16_t)(dm & 0xffff)) * A.d[u]) * (float)sumi + xf_h2f((uint16_t)(dm >> 16)) * A.s[u];
}
// Q8_0, library layout [qs 32B x nb][d f16 x nb]  (ggml-cpu/quants.c:305-333)
template <> XF_HD float xf_sub_dot<XF_Q8_0>(const uint8_t * row, int64_t nb, int64_t u, const XfAct & A) {
    const uint8_t * qs = row + u * 32;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int sumi = 0;
    for (int i = 0; i < 8; i++) sumi = xf_dp4a(xf_ld32(qs + 4 * i), a[i], sumi);
    return (float)sumi * (xf_h2f((uint16_t)xf_ld16(row + nb * 32 + u * 2)) * A.d[u]);
}
// IQ4_NL native {d, qs[16]} 18 B (ggml-cpu/quants.c:1108-1135)
template <> XF_HD float xf_sub_dot<XF_IQ4_NL>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const uint8_t * b = row + u * 18;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld16x2(b + 2 + 4 * i);
        sumi = xf_dp4a(xf_lut4<false>(w & 0x0F0F0F0Fu), a[i], sumi);
        sumi = xf_dp4a(xf_lut4<false>((w >> 4) & 0x0F0F0F0Fu), a[i + 4], sumi);
    }
    return (A.d[u] * xf_h2f((uint16_t)xf_ld16(b))) * (float)sumi;
}
// MXFP4 native {e, qs[16]} 17 B (ggml-cpu/quants.c:188-217)
template <> XF_HD float xf_sub_dot<XF_MXFP4>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const uint8_t * b = row + u * 17;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld8x4(b + 1 + 4 * i);
        sumi = xf_dp4a(xf_lut4<true>(w & 0x0F0F0F0Fu), a[i], sumi);
        sumi = xf_dp4a(xf_lut4<true>((w >> 4) & 0x0F0F0F0Fu), a[i + 4], sumi);
    }
    return (A.d[u] * xf_e8m0_half(b[0])) * (float)sumi;
}
// Q2_K native {scales[16], qs[64], d, dmin} 84 B (ggml-cpu/quants.c:419-469): sub-block s of a super-block = half n = s/4, shift 2*(s%4)
template <> XF_HD float xf_sub_dot<XF_Q2_K>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), n = s >> 2, sh = 2 * (s & 3);
    const uint8_t * b = row + sb * 84;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int i0 = 0, i1 = 0;
    for (int i = 0; i < 4; i++) {
        i0 = xf_dp4a((xf_ld32(b + 16 + 32 * n + 4 * i) >> sh) & 0x03030303u, a[i], i0);
        i1 = xf_dp4a((xf_ld32(b + 16 + 32 * n + 16 + 4 * i) >> sh) & 0x03030303u, a[i + 4], i1);
    }
    const int sc0 = b[2 * s], sc1 = b[2 * s + 1];
    const int isum  = (sc0 & 0xF) * i0 + (sc1 & 0xF) * i1;
    const int summs = (int)A.bs[2 * u] * (sc0 >> 4) + (int)A.bs[2 * u + 1] * (sc1 >> 4);
    const uint32_t dm = xf_ld32(b + 80);
    const float yd = A.d[sb];
    return (yd * xf_h2f((uint16_t)(dm & 0xffff))) * (float)isum - (yd * xf_h2f((uint16_t)(dm >> 16))) * (float)summs;
}
// Q3_K native {hmask[32], qs[64], scales[12], d} 110 B (ggml-cpu/quants.c:471-548): value = 2 low bits + 4 * hmask bit s, minus 4
template <> XF_HD float xf_sub_dot<XF_Q3_K>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), n = s >> 2, sh = 2 * (s & 3);
    const uint8_t * b = row + sb * 110;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int i0 = 0, i1 = 0;
    for (int i = 0; i < 8; i++) {
        const uint32_t lo = (xf_ld16x2(b + 32 + 32 * n + 4 * i) >> sh) & 0x03030303u;
        const uint32_t hb = (xf_ld16x2(b + 4 * i) >> s) & 0x01010101u;
        if (i < 4) i0 = xf_dp4a(lo | (hb << 2), a[i], i0); else i1 = xf_dp4a(lo | (hb << 2), a[i], i1);
    }
    i0 -= 4 * (int)A.bs[2 * u]; i1 -= 4 * (int)A.bs[2 * u + 1];
    const int isum = xf_q3k_scale(b + 96, 2 * s) * i0 + xf_q3k_scale(b + 96, 2 * s + 1) * i1;
    return (xf_h2f((uint16_t)xf_ld16(b + 108)) * A.d[sb]) * (float)isum;
}
// Q4_K native {d, dmin, scales[12], qs[128]} 144 B (ggml-cpu/quants.c:550-623)
template <> XF_HD float xf_sub_dot<XF_Q4_K>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), j = s >> 1, sh = 4 * (s & 1);
    const uint8_t * b = row + sb * 144;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int isum = 0;
    for (int i = 0; i < 8; i++) isum = xf_dp4a((xf_ld32(b + 16 + 32 * j + 4 * i) >> sh) & 0x0F0F0F0Fu, a[i], isum);
    int sc, mn; xf_scale_min_k4(s, b + 4, &sc, &mn);
    const uint32_t dm = xf_ld32(b);
    const float yd = A.d[sb];
    return (yd * xf_h2f((uint16_t)(dm & 0xffff))) * (float)(sc * isum) - (yd * xf_h2f((uint16_t)(dm >> 16))) * (float)(mn * ((int)A.bs[2 * u] + (int)A.bs[2 * u + 1]));
}
// Q5_K native {d, dmin, scales[12], qh[32], qs[128]} 176 B (ggml-cpu/quants.c:625-703)
template <> XF_HD float xf_sub_dot<XF_Q5_K>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), j = s >> 1, sh = 4 * (s & 1);
    const uint8_t * b = row + sb * 176;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int isum = 0;
    for (int i = 0; i < 8; i++) {
        const uint32_t lo = (xf_ld32(b + 48 + 32 * j + 4 * i) >> sh) & 0x0F0F0F0Fu;
        const uint32_t hb = (xf_ld32(b + 16 + 4 * i) >> s) & 0x01010101u;
        isum = xf_dp4a(lo | (hb << 4), a[i], isum);
    }
    int sc, mn; xf_scale_min_k4(s, b + 4, &sc, &mn);
    const uint32_t dm = xf_ld32(b);
    const float yd = A.d[sb];
    return (yd * xf_h2f((uint16_t)(dm & 0xffff))) * (float)(sc * isum) - (yd * xf_h2f((uint16_t)(dm >> 16))) * (float)(mn * ((int)A.bs[2 * u] + (int)A.bs[2 * u + 1]));
}
// Q6_K, library layout [ql 128B x nb][qh 64B x nb][scales 16B x nb][d f16 x nb]  (ggml-cpu/quants.c:705-758; ggml-quants.c dequantize_row_q6_K)
template <> XF_HD float xf_sub_dot<XF_Q6_K>(const uint8_t * row, int64_t nb, int64_t u, const XfAct & A) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), n = s >> 2, j = s & 3;
    const uint8_t * ql = row + sb * 128 + 64 * n + 32 * (j & 1);
    const uint8_t * qh = row + nb * 128 + sb * 64 + 32 * n;
    const int8_t  * sc = (const int8_t *)(row + nb * 192 + sb * 16 + 8 * n + 2 * j);
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    int i0 = 0, i1 = 0;
    for (int i = 0; i < 8; i++) {
        const uint32_t lo = (xf_ld32(ql + 4 * i) >> (j >= 2 ? 4 : 0)) & 0x0F0F0F0Fu;
        const uint32_t hi = (xf_ld32(qh + 4 * i) >> (2 * j)) & 0x03030303u;
        if (i < 4) i0 = xf_dp4a(lo | (hi << 4), a[i], i0); else i1 = xf_dp4a(lo | (hi << 4), a[i], i1);
    }
    i0 -= 32 * (int)A.bs[2 * u]; i1 -= 32 * (int)A.bs[2 * u + 1];
    return (xf_h2f((uint16_t)xf_ld16(row + nb * 208 + sb * 2)) * A.d[sb]) * (float)((int)sc[0] * i0 + (int)sc[1] * i1);
}
// IQ4_XS native {d, scales_h, scales_l[4], qs[128]} 136 B (ggml-cpu/quants.c:1137-1183)
template <> XF_HD float xf_sub_dot<XF_IQ4_XS>(const uint8_t * row, int64_t, int64_t u, const XfAct & A) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7);
    const uint8_t * b = row + sb * 136;
    const uint32_t * a = (const uint32_t *)(A.qs + u * 32);
    const uint32_t hd = xf_ld32(b);                                           // d | scales_h << 16
    const int ls = (int)((b[4 + (s >> 1)] >> (4 * (s & 1))) & 0xF) | (int)((((hd >> 16) >> (2 * s)) & 3) << 4);    // xf_iq4xs_ls written out (the call reorders this kernel's registers)
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld32(b + 8 + 16 * s + 4 * i);
        sumi = xf_dp4a(xf_lut4<false>(w & 0x0F0F0F0Fu), a[i], sumi);
        sumi = xf_dp4a(xf_lut4<false>((w >> 4) & 0x0F0F0F0Fu), a[i + 4], sumi);
    }
    return ((xf_h2f((uint16_t)(hd & 0xffff)) * A.d[sb]) * (float)(ls - 32)) * (float)sumi;
}

// =========================================================================================================================
// xf_sub_dequant<T>: the 32 values of sub-block u as f32 (ggml-quants.c dequantize_row_*), products rounded separately
// (no fused multiply-add) like the reference's scalar code.
// =========================================================================================================================
XF_HD float xf_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    volatile float r = a * b; return r;
#endif
}
XF_HD float xf_sub(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    volatile float r = a - b; return r;
#endif
}
XF_HD float xf_add(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    volatile float r = a + b; return r;
#endif
}

template <int T> XF_HD void xf_sub_dequant(const uint8_t * row, int64_t nb, int64_t u, float * y);

template <> XF_HD void xf_sub_dequant<XF_Q4_0>(const uint8_t * row, int64_t nb, int64_t u, float * y) {
    const uint8_t * qs = row + u * 16; const float d = xf_h2f((uint16_t)xf_ld16(row + nb * 16 + u * 2));
    for (int j = 0; j < 16; j++) { y[j] = xf_mul((float)((int)(qs[j] & 0xF) - 8), d); y[j + 16] = xf_mul((float)((int)(qs[j] >> 4) - 8), d); }
}
template <> XF_HD void xf_sub_dequant<XF_Q4_1>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const uint8_t * b = row + u * 20; const float d = xf_h2f((uint16_t)xf_ld16(b)), m = xf_h2f((uint16_t)xf_ld16(b + 2));
    for (int j = 0; j < 16; j++) { y[j] = xf_add(xf_mul((float)(b[4 + j] & 0xF), d), m); y[j + 16] = xf_add(xf_mul((float)(b[4 + j] >> 4), d), m); }
}
template <> XF_HD void xf_sub_dequant<XF_Q5_0>(const uint8_t * row, int64_t nb, int64_t u, float * y) {
    const uint8_t * qs = row + u * 16; const uint32_t qh = xf_ld32(row + nb * 16 + u * 4); const float d = xf_h2f((uint16_t)xf_ld16(row + nb * 20 + u * 2));
    for (int j = 0; j < 16; j++) {
        y[j]      = xf_mul((float)((int)((qs[j] & 0xF) | (((qh >> j) & 1) << 4)) - 16), d);
        y[j + 16] = xf_mul((float)((int)((qs[j] >> 4) | (((qh >> (j + 16)) & 1) << 4)) - 16), d);
    }
}
template <> XF_HD void xf_sub_dequant<XF_Q5_1>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const uint8_t * b = row + u * 24; const float d = xf_h2f((uint16_t)xf_ld16(b)), m = xf_h2f((uint16_t)xf_ld16(b + 2)); const uint32_t qh = xf_ld32(b + 4);
    for (int j = 0; j < 16; j++) {
        y[j]      = xf_add(xf_mul((float)((b[8 + j] & 0xF) | (((qh >> j) & 1) << 4)), d), m);
        y[j + 16] = xf_add(xf_mul((float)((b[8 + j] >> 4) | (((qh >> (j + 16)) & 1) << 4)), d), m);
    }
}
template <> XF_HD void xf_sub_dequant<XF_Q8_0>(const uint8_t * row, int64_t nb, int64_t u, float * y) {
    const int8_t * qs = (const int8_t *)(row + u * 32); const float d = xf_h2f((uint16_t)xf_ld16(row + nb * 32 + u * 2));
    for (int j = 0; j < 32; j++) y[j] = xf_mul((float)qs[j], d);
}
template <> XF_HD void xf_sub_dequant<XF_IQ4_NL>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const uint8_t * b = row + u * 18; const float d = xf_h2f((uint16_t)xf_ld16(b));
    for (int j = 0; j < 16; j++) { y[j] = xf_mul(d, (float)xf_kv_iq4nl(b[2 + j] & 0xF)); y[j + 16] = xf_mul(d, (float)xf_kv_iq4nl(b[2 + j] >> 4)); }
}
template <> XF_HD void xf_sub_dequant<XF_MXFP4>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const uint8_t * b = row + u * 17; const float d = xf_e8m0_half(b[0]);
    for (int j = 0; j < 16; j++) { y[j] = xf_mul((float)xf_kv_mxfp4(b[1 + j] & 0xF), d); y[j + 16] = xf_mul((float)xf_kv_mxfp4(b[1 + j] >> 4), d); }
}
template <> XF_HD void xf_sub_dequant<XF_Q2_K>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), n = s >> 2, sh = 2 * (s & 3);
    const uint8_t * b = row + sb * 84; const float d = xf_h2f((uint16_t)xf_ld16(b + 80)), dmin = xf_h2f((uint16_t)xf_ld16(b + 82));
    for (int h = 0; h < 2; h++) {
        const int sc = b[2 * s + h]; const float dl = xf_mul(d, (float)(sc & 0xF)), ml = xf_mul(dmin, (float)(sc >> 4));
        for (int l = 0; l < 16; l++) y[16 * h + l] = xf_sub(xf_mul(dl, (float)((b[16 + 32 * n + 16 * h + l] >> sh) & 3)), ml);
    }
}
template <> XF_HD void xf_sub_dequant<XF_Q3_K>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), n = s >> 2, sh = 2 * (s & 3);
    const uint8_t * b = row + sb * 110; const float d = xf_h2f((uint16_t)xf_ld16(b + 108));
    for (int h = 0; h < 2; h++) {
        const float dl = xf_mul(d, (float)xf_q3k_scale(b + 96, 2 * s + h));
        for (int l = 16 * h; l < 16 * h + 16; l++) y[l] = xf_mul(dl, (float)((int)((b[32 + 32 * n + l] >> sh) & 3) - (((b[l] >> s) & 1) ? 0 : 4)));
    }
}
template <> XF_HD void xf_sub_dequant<XF_Q4_K>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), j = s >> 1, sh = 4 * (s & 1);
    const uint8_t * b = row + sb * 144; const float d = xf_h2f((uint16_t)xf_ld16(b)), dmin = xf_h2f((uint16_t)xf_ld16(b + 2));
    int sc, mn; xf_scale_min_k4(s, b + 4, &sc, &mn);
    const float d1 = xf_mul(d, (float)sc), m1 = xf_mul(dmin, (float)mn);
    for (int l = 0; l < 32; l++) y[l] = xf_sub(xf_mul(d1, (float)((b[16 + 32 * j + l] >> sh) & 0xF)), m1);
}
template <> XF_HD void xf_sub_dequant<XF_Q5_K>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), j = s >> 1, sh = 4 * (s & 1);
    const uint8_t * b = row + sb * 176; const float d = xf_h2f((uint16_t)xf_ld16(b)), dmin = xf_h2f((uint16_t)xf_ld16(b + 2));
    int sc, mn; xf_scale_min_k4(s, b + 4, &sc, &mn);
    const float d1 = xf_mul(d, (float)sc), m1 = xf_mul(dmin, (float)mn);
    for (int l = 0; l < 32; l++) y[l] = xf_sub(xf_mul(d1, (float)(((b[48 + 32 * j + l] >> sh) & 0xF) + (((b[16 + l] >> s) & 1) ? 16 : 0))), m1);
}
template <> XF_HD void xf_sub_dequant<XF_Q6_K>(const uint8_t * row, int64_t nb, int64_t u, float * y) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7), n = s >> 2, j = s & 3;
    const uint8_t * ql = row + sb * 128 + 64 * n + 32 * (j & 1);
    const uint8_t * qh = row + nb * 128 + sb * 64 + 32 * n;
    const int8_t  * sc = (const int8_t *)(row + nb * 192 + sb * 16 + 8 * n + 2 * j);
    const float d = xf_h2f((uint16_t)xf_ld16(row + nb * 208 + sb * 2));
    for (int l = 0; l < 32; l++) {
        const int q = (int)(((ql[l] >> (j >= 2 ? 4 : 0)) & 0xF) | (((qh[l] >> (2 * j)) & 3) << 4)) - 32;
        y[l] = xf_mul(xf_mul(d, (float)sc[l >> 4]), (float)q);
    }
}
template <> XF_HD void xf_sub_dequant<XF_IQ4_XS>(const uint8_t * row, int64_t, int64_t u, float * y) {
    const int64_t sb = u >> 3; const int s = (int)(u & 7);
    const uint8_t * b = row + sb * 136; const float d = xf_h2f((uint16_t)xf_ld16(b)); const uint32_t sh = xf_ld16(b + 2);
    const int ls = xf_iq4xs_ls(b[4 + (s >> 1)], sh, s);
    const float dl = xf_mul(d, (float)(ls - 32));
    for (int jj = 0; jj < 16; jj++) { y[jj] = xf_mul(dl, (float)xf_kv_iq4nl(b[8 + 16 * s + jj] & 0xF)); y[jj + 16] = xf_mul(dl, (float)xf_kv_iq4nl(b[8 + 16 * s + jj] >> 4)); }
}

// =========================================================================================================================
// Q4_0 in ggml's NATIVE block layout {d f16, qs[16]} — the KV cache type q4_0 (caches keep ggml's layout so that llama.cpp's state
// save / restore and defragmentation see what they expect).
// =========================================================================================================================
// f32 -> one block, as ggml's from_float writes it (ggml-quants.c quantize_row_q4_0_ref): the element of largest magnitude (first on
// ties) maps to -8; (int8_t)(x*id + 8.5f) truncated, clamped to 15.  blk 2-byte aligned.
XF_HD void xf_q4_0_quantize_block(const float * x, uint8_t * blk) {
    float amax = 0.0f, mx = 0.0f;
    for (int j = 0; j < 32; j++) { const float v = x[j]; const float av = v < 0.0f ? -v : v; if (amax < av) { amax = av; mx = v; } }
    const float d = mx / -8.0f;
    const float id = d != 0.0f ? 1.0f / d : 0.0f;
    // f32 -> f16 round-to-nearest-even, bit-level (== ggml's GGML_FP32_TO_FP16 / F16C)
    uint32_t fb; memcpy(&fb, &d, 4);
    const uint32_t sign = (fb >> 16) & 0x8000u; fb &= 0x7fffffffu;
    uint32_t hb;
    if (fb >= 0x7f800000u) hb = fb > 0x7f800000u ? 0x7e00u : 0x7c00u;
    else if (fb >= 0x477ff000u) hb = 0x7c00u;                                  // rounds to infinity
    else if (fb >= 0x38800000u) {                                              // normal half
        const uint32_t mant = fb & 0x7fffffu, e = (fb >> 23) - 112;
        hb = (e << 10) | (mant >> 13);
        const uint32_t rem = mant & 0x1fffu;
        if (rem > 0x1000u || (rem == 0x1000u && (hb & 1))) hb++;
    } else if (fb >= 0x33000000u) {                                            // subnormal half
        const uint32_t mant = (fb & 0x7fffffu) | 0x800000u; const int shift = 126 - (int)(fb >> 23);   // 14..24
        hb = mant >> shift;
        const uint32_t rem = mant & ((1u << shift) - 1), half = 1u << (shift - 1);
        if (rem > half || (rem == half && (hb & 1))) hb++;
    } else hb = 0;
    hb |= sign;
    blk[0] = (uint8_t)(hb & 0xff); blk[1] = (uint8_t)(hb >> 8);
    for (int j = 0; j < 16; j++) {
        int q0 = (int)(int8_t)xf_add(xf_mul(x[j], id), 8.5f), q1 = (int)(int8_t)xf_add(xf_mul(x[16 + j], id), 8.5f);
        if (q0 > 15) q0 = 15;
        if (q1 > 15) q1 = 15;
        blk[2 + j] = (uint8_t)(q0 | (q1 << 4));
    }
}
// (sum (nib - 8) * q8) * d_k * d_q for one native block against 32 int8 of the q8_0 form of the query (ggml-cpu/quants.c:115-149)
XF_HD float xf_q4_0n_dot(const uint8_t * blk, const int8_t * q8, float ad, int bs) {
    const uint32_t * a = (const uint32_t *)q8;
    int sumi = 0;
    for (int i = 0; i < 4; i++) {
        const uint32_t w = xf_ld16x2(blk + 2 + 4 * i);
        sumi = xf_dp4a(w & 0x0F0F0F0Fu, a[i], sumi);
        sumi = xf_dp4a((w >> 4) & 0x0F0F0F0Fu, a[i + 4], sumi);
    }
    sumi -= 8 * bs;
    return (float)sumi * (xf_h2f((uint16_t)xf_ld16(blk)) * ad);
}
// element e (0..31) of a native block as f32 (ggml-quants.c dequantize_row_q4_0)
XF_HD float xf_q4_0n_value(const uint8_t * blk, int e) {
    const int nib = e < 16 ? (blk[2 + e] & 0xF) : (blk[2 + e - 16] >> 4);
    return xf_mul((float)(nib - 8), xf_h2f((uint16_t)xf_ld16(blk)));
}

// Q8_0 in ggml's native block layout {d f16, qs[32]} (the KV cache type q8_0), for the any-head-size attention kernel (fattn_ext_kernels.cuh)
XF_HD float xf_q8_0n_dot(const uint8_t * blk, const int8_t * q8, float ad) {          // ggml-cpu/quants.c:305-333
    const uint32_t * a = (const uint32_t *)q8;
    int sumi = 0;
    for (int i = 0; i < 8; i++) sumi = xf_dp4a(xf_ld16x2(blk + 2 + 4 * i), a[i], sumi);
    return (float)sumi * (xf_h2f((uint16_t)xf_ld16(blk)) * ad);
}
XF_HD float xf_q8_0n_value(const uint8_t * blk, int e) { return xf_mul((float)(int8_t)blk[2 + e], xf_h2f((uint16_t)xf_ld16(blk))); }

// run F<T>(args...) for a runtime type id; false when the type is not one of ours
#define XF_DISPATCH(t, CALL) \
    switch (t) { \
        case XF_Q4_0:  { constexpr int T = XF_Q4_0;  CALL; } break;  case XF_Q4_1:  { constexpr int T = XF_Q4_1;  CALL; } break; \
        case XF_Q5_0:  { constexpr int T = XF_Q5_0;  CALL; } break;  case XF_Q5_1:  { constexpr int T = XF_Q5_1;  CALL; } break; \
        case XF_Q8_0:  { constexpr int T = XF_Q8_0;  CALL; } break;  case XF_Q2_K:  { constexpr int T = XF_Q2_K;  CALL; } break; \
        case XF_Q3_K:  { constexpr int T = XF_Q3_K;  CALL; } break;  case XF_Q4_K:  { constexpr int T = XF_Q4_K;  CALL; } break; \
        case XF_Q5_K:  { constexpr int T = XF_Q5_K;  CALL; } break;  case XF_Q6_K:  { constexpr int T = XF_Q6_K;  CALL; } break; \
        case XF_IQ4_NL:{ constexpr int T = XF_IQ4_NL;CALL; } break;  case XF_IQ4_XS:{ constexpr int T = XF_IQ4_XS;CALL; } break; \
        case XF_MXFP4: { constexpr int T = XF_MXFP4; CALL; } break;  default: break; \
    }
