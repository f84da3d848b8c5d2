// mmvq.cu — decode matvec on GGUF-quantised weights (sm_90a), ncols <= 8.
//
// Replaces ggml_cuda_mul_mat_vec_q / mul_mat_vec_q<type,ncols_dst> (ggml-cuda/mmvq.cu:139-226,
// 500-570) and vec_dot_q*_q8_1 (vecdotq.cuh:579-839).  Design (HBM-bound; bytes = m * row_bytes):
//   * ONE persistent CTA per SM (16 warps).  Every warp runs its own TMA pipeline: lane 0 issues
//     1-D bulk async copies (cp.async.bulk, mbarrier complete_tx) of the next row-pair segments of the
//     weight matrix into a private shared-memory ring, so the bytes in flight per SM are set by the
//     ring size (~128 KB), not by registers or occupancy — that is what saturates HBM3e.  The
//     reference instead issues 2-/4-byte LDGs from 128-thread blocks, one row per block.
//   * weights never depend on the previous kernel, so the ring is primed BEFORE griddepcontrol.wait:
//     under programmatic dependent launch the weight stream of this matvec starts while the previous
//     kernel is still draining.  Only then is the quantised activation vector staged (one bulk copy
//     per CTA) and consumed with conflict-free LDS.128.
//   * activations are quantised like the CPU oracle (q8_K / RNE q8_0), so per-block integer sums
//     equal the oracle's bit for bit (ggml-cpu/quants.c:115-149,305-333,550-758);
//   * a warp owns TWO rows at a time (activation registers reused); several matrices (QKV, gate+up)
//     share a launch; epilogues fused: bias, residual add, SwiGLU (gate row x up row).
// Rows of Q4_0/Q8_0/Q6_K are repacked at load time so every part of a segment is 16-byte aligned
// (repack.cu); Q4_K/Q5_K keep the GGUF layout.
#include "common.cuh"
#include "actquant.cuh"

#ifndef MMV_WARPS
#define MMV_WARPS 16
#endif
#ifndef MMV_CTAS_PER_SM
#define MMV_CTAS_PER_SM 1      // one CTA of 16 warps per SM: the whole warp count keeps the bulk copies of the ring in flight
#endif
#define MMV_MAX_MATS 4
#define MMV_MAX_STAGES 8

enum { MMV_MODE_PLAIN = 0, MMV_MODE_SWIGLU = 1 };

struct MmvMat {
    const uint8_t * W;
    float *         dst;
    const float *   bias;
    const float *   residual;
    int64_t         m;
    int64_t         dst_col_stride;
    int64_t         rb;         // bytes per row
    int32_t         nb;         // blocks per row
    int32_t         type;
    int32_t         pair0;      // first unit index of this matrix in the launch
    int32_t         _pad;
};
struct MmvArgs {
    MmvMat  mat[MMV_MAX_MATS];
    const uint8_t * act[2];     // [kind]: 0 = q8_K act buffer, 1 = q8_0 act buffer (may be null)
    int64_t k;
    int32_t n_mats;
    int32_t total_pairs;
    int32_t act_bytes[2];       // bytes to stage per kind (ncols * col_bytes), 0 if unused
    int32_t segc;               // chunks (32 elements) per compute segment (64 = fast paths)
    int32_t nseg;               // segments per row
    int32_t stages;             // ring depth per warp
    int32_t slot_bytes;         // bytes of one ring slot: R whole rows of the widest type in the launch
    int32_t rows_per_unit;      // R: 1 or 2 (SwiGLU: one gate row + one up row)
    int32_t segs_per_part;      // G: a unit is split into K-parts of G segments so that >= 2 ring slots fit per warp
    int32_t parts;              // P = ceil(nseg / G)
    int32_t row_stride;         // byte distance between the two rows inside a slot
    // activation source: 0 = quantised act buffers (bulk copy), 1 = f32 x quantised in the prologue,
    // 2 = f32 x with RMS norm * norm_w, then quantised (fuses rms_norm + mul + quantize into this kernel)
    int32_t act_source;
    int32_t ncols;
    const float * x;            // [ncols][x_col_stride]
    const float * norm_w;       // [k] or null
    float *       y_out;        // optional f32 copy of the (normalised) activations, written by CTA 0
    int64_t       x_col_stride;
    float         eps;
    int32_t       trace;      // B200_TRACE: CTA 0 and the last CTA record a timeline (common.cuh)
    int64_t       k_valid;      // elements that exist in x per column (<= k; the rest of the padded weight rows are zero blocks)
};

B200_TRACE_DECL(g_mmv_trace)

// ---- activation view in shared memory --------------------------------------------------------
struct ActView { const uint8_t * qs; const float * d; const int16_t * bs; };

__device__ __forceinline__ int dot16(const uint4 & a, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    int s = dp4a_us(w0, (int)a.x, 0);
    s = dp4a_us(w1, (int)a.y, s);
    s = dp4a_us(w2, (int)a.z, s);
    return dp4a_us(w3, (int)a.w, s);
}
__device__ __forceinline__ int dot16s(const uint4 & a, const uint4 & w) {
    int s = dp4a_s((int)w.x, (int)a.x, 0);
    s = dp4a_s((int)w.y, (int)a.y, s);
    s = dp4a_s((int)w.z, (int)a.z, s);
    return dp4a_s((int)w.w, (int)a.w, s);
}

__device__ __forceinline__ int dp4a_u8s8(uint32_t w, uint32_t a, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(w), "r"(a), "r"(c));
    return d;
}
__device__ __forceinline__ int dot16m(const uint4 & a, const uint4 & w, uint32_t m) {
    int s = dp4a_u8s8(w.x & m, a.x, 0);
    s = dp4a_u8s8(w.y & m, a.y, s);
    s = dp4a_u8s8(w.z & m, a.z, s);
    return dp4a_u8s8(w.w & m, a.w, s);
}
__device__ __forceinline__ int byte_of(uint32_t w, int sh8) { return (int)__byte_perm(w, 0, 0x4440 | (sh8 >> 3)); }   // one PRMT


// 6-bit scale / min of sub-block `is` from the q4_K/q5_K header regs (ggml-quants.c:703-711)
__device__ __forceinline__ void k4_scale_min(const uint4 & hdr, int is, int & sc, int & mn) {
    const int e = (is & 3) * 8;
    const int sc_lo = (hdr.y >> e) & 63, mn_lo = (hdr.z >> e) & 63;
    const int sc_hi = ((hdr.w >> e) & 15) | (((hdr.y >> (e + 6)) & 3) << 4);
    const int mn_hi = ((hdr.w >> (e + 4)) & 15) | (((hdr.z >> (e + 6)) & 3) << 4);
    sc = is < 4 ? sc_lo : sc_hi;
    mn = is < 4 ? mn_lo : mn_hi;
}

// ---- one 32-element chunk: weights from the ring slot (local chunk lc), activations chunk i -----
// Each lane handles 32 elements as two 16-element parts; the order in which the two parts are read
// from the activation vector is swapped on half of the lanes of every quarter-warp so that each
// LDS.128 touches 8 distinct 16-byte bank groups (no conflicts).
template <int T> struct WChunk;

template <> struct WChunk<B200_TYPE_Q4_0> {
    uint4 qs; uint16_t d;
    __device__ __forceinline__ void load(const uint8_t * s, int nb, int i) { qs = *(const uint4 *)(s + i * 16); d = *(const uint16_t *)(s + nb * 16 + i * 2); }
    __device__ __forceinline__ float dot(const ActView & a, int i) const {
        const int sw = (i >> 2) & 1;
        const uint4 A = *(const uint4 *)(a.qs + i * 32 + sw * 16);
        const uint4 B = *(const uint4 *)(a.qs + i * 32 + (sw ^ 1) * 16);
        // low nibbles <-> elements 0..15; high nibbles stay in place: u8 x s8 dp4a on (q & 0xF0), sum >> 4
        const uint32_t mA = sw ? 0xF0F0F0F0u : 0x0F0F0F0Fu;
        int s = (dot16m(A, qs, mA) >> (sw * 4)) + (dot16m(B, qs, ~mA) >> (4 - sw * 4));
        s -= 8 * (int)a.bs[i];
        return __fmul_rn(__fmul_rn((float)s, h2f(d)), a.d[i]);          // ggml-cpu/quants.c:146
    }
};
// 5-bit: low / high nibbles as in Q4_0 plus a fifth bit from qh (bit j -> element j, ggml-quants.c dequantize_row_q5_0); value q - 16
__device__ __forceinline__ uint32_t spread4(uint32_t b) { return (((b & 0xFu) * 0x00204081u) & 0x01010101u) << 4; }   // 4 bits -> bit 4 of 4 bytes
template <> struct WChunk<B200_TYPE_Q5_0> {
    uint4 qs; uint32_t qh; uint16_t d;
    __device__ __forceinline__ void load(const uint8_t * s, int nb, int i) {
        qs = *(const uint4 *)(s + i * 16); qh = *(const uint32_t *)(s + nb * 16 + i * 4); d = *(const uint16_t *)(s + nb * 20 + i * 2);
    }
    __device__ __forceinline__ float dot(const ActView & a, int i) const {
        const int sw = (i >> 2) & 1;
        const uint4 A = *(const uint4 *)(a.qs + i * 32 + sw * 16);           // the two 16-element halves, read in lane-dependent order (bank conflicts)
        const uint4 B = *(const uint4 *)(a.qs + i * 32 + (sw ^ 1) * 16);
        const uint4 lo = sw ? B : A, hi = sw ? A : B;                        // lo: elements 0..15, hi: 16..31
        const uint32_t w[4] = { qs.x, qs.y, qs.z, qs.w };
        const uint32_t al[4] = { lo.x, lo.y, lo.z, lo.w }, ah[4] = { hi.x, hi.y, hi.z, hi.w };
        int s = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            s = dp4a_us((w[j] & 0x0F0F0F0Fu) | spread4(qh >> (4 * j)), (int)al[j], s);
            s = dp4a_us(((w[j] >> 4) & 0x0F0F0F0Fu) | spread4(qh >> (16 + 4 * j)), (int)ah[j], s);
        }
        s -= 16 * (int)a.bs[i];
        return __fmul_rn(__fmul_rn(h2f(d), a.d[i]), (float)s);              // (d_w * d_x) * sumi, ggml-cpu/quants.c ggml_vec_dot_q5_0_q8_0
    }
};
template <> struct WChunk<B200_TYPE_Q8_0> {
    uint4 q0, q1; uint16_t d;
    __device__ __forceinline__ void load(const uint8_t * s, int nb, int i) {
        q0 = *(const uint4 *)(s + i * 32); q1 = *(const uint4 *)(s + i * 32 + 16); d = *(const uint16_t *)(s + nb * 32 + i * 2);
    }
    __device__ __forceinline__ float dot(const ActView & a, int i) const {
        const int sw = (i >> 2) & 1;
        const uint4 A = *(const uint4 *)(a.qs + i * 32 + sw * 16);
        const uint4 B = *(const uint4 *)(a.qs + i * 32 + (sw ^ 1) * 16);
        const int s = sw ? dot16s(A, q1) + dot16s(B, q0) : dot16s(A, q0) + dot16s(B, q1);
        return __fmul_rn((float)s, __fmul_rn(h2f(d), a.d[i]));           // ggml-cpu/quants.c:330
    }
};
template <> struct WChunk<B200_TYPE_Q4_K> {
    uint4 hdr, qs;
    __device__ __forceinline__ void load(const uint8_t * s, int, int i) { const uint8_t * b = s + (i >> 3) * 144; hdr = *(const uint4 *)b; qs = *(const uint4 *)(b + 16 + (i & 7) * 16); }
    __device__ __forceinline__ float dot(const ActView & a, int i) const {
        const int sb = i >> 3, j = i & 7, c = j >> 1, h = j & 1, sw = c >> 1;
        const int is0 = 2 * c + sw, is1 = 2 * c + (sw ^ 1);           // sub-block (32 elems) of each part
        const uint8_t * base = a.qs + sb * 256 + h * 16;
        const uint4 A = *(const uint4 *)(base + is0 * 32);
        const uint4 B = *(const uint4 *)(base + is1 * 32);
        const int shA = (is0 & 1) * 4, shB = (is1 & 1) * 4;
        const int sA = dot16(A, (qs.x >> shA) & 0x0F0F0F0Fu, (qs.y >> shA) & 0x0F0F0F0Fu, (qs.z >> shA) & 0x0F0F0F0Fu, (qs.w >> shA) & 0x0F0F0F0Fu);
        const int sB = dot16(B, (qs.x >> shB) & 0x0F0F0F0Fu, (qs.y >> shB) & 0x0F0F0F0Fu, (qs.z >> shB) & 0x0F0F0F0Fu, (qs.w >> shB) & 0x0F0F0F0Fu);
        int scA, mnA, scB, mnB;
        k4_scale_min(hdr, is0, scA, mnA);
        k4_scale_min(hdr, is1, scB, mnB);
        const int isum = scA * sA + scB * sB;
        const int imin = mnA * (int)a.bs[sb * 16 + is0 * 2 + h] + mnB * (int)a.bs[sb * 16 + is1 * 2 + h];
        const float da = a.d[sb];
        const float dw = h2f((uint16_t)(hdr.x & 0xffff)), dm = h2f((uint16_t)(hdr.x >> 16));
        return __fmul_rn(dw, da) * (float)isum - __fmul_rn(dm, da) * (float)imin;   // ggml-cpu/quants.c:615-620
    }
};
template <> struct WChunk<B200_TYPE_Q5_K> {
    uint4 hdr, qh, qs;
    __device__ __forceinline__ void load(const uint8_t * s, int, int i) {
        const uint8_t * b = s + (i >> 3) * 176; hdr = *(const uint4 *)b; qh = *(const uint4 *)(b + 16 + (i & 1) * 16); qs = *(const uint4 *)(b + 48 + (i & 7) * 16);
    }
    __device__ __forceinline__ float dot(const ActView & a, int i) const {
        const int sb = i >> 3, j = i & 7, c = j >> 1, h = j & 1, sw = c >> 1;
        const int is0 = 2 * c + sw, is1 = 2 * c + (sw ^ 1);
        const uint8_t * base = a.qs + sb * 256 + h * 16;
        const uint4 A = *(const uint4 *)(base + is0 * 32);
        const uint4 B = *(const uint4 *)(base + is1 * 32);
        const int shA = (is0 & 1) * 4, shB = (is1 & 1) * 4;
#define Q5W(q, hb, sh, is) ((((q) >> (sh)) & 0x0F0F0F0Fu) | ((((hb) >> (is)) & 0x01010101u) << 4))
        const int sA = dot16(A, Q5W(qs.x, qh.x, shA, is0), Q5W(qs.y, qh.y, shA, is0), Q5W(qs.z, qh.z, shA, is0), Q5W(qs.w, qh.w, shA, is0));
        const int sB = dot16(B, Q5W(qs.x, qh.x, shB, is1), Q5W(qs.y, qh.y, shB, is1), Q5W(qs.z, qh.z, shB, is1), Q5W(qs.w, qh.w, shB, is1));
#undef Q5W
        int scA, mnA, scB, mnB;
        k4_scale_min(hdr, is0, scA, mnA);
        k4_scale_min(hdr, is1, scB, mnB);
        const int isum = scA * sA + scB * sB;
        const int imin = mnA * (int)a.bs[sb * 16 + is0 * 2 + h] + mnB * (int)a.bs[sb * 16 + is1 * 2 + h];
        const float da = a.d[sb];
        const float dw = h2f((uint16_t)(hdr.x & 0xffff)), dm = h2f((uint16_t)(hdr.x >> 16));
        return __fmul_rn(dw, da) * (float)isum - __fmul_rn(dm, da) * (float)imin;
    }
};
template <> struct WChunk<B200_TYPE_Q6_K> {
    uint4 ql, qh; uint32_t sc; uint16_t d;
    __device__ __forceinline__ void load(const uint8_t * s, int nb, int i) {
        const int sb = i >> 3, j = i & 7, hh = j >> 2, ii = j & 3;
        ql = *(const uint4 *)(s + sb * 128 + hh * 64 + ii * 16);
        qh = *(const uint4 *)(s + nb * 128 + sb * 64 + hh * 32 + (ii & 1) * 16);
        const uint8_t * scp = s + nb * 192 + sb * 16 + hh * 8 + ii;     // scales 8hh+ii and 8hh+ii+4
        sc = (uint32_t)scp[0] | ((uint32_t)scp[4] << 8);
        d = *(const uint16_t *)(s + nb * 208 + sb * 2);
    }
    __device__ __forceinline__ float dot(const ActView & a, int i) const {
        const int sb = i >> 3, j = i & 7, hh = j >> 2, ii = j & 3, sw = hh;
        // part p (0: low nibbles, 1: high nibbles) covers elements 128hh + 16ii + 64p .. +15,
        // 2-bit highs at qh bit 2*(ii/2) + 4p, scale 8hh + ii + 4p
        const int p0 = sw, p1 = sw ^ 1;
        const uint8_t * base = a.qs + sb * 256 + hh * 128 + ii * 16;
        const uint4 A = *(const uint4 *)(base + p0 * 64);
        const uint4 B = *(const uint4 *)(base + p1 * 64);
        const int hs0 = (ii >> 1) * 2 + p0 * 4, hs1 = (ii >> 1) * 2 + p1 * 4;
#define Q6W(q, hb, p, hs) ((((q) >> ((p) * 4)) & 0x0F0F0F0Fu) | ((((hb) >> (hs)) & 0x03030303u) << 4))
        int sA = dot16(A, Q6W(ql.x, qh.x, p0, hs0), Q6W(ql.y, qh.y, p0, hs0), Q6W(ql.z, qh.z, p0, hs0), Q6W(ql.w, qh.w, p0, hs0));
        int sB = dot16(B, Q6W(ql.x, qh.x, p1, hs1), Q6W(ql.y, qh.y, p1, hs1), Q6W(ql.z, qh.z, p1, hs1), Q6W(ql.w, qh.w, p1, hs1));
#undef Q6W
        const int g = sb * 16 + hh * 8 + ii;                          // 16-element group of part p: g + 4p
        sA -= 32 * (int)a.bs[g + 4 * p0];
        sB -= 32 * (int)a.bs[g + 4 * p1];
        const int scA = (int)(int8_t)((sc >> (8 * p0)) & 0xff), scB = (int)(int8_t)((sc >> (8 * p1)) & 0xff);
        return __fmul_rn(h2f(d), a.d[sb]) * (float)(scA * sA + scB * sB);   // ggml-cpu/quants.c:752-754
    }
};


// ---- fast paths for 2048-element segments (segc == 64: 8 super-blocks per row segment) -------------
// The generic WChunk code above spends ~100 instructions per 32 weights (6-bit scale unpack and nibble
// shifts per chunk), which makes the matvec ISSUE-bound long before HBM is saturated.
// Here one lane owns 64 elements of ONE super-block for both rows: scales are decoded once per
// super-block with 32-bit SIMD masks (the utmp trick of ggml-cpu/quants.c:586-592), high nibbles are
// used in place through an unsigned-by-signed dp4a on (q & 0xF0F0F0F0) followed by one >>4 of the sum,
// and every bank-conflict "swap" folds into lane-constant masks / selectors.  ~40 instructions / 32 weights.
template <int NCOLS, int NR>
__device__ __forceinline__ void slot_dot_q4K_fast(const uint8_t * s0, const uint8_t * s1, int nb, int lseg, int seg, const uint8_t * act_s, int64_t k, int lane, float (&acc)[2][NCOLS]) {
    const int q = lane >> 3, s = (lane >> 2) & 1, jj = lane & 3, c = jj >> 1, h = jj & 1;
    const int sb = q + 4 * s, gsb = seg * 8 + sb, lsb = lseg * 8 + sb;     // gsb: in the row (activations), lsb: in the slot
    // "first" = the 16-element part this lane reads first (low-nibble part on s=0 lanes, high-nibble part on s=1)
    const uint32_t mF = s ? 0xF0F0F0F0u : 0x0F0F0F0Fu, mS = ~mF;
    const int shF = 4 * s, shS = 4 - shF;
    const int isF = 2 * c + s, isS = 2 * c + 1 - s;                 // sub-block ids of pass A (pass B: +4)
    const int eF = 8 * isF, eS = 8 * isS;                            // byte selectors in the decoded scale words
    uint4 hdr[2], qa[2], qb[2];
    {
        const uint8_t * b0 = s0 + lsb * 144, * b1 = s1 + lsb * 144;
        hdr[0] = *(const uint4 *)b0; qa[0] = *(const uint4 *)(b0 + 16 + jj * 16); qb[0] = *(const uint4 *)(b0 + 80 + jj * 16);
        if (NR > 1) { hdr[1] = *(const uint4 *)b1; qa[1] = *(const uint4 *)(b1 + 16 + jj * 16); qb[1] = *(const uint4 *)(b1 + 80 + jj * 16); }
    }
    int scAF[2], scAS[2], scBF[2], scBS[2], mnAF[2], mnAS[2], mnBF[2], mnBS[2]; float dw[2], dm[2];
#pragma unroll
    for (int r = 0; r < NR; r++) {
        const uint32_t y = hdr[r].y, z = hdr[r].z, w = hdr[r].w;
        const uint32_t sc03 = y & 0x3f3f3f3fu, mn03 = z & 0x3f3f3f3fu;
        const uint32_t sc47 = (w & 0x0f0f0f0fu) | (((y >> 6) & 0x03030303u) << 4);
        const uint32_t mn47 = ((w >> 4) & 0x0f0f0f0fu) | (((z >> 6) & 0x03030303u) << 4);
        scAF[r] = byte_of(sc03, eF); scAS[r] = byte_of(sc03, eS); scBF[r] = byte_of(sc47, eF); scBS[r] = byte_of(sc47, eS);
        mnAF[r] = byte_of(mn03, eF); mnAS[r] = byte_of(mn03, eS); mnBF[r] = byte_of(mn47, eF); mnBS[r] = byte_of(mn47, eS);
        dw[r] = h2f((uint16_t)(hdr[r].x & 0xffff)); dm[r] = h2f((uint16_t)(hdr[r].x >> 16));
    }
    const int64_t colb = act_col_bytes(0, k), doff = act_d_off(0, k), boff = act_bsum_off(0, k);
#pragma unroll
    for (int col = 0; col < NCOLS; col++) {
        const uint8_t * ab = act_s + col * colb;
        const uint8_t * base = ab + gsb * 256 + c * 64 + h * 16;
        const uint4 FA = *(const uint4 *)(base + 32 * s), SA = *(const uint4 *)(base + 32 - 32 * s);
        const uint4 FB = *(const uint4 *)(base + 128 + 32 * s), SB = *(const uint4 *)(base + 160 - 32 * s);
        const int16_t * bs = (const int16_t *)(ab + boff) + gsb * 16 + h;
        const int bFA = bs[isF * 2], bSA = bs[isS * 2], bFB = bs[isF * 2 + 8], bSB = bs[isS * 2 + 8];
        const float da = ((const float *)(ab + doff))[gsb];
#pragma unroll
        for (int r = 0; r < NR; r++) {
            const int dFA = dot16m(FA, qa[r], mF) >> shF, dSA = dot16m(SA, qa[r], mS) >> shS;
            const int dFB = dot16m(FB, qb[r], mF) >> shF, dSB = dot16m(SB, qb[r], mS) >> shS;
            const int isum = scAF[r] * dFA + scAS[r] * dSA + scBF[r] * dFB + scBS[r] * dSB;
            const int imin = mnAF[r] * bFA + mnAS[r] * bSA + mnBF[r] * bFB + mnBS[r] * bSB;
            acc[r][col] += __fmul_rn(dw[r], da) * (float)isum - __fmul_rn(dm[r], da) * (float)imin;
        }
    }
}

template <int NCOLS, int NR>
__device__ __forceinline__ void slot_dot_q6K_fast(const uint8_t * s0, const uint8_t * s1, int nb, int lseg, int seg, const uint8_t * act_s, int64_t k, int lane, float (&acc)[2][NCOLS]) {
    const int q = lane >> 3, s = (lane >> 2) & 1, ii = lane & 3;
    const int sb = q + 4 * s, gsb = seg * 8 + sb, lsb = lseg * 8 + sb;
    const uint32_t mF = s ? 0xF0F0F0F0u : 0x0F0F0F0Fu, mS = ~mF;
    const int shF = 4 * s, shS = 4 - shF;
    const int hsF = (ii >> 1) * 2 + 4 * s, hsS = (ii >> 1) * 2 + 4 - 4 * s;     // 2-bit highs of the first / second part
    const int eF = 8 * (ii & 3) , eS = eF;                                          // scale byte ii (+4 parts: other word)
    uint4 ql0[2], ql1[2], qh0[2], qh1[2], scv[2]; float dw[2];
#pragma unroll
    for (int r = 0; r < NR; r++) {
        const uint8_t * sr = r ? s1 : s0;
        ql0[r] = *(const uint4 *)(sr + lsb * 128 + ii * 16);
        ql1[r] = *(const uint4 *)(sr + lsb * 128 + 64 + ii * 16);
        qh0[r] = *(const uint4 *)(sr + nb * 128 + lsb * 64 + (ii & 1) * 16);
        qh1[r] = *(const uint4 *)(sr + nb * 128 + lsb * 64 + 32 + (ii & 1) * 16);
        scv[r] = *(const uint4 *)(sr + nb * 192 + lsb * 16);
        dw[r]  = h2f(*(const uint16_t *)(sr + nb * 208 + lsb * 2));
    }
    // scales (int8): half hh uses bytes 8hh + ii (low-nibble part) and 8hh + ii + 4 (high-nibble part)
    int scF0[2], scS0[2], scF1[2], scS1[2];
#pragma unroll
    for (int r = 0; r < NR; r++) {
        const uint32_t lo0 = scv[r].x, hi0 = scv[r].y, lo1 = scv[r].z, hi1 = scv[r].w;   // bytes 0-3, 4-7, 8-11, 12-15
        const int a0 = (int)(int8_t)byte_of(lo0, eF), b0 = (int)(int8_t)byte_of(hi0, eF);
        const int a1 = (int)(int8_t)byte_of(lo1, eF), b1 = (int)(int8_t)byte_of(hi1, eF);
        scF0[r] = s ? b0 : a0; scS0[r] = s ? a0 : b0; scF1[r] = s ? b1 : a1; scS1[r] = s ? a1 : b1;
    }
    (void)eS;
    const int64_t colb = act_col_bytes(0, k), doff = act_d_off(0, k), boff = act_bsum_off(0, k);
#pragma unroll
    for (int col = 0; col < NCOLS; col++) {
        const uint8_t * ab = act_s + col * colb;
        const uint8_t * base = ab + gsb * 256 + ii * 16;
        const uint4 F0 = *(const uint4 *)(base + 64 * s), S0 = *(const uint4 *)(base + 64 - 64 * s);          // half 0
        const uint4 F1 = *(const uint4 *)(base + 128 + 64 * s), S1 = *(const uint4 *)(base + 192 - 64 * s);   // half 1
        const int16_t * bs = (const int16_t *)(ab + boff) + gsb * 16 + ii;
        const int bF0 = bs[4 * s], bS0 = bs[4 - 4 * s], bF1 = bs[8 + 4 * s], bS1 = bs[12 - 4 * s];
        const float da = ((const float *)(ab + doff))[gsb];
#pragma unroll
        for (int r = 0; r < NR; r++) {
#define H2(qh, sh) dot16m_h(qh, sh)
            auto h2dot = [](const uint4 & a, const uint4 & qh, int sh) {
                int t = __dp4a((int)((qh.x >> sh) & 0x03030303u), (int)a.x, 0);
                t = __dp4a((int)((qh.y >> sh) & 0x03030303u), (int)a.y, t);
                t = __dp4a((int)((qh.z >> sh) & 0x03030303u), (int)a.z, t);
                return __dp4a((int)((qh.w >> sh) & 0x03030303u), (int)a.w, t);
            };
#undef H2
            const int vF0 = (dot16m(F0, ql0[r], mF) >> shF) + 16 * h2dot(F0, qh0[r], hsF) - 32 * bF0;
            const int vS0 = (dot16m(S0, ql0[r], mS) >> shS) + 16 * h2dot(S0, qh0[r], hsS) - 32 * bS0;
            const int vF1 = (dot16m(F1, ql1[r], mF) >> shF) + 16 * h2dot(F1, qh1[r], hsF) - 32 * bF1;
            const int vS1 = (dot16m(S1, ql1[r], mS) >> shS) + 16 * h2dot(S1, qh1[r], hsS) - 32 * bS1;
            const int isum = scF0[r] * vF0 + scS0[r] * vS0 + scF1[r] * vF1 + scS1[r] * vS1;
            acc[r][col] += __fmul_rn(dw[r], da) * (float)isum;
        }
    }
}

// both rows of a slot, all chunks of one segment, all columns
template <int T, int NCOLS, int NR>
__device__ __forceinline__ void slot_dot(const uint8_t * s0, const uint8_t * s1, int nb, int segc, int lseg, int seg, const uint8_t * act_s, int64_t k, int kind, int lane, float (&acc)[2][NCOLS]) {
    const int64_t colb = act_col_bytes(kind, k);
    const int64_t doff = act_d_off(kind, k), boff = act_bsum_off(kind, k);
#pragma unroll 2
    for (int lc = lane; lc < segc; lc += 32) {
        const int i = seg * segc + lc, li = lseg * segc + lc;      // chunk in the row (activations) / in the slot (weights)
        WChunk<T> w0, w1;
        w0.load(s0, nb, li); if (NR > 1) w1.load(s1, nb, li);
#pragma unroll
        for (int c = 0; c < NCOLS; c++) {
            ActView a;
            a.qs = act_s + c * colb;
            a.d  = (const float *)(act_s + c * colb + doff);
            a.bs = (const int16_t *)(act_s + c * colb + boff);
            acc[0][c] += w0.dot(a, i);
            if (NR > 1) acc[1][c] += w1.dot(a, i);
        }
    }
}

template <int NCOLS, int NR>
__device__ __forceinline__ void slot_one_type(int t, const uint8_t * s0, const uint8_t * s1, int nb, int segc, int lseg, int seg, const uint8_t * a0, const uint8_t * a1,
                                              int64_t k, int lane, float (&acc)[2][NCOLS]) {
    if (segc == 64 && t == B200_TYPE_Q4_K) { slot_dot_q4K_fast<NCOLS, NR>(s0, s1, nb, lseg, seg, a0, k, lane, acc); return; }
    if (segc == 64 && t == B200_TYPE_Q6_K) { slot_dot_q6K_fast<NCOLS, NR>(s0, s1, nb, lseg, seg, a0, k, lane, acc); return; }
    switch (t) {
        case B200_TYPE_Q4_K: slot_dot<B200_TYPE_Q4_K, NCOLS, NR>(s0, s1, nb, segc, lseg, seg, a0, k, 0, lane, acc); break;
        case B200_TYPE_Q5_K: slot_dot<B200_TYPE_Q5_K, NCOLS, NR>(s0, s1, nb, segc, lseg, seg, a0, k, 0, lane, acc); break;
        case B200_TYPE_Q6_K: slot_dot<B200_TYPE_Q6_K, NCOLS, NR>(s0, s1, nb, segc, lseg, seg, a0, k, 0, lane, acc); break;
        case B200_TYPE_Q4_0: slot_dot<B200_TYPE_Q4_0, NCOLS, NR>(s0, s1, nb, segc, lseg, seg, a1, k, 1, lane, acc); break;
        case B200_TYPE_Q5_0: slot_dot<B200_TYPE_Q5_0, NCOLS, NR>(s0, s1, nb, segc, lseg, seg, a1, k, 1, lane, acc); break;
        default:             slot_dot<B200_TYPE_Q8_0, NCOLS, NR>(s0, s1, nb, segc, lseg, seg, a1, k, 1, lane, acc); break;
    }
}

// rows s0 (type t0, nb0) and s1 (type t1, nb1); TT >= 0: the launch is uniform in that type
template <int NCOLS, int TT, int NR>
__device__ __forceinline__ void slot_dispatch(int t0, int t1, const uint8_t * s0, const uint8_t * s1, int nb0, int nb1, int segc, int lseg, int seg,
                                              const uint8_t * a0, const uint8_t * a1, int64_t k, int lane, float (&acc)[2][NCOLS]) {
    if (TT >= 0) {
        if (segc == 64 && TT == B200_TYPE_Q4_K) { slot_dot_q4K_fast<NCOLS, NR>(s0, s1, nb0, lseg, seg, a0, k, lane, acc); return; }
        if (segc == 64 && TT == B200_TYPE_Q6_K) { slot_dot_q6K_fast<NCOLS, NR>(s0, s1, nb0, lseg, seg, a0, k, lane, acc); return; }
        switch (TT) {
            case B200_TYPE_Q4_K: slot_dot<B200_TYPE_Q4_K, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a0, k, 0, lane, acc); break;
            case B200_TYPE_Q5_K: slot_dot<B200_TYPE_Q5_K, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a0, k, 0, lane, acc); break;
            case B200_TYPE_Q6_K: slot_dot<B200_TYPE_Q6_K, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a0, k, 0, lane, acc); break;
            case B200_TYPE_Q4_0: slot_dot<B200_TYPE_Q4_0, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a1, k, 1, lane, acc); break;
            case B200_TYPE_Q5_0: slot_dot<B200_TYPE_Q5_0, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a1, k, 1, lane, acc); break;
            default:             slot_dot<B200_TYPE_Q8_0, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a1, k, 1, lane, acc); break;
        }
    } else if (TT == -2) {
        // the launch mixes Q4_K and Q6_K matrices only (QKV of a Q4_K_M model: attn_v is Q6_K in half of the layers):
        // two types' worth of code instead of five — these 10-microsecond kernels feel every instruction-cache miss
        if (t0 == B200_TYPE_Q4_K) {
            if (segc == 64) slot_dot_q4K_fast<NCOLS, NR>(s0, s1, nb0, lseg, seg, a0, k, lane, acc);
            else slot_dot<B200_TYPE_Q4_K, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a0, k, 0, lane, acc);
        } else {
            if (segc == 64) slot_dot_q6K_fast<NCOLS, NR>(s0, s1, nb0, lseg, seg, a0, k, lane, acc);
            else slot_dot<B200_TYPE_Q6_K, NCOLS, NR>(s0, s1, nb0, segc, lseg, seg, a0, k, 0, lane, acc);
        }
    } else if (t0 == t1) {
        slot_one_type<NCOLS, NR>(t0, s0, s1, nb0, segc, lseg, seg, a0, a1, k, lane, acc);
    } else {
        // SwiGLU pair with different gate / up types: one row each (second accumulator of each call unused)
        float t[2][NCOLS];
#pragma unroll
        for (int c = 0; c < NCOLS; c++) { t[0][c] = 0.0f; t[1][c] = 0.0f; }
        slot_one_type<NCOLS, 1>(t0, s0, s0, nb0, segc, lseg, seg, a0, a1, k, lane, t);
#pragma unroll
        for (int c = 0; c < NCOLS; c++) { acc[0][c] += t[0][c]; t[0][c] = 0.0f; t[1][c] = 0.0f; }
        slot_one_type<NCOLS, 1>(t1, s1, s1, nb1, segc, lseg, seg, a0, a1, k, lane, t);
#pragma unroll
        for (int c = 0; c < NCOLS; c++) acc[1][c] += t[0][c];
    }
}

// One unit of work for a warp = R rows x one K-part (G segments of 2048 elements).  The K-parts of a row group
// are consecutive units of the same warp (accumulators persist), so every ring slot is a few KB and >= 2 slots fit
// per warp even for n_ff-long rows.  A part of a row is 1 contiguous byte range (Q4_K/Q5_K) or 2 / 4 ranges
// (repacked Q4_0/Q8_0: qs | d;  Q6_K: ql | qh | scales | d) -> that many bulk copies.
struct RowGroup { const uint8_t * row0, * row1; int t0, t1, nb0, nb1; int64_t r0; int rows; };

template <int MODE>
__device__ __forceinline__ RowGroup group_info(const MmvArgs & args, int g, const MmvMat * & Mp) {
    RowGroup rg;
    if (MODE == MMV_MODE_SWIGLU) {
        const MmvMat & gt = args.mat[0]; const MmvMat & up = args.mat[1];
        Mp = &args.mat[0];
        rg.t0 = gt.type; rg.t1 = up.type; rg.nb0 = gt.nb; rg.nb1 = up.nb;
        rg.row0 = gt.W + (int64_t)g * gt.rb; rg.row1 = up.W + (int64_t)g * up.rb;
        rg.r0 = g; rg.rows = 2;
    } else {
        int mi = 0;                                   // the matrix is addressed inside the (constant-bank) parameter block: no local copy
        if (args.n_mats > 1) {
#pragma unroll
            for (int q = 1; q < MMV_MAX_MATS; q++) if (q < args.n_mats && g >= args.mat[q].pair0) mi = q;
        }
        const MmvMat & M = args.mat[mi];
        Mp = &M;
        const int R = args.rows_per_unit;
        rg.r0 = (int64_t)(g - M.pair0) * R;
        rg.rows = (int)(M.m - rg.r0 < R ? M.m - rg.r0 : R);
        rg.t0 = rg.t1 = M.type; rg.nb0 = rg.nb1 = M.nb;
        rg.row0 = M.W + rg.r0 * M.rb; rg.row1 = rg.rows > 1 ? rg.row0 + M.rb : rg.row0;
    }
    return rg;
}

// bytes of `nsb8` segments (8 super-blocks / 64 small blocks each) of one row of `type`
template <int TT>
__device__ __forceinline__ uint32_t part_bytes(int type, int nchunks) {
    if (TT >= 0) type = TT;                           // uniform launch: the switch folds away
    if (TT == -2) return type == B200_TYPE_Q4_K ? nchunks / 8 * 144 : nchunks / 8 * 210;
    switch (type) {
        case B200_TYPE_Q4_0: return nchunks * 18;
        case B200_TYPE_Q5_0: return nchunks * 22;
        case B200_TYPE_Q8_0: return nchunks * 34;
        case B200_TYPE_Q4_K: return nchunks / 8 * 144;
        case B200_TYPE_Q5_K: return nchunks / 8 * 176;
        default:             return nchunks / 8 * 210;
    }
}
// lane 0: copy chunks [c0, c0 + n) of a row into the slot, laid out like a short row of n chunks
template <int TT>
__device__ __forceinline__ void issue_part(int type, uint8_t * dst, const uint8_t * row, int64_t nb, int c0, int n, uint64_t * bar) {
    if (TT >= 0) type = TT;                           // uniform launch: one case survives (13 bulk copies x 4 call sites otherwise)
    if (TT == -2) {                                   // Q4_K or Q6_K only
        if (type == B200_TYPE_Q4_K) { bulk_g2s(dst, row + (int64_t)(c0 >> 3) * 144, (n >> 3) * 144, bar); return; }
        const int64_t s0 = c0 >> 3; const int ns = n >> 3;
        bulk_g2s(dst,            row + s0 * 128,           ns * 128, bar);
        bulk_g2s(dst + ns * 128, row + nb * 128 + s0 * 64, ns * 64,  bar);
        bulk_g2s(dst + ns * 192, row + nb * 192 + s0 * 16, ns * 16,  bar);
        bulk_g2s(dst + ns * 208, row + nb * 208 + s0 * 2,  ns * 2,   bar);
        return;
    }
    switch (type) {
        case B200_TYPE_Q4_K: bulk_g2s(dst, row + (int64_t)(c0 >> 3) * 144, (n >> 3) * 144, bar); break;
        case B200_TYPE_Q5_K: bulk_g2s(dst, row + (int64_t)(c0 >> 3) * 176, (n >> 3) * 176, bar); break;
        case B200_TYPE_Q4_0:
            bulk_g2s(dst, row + (int64_t)c0 * 16, n * 16, bar);
            bulk_g2s(dst + n * 16, row + nb * 16 + (int64_t)c0 * 2, n * 2, bar);
            break;
        case B200_TYPE_Q5_0:
            bulk_g2s(dst, row + (int64_t)c0 * 16, n * 16, bar);
            bulk_g2s(dst + n * 16, row + nb * 16 + (int64_t)c0 * 4, n * 4, bar);
            bulk_g2s(dst + n * 20, row + nb * 20 + (int64_t)c0 * 2, n * 2, bar);
            break;
        case B200_TYPE_Q8_0:
            bulk_g2s(dst, row + (int64_t)c0 * 32, n * 32, bar);
            bulk_g2s(dst + n * 32, row + nb * 32 + (int64_t)c0 * 2, n * 2, bar);
            break;
        default: {
            const int64_t s0 = c0 >> 3; const int ns = n >> 3;
            bulk_g2s(dst,            row + s0 * 128,           ns * 128, bar);
            bulk_g2s(dst + ns * 128, row + nb * 128 + s0 * 64, ns * 64,  bar);
            bulk_g2s(dst + ns * 192, row + nb * 192 + s0 * 16, ns * 16,  bar);
            bulk_g2s(dst + ns * 208, row + nb * 208 + s0 * 2,  ns * 2,   bar);
        }
    }
}

// ACT >= 0 selects the LEAN decode instance: one column, K-quant weights only (q8_K activations), whole 2048-element segments, row
// pairs, the activation source fixed at compile time.  Same arithmetic as the general instance, a fraction of its code: a decode
// token runs ~160 launches of ~10 us, and every one of them starts with a cold instruction cache (the general instances are ~100 KB
// of SASS each; the trace of tools/trace_decode.py shows 1.5-4 us from kernel entry to the first bulk copy).
template <int NCOLS, int TT, int MODE, int ACT = -1, int NR = 2>
__global__ void __launch_bounds__(MMV_WARPS * 32, MMV_CTAS_PER_SM) mmvq_kernel(const __grid_constant__ MmvArgs args) {
    constexpr bool LEAN = ACT >= 0;
    constexpr bool B32 = TT == B200_TYPE_Q4_0 || TT == B200_TYPE_Q5_0 || TT == B200_TYPE_Q8_0;   // lean instances of the 32-element block types: q8_0 activations
    const int act_source = LEAN ? ACT : args.act_source;
    const int ncols_rt = LEAN ? 1 : args.ncols;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t act_bar;
    __shared__ __align__(8) uint64_t full_bar[MMV_WARPS][MMV_MAX_STAGES];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int S = args.stages, segc = args.segc, nseg = args.nseg, G = args.segs_per_part, P = args.parts;

    uint8_t * act_s0 = smem;
    uint8_t * act_s1 = smem + args.act_bytes[0];
    uint8_t * ring   = smem + ((args.act_bytes[0] + args.act_bytes[1] + 127) & ~127) + (size_t)warp * S * args.slot_bytes;

    B200_TRACE_OPEN(g_mmv_trace, (args.trace & 1) && tid == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1), tr)
    if (tr) { tr[8] = ((unsigned long long)blockIdx.x << 48) | ((unsigned long long)(unsigned)args.total_pairs << 16) | (unsigned long long)((args.mat[0].type & 0xff) << 8) | (unsigned)args.n_mats; tr[9] = (unsigned long long)args.k; }
    if (tid == 0) mbar_init(&act_bar, 1);
    if (lane == 0) for (int s = 0; s < S; s++) mbar_init(&full_bar[warp][s], 1);
    mbar_fence_init();
    __syncthreads();

    // this warp's row groups: gw, gw + TW, ... (consecutive groups -> consecutive SMs); counters only, no div/mod
    const int TW = gridDim.x * MMV_WARPS;
    const int gw = warp * gridDim.x + blockIdx.x;
    const int total = args.total_pairs;

    int ig = gw, ip = 0, islot = 0;                               // issue cursor: group, part, slot
    auto issue_next = [&]() {                                     // lane 0 only
        const MmvMat * Mp;
        const RowGroup rg = group_info<MODE>(args, ig, Mp);
        const int c0 = ip * G * segc;
        const int n = (ip == P - 1 ? nseg - ip * G : G) * segc;
        uint8_t * dst = ring + (size_t)islot * args.slot_bytes;
        const uint32_t b0 = part_bytes<TT>(rg.t0, n), b1 = (MODE == MMV_MODE_SWIGLU || rg.rows > 1) ? part_bytes<TT>(rg.t1, n) : 0;
        mbar_expect_tx(&full_bar[warp][islot], b0 + b1);
        issue_part<TT>(rg.t0, dst, rg.row0, rg.nb0, c0, n, &full_bar[warp][islot]);
        if (b1) issue_part<TT>(rg.t1, dst + args.row_stride, rg.row1, rg.nb1, c0, n, &full_bar[warp][islot]);
        if (++ip == P) { ip = 0; ig += TW; }
        if (++islot == S) islot = 0;
    };

    // prime the ring: weights do not depend on the previous kernel (PDL overlap)
    // (lean instances: only the first slot now — the rest of the ring is issued behind this CTA's activation loads, see below)
    const int pre_slots = (LEAN && !(args.trace & 2)) ? 1 : S;       // (bit 1 of args.trace: B200_MMV_PRIME_ALL=1, the old order, for A/B runs)
    if (lane == 0) for (int s = 0; s < pre_slots && ig < total; s++) issue_next();
    // norm weights are parameters too: fetch this warp's first block before waiting for the previous kernel (otherwise a
    // cold DRAM access sits between the rms_norm reduction and the quantisation, on every CTA's critical path)
    float4 nwa = make_float4(1.0f, 1.0f, 1.0f, 1.0f), nwb = nwa;
    if (act_source == 2 && args.norm_w && warp < (int)(args.k >> 8)) {
        nwa = __ldg((const float4 *)(args.norm_w + warp * 256 + lane * 8)); nwb = __ldg((const float4 *)(args.norm_w + warp * 256 + lane * 8 + 4));
    }
    B200_TRACE_AT(tr, 2);                                          // ring primed
    pdl_trigger();
    pdl_wait();
    B200_TRACE_AT(tr, 3);                                          // previous kernel complete
    if constexpr (LEAN) {
        // one column, k <= 16384: a warp owns at most four 256-element blocks and keeps them in registers for both passes.  The loads go
        // out FIRST, the remaining ring slots behind them: a CTA that starts late (most do: its SM was busy with the previous kernel)
        // otherwise queues 128 KB of weight requests in front of the 16 KB everything else waits for (act rebuild 3.5-4.8 us vs 2.5)
        __shared__ double red[MMV_WARPS];
        const int nblk = (int)(args.k >> 8);
        const float * xc = args.x;
        float4 xa[4], xb[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int blk = warp + j * MMV_WARPS;
            xa[j] = make_float4(0, 0, 0, 0); xb[j] = xa[j];
            if (blk < nblk) { xa[j] = *(const float4 *)(xc + blk * 256 + lane * 8); xb[j] = *(const float4 *)(xc + blk * 256 + lane * 8 + 4); }
        }
        if (lane == 0) for (int s = pre_slots; s < S && ig < total; s++) issue_next();
        float scale = 1.0f;
        if (ACT == 2) {
            double acc2 = 0.0;                                      // ggml-cpu/ops.cpp:4164-4170: f32 squares summed in double
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (warp + j * MMV_WARPS < nblk) {
                    const float4 a = xa[j], b = xb[j];
                    acc2 += (double)__fmul_rn(a.x, a.x); acc2 += (double)__fmul_rn(a.y, a.y); acc2 += (double)__fmul_rn(a.z, a.z); acc2 += (double)__fmul_rn(a.w, a.w);
                    acc2 += (double)__fmul_rn(b.x, b.x); acc2 += (double)__fmul_rn(b.y, b.y); acc2 += (double)__fmul_rn(b.z, b.z); acc2 += (double)__fmul_rn(b.w, b.w);
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc2 += __shfl_xor_sync(0xffffffffu, acc2, o);
            if (lane == 0) red[warp] = acc2;
            __syncthreads();
            double t = 0.0;
            for (int i = 0; i < MMV_WARPS; i++) t += red[i];
            scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn((float)(t / (double)args.k), args.eps)));
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int blk = warp + j * MMV_WARPS;
            if (blk >= nblk) break;
            const int64_t i = (int64_t)blk * 256 + lane * 8;
            float v[8] = { xa[j].x, xa[j].y, xa[j].z, xa[j].w, xb[j].x, xb[j].y, xb[j].z, xb[j].w };
            if (ACT == 2) {
#pragma unroll
                for (int q = 0; q < 8; q++) v[q] = __fmul_rn(v[q], scale);
                if (args.norm_w) {
                    const float4 wa = j == 0 ? nwa : *(const float4 *)(args.norm_w + i), wb = j == 0 ? nwb : *(const float4 *)(args.norm_w + i + 4);
                    v[0] = __fmul_rn(v[0], wa.x); v[1] = __fmul_rn(v[1], wa.y); v[2] = __fmul_rn(v[2], wa.z); v[3] = __fmul_rn(v[3], wa.w);
                    v[4] = __fmul_rn(v[4], wb.x); v[5] = __fmul_rn(v[5], wb.y); v[6] = __fmul_rn(v[6], wb.z); v[7] = __fmul_rn(v[7], wb.w);
                }
            }
            if (B32) warp_quant_q80(v, act_sections(act_s1, 1, args.k, 0), blk, lane);
            else     warp_quant_q8K(v, act_sections(act_s0, 0, args.k, 0), blk, lane);
        }
        __syncthreads();
    } else
    if (act_source == 0) {
        if (tid == 0) {
            mbar_expect_tx(&act_bar, (uint32_t)(args.act_bytes[0] + args.act_bytes[1]));
            if (args.act_bytes[0]) bulk_g2s(act_s0, args.act[0], (uint32_t)args.act_bytes[0], &act_bar);
            if (args.act_bytes[1]) bulk_g2s(act_s1, args.act[1], (uint32_t)args.act_bytes[1], &act_bar);
        }
        mbar_wait(&act_bar, 0);
    } else {
        // every CTA builds the quantised activation vector itself, straight into shared memory:
        // [rms_norm * w ->] q8_K / q8_0 exactly as the CPU oracle quantises (no separate kernels, no HBM round trip)
        __shared__ double red[MMV_WARPS];
        const int nblk = (int)(args.k >> 8);
        for (int col = 0; col < ncols_rt; col++) {
            const float * xc = args.x + (int64_t)col * args.x_col_stride;
            float scale = 1.0f;
            if (act_source == 2) {
                double acc2 = 0.0;                                  // ggml-cpu/ops.cpp:4164-4170: f32 squares summed in double
                for (int blk = warp; blk < nblk; blk += MMV_WARPS) {
                    float4 a = make_float4(0, 0, 0, 0), b = a;
                    if (blk * 256 + lane * 8 < args.k_valid) { a = *(const float4 *)(xc + blk * 256 + lane * 8); b = *(const float4 *)(xc + blk * 256 + lane * 8 + 4); }
                    acc2 += (double)__fmul_rn(a.x, a.x); acc2 += (double)__fmul_rn(a.y, a.y); acc2 += (double)__fmul_rn(a.z, a.z); acc2 += (double)__fmul_rn(a.w, a.w);
                    acc2 += (double)__fmul_rn(b.x, b.x); acc2 += (double)__fmul_rn(b.y, b.y); acc2 += (double)__fmul_rn(b.z, b.z); acc2 += (double)__fmul_rn(b.w, b.w);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) acc2 += __shfl_xor_sync(0xffffffffu, acc2, o);
                if (lane == 0) red[warp] = acc2;
                __syncthreads();
                double t = 0.0;
                for (int i = 0; i < MMV_WARPS; i++) t += red[i];    // every thread: same order, same value — no second barrier
                scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn((float)(t / (double)args.k_valid), args.eps)));
            }
            // a warp owns blocks warp, warp + 16, ...: the loads of up to four of them are issued before the first is quantised, so a long
            // row (n_ff = 14336: 3.5 blocks per warp) costs one memory round trip instead of one per block (4 us -> the k = 4096 figure)
            for (int b0 = warp; b0 < nblk; b0 += MMV_WARPS * 4) {
                float4 xa[4], xb[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int64_t i = (int64_t)(b0 + j * MMV_WARPS) * 256 + lane * 8;
                    xa[j] = make_float4(0, 0, 0, 0); xb[j] = xa[j];
                    if (b0 + j * MMV_WARPS < nblk && i < args.k_valid) { xa[j] = *(const float4 *)(xc + i); xb[j] = *(const float4 *)(xc + i + 4); }
                }
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int blk = b0 + j * MMV_WARPS;
                    if (blk >= nblk) break;
                    const int64_t i = (int64_t)blk * 256 + lane * 8;
                    const bool have = i < args.k_valid;                 // padded weight layout: x ends at k_valid
                    float v[8] = { xa[j].x, xa[j].y, xa[j].z, xa[j].w, xb[j].x, xb[j].y, xb[j].z, xb[j].w };
                    if (act_source == 2) {
#pragma unroll
                        for (int q = 0; q < 8; q++) v[q] = __fmul_rn(v[q], scale);
                        if (args.norm_w && have) {
                            const bool pre = blk == warp;
                            const float4 wa = pre ? nwa : *(const float4 *)(args.norm_w + i), wb = pre ? nwb : *(const float4 *)(args.norm_w + i + 4);
                            v[0] = __fmul_rn(v[0], wa.x); v[1] = __fmul_rn(v[1], wa.y); v[2] = __fmul_rn(v[2], wa.z); v[3] = __fmul_rn(v[3], wa.w);
                            v[4] = __fmul_rn(v[4], wb.x); v[5] = __fmul_rn(v[5], wb.y); v[6] = __fmul_rn(v[6], wb.z); v[7] = __fmul_rn(v[7], wb.w);
                        }
                    }
                    if (!LEAN && args.y_out && blockIdx.x == 0 && have) {
                        float * yo = args.y_out + (int64_t)col * args.k + i;
                        *(float4 *)yo = make_float4(v[0], v[1], v[2], v[3]); *(float4 *)(yo + 4) = make_float4(v[4], v[5], v[6], v[7]);
                    }
                    if (LEAN ? !B32 : (bool)args.act_bytes[0]) warp_quant_q8K(v, act_sections(act_s0, 0, args.k, col), blk, lane);
                    if (LEAN ? B32 : (bool)args.act_bytes[1]) warp_quant_q80(v, act_sections(act_s1, 1, args.k, col), blk, lane);
                }
            }
            if (act_source == 2) __syncthreads();             // red / s_scale are reused by the next column
        }
        __syncthreads();
    }

    B200_TRACE_AT(tr, 4);                                          // activations quantised in shared memory
    const int64_t k = args.k;
    int slot = 0; uint32_t phase = 0;
    if constexpr (LEAN) {
        // row pairs (NR = 1: single rows, for launches whose pair count divides badly over the warps), whole segments, one column: nothing to select at run time except (TT == -2) Q4_K or Q6_K per matrix
#pragma unroll 1
        for (int g = gw; g < total; g += TW) {
            const MmvMat * Mp;
            const RowGroup rg = group_info<MODE>(args, g, Mp);
            const MmvMat & M = *Mp;
            float acc[2][1] = { { 0.0f }, { 0.0f } };
#pragma unroll 1
            for (int p = 0; p < P; p++) {
                const int nsegs = p == P - 1 ? nseg - p * G : G;
                mbar_wait(&full_bar[warp][slot], phase);
                const uint8_t * s0 = ring + (size_t)slot * args.slot_bytes;
                const uint8_t * s1 = s0 + args.row_stride;
                const int lnb = nsegs * 8;
#pragma unroll 1
                for (int ls = 0; ls < nsegs; ls++) {
                    if constexpr (B32) {
                        slot_dot<TT, 1, NR>(s0, s1, nsegs * segc, segc, ls, p * G + ls, act_s1, k, 1, lane, acc);
                    } else if (MODE == MMV_MODE_SWIGLU) {
                        // gate row and up row of the same type TT
                        if (TT == B200_TYPE_Q4_K) slot_dot_q4K_fast<1, NR>(s0, s1, lnb, ls, p * G + ls, act_s0, k, lane, acc);
                        else                      slot_dot_q6K_fast<1, NR>(s0, s1, lnb, ls, p * G + ls, act_s0, k, lane, acc);
                    } else if (TT == B200_TYPE_Q4_K || (TT == -2 && rg.t0 == B200_TYPE_Q4_K)) {
                        slot_dot_q4K_fast<1, NR>(s0, s1, lnb, ls, p * G + ls, act_s0, k, lane, acc);
                    } else {
                        slot_dot_q6K_fast<1, NR>(s0, s1, lnb, ls, p * G + ls, act_s0, k, lane, acc);
                    }
                }
                __syncwarp();
                if (lane == 0 && ig < total) issue_next();
                if (++slot == S) { slot = 0; phase ^= 1; }
            }
            acc[0][0] = warp_sum(acc[0][0]); acc[1][0] = warp_sum(acc[1][0]);
            if (MODE == MMV_MODE_SWIGLU) {
                if (lane == 0) M.dst[rg.r0] = __fmul_rn(silu_x86(acc[0][0]), acc[1][0]);
            } else if (lane < NR) {
                const int64_t r = rg.r0 + lane;
                float v = lane == 0 ? acc[0][0] : acc[1][0];
                if (M.bias)     v += M.bias[r];
                if (M.residual) v += M.residual[r];
                M.dst[r] = v;
            }
        }
    } else {
    bool first_slot = true;
    for (int g = gw; g < total; g += TW) {
        const MmvMat * Mp;
        const RowGroup rg = group_info<MODE>(args, g, Mp);
        const MmvMat & M = *Mp;
        float acc[2][NCOLS];
#pragma unroll
        for (int c = 0; c < NCOLS; c++) { acc[0][c] = 0.0f; acc[1][c] = 0.0f; }
        for (int p = 0; p < P; p++) {
            const int nsegs = p == P - 1 ? nseg - p * G : G;
            mbar_wait(&full_bar[warp][slot], phase);
            if (first_slot) { B200_TRACE_AT(tr, 5); first_slot = false; }   // warp 0's first slot has landed
            const uint8_t * s0 = ring + (size_t)slot * args.slot_bytes;
            const uint8_t * s1 = s0 + args.row_stride;
            // inside the slot a part looks like a short row of nsegs*segc chunks
            const int lnb0 = rg.t0 >= B200_TYPE_Q4_K ? nsegs * (segc >> 3) : nsegs * segc;
            const int lnb1 = rg.t1 >= B200_TYPE_Q4_K ? nsegs * (segc >> 3) : nsegs * segc;
            if (MODE == MMV_MODE_SWIGLU || rg.rows > 1) {
                for (int ls = 0; ls < nsegs; ls++)
                    slot_dispatch<NCOLS, TT, 2>(rg.t0, rg.t1, s0, s1, lnb0, lnb1, segc, ls, p * G + ls, act_s0, act_s1, k, lane, acc);
            } else {
                for (int ls = 0; ls < nsegs; ls++)
                    slot_dispatch<NCOLS, TT, 1>(rg.t0, rg.t0, s0, s0, lnb0, lnb0, segc, ls, p * G + ls, act_s0, act_s1, k, lane, acc);
            }
            __syncwarp();                                         // every lane is done reading the slot
            if (lane == 0 && ig < total) issue_next();            // refill it
            if (++slot == S) { slot = 0; phase ^= 1; }
        }
#pragma unroll
        for (int c = 0; c < NCOLS; c++) { acc[0][c] = warp_sum(acc[0][c]); acc[1][c] = warp_sum(acc[1][c]); }
        if (MODE == MMV_MODE_SWIGLU) {
            if (lane == 0) {
#pragma unroll
                for (int c = 0; c < NCOLS; c++)
                    M.dst[c * M.dst_col_stride + rg.r0] = __fmul_rn(silu_x86(acc[0][c]), acc[1][c]);   // ggml-cpu/vec.cpp:260-282
            }
        } else if (lane < rg.rows) {
            const int64_t r = rg.r0 + lane;
#pragma unroll
            for (int c = 0; c < NCOLS; c++) {
                float v = lane == 0 ? acc[0][c] : acc[1][c];
                if (M.bias)     v += M.bias[r];
                if (M.residual) v += M.residual[c * M.dst_col_stride + r];
                M.dst[c * M.dst_col_stride + r] = v;
            }
        }
    }
    }
    B200_TRACE_AT(tr, 6);                                          // warp 0 done
    if (args.trace & 1) { __syncthreads(); B200_TRACE_CLOSE(tr, 7 + 3); }   // [10] clock, [11] globaltimer: whole CTA done
}
B200_TRACE_DUMP(b200_mmv_trace_dump, g_mmv_trace)

// ---- host ------------------------------------------------------------------------------------
static bool mmv_type_ok(int t) {
    return t == B200_TYPE_Q4_0 || t == B200_TYPE_Q5_0 || t == B200_TYPE_Q8_0 || t == B200_TYPE_Q4_K || t == B200_TYPE_Q5_K || t == B200_TYPE_Q6_K;
}
// k for which every row start and every repacked section is 16-byte aligned
static bool mmv_k_ok(int t, int64_t k) {
    if (k <= 0 || k % 256 != 0) return false;
    if (t == B200_TYPE_Q6_K) return k % 2048 == 0;
    return true;
}

template <int NCOLS, int TT, int MODE, int ACT = -1, int NR = 2> static int mmv_launch_ntm(const MmvArgs & a, size_t smem, int grid, cudaStream_t st) {
    static bool attr[64] = { false };
    int dev = 0; cudaGetDevice(&dev);
    if (!attr[dev & 63]) { cudaFuncSetAttribute(mmvq_kernel<NCOLS, TT, MODE, ACT, NR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 222 * 1024); attr[dev & 63] = true; }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(MMV_WARPS * 32); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = b200_pdl_enabled() ? 1 : 0;
    int s = b200_check(cudaLaunchKernelEx(&cfg, mmvq_kernel<NCOLS, TT, MODE, ACT, NR>, a), "mmvq launch");
    if (s != B200_OK) return s;
    b200_count_launch();
    return B200_OK;
}
template <int NCOLS, int TT> static int mmv_launch_nt(const MmvArgs & a, int mode, size_t smem, int grid, cudaStream_t st) {
    return mode == MMV_MODE_SWIGLU ? mmv_launch_ntm<NCOLS, TT, MMV_MODE_SWIGLU>(a, smem, grid, st)
                                   : mmv_launch_ntm<NCOLS, TT, MMV_MODE_PLAIN>(a, smem, grid, st);
}
// the lean decode instances (see mmvq_kernel): returns -1 if the launch does not qualify
template <int TT, int MODE> static int mmv_launch_lean_tm(const MmvArgs & a, size_t smem, int grid, cudaStream_t st) {
    return a.act_source == 2 ? mmv_launch_ntm<1, TT, MODE, 2>(a, smem, grid, st) : mmv_launch_ntm<1, TT, MODE, 1>(a, smem, grid, st);
}
static int mmv_launch_lean(const MmvArgs & a, int mode, size_t smem, int grid, cudaStream_t st) {
    static const bool off = getenv("B200_MMV_NO_LEAN") != nullptr;
    if (off || a.ncols != 1 || (a.act_source != 1 && a.act_source != 2) || a.y_out || a.k_valid != a.k || a.k > 16384) return -1;
    if (a.rows_per_unit == 1) {                     // single rows: Q4_K (+ Q6_K) launches without SwiGLU only (the QKV projection)
        bool q6 = false;
        for (int i = 0; i < a.n_mats; i++) { if (a.mat[i].type == B200_TYPE_Q6_K) q6 = true; else if (a.mat[i].type != B200_TYPE_Q4_K) return -1; }
        if (mode == MMV_MODE_SWIGLU || a.act_bytes[1] != 0 || a.segc != 64) return -1;
        if (q6) return a.act_source == 2 ? mmv_launch_ntm<1, -2, MMV_MODE_PLAIN, 2, 1>(a, smem, grid, st) : mmv_launch_ntm<1, -2, MMV_MODE_PLAIN, 1, 1>(a, smem, grid, st);
        return a.act_source == 2 ? mmv_launch_ntm<1, B200_TYPE_Q4_K, MMV_MODE_PLAIN, 2, 1>(a, smem, grid, st) : mmv_launch_ntm<1, B200_TYPE_Q4_K, MMV_MODE_PLAIN, 1, 1>(a, smem, grid, st);
    }
    if (a.rows_per_unit != 2) return -1;
    const int t0 = a.mat[0].type;
    bool q4 = false, q6 = false, uniform = true;
    for (int i = 0; i < a.n_mats; i++) {
        if (a.mat[i].type != t0) uniform = false;
        if (a.mat[i].type == B200_TYPE_Q4_K) q4 = true; else if (a.mat[i].type == B200_TYPE_Q6_K) q6 = true;
        if (a.mat[i].m & 1) return -1;
    }
    const bool swiglu = mode == MMV_MODE_SWIGLU;
    if (uniform && (t0 == B200_TYPE_Q4_0 || t0 == B200_TYPE_Q5_0 || t0 == B200_TYPE_Q8_0)) {       // q8_0 activations only
        if (a.act_bytes[0] != 0) return -1;
#define LEAN32(T) (swiglu ? mmv_launch_lean_tm<T, MMV_MODE_SWIGLU>(a, smem, grid, st) : mmv_launch_lean_tm<T, MMV_MODE_PLAIN>(a, smem, grid, st))
        return t0 == B200_TYPE_Q4_0 ? LEAN32(B200_TYPE_Q4_0) : t0 == B200_TYPE_Q5_0 ? LEAN32(B200_TYPE_Q5_0) : LEAN32(B200_TYPE_Q8_0);
#undef LEAN32
    }
    if (!(q4 || q6) || (int)q4 + (int)q6 == 0 || a.act_bytes[1] != 0 || a.segc != 64) return -1;
    for (int i = 0; i < a.n_mats; i++) if (a.mat[i].type != B200_TYPE_Q4_K && a.mat[i].type != B200_TYPE_Q6_K) return -1;
    if (swiglu) {
        if (q4 && q6) return -1;
        return q4 ? mmv_launch_lean_tm<B200_TYPE_Q4_K, MMV_MODE_SWIGLU>(a, smem, grid, st) : mmv_launch_lean_tm<B200_TYPE_Q6_K, MMV_MODE_SWIGLU>(a, smem, grid, st);
    }
    if (q4 && q6) return mmv_launch_lean_tm<-2, MMV_MODE_PLAIN>(a, smem, grid, st);
    return q4 ? mmv_launch_lean_tm<B200_TYPE_Q4_K, MMV_MODE_PLAIN>(a, smem, grid, st) : mmv_launch_lean_tm<B200_TYPE_Q6_K, MMV_MODE_PLAIN>(a, smem, grid, st);
}

template <int NCOLS> static int mmv_launch_n(const MmvArgs & a, int mode, size_t smem, int grid, cudaStream_t st) {
    if (NCOLS == 1) { const int ls = mmv_launch_lean(a, mode, smem, grid, st); if (ls != -1) return ls; }
    int tt = a.mat[0].type;
    for (int i = 1; i < a.n_mats; i++) if (a.mat[i].type != tt) tt = -1;
    switch (tt) {
        case B200_TYPE_Q4_0: return mmv_launch_nt<NCOLS, B200_TYPE_Q4_0>(a, mode, smem, grid, st);
        case B200_TYPE_Q5_0: return mmv_launch_nt<NCOLS, B200_TYPE_Q5_0>(a, mode, smem, grid, st);
        case B200_TYPE_Q8_0: return mmv_launch_nt<NCOLS, B200_TYPE_Q8_0>(a, mode, smem, grid, st);
        case B200_TYPE_Q4_K: return mmv_launch_nt<NCOLS, B200_TYPE_Q4_K>(a, mode, smem, grid, st);
        case B200_TYPE_Q5_K: return mmv_launch_nt<NCOLS, B200_TYPE_Q5_K>(a, mode, smem, grid, st);
        case B200_TYPE_Q6_K: return mmv_launch_nt<NCOLS, B200_TYPE_Q6_K>(a, mode, smem, grid, st);
        default: {
            bool k46 = mode != MMV_MODE_SWIGLU;
            for (int i = 0; i < a.n_mats; i++) if (a.mat[i].type != B200_TYPE_Q4_K && a.mat[i].type != B200_TYPE_Q6_K) k46 = false;
            if (k46) return mmv_launch_ntm<NCOLS, -2, MMV_MODE_PLAIN>(a, smem, grid, st);
            return mmv_launch_nt<NCOLS, -1>(a, mode, smem, grid, st);
        }
    }
}

static int mmv_launch(MmvArgs & a, int mode, int64_t ncols, cudaStream_t st) {
    if (ncols < 1 || ncols > 8) { b200_set_error("mmvq: ncols must be 1..8"); return B200_ERR_INVALID; }
    a.ncols = (int32_t)ncols;
    if (a.k_valid <= 0 || a.k_valid > a.k) a.k_valid = a.k;
    if (a.k_valid % 8 != 0) { b200_set_error("mmvq: k_valid must be a multiple of 8"); return B200_ERR_INVALID; }
    if (a.act_source != 0 && (!a.x || ((uintptr_t)a.x & 15) || (a.x_col_stride & 3) || ((uintptr_t)a.norm_w & 15))) { b200_set_error("mmvq: f32 activation source must be 16-byte aligned"); return B200_ERR_INVALID; }
    bool need[2] = { false, false };
    for (int i = 0; i < a.n_mats; i++) {
        const MmvMat & M = a.mat[i];
        if (!mmv_type_ok(M.type)) { b200_set_error("mmvq: unsupported weight type %d", M.type); return B200_ERR_UNSUPPORTED; }
        if (!mmv_k_ok(M.type, a.k)) { b200_set_error("mmvq: k=%lld not supported for type %d (needs k%%256==0, Q6_K k%%2048==0)", (long long)a.k, M.type); return B200_ERR_UNSUPPORTED; }
        if (((uintptr_t)M.W & 15) || !M.W || !M.dst || M.m <= 0) { b200_set_error("mmvq: weights must be 16-byte aligned / non-null"); return B200_ERR_INVALID; }
        need[b200_act_kind_for(M.type)] = true;
    }
    size_t act = 0;
    for (int kd = 0; kd < 2; kd++) {
        a.act_bytes[kd] = 0;
        if (need[kd]) {
            if (a.act_source == 0 && (!a.act[kd] || ((uintptr_t)a.act[kd] & 15))) { b200_set_error("mmvq: missing/unaligned act buffer of kind %d", kd); return B200_ERR_INVALID; }
            a.act_bytes[kd] = (int32_t)(ncols * act_col_bytes(kd, a.k));
            act += a.act_bytes[kd];
        } else a.act[kd] = nullptr;
    }
    // compute segment: 64 chunks (2048 elements) selects the fast paths; otherwise the largest divisor <= 64
    const int nchunks = (int)(a.k / 32);
    int segc = 8;
    for (int c = 64; c >= 8; c -= 8) if (nchunks % c == 0) { segc = c; break; }
    a.segc = segc; a.nseg = nchunks / segc;
    int64_t rbmax = 0;
    for (int i = 0; i < a.n_mats; i++) {
        a.mat[i].nb = (int32_t)(a.k / type_block_elems(a.mat[i].type));
        a.mat[i].rb = (int64_t)a.mat[i].nb * type_block_bytes(a.mat[i].type);
        if (a.mat[i].rb > rbmax) rbmax = a.mat[i].rb;
    }
    // unit = R rows x G segments: pick the largest G (<= nseg) such that two slots per warp fit; prefer R = 2
    // (activation registers shared by both rows), fall back to R = 1, then to a single slot, then to column halves
    static const int smem_kb = getenv("B200_MMV_SMEM_KB") ? atoi(getenv("B200_MMV_SMEM_KB")) : (MMV_CTAS_PER_SM == 2 ? 108 : 216);
    static const int grid_mult = getenv("B200_MMV_GRID_MULT") ? atoi(getenv("B200_MMV_GRID_MULT")) : 1;
    const size_t budget = (size_t)smem_kb * 1024;
    const size_t act_al = (act + 127) & ~(size_t)127;
    int64_t segb = 0;                                  // bytes of one segment of the widest row type
    for (int i = 0; i < a.n_mats; i++) { const int64_t b = a.mat[i].rb / a.nseg; if (b > segb) segb = b; }
    const int rows_in_slot = 2;                        // SwiGLU: gate + up;  plain: R (decided below)
    int R = 2, G = 0, stages = 0;
    auto try_cfg = [&](int r, int want_stages) {
        for (int g = a.nseg; g >= 1; g--) {
            const size_t slot = (size_t)(((r * g * segb) + 255) & ~(int64_t)255);
            const size_t room = budget > act_al ? (budget - act_al) / ((size_t)MMV_WARPS * slot) : 0;
            if ((int)room >= want_stages) { R = r; G = g; stages = (int)room; return true; }
        }
        return false;
    };
    // single rows when row PAIRS divide badly over the warps: QKV of Llama-3-8B is 3072 pairs on 2368 warps — 704 warps get two pairs
    // (4 rows) while 6144 single rows give at most 3 per warp; a single row costs ~15 % more than half a pair (no activation reuse)
    static const int r1_mode = getenv("B200_MMV_R1") ? atoi(getenv("B200_MMV_R1")) : 0;      // 0 = never, 1 = by the estimate below
    int64_t units2 = 0, rows1 = 0;
    for (int i = 0; i < a.n_mats; i++) { units2 += (a.mat[i].m + 1) / 2; rows1 += a.mat[i].m; }
    const int64_t Wn = (int64_t)b200_sm_count() * MMV_WARPS;
    const double t2 = 2.0 * (double)((units2 + Wn - 1) / Wn), t1 = 1.15 * (double)((rows1 + Wn - 1) / Wn);
    bool ok = false;
    if (mode != MMV_MODE_SWIGLU && r1_mode == 1 && ncols == 1 && t1 < t2) ok = try_cfg(1, 2);
    if (!ok) ok = try_cfg(2, 2);
    if (!ok && mode != MMV_MODE_SWIGLU) ok = try_cfg(1, 2);
    if (!ok) ok = try_cfg(2, 1);
    if (!ok && mode != MMV_MODE_SWIGLU) ok = try_cfg(1, 1);
    (void)rows_in_slot;
    if (!ok) {
        // the columns of a long row do not leave room for even one slot per warp: run the columns in two halves
        // (weights are streamed twice; only speculative-verify batches of 5..8 tokens on n_ff-long rows get here)
        if (ncols < 2) { b200_set_error("mmvq: k=%lld rows (%lld bytes) exceed shared memory", (long long)a.k, (long long)rbmax); return B200_ERR_UNSUPPORTED; }
        const int64_t h0 = ncols / 2, h1 = ncols - h0;
        MmvArgs lo = a, hi = a;
        for (int kd = 0; kd < 2; kd++) if (hi.act[kd]) hi.act[kd] += h0 * act_col_bytes(kd, a.k);
        if (hi.x) hi.x += h0 * a.x_col_stride;
        if (hi.y_out) hi.y_out += h0 * a.k;
        for (int i = 0; i < a.n_mats; i++) {
            hi.mat[i].dst += h0 * a.mat[i].dst_col_stride;
            if (hi.mat[i].residual) hi.mat[i].residual += h0 * a.mat[i].dst_col_stride;
        }
        const int s0 = mmv_launch(lo, mode, h0, st);
        return s0 != B200_OK ? s0 : mmv_launch(hi, mode, h1, st);
    }
    const size_t row_stride = (size_t)(((G * segb) + 127) & ~(int64_t)127);
    const size_t slot = (size_t)(((R * G * segb) + 255) & ~(int64_t)255) < 2 * row_stride && R == 2 ? 2 * row_stride : (size_t)(((R * G * segb) + 255) & ~(int64_t)255);
    a.segs_per_part = G; a.parts = (a.nseg + G - 1) / G; a.row_stride = (int32_t)row_stride;
    if (budget - act_al < (size_t)MMV_WARPS * stages * slot) stages = (int)((budget - act_al) / ((size_t)MMV_WARPS * slot));
    if (stages < 1) { b200_set_error("mmvq: internal smem planning error"); return B200_ERR_UNSUPPORTED; }
    a.rows_per_unit = R; a.slot_bytes = (int32_t)slot;
    if (stages > MMV_MAX_STAGES) stages = MMV_MAX_STAGES;
    a.stages = stages;
    // units: per matrix ceil(m / R) (SwiGLU: one per output row)
    if (mode != MMV_MODE_SWIGLU) {
        int32_t units = 0;
        for (int i = 0; i < a.n_mats; i++) { a.mat[i].pair0 = units; units += (int32_t)((a.mat[i].m + R - 1) / R); }
        a.total_pairs = units;
    }
    const size_t smem = act_al + (size_t)MMV_WARPS * stages * slot;
    const int sms = b200_sm_count();
    int grid = (a.total_pairs + MMV_WARPS - 1) / MMV_WARPS;
    if (grid > sms * grid_mult) grid = sms * grid_mult;
    if (grid < 1) grid = 1;
    switch (ncols) {
        case 1: return mmv_launch_n<1>(a, mode, smem, grid, st);
        case 2: return mmv_launch_n<2>(a, mode, smem, grid, st);
        case 3: return mmv_launch_n<3>(a, mode, smem, grid, st);
        case 4: return mmv_launch_n<4>(a, mode, smem, grid, st);
        case 5: return mmv_launch_n<5>(a, mode, smem, grid, st);
        case 6: return mmv_launch_n<6>(a, mode, smem, grid, st);
        case 7: return mmv_launch_n<7>(a, mode, smem, grid, st);
        default: return mmv_launch_n<8>(a, mode, smem, grid, st);
    }
}

extern "C" int b200_mul_mat_vec_q(int type, const void * W, const void * act, float * dst, int64_t dst_col_stride,
                                  const float * bias, const float * residual, int64_t m, int64_t k, int64_t ncols, void * stream) {
    MmvArgs a = {};
    a.mat[0] = { (const uint8_t *)W, dst, bias, residual, m, dst_col_stride, 0, 0, type, 0, 0 };
    a.n_mats = 1; a.k = k;
    a.total_pairs = (int32_t)((m + 1) / 2);
    const int kind = b200_act_kind_for(type);
    if (kind < 0) { b200_set_error("mmvq: unsupported weight type %d", type); return B200_ERR_UNSUPPORTED; }
    a.act[kind] = (const uint8_t *)act;
    return mmv_launch(a, MMV_MODE_PLAIN, ncols, (cudaStream_t)stream);
}

extern "C" int b200_mul_mat_vec_q_multi(const b200_mmv_desc * descs, int n_mats, const void * act_q8K, const void * act_q80,
                                        int64_t k, int64_t ncols, void * stream) {
    if (n_mats < 1 || n_mats > MMV_MAX_MATS || !descs) { b200_set_error("mmvq_multi: n_mats must be 1..%d", MMV_MAX_MATS); return B200_ERR_INVALID; }
    MmvArgs a = {};
    int32_t pairs = 0;
    for (int i = 0; i < n_mats; i++) {
        a.mat[i] = { (const uint8_t *)descs[i].W, descs[i].dst, descs[i].bias, nullptr, descs[i].m, descs[i].m, 0, 0, descs[i].type, pairs, 0 };
        pairs += (int32_t)((descs[i].m + 1) / 2);
    }
    a.n_mats = n_mats; a.k = k; a.total_pairs = pairs;
    a.act[0] = (const uint8_t *)act_q8K; a.act[1] = (const uint8_t *)act_q80;
    return mmv_launch(a, MMV_MODE_PLAIN, ncols, (cudaStream_t)stream);
}

extern "C" int b200_mul_mat_vec_q_swiglu(int type_gate, const void * Wg, int type_up, const void * Wu,
                                         const void * act_q8K, const void * act_q80, float * dst,
                                         int64_t m, int64_t k, int64_t ncols, void * stream) {
    MmvArgs a = {};
    a.mat[0] = { (const uint8_t *)Wg, dst, nullptr, nullptr, m, m, 0, 0, type_gate, 0, 0 };
    a.mat[1] = { (const uint8_t *)Wu, dst, nullptr, nullptr, m, m, 0, 0, type_up, 0, 0 };
    a.n_mats = 2; a.k = k; a.total_pairs = (int32_t)m;
    a.act[0] = (const uint8_t *)act_q8K; a.act[1] = (const uint8_t *)act_q80;
    return mmv_launch(a, MMV_MODE_SWIGLU, ncols, (cudaStream_t)stream);
}

// general launch: several matrices / SwiGLU / fused activation prologue in one descriptor (see b200_ops.h)
extern "C" int b200_mul_mat_vec_q_launch(const b200_mmv_launch * L, void * stream) {
    if (!L || L->n_mats < 1 || L->n_mats > MMV_MAX_MATS) { b200_set_error("mmvq_launch: bad descriptor"); return B200_ERR_INVALID; }
    if (L->swiglu && L->n_mats != 2) { b200_set_error("mmvq_launch: swiglu needs exactly gate and up"); return B200_ERR_INVALID; }
    if (L->act_source < 0 || L->act_source > 2) { b200_set_error("mmvq_launch: act_source must be 0..2"); return B200_ERR_INVALID; }
    MmvArgs a = {};
    for (int i = 0; i < L->n_mats; i++)
        a.mat[i] = { (const uint8_t *)L->mats[i].W, L->mats[i].dst, L->mats[i].bias, L->residual[i], L->mats[i].m, L->dst_col_stride[i] ? L->dst_col_stride[i] : L->mats[i].m, 0, 0, L->mats[i].type, 0, 0 };
    a.n_mats = L->n_mats; a.k = L->k;
    a.total_pairs = L->swiglu ? (int32_t)L->mats[0].m : 0;
    a.act[0] = (const uint8_t *)L->act_q8K; a.act[1] = (const uint8_t *)L->act_q80;
    a.act_source = L->act_source; a.x = L->x; a.x_col_stride = L->x_col_stride; a.norm_w = L->norm_w; a.eps = L->eps; a.y_out = L->y_out;
    a.k_valid = L->k_valid;
    static const int prime_all = getenv("B200_MMV_PRIME_ALL") ? 2 : 0;
    a.trace = (b200_trace_on() ? 1 : 0) | prime_all;
    return mmv_launch(a, L->swiglu ? MMV_MODE_SWIGLU : MMV_MODE_PLAIN, L->ncols, (cudaStream_t)stream);
}
