// fattn.cu — FLASH_ATTN_EXT over the F16 / Q8_0 KV cache, split-KV "vector" kernel (sm_90a).
//
// Replaces ggml_cuda_flash_attn_ext -> flash_attn_vec_ext_f32<D,1,K,V> + flash_attn_combine_results
// (ggml-cuda/fattn.cu:271-338, fattn-vec-f32.cuh:10-361, fattn-common.cuh:645-701).
// Numerics follow the CPU oracle (ggml-cpu/ops.cpp:8169-8405): the Q row is converted to K's
// vec_dot type (f16 for F16 K; RNE q8_0 for Q8_0 K, integer block dots), s = dot*scale
// (+softcap) + slope*mask, online softmax in f32, quantised V expanded to f32.  (With F16 V the
// oracle accumulates in fp16; we accumulate in f32, which is strictly more accurate.)
//
// Mapping: D/8 lanes per KV position (8 elements = one 16-byte load per lane for F16), so a warp
// streams 2 (D=128) or 4 (D=64) positions per step with fully coalesced rows; up to 2 query heads of
// one GQA group share every K/V load; KV is split over the CTAs of a thread-block cluster (grid.x) to fill the SMs (132 on
// an H100), and the cluster merges the splits' (m, l, acc) partials through distributed shared memory.  HBM-bound: bytes =
// K+V rows once per head tile.
#include "common.cuh"
#include "ropeutil.cuh"
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define FA_WARPS 4
#ifndef FA_MIN_CTAS
#define FA_MIN_CTAS 1      // (4 = at most 128 registers, so that a CTA fits next to a resident matvec CTA: measured no gain)
#endif
#define FA_MAX_CLUSTER 16  // KV splits of one (token, head tile) = CTAs of one cluster

B200_TRACE_DECL(g_fa_trace)


__device__ __forceinline__ void unpack_h8(const uint4 & r, float (&f)[8]) {
    const __half2 * h = (const __half2 *)&r;
#pragma unroll
    for (int i = 0; i < 4; i++) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}

// load 8 int8 of a native q8_0 row (34-byte blocks, 2-byte aligned) + the block scale
__device__ __forceinline__ void load_q80_8(const uint8_t * row, int dl, int (&q)[2], float & d) {
    const uint8_t * blk = row + (dl >> 2) * 34;
    const uint16_t * p = (const uint16_t *)(blk + 2 + (dl & 3) * 8);
    d = h2f(__ldg((const uint16_t *)blk));
    q[0] = (int)((uint32_t)__ldg(p)     | ((uint32_t)__ldg(p + 1) << 16));
    q[1] = (int)((uint32_t)__ldg(p + 2) | ((uint32_t)__ldg(p + 3) << 16));
}

// ---- decode fusion: ROPE(q), ROPE(k) -> K cache, v -> V cache and the attention itself in ONE launch ----------------
// (replaces rope_norm/rope_neox x2 + k_set_rows x2 + flash_attn_vec + combine: ggml-cuda/rope.cu, set-rows.cu, fattn.cu).
// Every CTA ropes the query heads of its tile on the fly and stages this token's K (roped) / V for its kv head in shared
// memory in cache format; positions equal to the token's cell are read from there, so no CTA depends on another CTA's
// cache write.  One CTA per kv head also writes the cell (and the roped Q, which the graph declares as an output).
struct FaFuse {
    const float * q_src; float * q_dst; const float * k_new; const float * v_new;
    const int32_t * pos; const float * ff; const int64_t * k_ids; const int64_t * v_ids;
    RopeDev rp; int enabled;
    // cos/sin table of this token: the same for every layer, so the first attention launch of a token computes it (every CTA for
    // itself, one CTA also stores it) and the other layers just load 512 bytes: tab_mode 0 = compute (+ store if rope_tab), 1 = load
    float * rope_tab; int tab_mode;
    int trace;                                  // B200_TRACE: timeline records (common.cuh)
};
// elements e0..e0+7 of one head, roped (ops.cpp:6088-6150 pairing; the table holds cos/sin already scaled) — in three steps so
// that the global loads can be issued long before the table is ready: raw8 (the elements), partner8 (NEOX: the other half of
// each pair), rope8 (arithmetic only)
__device__ __forceinline__ void raw8(const float * head, int e0, float (&v)[8]) {
    const float4 a = *(const float4 *)(head + e0), b = *(const float4 *)(head + e0 + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void partner8(const float * head, int e0, const RopeDev & rp, float (&o)[8]) {
#pragma unroll
    for (int j = 0; j < 8; j++) o[j] = 0.0f;
    if (!rp.neox || e0 >= rp.n_dims) return;
    const int half = rp.n_dims >> 1;
    raw8(head, e0 < half ? e0 + half : e0 - half, o);
}
__device__ __forceinline__ void rope8(float (&v)[8], const float (&o)[8], int e0, const float * cs, const RopeDev & rp) {
    if (e0 >= rp.n_dims) return;
    if (!rp.neox) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int i = (e0 >> 1) + j;
            const float c = cs[2 * i], sn = cs[2 * i + 1], x0 = v[2 * j], x1 = v[2 * j + 1];
            v[2 * j]     = __fsub_rn(__fmul_rn(x0, c), __fmul_rn(x1, sn));
            v[2 * j + 1] = __fadd_rn(__fmul_rn(x0, sn), __fmul_rn(x1, c));
        }
    } else {
        const int half = rp.n_dims >> 1;
        const bool first = e0 < half;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int i = first ? e0 + j : e0 - half + j;
            const float c = cs[2 * i], sn = cs[2 * i + 1];
            v[j] = first ? __fsub_rn(__fmul_rn(v[j], c), __fmul_rn(o[j], sn)) : __fadd_rn(__fmul_rn(o[j], sn), __fmul_rn(v[j], c));
        }
    }
}
__device__ __forceinline__ void load_roped8(const float * head, int e0, const float * cs, const RopeDev & rp, float (&v)[8]) {
    float o[8];
    raw8(head, e0, v);
    partner8(head, e0, rp, o);
    rope8(v, o, e0, cs, rp);
}
// 8 int8 of a q8_0 row in shared memory (34-byte blocks) + the block scale
__device__ __forceinline__ void lds_q80_8(const uint8_t * row, int dl, int (&q)[2], float & d) {
    const uint8_t * blk = row + (dl >> 2) * 34;
    const uint16_t * p = (const uint16_t *)(blk + 2 + (dl & 3) * 8);
    d = h2f(*(const uint16_t *)blk);
    q[0] = (int)((uint32_t)p[0] | ((uint32_t)p[1] << 16));
    q[1] = (int)((uint32_t)p[2] | ((uint32_t)p[3] << 16));
}

// LEAN = 1: the decode instance of layers 1..n-1 — fused rope / KV store with the cos/sin table loaded (tab_mode 1), a mask, no ALiBi,
// no soft-cap: the switches below become constants and powf / tanhf / the table computation (sincosf, YaRN) leave the kernel.  These
// launches last ~10 us and start with a cold instruction cache, so the size of the code they step through is their critical path.
//
// The splits of one (token, head tile) are one thread-block cluster along grid.x (cluster rank = split).  Each CTA leaves its split's
// (m, l) per head and its G x D accumulator in shared memory; after a cluster barrier CTA r merges a 1/C slice of the tile's output,
// reading every peer's partials through distributed shared memory in rank order 0..C-1 (so the result does not depend on timing).
template <int D, int KVT, int G, int LEAN = 0>
__global__ void __launch_bounds__(FA_WARPS * 32, FA_MIN_CTAS) fattn_vec_kernel(
        const float * __restrict__ q, int64_t q_ts, int64_t q_hs,
        const uint8_t * __restrict__ kc, int64_t k_rs, int64_t k_hs,
        const uint8_t * __restrict__ vc, int64_t v_rs, int64_t v_hs,
        const uint16_t * __restrict__ mask, int64_t mask_rs, float * __restrict__ dst,
        int n_head, int n_head_kv, int n_kv, int split_len, int n_splits,
        float scale, float max_bias_rt, float softcap_rt, float m0, float m1, int nh_log2, const FaFuse fu) {
    const float max_bias = LEAN ? 0.0f : max_bias_rt, softcap = LEAN ? 0.0f : softcap_rt;
    const bool fused = LEAN ? true : (bool)fu.enabled;
    constexpr int LP  = D / 8;          // lanes per position
    constexpr int PPW = 32 / LP;        // positions per warp step
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sg = lane / LP, dl = lane % LP;
    const int split = blockIdx.x, tile = blockIdx.y, tok = LEAN ? 0 : (int)blockIdx.z;
    const int gq = n_head / n_head_kv;                  // query heads per kv head
    const int h0 = tile * G;                            // first query head of this tile
    const int hk = h0 / gq;
    __shared__ __align__(16) float s_cs[D];
    __shared__ __align__(16) uint8_t s_newk[D * 2 + 32], s_newv[D * 2 + 32];
    constexpr int MAXIT = 4;
    constexpr int pstride = FA_WARPS * PPW;
    constexpr int CH = pstride * MAXIT;                 // positions of one chunk (MAXIT per lane group)
    const int p_begin = split * split_len;
    const int p_end   = min(n_kv, p_begin + split_len);
    const int base0 = p_begin + warp * PPW + sg;
    const uint16_t * mrow = (LEAN || mask) ? mask + (int64_t)tok * mask_rs : nullptr;
    int kcell = -1, vcell = -1, tok_pos = 0;
    B200_TRACE_OPEN(g_fa_trace, fu.trace && threadIdx.x == 0 && tok == 0 && ((split == 0 && tile == 0) || (split == n_splits - 1 && tile == (int)gridDim.y - 1)), tr)
    if (tr) { tr[8] = ((unsigned long long)split << 48) | ((unsigned long long)(unsigned)n_kv << 16) | (unsigned)n_splits; tr[9] = 0; }
    auto load_kv = [&](int p, uint4 & kr, uint4 & vr, float & kd, float & vd) {
        const uint8_t * krow = kc + (int64_t)p * k_rs + (int64_t)hk * k_hs;
        const uint8_t * vrow = vc + (int64_t)p * v_rs + (int64_t)hk * v_hs;
        if (KVT == B200_TYPE_F16) { kr = ldg_stream16(krow + dl * 16); vr = ldg_stream16(vrow + dl * 16); kd = 0.0f; vd = 0.0f; }
        else {
            int q2[2];
            load_q80_8(krow, dl, q2, kd); kr = make_uint4((uint32_t)q2[0], (uint32_t)q2[1], 0, 0);
            load_q80_8(vrow, dl, q2, vd); vr = make_uint4((uint32_t)q2[0], (uint32_t)q2[1], 0, 0);
        }
    };
    // mask of this lane group's positions in the chunk at `base`: -inf beyond the split
    auto load_mask = [&](int base, float (&m)[MAXIT]) {
#pragma unroll
        for (int it = 0; it < MAXIT; it++) {
            const int p = base + it * pstride;
            m[it] = p < p_end ? ((LEAN || mrow) ? h2f(__ldg(mrow + p)) : 0.0f) : -INFINITY;
        }
    };
    // K / V of the chunk at `base`; no load for a position that cannot contribute (beyond the split, or masked without ALiBi)
    auto load_chunk = [&](int base, const float (&m)[MAXIT], uint4 (&kr)[MAXIT], uint4 (&vr)[MAXIT], float (&kd)[MAXIT], float (&vd)[MAXIT]) {
#pragma unroll
        for (int it = 0; it < MAXIT; it++) {
            const int p = base + it * pstride;
            kr[it] = make_uint4(0, 0, 0, 0); vr[it] = kr[it]; kd[it] = 0.0f; vd[it] = 0.0f;
            if (p < p_end && !(m[it] == -INFINITY && max_bias <= 0.0f)) load_kv(p, kr[it], vr[it], kd[it], vd[it]);
        }
    };
    // the chunk being computed (mask, K, V) and the next chunk's mask
    float mcur[MAXIT], mnext[MAXIT]; uint4 kcur[MAXIT], vcur[MAXIT]; float kdcur[MAXIT], vdcur[MAXIT];
    // First chunk.  On the decode path (fu.enabled) the cells of EARLIER tokens were written by earlier launches of the token loop, and
    // pos / cell ids are graph inputs: all of it may be fetched before griddepcontrol.wait, while the previous kernel (the QKV projection)
    // is still running — a memory round trip off the token's critical path.  The mask is read that early only by the layers after the
    // first (LEAN): whatever produces it ran launches ago, and fully masked positions then cost no K / V traffic either.
    if (fused) {
        kcell = (int)fu.k_ids[0]; vcell = (int)fu.v_ids[0]; tok_pos = fu.pos[0];
        if (LEAN) { load_mask(base0, mcur); load_mask(base0 + CH, mnext); }
        else {
#pragma unroll
            for (int it = 0; it < MAXIT; it++) mcur[it] = 0.0f;       // not known yet: load every position of the split
        }
        load_chunk(base0, mcur, kcur, vcur, kdcur, vdcur);
    }
    B200_TRACE_AT(tr, 2);                     // first K / V chunk requested
    pdl_wait();
    B200_TRACE_AT(tr, 3);                     // QKV projection complete
    if (!LEAN) {
        load_mask(base0, mcur); load_mask(base0 + CH, mnext);
        if (!fused) load_chunk(base0, mcur, kcur, vcur, kdcur, vdcur);
    }
    float qraw[G][8], qpar[G][8];
    if (fused) {
        // this token's query heads: issue the loads now, rope them once the table is in shared memory
#pragma unroll
        for (int g = 0; g < G; g++) { raw8(fu.q_src + (int64_t)(h0 + g) * D, dl * 8, qraw[g]); partner8(fu.q_src + (int64_t)(h0 + g) * D, dl * 8, fu.rp, qpar[g]); }
        // rope table: computed by the first layer's launch (kept for the others), loaded by the rest
        if (LEAN || fu.tab_mode == 1) {
            if (threadIdx.x < D / 4) *(float4 *)(s_cs + threadIdx.x * 4) = __ldcg((const float4 *)(fu.rope_tab) + threadIdx.x);
        } else {
            rope_table(s_cs, tok_pos, fu.ff, fu.rp, threadIdx.x, FA_WARPS * 32);
        }
        __syncthreads();
        if (!LEAN && fu.tab_mode == 0 && fu.rope_tab && split == 0 && tile == 0 && threadIdx.x < D / 4) ((float4 *)fu.rope_tab)[threadIdx.x] = *(const float4 *)(s_cs + threadIdx.x * 4);
        // this token's K (roped) / V for kv head hk in cache format: only the CTA whose split holds the cell reads it from shared
        // memory, and one CTA per kv head writes the cell — every other CTA skips the staging (and its barrier) altogether
        const bool storer = split == 0 && (h0 % gq) == 0;
        const bool mine = (kcell >= p_begin && kcell < p_end) || (vcell >= p_begin && vcell < p_end);
        if (storer || mine) {
            if (warp < 2) {
                const int e = lane * 8; const bool on = e < D;
                float a[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
                if (warp == 0) {
                    if (on) load_roped8(fu.k_new + (int64_t)hk * D, e, s_cs, fu.rp, a);
                    store8(s_newk, KVT, e, a, lane, on);
                    if (storer) store8((uint8_t *)kc + (int64_t)kcell * k_rs + (int64_t)hk * k_hs, KVT, e, a, lane, on);
                } else {
                    if (on) { const float4 x = *(const float4 *)(fu.v_new + (int64_t)hk * D + e), y = *(const float4 *)(fu.v_new + (int64_t)hk * D + e + 4);
                              a[0] = x.x; a[1] = x.y; a[2] = x.z; a[3] = x.w; a[4] = y.x; a[5] = y.y; a[6] = y.z; a[7] = y.w; }
                    store8(s_newv, KVT, e, a, lane, on);
                    if (storer) store8((uint8_t *)vc + (int64_t)vcell * v_rs + (int64_t)hk * v_hs, KVT, e, a, lane, on);
                }
            }
            __syncthreads();
        }
    }

    B200_TRACE_AT(tr, 4);                     // rope table + this token's K / V staged
    // ---- query slices: q8[g][8] as f32 (f16-rounded) or int8 + scale -------------------------
    float qf[G][8]; int qi[G][2]; float qd[G]; float slope[G];
#pragma unroll
    for (int g = 0; g < G; g++) {
        const int h = h0 + g;
        float v[8];
        if (fused) {
#pragma unroll
            for (int e = 0; e < 8; e++) v[e] = qraw[g][e];
            rope8(v, qpar[g], dl * 8, s_cs, fu.rp);
            if (split == 0 && warp == 0 && sg == 0) {
                *(float4 *)(fu.q_dst + (int64_t)h * D + dl * 8)     = make_float4(v[0], v[1], v[2], v[3]);
                *(float4 *)(fu.q_dst + (int64_t)h * D + dl * 8 + 4) = make_float4(v[4], v[5], v[6], v[7]);
            }
        } else {
            const float * qp = q + (int64_t)tok * q_ts + (int64_t)h * q_hs + dl * 8;
            const float4 a = *(const float4 *)qp, b = *(const float4 *)(qp + 4);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
        }
        if (KVT == B200_TYPE_F16) {
#pragma unroll
            for (int e = 0; e < 8; e++) qf[g][e] = __half2float(__float2half_rn(v[e]));
            qi[g][0] = qi[g][1] = 0; qd[g] = 0.0f;
        } else {
            float am = 0.0f;
#pragma unroll
            for (int e = 0; e < 8; e++) am = fmaxf(am, fabsf(v[e]));
            am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 1));
            am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 2));
            const float id = am != 0.0f ? __fdiv_rn(127.0f, am) : 0.0f;
            int t[8];
#pragma unroll
            for (int e = 0; e < 8; e++) t[e] = __float2int_rn(__fmul_rn(v[e], id)) & 0xff;
            qi[g][0] = t[0] | (t[1] << 8) | (t[2] << 16) | (t[3] << 24);
            qi[g][1] = t[4] | (t[5] << 8) | (t[6] << 16) | (t[7] << 24);
            qd[g] = __half2float(__float2half_rn(__fdiv_rn(am, 127.0f)));
#pragma unroll
            for (int e = 0; e < 8; e++) qf[g][e] = 0.0f;
        }
        slope[g] = max_bias > 0.0f ? (h < nh_log2 ? powf(m0, (float)(h + 1)) : powf(m1, (float)(2 * (h - nh_log2) + 1))) : 1.0f;
    }

    float M[G], L[G], acc[G][8];
#pragma unroll
    for (int g = 0; g < G; g++) { M[g] = -INFINITY; L[g] = 0.0f;
#pragma unroll
        for (int e = 0; e < 8; e++) acc[g][e] = 0.0f; }

    const unsigned gmask = ((1u << LP) - 1u) << (sg * LP);   // lanes sharing one KV position (converged inside the loop)

    // positions are visited in chunks of MAXIT per lane group.  Every load of a chunk is issued before any arithmetic on it, and the
    // next chunk's K / V (and the mask of the one after) are issued before this chunk's arithmetic: a split of several chunks pays about
    // one memory round trip, not one per chunk (decode attention is latency-bound).
    for (int base = base0; base < p_end; base += CH) {
        if (fused) {
#pragma unroll
            for (int it = 0; it < MAXIT; it++) {
                const int p = base + it * pstride;
                if (p == kcell) {                               // this token's own cell: from shared memory (the global cell is being written by another CTA)
                    if (KVT == B200_TYPE_F16) kcur[it] = *(const uint4 *)(s_newk + dl * 16);
                    else { int q2[2]; lds_q80_8(s_newk, dl, q2, kdcur[it]); kcur[it].x = (uint32_t)q2[0]; kcur[it].y = (uint32_t)q2[1]; }
                }
                if (p == vcell) {
                    if (KVT == B200_TYPE_F16) vcur[it] = *(const uint4 *)(s_newv + dl * 16);
                    else { int q2[2]; lds_q80_8(s_newv, dl, q2, vdcur[it]); vcur[it].x = (uint32_t)q2[0]; vcur[it].y = (uint32_t)q2[1]; }
                }
            }
        }
        float mnn[MAXIT]; uint4 knext[MAXIT], vnext[MAXIT]; float kdnext[MAXIT], vdnext[MAXIT];
        load_chunk(base + CH, mnext, knext, vnext, kdnext, vdnext);
        load_mask(base + 2 * CH, mnn);
        // one position per lane group and step.  The decode instance keeps this loop ROLLED (the K / V registers rotate through
        // slot 0): unrolled it is 20 KB of straight-line code that every launch fetches cold, rolled it is 5 KB fetched once
        auto step = [&](const float mr, const uint4 & kr, const uint4 & vr, const float kd, const float vd) {
            float kf[8], vf[8];
            if (KVT == B200_TYPE_F16) {
                unpack_h8(kr, kf);
                unpack_h8(vr, vf);
            } else {
#pragma unroll
                for (int e = 0; e < 8; e++) vf[e] = __fmul_rn((float)(int8_t)(((e < 4 ? vr.x : vr.y) >> (8 * (e & 3))) & 0xff), vd);
            }
            float s[G];
#pragma unroll
            for (int g = 0; g < G; g++) {
                if (KVT == B200_TYPE_F16) {
                    float a = 0.0f;
#pragma unroll
                    for (int e = 0; e < 8; e++) a = fmaf(kf[e], qf[g][e], a);
#pragma unroll
                    for (int o = LP / 2; o > 0; o >>= 1) a += __shfl_xor_sync(gmask, a, o, LP);
                    s[g] = a;
                } else {
                    int is = dp4a_s((int)kr.x, qi[g][0], 0);
                    is = dp4a_s((int)kr.y, qi[g][1], is);
                    is += __shfl_xor_sync(gmask, is, 1, LP);          // whole 32-element block
                    is += __shfl_xor_sync(gmask, is, 2, LP);
                    float a = __fmul_rn((float)is, __fmul_rn(kd, qd[g]));   // ggml-cpu/quants.c:305-333
                    a = (dl & 3) == 0 ? a : 0.0f;
#pragma unroll
                    for (int o = LP / 2; o >= 4; o >>= 1) a += __shfl_xor_sync(gmask, a, o, LP);
                    s[g] = __shfl_sync(gmask, a, 0, LP);
                }
            }
#pragma unroll
            for (int g = 0; g < G; g++) {
                float sv = s[g] * scale;
                if (softcap != 0.0f) sv = softcap * tanhf(sv);
                sv += slope[g] * mr;
                if (sv == -INFINITY) continue;
                float ms = 1.0f, vs = 1.0f;
                if (sv > M[g]) { ms = expf(M[g] - sv); M[g] = sv;
#pragma unroll
                    for (int e = 0; e < 8; e++) acc[g][e] *= ms;
                } else vs = expf(sv - M[g]);
#pragma unroll
                for (int e = 0; e < 8; e++) acc[g][e] = fmaf(vf[e], vs, acc[g][e]);
                L[g] = L[g] * ms + vs;
            }
        };
        if constexpr (LEAN) {
#pragma unroll 1
            for (int it = 0; it < MAXIT; it++) {
                const float mr = mcur[0]; const uint4 kr = kcur[0], vr = vcur[0]; const float kd = kdcur[0], vd = vdcur[0];
#pragma unroll
                for (int j = 0; j + 1 < MAXIT; j++) { mcur[j] = mcur[j + 1]; kcur[j] = kcur[j + 1]; vcur[j] = vcur[j + 1]; kdcur[j] = kdcur[j + 1]; vdcur[j] = vdcur[j + 1]; }
                if (mr == -INFINITY) continue;      // masked, or beyond the split (uniform inside the LP-lane group)
                step(mr, kr, vr, kd, vd);
            }
        } else {
#pragma unroll
            for (int it = 0; it < MAXIT; it++) {
                if (mcur[it] == -INFINITY && max_bias <= 0.0f) continue;       // masked, or beyond the split (uniform inside the LP-lane group)
                if (base + it * pstride >= p_end) continue;
                step(mcur[it], kcur[it], vcur[it], kdcur[it], vdcur[it]);
            }
        }
#pragma unroll
        for (int it = 0; it < MAXIT; it++) {
            mcur[it] = mnext[it]; kcur[it] = knext[it]; vcur[it] = vnext[it]; kdcur[it] = kdnext[it]; vdcur[it] = vdnext[it]; mnext[it] = mnn[it];
        }
    }

    B200_TRACE_AT(tr, 5);                     // positions of this split done (warp 0)
    // ---- merge the PPW position groups of the warp, then the warps: this split's partial, in shared memory ----------------
    __shared__ float sM[FA_WARPS][G], sL[FA_WARPS][G];
    __shared__ float sA[FA_WARPS][G][D];
    __shared__ float cM[G], cL[G], cA[G][D];            // the split's partial, read by every CTA of the cluster
#pragma unroll
    for (int g = 0; g < G; g++) {
#pragma unroll
        for (int o = LP; o < 32; o <<= 1) {
            const float Mo = __shfl_xor_sync(0xffffffffu, M[g], o), Lo = __shfl_xor_sync(0xffffffffu, L[g], o);
            const float Mn = fmaxf(M[g], Mo);
            const float sa = M[g] == -INFINITY ? 0.0f : expf(M[g] - Mn), sb = Mo == -INFINITY ? 0.0f : expf(Mo - Mn);
#pragma unroll
            for (int e = 0; e < 8; e++) { const float ao = __shfl_xor_sync(0xffffffffu, acc[g][e], o); acc[g][e] = acc[g][e] * sa + ao * sb; }
            L[g] = L[g] * sa + Lo * sb; M[g] = Mn;
        }
        if (sg == 0) {
#pragma unroll
            for (int e = 0; e < 8; e++) sA[warp][g][dl * 8 + e] = acc[g][e];
            if (dl == 0) { sM[warp][g] = M[g]; sL[warp][g] = L[g]; }
        }
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < G * D; idx += FA_WARPS * 32) {
        const int g = idx / D, e = idx % D;
        float Mn = -INFINITY;
#pragma unroll
        for (int w = 0; w < FA_WARPS; w++) Mn = fmaxf(Mn, sM[w][g]);
        float a = 0.0f, l = 0.0f;
#pragma unroll
        for (int w = 0; w < FA_WARPS; w++) {
            const float sc = sM[w][g] == -INFINITY ? 0.0f : expf(sM[w][g] - Mn);
            a += sA[w][g][e] * sc; l += sL[w][g] * sc;
        }
        cA[g][e] = a;
        if (e == 0) { cM[g] = Mn; cL[g] = l; }
    }
    // ---- merge the splits over the cluster (replaces flash_attn_combine_results, fattn-common.cuh:645-701) ----------------
    cluster_arrive_release();                 // this split's partial is published to the cluster
    pdl_trigger();                            // the next kernel (the wo projection) may launch; its griddepcontrol.wait still waits for this grid
    cluster_wait_acquire();
    B200_TRACE_AT(tr, 6);                     // every split of the tile published
    // CTA `split` writes outputs [split * per, (split + 1) * per) of the tile's G x D; every peer's loads are issued before any is used
    const int per = (G * D + n_splits - 1) / n_splits;
    const int i_end = min(G * D, (split + 1) * per);
    for (int idx = split * per + (int)threadIdx.x; idx < i_end; idx += FA_WARPS * 32) {
        const int g = idx / D, e = idx % D;
        float pm[FA_MAX_CLUSTER], pl[FA_MAX_CLUSTER], pa[FA_MAX_CLUSTER];
#pragma unroll
        for (int r = 0; r < FA_MAX_CLUSTER; r++) {
            if (r < n_splits) {
                pm[r] = ld_cluster_f32(cluster_map(&cM[g], r));
                pl[r] = ld_cluster_f32(cluster_map(&cL[g], r));
                pa[r] = ld_cluster_f32(cluster_map(&cA[g][e], r));
            }
        }
        float Mn = -INFINITY;
#pragma unroll
        for (int r = 0; r < FA_MAX_CLUSTER; r++) if (r < n_splits) Mn = fmaxf(Mn, pm[r]);
        float a = 0.0f, l = 0.0f;
#pragma unroll
        for (int r = 0; r < FA_MAX_CLUSTER; r++) {
            if (r < n_splits) {
                const float sc = pm[r] == -INFINITY ? 0.0f : expf(pm[r] - Mn);
                a = fmaf(pa[r], sc, a);
                l += pl[r] * sc;
            }
        }
        dst[((int64_t)tok * n_head + h0 + g) * D + e] = a * (1.0f / l);            // ops.cpp:8390-8392
    }
    B200_TRACE_AT(tr, 7);                     // this CTA's slice of the output written
    // the peers' shared memory must outlive every read of it.  Relaxed: those reads have returned (their values are in dst), so no
    // memory ordering is needed, and a release here would wait for the dst stores to drain (MEMBAR.GPU)
    cluster_arrive_relaxed();
    cluster_wait();
    B200_TRACE_CLOSE(tr, 10);
}
B200_TRACE_DUMP(b200_fa_trace_dump, g_fa_trace)

// KV splits = the cluster size: enough CTAs for two on every SM (132 on an H100), at least 32 positions per split, at most 16 (the
// largest cluster Hopper runs; above 8 it is a non-portable size).  Llama-3-8B decode (32 heads, 8 KV heads, G = 2) at n_kv 768:
// 16 tiles x 16 splits of 48 positions = 256 CTAs
static int fa_splits(int64_t n_tiles, int64_t n_tok, int64_t n_kv, int * split_len) {
    const int64_t base = n_tiles * n_tok;
    int64_t want = (2 * b200_sm_count() + base - 1) / base;
    int64_t maxs = (n_kv + 31) / 32;
    if (maxs > FA_MAX_CLUSTER) maxs = FA_MAX_CLUSTER;
    if (want > maxs) want = maxs;
    if (want < 1) want = 1;
    int64_t len = (n_kv + want - 1) / want;
    len = (len + 7) / 8 * 8;
    *split_len = (int)len;
    return (int)((n_kv + len - 1) / len);
}

// The splits merge inside their cluster: the attention needs no global workspace any more.  The entry point stays for callers
// that size one (0 bytes; a null workspace is accepted).
extern "C" int64_t b200_flash_attn_workspace(int64_t dv, int64_t n_head, int64_t n_tok, int64_t n_kv) {
    (void)dv; (void)n_head; (void)n_tok; (void)n_kv;
    return 0;
}

template <int D, int KVT, int G>
static int fa_launch(const float * q, int64_t q_ts, int64_t q_hs, const void * k, int64_t k_rs, int64_t k_hs,
                     const void * v, int64_t v_rs, int64_t v_hs, const void * mask, int64_t mask_rs, float * dst,
                     int64_t n_head, int64_t n_head_kv, int64_t n_tok, int64_t n_kv, float scale, float max_bias, float softcap, cudaStream_t st, const FaFuse & fu) {
    int split_len = 0;
    const int n_tiles = (int)(n_head / G);
    const int n_splits = fa_splits(n_tiles, n_tok, n_kv, &split_len);
    const int nh_log2 = 1 << (int)floor(log2((double)n_head));
    const float m0 = powf(2.0f, -(max_bias) / (float)nh_log2), m1 = powf(2.0f, -(max_bias / 2.0f) / (float)nh_log2);
    if (softcap != 0.0f) scale /= softcap;
    dim3 grid((unsigned)n_splits, (unsigned)n_tiles, (unsigned)n_tok);
    static const bool no_lean = getenv("B200_FA_NO_LEAN") != nullptr;
    const bool lean = !no_lean && fu.enabled && fu.tab_mode == 1 && fu.rope_tab && mask && max_bias == 0.0f && softcap == 0.0f && n_tok == 1;
    auto kern = lean ? fattn_vec_kernel<D, KVT, G, 1> : fattn_vec_kernel<D, KVT, G, 0>;
    if (n_splits > 8) B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    B200_CUDA(b200_launch_pdl_cluster(kern, grid, dim3(FA_WARPS * 32), 0, st, (unsigned)n_splits, q, q_ts, q_hs, (const uint8_t *)k, k_rs, k_hs,
        (const uint8_t *)v, v_rs, v_hs, (const uint16_t *)mask, mask_rs, dst, (int)n_head, (int)n_head_kv, (int)n_kv, split_len, n_splits,
        scale, max_bias, softcap, m0, m1, nh_log2, fu));
    b200_count_launch();
    return B200_OK;
}

bool b200_fattn_tc_supported(int kv_type, int64_t dk, int64_t dv, int64_t n_tok, int64_t n_kv, float max_bias);
int  b200_fattn_tc(const float * q, int64_t q_ts, int64_t q_hs, const void * k, int64_t k_rs, int64_t k_hs, const void * v, int64_t v_rs, int64_t v_hs,
                   const void * mask, int64_t mask_rs, float * dst, int kv_type, int64_t d, int64_t n_head, int64_t n_head_kv, int64_t n_tok, int64_t n_kv,
                   float scale, float softcap, void * stream);

static int fa_dispatch(const float * q, int64_t q_ts, int64_t q_hs, const void * k, int64_t k_rs, int64_t k_hs,
                                   const void * v, int64_t v_rs, int64_t v_hs, const void * mask, int64_t mask_rs, float * dst,
                                   int kv_type, int64_t dk, int64_t dv, int64_t n_head, int64_t n_head_kv, int64_t n_tok, int64_t n_kv,
                                   float scale, float max_bias, float softcap, void * stream, const FaFuse & fu) {
    if (!q || !k || !v || !dst) { b200_set_error("flash_attn: null pointer"); return B200_ERR_INVALID; }
    if (dk != dv || (dk != 64 && dk != 128)) { b200_set_error("flash_attn: head size %lld/%lld unsupported (64 or 128)", (long long)dk, (long long)dv); return B200_ERR_UNSUPPORTED; }
    if (kv_type != B200_TYPE_F16 && kv_type != B200_TYPE_Q8_0) { b200_set_error("flash_attn: kv type %d unsupported", kv_type); return B200_ERR_UNSUPPORTED; }
    if (n_head_kv <= 0 || n_head % n_head_kv != 0 || n_tok <= 0 || n_kv <= 0) { b200_set_error("flash_attn: bad head counts"); return B200_ERR_INVALID; }
    if (((uintptr_t)q & 15) || (q_ts & 3) || (q_hs & 3)) { b200_set_error("flash_attn: q must be 16-byte aligned"); return B200_ERR_INVALID; }
    if (kv_type == B200_TYPE_F16 && ((((uintptr_t)k | (uintptr_t)v) & 15) || ((k_rs | k_hs | v_rs | v_hs) & 15))) { b200_set_error("flash_attn: f16 K/V rows must be 16-byte aligned"); return B200_ERR_INVALID; }
    if (n_tok > 65535) { b200_set_error("flash_attn: n_tok * n_head too large for one launch"); return B200_ERR_UNSUPPORTED; }
    // multi-token batches (prefill, big verify batches): the tensor-core kernel (fattn_tc.cu) — K / V read once per 128 query tokens.
    // Head 128 from 16 tokens, head 64 from the minimum its sweep measured (FT_MIN_TOK_D64); fewer tokens (speculative verify
    // batches), the fused decode launch and ALiBi stay on the vector kernel below
    if (!fu.enabled && b200_fattn_tc_supported(kv_type, dk, dv, n_tok, n_kv, max_bias) && (!mask || ((mask_rs & 7) == 0 && ((uintptr_t)mask & 15) == 0)) &&
        (kv_type != B200_TYPE_F16 || (((k_rs | k_hs | v_rs | v_hs) & 15) == 0)))
        return b200_fattn_tc(q, q_ts, q_hs, k, k_rs, k_hs, v, v_rs, v_hs, mask, mask_rs, dst, kv_type, dk, n_head, n_head_kv, n_tok, n_kv, scale, softcap, stream);
    const int64_t gq = n_head / n_head_kv;
    // query heads per CTA.  G = 4 halves the K/V reads from L2 but leaves half as many CTAs to keep loads in flight: on an H100 SXM
    // (400 W) Llama-3-8B decode ran 407 tok/s with G = 4 (8 tiles x 16 splits, one CTA per SM) and 415 tok/s with G = 2 (16 x 16)
    const int G = gq % 2 == 0 ? 2 : 1;
    cudaStream_t st = (cudaStream_t)stream;
#define FA_CASE(DD, KK, GG) return fa_launch<DD, KK, GG>(q, q_ts, q_hs, k, k_rs, k_hs, v, v_rs, v_hs, mask, mask_rs, dst, n_head, n_head_kv, n_tok, n_kv, scale, max_bias, softcap, st, fu)
    if (dk == 128) {
        if (kv_type == B200_TYPE_F16) { if (G == 2) FA_CASE(128, B200_TYPE_F16, 2); FA_CASE(128, B200_TYPE_F16, 1); }
        else                          { if (G == 2) FA_CASE(128, B200_TYPE_Q8_0, 2); FA_CASE(128, B200_TYPE_Q8_0, 1); }
    } else {
        if (kv_type == B200_TYPE_F16) { if (G == 2) FA_CASE(64, B200_TYPE_F16, 2); FA_CASE(64, B200_TYPE_F16, 1); }
        else                          { if (G == 2) FA_CASE(64, B200_TYPE_Q8_0, 2); FA_CASE(64, B200_TYPE_Q8_0, 1); }
    }
#undef FA_CASE
    return B200_ERR_UNSUPPORTED;
}

extern "C" int b200_flash_attn_ext(const float * q, int64_t q_ts, int64_t q_hs, const void * k, int64_t k_rs, int64_t k_hs,
                                   const void * v, int64_t v_rs, int64_t v_hs, const void * mask, int64_t mask_rs, float * dst,
                                   int kv_type, int64_t dk, int64_t dv, int64_t n_head, int64_t n_head_kv, int64_t n_tok, int64_t n_kv,
                                   float scale, float max_bias, float softcap, void * workspace, void * stream) {
    (void)workspace;                          // no longer needed: the splits merge inside their cluster
    FaFuse fu; memset(&fu, 0, sizeof(fu));
    return fa_dispatch(q, q_ts, q_hs, k, k_rs, k_hs, v, v_rs, v_hs, mask, mask_rs, dst, kv_type, dk, dv, n_head, n_head_kv, n_tok, n_kv, scale, max_bias, softcap, stream, fu);
}

extern "C" int b200_rope_kv_flash_attn2(const float * q_src, float * q_dst, const float * k_new, const float * v_new, const int32_t * pos, const float * ff,
                                        const int64_t * k_ids, const int64_t * v_ids, void * k_cache, void * v_cache, int kv_type,
                                        int64_t k_rs, int64_t k_hs, int64_t v_rs, int64_t v_hs, const void * mask, float * dst,
                                        int64_t hd, int64_t n_head, int64_t n_head_kv, int64_t n_kv, const b200_rope_params * p,
                                        float scale, float max_bias, float softcap, void * workspace, float * rope_tab, int tab_mode, void * stream);
// decode token: rope(q), rope(k) -> K cache cell, v -> V cache cell, attention over n_kv cells — one launch (see FaFuse)
extern "C" int b200_rope_kv_flash_attn(const float * q_src, float * q_dst, const float * k_new, const float * v_new, const int32_t * pos, const float * ff,
                                       const int64_t * k_ids, const int64_t * v_ids, void * k_cache, void * v_cache, int kv_type,
                                       int64_t k_rs, int64_t k_hs, int64_t v_rs, int64_t v_hs, const void * mask, float * dst,
                                       int64_t hd, int64_t n_head, int64_t n_head_kv, int64_t n_kv, const b200_rope_params * p,
                                       float scale, float max_bias, float softcap, void * workspace, void * stream) {
    return b200_rope_kv_flash_attn2(q_src, q_dst, k_new, v_new, pos, ff, k_ids, v_ids, k_cache, v_cache, kv_type, k_rs, k_hs, v_rs, v_hs, mask, dst, hd, n_head, n_head_kv, n_kv, p,
                                    scale, max_bias, softcap, workspace, nullptr, 0, stream);
}
// ... with a per-token cos/sin table shared by the layers: rope_tab = 2 * head_dim floats of scratch; tab_mode 0 = this launch computes
// the table (and stores it), 1 = an earlier launch of the same token (same pos, same rope parameters) did
extern "C" int b200_rope_kv_flash_attn2(const float * q_src, float * q_dst, const float * k_new, const float * v_new, const int32_t * pos, const float * ff,
                                        const int64_t * k_ids, const int64_t * v_ids, void * k_cache, void * v_cache, int kv_type,
                                        int64_t k_rs, int64_t k_hs, int64_t v_rs, int64_t v_hs, const void * mask, float * dst,
                                        int64_t hd, int64_t n_head, int64_t n_head_kv, int64_t n_kv, const b200_rope_params * p,
                                        float scale, float max_bias, float softcap, void * workspace, float * rope_tab, int tab_mode, void * stream) {
    if (!q_src || !q_dst || !k_new || !v_new || !pos || !k_ids || !v_ids || !k_cache || !v_cache || !dst || !p) { b200_set_error("rope_kv_flash_attn: null pointer"); return B200_ERR_INVALID; }
    if ((p->mode & ~2) || p->n_dims > hd || p->n_dims % 8 != 0 || (p->mode == 2 && p->n_dims % 16 != 0)) { b200_set_error("rope_kv_flash_attn: rope mode / n_dims unsupported"); return B200_ERR_UNSUPPORTED; }
    const int64_t hs = kv_type == B200_TYPE_F16 ? hd * 2 : hd / 32 * 34;
    if (k_hs != hs || v_hs != hs) { b200_set_error("rope_kv_flash_attn: heads must be contiguous inside a cache cell"); return B200_ERR_INVALID; }
    if (((uintptr_t)q_src | (uintptr_t)q_dst | (uintptr_t)k_new | (uintptr_t)v_new | (uintptr_t)rope_tab) & 15) { b200_set_error("rope_kv_flash_attn: 16-byte alignment required"); return B200_ERR_INVALID; }
    (void)workspace;
    FaFuse fu; memset(&fu, 0, sizeof(fu));
    fu.q_src = q_src; fu.q_dst = q_dst; fu.k_new = k_new; fu.v_new = v_new; fu.pos = pos; fu.ff = ff; fu.k_ids = k_ids; fu.v_ids = v_ids;
    fu.rp = rope_host_params(p); fu.enabled = 1; fu.trace = b200_trace_on() ? 1 : 0;
    fu.rope_tab = rope_tab; fu.tab_mode = rope_tab ? tab_mode : 0;
    return fa_dispatch(q_dst, hd * n_head, hd, k_cache, k_rs, k_hs, v_cache, v_rs, v_hs, mask, 0, dst, kv_type, hd, hd, n_head, n_head_kv, 1, n_kv,
                       scale, max_bias, softcap, stream, fu);
}
