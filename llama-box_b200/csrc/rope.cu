// rope.cu — ROPE, SET_ROWS (KV store) and their fused decode form (sm_90a).
//
// Replaces rope_norm / rope_neox (ggml-cuda/rope.cu:40-122,324-446), k_set_rows / k_set_rows_quant
// (ggml-cuda/set-rows.cu:13-160) and quantize_f32_q8_0_block (cpy-utils.cuh:145-162).
// Numerics follow the CPU oracle, not ggml-cuda:
//   * theta for pair i is the oracle's sequential f32 product pos*ts*ts*...  (ops.cpp:6077-6086);
//     thread i replays exactly those i multiplications, theta_scale / YaRN constants are computed on
//     the host with the same libm calls the oracle makes (powf/logf) — ggml-cuda instead evaluates
//     pos*powf(ts, i), which differs in the last bits;
//   * Q8_0 rows use the x86 oracle quantiser (RNE, id = 127/max), F16 rows use RNE conversion.
// One CTA per token: the cos/sin table is built once in shared memory and reused by every head.
#include "common.cuh"
#include "ropeutil.cuh"
#include <math.h>

RopeDev rope_host_params(const b200_rope_params * p) {
    RopeDev d;
    d.n_dims = p->n_dims;
    d.neox   = (p->mode & 2) != 0;
    d.theta_scale = powf(p->freq_base, -2.0f / (float)p->n_dims);                 // ops.cpp:6198
    d.freq_scale  = p->freq_scale;
    d.ext_factor  = p->ext_factor;
    d.mscale      = p->attn_factor;
    if (p->ext_factor != 0.0f) d.mscale *= 1.0f + 0.1f * logf(1.0f / p->freq_scale);   // ops.cpp:6068
    // ggml.c:4082-4095
    auto corr = [&](float n_rot) { return (float)p->n_dims * logf((float)p->n_ctx_orig / (n_rot * 2.0f * (float)M_PI)) / (2.0f * logf(p->freq_base)); };
    float lo = floorf(corr(p->beta_fast)), hi = ceilf(corr(p->beta_slow));
    d.corr_lo = lo < 0.0f ? 0.0f : lo;
    d.corr_hi = hi > (float)(p->n_dims - 1) ? (float)(p->n_dims - 1) : hi;
    return d;
}

__global__ void __launch_bounds__(256) rope_kernel(const float * __restrict__ x, float * __restrict__ y, const int32_t * __restrict__ pos,
                                                   const float * __restrict__ ff, int64_t hd, int64_t n_head,
                                                   int64_t xhs, int64_t xts, int64_t yhs, int64_t yts, RopeDev rp) {
    extern __shared__ float cs[];
    pdl_wait();
    const int64_t t = blockIdx.x;
    rope_table(cs, pos[t], ff, rp, threadIdx.x, blockDim.x);
    __syncthreads();
    const int half = rp.n_dims / 2;
    const int64_t work = n_head * (hd / 2);
    for (int64_t w = threadIdx.x; w < work; w += blockDim.x) {
        const int64_t h = w / (hd / 2); const int i = (int)(w % (hd / 2));
        const float * s = x + t * xts + h * xhs; float * d = y + t * yts + h * yhs;
        if (i < half) rope_pair(s, d, i, cs, rp);
        else { const int e = rp.n_dims + 2 * (i - half); d[e] = s[e]; d[e + 1] = s[e + 1]; }   // pass-through dims
    }
    pdl_trigger();
}

extern "C" int b200_rope(const float * x, float * y, const int32_t * pos, const float * ff,
                         int64_t hd, int64_t n_head, int64_t n_tok, int64_t xhs, int64_t xts, int64_t yhs, int64_t yts,
                         const b200_rope_params * p, void * stream) {
    if (!x || !y || !pos || !p || p->n_dims <= 0 || p->n_dims > hd || (p->n_dims & 1) || (hd & 1)) { b200_set_error("rope: bad arguments"); return B200_ERR_INVALID; }
    if (p->mode & ~2) { b200_set_error("rope: only NORM (0) and NEOX (2) modes are on the hot path"); return B200_ERR_UNSUPPORTED; }
    if (n_tok <= 0) return B200_OK;
    rope_kernel<<<(unsigned)n_tok, 256, (size_t)p->n_dims * sizeof(float), (cudaStream_t)stream>>>(x, y, pos, ff, hd, n_head, xhs, xts, yhs, yts, rope_host_params(p));
    B200_LAUNCH_CHECK();
    return B200_OK;
}

__global__ void __launch_bounds__(128) set_rows_kernel(const float * __restrict__ src, int64_t src_row_stride, const int64_t * __restrict__ ids,
                                                       void * __restrict__ dst, int dst_type, int64_t dst_row_stride, int64_t ncols) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t r = blockIdx.y;
    const int64_t e = ((int64_t)blockIdx.x * 4 + (threadIdx.x >> 5)) * 256 + lane * 8;
    if (e - lane * 8 >= ncols) return;                      // whole warp out of range
    float v[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    const bool in = e < ncols;                              // ncols % 32 == 0 keeps q8_0 groups whole
    if (in) {
        const float4 a = *(const float4 *)(src + r * src_row_stride + e), b = *(const float4 *)(src + r * src_row_stride + e + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
    uint8_t * drow = (uint8_t *)dst + ids[r] * dst_row_stride;
    store8(drow, dst_type, e, v, lane, in);   // all 32 lanes take part in the q8_0 group reductions
    pdl_trigger();
}

extern "C" int b200_set_rows(const float * src, int64_t src_row_stride, const int64_t * ids, void * dst, int dst_type, int64_t dst_row_stride,
                             int64_t ncols, int64_t nrows, void * stream) {
    if (dst_type != B200_TYPE_F32 && dst_type != B200_TYPE_F16 && dst_type != B200_TYPE_Q8_0) { b200_set_error("set_rows: dst type %d unsupported", dst_type); return B200_ERR_UNSUPPORTED; }
    if (!src || !ids || !dst || ncols <= 0 || ncols % 32 != 0 || (src_row_stride & 3) || ((uintptr_t)src & 15)) { b200_set_error("set_rows: ncols must be a multiple of 32, src 16-byte aligned"); return B200_ERR_INVALID; }
    if (dst_type != B200_TYPE_Q8_0 && (((uintptr_t)dst | (uintptr_t)dst_row_stride) & 15)) { b200_set_error("set_rows: dst rows must be 16-byte aligned"); return B200_ERR_INVALID; }
    if (nrows <= 0) return B200_OK;
    dim3 grid((unsigned)((ncols + 1023) / 1024), (unsigned)nrows);
    set_rows_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(src, src_row_stride, ids, dst, dst_type, dst_row_stride, ncols);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// ---- fused: rope(q) in place, rope(k) -> K cache, v -> V cache --------------------------------
// q [n_tok][n_head][hd], k/v [n_tok][n_head_kv][hd] contiguous f32.  One CTA (256 threads) per token.
__global__ void __launch_bounds__(256) rope_kv_store_kernel(const float * q, float * qo, const float * __restrict__ k, const float * __restrict__ v,
                                                            const int32_t * __restrict__ pos, const float * __restrict__ ff,
                                                            const int64_t * __restrict__ k_ids, const int64_t * __restrict__ v_ids,
                                                            void * __restrict__ kc, void * __restrict__ vc, int kv_type, int64_t k_row_stride, int64_t v_row_stride,
                                                            int64_t hd, int64_t n_head, int64_t n_head_kv, RopeDev rp) {
    extern __shared__ __align__(16) float sm[];
    float * cs = sm;                          // n_dims floats
    float * kr = sm + rp.n_dims;              // roped k row: n_head_kv*hd floats
    pdl_wait();
    const int64_t t = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    rope_table(cs, pos[t], ff, rp, tid, blockDim.x);
    __syncthreads();
    const int half = rp.n_dims / 2;
    const int64_t hp = hd / 2;
    const float * qt = q + t * n_head * hd; float * qd = qo + t * n_head * hd;
    for (int64_t w = tid; w < n_head * hp; w += blockDim.x) {
        const int64_t h = w / hp; const int i = (int)(w % hp);
        if (i < half) rope_pair(qt + h * hd, qd + h * hd, i, cs, rp);
        else if (qd != qt) { const int e = rp.n_dims + 2 * (i - half); qd[h * hd + e] = qt[h * hd + e]; qd[h * hd + e + 1] = qt[h * hd + e + 1]; }
    }
    const float * kt = k + t * n_head_kv * hd;
    for (int64_t w = tid; w < n_head_kv * hp; w += blockDim.x) {
        const int64_t h = w / hp; const int i = (int)(w % hp);
        if (i < half) rope_pair(kt + h * hd, kr + h * hd, i, cs, rp);
        else { const int e = rp.n_dims + 2 * (i - half); kr[h * hd + e] = kt[h * hd + e]; kr[h * hd + e + 1] = kt[h * hd + e + 1]; }
    }
    __syncthreads();
    const int64_t n = n_head_kv * hd;          // multiple of 256 required by the host wrapper
    uint8_t * krow = (uint8_t *)kc + k_ids[t] * k_row_stride;
    uint8_t * vrow = (uint8_t *)vc + v_ids[t] * v_row_stride;
    const float * vt = v + t * n;
    for (int64_t e = (int64_t)warp * 256 + lane * 8; e < n; e += (blockDim.x / 32) * 256) {
        float a[8], b[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { a[j] = kr[e + j]; b[j] = vt[e + j]; }
        store8(krow, kv_type, e, a, lane);
        store8(vrow, kv_type, e, b, lane);
    }
    pdl_trigger();
}

extern "C" int b200_rope_kv_store2(const float * q_src, float * q_dst, const float * k, const float * v, const int32_t * pos, const float * ff,
                                   const int64_t * k_ids, const int64_t * v_ids, void * k_cache, void * v_cache, int kv_type,
                                   int64_t k_row_stride, int64_t v_row_stride, int64_t hd, int64_t n_head, int64_t n_head_kv, int64_t n_tok,
                                   const b200_rope_params * p, void * stream) {
    if (!q_src || !q_dst || !k || !v || !pos || !k_ids || !v_ids || !k_cache || !v_cache || !p) { b200_set_error("rope_kv_store: null pointer"); return B200_ERR_INVALID; }
    if (kv_type != B200_TYPE_F16 && kv_type != B200_TYPE_Q8_0) { b200_set_error("rope_kv_store: kv type %d unsupported", kv_type); return B200_ERR_UNSUPPORTED; }
    if (p->mode & ~2) { b200_set_error("rope_kv_store: only NORM/NEOX"); return B200_ERR_UNSUPPORTED; }
    if ((n_head_kv * hd) % 256 != 0 || p->n_dims > hd || (p->n_dims & 1)) { b200_set_error("rope_kv_store: n_head_kv*head_dim must be a multiple of 256"); return B200_ERR_INVALID; }
    if (n_tok <= 0) return B200_OK;
    const size_t smem = ((size_t)p->n_dims + (size_t)(n_head_kv * hd)) * sizeof(float);
    B200_CUDA(b200_launch_pdl(rope_kv_store_kernel, dim3((unsigned)n_tok), dim3(256), smem, (cudaStream_t)stream, q_src, q_dst, k, v, pos, ff, k_ids, v_ids, k_cache, v_cache,
                              kv_type, k_row_stride, v_row_stride, hd, n_head, n_head_kv, rope_host_params(p)));
    b200_count_launch();
    return B200_OK;
}

extern "C" int b200_rope_kv_store(float * q, const float * k, const float * v, const int32_t * pos, const float * ff,
                                  const int64_t * kv_ids, void * k_cache, void * v_cache, int kv_type, int64_t kv_row_stride,
                                  int64_t hd, int64_t n_head, int64_t n_head_kv, int64_t n_tok, const b200_rope_params * p, void * stream) {
    return b200_rope_kv_store2(q, q, k, v, pos, ff, kv_ids, kv_ids, k_cache, v_cache, kv_type, kv_row_stride, kv_row_stride, hd, n_head, n_head_kv, n_tok, p, stream);
}
