// quantize.cu — activation quantisation + RMS_NORM for the decode/prefill hot path (sm_90a).
//
// Replaces quantize_q8_1 (ggml-cuda/quantize.cu:4-48) and rms_norm_f32 (ggml-cuda/norm.cu:107-164),
// but quantises the way the CPU oracle does so integer dot products are bit-identical:
//   q8_K  — ggml-quants.c:2555-2592 (quantize_row_q8_K_ref; x86 uses it: arch/x86/quants.c:493-495)
//   q8_0  — ggml-cpu/arch/x86/quants.c:290-360 (d = max/127 -> f16, id = 127/max, RNE)
// HBM-bound elementwise work: one warp per 256 elements, 32-byte loads per lane, 8-byte stores.
#include "common.cuh"

#include "actquant.cuh"

__global__ void __launch_bounds__(128) quantize_act_kernel(const float * __restrict__ x, int64_t x_col_stride,
                                                           void * __restrict__ act, int kind, int64_t k, int64_t k_valid) {
    pdl_wait();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t blk = (int64_t)blockIdx.x * 4 + warp;
    const int64_t col = blockIdx.y;
    if (blk * 256 >= k) return;
    float v[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    if (blk * 256 + lane * 8 < k_valid) {                    // elements past k_valid do not exist in x: zero (padded weight layout)
        const float4 * p = (const float4 *)(x + col * x_col_stride + blk * 256 + lane * 8);
        const float4 a = p[0], b = p[1];
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
    ActOut o = act_sections(act, kind, k, col);
    if (kind == 0) warp_quant_q8K(v, o, blk, lane); else warp_quant_q80(v, o, blk, lane);
    pdl_trigger();
}

extern "C" int b200_act_kind_for(int t) {
    switch (t) {
        case B200_TYPE_Q4_K: case B200_TYPE_Q5_K: case B200_TYPE_Q6_K: return 0;
        case B200_TYPE_Q4_0: case B200_TYPE_Q5_0: case B200_TYPE_Q8_0: return 1;
        default: return B200_ERR_UNSUPPORTED;
    }
}
extern "C" int64_t b200_act_col_bytes(int kind, int64_t k)   { return act_col_bytes(kind, k); }
extern "C" int64_t b200_act_d_offset(int kind, int64_t k)    { return act_d_off(kind, k); }
extern "C" int64_t b200_act_bsum_offset(int kind, int64_t k) { return act_bsum_off(kind, k); }

extern "C" int b200_quantize_act(int kind, const float * x, int64_t x_col_stride, void * act, int64_t k, int64_t ncols, void * stream) {
    return b200_quantize_act2(kind, x, x_col_stride, act, k, k, ncols, stream);
}
extern "C" int b200_quantize_act2(int kind, const float * x, int64_t x_col_stride, void * act, int64_t k, int64_t k_valid, int64_t ncols, void * stream) {
    if ((kind != 0 && kind != 1) || k <= 0 || k % 256 != 0 || ncols <= 0 || k_valid <= 0 || k_valid > k || k_valid % 8 != 0) { b200_set_error("quantize_act: k must be a positive multiple of 256 (k_valid a multiple of 8)"); return B200_ERR_INVALID; }
    if (((uintptr_t)x | (uintptr_t)act) & 15 || (x_col_stride & 3)) { b200_set_error("quantize_act: pointers must be 16-byte aligned"); return B200_ERR_INVALID; }
    dim3 grid((unsigned)((k / 256 + 3) / 4), (unsigned)ncols);
    quantize_act_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(x, x_col_stride, act, kind, k, k_valid);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// ------------------------------------------------------------------------------------------------
// RMS_NORM (+MUL) — oracle numerics (ggml-cpu/ops.cpp:4164-4183): f32 squares summed in double,
// scale = 1/sqrtf(mean + eps), y = (x*scale)*w.  One CTA per row; the row is kept in shared
// memory between the reduction pass and the scaling pass so x is read from HBM once
// (the reference reads it twice: norm.cu:107-164).
// Optional fused activation quantisation of the normalised row (up to two act kinds).
// ------------------------------------------------------------------------------------------------
template <int NT>
__global__ void __launch_bounds__(NT) rms_norm_kernel(const float * __restrict__ x, const float * __restrict__ w, float * __restrict__ y,
                                                      void * __restrict__ act0, int kind0, void * __restrict__ act1, int kind1,
                                                      int64_t ncols, int64_t x_row_stride, int64_t y_row_stride, float eps) {
    extern __shared__ __align__(16) float row[];
    __shared__ double red[NT / 32];
    __shared__ float s_scale;
    pdl_wait();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t r = blockIdx.x;
    const float * xr = x + r * x_row_stride;
    double acc = 0.0;
    for (int64_t i = tid * 4; i < ncols; i += NT * 4) {
        const float4 v = *(const float4 *)(xr + i);
        *(float4 *)(row + i) = v;
        acc += (double)__fmul_rn(v.x, v.x); acc += (double)__fmul_rn(v.y, v.y);
        acc += (double)__fmul_rn(v.z, v.z); acc += (double)__fmul_rn(v.w, v.w);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) red[warp] = acc;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int i = 0; i < NT / 32; i++) t += red[i];
        const float mean = (float)(t / (double)ncols);
        s_scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, eps)));
    }
    __syncthreads();
    const float scale = s_scale;
    if (act0 == nullptr) {
        float * yr = y + r * y_row_stride;
        for (int64_t i = tid * 4; i < ncols; i += NT * 4) {
            float4 v = *(float4 *)(row + i);
            v.x = __fmul_rn(v.x, scale); v.y = __fmul_rn(v.y, scale); v.z = __fmul_rn(v.z, scale); v.w = __fmul_rn(v.w, scale);
            if (w) { const float4 ww = *(const float4 *)(w + i); v.x = __fmul_rn(v.x, ww.x); v.y = __fmul_rn(v.y, ww.y); v.z = __fmul_rn(v.z, ww.z); v.w = __fmul_rn(v.w, ww.w); }
            *(float4 *)(yr + i) = v;
        }
    } else {
        // one warp per 256 elements: scale, (write f32), quantise
        ActOut o0 = act_sections(act0, kind0, ncols, r);
        ActOut o1 = act1 ? act_sections(act1, kind1, ncols, r) : o0;
        for (int64_t blk = warp; blk * 256 < ncols; blk += NT / 32) {
            const int64_t i = blk * 256 + lane * 8;
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; j++) { v[j] = __fmul_rn(row[i + j], scale); if (w) v[j] = __fmul_rn(v[j], w[i + j]); }
            if (y) {
                float * yr = y + r * y_row_stride;
                *(float4 *)(yr + i)     = make_float4(v[0], v[1], v[2], v[3]);
                *(float4 *)(yr + i + 4) = make_float4(v[4], v[5], v[6], v[7]);
            }
            if (kind0 == 0) warp_quant_q8K(v, o0, blk, lane); else warp_quant_q80(v, o0, blk, lane);
            if (act1) { if (kind1 == 0) warp_quant_q8K(v, o1, blk, lane); else warp_quant_q80(v, o1, blk, lane); }
        }
    }
    pdl_trigger();
}

static int launch_rms(const float * x, const float * w, float * y, void * act0, int kind0, void * act1, int kind1,
                      int64_t ncols, int64_t nrows, int64_t xs, int64_t ys, float eps, cudaStream_t st) {
    if (ncols <= 0 || nrows <= 0 || ncols % 4 != 0) { b200_set_error("rms_norm: ncols must be a positive multiple of 4"); return B200_ERR_INVALID; }
    if ((((uintptr_t)x | (uintptr_t)y | (uintptr_t)w) & 15) || (xs & 3) || (ys & 3)) { b200_set_error("rms_norm: 16-byte alignment required"); return B200_ERR_INVALID; }
    const size_t smem = (size_t)ncols * sizeof(float);
    if (smem > 200 * 1024) { b200_set_error("rms_norm: row of %lld floats exceeds shared memory", (long long)ncols); return B200_ERR_UNSUPPORTED; }
    if (ncols >= 2048) {
        static bool attr[64] = { false };               // per device
        int dev = 0; cudaGetDevice(&dev);
        if (!attr[dev & 63]) { cudaFuncSetAttribute(rms_norm_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); attr[dev & 63] = true; }
        rms_norm_kernel<512><<<(unsigned)nrows, 512, smem, st>>>(x, w, y, act0, kind0, act1, kind1, ncols, xs, ys, eps);
    } else {
        rms_norm_kernel<128><<<(unsigned)nrows, 128, smem, st>>>(x, w, y, act0, kind0, act1, kind1, ncols, xs, ys, eps);
    }
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_rms_norm(const float * x, const float * w, float * y, int64_t ncols, int64_t nrows,
                             int64_t x_row_stride, int64_t y_row_stride, float eps, void * stream) {
    if (!x || !y) { b200_set_error("rms_norm: null pointer"); return B200_ERR_INVALID; }
    return launch_rms(x, w, y, nullptr, 0, nullptr, 0, ncols, nrows, x_row_stride, y_row_stride, eps, (cudaStream_t)stream);
}

extern "C" int b200_rms_norm_quantize(const float * x, const float * w, float * y, void * act0, int kind0, void * act1, int kind1,
                                      int64_t k, int64_t ncols, float eps, void * stream) {
    if (!x || !act0 || k % 256 != 0) { b200_set_error("rms_norm_quantize: k must be a multiple of 256"); return B200_ERR_INVALID; }
    return launch_rms(x, w, y, act0, kind0, act1, kind1, k, ncols, k, k, eps, (cudaStream_t)stream);
}
