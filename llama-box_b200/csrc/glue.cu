// glue.cu — the small elementwise ops that keep a whole transformer layer on the device (sm_90a).
// Replaces k_bin_bcast (ggml-cuda/binbcast.cu:26-93), unary_gated_op_kernel (unary.cu:209-230),
// k_get_rows_float (getrows.cu:5-67), cpy_flt f32->f16 (cpy.cu:11-64) and argmax (argmax.cu).
// All HBM/launch-bound: 16-byte vector accesses, grid sized to the data, f32 math in the oracle's
// operation order (ggml-cpu/binary-ops.cpp, vec.h:691).
#include "common.cuh"

template <int OP>
__global__ void __launch_bounds__(256) bin_bcast_kernel(const float * __restrict__ a, const float * __restrict__ b, float * __restrict__ y,
                                                        int64_t ncols, int64_t nrows, int64_t b_rows) {
    pdl_wait();
    const int64_t n4 = ncols / 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4 * nrows; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / n4, c = i % n4;
        const float4 va = ((const float4 *)a)[i];
        const float4 vb = ((const float4 *)b)[(r % b_rows) * n4 + c];
        float4 o;
        if (OP == 0) { o.x = __fadd_rn(va.x, vb.x); o.y = __fadd_rn(va.y, vb.y); o.z = __fadd_rn(va.z, vb.z); o.w = __fadd_rn(va.w, vb.w); }
        else         { o.x = __fmul_rn(va.x, vb.x); o.y = __fmul_rn(va.y, vb.y); o.z = __fmul_rn(va.z, vb.z); o.w = __fmul_rn(va.w, vb.w); }
        ((float4 *)y)[i] = o;
    }
    pdl_trigger();
}

static int grid_for(int64_t work, int threads) {
    int64_t g = (work + threads - 1) / threads;
    const int64_t cap = (int64_t)b200_sm_count() * 8;
    if (g > cap) g = cap;
    return (int)(g < 1 ? 1 : g);
}

static int bin_launch(int op, const float * a, const float * b, float * y, int64_t ncols, int64_t nrows, int64_t b_rows, cudaStream_t st) {
    if (!a || !b || !y || ncols <= 0 || nrows <= 0 || b_rows <= 0 || ncols % 4 != 0 || (((uintptr_t)a | (uintptr_t)b | (uintptr_t)y) & 15)) {
        b200_set_error("add/mul: ncols must be a multiple of 4 and pointers 16-byte aligned"); return B200_ERR_INVALID; }
    const int g = grid_for(ncols / 4 * nrows, 256);
    if (op == 0) bin_bcast_kernel<0><<<g, 256, 0, st>>>(a, b, y, ncols, nrows, b_rows);
    else         bin_bcast_kernel<1><<<g, 256, 0, st>>>(a, b, y, ncols, nrows, b_rows);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
extern "C" int b200_add(const float * a, const float * b, float * y, int64_t ncols, int64_t nrows, int64_t b_rows, void * stream) { return bin_launch(0, a, b, y, ncols, nrows, b_rows, (cudaStream_t)stream); }
extern "C" int b200_mul(const float * a, const float * b, float * y, int64_t ncols, int64_t nrows, int64_t b_rows, void * stream) { return bin_launch(1, a, b, y, ncols, nrows, b_rows, (cudaStream_t)stream); }

__global__ void __launch_bounds__(256) swiglu_kernel(const float * __restrict__ g, const float * __restrict__ u, float * __restrict__ y, int64_t n4) {
    pdl_wait();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 a = ((const float4 *)g)[i], b = ((const float4 *)u)[i];
        float4 o;
        o.x = __fmul_rn(silu_x86(a.x), b.x); o.y = __fmul_rn(silu_x86(a.y), b.y);
        o.z = __fmul_rn(silu_x86(a.z), b.z); o.w = __fmul_rn(silu_x86(a.w), b.w);
        ((float4 *)y)[i] = o;
    }
    pdl_trigger();
}
extern "C" int b200_swiglu(const float * gate, const float * up, float * y, int64_t n, void * stream) {
    if (!gate || !up || !y || n <= 0 || n % 4 != 0 || (((uintptr_t)gate | (uintptr_t)up | (uintptr_t)y) & 15)) { b200_set_error("swiglu: n must be a multiple of 4, pointers aligned"); return B200_ERR_INVALID; }
    swiglu_kernel<<<grid_for(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(gate, up, y, n / 4);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

__global__ void __launch_bounds__(256) get_rows_kernel(const float * __restrict__ src, int64_t srs, const int32_t * __restrict__ ids, float * __restrict__ dst, int64_t n4) {
    pdl_wait();
    const int64_t r = blockIdx.y;
    const float4 * s = (const float4 *)(src + (int64_t)ids[r] * srs);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) ((float4 *)dst)[r * n4 + i] = s[i];
    pdl_trigger();
}
extern "C" int b200_get_rows_f32(const float * src, int64_t src_row_stride, const int32_t * ids, float * dst, int64_t ncols, int64_t n_ids, void * stream) {
    if (!src || !ids || !dst || ncols <= 0 || ncols % 4 != 0 || (src_row_stride & 3) || (((uintptr_t)src | (uintptr_t)dst) & 15)) { b200_set_error("get_rows: ncols must be a multiple of 4, pointers aligned"); return B200_ERR_INVALID; }
    if (n_ids <= 0) return B200_OK;
    dim3 grid((unsigned)((ncols / 4 + 255) / 256), (unsigned)n_ids);
    get_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, src_row_stride, ids, dst, ncols / 4);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

__global__ void __launch_bounds__(256) cpy_f16_kernel(const float * __restrict__ s, uint16_t * __restrict__ d, int64_t n) {
    pdl_wait();
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += (int64_t)gridDim.x * blockDim.x * 4) {
        if (i + 3 < n) {
            const float4 v = *(const float4 *)(s + i);
            uint2 o; o.x = f2h_rn(v.x) | ((uint32_t)f2h_rn(v.y) << 16); o.y = f2h_rn(v.z) | ((uint32_t)f2h_rn(v.w) << 16);
            *(uint2 *)(d + i) = o;
        } else for (int64_t j = i; j < n; j++) d[j] = f2h_rn(s[j]);
    }
    pdl_trigger();
}
extern "C" int b200_cpy_f32_f16(const float * src, void * dst, int64_t n, void * stream) {
    if (!src || !dst || n < 0 || ((uintptr_t)src & 15) || ((uintptr_t)dst & 7)) { b200_set_error("cpy_f32_f16: alignment"); return B200_ERR_INVALID; }
    if (n == 0) return B200_OK;
    cpy_f16_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(src, (uint16_t *)dst, n);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// first index of the maximum (sampling's greedy path: llama-sampling.cpp greedy / argmax.cu)
__global__ void __launch_bounds__(1024) argmax_kernel(const float * __restrict__ x, int32_t * __restrict__ out, int64_t n) {
    __shared__ float sv[32]; __shared__ int si[32];
    pdl_wait();
    const float * row = x + (int64_t)blockIdx.x * n;
    float best = -INFINITY; int bi = 0x7fffffff;
    // one row is ~0.5 MB for a 128k vocabulary and a single CTA scans it: keep 8 independent 16-byte loads in flight per thread
    if ((((uintptr_t)row) & 15) == 0 && (n & 3) == 0) {
        const int64_t n4 = n >> 2;
        for (int64_t i0 = threadIdx.x; i0 < n4; i0 += (int64_t)blockDim.x * 8) {
            float4 v[8];
#pragma unroll
            for (int u = 0; u < 8; u++) { const int64_t i = i0 + (int64_t)u * blockDim.x; v[u] = i < n4 ? __ldg((const float4 *)row + i) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY); }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int e = (int)((i0 + (int64_t)u * blockDim.x) * 4);
                const float f[4] = { v[u].x, v[u].y, v[u].z, v[u].w };
#pragma unroll
                for (int c = 0; c < 4; c++) if (f[c] > best || (f[c] == best && e + c < bi)) { best = f[c]; bi = e + c; }
            }
        }
    } else {
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) { const float v = row[i]; if (v > best || (v == best && (int)i < bi)) { best = v; bi = (int)i; } }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, best, o); const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
        if (v2 > best || (v2 == best && i2 < bi)) { best = v2; bi = i2; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        best = threadIdx.x < blockDim.x / 32 ? sv[threadIdx.x] : -INFINITY; bi = threadIdx.x < blockDim.x / 32 ? si[threadIdx.x] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float v2 = __shfl_xor_sync(0xffffffffu, best, o); const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
            if (v2 > best || (v2 == best && i2 < bi)) { best = v2; bi = i2; }
        }
        if (threadIdx.x == 0) out[blockIdx.x] = bi;
    }
    pdl_trigger();
}
extern "C" int b200_argmax_f32(const float * x, int32_t * idx_out, int64_t n, int64_t nrows, void * stream) {
    if (!x || !idx_out || n <= 0 || nrows <= 0) { b200_set_error("argmax: bad arguments"); return B200_ERR_INVALID; }
    argmax_kernel<<<(unsigned)nrows, 1024, 0, (cudaStream_t)stream>>>(x, idx_out, n);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
