// common.cuh — shared device/host helpers for the sm_90a kernels (our code; no ggml dependency).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/b200_ops.h"

#define B200_WARP 32

// ---- host-side error plumbing -------------------------------------------------------------
void b200_set_error(const char * fmt, ...);
int  b200_check(cudaError_t e, const char * what);       // returns B200_OK / B200_ERR_CUDA
void b200_count_launch(int n = 1);
int  b200_sm_count();                                     // SMs of the current device (cached)
bool b200_pdl_enabled();                                  // programmatic dependent launch (off: GGML_B200_DISABLE_PDL)

// launch with programmatic stream serialization (PDL) so that this kernel's launch latency and prologue overlap the
// previous kernel's tail; every kernel of this library executes griddepcontrol.wait before touching dependent data
#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t b200_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args &&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = b200_pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
// ... as thread-block clusters of cluster_x CTAs along grid.x (grid.x must be a multiple of cluster_x; more than 8 needs the
// kernel's cudaFuncAttributeNonPortableClusterSizeAllowed)
template <typename... KArgs, typename... Args>
inline cudaError_t b200_launch_pdl_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, unsigned cluster_x, Args &&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cluster_x; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = b200_pdl_enabled() ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#endif

#define B200_CUDA(expr) do { int _s = b200_check((expr), #expr); if (_s != B200_OK) return _s; } while (0)
#define B200_LAUNCH_CHECK() do { b200_count_launch(); int _s = b200_check(cudaGetLastError(), "kernel launch"); if (_s != B200_OK) return _s; } while (0)

// ---- block layouts (ggml/src/ggml-common.h:170-175,219-224,295-344) -----------------------
// native (ggml) layouts
struct __align__(2) blk_q4_0 { uint16_t d; uint8_t qs[16]; };                                   // 18
struct __align__(2) blk_q5_0 { uint16_t d; uint8_t qh[4]; uint8_t qs[16]; };                    // 22
struct __align__(2) blk_q8_0 { uint16_t d; int8_t  qs[32]; };                                   // 34
struct __align__(4) blk_q4_K { uint16_t d, dmin; uint8_t sc[12]; uint8_t qs[128]; };            // 144
struct __align__(4) blk_q5_K { uint16_t d, dmin; uint8_t sc[12]; uint8_t qh[32]; uint8_t qs[128]; }; // 176
struct __align__(2) blk_q6_K { uint8_t ql[128]; uint8_t qh[64]; int8_t sc[16]; uint16_t d; };   // 210
static_assert(sizeof(blk_q4_0) == 18 && sizeof(blk_q8_0) == 34 && sizeof(blk_q4_K) == 144 &&
              sizeof(blk_q5_K) == 176 && sizeof(blk_q6_K) == 210, "block sizes");

__host__ __device__ inline int64_t type_block_elems(int t) {
    switch (t) {
        case B200_TYPE_F32: case B200_TYPE_F16: return 1;
        case B200_TYPE_Q4_0: case B200_TYPE_Q5_0: case B200_TYPE_Q8_0: return 32;
        case B200_TYPE_Q4_K: case B200_TYPE_Q5_K: case B200_TYPE_Q6_K: return 256;
        default: return 0;
    }
}
__host__ __device__ inline int64_t type_block_bytes(int t) {
    switch (t) {
        case B200_TYPE_F32: return 4;  case B200_TYPE_F16: return 2;
        case B200_TYPE_Q4_0: return 18; case B200_TYPE_Q5_0: return 22; case B200_TYPE_Q8_0: return 34;
        case B200_TYPE_Q4_K: return 144; case B200_TYPE_Q5_K: return 176; case B200_TYPE_Q6_K: return 210;
        default: return 0;
    }
}

// 32-element block types may have rows that are not a multiple of 256 elements (Qwen2-72B: n_ff = 29568 — the reference quantiser
// then falls back from Q4_K / Q6_K to Q5_0 / Q8_0, llama-quant.cpp:442-470).  The kernels work on 256-element units, so such
// weights are kept in a PRIVATE layout whose rows are padded with zero blocks (d = 0) up to the next multiple of 256.
__host__ __device__ inline bool type_is_block32(int t) { return t == B200_TYPE_Q4_0 || t == B200_TYPE_Q5_0 || t == B200_TYPE_Q8_0; }
__host__ __device__ inline int64_t padded_k(int t, int64_t k) { return type_is_block32(t) ? (k + 255) / 256 * 256 : k; }

// act-buffer geometry (see b200_ops.h)
__host__ __device__ inline int64_t align16(int64_t x) { return (x + 15) & ~(int64_t)15; }
__host__ __device__ inline int64_t act_d_off(int kind, int64_t k)    { (void)kind; return align16(k); }
__host__ __device__ inline int64_t act_bsum_off(int kind, int64_t k) { return act_d_off(kind, k) + align16(4 * (kind == 0 ? k / 256 : k / 32)); }
__host__ __device__ inline int64_t act_col_bytes(int kind, int64_t k) { return act_bsum_off(kind, k) + align16(2 * (kind == 0 ? k / 16 : k / 32)); }

// ---- device helpers -----------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// streaming 16-byte load of weights: read-only path, do not pollute L1 (guide: G13/G14)
__device__ __forceinline__ uint4 ldg_stream16(const void * p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ldg_stream8(const void * p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ldg_nc32(const void * p) { return __ldg((const uint32_t *)p); }
__device__ __forceinline__ uint16_t ldg_nc16(const void * p) { return __ldg((const uint16_t *)p); }

__device__ __forceinline__ float h2f(uint16_t h) { return __half2float(__ushort_as_half(h)); }
__device__ __forceinline__ uint16_t f2h_rn(float f) { return __half_as_ushort(__float2half_rn(f)); }

__device__ __forceinline__ int dp4a_s(int a, int b, int c) { return __dp4a(a, b, c); }      // s8 x s8
__device__ __forceinline__ int dp4a_us(unsigned a, int b, int c) { return __dp4a((int)a, b, c); } // weight bytes are < 128: s8 == u8

// silu exactly as the x86 CPU oracle evaluates it: x / (1 + ggml_v_expf(-x)) (ggml-cpu/vec.h:785-820); the same
// polynomial with an FMA at every step is bit-identical on the GPU, so SwiGLU outputs — which are re-quantised
// for ffn_down — do not pick up 1-ulp differences that would flip int8 roundings
__device__ __forceinline__ float silu_x86(float x) {
    const float nx = __fsub_rn(0.0f, x);
    const float r = 0x1.8p23f;
    const float z = __fmaf_rn(nx, 0x1.715476p+0f, r);
    const float n = __fsub_rn(z, r);
    const float b = __fmaf_rn(-n, 0x1.7f7d1cp-20f, __fmaf_rn(-n, 0x1.62e4p-1f, nx));
    const float u = __fmul_rn(b, b);
    const float j = __fmaf_rn(__fmaf_rn(__fmaf_rn(0x1.0e4020p-7f, b, 0x1.573e2ep-5f), u, __fmaf_rn(0x1.555e66p-3f, b, 0x1.fffdb6p-2f)), u, __fmaf_rn(0x1.ffffecp-1f, b, 1.0f));
    float e = ldexpf(j, (int)n);
    if (fabsf(n) > 192.0f) e = n <= 0.0f ? 0.0f : INFINITY;
    return __fdiv_rn(x, __fadd_rn(1.0f, e));
}

// ---- mbarrier + bulk async copy (TMA engine, 1-D): SASS UBLKCP / SYNCS ----------------------
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
// wait on an mbarrier, optionally accounting the cycles to a profile counter
__device__ __forceinline__ void mbar_wait_p(uint64_t * bar, uint32_t parity, unsigned long long * acc) {
    if (acc) { const long long t0 = clock64(); mbar_wait(bar, parity); *acc += (unsigned long long)(clock64() - t0); }
    else mbar_wait(bar, parity);
}
// generic-proxy shared-memory writes -> visible to the async proxy (tensor core operands, bulk copies)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// global -> shared bulk copy; src/dst 16-byte aligned, bytes % 16 == 0; completes on `bar`
__device__ __forceinline__ void bulk_g2s(void * smem_dst, const void * gsrc, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// L2 prefetch of a byte range (bytes % 16 == 0): lets idle SMs warm the next weight matrix
__device__ __forceinline__ void bulk_prefetch_l2(const void * gsrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(gsrc), "r"(bytes) : "memory");
}

// programmatic dependent launch (guide G9): overlap this kernel's prologue with the previous tail
__device__ __forceinline__ void pdl_wait()    { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// thread-block cluster: hardware barrier over every thread of the cluster (all threads of each warp must take part), and loads from
// a peer CTA's shared memory (distributed shared memory)
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire()   { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait()           { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_map(const void * smem_p, uint32_t rank) {
    uint32_t a; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(smem_p)), "r"(rank)); return a;
}
__device__ __forceinline__ float ld_cluster_f32(uint32_t addr) {
    float v; asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory"); return v;
}

// ---- B200_TRACE=1: in-kernel timeline of the decode chain (tools/trace_decode.py).  A traced CTA claims a record with one atomic
// and stamps %globaltimer at entry / exit plus clock64 at the points in between; records are read back per source file.
#define B200_TRACE_SLOTS 4096
#define B200_TRACE_WORDS 12
__device__ __forceinline__ unsigned long long gtime_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define B200_TRACE_DECL(name) static __device__ unsigned long long name##_buf[B200_TRACE_SLOTS][B200_TRACE_WORDS]; static __device__ unsigned int name##_n;
#define B200_TRACE_OPEN(name, on, tr) unsigned long long * tr = nullptr; \
    if (on) { const unsigned int i_ = atomicAdd(&name##_n, 1u); if (i_ < B200_TRACE_SLOTS) { tr = name##_buf[i_]; tr[0] = gtime_ns(); tr[1] = (unsigned long long)clock64(); } }
#define B200_TRACE_AT(tr, i) do { if (tr) tr[i] = (unsigned long long)clock64(); } while (0)
#define B200_TRACE_CLOSE(tr, i) do { if (tr) { tr[i] = (unsigned long long)clock64(); tr[i + 1] = gtime_ns(); } } while (0)
// host side of one file's trace: copies the records out and resets the counter; returns the number of records
#define B200_TRACE_DUMP(fn, name) extern "C" __attribute__((visibility("default"))) int fn(unsigned long long * out, int max_records) { \
    unsigned int n = 0; cudaMemcpyFromSymbol(&n, name##_n, sizeof(n)); if (n > B200_TRACE_SLOTS) n = B200_TRACE_SLOTS; if ((int)n > max_records) n = (unsigned int)max_records; \
    if (n) cudaMemcpyFromSymbol(out, name##_buf, (size_t)n * B200_TRACE_WORDS * sizeof(unsigned long long)); \
    const unsigned int z = 0; cudaMemcpyToSymbol(name##_n, &z, sizeof(z)); return (int)n; }
static inline bool b200_trace_on() { static const bool on = getenv("B200_TRACE") != nullptr; return on; }

#endif // __CUDACC__
