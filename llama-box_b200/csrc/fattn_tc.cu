// fattn_tc.cu — FLASH_ATTN_EXT for multi-token batches (prefill, large verify batches) on the Hopper tensor cores (sm_90a):
// both contractions (S = Q K^T and O = P V) are wgmma f16 with f32 register accumulators, softmax runs online in registers.
// Two instances, head size D = 128 and D = 64: S is m64n128 either way (D / 16 MMAs of K = 16), O = P V is m64n<D>k16.
//
// Replaces the multi-token path of ggml_cuda_flash_attn_ext: flash_attn_ext_f16 (ggml-cuda/fattn-mma-f16.cuh:395-1410, mma.sync
// tiles, after a to_fp16 expansion of the WHOLE cache: fattn-common.cuh:780-833) — here K / V rows are read from the cache in
// place, once per (query tile, head), and the decode "vec" kernel no longer re-reads the cache once per query token.
//
// One CTA = 128 query tokens of one head.  Per block of 128 KV positions:
//     loader warps   K, V rows (f16, or q8_0 de-quantised to f16 d*q) -> shared memory as core matrices.  Both tiles have the
//                    same image [d / 8][position][8 halves]: for S = Q K^T it is the K-major B operand, for O = P V the SAME image
//                    is an MN-major B operand (n = d, k = position), so V needs no transposition at all
//     consumers      two warpgroups, 64 query rows each: S[64 q][128 kv] = Q K^T (D / 16 x wgmma, K = 16 over d) into registers;
//                    s * scale + mask, online max / sum in f32 (ggml-cpu/ops.cpp:8252-8404 semantics); P = exp(s - m) rounded
//                    to f16 straight from the S registers into the A-operand registers of O = O * alpha + P V (8 x wgmma,
//                    K = 16 over positions); the running O stays in the accumulator registers
// K / V tiles are double-buffered in shared memory, so the loaders fill block i + 1 while the consumers work on block i.  Fully
// masked blocks (causal future, cache padding) are skipped before anything is loaded.  Numerics: Q, K, V, P in f16 on the tensor
// cores (the reference's CUDA path does the same); f32 softmax statistics and accumulation.  The CPU oracle keeps P in f32 and —
// for F16 V — accumulates in fp16, so agreement is ~1e-3 relative, inside the reference harness's NMSE threshold.
#include "common.cuh"
#include "wgmma.cuh"

#include <cuda_fp16.h>
#include <math.h>

#define FT_THREADS 352            // warps 0-3 / 4-7 consumers (query rows 0-63 / 64-127), 8-10 loaders
#define FT_PANEL 2048

struct FtArgs {
    const float * q; int64_t q_ts, q_hs;               // floats
    const uint8_t * k; int64_t k_rs, k_hs;             // bytes
    const uint8_t * v; int64_t v_rs, v_hs;
    const uint16_t * mask; int64_t mask_rs;            // halves; row = token
    float * dst;
    int32_t n_head, n_head_kv, n_tok, n_kv, kv_type;
    float scale, softcap;
};

// Q tile, then two K and two V stages: each [D / 8][128 rows][16 bytes] (32 KB at D = 128, 16 KB at D = 64)
template <int D> struct FtSmem {
    static constexpr int TILE = D / 8 * FT_PANEL;
    static constexpr int Q = 0, K = TILE, V = K + 2 * TILE, BAR = V + 2 * TILE, TOTAL = BAR + 256;
};

__device__ __forceinline__ void ft_fence_async()  { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void ft_arrive(uint64_t * bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ uint32_t pack_h2(float a, float b) { return (uint32_t)__half_as_ushort(__float2half_rn(a)) | ((uint32_t)__half_as_ushort(__float2half_rn(b)) << 16); }

// 8 consecutive elements of a cache row as f16 (one 16-byte K-chunk of a core matrix)
template <int KVT>
__device__ __forceinline__ uint4 kv_chunk(const uint8_t * row, int c) {
    if (KVT == B200_TYPE_F16) return ldg_stream16(row + c * 16);
    // q8_0: 34-byte blocks (f16 d, 32 int8), 2-byte aligned: elements 8c .. 8c+7 live in block c / 4
    const uint8_t * blk = row + (c >> 2) * 34;
    const float d = h2f(__ldg((const uint16_t *)blk));
    const uint16_t * p = (const uint16_t *)(blk + 2 + (c & 3) * 8);
    uint4 r; uint32_t * o = (uint32_t *)&r;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint16_t w = __ldg(p + i);
        o[i] = pack_h2(d * (float)(int8_t)(w & 0xff), d * (float)(int8_t)(w >> 8));
    }
    return r;
}

template <int D, int KVT>
__global__ void __launch_bounds__(FT_THREADS, 1) fattn_tc_kernel(const __grid_constant__ FtArgs a) {
    static_assert(D == 64 || D == 128, "head size");
    using FtSmem = ::FtSmem<D>;
    constexpr int NC = D / 8;                                   // 16-byte K-chunks of a head row = core-matrix panels of a tile
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t * bars = (uint64_t *)(smem + FtSmem::BAR);
    // kv_full[2]: K,V stage loaded (3 loader warp arrivals) | kv_empty[2]: both consumer warpgroups done with the stage
    uint64_t * kv_full = bars, * kv_empty = bars + 2, * q_full = bars + 14;
    int * s_nblk = (int *)(bars + 17);                        // list of KV blocks that hold at least one unmasked position
    __shared__ int s_blocks[512];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int qt = blockIdx.x, h = blockIdx.y;
    const int hk = h / (a.n_head / a.n_head_kv);
    const int q0 = qt * 128;
    const int n_blocks_all = (a.n_kv + 127) / 128;

    if (tid == 0) {
        for (int i = 0; i < 2; i++) { mbar_init(&kv_full[i], 3); mbar_init(&kv_empty[i], 8); }
        mbar_init(q_full, 3);
        mbar_fence_init();
        *s_nblk = 0;
    }
    pdl_wait();
    __syncthreads();
    // ---- which KV blocks matter?  One thread per (block): any unmasked (token, position) pair of this query tile.
    // (libllama's masks are causal + padding; whole future / padding blocks drop out here, before any K / V byte is read)
    const int last_row = (a.n_tok - q0 < 128 ? a.n_tok - q0 : 128) - 1;
    for (int b = warp; b < n_blocks_all; b += FT_THREADS / 32) {
        bool any = a.mask == nullptr;
        if (!any) {
            auto row_any = [&](int r) {                                // 128 halves of one mask row: lane l checks 4
                const uint16_t * mr = a.mask + (int64_t)(q0 + r) * a.mask_rs + b * 128;
                bool u = false;
                if (b * 128 + lane * 4 < a.n_kv) { const uint2 w = *(const uint2 *)(mr + lane * 4); u = ((w.x & 0xffffu) != 0xfc00u) || ((w.x >> 16) != 0xfc00u) || ((w.y & 0xffffu) != 0xfc00u) || ((w.y >> 16) != 0xfc00u); }
                return u;
            };
            // causal masks: the LAST query row of the tile sees the most positions — one load settles almost every block
            any = __any_sync(0xffffffffu, row_any(last_row));
            if (!any) {                                                // rare (future / padding blocks): look at every row, loads independent
                bool u = false;
                for (int r = 0; r < last_row; r++) u |= row_any(r);
                any = __any_sync(0xffffffffu, u);
            }
        }
        if (lane == 0 && any) s_blocks[atomicAdd(s_nblk, 1)] = b;
    }
    __syncthreads();
    const int nblk = *s_nblk;
    // the list is filled in arbitrary order; every role needs the same order -> sort (tiny) by one thread
    if (tid == 0) { for (int i = 1; i < nblk; i++) { const int x = s_blocks[i]; int j = i - 1; while (j >= 0 && s_blocks[j] > x) { s_blocks[j + 1] = s_blocks[j]; j--; } s_blocks[j + 1] = x; } }
    __syncthreads();

    if (warp >= 8) {
        // ===================== loaders (96 threads, rows t and t + 96): Q tile once, then K / V stages =====================
        const int t0 = tid - 256;
        for (int t = t0; t < 128; t += 96) {
            const int tok = q0 + t;
            uint8_t * Qs = smem + FtSmem::Q + t * 16;
            const float * qp = a.q + (int64_t)(tok < a.n_tok ? tok : 0) * a.q_ts + (int64_t)h * a.q_hs;
#pragma unroll
            for (int c = 0; c < NC; c++) {
                uint4 o = make_uint4(0, 0, 0, 0);
                if (tok < a.n_tok) {
                    const float4 x = *(const float4 *)(qp + c * 8), y = *(const float4 *)(qp + c * 8 + 4);
                    o.x = pack_h2(x.x, x.y); o.y = pack_h2(x.z, x.w); o.z = pack_h2(y.x, y.y); o.w = pack_h2(y.z, y.w);   // f32 -> f16 like the CPU's q_to_vec_dot
                }
                *(uint4 *)(Qs + c * FT_PANEL) = o;
            }
        }
        ft_fence_async();
        __syncwarp();
        if (lane == 0) ft_arrive(q_full);
        for (int i = 0; i < nblk; i++) {
            const int st = i & 1;
            mbar_wait(&kv_empty[st], ((i >> 1) & 1) ^ 1);
            for (int t = t0; t < 128; t += 96) {
            const int p = s_blocks[i] * 128 + t;
            const bool in = p < a.n_kv;
            const uint8_t * krow = a.k + (int64_t)(in ? p : 0) * a.k_rs + (int64_t)hk * a.k_hs;
            const uint8_t * vrow = a.v + (int64_t)(in ? p : 0) * a.v_rs + (int64_t)hk * a.v_hs;
            uint8_t * Ks = smem + FtSmem::K + st * FtSmem::TILE + t * 16, * Vs = smem + FtSmem::V + st * FtSmem::TILE + t * 16;
#pragma unroll 4
            for (int c = 0; c < NC; c++) {
                uint4 kk = make_uint4(0, 0, 0, 0), vv = kk;
                if (in) { kk = kv_chunk<KVT>(krow, c); vv = kv_chunk<KVT>(vrow, c); }
                *(uint4 *)(Ks + c * FT_PANEL) = kk;
                *(uint4 *)(Vs + c * FT_PANEL) = vv;
            }
            }
            ft_fence_async();
            __syncwarp();
            if (lane == 0) ft_arrive(&kv_full[st]);
        }
    } else {
        // ===================== consumers: warpgroup g = query rows 64 g .. 64 g + 63 =====================
        // thread: rows ra = 64 g + 16 (warp % 4) + lane / 4 and ra + 8, columns 8 j + c0 + {0, 1} of S and of O (wgmma.cuh)
        const int g = warp >> 2;
        const int ra = 64 * g + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
        const uint16_t * mrow[2];
        bool row_ok[2];
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const int tok = q0 + ra + 8 * u;
            row_ok[u] = tok < a.n_tok;
            mrow[u] = a.mask ? a.mask + (int64_t)(row_ok[u] ? tok : 0) * a.mask_rs : nullptr;
        }
        float O[D / 2], S[64];                                                 // O: m64 x n<D> accumulator, S: m64 x n128
#pragma unroll
        for (int c = 0; c < D / 2; c++) O[c] = 0.0f;
        float M[2] = { -INFINITY, -INFINITY }, L[2] = { 0.0f, 0.0f };           // L: this thread's share of the row sum
        const float scale = a.softcap != 0.0f ? a.scale / a.softcap : a.scale;
        const uint32_t qs = smem_u32(smem + FtSmem::Q) + g * 1024;
        mbar_wait(q_full, 0);
        for (int i = 0; i < nblk; i++) {
            const int st = i & 1;
            const int pb = s_blocks[i] * 128;
            mbar_wait(&kv_full[st], (i >> 1) & 1);
            const uint32_t ks = smem_u32(smem + FtSmem::K + st * FtSmem::TILE), vs = smem_u32(smem + FtSmem::V + st * FtSmem::TILE);
            wg_fence();
#pragma unroll
            for (int j = 0; j < NC / 2; j++) wg_mma_ss(S, wg_desc(qs + j * 2 * FT_PANEL, FT_PANEL, 128), wg_desc(ks + j * 2 * FT_PANEL, FT_PANEL, 128), j ? 1u : 0u);
            wg_commit();
            wg_wait0();
            wg_pin(S);
            // ---- s = S * scale (+ softcap) + mask, row maxima (a row lives in the 4 threads of a lane quad)
            float mloc[2] = { -INFINITY, -INFINITY };
#pragma unroll
            for (int j = 0; j < 16; j++) {
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const int col = pb + 8 * j + c0;
                    const uint32_t mk = mrow[u] ? *(const uint32_t *)(mrow[u] + col) : 0u;
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        float s = S[4 * j + 2 * u + e] * scale;
                        if (a.softcap != 0.0f) s = a.softcap * tanhf(s);
                        const float mv = mrow[u] ? h2f((uint16_t)(mk >> (16 * e))) : 0.0f;
                        s = (row_ok[u] && col + e < a.n_kv) ? s + mv : -INFINITY;
                        S[4 * j + 2 * u + e] = s;
                        mloc[u] = fmaxf(mloc[u], s);
                    }
                }
            }
            float alpha[2], Mn[2];
#pragma unroll
            for (int u = 0; u < 2; u++) {
                mloc[u] = fmaxf(mloc[u], __shfl_xor_sync(0xffffffffu, mloc[u], 1));
                mloc[u] = fmaxf(mloc[u], __shfl_xor_sync(0xffffffffu, mloc[u], 2));
                Mn[u] = fmaxf(M[u], mloc[u]);
                alpha[u] = (M[u] == -INFINITY) ? 1.0f : expf(M[u] - Mn[u]);     // Mn finite here unless the whole row is masked so far (then O = L = 0 anyway)
            }
            // ---- P = exp(s - Mn) rounded to f16: the A operand of P V, straight from the S registers
            uint32_t P[8][4];
            float lsum[2] = { 0.0f, 0.0f };
#pragma unroll
            for (int j = 0; j < 16; j++) {
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    float p[2];
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        p[e] = (Mn[u] == -INFINITY) ? 0.0f : expf(S[4 * j + 2 * u + e] - Mn[u]);
                        // the tensor core sees f16(p): sum the SAME rounded values so that O / L is a proper weighted mean
                        p[e] = __half2float(__float2half_rn(p[e]));
                        lsum[u] += p[e];
                    }
                    P[j >> 1][(j & 1) * 2 + u] = pack_h2(p[0], p[1]);
                }
            }
#pragma unroll
            for (int j = 0; j < NC; j++) {
#pragma unroll
                for (int u = 0; u < 2; u++) { O[4 * j + 2 * u] *= alpha[u]; O[4 * j + 2 * u + 1] *= alpha[u]; }
            }
#pragma unroll
            for (int u = 0; u < 2; u++) { L[u] = L[u] * alpha[u] + lsum[u]; M[u] = Mn[u]; }
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < 8; kk++)                                      // K = 16 positions per MMA; V position groups 2kk, 2kk+1 (MN-major: 128 B apart)
                wg_mma_rs_bmn(O, P[kk], wg_desc(vs + kk * 256, 128, FT_PANEL), 1u);
            wg_commit();
            wg_wait0();
            wg_pin(O);
            __syncwarp();
            if (lane == 0) ft_arrive(&kv_empty[st]);                            // K / V stage free
        }
#pragma unroll
        for (int u = 0; u < 2; u++) {
            float l = L[u];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            if (!row_ok[u]) continue;
            const float inv = l > 0.0f ? 1.0f / l : 0.0f;                        // ops.cpp:8390-8392 (V /= S)
            float * out = a.dst + ((int64_t)(q0 + ra + 8 * u) * a.n_head + h) * D;
#pragma unroll
            for (int j = 0; j < NC; j++) *(float2 *)(out + 8 * j + c0) = make_float2(O[4 * j + 2 * u] * inv, O[4 * j + 2 * u + 1] * inv);
        }
    }
    pdl_trigger();
}

// ---- host ----------------------------------------------------------------------------------------------------------
// Fewest query tokens per head size for which this kernel beats the vector kernel (fattn.cu), which reads K / V once per token.
// Head 64 from a sweep of both arms (tools/fattn_bench.py --sweep, H100.md): at 32 tokens the vector kernel is still ahead on a
// Q8_0 cache, from 40 on this kernel wins or ties on both cache types.
#define FT_MIN_TOK_D128 16
#define FT_MIN_TOK_D64 40

bool b200_fattn_tc_supported(int kv_type, int64_t dk, int64_t dv, int64_t n_tok, int64_t n_kv, float max_bias) {
    static const bool off = getenv("B200_FATTN_DISABLE_TC") != nullptr;
    const bool shape = (dk == 128 && dv == 128 && n_tok >= FT_MIN_TOK_D128) || (dk == 64 && dv == 64 && n_tok >= FT_MIN_TOK_D64);
    return !off && shape && n_kv % 8 == 0 && n_kv <= 512 * 128 && max_bias == 0.0f && (kv_type == B200_TYPE_F16 || kv_type == B200_TYPE_Q8_0);
}

template <int D, int KVT> static int ft_launch(const FtArgs & a, cudaStream_t st) {
    static bool attr[64] = { false };
    int dev = 0; cudaGetDevice(&dev);
    if (!attr[dev & 63]) { B200_CUDA(cudaFuncSetAttribute(fattn_tc_kernel<D, KVT>, cudaFuncAttributeMaxDynamicSharedMemorySize, FtSmem<D>::TOTAL)); attr[dev & 63] = true; }
    dim3 grid((unsigned)((a.n_tok + 127) / 128), (unsigned)a.n_head);
    B200_CUDA(b200_launch_pdl(fattn_tc_kernel<D, KVT>, grid, dim3(FT_THREADS), (size_t)FtSmem<D>::TOTAL, st, a));
    b200_count_launch();
    return B200_OK;
}

int b200_fattn_tc(const float * q, int64_t q_ts, int64_t q_hs, const void * k, int64_t k_rs, int64_t k_hs, const void * v, int64_t v_rs, int64_t v_hs,
                  const void * mask, int64_t mask_rs, float * dst, int kv_type, int64_t d, int64_t n_head, int64_t n_head_kv, int64_t n_tok, int64_t n_kv,
                  float scale, float softcap, void * stream) {
    FtArgs a;
    a.q = q; a.q_ts = q_ts; a.q_hs = q_hs; a.k = (const uint8_t *)k; a.k_rs = k_rs; a.k_hs = k_hs; a.v = (const uint8_t *)v; a.v_rs = v_rs; a.v_hs = v_hs;
    a.mask = (const uint16_t *)mask; a.mask_rs = mask_rs; a.dst = dst;
    a.n_head = (int32_t)n_head; a.n_head_kv = (int32_t)n_head_kv; a.n_tok = (int32_t)n_tok; a.n_kv = (int32_t)n_kv; a.kv_type = kv_type;
    a.scale = scale; a.softcap = softcap;
    if (mask && ((mask_rs & 7) || ((uintptr_t)mask & 15))) { b200_set_error("flash_attn (tensor core): mask rows must be 16-byte aligned"); return B200_ERR_INVALID; }
    const cudaStream_t st = (cudaStream_t)stream;
    if (d == 128) return kv_type == B200_TYPE_F16 ? ft_launch<128, B200_TYPE_F16>(a, st) : ft_launch<128, B200_TYPE_Q8_0>(a, st);
    if (d == 64)  return kv_type == B200_TYPE_F16 ? ft_launch<64, B200_TYPE_F16>(a, st) : ft_launch<64, B200_TYPE_Q8_0>(a, st);
    b200_set_error("flash_attn (tensor core): head size %lld unsupported (64 or 128)", (long long)d);
    return B200_ERR_UNSUPPORTED;
}
