// mmid_route.cu — MUL_MAT_ID for prefill (ubatches of MMID_MIN_TOK tokens and more) as a grouped GEMM on the tensor cores.
// Replaces the ids path of ggml_cuda_mul_mat_q (ggml-cuda/mmq.cu:149-193), which copies the ids to the host and synchronises twice per
// op to build its expert map.  Here the map is built ON THE DEVICE by one small kernel, so the op is capturable into a CUDA graph:
//
//   1. mmid_route_kernel: (token, slot) pairs grouped by expert, in the order t * n_used + s inside each expert (stable, no atomics decide a
//      position), each expert's run padded to whole 128-column tiles; ids outside [0, n_expert) are dropped (their outputs are not written);
//   2. the gathering quantiser of the weight's tile kernel writes the activation image of those columns (padding columns are zeros);
//   3. the GROUPED instance of the tile kernel (mmq_tc.cu for Q4_K / Q5_K / Q6_K, mmq_tc32.cu for Q4_0 / Q5_0 / Q8_0) multiplies column
//      tile ct by its expert's matrix and scatters the outputs to their (token, slot) rows.
// Every output is folded by one CTA over its blocks in order from exact integer sums, so it is bit-identical to what b200_mul_mat_q gives
// for the same expert matrix and the same activation column.  The launches are sized from the host's upper bound on the column tiles,
// floor(N / 128) + min(n_expert, N) with N = n_tok * n_used; CTAs past the real count (in device memory) do nothing.
#include "mmq_tile.cuh"

// When the grouped GEMM runs: at least MMID_MIN_TOK tokens (fewer — decode, speculative verify batches — stay on the matvec of mmvq_ext.cu,
// one pass over an expert's weights per (token, slot)), and at least MMID_MIN_PAIRS (token, slot) pairs per expert on average.  A tile pass
// costs about as much for 1 column as for 128 and every expert with a pair takes one, so with many experts and few pairs each (fine-grained
// stacks: 128 experts, top-8) the matvec stays ahead up to a few pairs per expert.  From the two-arm sweep of tools/wide_bench.py --mmid
// --sweep (H100.md), which times a build with -DMMID_MIN_TOK=9 -DMMID_MIN_PAIRS=0 so that the grouped arm runs at every token count.
#ifndef MMID_MIN_TOK
#define MMID_MIN_TOK 16
#endif
#ifndef MMID_MIN_PAIRS
#define MMID_MIN_PAIRS 4
#endif
#define MMID_MAX_EXPERT 1024        // the router keeps a per-warp count of every expert in shared memory
#define MMID_ROUTE_SMEM (44 * 1024)

namespace {

struct RouteGeom { int64_t ub, off_cnt, off_tiles, off_cols, off_image, total; };

int64_t up256(int64_t x) { return (x + 255) & ~(int64_t)255; }

RouteGeom route_geom(int type, int64_t k, int64_t n_expert, int64_t n_used, int64_t n_tok) {
    RouteGeom g;
    const int64_t N = n_tok * n_used;
    g.ub = N / 128 + (n_expert < N ? n_expert : N);
    g.off_cnt = 16;                                        // [0]: the column tiles in use
    g.off_tiles = up256(g.off_cnt + 4 * n_expert);
    g.off_cols = up256(g.off_tiles + 4 * g.ub);
    g.off_image = up256(g.off_cols + 4 * 128 * g.ub);
    g.total = g.off_image + mmq_tile_workspace(type, k, 128 * g.ub);
    return g;
}

bool mmid_tc_ok(int type, int64_t m, int64_t k, int64_t n_expert, int64_t n_used, int64_t n_tok) {
    // the tuned six only: the K-quant kernel also takes Q2_K / Q3_K, but as dense MUL_MAT (no grouped instance)
    if (!(type_is_block32(type) || type == B200_TYPE_Q4_K || type == B200_TYPE_Q5_K || type == B200_TYPE_Q6_K)) return false;
    if (!mmq_tile_takes(type, m, k)) return false;
    if (n_tok < MMID_MIN_TOK || n_expert <= 0 || n_expert > MMID_MAX_EXPERT || n_used <= 0 || n_used > n_expert) return false;
    if (n_tok * n_used > INT32_MAX / 2 || n_tok * n_used < MMID_MIN_PAIRS * n_expert) return false;
    const int64_t N = n_tok * n_used, ub = N / 128 + (n_expert < N ? n_expert : N);
    return ub * 16 <= 65535 && ((m + 127) / 128) * ub <= INT32_MAX;                    // quantiser grid.y, tile count
}

// one CTA of nw warps.  Warp w owns pairs [w * seg, (w + 1) * seg) of the list p = t * n_used + s.  Pass 1 counts each warp's pairs per
// expert (lanes with the same expert are found with match.any; the highest of them adds the group), a scan over warps and one over experts
// give every (warp, expert) its first column, pass 2 places the pairs: first column + lanes of the same expert before this one.
__global__ void __launch_bounds__(1024) mmid_route_kernel(const int32_t * __restrict__ ids, int64_t ids_tok_stride, int n_expert, int n_used, int64_t n_tok,
                                                           int32_t * __restrict__ ws_ntt, int32_t * __restrict__ cnt, int32_t * __restrict__ tile_expert,
                                                           int32_t * __restrict__ cols) {
    extern __shared__ int32_t sm[];
    const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int32_t * wc = sm;                                     // [nw][n_expert]: count, then first column within the expert
    int32_t * first = sm + nw * n_expert;                  // [n_expert]: first column tile of the expert
    for (int i = threadIdx.x; i < nw * n_expert; i += blockDim.x) wc[i] = 0;
    pdl_wait();
    __syncthreads();
    const int64_t N = n_tok * n_used, seg = (N + nw - 1) / nw;
    const int64_t p0 = warp * seg, p1 = p0 + seg < N ? p0 + seg : N;
    int32_t * my = wc + warp * n_expert;
    auto expert_of = [&](int64_t p) {
        if (p >= p1) return -1;
        const int e = ids[(p / n_used) * ids_tok_stride + p % n_used];
        return e >= 0 && e < n_expert ? e : -1;
    };
    for (int64_t q = p0; q < p1; q += 32) {
        const int e = expert_of(q + lane);
        const unsigned same = __match_any_sync(0xffffffffu, e);
        if (e >= 0 && lane == 31 - __clz(same)) my[e] += __popc(same);
        __syncwarp();
    }
    __syncthreads();
    for (int e = threadIdx.x; e < n_expert; e += blockDim.x) {
        int s = 0;
        for (int w = 0; w < nw; w++) { const int c = wc[w * n_expert + e]; wc[w * n_expert + e] = s; s += c; }
        cnt[e] = s;
        first[e] = (s + 127) >> 7;                         // tiles of the expert, scanned below
    }
    __syncthreads();
    if (warp == 0) {
        int carry = 0;
        for (int e0 = 0; e0 < n_expert; e0 += 32) {
            const int e = e0 + lane;
            const int v = e < n_expert ? first[e] : 0;
            int incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
            if (e < n_expert) first[e] = carry + incl - v;
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) *ws_ntt = carry;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < n_expert; e += blockDim.x) {   // tile -> expert, and the padding columns of the expert's last tile
        const int c = cnt[e], t0 = first[e], nt = (c + 127) >> 7;
        for (int t = 0; t < nt; t++) tile_expert[t0 + t] = e;
        for (int j = c; j < nt * 128; j++) cols[(int64_t)t0 * 128 + j] = -1;
    }
    for (int64_t q = p0; q < p1; q += 32) {
        const int e = expert_of(q + lane);
        const unsigned same = __match_any_sync(0xffffffffu, e);
        const int before = __popc(same & ((1u << lane) - 1u));
        if (e >= 0) cols[(int64_t)first[e] * 128 + my[e] + before] = (int32_t)(q + lane);
        __syncwarp();
        if (e >= 0 && lane == 31 - __clz(same)) my[e] += __popc(same);
        __syncwarp();
    }
    pdl_trigger();
}

bool al16(const void * p) { return ((uintptr_t)p & 15) == 0; }

} // namespace

extern "C" int64_t b200_mul_mat_id_workspace(int type, int64_t m, int64_t k, int64_t n_expert, int64_t n_used, int64_t n_tok) {
    if (!mmid_tc_ok(type, m, k, n_expert, n_used, n_tok)) return 0;
    return route_geom(type, k, n_expert, n_used, n_tok).total;
}

extern "C" int b200_mul_mat_id2(int type, const void * as, int64_t expert_stride_bytes, const float * b, int64_t b_tok_stride, int64_t b_slot_stride, int64_t n_b1,
                                const int32_t * ids, int64_t ids_tok_stride, float * dst, int64_t dst_tok_stride, int64_t dst_slot_stride,
                                int64_t m, int64_t k, int64_t n_expert, int64_t n_used, int64_t n_tok, void * workspace, void * stream) {
    if (!mmid_tc_ok(type, m, k, n_expert, n_used, n_tok))
        return b200_mul_mat_id(type, as, expert_stride_bytes, b, b_tok_stride, b_slot_stride, n_b1, ids, ids_tok_stride, dst, dst_tok_stride, dst_slot_stride,
                               m, k, n_expert, n_used, n_tok, stream);
    if (b200_device_count() <= 0) { b200_set_error("no CUDA device"); return B200_ERR_CUDA; }
    if (!as || !b || !ids || !dst || n_b1 <= 0 || !al16(as) || !al16(b) || (b_tok_stride & 3) || (b_slot_stride & 3) ||
        (expert_stride_bytes & 15) || ((uintptr_t)dst & 3)) {
        b200_set_error("mul_mat_id: bad arguments (as, b 16-byte aligned; b strides multiples of 4 floats; expert stride a multiple of 16 bytes)"); return B200_ERR_INVALID;
    }
    if (!workspace || ((uintptr_t)workspace & 255)) { b200_set_error("mul_mat_id: workspace missing or not 256-byte aligned"); return B200_ERR_INVALID; }
    cudaStream_t st = (cudaStream_t)stream;
    const RouteGeom g = route_geom(type, k, n_expert, n_used, n_tok);
    uint8_t * ws = (uint8_t *)workspace;
    MmidMap map;
    map.ntt = (const int32_t *)ws; map.tile_expert = (const int32_t *)(ws + g.off_tiles); map.cols = (const int32_t *)(ws + g.off_cols);
    map.n_used = (int32_t)n_used; map.n_b1 = (int32_t)n_b1; map.b_tok_stride = b_tok_stride; map.b_slot_stride = b_slot_stride;
    map.expert_stride = expert_stride_bytes; map.dst_tok_stride = dst_tok_stride; map.dst_slot_stride = dst_slot_stride;
    int nw = (int)((MMID_ROUTE_SMEM / 4 - n_expert) / n_expert);
    if (nw > 32) nw = 32;
    const size_t smem = (size_t)(nw + 1) * n_expert * 4;
    B200_CUDA(b200_launch_pdl(mmid_route_kernel, dim3(1), dim3(32 * nw), smem, st, ids, ids_tok_stride, (int)n_expert, (int)n_used, n_tok,
                              (int32_t *)ws, (int32_t *)(ws + g.off_cnt), (int32_t *)(ws + g.off_tiles), (int32_t *)(ws + g.off_cols)));
    b200_count_launch();
    const MmqJob job = { as, b, 0, k, dst, 0, m, k, 128 * g.ub, ws + g.off_image, &map };
    return mmq_tile_run(type, job, st);
}
