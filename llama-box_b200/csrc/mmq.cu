// mmq.cu — batched MUL_MAT on quantised weights (prefill / ubatches of more than 8 tokens), host dispatch, and the one place that
// decides which tensor-core tile kernel runs (for MUL_MAT_ID too, mmid_route.cu).
// Replaces ggml_cuda_mul_mat_q (ggml-cuda/mmq.cu:71-143).
//   * K-quants (Q4_K / Q5_K / Q6_K): the wgmma tile kernel of mmq_tc.cu (tensor cores, register accumulators, TMA staging),
//     integer-exact against the CPU oracle;
//   * Q2_K / Q3_K (the wide path's 2- and 3-bit K-quants, ggml's native block layout): the same K-quant kernel; what it does not take
//     goes to the wide matvec of mmvq_ext.cu (b200_mul_mat_vec_wide), which quantises the columns itself and needs no workspace;
//   * Q4_0 / Q5_0 / Q8_0 (per-32 f16 block scales): the int8 wgmma tile kernel of mmq_tc32.cu, padded rows (k_valid < k) included;
//     the block sums are exact and folded with the oracle's roundings;
//   * IQ4_NL / IQ4_XS (the wide path's non-linear 4-bit formats, ggml's native block layout, rows of k % 256 == 0): the same int8
//     kernel; like Q2_K / Q3_K, what it does not take goes to the wide matvec;
//   * what neither kernel takes (too few columns for the tile kernel to pay off, Q6_K rows that are not a multiple of 2048,
//     B200_MMQ_DISABLE_TC=1): activations quantised like the CPU oracle (quantize.cu) and columns streamed through the matvec
//     kernel in groups of 8 (weights re-read from L2 / HBM per group).
#include "mmq_tile.cuh"

#include <cstdio>

// Fewest activation columns that go to the tensor cores; below it the columns stream through the matvec in groups of 8.  A tile pass
// costs the same for 9 columns as for 128 (and a matrix of m rows occupies only m / 128 SMs), a column group costs one pass over the
// weights.  K-quants: from the second column group on; Q2_K / Q3_K keep that rule, measured against the wide matvec on the Llama-3-8B
// shapes (H100.md): at 9 columns the tile kernel is ahead on all four (1.04-5.6x).  Q4_0 / Q5_0 / Q8_0, measured on the Llama-3-8B
// shapes at Q8_0 (H100.md): at 32 columns the column groups win on three shapes of four, at 64 the tensor cores win on all four; by
// the per-group time in between, 7 groups (49 columns) is where the tile kernel is ahead on all.  IQ4_NL / IQ4_XS, measured against the
// wide matvec on the Llama-3-8B shapes (H100.md, sweep 9 / 16 / 24 / 32 / 64): at 9 columns the wide matvec still wins IQ4_XS ffn_down
// (0.95x), at 16 the tile kernel is ahead on all four shapes for both types (1.07-5.7x).
#define TC_MIN_COLS 9
#define T32_MIN_COLS 49
#define IQ4_MIN_COLS 16

bool mmq_tile_takes(int type, int64_t m, int64_t k) {
    static const bool off = getenv("B200_MMQ_DISABLE_TC") != nullptr;     // comparison arm: the matvec kernels instead (still the GPU)
    if (off || m <= 0 || k <= 0) return false;
    if (type == B200_TYPE_Q6_K) return k % 2048 == 0;
    return (type == B200_TYPE_Q4_K || type == B200_TYPE_Q5_K || type == B200_TYPE_Q2_K || type == B200_TYPE_Q3_K || type_is_block32(type) ||
            type == B200_TYPE_IQ4_NL || type == B200_TYPE_IQ4_XS) && k % 256 == 0;
}
static bool wide_iq4(int type) { return type == B200_TYPE_IQ4_NL || type == B200_TYPE_IQ4_XS; }
// the formats of the int8 kernel (mmq_tc32.cu); the rest go to the K-quant kernel (mmq_tc.cu)
static bool int8_tile(int type) { return type_is_block32(type) || wide_iq4(type); }
int64_t mmq_tile_workspace(int type, int64_t k, int64_t ncols) {
    return int8_tile(type) ? b200_mmq_tc32_workspace(k, ncols) : b200_mmq_tc_workspace(k, ncols);
}
int mmq_tile_run(int type, const MmqJob & job, cudaStream_t st) {
    return int8_tile(type) ? b200_mmq_tc32(type, job, st) : b200_mmq_tc(type, job, st);
}

// the dense MUL_MAT also needs enough columns, and unpadded rows except for the repacked block-32 formats
static bool dense_tile(int type, int64_t m, int64_t k, int64_t k_valid, int64_t ncols) {
    if (!mmq_tile_takes(type, m, k)) return false;
    if (type_is_block32(type)) return ncols >= T32_MIN_COLS;
    return ncols >= (wide_iq4(type) ? IQ4_MIN_COLS : TC_MIN_COLS) && k_valid == k;
}

// the formats only the wide matvec reads that also have a tile kernel (native block layout, dense MUL_MAT only): no act-buffer path,
// and the wide matvec wherever the tile kernel does not take the call
static bool wide_tile_type(int type) { return type == B200_TYPE_Q2_K || type == B200_TYPE_Q3_K || wide_iq4(type); }

extern "C" int64_t b200_mul_mat_q_workspace(int type, int64_t m, int64_t k, int64_t ncols) {
    if (wide_tile_type(type)) return dense_tile(type, m, k, k, ncols) ? mmq_tile_workspace(type, k, ncols) : 0;     // the wide matvec needs none
    const int kind = b200_act_kind_for(type);
    if (kind < 0 || k <= 0 || k % 256 != 0 || ncols <= 0) return 0;
    const int64_t vec = ncols * act_col_bytes(kind, k);
    const int64_t tc = dense_tile(type, m, k, k, ncols) ? mmq_tile_workspace(type, k, ncols) : 0;
    return vec > tc ? vec : tc;
}

extern "C" int b200_mul_mat_q(int type, const void * W, const float * X, int64_t x_col_stride, float * dst, int64_t dst_col_stride,
                              int64_t m, int64_t k, int64_t ncols, void * workspace, void * stream) {
    return b200_mul_mat_q2(type, W, X, x_col_stride, dst, dst_col_stride, m, k, k, ncols, workspace, stream);
}
// k: length of the (padded) weight rows, a multiple of 256; k_valid <= k: elements that exist in X (padded weight layout, see b200_padded_k)
extern "C" int b200_mul_mat_q2(int type, const void * W, const float * X, int64_t x_col_stride, float * dst, int64_t dst_col_stride,
                               int64_t m, int64_t k, int64_t k_valid, int64_t ncols, void * workspace, void * stream) {
    if (wide_tile_type(type) && !dense_tile(type, m, k, k_valid, ncols)) {
        if (k_valid != k) { b200_set_error("mul_mat_q: type %d has no padded rows (k_valid must equal k)", type); return B200_ERR_INVALID; }
        return b200_mul_mat_vec_wide(type, W, X, x_col_stride, dst, dst_col_stride, nullptr, nullptr, m, k, ncols, stream);
    }
    const int kind = wide_tile_type(type) ? 0 : b200_act_kind_for(type);
    if (kind < 0) { b200_set_error("mul_mat_q: unsupported weight type %d", type); return B200_ERR_UNSUPPORTED; }
    if (!workspace || ((uintptr_t)workspace & 15)) { b200_set_error("mul_mat_q: workspace missing or unaligned"); return B200_ERR_INVALID; }
    if (dense_tile(type, m, k, k_valid, ncols)) {
        if (((uintptr_t)W | (uintptr_t)X) & 15 || (x_col_stride & 3)) { b200_set_error("mul_mat_q: pointers must be 16-byte aligned"); return B200_ERR_INVALID; }
        if (k_valid <= 0 || k_valid > k || k_valid % 8 != 0) { b200_set_error("mul_mat_q: k_valid must be a positive multiple of 8, at most k"); return B200_ERR_INVALID; }
        const MmqJob job = { W, X, x_col_stride, k_valid, dst, dst_col_stride, m, k, ncols, workspace, nullptr };
        return mmq_tile_run(type, job, (cudaStream_t)stream);
    }
    int s = b200_quantize_act2(kind, X, x_col_stride, workspace, k, k_valid, ncols, stream);
    if (s != B200_OK) return s;
    const int64_t colb = act_col_bytes(kind, k);
    for (int64_t c0 = 0; c0 < ncols; c0 += 8) {
        const int64_t nc = ncols - c0 < 8 ? ncols - c0 : 8;
        s = b200_mul_mat_vec_q(type, W, (const uint8_t *)workspace + c0 * colb, dst + c0 * dst_col_stride, dst_col_stride, nullptr, nullptr, m, k, nc, stream);
        if (s != B200_OK) return s;
    }
    return B200_OK;
}

// B200_MMQ_PROF=1: per-role wait cycles of CTA 0 of the tile kernels (mmq_tc.cu and mmq_tc32.cu share the warp roles), printed after
// each launch (bring-up only)
unsigned long long * mmq_prof_buf() {
    static unsigned long long * prof_buf = nullptr;
    static const bool want_prof = getenv("B200_MMQ_PROF") != nullptr;
    if (want_prof && !prof_buf) { cudaMalloc((void **)&prof_buf, 16 * 4 * 8); }
    return want_prof ? prof_buf : nullptr;
}
void mmq_prof_report(const char * kernel, int type, const MmqTileArgs & a, cudaStream_t st) {
    unsigned long long h[16 * 4];
    cudaStreamSynchronize(st); cudaMemcpy(h, a.prof, sizeof(h), cudaMemcpyDeviceToHost);
    const char * role[12] = { "mma", "mma", "mma", "mma", "mma", "mma", "mma", "mma", "xform", "xform", "xform", "xform" };
    fprintf(stderr, "%s prof (CTA 0, cycles): type %d m %lld k %lld n %lld tiles %d\n", kernel, type, (long long)a.m, (long long)a.k, (long long)a.ncols, a.n_tiles);
    for (int w = 0; w < 12; w += (w < 8 ? 4 : 2))
        fprintf(stderr, "  warp %2d %-8s total %9llu  wait0 %9llu  wait1 %9llu  wait2 %9llu\n", w, role[w], h[w * 4], h[w * 4 + 1], h[w * 4 + 2], h[w * 4 + 3]);
    fprintf(stderr, "  (mma: wait0 = b_full, wait1 = a_full | xform: wait1 = ab_empty)\n");
}
