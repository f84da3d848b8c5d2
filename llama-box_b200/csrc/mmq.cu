// mmq.cu — batched MUL_MAT on quantised weights (prefill / ubatches of more than 8 tokens), host dispatch.
// Replaces ggml_cuda_mul_mat_q (ggml-cuda/mmq.cu:71-143).
//   * K-quants (Q4_K / Q5_K / Q6_K): the wgmma tile kernel of mmq_tc.cu (tensor cores, register accumulators, TMA staging),
//     integer-exact against the CPU oracle;
//   * Q4_0 / Q5_0 / Q8_0 (per-32 f16 block scales): the int8 wgmma tile kernel of mmq_tc32.cu, padded rows (k_valid < k) included;
//     the block sums are exact and folded with the oracle's roundings;
//   * what neither kernel takes (too few columns for the tile kernel to pay off, Q6_K rows that are not a multiple of 2048,
//     B200_MMQ_DISABLE_TC=1): activations quantised like the CPU oracle (quantize.cu) and columns streamed through the matvec
//     kernel in groups of 8 (weights re-read from L2 / HBM per group).
#include "common.cuh"

bool    b200_mmq_tc_supported(int type, int64_t m, int64_t k, int64_t ncols);
int64_t b200_mmq_tc_workspace(int64_t k, int64_t ncols);
int     b200_mmq_tc(int type, const void * W, const float * X, int64_t x_col_stride, float * dst, int64_t ldd, int64_t m, int64_t k, int64_t ncols, void * workspace, void * stream);
bool    b200_mmq_tc32_supported(int type, int64_t m, int64_t k, int64_t ncols);
int64_t b200_mmq_tc32_workspace(int64_t k, int64_t ncols);
int     b200_mmq_tc32(int type, const void * W, const float * X, int64_t x_col_stride, float * dst, int64_t ldd, int64_t m, int64_t k, int64_t k_valid, int64_t ncols, void * workspace, void * stream);

extern "C" int64_t b200_mul_mat_q_workspace(int type, int64_t m, int64_t k, int64_t ncols) {
    const int kind = b200_act_kind_for(type);
    if (kind < 0 || k <= 0 || k % 256 != 0 || ncols <= 0) return 0;
    const int64_t vec = ncols * act_col_bytes(kind, k);
    const int64_t tc = b200_mmq_tc_supported(type, m, k, ncols) ? b200_mmq_tc_workspace(k, ncols)
                     : b200_mmq_tc32_supported(type, m, k, ncols) ? b200_mmq_tc32_workspace(k, ncols) : 0;
    return vec > tc ? vec : tc;
}

extern "C" int b200_mul_mat_q(int type, const void * W, const float * X, int64_t x_col_stride, float * dst, int64_t dst_col_stride,
                              int64_t m, int64_t k, int64_t ncols, void * workspace, void * stream) {
    return b200_mul_mat_q2(type, W, X, x_col_stride, dst, dst_col_stride, m, k, k, ncols, workspace, stream);
}
// k: length of the (padded) weight rows, a multiple of 256; k_valid <= k: elements that exist in X (padded weight layout, see b200_padded_k)
extern "C" int b200_mul_mat_q2(int type, const void * W, const float * X, int64_t x_col_stride, float * dst, int64_t dst_col_stride,
                               int64_t m, int64_t k, int64_t k_valid, int64_t ncols, void * workspace, void * stream) {
    const int kind = b200_act_kind_for(type);
    if (kind < 0) { b200_set_error("mul_mat_q: unsupported weight type %d", type); return B200_ERR_UNSUPPORTED; }
    if (!workspace || ((uintptr_t)workspace & 15)) { b200_set_error("mul_mat_q: workspace missing or unaligned"); return B200_ERR_INVALID; }
    if (k_valid == k && b200_mmq_tc_supported(type, m, k, ncols)) return b200_mmq_tc(type, W, X, x_col_stride, dst, dst_col_stride, m, k, ncols, workspace, stream);
    if (b200_mmq_tc32_supported(type, m, k, ncols)) return b200_mmq_tc32(type, W, X, x_col_stride, dst, dst_col_stride, m, k, k_valid, ncols, workspace, stream);
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
