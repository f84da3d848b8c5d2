// mmid.cuh — the device-built schedule of a grouped MUL_MAT_ID (mmid_route.cu), as the tile kernels of mmq_tc.cu / mmq_tc32.cu read it
// in their GROUPED instances.  The (token, slot) pairs are grouped by expert, in the order t * n_used + s inside each expert, and each
// expert's run is padded to whole 128-column tiles; column tile ct belongs to expert tile_expert[ct] and its column j holds pair cols[128 ct + j]
// (-1: padding).  The number of tiles in use, *ntt, is known on the device only: launches are sized from the host's upper bound and the
// CTAs past it do nothing.
#pragma once
#include <stdint.h>

struct MmidMap {
    const int32_t * ntt;            // column tiles in use (device)
    const int32_t * tile_expert;    // [ct] expert of column tile ct
    const int32_t * cols;           // [ct * 128 + j] pair t * n_used + s, or -1
    int32_t n_used, n_b1;
    int64_t b_tok_stride, b_slot_stride;                        // activation of pair (t, s): b + t * b_tok_stride + (s % n_b1) * b_slot_stride (floats)
    int64_t expert_stride;                                      // bytes between the experts' weight matrices
    int64_t dst_tok_stride, dst_slot_stride;                    // output rows of pair (t, s): dst + t * dst_tok_stride + s * dst_slot_stride (floats)
};
