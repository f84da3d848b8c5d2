/*
 * b200_graph.h — C-ABI of the graph executor in libb200ops.so (row a10 of SURVEY.md §8).
 *
 * A neutral, plain-C mirror of the slice of ggml's graph IR that llm_build_llama / llm_build_qwen2
 * emit (/root/reference/llama.cpp/src/llama-model.cpp:5968-6122, llama-graph.cpp): a node = op + dst
 * + sources with ggml's ne[] (elements) / nb[] (byte strides) conventions (ggml/include/ggml.h:613-645).
 * The ggml backend plug-in (include/ggml_b200.h) translates a ggml_cgraph into this form 1:1; tests
 * and bench.py build the same node lists directly.  Replaces the node loop, fusion and CUDA-graph
 * capture of ggml-cuda (ggml/src/ggml-cuda/ggml-cuda.cu:2845-3010, 2784-2843, 2593-2782).
 *
 * What the executor does with a node list:
 *   - skips view ops, launches one hand-written sm_90a kernel per remaining node, or fewer:
 *       RMS_NORM+MUL(+activation quantisation), MUL_MAT+ADD(bias)+ADD(residual),
 *       MUL_MAT(up)+MUL_MAT(gate)+GLU, several MUL_MATs of one activation in one launch (QKV),
 *   - quantises each activation tensor once per consumer group (the reference re-quantises per matmul),
 *   - captures the whole list into a CUDA graph keyed by its topology and replays it while the
 *     topology is unchanged (decode), so ~600 nodes cost one launch.
 */
#ifndef B200_GRAPH_H
#define B200_GRAPH_H

#include "b200_ops.h"

#ifdef __cplusplus
extern "C" {
#endif

/* tensor element types beyond b200_type, numerically equal to enum ggml_type */
enum { B200_TYPE_I32 = 26, B200_TYPE_I64 = 27 };

enum b200_op {
    B200_OP_NONE = 0,        /* RESHAPE / VIEW / PERMUTE / TRANSPOSE / NONE: metadata only (ggml-cuda.cu:2404-2409) */
    B200_OP_MUL_MAT,         /* src0 weights [K,M], src1 f32 [K,N]  -> dst f32 [M,N]                 */
    B200_OP_RMS_NORM,        /* op_params[0] = eps (f32 bits)                                         */
    B200_OP_MUL,             /* broadcasting f32                                                      */
    B200_OP_ADD,
    B200_OP_ROPE,            /* src0 x [hd,n_head,n_tok], src1 pos i32, src2 freq_factors (optional); op_params as ggml (rope.cu:347-368) */
    B200_OP_SET_ROWS,        /* src0 f32 rows, src1 i64 ids, dst = cache (F32/F16/Q8_0)               */
    B200_OP_FLASH_ATTN_EXT,  /* src0 q, src1 k, src2 v, src3 mask f16 (optional); op_params {scale,max_bias,softcap,prec} */
    B200_OP_GLU_SWIGLU,      /* src0 gate, src1 up (split form, ggml.c:2796)                          */
    B200_OP_GET_ROWS,        /* src0 f32 [ncols, nrows], src1 i32 ids                                  */
    B200_OP_CPY,             /* src0 f32 -> dst f16 / f32, contiguous                                  */
    B200_OP_MUL_MAT_ID,      /* src0 experts [K,M,n_expert], src1 f32 [K,n_b1,n_tok], src2 ids i32 [n_used,n_tok] -> dst f32 [M,n_used,n_tok]
                                (ggml.c:3064-3106).  Wide path (b200_mul_mat_id): see B200_WIDE below                             */
    /* mixture-of-experts router glue (llama-graph.cpp build_moe_ffn), wide path only: */
    B200_OP_SOFT_MAX,        /* src0 f32 rows; optional src1 mask f32 / f16 (one row per token, attention without -fa); op_params {scale, max_bias}   */
    B200_OP_ARGSORT,         /* src0 f32 [n, rows] -> dst i32 [n, rows]; op_params[0] = order (0 ascending, 1 descending); the reference's tie order */
    B200_OP_SUM_ROWS,        /* src0 f32 [n, rows] -> dst f32 [1, rows]                                                                             */
    B200_OP_DIV,             /* broadcasting f32, like MUL                                                                                          */
    B200_OP_CONT,            /* src0 f32, any strides -> dst f32 contiguous, elements in src0's logical order (ggml_cont / ggml_cont_2d); wide path            */
    B200_OP_SCALE,           /* src0 f32 contiguous; op_params {s, b} (f32 bits): x * s + b; wide path                                                         */
    B200_OP_UNARY,           /* src0 f32 contiguous; op_params[0] = ggml_unary_op: SILU (10) or SIGMOID (7); wide path                                          */
    B200_OP_COUNT
};

#define B200_MAX_SRC 6
#define B200_TENSOR_FLAG_OUTPUT 2   /* == GGML_TENSOR_FLAG_OUTPUT: never elided, never fused away (ggml-impl.h:565) */

typedef struct b200_tensor {
    uint64_t id;             /* identity for dependency analysis (plug-in: the ggml_tensor address); 0 = absent */
    void    *data;           /* device pointer                                                          */
    int32_t  type;           /* ggml_type value                                                         */
    int32_t  flags;          /* ggml's tensor flags (ggml.h:602-607); B200_TENSOR_FLAG_OUTPUT = the caller reads this tensor  */
    int64_t  ne[4];
    int64_t  nb[4];
} b200_tensor;

typedef struct b200_node {
    int32_t     op;          /* enum b200_op */
    int32_t     n_src;
    b200_tensor dst;
    b200_tensor src[B200_MAX_SRC];
    int32_t     op_params[16];
} b200_node;

enum {
    B200_EXEC_CUDA_GRAPHS = 1,   /* capture / replay (off: GGML_B200_DISABLE_GRAPHS, like GGML_CUDA_DISABLE_GRAPHS ggml-cuda.cu:2937) */
    B200_EXEC_FUSION      = 2,   /* cross-node fusion (off: GGML_B200_DISABLE_FUSION, like ggml-cuda.cu:2862)                          */
    B200_EXEC_MEGAKERNEL  = 4,   /* decode lists: phases of the persistent decode kernel — rope + KV store + attention as one launch
                                    (needs FUSION; also GGML_B200_MEGAKERNEL=1; off: GGML_B200_DISABLE_MEGAKERNEL).  Experimental: the default
                                    decode path is per-op kernels with the attention fused into one launch (b200_rope_kv_flash_attn) */
    B200_EXEC_MEGA_MMV    = 8,   /* ... and the Q4_K / Q6_K matvecs of the chain in the same launch (also: GGML_B200_MEGA_MMV=1)        */
};

/* The wide path — MUL_MAT on Q4_1 / Q5_1 / Q2_K / Q3_K / IQ4_NL / IQ4_XS / MXFP4 weights, MUL_MAT_ID, GET_ROWS on quantised tables
 * (b200_ops.h "the wide kernels", SURVEY.md §8 f2-f4) — is switched on per process with GGML_B200_WIDE=1.  It is off by default in
 * this round because its kernels were written after the round's GPU budget was spent: their arithmetic is verified on the CPU
 * (tests/test_extfmt_hostsim.py), the kernels themselves have not run on hardware yet (tests/test_gpu_zz_wide.py).  With the switch off
 * b200_executor_supports answers 0 for those nodes and ggml's scheduler keeps them on its CPU backend, exactly as before. */
B200_API int            b200_executor_wide_enabled(void);

typedef struct b200_executor b200_executor;

B200_API b200_executor *b200_executor_create(int device);
B200_API void           b200_executor_free(b200_executor *ex);
/* 1 if the executor can run this node exactly (the plug-in's supports_op answers with this) */
B200_API int            b200_executor_supports(const b200_node *node);
/* run the list in order on `stream`; asynchronous.  Returns b200_status. */
B200_API int            b200_executor_compute(b200_executor *ex, const b200_node *nodes, int n_nodes, void *stream, int flags);
/* dry run: how many kernel launches the executor would issue for this list with these flags (no device is touched, so the
 * fusion logic is testable on a CPU-only host); negative b200_status on unsupported nodes */
B200_API int64_t        b200_executor_plan(const b200_node *nodes, int n_nodes, int flags);
/* counters for tests / bench: kernels launched by the last compute (inside a replayed graph too),
 * number of CUDA-graph captures and replays so far */
B200_API int64_t        b200_executor_last_kernels(const b200_executor *ex);
/* persistent decode kernel: launches recorded so far and phases they covered (recorded at capture time, not per replay) */
B200_API int64_t        b200_executor_mk_launches(const b200_executor *ex);
B200_API int64_t        b200_executor_mk_phases(const b200_executor *ex);
B200_API int64_t        b200_executor_graph_captures(const b200_executor *ex);
B200_API int64_t        b200_executor_graph_replays(const b200_executor *ex);

#ifdef __cplusplus
}
#endif
#endif
