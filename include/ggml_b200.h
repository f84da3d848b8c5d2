/*
 * ggml_b200.h — the drop-in boundary of libggml-b200.so.
 *
 * The plug-in exports EXACTLY the two C symbols ggml's backend registry binds when it dlopen()s a
 * backend library (reference: ggml/src/ggml-backend-impl.h:214-246 GGML_BACKEND_DL_IMPL /
 * GGML_BACKEND_DL_SCORE_IMPL; loader: ggml/src/ggml-backend-reg.cpp:232-276 load_backend,
 * :569-593 ggml_backend_load_all_from_path incl. GGML_BACKEND_PATH):
 *
 *     ggml_backend_reg_t ggml_backend_init(void);   // required; reg->api_version == GGML_BACKEND_API_VERSION (1)
 *     int                ggml_backend_score(void);  // optional; 0 = "not usable on this machine"
 *
 * Everything else crosses the boundary through the five function-pointer tables of
 * ggml/src/ggml-backend-impl.h (cited per table below); their struct layouts are ggml's, so the
 * plug-in is compiled against the reference's own headers with -DGGML_MAX_NAME=128 (llama-box root
 * CMakeLists.txt:62 — sizeof(ggml_tensor) depends on it) and linked to the host's libggml-base.so.
 * This header restates the contract in plain C so that it can be read (and symbol-checked by
 * tests/test_abi.py) without the ggml tree; opaque types stand in for ggml's structs.
 *
 *   table (ggml-backend-impl.h)        implemented in llama-box_b200/plugin/ggml_b200.cpp
 *   ggml_backend_reg_i        :191-207  name "B200"; one device per compute-capability 9.0 GPU; get_proc_address -> NULL
 *   ggml_backend_device_i     :137-185  type GPU; caps {async, host_buffer, events}; supports_op = the op set of
 *                                       SURVEY.md §3.3 validated node by node by b200_executor_supports();
 *                                       offload_op = false; events = cudaEvent
 *   ggml_backend_buffer_type_i :17-35   cudaMalloc buffers, alignment 128; pinned host buffer type "B200_Host"
 *   ggml_backend_buffer_i      :41-66   set/get/memset/cpy/clear, synchronous; weights are kept in ggml's layout at
 *                                       the boundary and repacked lazily (b200_repack_rows) on first MUL_MAT use,
 *                                       get_tensor / set_tensor undo it, so ggml never observes the private layout
 *   ggml_backend_i             :87-124  one CUDA stream per backend; set/get_tensor_async; cpy_tensor_async =
 *                                       cudaMemcpyPeerAsync + event (the --tensor-split hidden-state handoff,
 *                                       replaces ggml-cuda.cu:2530-2583); graph_compute -> b200_executor_compute
 *
 * Errors: alloc_buffer returns NULL on OOM, graph_compute returns GGML_STATUS_FAILED (mapped by llama_decode to its
 * error codes, llama-context.cpp:1101-1106); nothing aborts the process and no exception crosses the boundary.
 * Environment switches (mirroring GGML_CUDA_DISABLE_GRAPHS / _FUSION, ggml-cuda.cu:2937,2862):
 *   GGML_B200_DISABLE_GRAPHS, GGML_B200_DISABLE_FUSION, GGML_B200_DISABLE_PDL, GGML_B200_DEBUG.
 */
#ifndef GGML_B200_H
#define GGML_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ggml_backend_reg * ggml_backend_reg_t;   /* ggml/include/ggml-backend.h */

__attribute__((visibility("default"))) ggml_backend_reg_t ggml_backend_init(void);
__attribute__((visibility("default"))) int                ggml_backend_score(void);

#ifdef __cplusplus
}
#endif
#endif
