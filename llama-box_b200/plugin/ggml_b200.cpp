// ggml_b200.cpp — the drop-in boundary: a ggml backend plug-in (libggml-b200.so) for NVIDIA H100 (sm_90a).
//
// Exports exactly what ggml's registry binds when it dlopen()s a backend
// (ggml/src/ggml-backend-impl.h:214-246, ggml/src/ggml-backend-reg.cpp:232-276):
//     ggml_backend_reg_t ggml_backend_init(void);      int ggml_backend_score(void);
// and implements the five vtables of ggml-backend-impl.h:17-207 (registry, device, buffer type,
// buffer, backend/stream).  llama-box / llama.cpp load it with GGML_BACKEND_PATH=<abs path> or by file
// name next to the executable, unchanged.  Everything that computes is a call into the kernel library's
// C-ABI (include/b200_ops.h, include/b200_graph.h); this file only adapts ggml's structs.
//
// Compiled against the reference's own ggml headers (staged in oracle/_ref/include by `make -C oracle ref`) with
// -DGGML_MAX_NAME=128 to match llama-box (root CMakeLists.txt:62); libggml-base's symbols resolve against the host process.
// Replaces ggml/src/ggml-cuda/ggml-cuda.cu's backend plumbing (:500-760 buffers, :2495-2600 streams/events,
// :3138-3800 device/registry); nothing here is copied from it.
#include "ggml.h"
#include "ggml-backend.h"
#include "ggml-backend-impl.h"
#include "ggml-impl.h"

#include "../../include/b200_graph.h"

#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <mutex>
#include <string>
#include <unordered_set>
#include <vector>

#define B200_MAX_DEVICES 16

#define CUDA_OK(expr) b200_cuda_ok((expr), #expr, __FILE__, __LINE__)
static bool b200_cuda_ok(cudaError_t e, const char * what, const char * file, int line) {
    if (e == cudaSuccess) return true;
    fprintf(stderr, "ggml-b200: CUDA error %d (%s) in %s at %s:%d\n", (int)e, cudaGetErrorString(e), what, file, line);
    cudaGetLastError();
    return false;
}

// ------------------------------------------------------------------------------------------------
// contexts
// ------------------------------------------------------------------------------------------------
struct b200_device_ctx {
    int device = 0;
    std::string name, description;
    ggml_backend_buffer_type buft;        // device memory
    ggml_backend_buffer_type buft_host;   // pinned host memory
};

struct b200_buffer_ctx {
    int    device;
    void * base;
    // weight tensors whose rows currently are in the kernels' repacked layout (see b200_repack_rows), keyed by
    // tensor->data.  Whole-tensor uploads into a WEIGHTS buffer (what llama_model_loader does, llama-model-loader.cpp:1060,
    // 1095) are repacked right there, synchronously, at load time; anything uploaded in pieces is repacked the first time
    // a MUL_MAT consumes it, under `mu` and followed by a stream sync, so that no other stream or backend can observe a
    // half-converted tensor.  get_tensor / partial set_tensor convert back first: ggml never sees the private layout.
    std::mutex mu;
    std::unordered_set<const void *> repacked;
};

struct b200_backend_ctx {
    int device;
    cudaStream_t stream = nullptr;
    cudaEvent_t  copy_event = nullptr;     // reused for every hidden-state handoff issued by this backend (as ggml-cuda does, ggml-cuda.cu:2566-2575)
    b200_executor * ex = nullptr;
    std::vector<b200_node> nodes;
    std::string name;
};

// ---- statistics of the inter-device handoff (row a11), readable through reg->get_proc_address("ggml_b200_handoff_stats")
struct b200_handoff_stats { int64_t copies; int64_t bytes; double device_us; double host_us; };
static std::mutex g_stat_mu;
static b200_handoff_stats g_handoff = { 0, 0, 0.0, 0.0 };
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_handoff_pending;   // timing event pairs not yet read back

static b200_device_ctx   g_dev[B200_MAX_DEVICES];
static ggml_backend_device g_devices[B200_MAX_DEVICES];
static int               g_ndev = 0;
static ggml_backend_reg  g_reg;

static bool is_b200_buffer(ggml_backend_buffer_t b);
static bool is_repack_type(enum ggml_type t) { return t == GGML_TYPE_Q4_0 || t == GGML_TYPE_Q5_0 || t == GGML_TYPE_Q8_0 || t == GGML_TYPE_Q6_K; }
// 32-element block types whose rows are not a multiple of 256 elements (Qwen2-72B ffn_down: 29568, quantised Q5_0 / Q8_0 by the
// reference's fallback rule, llama-quant.cpp:442-470) are kept in a private layout padded with zero blocks (b200_padded_k)
static bool is_block32(enum ggml_type t) { return t == GGML_TYPE_Q4_0 || t == GGML_TYPE_Q5_0 || t == GGML_TYPE_Q8_0; }
static bool needs_padding(const ggml_tensor * t) { return is_block32(t->type) && t->ne[0] % 256 != 0; }

// ------------------------------------------------------------------------------------------------
// buffers (ggml_backend_buffer_i, ggml-backend-impl.h:41-66) — all calls synchronous on return,
// like the reference's (ggml-cuda.cu:586-600)
// ------------------------------------------------------------------------------------------------
static void buf_free(ggml_backend_buffer_t buffer) {
    b200_buffer_ctx * c = (b200_buffer_ctx *)buffer->context;
    cudaSetDevice(c->device);
    CUDA_OK(cudaFree(c->base));
    delete c;
}
static void * buf_get_base(ggml_backend_buffer_t buffer) { return ((b200_buffer_ctx *)buffer->context)->base; }

static enum ggml_status buf_init_tensor(ggml_backend_buffer_t, struct ggml_tensor *) { return GGML_STATUS_SUCCESS; }

// padded private layout <-> ggml rows, through a temporary (rows change their stride, so it cannot be done in place)
static bool convert_padded(const ggml_tensor * t, int inverse) {
    const int64_t nrows = ggml_nrows(t), k = t->ne[0];
    const size_t nat = (size_t)nrows * (size_t)b200_row_bytes((int)t->type, k), pad = (size_t)nrows * (size_t)b200_row_bytes((int)t->type, b200_padded_k((int)t->type, k));
    void * tmp = nullptr;
    if (!CUDA_OK(cudaMalloc(&tmp, inverse ? nat : pad))) return false;
    bool ok = b200_repack_rows_padded((int)t->type, t->data, tmp, nrows, k, inverse, cudaStreamPerThread) == B200_OK;
    ok = ok && CUDA_OK(cudaMemcpyAsync(t->data, tmp, inverse ? nat : pad, cudaMemcpyDeviceToDevice, cudaStreamPerThread));
    ok = CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread)) && ok;
    cudaFree(tmp);
    return ok;
}
// bring a weight tensor back to ggml's layout (before ggml reads or partially writes it)
static void ensure_native(b200_buffer_ctx * c, const ggml_tensor * t) {
    if (!is_repack_type(t->type)) return;
    std::lock_guard<std::mutex> lk(c->mu);
    if (!c->repacked.count(t->data)) return;
    cudaSetDevice(c->device);
    CUDA_OK(cudaDeviceSynchronize());                    // compute streams are non-blocking: order against every reader of the tensor
    if (needs_padding(t)) convert_padded(t, /* inverse */ 1);
    else b200_unpack_rows((int)t->type, t->data, ggml_nrows(t), t->ne[0], cudaStreamPerThread);
    CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
    c->repacked.erase(t->data);
}
static bool repack_k_ok(const ggml_tensor * t) {
    if (!ggml_is_contiguous(t)) return false;
    if (is_block32(t->type)) return t->ne[0] % 32 == 0;
    return t->ne[0] % 256 == 0 && (t->type != GGML_TYPE_Q6_K || t->ne[0] % 2048 == 0);
}
// convert a weight tensor to the kernels' layout, exactly once, visible to every stream when this returns
static bool ensure_repacked(b200_buffer_ctx * c, const ggml_tensor * t) {
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->repacked.count(t->data)) return true;
    cudaSetDevice(c->device);
    if (needs_padding(t)) { if (!convert_padded(t, 0)) return false; }
    else if (b200_repack_rows((int)t->type, t->data, ggml_nrows(t), t->ne[0], cudaStreamPerThread) != B200_OK) return false;
    if (!CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread))) return false;
    c->repacked.insert(t->data);
    return true;
}

static void buf_memset_tensor(ggml_backend_buffer_t buffer, struct ggml_tensor * tensor, uint8_t value, size_t offset, size_t size) {
    b200_buffer_ctx * c = (b200_buffer_ctx *)buffer->context;
    cudaSetDevice(c->device);
    ensure_native(c, tensor);
    CUDA_OK(cudaMemset((char *)tensor->data + offset, value, size));
}
static void buf_set_tensor(ggml_backend_buffer_t buffer, struct ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    b200_buffer_ctx * c = (b200_buffer_ctx *)buffer->context;
    cudaSetDevice(c->device);
    ensure_native(c, tensor);
    CUDA_OK(cudaMemcpy((char *)tensor->data + offset, data, size, cudaMemcpyHostToDevice));
    // load-time repack: a whole quantised weight tensor has just arrived (llama_model_loader::load_all_data)
    if (buffer->usage == GGML_BACKEND_BUFFER_USAGE_WEIGHTS && is_repack_type(tensor->type) && offset == 0 && size == ggml_nbytes(tensor) &&
        !tensor->view_src && repack_k_ok(tensor)) ensure_repacked(c, tensor);
}
static void buf_get_tensor(ggml_backend_buffer_t buffer, const struct ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    b200_buffer_ctx * c = (b200_buffer_ctx *)buffer->context;
    cudaSetDevice(c->device);
    ensure_native(c, tensor);
    CUDA_OK(cudaMemcpy(data, (const char *)tensor->data + offset, size, cudaMemcpyDeviceToHost));
}
static bool buf_cpy_tensor(ggml_backend_buffer_t buffer, const struct ggml_tensor * src, struct ggml_tensor * dst) {
    if (!is_b200_buffer(src->buffer)) return false;
    b200_buffer_ctx * sc = (b200_buffer_ctx *)src->buffer->context, * dc = (b200_buffer_ctx *)buffer->context;
    ensure_native(sc, src); ensure_native(dc, dst);
    if (sc->device == dc->device) { cudaSetDevice(dc->device); CUDA_OK(cudaMemcpy(dst->data, src->data, ggml_nbytes(src), cudaMemcpyDeviceToDevice)); }
    else CUDA_OK(cudaMemcpyPeer(dst->data, dc->device, src->data, sc->device, ggml_nbytes(src)));
    return true;
}
static void buf_clear(ggml_backend_buffer_t buffer, uint8_t value) {
    b200_buffer_ctx * c = (b200_buffer_ctx *)buffer->context;
    cudaSetDevice(c->device);
    CUDA_OK(cudaMemset(c->base, value, buffer->size));
    std::lock_guard<std::mutex> lk(c->mu);
    c->repacked.clear();
}
static const ggml_backend_buffer_i b200_buffer_iface = {
    /* free_buffer   */ buf_free,
    /* get_base      */ buf_get_base,
    /* init_tensor   */ buf_init_tensor,
    /* memset_tensor */ buf_memset_tensor,
    /* set_tensor    */ buf_set_tensor,
    /* get_tensor    */ buf_get_tensor,
    /* cpy_tensor    */ buf_cpy_tensor,
    /* clear         */ buf_clear,
    /* reset         */ nullptr,
};
static bool is_b200_buffer(ggml_backend_buffer_t b) { return b && b->iface.free_buffer == buf_free; }

// ---- device buffer type (ggml_backend_buffer_type_i, ggml-backend-impl.h:17-35)
static const char * buft_name(ggml_backend_buffer_type_t buft) { return ((b200_device_ctx *)buft->device->context)->name.c_str(); }
static ggml_backend_buffer_t buft_alloc(ggml_backend_buffer_type_t buft, size_t size) {
    b200_device_ctx * d = (b200_device_ctx *)buft->device->context;
    cudaSetDevice(d->device);
    void * p = nullptr;
    const size_t padded = size + 256;                       // bulk copies never run past a tensor, but keep slack like ggml-cuda does (ggml-cuda.cu:684-698)
    if (cudaMalloc(&p, padded > 0 ? padded : 256) != cudaSuccess) {   // recoverable: NULL on OOM (ggml-cuda.cu:666-671)
        cudaGetLastError();
        fprintf(stderr, "ggml-b200: failed to allocate %.2f MiB on device %d\n", size / 1048576.0, d->device);
        return nullptr;
    }
    b200_buffer_ctx * c = new b200_buffer_ctx(); c->device = d->device; c->base = p;
    return ggml_backend_buffer_init(buft, b200_buffer_iface, c, size);
}
static size_t buft_alignment(ggml_backend_buffer_type_t) { return 128; }
static size_t buft_alloc_size(ggml_backend_buffer_type_t, const struct ggml_tensor * t) {
    // room for the padded private layout of 32-element block weights with k % 256 != 0 (ggml-cuda pads quantised rows too: ggml-cuda.cu:684-698)
    if (needs_padding(t) && ggml_is_contiguous(t)) return (size_t)ggml_nrows(t) * (size_t)b200_row_bytes((int)t->type, b200_padded_k((int)t->type, t->ne[0]));
    return ggml_nbytes(t);
}
static bool buft_is_host(ggml_backend_buffer_type_t) { return false; }

// ---- pinned host buffer type (used for CPU-side activations and async uploads, llama-context.cpp:231-238)
static void hbuf_free(ggml_backend_buffer_t buffer) { CUDA_OK(cudaFreeHost(buffer->context)); }
static void * hbuf_base(ggml_backend_buffer_t buffer) { return buffer->context; }
static void hbuf_memset(ggml_backend_buffer_t, struct ggml_tensor * t, uint8_t v, size_t off, size_t size) { memset((char *)t->data + off, v, size); }
static void hbuf_set(ggml_backend_buffer_t, struct ggml_tensor * t, const void * data, size_t off, size_t size) { memcpy((char *)t->data + off, data, size); }
static void hbuf_get(ggml_backend_buffer_t, const struct ggml_tensor * t, void * data, size_t off, size_t size) { memcpy(data, (const char *)t->data + off, size); }
static bool hbuf_cpy(ggml_backend_buffer_t, const struct ggml_tensor * src, struct ggml_tensor * dst) {
    if (ggml_backend_buffer_is_host(src->buffer)) { memcpy(dst->data, src->data, ggml_nbytes(src)); return true; }
    return false;
}
static void hbuf_clear(ggml_backend_buffer_t buffer, uint8_t v) { memset(buffer->context, v, buffer->size); }
static const ggml_backend_buffer_i b200_host_buffer_iface = { hbuf_free, hbuf_base, nullptr, hbuf_memset, hbuf_set, hbuf_get, hbuf_cpy, hbuf_clear, nullptr };
static const char * hbuft_name(ggml_backend_buffer_type_t) { return "B200_Host"; }
static ggml_backend_buffer_t hbuft_alloc(ggml_backend_buffer_type_t buft, size_t size) {
    void * p = nullptr;
    if (cudaMallocHost(&p, size > 0 ? size : 64) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return ggml_backend_buffer_init(buft, b200_host_buffer_iface, p, size);
}
static size_t hbuft_alignment(ggml_backend_buffer_type_t) { return 64; }
static bool hbuft_is_host(ggml_backend_buffer_type_t) { return true; }

// ------------------------------------------------------------------------------------------------
// ggml_tensor -> b200_tensor / b200_node (include/b200_graph.h mirrors ggml.h:613-645 1:1)
// ------------------------------------------------------------------------------------------------
static void to_b200(const ggml_tensor * t, b200_tensor & o) {
    memset(&o, 0, sizeof(o));
    if (!t) return;
    o.id = (uint64_t)(uintptr_t)t; o.data = t->data; o.type = (int32_t)t->type; o.flags = t->flags;   // GGML_TENSOR_FLAG_OUTPUT etc. (ggml.h:602-607)
    for (int i = 0; i < 4; i++) { o.ne[i] = t->ne[i]; o.nb[i] = (int64_t)t->nb[i]; }
}
// false = this op is not one the hot path handles
static bool node_to_b200(const ggml_tensor * t, b200_node & n) {
    memset(&n, 0, sizeof(n));
    switch (t->op) {
        case GGML_OP_NONE: case GGML_OP_RESHAPE: case GGML_OP_VIEW: case GGML_OP_PERMUTE: case GGML_OP_TRANSPOSE: n.op = B200_OP_NONE; break;
        case GGML_OP_MUL_MAT:  n.op = B200_OP_MUL_MAT; break;
        case GGML_OP_RMS_NORM: n.op = B200_OP_RMS_NORM; break;
        case GGML_OP_MUL:      n.op = B200_OP_MUL; break;
        case GGML_OP_ADD:      n.op = B200_OP_ADD; break;
        case GGML_OP_ROPE:     n.op = B200_OP_ROPE; break;
        case GGML_OP_SET_ROWS: n.op = B200_OP_SET_ROWS; break;
        case GGML_OP_FLASH_ATTN_EXT: n.op = B200_OP_FLASH_ATTN_EXT; break;
        case GGML_OP_GLU:
            if (ggml_get_glu_op(t) != GGML_GLU_OP_SWIGLU || !t->src[1] || t->op_params[1] != 0) return false;   // split form, not swapped
            n.op = B200_OP_GLU_SWIGLU; break;
        case GGML_OP_GET_ROWS: n.op = B200_OP_GET_ROWS; break;
        case GGML_OP_CPY:      n.op = B200_OP_CPY; break;
        case GGML_OP_MUL_MAT_ID: n.op = B200_OP_MUL_MAT_ID; break;
        // mixture-of-experts router glue (llama-graph.cpp build_moe_ffn), wide path only
        case GGML_OP_SOFT_MAX: n.op = B200_OP_SOFT_MAX; break;
        case GGML_OP_ARGSORT:  n.op = B200_OP_ARGSORT; break;
        case GGML_OP_SUM_ROWS: n.op = B200_OP_SUM_ROWS; break;
        case GGML_OP_DIV:      n.op = B200_OP_DIV; break;
        case GGML_OP_CONT:     n.op = B200_OP_CONT; break;        // attention without -fa (wide path)
        case GGML_OP_SCALE:    n.op = B200_OP_SCALE; break;       // MoE gating variants (wide path)
        case GGML_OP_UNARY:    n.op = B200_OP_UNARY; break;       // SILU / SIGMOID only (op_params[0] = ggml_unary_op; checked by the executor)     // wide path (GGML_B200_WIDE=1); refused by b200_executor_supports otherwise
        default: return false;
    }
    to_b200(t, n.dst);
    int ns = 0;
    for (int i = 0; i < GGML_MAX_SRC && i < B200_MAX_SRC; i++) if (t->src[i]) { to_b200(t->src[i], n.src[i]); ns = i + 1; }
    for (int i = B200_MAX_SRC; i < GGML_MAX_SRC; i++) if (t->src[i]) return false;
    n.n_src = ns;
    memcpy(n.op_params, t->op_params, sizeof(n.op_params));
    // CPY writes into src[1] (ggml.c ggml_cpy_impl: result is a view of b); the node's own data is that view
    return true;
}

// ------------------------------------------------------------------------------------------------
// backend = one stream (ggml_backend_i, ggml-backend-impl.h:87-124)
// ------------------------------------------------------------------------------------------------
static const char * be_name(ggml_backend_t b) { return ((b200_backend_ctx *)b->context)->name.c_str(); }
static double now_us() { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static bool g_timing_flag(); static long g_calls_ref(); static long g_nodes_ref(); static long g_kernels_ref(); static double g_conv_ref(); static double g_exec_ref();
static void be_free(ggml_backend_t b) {
    b200_backend_ctx * c = (b200_backend_ctx *)b->context;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (g_timing_flag() && g_calls_ref()) fprintf(stderr, "ggml-b200 timing: %ld graph_compute calls, %.1f nodes and %.1f kernels per call, host: %.1f us translate + %.1f us executor per call; graph captures %lld replays %lld\n",
                                      g_calls_ref(), (double)g_nodes_ref() / g_calls_ref(), (double)g_kernels_ref() / g_calls_ref(), g_conv_ref() / g_calls_ref(), g_exec_ref() / g_calls_ref(), (long long)b200_executor_graph_captures(c->ex), (long long)b200_executor_graph_replays(c->ex));
    b200_executor_free(c->ex);
    if (c->copy_event) cudaEventDestroy(c->copy_event);
    cudaStreamDestroy(c->stream);
    delete c; delete b;
}
static void be_set_tensor_async(ggml_backend_t b, struct ggml_tensor * t, const void * data, size_t offset, size_t size) {
    b200_backend_ctx * c = (b200_backend_ctx *)b->context;
    cudaSetDevice(c->device);
    ggml_backend_buffer_t buf = t->view_src ? t->view_src->buffer : t->buffer;
    if (is_b200_buffer(buf)) ensure_native((b200_buffer_ctx *)buf->context, t);
    CUDA_OK(cudaMemcpyAsync((char *)t->data + offset, data, size, cudaMemcpyHostToDevice, c->stream));
}
static void be_get_tensor_async(ggml_backend_t b, const struct ggml_tensor * t, void * data, size_t offset, size_t size) {
    b200_backend_ctx * c = (b200_backend_ctx *)b->context;
    cudaSetDevice(c->device);
    ggml_backend_buffer_t buf = t->view_src ? t->view_src->buffer : t->buffer;
    if (is_b200_buffer(buf) && is_repack_type(t->type)) { cudaStreamSynchronize(c->stream); ensure_native((b200_buffer_ctx *)buf->context, t); }
    CUDA_OK(cudaMemcpyAsync(data, (const char *)t->data + offset, size, cudaMemcpyDeviceToHost, c->stream));
}
// the inter-layer hidden-state handoff of --tensor-split (replaces ggml_backend_cuda_cpy_tensor_async,
// ggml-cuda.cu:2530-2583): one peer copy over NVLink on the source stream, an event, the destination waits
static bool be_cpy_tensor_async(ggml_backend_t bsrc, ggml_backend_t bdst, const struct ggml_tensor * src, struct ggml_tensor * dst) {
    if (bsrc->iface.get_name != be_name || bdst->iface.get_name != be_name) return false;
    ggml_backend_buffer_t sb = src->view_src ? src->view_src->buffer : src->buffer, db = dst->view_src ? dst->view_src->buffer : dst->buffer;
    if (!is_b200_buffer(sb) || !is_b200_buffer(db)) return false;
    b200_backend_ctx * cs = (b200_backend_ctx *)bsrc->context, * cd = (b200_backend_ctx *)bdst->context;
    if (((b200_buffer_ctx *)sb->context)->device != cs->device || ((b200_buffer_ctx *)db->context)->device != cd->device) return false;
    if (cs == cd) {
        cudaSetDevice(cs->device);
        return CUDA_OK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, cs->stream));
    }
    const double h0 = now_us();
    cudaSetDevice(cs->device);
    // GGML_B200_TIMING / handoff statistics: timing events around the peer copy on the source stream
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    static const bool timed = g_timing_flag() || getenv("GGML_B200_HANDOFF_TIMING") != nullptr;
    if (timed) { cudaEventCreate(&t0); cudaEventCreate(&t1); cudaEventRecord(t0, cs->stream); }
    bool ok;
    if (cs->device == cd->device) ok = CUDA_OK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, cs->stream));
    else                          ok = CUDA_OK(cudaMemcpyPeerAsync(dst->data, cd->device, src->data, cs->device, ggml_nbytes(dst), cs->stream));
    if (!ok) return false;
    if (timed) cudaEventRecord(t1, cs->stream);
    if (!cs->copy_event && !CUDA_OK(cudaEventCreateWithFlags(&cs->copy_event, cudaEventDisableTiming))) return false;
    CUDA_OK(cudaEventRecord(cs->copy_event, cs->stream));
    cudaSetDevice(cd->device);
    CUDA_OK(cudaStreamWaitEvent(cd->stream, cs->copy_event, 0));
    {
        std::lock_guard<std::mutex> lk(g_stat_mu);
        g_handoff.copies++; g_handoff.bytes += (int64_t)ggml_nbytes(dst); g_handoff.host_us += now_us() - h0;
        if (timed) g_handoff_pending.emplace_back(t0, t1);
    }
    return true;
}
// drain finished timing pairs into the statistics (called with every stream idle, or lazily when the list grows)
static void handoff_collect(bool all) {
    std::lock_guard<std::mutex> lk(g_stat_mu);
    size_t keep = 0;
    for (auto & pr : g_handoff_pending) {
        if (all) cudaEventSynchronize(pr.second);
        if (cudaEventQuery(pr.second) == cudaSuccess) {
            float ms = 0; if (cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) g_handoff.device_us += ms * 1e3;
            cudaEventDestroy(pr.first); cudaEventDestroy(pr.second);
        } else g_handoff_pending[keep++] = pr;
    }
    g_handoff_pending.resize(keep);
    cudaGetLastError();
}
extern "C" void ggml_b200_handoff_stats(int64_t * copies, int64_t * bytes, double * device_us, double * host_us) {
    handoff_collect(true);
    std::lock_guard<std::mutex> lk(g_stat_mu);
    if (copies) *copies = g_handoff.copies; if (bytes) *bytes = g_handoff.bytes;
    if (device_us) *device_us = g_handoff.device_us; if (host_us) *host_us = g_handoff.host_us;
}
extern "C" void ggml_b200_handoff_reset(void) {
    handoff_collect(true);
    std::lock_guard<std::mutex> lk(g_stat_mu);
    g_handoff = { 0, 0, 0.0, 0.0 };
}
static void be_synchronize(ggml_backend_t b) {
    b200_backend_ctx * c = (b200_backend_ctx *)b->context;
    cudaSetDevice(c->device);
    CUDA_OK(cudaStreamSynchronize(c->stream));
}

// GGML_B200_TIMING=1: host-side cost of graph_compute (node translation / executor call), printed when the backend is freed
static bool g_timing = getenv("GGML_B200_TIMING") != nullptr;
static double g_t_conv = 0, g_t_exec = 0; static long g_calls = 0, g_nodes = 0, g_kernels = 0;

static bool g_timing_flag() { return g_timing; } static long g_calls_ref() { return g_calls; } static long g_nodes_ref() { return g_nodes; } static long g_kernels_ref() { return g_kernels; }
static double g_conv_ref() { return g_t_conv; } static double g_exec_ref() { return g_t_exec; }

static enum ggml_status be_graph_compute(ggml_backend_t b, struct ggml_cgraph * cgraph) {
    b200_backend_ctx * c = (b200_backend_ctx *)b->context;
    cudaSetDevice(c->device);
    const double t0 = g_timing ? now_us() : 0;
    const int n = ggml_graph_n_nodes(cgraph);
    c->nodes.resize(n);
    for (int i = 0; i < n; i++) {
        ggml_tensor * t = ggml_graph_node(cgraph, i);
        if (!node_to_b200(t, c->nodes[i])) { fprintf(stderr, "ggml-b200: op %s is not supported (node %s)\n", ggml_op_name(t->op), t->name); return GGML_STATUS_FAILED; }
        // weights that did not arrive as one whole-tensor upload (chunked --no-mmap loads) are converted here, once, with the
        // buffer mutex held across check + conversion + mark and a stream sync before anyone may read them
        if ((t->op == GGML_OP_MUL_MAT || t->op == GGML_OP_MUL_MAT_ID || t->op == GGML_OP_GET_ROWS) && is_repack_type(t->src[0]->type)) {
            const ggml_tensor * w = t->src[0];
            ggml_backend_buffer_t wb = w->view_src ? w->view_src->buffer : w->buffer;
            if (!is_b200_buffer(wb)) { fprintf(stderr, "ggml-b200: %s weight %s is not in a B200 buffer\n", ggml_op_name(t->op), w->name); return GGML_STATUS_FAILED; }
            if (!ensure_repacked((b200_buffer_ctx *)wb->context, w)) { fprintf(stderr, "ggml-b200: repack failed: %s\n", b200_last_error()); return GGML_STATUS_FAILED; }
            cudaSetDevice(c->device);
        }
    }
    static int dumped = 0;
    if (getenv("GGML_B200_DUMP_GRAPH") && n > 200 && dumped < 1) {           // debugging: the node list as the executor sees it
        dumped++;
        for (int i = 0; i < n && i < 140; i++) {
            ggml_tensor * t = ggml_graph_node(cgraph, i);
            fprintf(stderr, "node %3d %-14s %-22s [%lld,%lld,%lld] nb1=%lld src0=%s(%s) src1=%s data=%p\n", i, ggml_op_name(t->op), t->name, (long long)t->ne[0], (long long)t->ne[1], (long long)t->ne[2], (long long)t->nb[1],
                    t->src[0] ? t->src[0]->name : "-", t->src[0] ? ggml_type_name(t->src[0]->type) : "", t->src[1] ? t->src[1]->name : "-", t->data);
        }
    }
    const double t1 = g_timing ? now_us() : 0;
    const int st = b200_executor_compute(c->ex, c->nodes.data(), n, c->stream, B200_EXEC_CUDA_GRAPHS | B200_EXEC_FUSION);
    if (g_timing) { const double t2 = now_us(); g_t_conv += t1 - t0; g_t_exec += t2 - t1; g_calls++; g_nodes += n; g_kernels += b200_executor_last_kernels(c->ex); }
    if (st != B200_OK) { fprintf(stderr, "ggml-b200: graph_compute failed: %s\n", b200_last_error()); return GGML_STATUS_FAILED; }
    return GGML_STATUS_SUCCESS;
}

static void be_event_record(ggml_backend_t b, ggml_backend_event_t ev) {
    b200_backend_ctx * c = (b200_backend_ctx *)b->context;
    cudaSetDevice(c->device);
    CUDA_OK(cudaEventRecord((cudaEvent_t)ev->context, c->stream));
}
static void be_event_wait(ggml_backend_t b, ggml_backend_event_t ev) {
    b200_backend_ctx * c = (b200_backend_ctx *)b->context;
    cudaSetDevice(c->device);
    CUDA_OK(cudaStreamWaitEvent(c->stream, (cudaEvent_t)ev->context, 0));
}
static const ggml_backend_i b200_backend_iface = {
    /* get_name           */ be_name,
    /* free               */ be_free,
    /* set_tensor_async   */ be_set_tensor_async,
    /* get_tensor_async   */ be_get_tensor_async,
    /* cpy_tensor_async   */ be_cpy_tensor_async,
    /* synchronize        */ be_synchronize,
    /* graph_plan_create  */ nullptr,
    /* graph_plan_free    */ nullptr,
    /* graph_plan_update  */ nullptr,
    /* graph_plan_compute */ nullptr,
    /* graph_compute      */ be_graph_compute,
    /* event_record       */ be_event_record,
    /* event_wait         */ be_event_wait,
};
static ggml_guid g_guid = { 0xb2, 0x00, 0x5a, 0x10, 0x0a, 0x67, 0x67, 0x6d, 0x6c, 0x2d, 0x62, 0x32, 0x30, 0x30, 0x01, 0x00 };

// ------------------------------------------------------------------------------------------------
// device (ggml_backend_device_i, ggml-backend-impl.h:137-185)
// ------------------------------------------------------------------------------------------------
static const char * dev_name(ggml_backend_dev_t d) { return ((b200_device_ctx *)d->context)->name.c_str(); }
static const char * dev_desc(ggml_backend_dev_t d) { return ((b200_device_ctx *)d->context)->description.c_str(); }
static void dev_memory(ggml_backend_dev_t d, size_t * free, size_t * total) {
    cudaSetDevice(((b200_device_ctx *)d->context)->device);
    if (!CUDA_OK(cudaMemGetInfo(free, total))) { *free = 0; *total = 0; }
}
static enum ggml_backend_dev_type dev_type(ggml_backend_dev_t) { return GGML_BACKEND_DEVICE_TYPE_GPU; }
static void dev_props(ggml_backend_dev_t d, struct ggml_backend_dev_props * p) {
    p->name = dev_name(d); p->description = dev_desc(d); p->type = GGML_BACKEND_DEVICE_TYPE_GPU;
    dev_memory(d, &p->memory_free, &p->memory_total);
    p->caps = { /* async */ true, /* host_buffer */ true, /* buffer_from_host_ptr */ false, /* events */ true };
}
static ggml_backend_t dev_init_backend(ggml_backend_dev_t d, const char *) {
    b200_device_ctx * dc = (b200_device_ctx *)d->context;
    cudaSetDevice(dc->device);
    b200_backend_ctx * c = new b200_backend_ctx();
    c->device = dc->device; c->name = dc->name;
    if (!CUDA_OK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking))) { delete c; return nullptr; }
    c->ex = b200_executor_create(dc->device);
    if (!c->ex) { cudaStreamDestroy(c->stream); delete c; return nullptr; }
    // NVLink peer access for the hidden-state handoff, enabled once (ggml-cuda enables it lazily per batch size)
    for (int j = 0; j < g_ndev; j++) {
        const int peer = g_dev[j].device;                    // CUDA ordinal of plug-in device j (they differ on mixed boxes)
        if (peer == dc->device) continue;
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, dc->device, peer) == cudaSuccess && can) { cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0); if (e != cudaSuccess) cudaGetLastError(); }
    }
    ggml_backend_t be = new ggml_backend{ &g_guid, b200_backend_iface, d, c };
    return be;
}
static ggml_backend_buffer_type_t dev_buft(ggml_backend_dev_t d) { return &((b200_device_ctx *)d->context)->buft; }
static ggml_backend_buffer_type_t dev_host_buft(ggml_backend_dev_t d) { return &((b200_device_ctx *)d->context)->buft_host; }

static bool dev_supports_op(ggml_backend_dev_t, const struct ggml_tensor * op) {
    b200_node n;
    if (op->op == GGML_OP_SOFT_MAX && op->src[1] && !b200_executor_wide_enabled()) {         // with a mask: the attention of a graph built without -fa (a mask-free SOFT_MAX is the MoE router's, below)
        // attention without -fa (SOFT_MAX + batched KQ / KQV matmuls, llama-graph.cpp:1267-1330) is not on this backend's hot
        // path: ggml's scheduler will run those nodes on the CPU backend.  Say so once, loudly — llama-box only turns flash
        // attention on with -fa (llama-box/engine_param.hpp:772-779).
        static std::once_flag warned;
        std::call_once(warned, [] { GGML_LOG_WARN("ggml-b200: this graph uses non-flash attention (SOFT_MAX); the B200 backend implements FLASH_ATTN_EXT only — "
                                                  "start llama-box / llama.cpp with -fa (--flash-attn) or attention will run on the CPU backend\n"); });
        return false;
    }
    if (!node_to_b200(op, n)) return false;
    if (op->op == GGML_OP_CPY) {
        // only the contiguous f32 -> f16/f32 casts of the mask / KV path
        if (!op->src[1] || !ggml_is_contiguous(op->src[0]) || !ggml_is_contiguous(op->src[1])) return false;
    }
    // data pointers are not assigned yet when the scheduler asks: validate with a 16-byte aligned stand-in
    // (ggml-alloc places every tensor at a multiple of get_alignment() = 128)
    auto fake = [](b200_tensor & t) { if (t.id && !t.data) t.data = (void *)(uintptr_t)0x1000; };
    fake(n.dst);
    for (int i = 0; i < n.n_src; i++) fake(n.src[i]);
    if (n.op == B200_OP_NONE) return true;
    const bool ok = b200_executor_supports(&n) != 0;
    static const bool dbg = getenv("GGML_B200_DEBUG") != nullptr;
    if (dbg && !ok) {
        fprintf(stderr, "ggml-b200: supports_op(%s) = no:", ggml_op_name(op->op));
        for (int i = 0; i < n.n_src; i++) fprintf(stderr, " src%d{t=%d ne=[%lld,%lld,%lld,%lld] nb=[%lld,%lld,%lld,%lld]}", i, n.src[i].type, (long long)n.src[i].ne[0], (long long)n.src[i].ne[1], (long long)n.src[i].ne[2], (long long)n.src[i].ne[3], (long long)n.src[i].nb[0], (long long)n.src[i].nb[1], (long long)n.src[i].nb[2], (long long)n.src[i].nb[3]);
        fprintf(stderr, " dst{t=%d ne=[%lld,%lld,%lld,%lld] nb1=%lld}\n", n.dst.type, (long long)n.dst.ne[0], (long long)n.dst.ne[1], (long long)n.dst.ne[2], (long long)n.dst.ne[3], (long long)n.dst.nb[1]);
    }
    return ok;
}
static bool dev_supports_buft(ggml_backend_dev_t d, ggml_backend_buffer_type_t buft) {
    // own device memory only, like ggml-cuda on discrete GPUs (ggml-cuda.cu:3538-3547): tensors living in the pinned host
    // buffer type (CPU-resident layers with -ngl below the layer count, llama-model.cpp:321-333) belong to the CPU backend;
    // the scheduler copies the activations across the boundary
    b200_device_ctx * dc = (b200_device_ctx *)d->context;
    return buft == &dc->buft;
}
static bool dev_offload_op(ggml_backend_dev_t, const struct ggml_tensor *) { return false; }
static ggml_backend_event_t dev_event_new(ggml_backend_dev_t d) {
    cudaSetDevice(((b200_device_ctx *)d->context)->device);
    cudaEvent_t ev;
    if (!CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming))) return nullptr;
    return new ggml_backend_event{ d, ev };
}
static void dev_event_free(ggml_backend_dev_t, ggml_backend_event_t ev) { CUDA_OK(cudaEventDestroy((cudaEvent_t)ev->context)); delete ev; }
static void dev_event_sync(ggml_backend_dev_t, ggml_backend_event_t ev) { CUDA_OK(cudaEventSynchronize((cudaEvent_t)ev->context)); }

static const ggml_backend_device_i b200_device_iface = {
    dev_name, dev_desc, dev_memory, dev_type, dev_props, dev_init_backend, dev_buft, dev_host_buft,
    /* buffer_from_host_ptr */ nullptr, dev_supports_op, dev_supports_buft, dev_offload_op, dev_event_new, dev_event_free, dev_event_sync,
};

// ------------------------------------------------------------------------------------------------
// registry (ggml_backend_reg_i, ggml-backend-impl.h:191-207)
// ------------------------------------------------------------------------------------------------
static const char * reg_name(ggml_backend_reg_t) { return "B200"; }
static size_t reg_dev_count(ggml_backend_reg_t) { return (size_t)g_ndev; }
static ggml_backend_dev_t reg_get_dev(ggml_backend_reg_t, size_t i) { return i < (size_t)g_ndev ? &g_devices[i] : nullptr; }
// no split buffers / n_threads / extra bufts (NULL is legal); two diagnostic entry points of our own
static void * reg_proc(ggml_backend_reg_t, const char * name) {
    if (!strcmp(name, "ggml_b200_handoff_stats")) return (void *)ggml_b200_handoff_stats;
    if (!strcmp(name, "ggml_b200_handoff_reset")) return (void *)ggml_b200_handoff_reset;
    return nullptr;
}

// devices the sm_90a kernels run on: compute capability 9.0 (H100 / H200)
static int count_sm90(int * ids) {
    int n = 0, nd = 0;
    if (cudaGetDeviceCount(&nd) != cudaSuccess) { cudaGetLastError(); return 0; }
    for (int i = 0; i < nd && n < B200_MAX_DEVICES; i++) {
        int major = 0, minor = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess &&
            cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, i) == cudaSuccess && major == 9 && minor == 0) { if (ids) ids[n] = i; n++; }
    }
    return n;
}

extern "C" {
GGML_BACKEND_API ggml_backend_reg_t ggml_backend_init(void);
GGML_BACKEND_API int ggml_backend_score(void);
}

ggml_backend_reg_t ggml_backend_init(void) {
    static std::once_flag once;
    std::call_once(once, [] {
        int ids[B200_MAX_DEVICES];
        g_ndev = count_sm90(ids);
        for (int i = 0; i < g_ndev; i++) {
            b200_device_ctx & d = g_dev[i];
            cudaDeviceProp prop; cudaGetDeviceProperties(&prop, ids[i]);
            d.device = ids[i]; d.name = "B200" + std::to_string(i); d.description = prop.name;
            g_devices[i] = { b200_device_iface, &g_reg, &d };
            d.buft      = { { buft_name, buft_alloc, buft_alignment, /* get_max_size */ nullptr, buft_alloc_size, buft_is_host }, &g_devices[i], nullptr };
            d.buft_host = { { hbuft_name, hbuft_alloc, hbuft_alignment, nullptr, nullptr, hbuft_is_host }, &g_devices[i], nullptr };
        }
        g_reg = { GGML_BACKEND_API_VERSION, { reg_name, reg_dev_count, reg_get_dev, reg_proc }, nullptr };
    });
    return &g_reg;
}

// 0 = "not usable here" (no sm_90 device): the registry then skips us (ggml-backend-reg.cpp:493-563)
int ggml_backend_score(void) { return count_sm90(nullptr) > 0 ? 100 : 0; }
