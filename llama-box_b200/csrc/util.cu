// util.cu — library plumbing: error strings, launch counter, device queries, type geometry.
#include "common.cuh"
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void b200_set_error(const char * fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}
int b200_check(cudaError_t e, const char * what) {
    if (e == cudaSuccess) return B200_OK;
    b200_set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
    return B200_ERR_CUDA;
}
void b200_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int b200_sm_count() {
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cache[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cache[dev] = n;
    }
    return cache[dev];
}

bool b200_pdl_enabled() {
    static int v = -1;
    if (v < 0) v = getenv("GGML_B200_DISABLE_PDL") ? 0 : 1;
    return v == 1;
}

extern "C" int b200_abi_version(void) { return 1; }
extern "C" int b200_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }
extern "C" int b200_device_sm_count(int device) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
extern "C" const char * b200_last_error(void) { return g_err; }
extern "C" int64_t b200_kernel_launches(void) { return g_launches.load(std::memory_order_relaxed); }
extern "C" int64_t b200_block_elems(int t) { return type_block_elems(t); }
extern "C" int64_t b200_block_bytes(int t) { return type_block_bytes(t); }
extern "C" int64_t b200_row_bytes(int t, int64_t k) { const int64_t be = type_block_elems(t); return be > 0 && k % be == 0 ? k / be * type_block_bytes(t) : -1; }
