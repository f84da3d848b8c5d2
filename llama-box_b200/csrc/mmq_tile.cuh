// mmq_tile.cuh — what the tensor-core tile kernels of mmq_tc.cu (Q4_K / Q5_K / Q6_K) and mmq_tc32.cu (Q4_0 / Q5_0 / Q8_0) share, dense
// and GROUPED (MUL_MAT_ID, mmid_route.cu).  Each kernel file keeps its own transform and consumer loops, shared-memory map and
// activation image.
#pragma once
#include "common.cuh"

#define MMQ_TM 128
#define MMQ_TN 128
#define MMQ_THREADS 384             // warps 0-7: two consumer warpgroups (tile rows 0-63 / 64-127), warps 8-11: transform
#define MMQ_PANEL 2048              // one 16-byte K-chunk of 128 rows

// The device-built schedule of a grouped MUL_MAT_ID.  The (token, slot) pairs are grouped by expert, in the order t * n_used + s inside
// each expert, and each expert's run is padded to whole 128-column tiles; column tile ct belongs to expert tile_expert[ct] and its column j
// holds pair cols[128 ct + j] (-1: padding).  The number of tiles in use, *ntt, is known on the device only: launches are sized from the
// host's upper bound and the CTAs past it do nothing.
struct MmidMap {
    const int32_t * ntt;            // column tiles in use (device)
    const int32_t * tile_expert;    // [ct] expert of column tile ct
    const int32_t * cols;           // [ct * 128 + j] pair t * n_used + s, or -1
    int32_t n_used, n_b1;
    int64_t b_tok_stride, b_slot_stride;                        // activation of pair (t, s): b + t * b_tok_stride + (s % n_b1) * b_slot_stride (floats)
    int64_t expert_stride;                                      // bytes between the experts' weight matrices
    int64_t dst_tok_stride, dst_slot_stride;                    // output rows of pair (t, s): dst + t * dst_tok_stride + s * dst_slot_stride (floats)
};

// One tile GEMM: dst[n][r] = sum_k W[r][k] x[n][k] for r < m, n < ncols.  k is the length of the (padded) weight rows, k_valid <= k the
// elements that exist in X.  Dense when map is null; GROUPED otherwise: W is the first expert's matrix, X the activations gathered
// through the map, ncols = 128 x the upper bound of column tiles, and dst, ldd, x_col_stride are unused.
struct MmqJob {
    const void * W; const float * X; int64_t x_col_stride, k_valid;
    float * dst; int64_t ldd, m, k, ncols;
    void * workspace;               // 16-byte aligned, mmq_tile_workspace(type, k, ncols) bytes: the activation image
    const MmidMap * map;
};

struct MmqTileArgs {                // the parameters both tile kernels read
    const uint8_t * W;              // weights (repacked rows, see repack.cu)
    const uint8_t * ws;             // activation image (the file's quantiser)
    float *         dst;            // dense: [ncols][ldd] f32
    int64_t m, k, ncols, ldd, rb, nt;                          // rb: bytes per weight row, nt: column tiles (GROUPED: the upper bound)
    int32_t nks, n_tiles;                                      // nks: K steps per tile; GROUPED: n_tiles is the upper bound, the kernel reads the real count
    unsigned long long * prof;      // per-role cycle counters of CTA 0 (B200_MMQ_PROF), normally null
    MmidMap map;                    // GROUPED only
    int32_t n_mtiles;
};

// column tiles of the launch (GROUPED: from the device, 32-bit tile arithmetic)
template <bool GROUPED> __device__ __forceinline__ auto mmq_col_tiles(const MmqTileArgs & a) {
    if constexpr (GROUPED) return *a.map.ntt; else return a.nt;
}

// The quantisers' 8 elements [k0, k0 + 8) of activation-image column n: the dense column n of x (zeros from k_valid up and for columns
// from ncols up) or, GATHER, the column of pair map.cols[n] (zeros for padding)
template <bool GATHER>
__device__ __forceinline__ void mmq_load_col8(float (&v)[8], const float * x, int64_t x_col_stride, int64_t ncols, int64_t k_valid,
                                              const MmidMap & map, int64_t n, int64_t k0) {
    auto ld8 = [&](const float * p) {
        const float4 a = ((const float4 *)p)[0], b = ((const float4 *)p)[1];
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    };
    if constexpr (GATHER) {
        const int pr = map.cols[n], nu = map.n_used;
        if (pr >= 0) { const int t = pr / nu, s = pr % nu; ld8(x + (int64_t)t * map.b_tok_stride + (s % map.n_b1) * map.b_slot_stride + k0); }
    } else if (n < ncols && k0 < k_valid) ld8(x + n * x_col_stride + k0);
}

// weight row t of m-tile mt; rows past the end read row m - 1 (their results are never stored).  GROUPED: of column tile ct's expert
template <bool GROUPED>
__device__ __forceinline__ const uint8_t * mmq_weight_row(const MmqTileArgs & a, int64_t mt, int64_t ct, int t) {
    int64_t r = mt * MMQ_TM + t; if (r >= a.m) r = a.m - 1;
    const uint8_t * row = a.W + r * a.rb;
    if constexpr (GROUPED) row += (int64_t)a.map.tile_expert[ct] * a.map.expert_stride;
    return row;
}

// Epilogue of a consumer thread: acc[4 j + 2 h + e] is row mt * 128 + ra + 8 h, column nt * 128 + 8 j + c0 + e (wgmma accumulator layout).
// Rows past m are not stored; dense: nor columns past ncols.  GROUPED: column j goes to its pair's (token, slot) row, padding nowhere.
template <bool GROUPED>
__device__ __forceinline__ void mmq_store_tile(const MmqTileArgs & a, const float (&acc)[64], int64_t mt, int64_t nt, int ra, int c0) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int64_t row = mt * MMQ_TM + ra + 8 * h;
        if (row >= a.m) continue;
#pragma unroll
        for (int j = 0; j < 16; j++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int64_t n = nt * MMQ_TN + 8 * j + c0 + e;
                if constexpr (GROUPED) {
                    const int pr = a.map.cols[n], nu = a.map.n_used;
                    if (pr >= 0) a.dst[(pr / nu) * a.map.dst_tok_stride + (pr % nu) * a.map.dst_slot_stride + row] = acc[4 * j + 2 * h + e];
                } else if (n < a.ncols) a.dst[n * a.ldd + row] = acc[4 * j + 2 * h + e];
            }
        }
    }
}

// B200_MMQ_PROF: warp's [total cycles, cycles in wait kind 0, in wait kind 1, 0]
__device__ __forceinline__ void mmq_prof_store(const MmqTileArgs & a, int warp, long long t_start, const unsigned long long & w0, const unsigned long long & w1) {
    unsigned long long * o = a.prof + warp * 4;
    o[0] = (unsigned long long)(clock64() - t_start); o[1] = w0; o[2] = w1; o[3] = 0;
}

// mmq.cu: which tile kernel takes `type` rows of length k (the format rule, and B200_MMQ_DISABLE_TC), its workspace, the call into it
bool    mmq_tile_takes(int type, int64_t m, int64_t k);
int64_t mmq_tile_workspace(int type, int64_t k, int64_t ncols);
int     mmq_tile_run(int type, const MmqJob & job, cudaStream_t st);
unsigned long long * mmq_prof_buf();
void    mmq_prof_report(const char * kernel, int type, const MmqTileArgs & a, cudaStream_t st);
// the two families (mmq_tc.cu: Q4_K / Q5_K / Q6_K, mmq_tc32.cu: Q4_0 / Q5_0 / Q8_0)
int64_t b200_mmq_tc_workspace(int64_t k, int64_t ncols);
int     b200_mmq_tc(int type, const MmqJob & job, cudaStream_t st);
int64_t b200_mmq_tc32_workspace(int64_t k, int64_t ncols);
int     b200_mmq_tc32(int type, const MmqJob & job, cudaStream_t st);

inline void mmq_tile_fill(MmqTileArgs & a, const MmqJob & j, int64_t rb) {
    a.W = (const uint8_t *)j.W; a.ws = (const uint8_t *)j.workspace; a.dst = j.dst;
    a.m = j.m; a.k = j.k; a.ncols = j.ncols; a.ldd = j.ldd; a.rb = rb; a.nt = (j.ncols + MMQ_TN - 1) / MMQ_TN;
    a.n_mtiles = (int32_t)((j.m + MMQ_TM - 1) / MMQ_TM); a.n_tiles = (int32_t)(a.n_mtiles * a.nt);
    a.prof = mmq_prof_buf();
    if (j.map) a.map = *j.map;
}

// KERN on min(SMs, n_tiles) persistent CTAs with PDL; its dynamic shared-memory limit is raised to SMEM once per device
template <auto KERN, int SMEM, typename Args> int mmq_tile_launch(const Args & a, cudaStream_t st) {
    static bool attr[64] = { false };
    int dev = 0; cudaGetDevice(&dev);
    if (!attr[dev & 63]) { B200_CUDA(cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM)); attr[dev & 63] = true; }
    const int grid = a.n_tiles < b200_sm_count() ? a.n_tiles : b200_sm_count();
    B200_CUDA(b200_launch_pdl(KERN, dim3((unsigned)grid), dim3(MMQ_THREADS), (size_t)SMEM, st, a));
    b200_count_launch();
    return B200_OK;
}
