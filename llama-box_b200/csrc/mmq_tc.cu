// mmq_tc.cu — batched MUL_MAT on K-quant weights (prefill / large ubatches) on the Hopper tensor cores (sm_90a):
// wgmma with register accumulators, TMA (cp.async.bulk) staging, warp-specialised, persistent.
//
// Replaces ggml_cuda_mul_mat_q / mul_mat_q<type,mmq_x> (ggml-cuda/mmq.cu:71-143, mmq.cuh:3047-3370: int8 mma.sync tiles
// with per-32 f32 scale FMAs in the inner loop, stream-K fixup :3373-3522) and quantize_mmq_q8_1 (quantize.cu:50-146).
// The arithmetic is the CPU ORACLE's, not ggml-cuda's: activations are quantised to q8_K exactly like
// quantize_row_q8_K_ref (ggml-quants.c:2555-2592) and the per-super-block integer sums of ggml_vec_dot_q{4,5,6}_K_q8_K
// (ggml-cpu/quants.c:550-758) are reproduced EXACTLY by the tensor cores:
//
//     dst[n][r] = sum_sb  d_w[r,sb] * d_x[n,sb] * isum[r,n,sb]  -  dmin_w[r,sb] * d_x[n,sb] * imin[r,n,sb]
//     isum = sum_j sc_j * (sum_{k in sub-block j} q_k * q8_k)          imin = sum_j m_j * bsum_j
//
//   * A operand (weights): a transform warpgroup unpacks the packed quants from shared memory into f16 INTEGERS with the
//     6-bit sub-block scale folded in, a[r][k] = sc_j * q  (<= 63*15 = 945 for Q4_K, <= 63*31 = 1953 for Q5_K: exact in f16),
//     written as K-major core matrices.  Q6_K's sc * (q - 32) reaches +-4096, which f16 holds only when even: the
//     product is split as (sc & ~1) * (q - 32)  [even, exact]  +  (sc & 1) * (q - 32)  [|.| <= 32], two K-passes into ONE
//     accumulator.  Q2_K (sc * q <= 15 * 3, a 4-bit min per 16 elements) and Q3_K ((sc - 32) * q with q in [-4, 3]: |.| <= 128, no
//     min) are read in ggml's native block layout, which decode (ext_mmv_kernel) and GET_ROWS share: 84 B / 110 B per block, so only
//     4-byte / 2-byte aligned, loaded as 32-bit words (Q3_K: from the aligned word below the block, realigned with funnel shifts).
//   * B operand (activations): q8 values as f16 integers (|q8| <= 127), pre-tiled in HBM in the exact shared-memory image so
//     that one bulk copy brings a [128 tokens x 64 k] panel.
//   * wgmma m64n128k16 f16, f32 accumulate in registers: every product and every partial sum is an integer below 2^24, so the
//     accumulation is EXACT and isum equals the oracle's int32 bit for bit.  imin is one more K = 16 MMA per super-block
//     (A = m_j as f16, B = the q8_K bsums as f16) into the same registers once isum has been folded in.
//   * the consumer warpgroups fold each super-block into f32 running sums in registers: acc += (d_w * d_x) * isum, then
//     acc -= (dmin_w * d_x) * imin — the floating-point roundings of the oracle's two products, with the difference applied
//     to the running sum in two steps (an isum and an imin accumulator do not both fit in the register file next to acc).
//
// Warp roles (384 threads, one persistent CTA per SM):
//     warps 0-3 / 4-7  consumers: tile rows 0-63 / 64-127, all 128 columns (issue the MMAs, fold, store)
//     warps 8-11       transform: thread t owns weight row t of the tile; packed blocks come straight from global memory into
//                      registers, one super-block ahead; thread 0 also issues the activation panels of each stage
//                      (cp.async.bulk, mbarrier complete_tx) as soon as the stage is free
// Shared memory (per CTA, ~150 KB): 2 A stages x 32 KB (128 rows x 128 k f16) + 2 B stages x 32 KB + the imin operands + scale rings.
// Data movement: weights are read from HBM once per 128-token tile (L2 serves the other token tiles of the same rows, which
// run on neighbouring CTAs), activations stream from L2.
#include "extfmt.cuh"
#include "mmq_tile.cuh"
#include "wgmma.cuh"

#include <cuda_fp16.h>

#define TC_STAGE_A 32768
#define TC_STAGE_B 32768

// ---- workspace geometry (the B image) ------------------------------------------------------------------------------
// per 128-token tile nt: Bq[nt][kq = k/64][chunk 0..7][n 0..127][8 f16]   (16 KB per 64-k quarter)
//                        Bm[nt][sb][chunk 0..1][n][8 f16]                  (q8_K bsums, 4 KB per super-block)
//                        D8[nt][sb][n] f32                                 (512 B per super-block)
struct TcGeom { int64_t nt, kq, nsb, off_bq, off_bm, off_d8, total; };
static TcGeom tc_geom(int64_t k, int64_t ncols) {
    TcGeom g;
    g.nt = (ncols + MMQ_TN - 1) / MMQ_TN; g.kq = k / 64; g.nsb = k / 256;
    g.off_bq = 0;
    g.off_bm = g.nt * g.kq * 16384;
    g.off_d8 = g.off_bm + g.nt * g.nsb * 4096;
    g.total  = g.off_d8 + g.nt * g.nsb * 512;
    return g;
}

// ---- activation quantisation into the B image -------------------------------------------------------------------------
// one warp per (token, super-block); exactly quantize_row_q8_K_ref: first index of the largest |x|, iscale = -127/max,
// nearest-int (RNE), MIN(127, .), d = 1/iscale, bsums per 16
// GATHER (grouped MUL_MAT_ID): column n of the image is the pair map.cols[n] of the activation x (zeros for padding); the blocks
// of column tiles past *map.ntt exit.  Each column's image is the one the dense instance writes for the same f32 column.
template <bool GATHER>
__global__ void __launch_bounds__(256) quantize_mmq_kernel(const float * __restrict__ x, int64_t x_col_stride, int64_t ncols, int64_t k_valid,
                                                          uint8_t * __restrict__ ws, TcGeom g, MmidMap map) {
    pdl_wait();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t sb = blockIdx.x;
    const int64_t n = (int64_t)blockIdx.y * 8 + warp;                // token (padded range: < nt * 128)
    const int64_t nt = n >> 7; const int nl = (int)(n & 127);
    if constexpr (GATHER) { if (nt >= *map.ntt) return; }            // the whole block: blockIdx.y / 16 is its column tile
    float v[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    mmq_load_col8<GATHER>(v, x, x_col_stride, ncols, k_valid, map, n, sb * 256 + lane * 8);
    float am = 0.0f; int ai = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { const float a = fabsf(v[j]); if (a > am) { am = a; ai = lane * 8 + j; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float am2 = __shfl_xor_sync(0xffffffffu, am, o);
        const int   ai2 = __shfl_xor_sync(0xffffffffu, ai, o);
        if (am2 > am || (am2 == am && ai2 < ai)) { am = am2; ai = ai2; }
    }
    float mine = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; j++) if ((ai & 7) == j) mine = v[j];
    const float maxv = __shfl_sync(0xffffffffu, mine, ai >> 3);
    int q[8]; int s = 0; float d = 0.0f;
    if (am != 0.0f) {
        const float iscale = __fdiv_rn(-127.0f, maxv);
#pragma unroll
        for (int j = 0; j < 8; j++) { const int t = __float2int_rn(__fmul_rn(iscale, v[j])); q[j] = t > 127 ? 127 : t; s += q[j]; }
        d = __fdiv_rn(1.0f, iscale);
    } else {
#pragma unroll
        for (int j = 0; j < 8; j++) q[j] = 0;
    }
    // 8 consecutive elements = one K-chunk of the panel; element order inside a chunk is (0,2,1,3,4,6,5,7): the order in
    // which the weight transform extracts nibbles from a 32-bit word (see unpack in the GEMM kernel)
    auto h2 = [](int a, int b) { return (uint32_t)__half_as_ushort(__int2half_rn(a)) | ((uint32_t)__half_as_ushort(__int2half_rn(b)) << 16); };
    uint4 pk; pk.x = h2(q[0], q[2]); pk.y = h2(q[1], q[3]); pk.z = h2(q[4], q[6]); pk.w = h2(q[5], q[7]);
    const int64_t kq = sb * 4 + (lane >> 3); const int c = lane & 7;
    *(uint4 *)(ws + g.off_bq + ((nt * g.kq + kq) * 8 + c) * MMQ_PANEL + nl * 16) = pk;
    s += __shfl_xor_sync(0xffffffffu, s, 1);                          // bsum of 16 elements (|.| <= 2032: exact in f16)
    if ((lane & 1) == 0) {
        const int grp = lane >> 1;
        *(__half *)(ws + g.off_bm + ((nt * g.nsb + sb) * 2 + (grp >> 3)) * MMQ_PANEL + nl * 16 + (grp & 7) * 2) = __int2half_rn(s);
    }
    if (lane == 0) *(float *)(ws + g.off_d8 + ((nt * g.nsb + sb) * 128 + nl) * 4) = d;
    pdl_trigger();
}

struct TcArgs : MmqTileArgs {
    TcGeom g;
    uint32_t lbo, sbo;          // descriptor strides (bytes): K-chunk stride / 8-row-group stride
};
// ---- per-type pipeline geometry: K-stages per super-block, whether the mins MMA runs, activation bytes per stage -------
// (the transform threads read each row's packed blocks straight from global memory, so no weight bytes live in shared memory;
// Q6_K rows are repacked [ql 128B x nb][qh 64B x nb][scales 16B x nb][d f16 x nb], see repack.cu)
template <int T> struct TcType;
template <> struct TcType<B200_TYPE_Q4_K> { static constexpr int STAGES = 2, HAS_MIN = 1, B_BYTES = 32768; };
template <> struct TcType<B200_TYPE_Q5_K> { static constexpr int STAGES = 2, HAS_MIN = 1, B_BYTES = 32768; };
template <> struct TcType<B200_TYPE_Q6_K> { static constexpr int STAGES = 4, HAS_MIN = 0, B_BYTES = 16384; };
template <> struct TcType<B200_TYPE_Q2_K> { static constexpr int STAGES = 2, HAS_MIN = 1, B_BYTES = 32768; };
template <> struct TcType<B200_TYPE_Q3_K> { static constexpr int STAGES = 2, HAS_MIN = 0, B_BYTES = 32768; };

// shared memory map
struct TcSmem {
    static constexpr int A = 0, B = A + 2 * TC_STAGE_A, AM = B + 2 * TC_STAGE_B, BM = AM + 2 * 4096;
    static constexpr int RS = BM + 2 * 4096;                 // row scales ring: 4 x 128 x float2
    static constexpr int D8 = RS + 4 * 1024;                 // d_x ring: 4 x 128 f32
    static constexpr int BAR = D8 + 4 * 512;                 // mbarriers
    static constexpr int TOTAL = BAR + 256;
};

__device__ __forceinline__ uint32_t hfma2_u(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d; asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}
__device__ __forceinline__ uint32_t hmul2_u(uint32_t a, uint32_t b) { uint32_t d; asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t hsub2_u(uint32_t a, uint32_t b) { uint32_t d; asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t h2_of_int(int v) { const uint32_t h = __half_as_ushort(__int2half_rn(v)); return h | (h << 16); }
// bytes 0, 1 (hi: 2, 3) of v, each < 1024, as an f16 pair (exact)
__device__ __forceinline__ uint32_t h2_of_bytes(uint32_t v, bool hi) { return hsub2_u(__byte_perm(v, 0u, hi ? 0x4342u : 0x4140u) | 0x64006400u, 0x64006400u); }

// 6-bit scales / mins of a q4_K / q5_K block header (ggml-quants.c:703-711), all 8 at once
__device__ __forceinline__ void k4_unpack(uint32_t y, uint32_t z, uint32_t w, uint32_t & sc03, uint32_t & sc47, uint32_t & mn03, uint32_t & mn47) {
    sc03 = y & 0x3f3f3f3fu; mn03 = z & 0x3f3f3f3fu;
    sc47 = (w & 0x0f0f0f0fu) | (((y >> 6) & 0x03030303u) << 4);
    mn47 = ((w >> 4) & 0x0f0f0f0fu) | (((z >> 6) & 0x03030303u) << 4);
}

// GROUPED (MUL_MAT_ID): column tile ct multiplies expert map.tile_expert[ct]; the tile count comes from the device (*map.ntt)
// and the epilogue scatters column j to its pair's output row (padding columns are not stored).  Everything else is the dense kernel.
template <int T, bool GROUPED>
__global__ void __launch_bounds__(MMQ_THREADS, 1) mmq_tc_kernel(const __grid_constant__ TcArgs args) {
    using TT = TcType<T>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t * bars = (uint64_t *)(smem + TcSmem::BAR);
    uint64_t * b_full = bars + 8, * a_full = bars + 10, * ab_empty = bars + 12;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    if (tid == 0) {
        for (int i = 0; i < 2; i++) { mbar_init(&b_full[i], 1); mbar_init(&a_full[i], 4); mbar_init(&ab_empty[i], 8); }
        mbar_fence_init();
    }
    __syncthreads();
    pdl_wait();

    const int nsb = args.nks;
    const auto NT = mmq_col_tiles<GROUPED>(args);
    auto n_tiles = [&]() { return GROUPED ? args.n_mtiles * (int)NT : args.n_tiles; };      // dense: read from the parameters at each use
    unsigned long long w0 = 0, w1 = 0;                               // profile: cycles in this role's kinds of waits
    const bool prof = args.prof != nullptr && blockIdx.x == 0;
    unsigned long long * pw0 = prof ? &w0 : nullptr, * pw1 = prof ? &w1 : nullptr;
    const long long t_start = clock64();

    // activation panels of one stage (+ the bsum panel and d_x with the first stage of a super-block), issued by one thread of
    // the transform warpgroup once the stage is free (cp.async.bulk, mbarrier complete_tx)
    auto load_b = [&](int64_t nt, int sb, uint32_t sbc, int s, int st) {
        const uint32_t extra = s == 0 ? (512u + (TT::HAS_MIN ? 4096u : 0u)) : 0u;
        mbar_expect_tx(&b_full[st], (uint32_t)TT::B_BYTES + extra);
        const int64_t kq0 = (int64_t)sb * 4 + (TT::STAGES == 2 ? s * 2 : s);
        const uint8_t * src = args.ws + args.g.off_bq + (nt * args.g.kq + kq0) * 16384;
        uint8_t * dstb = smem + TcSmem::B + st * TC_STAGE_B;
        for (int o = 0; o < TT::B_BYTES; o += 8192) bulk_g2s(dstb + o, src + o, 8192, &b_full[st]);
        if (s == 0) {
            if (TT::HAS_MIN) bulk_g2s(smem + TcSmem::BM + (sbc & 1) * 4096, args.ws + args.g.off_bm + (nt * nsb + sb) * 4096, 4096, &b_full[st]);
            bulk_g2s(smem + TcSmem::D8 + (sbc & 3) * 512, args.ws + args.g.off_d8 + (nt * nsb + sb) * 512, 512, &b_full[st]);
        }
    };

    if (warp >= 8) {
        // ===================== transform: packed quants -> f16 sc*q core matrices =====================
        // Thread t owns weight row t of the tile and reads its packed block of the NEXT super-block straight from global memory
        // into registers (9-14 16-byte loads, issued one super-block ahead, so HBM / L2 latency hides behind the conversion of
        // the current one).  (A first version staged the blocks through shared memory with one cp.async.bulk per row: a
        // warp-wide bulk copy is issued lane by lane through uniform registers, ~65 cycles each — 128 rows cost 8 K cycles per
        // super-block and starved everything else.)
        // (Q2_K: 21 32-bit words; Q3_K: 28, from the aligned word at or below the block start, whose offset in it is nxt_sh bytes)
        constexpr int NW = T == B200_TYPE_Q4_K ? 9 : T == B200_TYPE_Q5_K ? 11 : T == B200_TYPE_Q6_K ? 13 : T == B200_TYPE_Q2_K ? 6 : 7;
        const int t = tid - 8 * 32;                                      // weight row of the tile
        const int64_t nb = args.k / 256;
        uint32_t it = 0, sbc = 0;
        uint4 nxt[NW]; uint16_t nxt_d = 0; uint32_t nxt_sh = 0;
        auto fetch = [&](int tile, int sb) {
            const int64_t mt = tile / NT;
            const uint8_t * row = mmq_weight_row<GROUPED>(args, mt, tile - mt * NT, t);
            auto ld16b = [](const uint8_t * p) { return make_uint4(ldg_nc32(p), ldg_nc32(p + 4), ldg_nc32(p + 8), ldg_nc32(p + 12)); };
            if constexpr (T == B200_TYPE_Q2_K) {
                const uint8_t * p = row + (int64_t)sb * 84;                  // 4-byte aligned
#pragma unroll
                for (int i = 0; i < 5; i++) nxt[i] = ld16b(p + 16 * i);
                nxt[5] = make_uint4(ldg_nc32(p + 80), 0u, 0u, 0u);
            } else if constexpr (T == B200_TYPE_Q3_K) {
                const uint8_t * b = row + (int64_t)sb * 110;                 // 2-byte aligned
                nxt_sh = (uint32_t)(uintptr_t)b & 2u;
                const uint8_t * p = b - nxt_sh;
#pragma unroll
                for (int i = 0; i < 6; i++) nxt[i] = ld16b(p + 16 * i);
                // the last word: 16 bits where the block ends inside it (never reads past the block, so never past the matrix)
                nxt[6] = make_uint4(ldg_nc32(p + 96), ldg_nc32(p + 100), ldg_nc32(p + 104), nxt_sh ? ldg_nc32(p + 108) : (uint32_t)ldg_nc16(p + 108));
            } else if (T == B200_TYPE_Q6_K) {
                const uint4 * ql = (const uint4 *)(row + (int64_t)sb * 128), * qh = (const uint4 *)(row + nb * 128 + (int64_t)sb * 64);
#pragma unroll
                for (int i = 0; i < 8; i++) nxt[i] = __ldg(ql + i);
#pragma unroll
                for (int i = 0; i < 4; i++) nxt[8 + i] = __ldg(qh + i);
                nxt[12] = __ldg((const uint4 *)(row + nb * 192 + (int64_t)sb * 16));
                nxt_d = __ldg((const uint16_t *)(row + nb * 208 + (int64_t)sb * 2));
            } else {
                const uint4 * p = (const uint4 *)(row + (int64_t)sb * (T == B200_TYPE_Q4_K ? 144 : 176));
#pragma unroll
                for (int i = 0; i < NW; i++) nxt[i] = __ldg(p + i);
            }
        };
        if (blockIdx.x < n_tiles()) fetch(blockIdx.x, 0);
        for (int tile = blockIdx.x; tile < n_tiles(); tile += gridDim.x) {
            for (int sb = 0; sb < nsb; sb++, sbc++) {
                const int rs = sbc & 1;                                  // accumulator / imin-operand slot
                uint4 cur[NW]; const uint16_t cur_d = nxt_d; const uint32_t cur_sh = nxt_sh;
#pragma unroll
                for (int i = 0; i < NW; i++) cur[i] = nxt[i];
                {   // prefetch the next super-block (of this tile, or the first one of this CTA's next tile)
                    int ntile = tile, nsbi = sb + 1;
                    if (nsbi == nsb) { nsbi = 0; ntile = tile + gridDim.x; }
                    if (ntile < n_tiles()) fetch(ntile, nsbi);
                }
                float2 * rscale = (float2 *)(smem + TcSmem::RS + (sbc & 3) * 1024);
                if constexpr (T == B200_TYPE_Q2_K || T == B200_TYPE_Q3_K) {
                    // ---- Q2_K {scales[16], qs[64], d, dmin} / Q3_K {hmask[32], qs[64], scales[12], d} (ggml-quants.c dequantize_row_q2_K / _q3_K):
                    // element 128 n + 32 j + l is the 2-bit field 2 j of qs[32 n + l] (Q3_K: plus 4 x bit 4 n + j of hmask[l], minus 4); its
                    // scale (Q2_K: and min) is that of its 16-element group.  Half n is stage s = n.
                    auto raw = [&](int i) { const uint4 & v = cur[i >> 2]; return (i & 3) == 0 ? v.x : (i & 3) == 1 ? v.y : (i & 3) == 2 ? v.z : v.w; };
                    auto word = [&](int i) { return T == B200_TYPE_Q2_K ? raw(i) : __funnelshift_r(raw(i), raw(i + 1), 8 * cur_sh); };   // 32-bit word i of the block
                    constexpr int QS = T == B200_TYPE_Q2_K ? 4 : 8;               // first word of qs
                    const uint32_t sc12[3] = { word(24), word(25), word(26) };      // Q3_K: the 12 packed scale bytes (registers once inlined)
#pragma unroll
                    for (int s = 0; s < 2; s++, it++) {
                        const int st = it & 1;
                        mbar_wait_p(&ab_empty[st], ((it >> 1) & 1) ^ 1, pw1);
                        if (t == 0) load_b(tile % NT, sb, sbc, s, st);
                        uint8_t * As = smem + TcSmem::A + st * TC_STAGE_A + t * 16;
#pragma unroll
                        for (int j = 0; j < 4; j++) {                     // 32-element group j: K-chunks 4 j .. 4 j + 3 of the stage
#pragma unroll
                            for (int i = 0; i < 4; i++) {                 // l = 8 i .. 8 i + 7: qs words QS + 8 s + 2 i + u, hmask words 2 i + u
                                const int g = 8 * s + 2 * j + (i >> 1);
                                uint4 o;
                                uint32_t * po = (uint32_t *)&o;
                                if constexpr (T == B200_TYPE_Q2_K) {
                                    const int sc = (int)(word(g >> 2) >> (8 * (g & 3))) & 15;
                                    const uint32_t m = h2_of_int(sc), c = h2_of_int(-1024 * sc);
#pragma unroll
                                    for (int u = 0; u < 2; u++) {
                                        const uint32_t qw = word(QS + 8 * s + 2 * i + u);
                                        const uint32_t x0 = ((qw >> (2 * j)) & 0x00030003u) | 0x64006400u;                  // 1024 + q, elements (e, e+2)
                                        const uint32_t x1 = ((qw >> (2 * j + 8)) & 0x00030003u) | 0x64006400u;              // elements (e+1, e+3)
                                        po[2 * u] = hfma2_u(x0, m, c); po[2 * u + 1] = hfma2_u(x1, m, c);                  // exact: sc * q
                                    }
                                } else {
                                    const uint32_t m = h2_of_int(xf_q3k_scale((const uint8_t *)sc12, g));
#pragma unroll
                                    for (int u = 0; u < 2; u++) {
                                        const uint32_t qw = word(QS + 8 * s + 2 * i + u), hw = word(2 * i + u);
                                        const uint32_t x0 = ((qw >> (2 * j)) & 0x00030003u) | (((hw >> (4 * s + j)) & 0x00010001u) << 2) | 0x64006400u;
                                        const uint32_t x1 = ((qw >> (2 * j + 8)) & 0x00030003u) | (((hw >> (4 * s + j + 8)) & 0x00010001u) << 2) | 0x64006400u;
                                        // (1024 + q2 + 4 h) - 1028 = q in [-4, 3], then (sc - 32) * q: both exact (|.| <= 128)
                                        po[2 * u] = hmul2_u(hsub2_u(x0, 0x64046404u), m); po[2 * u + 1] = hmul2_u(hsub2_u(x1, 0x64046404u), m);
                                    }
                                }
                                *(uint4 *)(As + (4 * j + i) * MMQ_PANEL) = o;
                            }
                        }
                        if (s == 0) {
                            if constexpr (T == B200_TYPE_Q2_K) {
                                // imin operand: m_0 .. m_15 in natural order, the order of the quantiser's bsum panel; d, dmin for the epilogue
                                uint8_t * Am = smem + TcSmem::AM + rs * 4096 + t * 16;
                                uint32_t mn[4];
#pragma unroll
                                for (int w = 0; w < 4; w++) mn[w] = (word(w) >> 4) & 0x0F0F0F0Fu;
                                *(uint4 *)Am = make_uint4(h2_of_bytes(mn[0], false), h2_of_bytes(mn[0], true), h2_of_bytes(mn[1], false), h2_of_bytes(mn[1], true));
                                *(uint4 *)(Am + MMQ_PANEL) = make_uint4(h2_of_bytes(mn[2], false), h2_of_bytes(mn[2], true), h2_of_bytes(mn[3], false), h2_of_bytes(mn[3], true));
                                rscale[t] = make_float2(h2f((uint16_t)(word(20) & 0xffff)), h2f((uint16_t)(word(20) >> 16)));
                            } else {
                                rscale[t] = make_float2(h2f((uint16_t)(raw(27) >> (8 * cur_sh))), 0.0f);
                            }
                        }
                        fence_async_smem();
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&a_full[st]);
                    }
                } else if (T == B200_TYPE_Q4_K || T == B200_TYPE_Q5_K) {
                    constexpr int QW = T == B200_TYPE_Q4_K ? 1 : 3;       // first 16-byte word of qs
                    const uint4 hdr = cur[0];
                    uint32_t sc03, sc47, mn03, mn47;
                    k4_unpack(hdr.y, hdr.z, hdr.w, sc03, sc47, mn03, mn47);
                    uint32_t qhw[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
                    if (T == B200_TYPE_Q5_K) { qhw[0] = cur[1].x; qhw[1] = cur[1].y; qhw[2] = cur[1].z; qhw[3] = cur[1].w; qhw[4] = cur[2].x; qhw[5] = cur[2].y; qhw[6] = cur[2].z; qhw[7] = cur[2].w; }
#pragma unroll
                    for (int s = 0; s < 2; s++, it++) {                   // half super-block = 128 k = one stage
                        const int st = it & 1;
                        mbar_wait_p(&ab_empty[st], ((it >> 1) & 1) ^ 1, pw1);
                        if (t == 0) load_b(tile % NT, sb, sbc, s, st);
                        uint8_t * As = smem + TcSmem::A + st * TC_STAGE_A + t * 16;
#pragma unroll
                        for (int gg = 0; gg < 2; gg++) {
                            const int grp = 2 * s + gg;                   // 64-element group: low nibbles = sub-block 2grp, high = 2grp + 1
                            const uint32_t scw = grp < 2 ? sc03 : sc47;
                            const int sc_lo = (scw >> (16 * (grp & 1))) & 63, sc_hi = (scw >> (16 * (grp & 1) + 8)) & 63;
                            const uint32_t m_lo = h2_of_int(sc_lo), m_hi = h2_of_int(sc_hi);
                            const uint32_t c_lo = h2_of_int(-1024 * sc_lo), c_hi = h2_of_int(-64 * sc_hi);
                            const uint4 qa = cur[QW + grp * 2], qb = cur[QW + grp * 2 + 1];
                            const uint32_t w[8] = { qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w };
#pragma unroll
                            for (int i = 0; i < 4; i++) {
                                uint4 lo, hi;
                                uint32_t * plo = (uint32_t *)&lo, * phi = (uint32_t *)&hi;
#pragma unroll
                                for (int u = 0; u < 2; u++) {
                                    const uint32_t ww = w[2 * i + u];
                                    uint32_t l0 = (ww & 0x000F000Fu) | 0x64006400u, l1 = ((ww >> 8) & 0x000F000Fu) | 0x64006400u;      // 1024 + q  (elements e, e+2 | e+1, e+3)
                                    uint32_t h0 = (ww & 0x00F000F0u) | 0x54005400u, h1 = ((ww >> 8) & 0x00F000F0u) | 0x54005400u;      // 64 + q    (high nibbles, elements + 32)
                                    if (T == B200_TYPE_Q5_K) {                                                                         // fifth bit: bit (sub-block) of qh[l]
                                        const uint32_t hw = qhw[2 * i + u];
                                        l0 |= ((hw >> (2 * grp)) & 0x00010001u) << 4;      l1 |= ((hw >> (2 * grp + 8)) & 0x00010001u) << 4;
                                        h0 |= ((hw >> (2 * grp + 1)) & 0x00010001u) << 8;  h1 |= ((hw >> (2 * grp + 9)) & 0x00010001u) << 8;
                                    }
                                    plo[2 * u] = hfma2_u(l0, m_lo, c_lo); plo[2 * u + 1] = hfma2_u(l1, m_lo, c_lo);     // exact: sc * q
                                    phi[2 * u] = hfma2_u(h0, m_hi, c_hi); phi[2 * u + 1] = hfma2_u(h1, m_hi, c_hi);
                                }
                                *(uint4 *)(As + (gg * 8 + i) * MMQ_PANEL) = lo;
                                *(uint4 *)(As + (gg * 8 + 4 + i) * MMQ_PANEL) = hi;
                            }
                        }
                        if (s == 0) {
                            // imin operand: m_j duplicated for its two 16-element halves; d, dmin for the epilogue
                            uint8_t * Am = smem + TcSmem::AM + rs * 4096 + t * 16;
                            uint4 m0, m1;
                            m0.x = h2_of_int(mn03 & 63); m0.y = h2_of_int((mn03 >> 8) & 63); m0.z = h2_of_int((mn03 >> 16) & 63); m0.w = h2_of_int((mn03 >> 24) & 63);
                            m1.x = h2_of_int(mn47 & 63); m1.y = h2_of_int((mn47 >> 8) & 63); m1.z = h2_of_int((mn47 >> 16) & 63); m1.w = h2_of_int((mn47 >> 24) & 63);
                            *(uint4 *)Am = m0; *(uint4 *)(Am + MMQ_PANEL) = m1;
                            rscale[t] = make_float2(h2f((uint16_t)(hdr.x & 0xffff)), h2f((uint16_t)(hdr.x >> 16)));
                        }
                        fence_async_smem();                               // generic-proxy writes -> visible to the tensor core (async proxy)
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&a_full[st]);
                    }
                } else {
                    // ---- Q6_K: q = ql | qh << 4 (0..63), value sc * (q - 32), scales int8 per 16 elements (ggml-quants.c dequantize_row_q6_K)
                    const uint32_t scw[4] = { cur[12].x, cur[12].y, cur[12].z, cur[12].w };
#pragma unroll
                    for (int s = 0; s < 4; s++, it++) {                   // quarter super-block = 64 k: chunks 0-7 = even-scale part, 8-15 = odd-scale part
                        const int st = it & 1;
                        mbar_wait_p(&ab_empty[st], ((it >> 1) & 1) ^ 1, pw1);
                        if (t == 0) load_b(tile % NT, sb, sbc, s, st);
                        uint8_t * As = smem + TcSmem::A + st * TC_STAGE_A + t * 16;
                        const int hh = s >> 1, u2 = s & 1;
                        const uint4 qha = cur[8 + hh * 2], qhb = cur[8 + hh * 2 + 1];
                        const uint32_t qhw[8] = { qha.x, qha.y, qha.z, qha.w, qhb.x, qhb.y, qhb.z, qhb.w };
#pragma unroll
                        for (int tt = 0; tt < 2; tt++) {
                            const int tg = 2 * u2 + tt;                   // 32-element group of the half: elements 128 hh + 32 tg + l
                            const uint4 qa = cur[hh * 4 + (tg & 1) * 2], qb = cur[hh * 4 + (tg & 1) * 2 + 1];
                            const uint32_t w[8] = { qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w };
                            const int nsh = 4 * (tg >> 1), hsh = 2 * tg;
#pragma unroll
                            for (int i = 0; i < 4; i++) {
                                const int sidx = 8 * hh + 2 * tg + (i >> 1);                          // scale of elements 8i .. 8i+7 of the group
                                const int sc = (int)(int8_t)((scw[sidx >> 2] >> (8 * (sidx & 3))) & 0xff);
                                const int sce = sc & ~1;
                                const uint32_t m_e = h2_of_int(sce), m_o = h2_of_int(sc - sce);
                                uint4 ev, od;
                                uint32_t * pe = (uint32_t *)&ev, * po = (uint32_t *)&od;
#pragma unroll
                                for (int u = 0; u < 2; u++) {
                                    const uint32_t q4 = ((w[2 * i + u] >> nsh) & 0x0F0F0F0Fu) | (((qhw[2 * i + u] >> hsh) & 0x03030303u) << 4);
                                    const uint32_t x0 = hsub2_u((q4 & 0x00FF00FFu) | 0x64006400u, 0x64206420u);       // (1024 + q) - 1056 = q - 32, elements (e, e+2)
                                    const uint32_t x1 = hsub2_u(((q4 >> 8) & 0x00FF00FFu) | 0x64006400u, 0x64206420u); // elements (e+1, e+3)
                                    pe[2 * u] = hmul2_u(x0, m_e); pe[2 * u + 1] = hmul2_u(x1, m_e);                  // even scale part: exact (even integers <= 4096)
                                    po[2 * u] = hmul2_u(x0, m_o); po[2 * u + 1] = hmul2_u(x1, m_o);
                                }
                                *(uint4 *)(As + (tt * 4 + i) * MMQ_PANEL) = ev;
                                *(uint4 *)(As + (8 + tt * 4 + i) * MMQ_PANEL) = od;
                            }
                        }
                        if (s == 0) rscale[t] = make_float2(h2f(cur_d), 0.0f);
                        fence_async_smem();
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&a_full[st]);
                    }
                }
            }
        }
    } else {
        // ===================== consumers: MMAs of rows 64 g .. 64 g + 63, fold into f32 running sums, store =====================
        const int g = warp >> 2;
        const int ra = 64 * g + 16 * (warp & 3) + (lane >> 2);          // tile rows ra, ra + 8 (wgmma accumulator layout, wgmma.cuh)
        const int c0 = 2 * (lane & 3);                                  // tile columns 8 j + c0 + {0, 1}
        const uint64_t dmin_a = wg_desc(smem_u32(smem + TcSmem::AM + g * 1024), args.lbo, args.sbo);
        uint32_t it = 0, sbc = 0;
        for (int tile = blockIdx.x; tile < n_tiles(); tile += gridDim.x) {
            const int64_t mt = tile / NT, nt = tile % NT;
            float acc[64], frag[64];
#pragma unroll
            for (int c = 0; c < 64; c++) acc[c] = 0.0f;
            for (int sb = 0; sb < nsb; sb++, sbc++) {
                const int rs = sbc & 1;
                for (int s = 0; s < TT::STAGES; s++, it++) {
                    const int st = it & 1; const uint32_t ph = (it >> 1) & 1;
                    mbar_wait_p(&b_full[st], ph, pw0);
                    mbar_wait_p(&a_full[st], ph, pw1);
                    const uint32_t a0 = smem_u32(smem + TcSmem::A + st * TC_STAGE_A) + g * 1024, b0 = smem_u32(smem + TcSmem::B + st * TC_STAGE_B);
                    wg_fence();
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const uint32_t bj = TT::STAGES == 2 ? j : (j & 3);        // Q6_K: the even and the odd-scale pass read the same 64-k panel
                        wg_mma_ss(frag, wg_desc(a0 + j * 2 * MMQ_PANEL, args.lbo, args.sbo), wg_desc(b0 + bj * 2 * MMQ_PANEL, args.lbo, args.sbo), (s | j) ? 1u : 0u);
                    }
                    wg_commit();
                    wg_wait0();
                    wg_pin(frag);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&ab_empty[st]);                  // stage buffers reusable
                }
                // the scale rings (4 deep) and the imin operands (2 deep) of this super-block stay valid until this warpgroup has
                // released the stages of super-block sb + 1, which it does only after this fold
                const float2 * rsc = (const float2 *)(smem + TcSmem::RS + (sbc & 3) * 1024);
                const float2 da = rsc[ra], db = rsc[ra + 8];
                const float * d8 = (const float *)(smem + TcSmem::D8 + (sbc & 3) * 512);
#pragma unroll
                for (int j = 0; j < 16; j++) {
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const float dx = d8[8 * j + c0 + e];
                        acc[4 * j + e]     = __fadd_rn(acc[4 * j + e],     __fmul_rn(__fmul_rn(da.x, dx), frag[4 * j + e]));       // d * isum (ggml-cpu/quants.c:615-620)
                        acc[4 * j + 2 + e] = __fadd_rn(acc[4 * j + 2 + e], __fmul_rn(__fmul_rn(db.x, dx), frag[4 * j + 2 + e]));
                    }
                }
                if (TT::HAS_MIN) {
                    wg_fence();
                    wg_mma_ss(frag, dmin_a + ((uint64_t)(rs * 4096) >> 4), wg_desc(smem_u32(smem + TcSmem::BM + rs * 4096), args.lbo, args.sbo), 0u);
                    wg_commit();
                    wg_wait0();
                    wg_pin(frag);
#pragma unroll
                    for (int j = 0; j < 16; j++) {
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const float dx = d8[8 * j + c0 + e];
                            acc[4 * j + e]     = __fsub_rn(acc[4 * j + e],     __fmul_rn(__fmul_rn(da.y, dx), frag[4 * j + e]));   // - dmin * imin
                            acc[4 * j + 2 + e] = __fsub_rn(acc[4 * j + 2 + e], __fmul_rn(__fmul_rn(db.y, dx), frag[4 * j + 2 + e]));
                        }
                    }
                }
            }
            mmq_store_tile<GROUPED>(args, acc, mt, nt, ra, c0);
        }
    }

    if (prof && lane == 0) mmq_prof_store(args, warp, t_start, w0, w1);
    pdl_trigger();
}

// ---- host ----------------------------------------------------------------------------------------------------------
int64_t b200_mmq_tc_workspace(int64_t k, int64_t ncols) { return tc_geom(k, ncols).total; }

template <bool GROUPED> static int tc_launch(int type, const TcArgs & a, cudaStream_t st) {
    switch (type) {
        case B200_TYPE_Q4_K: return mmq_tile_launch<mmq_tc_kernel<B200_TYPE_Q4_K, GROUPED>, TcSmem::TOTAL>(a, st);
        case B200_TYPE_Q5_K: return mmq_tile_launch<mmq_tc_kernel<B200_TYPE_Q5_K, GROUPED>, TcSmem::TOTAL>(a, st);
        case B200_TYPE_Q6_K: return mmq_tile_launch<mmq_tc_kernel<B200_TYPE_Q6_K, GROUPED>, TcSmem::TOTAL>(a, st);
        // dense only: MUL_MAT_ID on these formats stays on the matvec (mmid_route.cu)
        case B200_TYPE_Q2_K: if constexpr (!GROUPED) return mmq_tile_launch<mmq_tc_kernel<B200_TYPE_Q2_K, false>, TcSmem::TOTAL>(a, st); break;
        case B200_TYPE_Q3_K: if constexpr (!GROUPED) return mmq_tile_launch<mmq_tc_kernel<B200_TYPE_Q3_K, false>, TcSmem::TOTAL>(a, st); break;
    }
    return B200_ERR_UNSUPPORTED;
}

int b200_mmq_tc(int type, const MmqJob & j, cudaStream_t st) {
    TcArgs a = {};
    mmq_tile_fill(a, j, (j.k / 256) * xf_block_bytes(type));          // Q6_K's repacked rows are as long as its native ones
    a.g = tc_geom(j.k, j.ncols);
    a.nks = (int32_t)(j.k / 256);
    a.lbo = (uint32_t)MMQ_PANEL; a.sbo = 128u;
    B200_CUDA(b200_launch_pdl(j.map ? quantize_mmq_kernel<true> : quantize_mmq_kernel<false>, dim3((unsigned)a.nks, (unsigned)(a.nt * 16)), dim3(256), 0, st,
                              j.X, j.x_col_stride, j.ncols, j.k_valid, (uint8_t *)j.workspace, a.g, a.map));
    b200_count_launch();
    const int rc = j.map ? tc_launch<true>(type, a, st) : tc_launch<false>(type, a, st);
    if (a.prof && rc == B200_OK) mmq_prof_report(j.map ? "mmq_tc grouped" : "mmq_tc", type, a, st);
    return rc;
}
