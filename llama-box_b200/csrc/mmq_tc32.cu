// mmq_tc32.cu — batched MUL_MAT on Q4_0 / Q5_0 / Q8_0 weights (prefill / large ubatches) on the Hopper tensor cores (sm_90a):
// int8 wgmma (SASS: IGMMA) with s32 register accumulators, TMA (cp.async.bulk) staging, warp-specialised, persistent.
// The sibling of mmq_tc.cu (K-quants) for the formats whose scale is an f16 per 32 elements on BOTH operands.
//
// The arithmetic is the CPU ORACLE's (oracle.c dot_q4_0 / dot_q5_0 / dot_q8_0), as in the matvec (mmvq.cu): activations are
// quantised to q8_0 exactly like b200_quantize_act2(kind 1) (d = max / 127 -> f16, id = 127 / max, RNE), the integer sum of each
// 32-element block is exact, and each block is folded into an f32 running sum with the oracle's products and roundings:
//
//     Q4_0:          acc += ((float)s * d_w) * d_x          Q5_0 / Q8_0:   acc += (float)s * (d_w * d_x)
//
// Every output has one running sum and its blocks are added in the oracle's order (block 0 first), so the result does not depend
// on the tile schedule; the matvec (column groups) splits a row over lanes and differs from this in the f32 summation order only.
//
// Why int8 wgmma and not the f16-integer trick of mmq_tc.cu: with a scale per 32 elements on both sides nothing can be folded
// into an operand, so the accumulator has to be read out after EVERY block.  One m64nNk32.s32.s8.s8 instruction is exactly one
// block and its s32 result is exact by construction; the f16 route needs two k16 instructions and twice the shared-memory bytes
// for the same block.  For Q8_0 the repacked row's qs run already is the A operand (the transform only places it); Q4_0 / Q5_0
// expand nibbles (+ the qh bit) to int8 with the -8 / -16 offset applied, in natural element order (low nibbles = elements
// 0..15 = the first 16-byte K-chunk of the block, high nibbles = the second), so the activation image needs no permutation.
//
// What limits it: the fold, not the tensor pipe.  Per block a consumer thread converts and scales 64 accumulators (convert, two
// multiplies, add = 4 issue slots each) against 64 cycles of IGMMA per warpgroup, so the issue slots of the two consumer
// warpgroups bound the kernel well below the int8 rate (counted: about a quarter; measured: a tenth, H100.md).  To keep the tensor pipe and the fold overlapped each
// warpgroup splits its 128 columns in two m64n64k32 halves with an accumulator set each: while one half is folded the other
// half's (or the next block's) MMA runs.  Registers: 64 f32 sums + 2 x 32 s32 accumulators, no setmaxnreg needed.
//
// Warp roles (384 threads, one persistent CTA per SM), as in mmq_tc.cu:
//     warps 0-3 / 4-7  consumers: tile rows 0-63 / 64-127, all 128 columns
//     warps 8-11       transform: thread t owns weight row t of the tile, reads its packed blocks one stage ahead from global
//                      memory into registers; thread 0 also issues the activation panel of each stage (cp.async.bulk)
// A stage is 128 k (4 blocks): A 16 KB (int8 core matrices) + B 16 KB + d_x 2 KB + d_w 2 KB; 4 stages, ~144 KB of shared memory.
//
// IQ4_NL / IQ4_XS (the wide path's non-linear 4-bit formats, dense MUL_MAT only) are read in ggml's native block layout; the transform
// looks each nibble up in kvalues_iq4nl (int8 in [-127, 113]) and places it like Q4_0 (mmq_wide32.cuh), so one IGMMA is still one
// block's exact integer sum.  IQ4_NL has q8_0 activations and folds like Q8_0; IQ4_XS has q8_K activations (one f32 d_x per 256
// elements, written to the image for each block, not f16-rounded) and a 6-bit scale per block, folded as the oracle does:
//
//     IQ4_XS:        acc += ((d_w * d_x) * (float)(ls - 32)) * (float)s
#include "mmq_tile.cuh"
#include "mmq_wide32.cuh"
#include "wgmma.cuh"

#define T32_KS 128                  // k per stage
#define T32_NSTAGE 4
#define T32_STAGE_A (8 * MMQ_PANEL)
#define T32_STAGE_B (8 * MMQ_PANEL + 4 * 512)      // the panel + d_x of its 4 blocks

// ---- workspace geometry (the activation image) --------------------------------------------------------------------------
// per 128-token tile nt and 128-k stage ks, contiguous so that one stage is one run of bytes:
//     Q[nt][ks][chunk 0..7][n 0..127][16 int8]      element e of block b of the stage: chunk 2 b + e / 16, byte e % 16
//     D[nt][ks][block 0..3][n 0..127] f32           d_x
struct Tc32Geom { int64_t nt, ns, total; };
static Tc32Geom tc32_geom(int64_t k, int64_t ncols) {
    Tc32Geom g;
    g.nt = (ncols + MMQ_TN - 1) / MMQ_TN; g.ns = k / T32_KS;
    g.total = g.nt * g.ns * T32_STAGE_B;
    return g;
}

// ---- activation quantisation into the image ------------------------------------------------------------------------------
// one warp per (token, 256 elements), 4 lanes per q8_0 block: the arithmetic of warp_quant_q80 (actquant.cuh).  Elements from
// k_valid up (padded weight rows) and tokens from ncols up are zeros with d = 0.
// GATHER (grouped MUL_MAT_ID): column n of the image is the pair map.cols[n] of x (zeros for padding); the blocks of column
// tiles past *map.ntt exit.  Each column's image is the one the dense instance writes for the same f32 column.
template <bool GATHER>
__global__ void __launch_bounds__(256) quantize_mmq32_kernel(const float * __restrict__ x, int64_t x_col_stride, int64_t ncols, int64_t k_valid,
                                                            uint8_t * __restrict__ ws, Tc32Geom g, MmidMap map) {
    pdl_wait();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t blk = blockIdx.x;
    const int64_t n = (int64_t)blockIdx.y * 8 + warp;                // token (padded range: < nt * 128)
    const int64_t nt = n >> 7; const int nl = (int)(n & 127);
    if constexpr (GATHER) { if (nt >= *map.ntt) return; }            // the whole block: blockIdx.y / 16 is its column tile
    float v[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    mmq_load_col8<GATHER>(v, x, x_col_stride, ncols, k_valid, map, n, blk * 256 + lane * 8);
    float am = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; j++) am = fmaxf(am, fabsf(v[j]));
    am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 1));
    am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 2));
    const float d  = __fdiv_rn(am, 127.0f);
    const float id = am != 0.0f ? __fdiv_rn(127.0f, am) : 0.0f;
    int q[8];
#pragma unroll
    for (int j = 0; j < 8; j++) q[j] = __float2int_rn(__fmul_rn(v[j], id));
    uint2 pk;
    pk.x = (q[0] & 0xff) | ((q[1] & 0xff) << 8) | ((q[2] & 0xff) << 16) | ((q[3] & 0xff) << 24);
    pk.y = (q[4] & 0xff) | ((q[5] & 0xff) << 8) | ((q[6] & 0xff) << 16) | ((q[7] & 0xff) << 24);
    uint8_t * stage = ws + ((nt * g.ns + blk * 2 + (lane >> 4)) * T32_STAGE_B);
    const int b = (lane >> 2) & 3;                                   // block of the stage
    *(uint2 *)(stage + (2 * b + ((lane & 3) >> 1)) * MMQ_PANEL + nl * 16 + (lane & 1) * 8) = pk;
    if ((lane & 3) == 0) *(float *)(stage + 8 * MMQ_PANEL + (b * 128 + nl) * 4) = __half2float(__float2half_rn(d));   // the oracle stores d as f16
    pdl_trigger();
}

// IQ4_XS: the same image from q8_K activations (quantize_row_q8_K_ref, as quantize_mmq_kernel of mmq_tc.cu does it), one warp per
// (token, super-block); d_x is the super-block's f32 d, written for each of the 4 blocks of both its stages.  Dense only.
__global__ void __launch_bounds__(256) quantize_mmq32k_kernel(const float * __restrict__ x, int64_t x_col_stride, int64_t ncols, int64_t k_valid,
                                                             uint8_t * __restrict__ ws, Tc32Geom g) {
    pdl_wait();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t sb = blockIdx.x;
    const int64_t n = (int64_t)blockIdx.y * 8 + warp;                // token (padded range: < nt * 128)
    const int64_t nt = n >> 7; const int nl = (int)(n & 127);
    float v[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    const MmidMap none = {};
    mmq_load_col8<false>(v, x, x_col_stride, ncols, k_valid, none, n, sb * 256 + lane * 8);
    float am = 0.0f; int ai = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { const float a = fabsf(v[j]); if (a > am) { am = a; ai = lane * 8 + j; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {                               // the first index of the largest |x|
        const float am2 = __shfl_xor_sync(0xffffffffu, am, o);
        const int   ai2 = __shfl_xor_sync(0xffffffffu, ai, o);
        if (am2 > am || (am2 == am && ai2 < ai)) { am = am2; ai = ai2; }
    }
    float mine = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; j++) if ((ai & 7) == j) mine = v[j];
    const float maxv = __shfl_sync(0xffffffffu, mine, ai >> 3);
    uint2 pk;
    const float d = w32_q8k_quant8(v, maxv, am, pk.x, pk.y);
    uint8_t * stage = ws + ((nt * g.ns + sb * 2 + (lane >> 4)) * T32_STAGE_B);
    const int b = (lane >> 2) & 3;                                   // block of the stage
    *(uint2 *)(stage + (2 * b + ((lane & 3) >> 1)) * MMQ_PANEL + nl * 16 + (lane & 1) * 8) = pk;
    if ((lane & 3) == 0) *(float *)(stage + 8 * MMQ_PANEL + (b * 128 + nl) * 4) = d;
    pdl_trigger();
}

using Tc32Args = MmqTileArgs;       // W: repacked rows (repack_layout.cuh), k a multiple of 256 (padded rows included); nks: 128-k stages

struct Tc32Smem {
    static constexpr int A = 0, B = A + T32_NSTAGE * T32_STAGE_A;
    static constexpr int RS = B + T32_NSTAGE * T32_STAGE_B;          // d_w ring: stage x block x 128 rows f32
    static constexpr int BAR = RS + T32_NSTAGE * 2048;
    static constexpr int TOTAL = BAR + 128;
};

__device__ __forceinline__ uint32_t bit4_of(uint32_t b) { return (((b & 0xFu) * 0x00204081u) & 0x01010101u) << 4; }   // 4 bits -> bit 4 of 4 bytes
// bytes v in [0, 2 OFF) -> v - OFF as int8, four at a time (no borrow crosses a byte: 0x80 + v - OFF >= 0x70)
template <uint32_t OFF> __device__ __forceinline__ uint32_t recentre(uint32_t v) { return ((v | 0x80808080u) - OFF * 0x01010101u) ^ 0x80808080u; }

// GROUPED (MUL_MAT_ID): column tile ct multiplies expert map.tile_expert[ct]; the tile count comes from the device (*map.ntt)
// and the epilogue scatters column j to its pair's output row (padding columns are not stored).  Everything else is the dense kernel.
template <int T, bool GROUPED>
__global__ void __launch_bounds__(MMQ_THREADS, 1) mmq_tc32_kernel(const __grid_constant__ Tc32Args args) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t * b_full = (uint64_t *)(smem + Tc32Smem::BAR), * a_full = b_full + T32_NSTAGE, * ab_empty = a_full + T32_NSTAGE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    if (tid == 0) {
        for (int i = 0; i < T32_NSTAGE; i++) { mbar_init(&b_full[i], 1); mbar_init(&a_full[i], 4); mbar_init(&ab_empty[i], 8); }
        mbar_fence_init();
    }
    __syncthreads();
    pdl_wait();

    const int ns = args.nks;
    const auto NT = mmq_col_tiles<GROUPED>(args);
    const int n_tiles = GROUPED ? args.n_mtiles * (int)NT : args.n_tiles;
    unsigned long long w0 = 0, w1 = 0;                               // profile: cycles in this role's kinds of waits
    const bool prof = args.prof != nullptr && blockIdx.x == 0;
    unsigned long long * pw0 = prof ? &w0 : nullptr, * pw1 = prof ? &w1 : nullptr;
    const long long t_start = clock64();

    if (warp >= 8) {
        // ===================== transform: packed blocks -> int8 core matrices + d_w =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 88;");
        constexpr bool IQ4 = T == B200_TYPE_IQ4_NL || T == B200_TYPE_IQ4_XS;  // native blocks, one stage as 9 aligned 8-byte words (mmq_wide32.cuh)
        constexpr int NQ = T == B200_TYPE_Q8_0 ? 8 : 4;                  // 16-byte words of qs per row and stage
        constexpr int QB = T == B200_TYPE_Q8_0 ? 32 : 16;                // qs bytes per block
        const int t = tid - 8 * 32;                                      // weight row of the tile
        const int64_t nb = args.k / 32;
        uint32_t it = 0;
        uint4 nxt[NQ], nxt_h = make_uint4(0, 0, 0, 0); uint2 nxt_d;
        uint32_t nxt_w[18];
        auto fetch = [&](int tile, int s) {
            const uint8_t * row = mmq_weight_row<GROUPED>(args, tile / NT, tile % NT, t);
            if constexpr (IQ4) {
                w32_load<T>(row, s, nxt_w);
            } else {
                const uint4 * p = (const uint4 *)(row + (int64_t)s * 4 * QB);
#pragma unroll
                for (int i = 0; i < NQ; i++) nxt[i] = __ldg(p + i);
                if (T == B200_TYPE_Q5_0) nxt_h = __ldg((const uint4 *)(row + nb * 16 + (int64_t)s * 16));
                nxt_d = __ldg((const uint2 *)(row + nb * (T == B200_TYPE_Q5_0 ? 20 : QB) + (int64_t)s * 8));
            }
        };
        if (blockIdx.x < n_tiles) fetch(blockIdx.x, 0);
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            for (int s = 0; s < ns; s++, it++) {
                uint4 cur[NQ]; const uint4 cur_h = nxt_h; const uint2 cur_d = nxt_d;
#pragma unroll
                for (int i = 0; i < NQ; i++) cur[i] = nxt[i];
                uint32_t cur_w[18];
                if constexpr (IQ4) {
#pragma unroll
                    for (int i = 0; i < 18; i++) cur_w[i] = nxt_w[i];
                }
                {   // prefetch the next stage (of this tile, or the first one of this CTA's next tile)
                    int ntile = tile, nsi = s + 1;
                    if (nsi == ns) { nsi = 0; ntile = tile + gridDim.x; }
                    if (ntile < n_tiles) fetch(ntile, nsi);
                }
                const int st = it % T32_NSTAGE;
                mbar_wait_p(&ab_empty[st], ((it / T32_NSTAGE) & 1) ^ 1, pw1);
                if (t == 0) {
                    mbar_expect_tx(&b_full[st], (uint32_t)T32_STAGE_B);
                    const uint8_t * src = args.ws + (((int64_t)(tile % NT) * ns + s) * T32_STAGE_B);
                    for (int o = 0; o < T32_STAGE_B; o += T32_STAGE_B / 3) bulk_g2s(smem + Tc32Smem::B + st * T32_STAGE_B + o, src + o, T32_STAGE_B / 3, &b_full[st]);
                }
                uint8_t * As = smem + Tc32Smem::A + st * T32_STAGE_A + t * 16;
                if constexpr (IQ4) {
                    float * rs = (float *)(smem + Tc32Smem::RS + st * 2048) + t;
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        uint32_t q[8];
                        const uint32_t sc = w32_unpack<T>(cur_w, s, b, q);
                        *(uint4 *)(As + (2 * b) * MMQ_PANEL) = make_uint4(q[0], q[1], q[2], q[3]);         // elements 0..15: low nibbles
                        *(uint4 *)(As + (2 * b + 1) * MMQ_PANEL) = make_uint4(q[4], q[5], q[6], q[7]);     // elements 16..31: high nibbles
                        if (T == B200_TYPE_IQ4_NL) rs[128 * b] = h2f((uint16_t)sc);
                        else ((uint32_t *)rs)[128 * b] = sc;                                               // d_w bits | (ls - 32) << 16
                    }
                } else if (T == B200_TYPE_Q8_0) {
#pragma unroll
                    for (int c = 0; c < 8; c++) *(uint4 *)(As + c * MMQ_PANEL) = cur[c];
                } else {
                    const uint32_t qh[4] = { cur_h.x, cur_h.y, cur_h.z, cur_h.w };
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const uint32_t w[4] = { cur[b].x, cur[b].y, cur[b].z, cur[b].w };
                        uint4 lo, hi;
                        uint32_t * plo = (uint32_t *)&lo, * phi = (uint32_t *)&hi;
#pragma unroll
                        for (int i = 0; i < 4; i++) {
                            const uint32_t l = w[i] & 0x0F0F0F0Fu, h = (w[i] >> 4) & 0x0F0F0F0Fu;
                            if (T == B200_TYPE_Q4_0) { plo[i] = recentre<8>(l); phi[i] = recentre<8>(h); }
                            else { plo[i] = recentre<16>(l | bit4_of(qh[b] >> (4 * i))); phi[i] = recentre<16>(h | bit4_of(qh[b] >> (16 + 4 * i))); }   // qh bit j -> element j
                        }
                        *(uint4 *)(As + (2 * b) * MMQ_PANEL) = lo;              // elements 0..15: low nibbles
                        *(uint4 *)(As + (2 * b + 1) * MMQ_PANEL) = hi;          // elements 16..31: high nibbles
                    }
                }
                if constexpr (!IQ4) {
                    float * rs = (float *)(smem + Tc32Smem::RS + st * 2048) + t;
                    rs[0]   = h2f((uint16_t)(cur_d.x & 0xffff)); rs[128] = h2f((uint16_t)(cur_d.x >> 16));
                    rs[256] = h2f((uint16_t)(cur_d.y & 0xffff)); rs[384] = h2f((uint16_t)(cur_d.y >> 16));
                }
                fence_async_smem();                                       // generic-proxy writes -> visible to the tensor core (async proxy)
                __syncwarp();
                if (lane == 0) mbar_arrive(&a_full[st]);
            }
        }
    } else {
        // ===================== consumers: one IGMMA per (block, column half), fold into f32 running sums, store =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 208;");           // 2 x 128 x 208 + 128 x 88 = the 384 x 168 the CTA was launched with
        const int g = warp >> 2;
        const int ra = 64 * g + 16 * (warp & 3) + (lane >> 2);          // tile rows ra, ra + 8 (wgmma accumulator layout, wgmma.cuh)
        const int c0 = 2 * (lane & 3);                                  // tile columns 8 j + c0 + {0, 1}
        uint32_t it = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int64_t mt = tile / NT, nt = tile % NT;
            float acc[64];
            int32_t f0[32], f1[32];                                      // accumulators of column halves 0-63 / 64-127
#pragma unroll
            for (int c = 0; c < 64; c++) acc[c] = 0.0f;
#pragma unroll
            for (int c = 0; c < 32; c++) { f0[c] = 0; f1[c] = 0; }
            auto mma = [&](int32_t (&f)[32], int st, int b, int h) {
                const uint32_t a = smem_u32(smem + Tc32Smem::A + st * T32_STAGE_A) + g * 1024 + b * 2 * MMQ_PANEL;
                const uint32_t bb = smem_u32(smem + Tc32Smem::B + st * T32_STAGE_B) + h * 1024 + b * 2 * MMQ_PANEL;
                wg_fence();
                wg_mma_ss_s8(f, wg_desc(a, MMQ_PANEL, 128u), wg_desc(bb, MMQ_PANEL, 128u), 0u);
                wg_commit();
            };
            auto fold = [&](int32_t (&f)[32], int st, int b, int h) {
                const float * rs = (const float *)(smem + Tc32Smem::RS + st * 2048) + b * 128;
                const float da = rs[ra], db = rs[ra + 8];
                const float2 * dx2 = (const float2 *)(smem + Tc32Smem::B + st * T32_STAGE_B + 8 * MMQ_PANEL + (b * 128 + 64 * h + c0) * 4);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const float2 dxp = dx2[4 * j];
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const float dx = e ? dxp.y : dxp.x;
                        float & ua = acc[4 * (8 * h + j) + e], & ub = acc[4 * (8 * h + j) + 2 + e];
                        const float sa = (float)f[4 * j + e], sb = (float)f[4 * j + 2 + e];
                        if (T == B200_TYPE_Q4_0) {                                  // ((float)s * d_w) * d_x
                            ua = __fadd_rn(ua, __fmul_rn(__fmul_rn(sa, da), dx));
                            ub = __fadd_rn(ub, __fmul_rn(__fmul_rn(sb, db), dx));
                        } else if (T == B200_TYPE_IQ4_XS) {                         // ((d_w * d_x) * (float)(ls - 32)) * (float)s
                            const uint32_t wa = __float_as_uint(da), wb = __float_as_uint(db);
                            const float la = (float)((int32_t)wa >> 16), lb = (float)((int32_t)wb >> 16);
                            ua = __fadd_rn(ua, __fmul_rn(__fmul_rn(__fmul_rn(h2f((uint16_t)wa), dx), la), sa));
                            ub = __fadd_rn(ub, __fmul_rn(__fmul_rn(__fmul_rn(h2f((uint16_t)wb), dx), lb), sb));
                        } else {                                                    // Q5_0 / Q8_0 / IQ4_NL: (float)s * (d_w * d_x)
                            ua = __fadd_rn(ua, __fmul_rn(sa, __fmul_rn(da, dx)));
                            ub = __fadd_rn(ub, __fmul_rn(sb, __fmul_rn(db, dx)));
                        }
                    }
                }
            };
            for (int s = 0; s < ns; s++, it++) {
                const int st = it % T32_NSTAGE;
                mbar_wait_p(&b_full[st], (it / T32_NSTAGE) & 1, pw0);
                mbar_wait_p(&a_full[st], (it / T32_NSTAGE) & 1, pw1);
                // straight-line software pipeline over the 4 blocks of the stage: one half's MMA runs while the other half is folded
                mma(f0, st, 0, 0);
#pragma unroll
                for (int b = 0; b < 4; b++) {
                    mma(f1, st, b, 1);
                    wg_wait1(); wg_pin(f0);
                    fold(f0, st, b, 0);
                    if (b < 3) { mma(f0, st, b + 1, 0); wg_wait1(); } else wg_wait0();
                    wg_pin(f1);
                    fold(f1, st, b, 1);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&ab_empty[st]);                // every MMA and every scale read of the stage is done
            }
            mmq_store_tile<GROUPED>(args, acc, mt, nt, ra, c0);
        }
    }

    if (prof && lane == 0) mmq_prof_store(args, warp, t_start, w0, w1);
    pdl_trigger();
}

// ---- host ----------------------------------------------------------------------------------------------------------
int64_t b200_mmq_tc32_workspace(int64_t k, int64_t ncols) { return tc32_geom(k, ncols).total; }

template <bool GROUPED> static int tc32_launch(int type, const Tc32Args & a, cudaStream_t st) {
    switch (type) {
        case B200_TYPE_Q4_0: return mmq_tile_launch<mmq_tc32_kernel<B200_TYPE_Q4_0, GROUPED>, Tc32Smem::TOTAL>(a, st);
        case B200_TYPE_Q5_0: return mmq_tile_launch<mmq_tc32_kernel<B200_TYPE_Q5_0, GROUPED>, Tc32Smem::TOTAL>(a, st);
        case B200_TYPE_Q8_0: return mmq_tile_launch<mmq_tc32_kernel<B200_TYPE_Q8_0, GROUPED>, Tc32Smem::TOTAL>(a, st);
        // dense only: MUL_MAT_ID on these formats stays on the wide matvec (mmid_route.cu)
        case B200_TYPE_IQ4_NL: if constexpr (!GROUPED) return mmq_tile_launch<mmq_tc32_kernel<B200_TYPE_IQ4_NL, false>, Tc32Smem::TOTAL>(a, st); break;
        case B200_TYPE_IQ4_XS: if constexpr (!GROUPED) return mmq_tile_launch<mmq_tc32_kernel<B200_TYPE_IQ4_XS, false>, Tc32Smem::TOTAL>(a, st); break;
    }
    return B200_ERR_UNSUPPORTED;
}

int b200_mmq_tc32(int type, const MmqJob & j, cudaStream_t st) {
    const Tc32Geom g = tc32_geom(j.k, j.ncols);
    Tc32Args a = {};
    mmq_tile_fill(a, j, (j.k / xf_block_elems(type)) * xf_block_bytes(type));     // Q4_0 / Q5_0 / Q8_0: the repacked rows are as long as the native ones
    a.nks = (int32_t)g.ns;
    if (type == B200_TYPE_IQ4_XS) {
        if (j.map) return B200_ERR_UNSUPPORTED;
        B200_CUDA(b200_launch_pdl(quantize_mmq32k_kernel, dim3((unsigned)(j.k / 256), (unsigned)(a.nt * 16)), dim3(256), 0, st,
                                  j.X, j.x_col_stride, j.ncols, j.k_valid, (uint8_t *)j.workspace, g));
    } else {
        B200_CUDA(b200_launch_pdl(j.map ? quantize_mmq32_kernel<true> : quantize_mmq32_kernel<false>, dim3((unsigned)(j.k / 256), (unsigned)(a.nt * 16)), dim3(256), 0, st,
                                  j.X, j.x_col_stride, j.ncols, j.k_valid, (uint8_t *)j.workspace, g, a.map));
    }
    b200_count_launch();
    const int rc = j.map ? tc32_launch<true>(type, a, st) : tc32_launch<false>(type, a, st);
    if (a.prof && rc == B200_OK) mmq_prof_report(j.map ? "mmq_tc32 grouped" : "mmq_tc32", type, a, st);
    return rc;
}
