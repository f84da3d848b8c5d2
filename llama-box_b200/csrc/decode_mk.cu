// decode_mk.cu — the persistent batch-1 decode kernel (sm_90a): one launch runs a whole chain of fused phases
// (mk.h) — [rms_norm ->] quantised matvecs with their epilogues, and rope + KV store + flash attention.
//
// Replaces, for a decode token, the reference's per-op launch sequence mul_mat_vec_q / quantize_q8_1 / rms_norm /
// rope / set_rows / flash_attn_vec / combine (ggml-cuda.cu:2207-2493 dispatch; mmvq.cu:139-503, fattn-vec-f32.cuh)
// and the CUDA-graph replay around it (ggml-cuda.cu:2845-3010).
//
// Shape of the kernel (HBM-bound by design: a decode token streams every weight byte exactly once):
//   * grid = one CTA per SM, 10 warps, ~205 KB of shared memory: a 2-slot TMA ring per warp (cp.async.bulk + mbarrier)
//     and one region that holds the quantised activation vector of the current matvec phase (or attention scratch);
//   * per matvec phase every SM owns a contiguous range of row PAIRS; a warp owns whole groups of pairs (8 rows of
//     Q4_K, 4 of Q6_K) and walks K in 2048-element steps, one ring slot per step.  A lane owns ONE super-block of
//     one row pair (Q4_K) or half a super-block (Q6_K): scales are decoded once per super-block, nibbles are used in
//     place ((q & 0xF0F0F0F0) . a, one >>4 per sum), the min / -32 terms are two-wide dp2a on pre-summed activations;
//   * a warp's slot sequence runs ACROSS phases: after its last slot of phase p it immediately streams its first slots
//     of the next matvec phase, so weights keep arriving while the grid barrier, the activation rebuild or the
//     attention phase run;
//   * phases are separated by a grid-wide barrier (atomic counter, self-cleaning on exit).
// Numerics: identical integer dots and activation quantisation to the CPU oracle (see quantize.cu / mmvq.cu); float
// accumulation order differs from mmvq.cu only in grouping (per super-block instead of per quarter).
#include "common.cuh"
#include "mk.h"
#include "ropeutil.cuh"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

namespace {

// One entry of the CTA's phase table: this SM's pair ranges per matrix + a shared-memory copy of the phase record (every
// descriptor field on the refill path would otherwise be an L2 round trip per ring slot).  Entries are planned two phases
// ahead by one warp (mk_plan), so neither the global read nor the partition arithmetic sits on anyone's critical path.
struct PCache { alignas(16) MkPhase ph; int ngroups; int gbase[MK_MAX_MATS + 1]; int pstart[MK_MAX_MATS]; int pend[MK_MAX_MATS]; int pad[2]; };
#define MK_TAB 4
struct Cur { int p, g, s, entered; };
#define MK_TUNE_DEFAULT 0        // bit 4: no weight streaming across phase boundaries (debug)

__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long * p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void grid_arrive(unsigned long long * bar) {
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); atomicAdd(bar, 1ULL); }
}
__device__ __forceinline__ void grid_wait(unsigned long long * bar, unsigned long long target) {
    if (threadIdx.x == 0) {
        while (ld_acquire_u64(bar) < target) { }
        __threadfence();
    }
    __syncthreads();
}

__device__ __forceinline__ int dp4a_u8s8(uint32_t w, uint32_t a, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(w), "r"(a), "r"(c));
    return d;
}
__device__ __forceinline__ int dot16m(const uint4 & w, const uint4 & a, uint32_t m, int c) {
    c = dp4a_u8s8(w.x & m, a.x, c); c = dp4a_u8s8(w.y & m, a.y, c);
    c = dp4a_u8s8(w.z & m, a.z, c); return dp4a_u8s8(w.w & m, a.w, c);
}
__device__ __forceinline__ int prmt(uint32_t a, uint32_t b, uint32_t sel) {      // bit 3 of a selector nibble replicates the sign
    int d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
}
// Slot geometry.  A ring slot always holds 64 (Q4_K) / 32 (Q6_K) super-blocks: S super-blocks of each row of `ppg` row
// pairs.  When a whole row fits (S == nsb: k = 2048, 4096 and, for Q4_K, 8192) the rows of a group are ONE contiguous byte
// range -> one bulk copy per slot (two for a gate/up pair); otherwise S = 8 and a row is walked in nsb/8 steps.
__device__ __forceinline__ int S_of(int type, int nsb) { return (nsb == 16 || (nsb == 32 && type == B200_TYPE_Q4_K)) ? nsb : 8; }
__device__ __forceinline__ int ppg_of(int type, int nsb) { return (type == B200_TYPE_Q4_K ? 32 : 16) / S_of(type, nsb); }
__device__ __forceinline__ int rowbytes_of(int type, int S) { return S * (type == B200_TYPE_Q4_K ? 144 : 210); }

// swizzled position of 16-byte chunk `idx` (0..15) of super-block sb in the activation vector: lanes that read the same
// chunk of 8 consecutive super-blocks (Q4_K mapping), or different chunks of 4 (Q6_K mapping), hit 8 distinct bank groups
__device__ __forceinline__ int act_chunk(int idx, int sb) { return idx ^ (sb & 7) ^ ((idx & 8) >> 1); }

// ---- activation vector: [rms_norm * w ->] q8_K exactly as the CPU oracle quantises (ggml-quants.c:2555-2592) ----
// 8 lanes per 256-element block, 32 consecutive elements per lane: the per-16 / per-32 sums and the packing are in-lane,
// only the block maximum crosses lanes (3 shuffle rounds), and a warp quantises 4 blocks at once.  This sits on the
// critical path right after every grid barrier.
__device__ __forceinline__ void mk_quant32(const float (&v)[32], uint8_t * act, int k, int blk, int li) {
    const int nsb = k >> 8;
    const unsigned gm = 0xffu << ((threadIdx.x & 24));              // the 8 lanes of this block
    float am = 0.0f, mv = 0.0f; int ai = 0;
#pragma unroll
    for (int j = 0; j < 32; j++) { const float a = fabsf(v[j]); if (a > am) { am = a; mv = v[j]; ai = li * 32 + j; } }
    // first index of the largest |x| (the reference scans sequentially with a strict '>')
#pragma unroll
    for (int o2 = 1; o2 < 8; o2 <<= 1) {
        const float am2 = __shfl_xor_sync(gm, am, o2), mv2 = __shfl_xor_sync(gm, mv, o2);
        const int   ai2 = __shfl_xor_sync(gm, ai, o2);
        if (am2 > am || (am2 == am && ai2 < ai)) { am = am2; mv = mv2; ai = ai2; }
    }
    uint32_t w[8]; int s16a = 0, s16b = 0; float d = 0.0f;
    if (am != 0.0f) {
        const float iscale = __fdiv_rn(-127.0f, mv);
#pragma unroll
        for (int j = 0; j < 32; j++) {
            int t = __float2int_rn(__fmul_rn(iscale, v[j])); t = t > 127 ? 127 : t;
            if (j < 16) s16a += t; else s16b += t;
            if ((j & 3) == 0) w[j >> 2] = (uint32_t)(t & 0xff); else w[j >> 2] |= (uint32_t)(t & 0xff) << (8 * (j & 3));
        }
        d = __fdiv_rn(1.0f, iscale);
    } else {
#pragma unroll
        for (int j = 0; j < 8; j++) w[j] = 0;
    }
    uint8_t * qb = act + blk * 256;
    *(uint4 *)(qb + act_chunk(2 * li, blk) * 16)     = make_uint4(w[0], w[1], w[2], w[3]);
    *(uint4 *)(qb + act_chunk(2 * li + 1, blk) * 16) = make_uint4(w[4], w[5], w[6], w[7]);
    *(uint32_t *)(act + k + 4 * nsb + blk * 32 + li * 4) = (uint32_t)(s16a & 0xffff) | ((uint32_t)(s16b & 0xffff) << 16);
    ((int16_t *)(act + k + 36 * nsb))[blk * 8 + li] = (int16_t)(s16a + s16b);
    if (li == 0) ((float *)(act + k))[blk] = d;
}

__device__ __forceinline__ void mk_load32(const float * p, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; j++) { const float4 t = __ldcg((const float4 *)(p + 4 * j)); v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w; }
}

__device__ __noinline__ void mk_build_act(const MkMmv * M, uint8_t * act, double * red, int warp, int lane, int nw) {
    const int k = M->k, nsb = k >> 8;
    const float * x = M->x;
    const int lg = lane >> 3, li = lane & 7;
    if (M->act_source == 2) {
        // rms_norm (ggml-cpu/ops.cpp:4164-4183: f32 squares summed in double) — one block per lane group: k <= 4 * nw * 256
        const int blk = warp * 4 + lg;
        const bool on = blk < nsb;
        float v[32];
        if (on) mk_load32(x + blk * 256 + li * 32, v);
        else {
#pragma unroll
            for (int j = 0; j < 32; j++) v[j] = 0.0f;
        }
        double a0 = 0.0, a1 = 0.0;
#pragma unroll
        for (int j = 0; j < 32; j += 2) { a0 += (double)__fmul_rn(v[j], v[j]); a1 += (double)__fmul_rn(v[j + 1], v[j + 1]); }
        double a2 = a0 + a1;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a2 += __shfl_xor_sync(0xffffffffu, a2, o);
        if (lane == 0) red[warp] = a2;
        const float * nwp = M->norm_w;
        float4 wv[8];
        if (nwp && on) {
#pragma unroll
            for (int j = 0; j < 8; j++) wv[j] = *(const float4 *)(nwp + blk * 256 + li * 32 + 4 * j);
        }
        __syncthreads();
        double t = 0.0;
        for (int i = 0; i < nw; i++) t += red[i];                  // every thread: same order, same value
        const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn((float)(t / (double)k), M->eps)));
        if (on) {
#pragma unroll
            for (int j = 0; j < 32; j++) v[j] = __fmul_rn(v[j], scale);
            if (nwp) {
#pragma unroll
                for (int j = 0; j < 8; j++) { v[4 * j] = __fmul_rn(v[4 * j], wv[j].x); v[4 * j + 1] = __fmul_rn(v[4 * j + 1], wv[j].y); v[4 * j + 2] = __fmul_rn(v[4 * j + 2], wv[j].z); v[4 * j + 3] = __fmul_rn(v[4 * j + 3], wv[j].w); }
            }
        }
        if (on) mk_quant32(v, act, k, blk, li);                   // shuffles stay inside the 8-lane group
    } else {
        for (int b0 = warp * 4; b0 < nsb; b0 += nw * 4) {
            const int blk = b0 + lg;
            if (blk < nsb) {                                        // nsb % 8 == 0: a lane group is on or off as a whole; shuffles stay inside it
                float v[32];
                mk_load32(x + blk * 256 + li * 32, v);
                mk_quant32(v, act, k, blk, li);
            }
        }
    }
    __syncthreads();
}

// ---- this SM's share of a matvec phase: planned into the CTA's phase table by ONE warp, two phases ahead -----------
// plan_begin: fire-and-forget copy of the phase record (cp.async, 16 lanes x 16 bytes) at the start of phase q - 3;
// plan_finish: at the end of that phase the same warp waits for it (long since landed), partitions and publishes.
__device__ __forceinline__ void mk_plan_begin(const MkPhase * prog, int q, PCache * tab, int lane) {
    if (lane < 16) {
        const uint32_t dst = smem_u32((uint8_t *)&tab[q % MK_TAB].ph + lane * 16);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"((const uint8_t *)(prog + q) + lane * 16) : "memory");
    }
}
__device__ __noinline__ void mk_plan_finish(int q, PCache * tab, volatile int * tab_phase, int lane) {
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncwarp();
    PCache * pc = &tab[q % MK_TAB];
    if (pc->ph.kind == MK_MMV) {
        const MkMmv * M = &pc->ph.mmv;
        // pairs: two consecutive rows of one matrix, or (gate row r, up row r)
        const int nm = M->swiglu ? 1 : M->n_mats;
        long long total = 0;
        for (int i = 0; i < nm; i++) total += M->swiglu ? M->mat[0].m : (M->mat[i].m >> 1);
        const long long lo = total * blockIdx.x / gridDim.x, hi = total * (blockIdx.x + 1) / gridDim.x;
        long long off = 0; int gb = 0;
        for (int i = 0; i < MK_MAX_MATS; i++) {
            int ps = 0, pe = 0;
            if (i < nm) {
                const long long n = M->swiglu ? M->mat[0].m : (M->mat[i].m >> 1);
                const long long s = lo > off ? lo : off, e = hi < off + n ? hi : off + n;
                if (e > s) { ps = (int)(s - off); pe = (int)(e - off); }
                off += n;
            }
            if (lane == 0) { pc->gbase[i] = gb; pc->pstart[i] = ps; pc->pend[i] = pe; }
            if (i < nm) { const int ppg = ppg_of(M->mat[i].type, M->k >> 8); gb += (pe - ps + ppg - 1) / ppg; }
        }
        if (lane == 0) { pc->gbase[MK_MAX_MATS] = gb; pc->ngroups = gb; }
    }
    __syncwarp();
    __threadfence_block();
    if (lane == 0) tab_phase[q % MK_TAB] = q;
}

struct Grp { int i, type, pair0, np, S, ppg; };
__device__ __forceinline__ Grp mk_locate(const MkMmv * M, const PCache * pc, int g) {
    Grp r; r.i = 0;
#pragma unroll
    for (int i = 1; i < MK_MAX_MATS; i++) if (g >= pc->gbase[i]) r.i = i;
    // gbase[] is non-decreasing (empty matrices repeat the next base): the last i with gbase[i] <= g owns group g
    r.type = M->mat[r.i].type;
    r.S = S_of(r.type, M->k >> 8);
    r.ppg = (r.type == B200_TYPE_Q4_K ? 32 : 16) / r.S;
    r.pair0 = pc->pstart[r.i] + (g - pc->gbase[r.i]) * r.ppg;
    r.np = pc->pend[r.i] - r.pair0; if (r.np > r.ppg) r.np = r.ppg;
    return r;
}

// one ring slot = step `step` (S super-blocks) of every row of group g.  Rows sit at rowbytes = S*144 (Q4_K) or S*210
// (Q6_K, as ql[S*128] | qh[S*64] | scales[S*16] | d[S*2]); pair j's rows are slot rows 2j, 2j+1 — or j and ppg + j for a
// gate/up pair, so that each matrix's rows stay one contiguous range.
__device__ __forceinline__ void mk_issue(const MkMmv * M, const PCache * pc, int g, int step, uint8_t * slot, uint64_t * bar, int lane) {
    const Grp gr = mk_locate(M, pc, g);
    const int rows = 2 * gr.np;
    const int nb = M->k >> 8;
    const int rowbytes = rowbytes_of(gr.type, gr.S);
    if (lane == 0) mbar_expect_tx(bar, (uint32_t)(rows * rowbytes));
    __syncwarp();
    if (gr.S == nb) {
        // whole rows: the group's rows are contiguous in the matrix
        if (M->swiglu) {
            if (lane < 2) bulk_g2s(slot + lane * gr.ppg * rowbytes, M->mat[lane].W + (int64_t)gr.pair0 * M->mat[lane].rb, (uint32_t)(gr.np * rowbytes), bar);
        } else if (lane == 0) {
            bulk_g2s(slot, M->mat[gr.i].W + (int64_t)(2 * gr.pair0) * M->mat[gr.i].rb, (uint32_t)(rows * rowbytes), bar);
        }
        return;
    }
    if (gr.type == B200_TYPE_Q4_K) {
        if (lane < rows) {
            const int pj = lane >> 1, rr = lane & 1;
            const MkMat & mt = M->swiglu ? M->mat[rr] : M->mat[gr.i];
            const int64_t row = M->swiglu ? gr.pair0 + pj : 2 * gr.pair0 + lane;
            const int srow = M->swiglu ? pj + rr * gr.ppg : lane;
            bulk_g2s(slot + srow * 1152, mt.W + row * mt.rb + (int64_t)step * 1152, 1152, bar);
        }
    } else {
        if (lane < rows * 4) {
            const int r = lane >> 2, part = lane & 3;
            const int pj = r >> 1, rr = r & 1;
            const MkMat & mt = M->swiglu ? M->mat[rr] : M->mat[gr.i];
            const int64_t row = M->swiglu ? gr.pair0 + pj : 2 * gr.pair0 + r;
            const int srow = M->swiglu ? pj + rr * gr.ppg : r;
            const uint8_t * rb = mt.W + row * mt.rb;
            // repacked Q6_K row: ql[nb*128] | qh[nb*64] | scales[nb*16] | d[nb*2]   (repack.cu)
            const int64_t soff = part == 0 ? (int64_t)step * 1024 : part == 1 ? (int64_t)nb * 128 + step * 512 : part == 2 ? (int64_t)nb * 192 + step * 128 : (int64_t)nb * 208 + step * 16;
            const int doff = part == 0 ? 0 : part == 1 ? 1024 : part == 2 ? 1536 : 1664;
            const uint32_t bytes = part == 0 ? 1024u : part == 1 ? 512u : part == 2 ? 128u : 16u;
            bulk_g2s(slot + srow * 1680 + doff, rb + soff, bytes, bar);
        }
    }
}

// position the issue cursor on this warp's next ring slot; false: the phase it would enter is not planned yet
__device__ __forceinline__ bool cur_seek(Cur & c, int n_phases, const PCache * tab, const volatile int * tab_phase, int warp) {
    while (c.p < n_phases) {
        if (tab_phase[c.p % MK_TAB] != c.p) return false;
        const PCache * pc = &tab[c.p % MK_TAB];
        if (pc->ph.kind == MK_MMV && warp < pc->ngroups) { c.g = warp; c.s = 0; c.entered = 1; return true; }
        c.p++;
    }
    return false;
}
__device__ __forceinline__ void cur_advance(Cur & c, const PCache * pc, int nsteps, int nw) {
    if (++c.s < nsteps) return;
    c.s = 0; c.g += nw;
    if (c.g < pc->ngroups) return;
    c.p++; c.entered = 0;
}
// keep this warp's two ring slots busy: issue the next slots of its sequence (possibly of later phases) while there is room
__device__ __forceinline__ void mk_pump(Cur & ic, int & nissued, int ncons, int plimit, int n_phases, const PCache * tab, const volatile int * tab_phase,
                                        uint8_t * ring, uint64_t * full, int warp, int lane, int nw) {
    while (nissued - ncons < 2) {
        if (!ic.entered && !cur_seek(ic, n_phases, tab, tab_phase, warp)) break;
        if (ic.p > plimit) break;
        const PCache * pc = &tab[ic.p % MK_TAB];
        const int ipos = nissued & 1;
        mk_issue(&pc->ph.mmv, pc, ic.g, ic.s, ring + ipos * MK_SLOT_BYTES, &full[ipos], lane);
        { const Grp gi = mk_locate(&pc->ph.mmv, pc, ic.g); cur_advance(ic, pc, (pc->ph.mmv.k >> 8) / gi.S, nw); }
        nissued++;
    }
}

// ---- Q4_K: lane = (pair lg = lane>>3, super-block sb = lane&7) of the slot; both rows of the pair ------------------
// S super-blocks per slot row (8 | 16 | 32); the pair's second row sits `rstride` bytes after the first (row-interleaved
// pairs: one row; gate/up pairs: ppg rows)
template <int S>
__device__ __forceinline__ void mk_dot_q4K(const uint8_t * slot, const uint8_t * act, int k, int step, int lane, bool glu, float & acc0, float & acc1) {
    constexpr int RB = S * 144, PPG = 32 / S;
    const int lg = lane / S, sb = lane % S;
    const int nsb = k >> 8, gsb = step * S + sb;
    const int rstride = glu ? PPG * RB : RB;
    const uint8_t * r0 = slot + (glu ? lg : 2 * lg) * RB + sb * 144;
    const uint8_t * aq = act + gsb * 256;
    const float da = ((const float *)(act + k))[gsb];
    const uint4 s32 = *(const uint4 *)(act + k + 36 * nsb + gsb * 16);
    uint32_t sc03[2], sc47[2], mn03[2], mn47[2]; float dw[2], dm[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const uint4 hdr = *(const uint4 *)(r0 + r * rstride);
        const uint32_t y = hdr.y, z = hdr.z, w = hdr.w;              // 6-bit scales / mins (ggml-quants.c:703-711), SIMD decode
        sc03[r] = y & 0x3f3f3f3fu; mn03[r] = z & 0x3f3f3f3fu;
        sc47[r] = (w & 0x0f0f0f0fu) | ((y >> 2) & 0x30303030u);
        mn47[r] = ((w >> 4) & 0x0f0f0f0fu) | ((z >> 2) & 0x30303030u);
        dw[r] = h2f((uint16_t)(hdr.x & 0xffff)); dm[r] = h2f((uint16_t)(hdr.x >> 16));
    }
    int isl[2] = { 0, 0 }, ish[2] = { 0, 0 };
#pragma unroll
    for (int g = 0; g < 4; g++) {
        uint4 a[4];
#pragma unroll
        for (int j = 0; j < 4; j++) { const int idx = 4 * g + j; a[j] = *(const uint4 *)(aq + (((idx ^ ((idx & 8) >> 1)) ^ (sb & 7)) << 4)); }
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const uint8_t * rr = r0 + r * rstride + 16 + 32 * g;
            const uint4 q0 = *(const uint4 *)rr, q1 = *(const uint4 *)(rr + 16);
            int dl = dot16m(q0, a[0], 0x0F0F0F0Fu, 0); dl = dot16m(q1, a[1], 0x0F0F0F0Fu, dl);
            int dh = dot16m(q0, a[2], 0xF0F0F0F0u, 0); dh = dot16m(q1, a[3], 0xF0F0F0F0u, dh);
            const uint32_t scw = g < 2 ? sc03[r] : sc47[r];
            const int sl = (int)__byte_perm(scw, 0, 0x4440 + ((2 * g) & 3)), sh = (int)__byte_perm(scw, 0, 0x4440 + ((2 * g + 1) & 3));
            isl[r] += sl * dl; ish[r] += sh * dh;
        }
    }
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int isum = isl[r] + (ish[r] >> 4);
        int imin = __dp2a_lo((int)s32.x, (int)mn03[r], 0);
        imin = __dp2a_hi((int)s32.y, (int)mn03[r], imin);
        imin = __dp2a_lo((int)s32.z, (int)mn47[r], imin);
        imin = __dp2a_hi((int)s32.w, (int)mn47[r], imin);
        const float v = __fmul_rn(dw[r], da) * (float)isum - __fmul_rn(dm[r], da) * (float)imin;
        if (r == 0) acc0 += v; else acc1 += v;
    }
}

// ---- Q6_K: lane = (pair lg = lane>>4, super-block sb = (lane>>1)&7, half h = lane&1) ---------------------------------
template <int S>
__device__ __forceinline__ void mk_dot_q6K(const uint8_t * slot, const uint8_t * act, int k, int step, int lane, bool glu, float & acc0, float & acc1) {
    constexpr int RB = S * 210, PPG = 16 / S;
    const int lg = lane / (2 * S), sb = (lane >> 1) % S, h = lane & 1;
    const int nsb = k >> 8, gsb = step * S + sb;
    const int rot = (0x78 >> (2 * (sb & 3))) & 3;                   // chunk order differs per lane: conflict-free LDS.128
    const int rstride = glu ? PPG * RB : RB;
    const uint8_t * rb0 = slot + (glu ? lg : 2 * lg) * RB;
    const uint8_t * aq = act + gsb * 256;
    const float da = ((const float *)(act + k))[gsb];
    const uint4 b16 = *(const uint4 *)(act + k + 4 * nsb + gsb * 32 + h * 16);
    uint2 scw[2]; float dw[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
        scw[r] = *(const uint2 *)(rb0 + r * rstride + S * 192 + sb * 16 + h * 8);
        dw[r]  = h2f(*(const uint16_t *)(rb0 + r * rstride + S * 208 + sb * 2));
    }
    int isum[2] = { 0, 0 };
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const int cp = c ^ rot, which = cp >> 1;
        const int ilo = 8 * h + cp;
        const uint4 Alo = *(const uint4 *)(aq + ((ilo ^ (sb & 7) ^ (4 * h)) << 4));
        const uint4 Ahi = *(const uint4 *)(aq + (((ilo + 4) ^ (sb & 7) ^ (4 * h)) << 4));
        const int shl = 2 * which;
        const uint32_t mlo = 0x03030303u << shl, mhi = mlo << 4;
        const uint32_t sel_lo = (uint32_t)cp | ((uint32_t)(cp | 8) * 0x1110u), sel_hi = sel_lo + 0x4444u;   // sign-extending byte select
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const uint8_t * rb = rb0 + r * rstride;
            const uint4 QL = *(const uint4 *)(rb + sb * 128 + h * 64 + cp * 16);
            const uint4 QH = *(const uint4 *)(rb + S * 128 + sb * 64 + h * 32 + (cp & 1) * 16);
            const int dlo = dot16m(QL, Alo, 0x0F0F0F0Fu, 0), dloh = dot16m(QH, Alo, mlo, 0) >> shl;
            const int dhi = dot16m(QL, Ahi, 0xF0F0F0F0u, 0) >> 4, dhih = dot16m(QH, Ahi, mhi, 0) >> (shl + 4);
            const int sclo = prmt(scw[r].x, scw[r].y, sel_lo), schi = prmt(scw[r].x, scw[r].y, sel_hi);
            isum[r] += sclo * (dlo + 16 * dloh) + schi * (dhi + 16 * dhih);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; r++) {
        int m32 = __dp2a_lo((int)b16.x, (int)scw[r].x, 0);          // sum_j sc_j * bsum16_j  (the -32 offset of q6)
        m32 = __dp2a_hi((int)b16.y, (int)scw[r].x, m32);
        m32 = __dp2a_lo((int)b16.z, (int)scw[r].y, m32);
        m32 = __dp2a_hi((int)b16.w, (int)scw[r].y, m32);
        const float v = __fmul_rn(dw[r], da) * (float)(isum[r] - 32 * m32);
        if (r == 0) acc0 += v; else acc1 += v;
    }
}

// ---- one matvec phase, consumer side ----------------------------------------------------------------------------------
__device__ __forceinline__ void mk_mmv_phase(int n_phases, int p, const uint8_t * act, uint8_t * ring, uint64_t * full, const PCache * tab, const volatile int * tab_phase,
                                             Cur & ic, int & ncons, int & nissued, int plimit, int warp, int lane, int nw, unsigned int * stats) {
    const PCache * cpc = &tab[p % MK_TAB];
    const MkMmv * M = &cpc->ph.mmv;                                 // shared-memory copy
    const int k = M->k;
    const int ng = cpc->ngroups;
    const bool glu = M->swiglu != 0;
    for (int g = warp; g < ng; g += nw) {
        const Grp gr = mk_locate(M, cpc, g);
        const int nsteps = (k >> 8) / gr.S;
        float acc0 = 0.0f, acc1 = 0.0f;
        for (int step = 0; step < nsteps; step++) {
            const int pos = ncons & 1;
            const long long c0 = stats ? clock64() : 0;
            mbar_wait(&full[pos], (uint32_t)((ncons >> 1) & 1));
            const long long c1 = stats ? clock64() : 0;
            uint8_t * slot = ring + pos * MK_SLOT_BYTES;
            if (gr.type == B200_TYPE_Q4_K) {
                if (gr.S == 8) mk_dot_q4K<8>(slot, act, k, step, lane, glu, acc0, acc1);
                else if (gr.S == 16) mk_dot_q4K<16>(slot, act, k, step, lane, glu, acc0, acc1);
                else mk_dot_q4K<32>(slot, act, k, step, lane, glu, acc0, acc1);
            } else {
                if (gr.S == 8) mk_dot_q6K<8>(slot, act, k, step, lane, glu, acc0, acc1);
                else mk_dot_q6K<16>(slot, act, k, step, lane, glu, acc0, acc1);
            }
            __syncwarp();                                           // every lane is done reading the slot
            const long long c2 = stats ? clock64() : 0;
            ncons++;
            mk_pump(ic, nissued, ncons, plimit, n_phases, tab, tab_phase, ring, full, warp, lane, nw);   // refill it
            if (stats && lane == 0) { atomicAdd(stats + 0, (unsigned int)(c1 - c0)); atomicAdd(stats + 1, (unsigned int)(c2 - c1)); atomicAdd(stats + 2, (unsigned int)(clock64() - c2)); atomicAdd(stats + 3, 1u); }
        }
        // reduce over the lanes of each pair, then bias / residual / SwiGLU
        const int lgw = 32 / gr.ppg;                              // lanes per pair: 8, 16 or 32
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            if (o < lgw) { acc0 += __shfl_xor_sync(0xffffffffu, acc0, o); acc1 += __shfl_xor_sync(0xffffffffu, acc1, o); }
        }
        const int pl = lane / lgw;
        if ((lane & (lgw - 1)) == 0 && pl < gr.np) {
            const int pair = gr.pair0 + pl;
            if (M->swiglu) {
                M->mat[0].dst[pair] = __fmul_rn(silu_x86(acc0), acc1);                  // ggml-cpu/vec.cpp:260-282
            } else {
                const MkMat & mt = M->mat[gr.i];
                const int r = 2 * pair;
                float v0 = acc0, v1 = acc1;
                if (mt.bias)     { v0 += mt.bias[r]; v1 += mt.bias[r + 1]; }
                if (mt.residual) { v0 += __ldcg(mt.residual + r); v1 += __ldcg(mt.residual + r + 1); }
                *(float2 *)(mt.dst + r) = make_float2(v0, v1);
            }
        }
    }
}

// ---- rope + KV store + split-KV flash attention for the decode token (numerics: fattn.cu / rope.cu) -------------------
__device__ __forceinline__ void unpack_h8(const uint4 & r, float (&f)[8]) {
    const __half2 * h = (const __half2 *)&r;
#pragma unroll
    for (int i = 0; i < 4; i++) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
// 8 int8 of a native q8_0 row (34-byte blocks, 2-byte aligned) + the block scale; generic loads (global or shared)
__device__ __forceinline__ void load_q80_8(const uint8_t * row, int dl, int (&q)[2], float & d) {
    const uint8_t * blk = row + (dl >> 2) * 34;
    const uint16_t * p = (const uint16_t *)(blk + 2 + (dl & 3) * 8);
    d = h2f(*(const uint16_t *)blk);
    q[0] = (int)((uint32_t)p[0] | ((uint32_t)p[1] << 16));
    q[1] = (int)((uint32_t)p[2] | ((uint32_t)p[3] << 16));
}
// elements e0..e0+7 of one head, roped (ops.cpp:6088-6150 pairing; the table holds cos/sin already scaled)
__device__ __forceinline__ void load_roped8(const float * head, int e0, const float * cs, const MkRope & rp, float (&v)[8]) {
    const float4 a = __ldcg((const float4 *)(head + e0)), b = __ldcg((const float4 *)(head + e0 + 4));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    if (e0 >= rp.n_dims) return;
    if (!rp.neox) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int i = (e0 >> 1) + j;
            const float c = cs[2 * i], sn = cs[2 * i + 1], x0 = v[2 * j], x1 = v[2 * j + 1];
            v[2 * j]     = __fsub_rn(__fmul_rn(x0, c), __fmul_rn(x1, sn));
            v[2 * j + 1] = __fadd_rn(__fmul_rn(x0, sn), __fmul_rn(x1, c));
        }
    } else {
        const int half = rp.n_dims >> 1;
        const bool first = e0 < half;
        const int po = first ? e0 + half : e0 - half;
        const float4 pa = __ldcg((const float4 *)(head + po)), pb = __ldcg((const float4 *)(head + po + 4));
        const float o[8] = { pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w };
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int i = first ? e0 + j : e0 - half + j;
            const float c = cs[2 * i], sn = cs[2 * i + 1];
            v[j] = first ? __fsub_rn(__fmul_rn(v[j], c), __fmul_rn(o[j], sn)) : __fadd_rn(__fmul_rn(o[j], sn), __fmul_rn(v[j], c));
        }
    }
}

template <int D, int KVT, int G>
__device__ __noinline__ void mk_attn(const MkAttn * Ap, uint8_t * scr, int nw) {
    constexpr int LP = D / 8, PPW = 32 / LP;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sg = lane / LP, dl = lane % LP;
    float * cs = (float *)scr;                                     // [128]
    uint8_t * newk = scr + 512, * newv = scr + 800;               // this token's K / V row slice in cache format
    float * sM = (float *)(scr + 1088), * sL = (float *)(scr + 1248), * s_inv = (float *)(scr + 1408);
    unsigned int * s_last = (unsigned int *)(scr + 1424);
    float * s_sc = (float *)(scr + 1536);                          // [64][G]
    float * sA = (float *)(scr + 2560);                            // [nw][G][D]
    const MkRope rp = Ap->rp;
    const int n_head = Ap->n_head, n_head_kv = Ap->n_head_kv, n_kv = Ap->n_kv, split_len = Ap->split_len, n_splits = Ap->n_splits;
    const int gq = n_head / n_head_kv, n_tiles = n_head / G;
    const float scale = Ap->scale, max_bias = Ap->max_bias, softcap = Ap->softcap;
    const int64_t k_rs = Ap->k_rs, k_hs = Ap->k_hs, v_rs = Ap->v_rs, v_hs = Ap->v_hs;
    const uint8_t * kc = Ap->k_cache, * vc = Ap->v_cache;
    const uint16_t * mrow = Ap->mask;
    float * ws = Ap->ws; unsigned int * counters = Ap->counters; float * dst = Ap->dst;
    const int n_items = n_tiles * n_splits;
    if ((int)blockIdx.x >= n_items) return;
    const int kcell = (int)__ldcg(Ap->k_ids), vcell = (int)__ldcg(Ap->v_ids);
    rope_table(cs, __ldcg(Ap->pos), Ap->ff, rp, threadIdx.x, blockDim.x);
    __syncthreads();

    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int tile = item % n_tiles, split = item / n_tiles;
        const int h0 = tile * G, hk = h0 / gq;
        // this token's K (roped) and V for kv head hk, in cache format, staged in shared memory; one item per kv head
        // also writes them to the cache cell (llama-kv-cache-unified.cpp:1103-1160 cpy_k / cpy_v as SET_ROWS)
        if (warp < 2) {
            const int e = lane * 8; const bool act = e < D;
            float a[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
            const bool storer = split == 0 && (h0 % gq) == 0;
            if (warp == 0) {
                if (act) load_roped8(Ap->k + (int64_t)hk * D, e, cs, rp, a);
                store8(newk, KVT, e, a, lane, act);
                if (storer) store8((uint8_t *)kc + (int64_t)kcell * k_rs + (int64_t)hk * k_hs, KVT, e, a, lane, act);
            } else {
                if (act) { const float4 x = __ldcg((const float4 *)(Ap->v + (int64_t)hk * D + e)), y = __ldcg((const float4 *)(Ap->v + (int64_t)hk * D + e + 4));
                           a[0] = x.x; a[1] = x.y; a[2] = x.z; a[3] = x.w; a[4] = y.x; a[5] = y.y; a[6] = y.z; a[7] = y.w; }
                store8(newv, KVT, e, a, lane, act);
                if (storer) store8((uint8_t *)vc + (int64_t)vcell * v_rs + (int64_t)hk * v_hs, KVT, e, a, lane, act);
            }
        }
        // query slices, roped on the fly (and written back once: the graph declares the roped Q as an output)
        float qf[G][8]; int qi[G][2]; float qd[G]; float slope[G];
#pragma unroll
        for (int g = 0; g < G; g++) {
            const int h = h0 + g;
            float v[8];
            load_roped8(Ap->q_src + (int64_t)h * D, dl * 8, cs, rp, v);
            if (split == 0 && warp == 0 && sg == 0) {
                *(float4 *)(Ap->q_dst + (int64_t)h * D + dl * 8)     = make_float4(v[0], v[1], v[2], v[3]);
                *(float4 *)(Ap->q_dst + (int64_t)h * D + dl * 8 + 4) = make_float4(v[4], v[5], v[6], v[7]);
            }
            if (KVT == B200_TYPE_F16) {
#pragma unroll
                for (int e = 0; e < 8; e++) qf[g][e] = __half2float(__float2half_rn(v[e]));
                qi[g][0] = qi[g][1] = 0; qd[g] = 0.0f;
            } else {
                float am = 0.0f;
#pragma unroll
                for (int e = 0; e < 8; e++) am = fmaxf(am, fabsf(v[e]));
                am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 1));
                am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 2));
                const float id = am != 0.0f ? __fdiv_rn(127.0f, am) : 0.0f;
                int t[8];
#pragma unroll
                for (int e = 0; e < 8; e++) t[e] = __float2int_rn(__fmul_rn(v[e], id)) & 0xff;
                qi[g][0] = t[0] | (t[1] << 8) | (t[2] << 16) | (t[3] << 24);
                qi[g][1] = t[4] | (t[5] << 8) | (t[6] << 16) | (t[7] << 24);
                qd[g] = __half2float(__float2half_rn(__fdiv_rn(am, 127.0f)));
#pragma unroll
                for (int e = 0; e < 8; e++) qf[g][e] = 0.0f;
            }
            slope[g] = max_bias > 0.0f ? (h < Ap->nh_log2 ? powf(Ap->m0, (float)(h + 1)) : powf(Ap->m1, (float)(2 * (h - Ap->nh_log2) + 1))) : 1.0f;
        }
        __syncthreads();                                            // newk / newv staged

        float M[G], L[G], acc[G][8];
#pragma unroll
        for (int g = 0; g < G; g++) { M[g] = -INFINITY; L[g] = 0.0f;
#pragma unroll
            for (int e = 0; e < 8; e++) acc[g][e] = 0.0f; }
        const unsigned gmask = (LP == 32 ? 0xffffffffu : ((1u << LP) - 1u)) << (sg * LP);
        const int p_begin = split * split_len;
        const int p_end   = min(n_kv, p_begin + split_len);
        // positions are visited in chunks of MAXIT per lane group: all loads of a chunk (mask, K, V) are issued before any
        // arithmetic, so a chunk costs ONE memory round trip (the phase sits on the token's critical path, and under full
        // weight streaming a DRAM round trip is several microseconds).  K/V of masked positions are loaded but never used.
        constexpr int MAXIT = 4;
        const int pstride = nw * PPW;
        for (int base = p_begin + warp * PPW + sg; base < p_end; base += pstride * MAXIT) {
            float mraw[MAXIT]; uint4 kraw[MAXIT], vraw[MAXIT]; float kdv[MAXIT], vdv[MAXIT];
#pragma unroll
            for (int it = 0; it < MAXIT; it++) {
                const int p = base + it * pstride;
                mraw[it] = -INFINITY; kraw[it] = make_uint4(0, 0, 0, 0); vraw[it] = kraw[it]; kdv[it] = 0.0f; vdv[it] = 0.0f;
                if (p < p_end) {
                    mraw[it] = mrow ? h2f(__ldg(mrow + p)) : 0.0f;
                    const uint8_t * krow = p == kcell ? newk : kc + (int64_t)p * k_rs + (int64_t)hk * k_hs;
                    const uint8_t * vrow = p == vcell ? newv : vc + (int64_t)p * v_rs + (int64_t)hk * v_hs;
                    if (KVT == B200_TYPE_F16) {
                        kraw[it] = p == kcell ? *(const uint4 *)(krow + dl * 16) : ldg_stream16(krow + dl * 16);
                        vraw[it] = p == vcell ? *(const uint4 *)(vrow + dl * 16) : ldg_stream16(vrow + dl * 16);
                    } else {
                        int q2[2];
                        load_q80_8(krow, dl, q2, kdv[it]); kraw[it].x = (uint32_t)q2[0]; kraw[it].y = (uint32_t)q2[1];
                        load_q80_8(vrow, dl, q2, vdv[it]); vraw[it].x = (uint32_t)q2[0]; vraw[it].y = (uint32_t)q2[1];
                    }
                }
            }
#pragma unroll
            for (int it = 0; it < MAXIT; it++) {
                if (mraw[it] == -INFINITY && max_bias <= 0.0f) continue;            // masked or beyond the split (uniform inside the lane group)
                if (base + it * pstride >= p_end) continue;
                float kf[8], vf[8];
                if (KVT == B200_TYPE_F16) {
                    unpack_h8(kraw[it], kf);
                    unpack_h8(vraw[it], vf);
                } else {
#pragma unroll
                    for (int e = 0; e < 8; e++) vf[e] = __fmul_rn((float)(int8_t)(((e < 4 ? vraw[it].x : vraw[it].y) >> (8 * (e & 3))) & 0xff), vdv[it]);
                }
                float s[G];
#pragma unroll
                for (int g = 0; g < G; g++) {
                    if (KVT == B200_TYPE_F16) {
                        float a = 0.0f;
#pragma unroll
                        for (int e = 0; e < 8; e++) a = fmaf(kf[e], qf[g][e], a);
#pragma unroll
                        for (int o = LP / 2; o > 0; o >>= 1) a += __shfl_xor_sync(gmask, a, o, LP);
                        s[g] = a;
                    } else {
                        int is = dp4a_s((int)kraw[it].x, qi[g][0], 0);
                        is = dp4a_s((int)kraw[it].y, qi[g][1], is);
                        is += __shfl_xor_sync(gmask, is, 1, LP);
                        is += __shfl_xor_sync(gmask, is, 2, LP);
                        float a = __fmul_rn((float)is, __fmul_rn(kdv[it], qd[g]));      // ggml-cpu/quants.c:305-333
                        a = (dl & 3) == 0 ? a : 0.0f;
#pragma unroll
                        for (int o = LP / 2; o >= 4; o >>= 1) a += __shfl_xor_sync(gmask, a, o, LP);
                        s[g] = __shfl_sync(gmask, a, 0, LP);
                    }
                }
#pragma unroll
                for (int g = 0; g < G; g++) {
                    float sv = s[g] * scale;
                    if (softcap != 0.0f) sv = softcap * tanhf(sv);
                    sv += slope[g] * mraw[it];
                    if (sv == -INFINITY) continue;
                    float ms = 1.0f, vs = 1.0f;
                    if (sv > M[g]) { ms = expf(M[g] - sv); M[g] = sv;
#pragma unroll
                        for (int e = 0; e < 8; e++) acc[g][e] *= ms;
                    } else vs = expf(sv - M[g]);
#pragma unroll
                    for (int e = 0; e < 8; e++) acc[g][e] = fmaf(vf[e], vs, acc[g][e]);
                    L[g] = L[g] * ms + vs;
                }
            }
        }
        // merge the position groups of the warp, then the warps
#pragma unroll
        for (int g = 0; g < G; g++) {
#pragma unroll
            for (int o = LP; o < 32; o <<= 1) {
                const float Mo = __shfl_xor_sync(0xffffffffu, M[g], o), Lo = __shfl_xor_sync(0xffffffffu, L[g], o);
                const float Mn = fmaxf(M[g], Mo);
                const float sa = M[g] == -INFINITY ? 0.0f : expf(M[g] - Mn), sb = Mo == -INFINITY ? 0.0f : expf(Mo - Mn);
#pragma unroll
                for (int e = 0; e < 8; e++) { const float ao = __shfl_xor_sync(0xffffffffu, acc[g][e], o); acc[g][e] = acc[g][e] * sa + ao * sb; }
                L[g] = L[g] * sa + Lo * sb; M[g] = Mn;
            }
            if (sg == 0) {
#pragma unroll
                for (int e = 0; e < 8; e++) sA[(warp * G + g) * D + dl * 8 + e] = acc[g][e];
                if (dl == 0) { sM[warp * G + g] = M[g]; sL[warp * G + g] = L[g]; }
            }
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < G * D; idx += nw * 32) {
            const int g = idx / D, e = idx % D;
            float Mn = -INFINITY;
            for (int w = 0; w < nw; w++) Mn = fmaxf(Mn, sM[w * G + g]);
            float a = 0.0f, l = 0.0f;
            for (int w = 0; w < nw; w++) {
                const float sc = sM[w * G + g] == -INFINITY ? 0.0f : expf(sM[w * G + g] - Mn);
                a += sA[(w * G + g) * D + e] * sc; l += sL[w * G + g] * sc;
            }
            const int h = h0 + g;
            if (n_splits == 1) {
                dst[(int64_t)h * D + e] = a * (1.0f / l);                        // ops.cpp:8390-8392
            } else {
                float * wp = ws + ((int64_t)split * n_head + h) * (D + 2);
                wp[e] = a;
                if (e == 0) { wp[D] = Mn; wp[D + 1] = l; }
            }
        }
        if (n_splits > 1) {
            // the last item of this head tile to finish merges all splits (fattn-common.cuh:645-701 as an epilogue)
            __threadfence();
            __syncthreads();
            if (threadIdx.x == 0) {
                const unsigned int prev = atomicAdd(&counters[tile], 1u);
                *s_last = prev == (unsigned int)(n_splits - 1);
                if (*s_last) counters[tile] = 0;
            }
            __syncthreads();
            if (*s_last) {
                __threadfence();
                float * s_l = sA;                                   // [n_splits][G] partial sums (the merge buffer is free now)
                for (int idx = threadIdx.x; idx < n_splits * G; idx += nw * 32) {
                    const int sp = idx / G, g = idx % G;
                    const float2 ml = __ldcg((const float2 *)(ws + ((int64_t)sp * n_head + h0 + g) * (D + 2) + D));   // all (m, l) pairs in one round trip
                    s_sc[sp * G + g] = ml.x; s_l[sp * G + g] = ml.y;
                }
                __syncthreads();
                if (threadIdx.x < G) {
                    const int g = threadIdx.x;
                    float Mn = -INFINITY;
                    for (int sp = 0; sp < n_splits; sp++) Mn = fmaxf(Mn, s_sc[sp * G + g]);
                    float l = 0.0f;
                    for (int sp = 0; sp < n_splits; sp++) {
                        const float m = s_sc[sp * G + g];
                        const float sc = m == -INFINITY ? 0.0f : expf(m - Mn);
                        l += s_l[sp * G + g] * sc;
                        s_sc[sp * G + g] = sc;
                    }
                    s_inv[g] = 1.0f / l;
                }
                __syncthreads();
                for (int idx = threadIdx.x; idx < G * D; idx += nw * 32) {
                    const int g = idx / D, e = idx % D;
                    const int row = h0 + g;
                    float a = 0.0f;
#pragma unroll 8
                    for (int sp = 0; sp < n_splits; sp++) a = fmaf(__ldcg(ws + ((int64_t)sp * n_head + row) * (D + 2) + e), s_sc[sp * G + g], a);
                    dst[(int64_t)row * D + e] = a * s_inv[g];
                }
            }
        }
        __syncthreads();                                            // scratch is reused by the next item
    }
}

template <int D, int KVT>
__device__ __forceinline__ void mk_attn_g(const MkAttn * A, uint8_t * scr, int nw) {
    const int gq = A->n_head / A->n_head_kv;
#ifdef MK_SLIM        // experiment: only the Llama-3-8B variant (code-size / instruction-cache study)
    mk_attn<D, KVT, 4>(A, scr, nw);
#else
    if (gq % 4 == 0) mk_attn<D, KVT, 4>(A, scr, nw);
    else if (gq % 2 == 0) mk_attn<D, KVT, 2>(A, scr, nw);
    else mk_attn<D, KVT, 1>(A, scr, nw);
#endif
}

__global__ void __launch_bounds__(MK_MAX_WARPS * 32, 1) mk_kernel(const MkPhase * __restrict__ prog, int n_phases, unsigned long long * sync, unsigned long long * trace, int tune) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[MK_MAX_WARPS][2];
    __shared__ PCache tab[MK_TAB];
    __shared__ volatile int tab_phase[MK_TAB];
    __shared__ double red[MK_MAX_WARPS];
    __shared__ unsigned int wstats[4];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    uint8_t * act  = smem;
    uint8_t * ring = smem + MK_AREG_BYTES + (size_t)warp * 2 * MK_SLOT_BYTES;
    if (lane == 0) { mbar_init(&full_bar[warp][0], 1); mbar_init(&full_bar[warp][1], 1); }
    mbar_fence_init();
    __syncthreads();

    // phase table: entries 0..2 now; entry p + 3 is fetched at the start of phase p and finished at its end (last warp)
    if (tid < MK_TAB) tab_phase[tid] = -1;
    __syncthreads();
    if (warp < 3 && warp < n_phases) { mk_plan_begin(prog, warp, tab, lane); mk_plan_finish(warp, tab, tab_phase, lane); }
    __syncthreads();
    // issue cursor: runs up to two ring slots ahead of consumption, across phase boundaries (weights do not depend on activations)
    Cur ic; ic.p = 0; ic.g = 0; ic.s = 0; ic.entered = 0;
    int ncons = 0, nissued = 0;
    const bool xphase = !(tune & 16);
    if (xphase) mk_pump(ic, nissued, ncons, n_phases, n_phases, tab, tab_phase, ring, full_bar[warp], warp, lane, nw);
    for (int p = 0; p < n_phases; p++) {
        if (trace && tid == 0) { trace[((size_t)blockIdx.x * n_phases + p) * 4 + 0] = gtimer(); wstats[0] = wstats[1] = wstats[2] = wstats[3] = 0; }
        if (p > 0) grid_wait(sync, (unsigned long long)p * gridDim.x);
        if (trace && tid == 0) trace[((size_t)blockIdx.x * n_phases + p) * 4 + 1] = gtimer();
        const int plimit = xphase ? n_phases : p;
        const PCache * cpc = &tab[p % MK_TAB];
        // first this warp's own refills (phases up to p + 2 are planned)
        mk_pump(ic, nissued, ncons, plimit, n_phases, tab, tab_phase, ring, full_bar[warp], warp, lane, nw);
        const bool planner = warp == nw - 1 && p + 3 < n_phases;
        if (planner) mk_plan_begin(prog, p + 3, tab, lane);
        // the KV rows the NEXT phase (attention) will read: each CTA warms its share of the range in L2 now, one phase early
        if (warp == nw - 2 && lane < 2 && p + 1 < n_phases && cpc->ph.kind == MK_MMV && tab_phase[(p + 1) % MK_TAB] == p + 1 && tab[(p + 1) % MK_TAB].ph.kind == MK_ATTN) {
            const MkAttn * An = &tab[(p + 1) % MK_TAB].ph.attn;
            const int64_t rs = lane == 0 ? An->k_rs : An->v_rs;
            const uint8_t * base = lane == 0 ? An->k_cache : An->v_cache;
            const int64_t total = (int64_t)An->n_kv * rs;
            const int64_t share = ((total + gridDim.x - 1) / gridDim.x + 15) & ~(int64_t)15;
            const int64_t lo = share * blockIdx.x;
            if (lo < total && (((uintptr_t)base | (uintptr_t)rs) & 15) == 0) {
                int64_t n = total - lo < share ? total - lo : share;
                n &= ~(int64_t)15;
                if (n > 0) bulk_prefetch_l2(base + lo, (uint32_t)n);
            }
        }
        if (cpc->ph.kind == MK_MMV) {
            mk_build_act(&cpc->ph.mmv, act, red, warp, lane, nw);
            if (trace && tid == 0) trace[((size_t)blockIdx.x * n_phases + p) * 4 + 2] = gtimer();
            mk_mmv_phase(n_phases, p, act, ring, full_bar[warp], tab, tab_phase, ic, ncons, nissued, plimit, warp, lane, nw, trace ? wstats : nullptr);
        } else {
            if (trace && tid == 0) trace[((size_t)blockIdx.x * n_phases + p) * 4 + 2] = gtimer();
            const MkAttn * A = &cpc->ph.attn;                     // shared-memory copy
#ifdef MK_SLIM
            mk_attn_g<128, B200_TYPE_F16>(A, act, nw);
#else
            if (A->hd == 128) { if (A->kv_type == B200_TYPE_F16) mk_attn_g<128, B200_TYPE_F16>(A, act, nw); else mk_attn_g<128, B200_TYPE_Q8_0>(A, act, nw); }
            else              { if (A->kv_type == B200_TYPE_F16) mk_attn_g<64,  B200_TYPE_F16>(A, act, nw); else mk_attn_g<64,  B200_TYPE_Q8_0>(A, act, nw); }
#endif
        }
        if (planner) mk_plan_finish(p + 3, tab, tab_phase, lane);
        if (trace) { __syncthreads(); if (tid == 0) { trace[((size_t)blockIdx.x * n_phases + p) * 4 + 3] = gtimer();
            unsigned long long * ext = trace + (size_t)gridDim.x * 512 * 4 + ((size_t)blockIdx.x * n_phases + p) * 4;
            ext[0] = wstats[0]; ext[1] = wstats[1]; ext[2] = wstats[2]; ext[3] = wstats[3]; } }
        if (p + 1 < n_phases) grid_arrive(sync);
    }
    // the last CTA out resets the barrier for the next launch
    if (tid == 0) {
        const unsigned long long prev = atomicAdd(sync + 1, 1ULL);
        if (prev == (unsigned long long)gridDim.x - 1) { sync[0] = 0; sync[1] = 0; __threadfence(); }
    }
}

} // namespace

int mk_phase_ok_k(int64_t k, int act_source) {
    // rms_norm phases keep their block in registers: one 256-element block per 8-lane group
    return k > 0 && k % 2048 == 0 && mk_act_bytes(k) <= MK_AREG_BYTES && (act_source != 2 || k <= (int64_t)4 * MK_MAX_WARPS * 256);
}

// GGML_B200_MK_TRACE=1: per-phase timestamps of every CTA of the most recent launch, printed by b200_mk_trace_dump()
static unsigned long long * g_trace = nullptr; static int g_trace_phases = 0; static std::vector<int> g_trace_kinds;
static const size_t TRACE_MAX_PHASES = 512;

int mk_launch(const MkPhase * dev_prog, int n_phases, unsigned long long * dev_sync, void * stream) {
    if (!dev_prog || n_phases <= 0 || !dev_sync) { b200_set_error("mk_launch: bad arguments"); return B200_ERR_INVALID; }
    const size_t smem = MK_AREG_BYTES + (size_t)MK_MAX_WARPS * 2 * MK_SLOT_BYTES;
    static bool attr[64] = { false };                   // the opt-in is per device (single-process --tensor-split uses several)
    int dev = 0; cudaGetDevice(&dev);
    static const bool want_trace = getenv("GGML_B200_MK_TRACE") != nullptr;
    if (!attr[dev & 63]) { B200_CUDA(cudaFuncSetAttribute(mk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr[dev & 63] = true; }
    unsigned long long * trace = nullptr;
    if (want_trace && (size_t)n_phases <= TRACE_MAX_PHASES && n_phases >= 8) {
        if (!g_trace) B200_CUDA(cudaMalloc((void **)&g_trace, (size_t)b200_sm_count() * TRACE_MAX_PHASES * 4 * 8 * 2));
        trace = g_trace; g_trace_phases = n_phases;
    }
    static const int tune = getenv("GGML_B200_MK_TUNE") ? atoi(getenv("GGML_B200_MK_TUNE")) : MK_TUNE_DEFAULT;
    mk_kernel<<<(unsigned)b200_sm_count(), MK_MAX_WARPS * 32, smem, (cudaStream_t)stream>>>(dev_prog, n_phases, dev_sync, trace, tune);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" __attribute__((visibility("default"))) void b200_mk_trace_dump(const MkPhase * dev_prog_or_null) {
    (void)dev_prog_or_null;
    if (!g_trace || g_trace_phases <= 0) { fprintf(stderr, "mk trace: nothing recorded (set GGML_B200_MK_TRACE=1)\n"); return; }
    cudaDeviceSynchronize();
    const int G = b200_sm_count(), P = g_trace_phases;
    std::vector<unsigned long long> t((size_t)G * P * 4), x((size_t)G * P * 4);
    cudaMemcpy(t.data(), g_trace, t.size() * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(x.data(), g_trace + (size_t)G * 512 * 4, x.size() * 8, cudaMemcpyDeviceToHost);
    const unsigned long long t0 = t[0];
    const bool verbose = atoi(getenv("GGML_B200_MK_TRACE")) > 1;
    const int period = getenv("GGML_B200_MK_TRACE_PERIOD") ? atoi(getenv("GGML_B200_MK_TRACE_PERIOD")) : 5;
    std::vector<double> agg((size_t)period * 6, 0.0), sagg((size_t)period * 4, 0.0); std::vector<int> cnt(period, 0);
    double t_end = 0;
    for (int p = 0; p < P; p++) {
        double wmin = 1e30, wmax = 0, cmin = 1e30, cmax = 0, csum = 0, first = 1e30, last = 0;
        for (int b = 0; b < G; b++) {
            const unsigned long long * r = &t[((size_t)b * P + p) * 4];
            const double w = (r[1] - r[0]) * 1e-3, c = (r[3] - r[1]) * 1e-3;
            wmin = w < wmin ? w : wmin; wmax = w > wmax ? w : wmax; cmin = c < cmin ? c : cmin; cmax = c > cmax ? c : cmax; csum += c;
            const double s0 = (r[1] - t0) * 1e-3, e = (r[3] - t0) * 1e-3; first = s0 < first ? s0 : first; last = e > last ? e : last;
        }
        const unsigned long long * r0 = &t[(size_t)p * 4];
        const double actb = (r0[2] - r0[1]) * 1e-3;
        if (verbose) fprintf(stderr, "  phase %3d  start %8.1f  wait %5.1f/%5.1f  act %5.1f  compute %5.1f/%5.1f/%5.1f  end(all) %8.1f\n", p, first, wmin, wmax, actb, cmin, csum / G, cmax, last);
        if (p >= period && p < P - period) { double * a = &agg[(size_t)(p % period) * 6]; a[0] += wmin; a[1] += wmax; a[2] += actb; a[3] += cmin; a[4] += csum / G; a[5] += cmax; cnt[p % period]++; }
        t_end = last;
        if (p >= period && p < P - period) for (int b = 0; b < G; b++) for (int q = 0; q < 4; q++) sagg[(size_t)(p % period) * 4 + q] += (double)x[((size_t)b * P + p) * 4 + q];
    }
    fprintf(stderr, "mk trace: %d phases, %d CTAs, %.1f us total; mean per phase slot (p %% %d): barrier wait min/max | act build (CTA0) | phase time min/avg/max\n", P, G, t_end, period);
    for (int q = 0; q < period; q++) if (cnt[q]) {
        const double * a = &agg[(size_t)q * 6]; const double n = cnt[q];
        const double * sg = &sagg[(size_t)q * 4]; const double ns = sg[3] > 0 ? sg[3] : 1;
        fprintf(stderr, "  slot %d: wait %5.1f/%5.1f  act %5.1f  time %5.1f/%5.1f/%5.1f | per ring slot (cycles): data wait %7.0f  dot %6.0f  refill %6.0f  (%.1f slots per SM)\n", q, a[0] / n, a[1] / n, a[2] / n, a[3] / n, a[4] / n, a[5] / n,
                sg[0] / ns, sg[1] / ns, sg[2] / ns, sg[3] / n / G);
    }
}
