"""GPU: the persistent matrix kernels where a worker takes more than one unit of work.

The decode matvec (csrc/mmvq.cu) runs one CTA of 16 warps per SM; warp w of CTA c owns the units g = w * grid + c, g + 16 * grid, ...
and carries its issue cursor, ring slots, mbarrier phases and K-parts from one unit to the next, across matrix boundaries in a multi-matrix
launch.  The tensor-core GEMMs (csrc/mmq_tc.cu, csrc/mmq_tc32.cu, and their GROUPED instances behind b200_mul_mat_id2) run
min(tiles, SMs) CTAs, each looping tile += gridDim.x and carrying the stage counter, the scale / D8 / imin rings, the next tile's first
super-block prefetch and the partial-tile guards from one tile to the next.  Every case here gives every worker at least two units (computed
from the device's SM count and the launch geometry, and scaled up on a larger device), starts its outputs as NaN, uses strides wider than
the data with a sentinel in the padding, runs twice for the same bits, and compares with the C oracle."""
import ctypes as C
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from refutil import (BLOCK_BYTES, BLOCK_ELEMS, Q4_0, Q4_K, Q5_0, Q5_K, Q6_K, Q8_0, nmse, oracle, orc_mul_mat, ptr, rand_blocks,
                     repack_rows_np, row_bytes)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENT = np.float32(-31337.0)      # padding [m, ldd) of every output column; no kernel may touch it
MMV_WARPS = 16                   # mmvq.cu: one CTA of 16 warps per SM
TILE = 128                       # mmq_tc.cu / mmq_tc32.cu: 128 x 128 output tiles
MIN_UNITS = 2

_KEEP = []          # device tensors stay alive until the test ends (raw pointers are passed to C)


@pytest.fixture(autouse=True)
def _keep_alive():
    yield
    torch.cuda.synchronize()
    _KEEP.clear()


def dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    _KEEP.append(t)
    return t


def load_ops():
    from conftest import load_pkg
    return load_pkg().ops


def sm_count(b200):
    return int(b200.lib.b200_device_sm_count(0))


def seeded(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def padded_out(n, m, ldd):
    """f32 [n][ldd]: NaN where the kernel must write, SENT in the padding of every column"""
    d = torch.full((n, ldd), float("nan"), dtype=torch.float32, device="cuda")
    d[:, m:] = float(SENT)
    _KEEP.append(d)
    return d


def strided_x(x, xs):
    """device copy of x [n][k] with column stride xs > k; the padding is NaN, so a read past k poisons the result"""
    n, k = x.shape
    h = np.full((n, xs), np.nan, np.float32)
    h[:, :k] = x
    return dev(h)


def check_padding(got, m):
    pad = got[:, m:]
    assert (pad.view(np.uint32) == SENT.view(np.uint32)).all(), "a store landed in the padding [m, ldd) of a column"


def check_close(got, want, bound=2e-5):
    assert np.isfinite(got).all(), "outputs left unwritten (NaN) or non-finite"
    scale = float(np.abs(want).max())
    err = float(np.abs(got - want).max())
    assert err <= bound * scale, (err, scale, np.unravel_index(np.argmax(np.abs(got - want)), got.shape))
    assert nmse(got, want) < 1e-10, nmse(got, want)


def weights_dev(b200, t, W):
    """device copy of ggml weight rows (+64 bytes slack), repacked in place for the kernels"""
    k = W.shape[1] // BLOCK_BYTES[t] * BLOCK_ELEMS[t]
    d = dev(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)]))
    b200.check(b200.lib.b200_repack_rows(t, b200.p(d), W.shape[0], k, b200.stream()))
    return d


# ====================================================================== 1. decode matvec
def mmv_plan(b200, mats, k, ncols, swiglu, sms, smem_kb=216, grid_mult=1, r1=0):
    """the planner of mmv_launch (mmvq.cu) restated: unit = R rows x G segments of segc 32-element chunks, `stages` ring slots per warp,
    P = ceil(nseg / G) K-parts per unit, grid = min(ceil(units / 16), SMs * grid_mult) CTAs.  Returns None for the column-halves split
    (no ring fits even one slot per warp); B200_MMV_SMEM_KB / B200_MMV_GRID_MULT / B200_MMV_R1 are smem_kb / grid_mult / r1."""
    L = b200.lib
    nchunks = k // 32
    segc = next((c for c in range(64, 7, -8) if nchunks % c == 0), 8)
    nseg = nchunks // segc
    act = sum(ncols * L.b200_act_col_bytes(kd, k) for kd in sorted({L.b200_act_kind_for(t) for t, _ in mats}))
    act_al = (act + 127) & ~127
    segb = max((k // BLOCK_ELEMS[t] * BLOCK_BYTES[t]) // nseg for t, _ in mats)
    budget = smem_kb * 1024

    def try_cfg(r, want):
        for g in range(nseg, 0, -1):
            slot = (r * g * segb + 255) & ~255
            room = (budget - act_al) // (MMV_WARPS * slot) if budget > act_al else 0
            if room >= want:
                return r, g, room
        return None

    units2, rows1 = sum((m + 1) // 2 for _, m in mats), sum(m for _, m in mats)
    wn = sms * MMV_WARPS
    t2, t1 = 2.0 * (-(-units2 // wn)), 1.15 * (-(-rows1 // wn))
    cfg = None
    if not swiglu and r1 == 1 and ncols == 1 and t1 < t2:
        cfg = try_cfg(1, 2)
    for r, want in ((2, 2), (1, 2), (2, 1), (1, 1)):
        if cfg is None and (r == 2 or not swiglu):
            cfg = try_cfg(r, want)
    if cfg is None:
        return None
    R, G, stages = cfg
    row_stride = (G * segb + 127) & ~127
    slot = (R * G * segb + 255) & ~255
    if slot < 2 * row_stride and R == 2:
        slot = 2 * row_stride
    stages = min(stages, (budget - act_al) // (MMV_WARPS * slot), 8)
    units = mats[0][1] if swiglu else sum(-(-m // R) for _, m in mats)
    grid = max(1, min(-(-units // MMV_WARPS), sms * grid_mult))
    return dict(R=R, G=G, P=-(-nseg // G), stages=int(stages), units=int(units), grid=int(grid), per_warp=units / (grid * MMV_WARPS))


def mmv_geometry(b200, mats, k, ncols, swiglu, sms, knobs):
    """plan(s) of the launch and the fewest units any warp gets: every warp of the grid gets floor(units / warps) or one more"""
    kw = dict(smem_kb=int(knobs.get("B200_MMV_SMEM_KB", 216)), grid_mult=int(knobs.get("B200_MMV_GRID_MULT", 1)), r1=int(knobs.get("B200_MMV_R1", 0)))
    plan = mmv_plan(b200, mats, k, ncols, swiglu, sms, **kw)
    if plan is not None:
        return [plan], plan["units"] // (plan["grid"] * MMV_WARPS)
    halves = [mmv_plan(b200, mats, k, h, swiglu, sms, **kw) for h in (ncols // 2, ncols - ncols // 2)]
    assert all(h is not None for h in halves)
    return halves, min(h["units"] // (h["grid"] * MMV_WARPS) for h in halves)


# name -> spec.  api: "vec_q" (b200_mul_mat_vec_q, act buffers), "multi" (b200_mul_mat_vec_q_multi), "swiglu" (b200_mul_mat_vec_q_swiglu),
# "launch" (b200_mul_mat_vec_q_launch; src 0 = act buffers, 1 = f32 x quantised in the kernel, 2 = rms_norm * w first).  A launch with
# one column and src 1 / 2 runs the lean instances, which is what decode runs.  `grow`: the rows of every matrix are multiplied by the
# smallest factor that gives each warp at least two units on this device (4096-row ffn_down: 2048 pairs on 2112 warps is less than one).
MMV_CASES = {
    # Llama-3-8B ffn_up / ffn_gate (7168 pairs: 3.4 per warp on 132 SMs)
    "q4K_ffn_up_n1":      dict(mats=[(Q4_K, 14336)], k=4096, n=1, api="vec_q"),
    "q4K_ffn_up_n1_lean": dict(mats=[(Q4_K, 14336)], k=4096, n=1, api="launch", src=1),
    "q4K_ffn_up_n8":      dict(mats=[(Q4_K, 14336)], k=4096, n=8, api="vec_q"),
    "q40_ffn_up_n1_lean": dict(mats=[(Q4_0, 14336)], k=4096, n=1, api="launch", src=1),
    "q40_ffn_up_n8":      dict(mats=[(Q4_0, 14336)], k=4096, n=8, api="launch", src=0),
    # ffn_down: k = 14336 does not fit two ring slots of a whole row pair per warp: G = 1 segment of 7, P = 7 K-parts per unit
    "q6K_ffn_down_n1":    dict(mats=[(Q6_K, 4096)], k=14336, n=1, api="launch", src=1, grow=True),
    "q6K_ffn_down_n5":    dict(mats=[(Q6_K, 4096)], k=14336, n=5, api="vec_q", grow=True),
    # a Q6_K lm_head of Llama-3 (128256 rows: 30 pairs per warp) behind the fused rms_norm
    "q6K_lm_head_norm":   dict(mats=[(Q6_K, 128256)], k=4096, n=1, api="launch", src=2),
    # TinyLlama's vocab at Q8_0
    "q80_vocab_n1":       dict(mats=[(Q8_0, 32000)], k=2048, n=1, api="launch", src=1),
    "q80_vocab_n4":       dict(mats=[(Q8_0, 32000)], k=2048, n=4, api="vec_q"),
    # an odd row count: the last pair has one row (and the lean instances, which need even m, are not taken)
    "q4K_odd_n1":         dict(mats=[(Q4_K, 14335)], k=4096, n=1, api="launch", src=1),
    "q4K_odd_n3":         dict(mats=[(Q4_K, 14335)], k=4096, n=3, api="vec_q"),
    # fused QKV with mixed types, Qwen2-style bias, and a residual.  Llama-3-70B widths (q 8192, k / v 1024): the 8B's 4096 + 1024 + 1024
    # rows are 3072 pairs, 1.45 per warp on 132 SMs
    "qkv_mixed_n1":       dict(mats=[(Q4_K, 8192), (Q4_K, 1024), (Q6_K, 1024)], k=8192, n=1, api="launch", src=1, bias=True, resid=True, grow=True),
    "qkv_mixed_n3":       dict(mats=[(Q4_K, 8192), (Q4_K, 1024), (Q6_K, 1024)], k=8192, n=3, api="launch", src=0, bias=True, resid=True, grow=True),
    "qkv_mixed_multi":    dict(mats=[(Q4_K, 8192), (Q4_K, 1024), (Q6_K, 1024)], k=8192, n=1, api="multi", bias=True, grow=True),
    # gate + up + SwiGLU (one unit per output row: 14336 rows, 6.8 per warp)
    "swiglu_q4K_q4K":     dict(mats=[(Q4_K, 14336), (Q4_K, 14336)], k=4096, n=1, api="swiglu"),
    "swiglu_q4K_q4K_lean": dict(mats=[(Q4_K, 14336), (Q4_K, 14336)], k=4096, n=1, api="launch", src=1, swiglu=True),
    "swiglu_q4K_q6K":     dict(mats=[(Q4_K, 14336), (Q6_K, 14336)], k=4096, n=1, api="swiglu"),
    "swiglu_q4K_q6K_n3":  dict(mats=[(Q4_K, 14336), (Q6_K, 14336)], k=4096, n=3, api="launch", src=1, swiglu=True),
}


def grown(b200, spec, sms, knobs):
    """the spec's matrices, their rows scaled (when the spec allows it) until every warp gets MIN_UNITS units; asserts that it does"""
    f = 1
    while True:
        mats = [(t, m * f) for t, m in spec["mats"]]
        plans, least = mmv_geometry(b200, mats, spec["k"], spec["n"], spec.get("swiglu") or spec["api"] == "swiglu", sms, knobs)
        if least >= MIN_UNITS or not spec.get("grow"):
            break
        f += 1
    print(f"  SMs {sms}: rows {[m for _, m in mats]} k {spec['k']} n {spec['n']}: " +
          "; ".join(f"R {p['R']} G {p['G']} P {p['P']} stages {p['stages']} units {p['units']} grid {p['grid']} units/warp {p['per_warp']:.2f}"
                    for p in plans))
    assert least >= MIN_UNITS, (least, plans)
    return mats, plans


def run_mmv(b200, name, knobs=None):
    """one matvec case: returns what a child process reports (the plan and the kernel launches of one call)"""
    spec = MMV_CASES[name]
    knobs = knobs or {}
    sms = sm_count(b200)
    mats, plans = grown(b200, spec, sms, knobs)
    k, n, api, src = spec["k"], spec["n"], spec["api"], spec.get("src", 0)
    swiglu = api == "swiglu" or spec.get("swiglu", False)
    L = b200.lib
    rng = seeded(name, tuple(mats))
    Ws = [rand_blocks(rng, t, m, k) for t, m in mats]
    x = (rng.standard_normal((n, k)) * 2).astype(np.float32)
    norm_w = (1 + 0.1 * rng.standard_normal(k)).astype(np.float32) if src == 2 else None
    biases = [rng.standard_normal(m).astype(np.float32) if spec.get("bias") else None for _, m in mats]
    # output strides wider than the data.  The multi and SwiGLU entry points write with stride m: one column, padded by the allocation
    ldds = [m + 37 for _, m in mats]
    assert api in ("vec_q", "launch") or n == 1
    resids = [rng.standard_normal((n, ldd)).astype(np.float32) if spec.get("resid") else None for (_, m), ldd in zip(mats, ldds)]

    # oracle
    xin = x
    if src == 2:
        xin = np.zeros_like(x)
        oracle().orc_rms_norm(ptr(x), ptr(norm_w), ptr(xin), k, n, 1e-5)
    prods = [orc_mul_mat(t, W, xin, m, n, k) for (t, m), W in zip(mats, Ws)]
    if swiglu:
        want = np.zeros_like(prods[0])
        oracle().orc_swiglu(ptr(prods[0]), ptr(prods[1]), ptr(want), want.size)
        wants = [want]
    else:
        wants = []
        for (t, m), p, b, r in zip(mats, prods, biases, resids):
            w = p
            if b is not None:
                w = w + b[None, :]
            if r is not None:
                w = w + r[:, :m]
            wants.append(w)

    # device
    Wd = [weights_dev(b200, t, W) for (t, _), W in zip(mats, Ws)]
    xs = k + 12
    xd = strided_x(x, xs)
    acts = [None, None]
    if src == 0:
        for kd in sorted({L.b200_act_kind_for(t) for t, _ in mats}):
            a = torch.zeros(n * L.b200_act_col_bytes(kd, k), dtype=torch.uint8, device="cuda")
            _KEEP.append(a)
            b200.check(L.b200_quantize_act(kd, b200.p(xd), xs, b200.p(a), k, n, b200.stream()))
            acts[kd] = a
    bd = [dev(b) if b is not None else None for b in biases]
    rd = [dev(r) if r is not None else None for r in resids]
    nw = dev(norm_w) if norm_w is not None else None
    n_out = 1 if swiglu else len(mats)

    def launch(dsts):
        if api == "vec_q":
            t, m = mats[0]
            b200.check(L.b200_mul_mat_vec_q(t, b200.p(Wd[0]), b200.p(acts[L.b200_act_kind_for(t)]), b200.p(dsts[0]), ldds[0], b200.p(bd[0]),
                                            b200.p(rd[0]), m, k, n, b200.stream()))
        elif api == "multi":
            descs = (b200.MmvDesc * len(mats))()
            for i, (t, m) in enumerate(mats):
                descs[i].W = Wd[i].data_ptr(); descs[i].dst = dsts[i].data_ptr(); descs[i].m = m; descs[i].type = t
                descs[i].bias = bd[i].data_ptr() if bd[i] is not None else None
            b200.check(L.b200_mul_mat_vec_q_multi(descs, len(mats), b200.p(acts[0]), b200.p(acts[1]), k, n, b200.stream()))
        elif api == "swiglu":
            (tg, m), (tu, _) = mats
            b200.check(L.b200_mul_mat_vec_q_swiglu(tg, b200.p(Wd[0]), tu, b200.p(Wd[1]), b200.p(acts[0]), b200.p(acts[1]), b200.p(dsts[0]),
                                                   m, k, n, b200.stream()))
        else:
            d = b200.MmvLaunch()
            d.n_mats = len(mats); d.swiglu = int(swiglu); d.k = k; d.ncols = n; d.act_source = src; d.eps = 1e-5
            for i, (t, m) in enumerate(mats):
                d.mats[i].W = Wd[i].data_ptr(); d.mats[i].m = m; d.mats[i].type = t
                d.mats[i].dst = dsts[0 if swiglu else i].data_ptr()
                d.mats[i].bias = bd[i].data_ptr() if bd[i] is not None else None
                d.residual[i] = rd[i].data_ptr() if rd[i] is not None else None
                d.dst_col_stride[i] = ldds[0 if swiglu else i]
            if src == 0:
                d.act_q8K = acts[0].data_ptr() if acts[0] is not None else None
                d.act_q80 = acts[1].data_ptr() if acts[1] is not None else None
            else:
                d.x = xd.data_ptr(); d.x_col_stride = xs
                d.norm_w = nw.data_ptr() if nw is not None else None
            b200.check(L.b200_mul_mat_vec_q_launch(C.byref(d), b200.stream()))

    runs, launches = [], None
    for _ in range(2):
        dsts = [padded_out(n, mats[i][1], ldds[i]) for i in range(n_out)]
        torch.cuda.synchronize()
        n0 = L.b200_kernel_launches()
        launch(dsts)
        torch.cuda.synchronize()
        launches = int(L.b200_kernel_launches() - n0)
        runs.append([d.cpu().numpy() for d in dsts])
    for a, b in zip(*runs):
        assert a.tobytes() == b.tobytes(), "two runs differ"
    for i, (got, want) in enumerate(zip(runs[0], wants)):
        m = want.shape[1]
        check_padding(got, m)
        check_close(got[:, :m], want)
    return dict(plans=plans, launches=launches, sms=sms)


@pytest.mark.parametrize("name", list(MMV_CASES))
def test_matvec_many_units_per_warp(b200, name):
    """every row of a model-width matvec against the oracle; each warp walks at least two units"""
    o = run_mmv(b200, name)
    assert o["launches"] == 1, o


# ====================================================================== 2. the matvec planner's other branches
# Each case runs in a fresh process: mmv_launch reads its knobs once per process.  The branch each knob value reaches, by the planner's
# arithmetic (budget = B200_MMV_SMEM_KB * 1024 bytes for the activations and 16 warps' rings; segb = bytes of one 2048-element segment
# of the widest row; a slot is R * G * segb rounded up to 256 bytes):
#   * r1: B200_MMV_R1=1, one column, Llama-3-70B QKV (10240 rows, k 8192): pairs cost t2 = 2 * ceil(5120 / 2112) = 6, single rows
#     t1 = 1.15 * ceil(10240 / 2112) = 5.75 < 6, so units are single rows (R = 1; the lean single-row instance).
#   * one_stage: B200_MMV_SMEM_KB=41, Q4_K 14336 x 4096, one column: segb = 2304 / 2 = 1152; 41984 - 4736 (activations) = 37248 bytes
#     hold one slot of a pair (16 x 2304 = 36864) but not two (73728), nor two of a single row (2 x 16 x 1280 = 40960): R = 2, G = 1,
#     one stage, so every part waits on the slot it has just refilled (P = 2).
#   * g1: B200_MMV_SMEM_KB=100, same shape: 102400 - 4736 = 97664 bytes: two stages of whole pairs need 147456, of half pairs 73728:
#     R = 2, G = 1, P = 2 (the default plan is G = 2, P = 1).
#   * halves: B200_MMV_SMEM_KB=50, same shape, 8 columns: the activations (8 x 4672 = 37376 bytes) leave 13824, less than one single-row
#     slot per warp (16 x 1280 = 20480): two launches of 4 columns, each R = 1, one stage (51200 - 18688 = 32512 >= 20480).
#   * grid2: B200_MMV_GRID_MULT=2, TinyLlama's Q8_0 vocab (16000 pairs): 2 x SMs CTAs, more than fit on the device at once.
KNOB_CASES = {
    "r1":        ("qkv_mixed_n1", {"B200_MMV_R1": "1"}, dict(R=1), 1),
    "one_stage": ("q4K_ffn_up_n1_lean", {"B200_MMV_SMEM_KB": "41"}, dict(R=2, G=1, stages=1), 1),
    "g1":        ("q4K_ffn_up_n1", {"B200_MMV_SMEM_KB": "100"}, dict(R=2, G=1, P=2), 1),
    "halves":    ("q4K_ffn_up_n8", {"B200_MMV_SMEM_KB": "50"}, dict(R=1, stages=1), 2),
    "grid2":     ("q80_vocab_n1", {"B200_MMV_GRID_MULT": "2"}, dict(R=2), 1),
}

MMV_CHILD = r"""
import json, sys
sys.path.insert(0, %r)
import conftest, test_gpu_persistent as T
b = conftest.load_pkg().ops
o = T.run_mmv(b, %r, %r)
print(json.dumps(o))
"""


@pytest.mark.parametrize("case", list(KNOB_CASES))
def test_matvec_planner_branches(case):
    name, knobs, expect, launches = KNOB_CASES[case]
    env = dict(os.environ)
    for kk in ("B200_MMV_SMEM_KB", "B200_MMV_R1", "B200_MMV_GRID_MULT", "B200_MMV_NO_LEAN", "B200_MMV_PRIME_ALL"):
        env.pop(kk, None)
    env.update(knobs)
    r = subprocess.run([sys.executable, "-c", MMV_CHILD % (os.path.join(ROOT, "tests"), name, knobs)], capture_output=True, text=True,
                       env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip().splitlines()[0])
    o = json.loads(r.stdout.strip().splitlines()[-1])
    assert o["launches"] == launches and len(o["plans"]) == launches, o
    for p in o["plans"]:
        for kk, v in expect.items():
            assert p[kk] == v, (kk, p)
    if case == "grid2":
        assert o["plans"][0]["grid"] > o["sms"], o
    if case in ("one_stage", "g1"):
        assert o["plans"][0]["P"] > 1, o


# ====================================================================== 3. dense tensor-core GEMMs past one tile per SM
def gemm_tiles(m, n):
    return -(-m // TILE) * -(-n // TILE)


def gemm_n_for(m, n, sms):
    """n, grown by whole column tiles (the partial last one kept) until every CTA of min(tiles, SMs) gets MIN_UNITS tiles"""
    while gemm_tiles(m, n) < MIN_UNITS * sms:
        n += TILE
    return n


def windows(n):
    """column windows [c0, c1) of at most 128 columns and at least 49 (so the tile kernel takes them): aligned ones, then ones shifted by
    77 columns (the last one ends at n)"""
    out = [(c, min(c + TILE, n)) for c in range(0, n, TILE)]
    if out[-1][1] - out[-1][0] < 49:
        out[-1] = (n - TILE, n)
    out += [(c, c + TILE) for c in range(77, n - TILE + 1, TILE)]
    if out[-1][1] != n:
        out.append((n - TILE, n))
    return out


GEMM_CASES = [
    # K-quants: 1, 3 and 22 super-blocks (TinyLlama's ffn_down), so the 4-deep scale / D8 rings and the 2-deep imin slots do not restart
    # at slot 0 on a CTA's second tile; 4100 x 1100 = 33 x 9 tiles, both last tiles partial
    (Q4_K, 4100, 1100, 256, None), (Q4_K, 4100, 1100, 768, None), (Q4_K, 4100, 1100, 5632, None),
    (Q5_K, 4100, 1100, 256, None), (Q5_K, 4100, 1100, 768, None), (Q5_K, 4100, 1100, 5632, None),
    (Q6_K, 4100, 1100, 2048, None), (Q6_K, 4100, 1100, 4096, None),
    (Q4_K, 14336, 512, 5632, None),                     # 112 x 4 tiles
    (Q4_0, 4100, 1100, 256, None), (Q4_0, 4100, 1100, 768, None), (Q4_0, 4100, 1100, 5632, None),
    (Q5_0, 4100, 1100, 256, None), (Q5_0, 4100, 1100, 768, None), (Q5_0, 4100, 1100, 5632, None),
    (Q8_0, 4100, 1100, 256, None), (Q8_0, 4100, 1100, 768, None), (Q8_0, 4100, 1100, 5632, None),
    (Q8_0, 14336, 512, 4096, None),
    (Q8_0, 4100, 1100, None, 29568),                    # Qwen2-72B's ffn_down rows, padded to a multiple of 256
]


@pytest.mark.parametrize("t,m,n0,k,k_valid", GEMM_CASES)
def test_gemm_many_tiles_per_cta(b200, t, m, n0, k, k_valid):
    """a tile kernel launch with at least two tiles per CTA: bit for bit the same as launches of one column window each (at most one tile
    per CTA), over the whole output; and the oracle on the first and last column of every column tile and a few others"""
    L = b200.lib
    sms = sm_count(b200)
    n = gemm_n_for(m, n0, sms)
    kv = k_valid or k
    if k_valid:
        k = int(L.b200_padded_k(t, k_valid))
    tiles = gemm_tiles(m, n)
    print(f"  SMs {sms}: {m} x {n} x {kv}: {tiles} tiles on {min(tiles, sms)} CTAs, {tiles / min(tiles, sms):.2f} tiles per CTA")
    assert tiles // min(tiles, sms) >= MIN_UNITS
    assert -(-m // TILE) <= sms                                 # a 128-column window is at most one tile per CTA
    rng = seeded(t, m, n, kv)
    W = rand_blocks(rng, t, m, kv)
    x = rng.standard_normal((n, kv)).astype(np.float32)
    x[n // 3, :256] = 0.0                                       # an all-zero activation block (d = 0)
    if k_valid:
        src = dev(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)]))
        Wd = torch.zeros(m * row_bytes(t, k) + 64, dtype=torch.uint8, device="cuda")
        _KEEP.append(Wd)
        b200.check(L.b200_repack_rows_padded(t, b200.p(src), b200.p(Wd), m, kv, 0, b200.stream()))
    else:
        Wd = weights_dev(b200, t, W)
    xs, ldd = kv + 12, m + 29
    xd = strided_x(x, xs)

    def gemm(c0, c1):
        w = c1 - c0
        ws = torch.zeros(L.b200_mul_mat_q_workspace(t, m, k, w), dtype=torch.uint8, device="cuda")
        dst = padded_out(w, m, ldd)
        xp = C.c_void_p(xd.data_ptr() + 4 * c0 * xs)
        b200.check(L.b200_mul_mat_q2(t, b200.p(Wd), xp, xs, b200.p(dst), ldd, m, k, kv, w, b200.p(ws), b200.stream()))
        torch.cuda.synchronize()
        del ws
        return dst.cpu().numpy()

    big = gemm(0, n)
    assert big.tobytes() == gemm(0, n).tobytes(), "two runs differ"
    check_padding(big, m)
    assert np.isfinite(big[:, :m]).all(), "outputs left unwritten (NaN) or non-finite"
    for c0, c1 in windows(n):
        assert c1 - c0 >= 49 and gemm_tiles(m, c1 - c0) <= sms
        win = gemm(c0, c1)
        check_padding(win, m)
        assert win.tobytes() == big[c0:c1].tobytes(), f"columns [{c0}, {c1}) differ from the same columns of the launch of all {n}"
    nct = -(-n // TILE)
    cols = sorted(set([j * TILE for j in range(nct)] + [min(n, (j + 1) * TILE) - 1 for j in range(nct)] + list(rng.choice(n, 4, replace=False))))
    want = orc_mul_mat(t, W, x[cols], m, len(cols), kv)
    err = float(np.abs(big[cols, :m] - want).max() / np.abs(want).max())
    assert err <= 2e-5, err


# ====================================================================== 4. grouped MUL_MAT_ID past one tile per CTA
MMID_CASES = [
    # 8 experts of 4096 rows (32 row tiles), top-2, 512 tokens: 1024 (token, slot) pairs, ~12 column tiles; k = 2304 is 9 super-blocks
    (Q4_K, 4096, 2304, 8, 2, 512, True), (Q4_K, 4096, 2304, 8, 2, 512, False),
    (Q8_0, 2048, 2304, 8, 2, 512, True), (Q8_0, 4096, 2304, 8, 2, 512, False),
]


def mmid_tiles(ids, ne, m):
    cnt = np.bincount(ids[(ids >= 0) & (ids < ne)], minlength=ne)
    return -(-m // TILE) * int(sum(-(-c // TILE) for c in cnt))


@pytest.mark.parametrize("t,M,K,ne,nu,n_tok,shared", MMID_CASES)
def test_grouped_mmid_many_tiles_per_cta(b200, t, M, K, ne, nu, n_tok, shared):
    """b200_mul_mat_id2 on the grouped tile kernel with at least two tiles per CTA, so that a CTA's next tile may belong to another
    expert: bit for bit b200_mul_mat_q on each expert's gathered columns, the oracle on a token sample, NaN rows of out-of-range ids"""
    L = b200.lib
    sms = sm_count(b200)
    rng = seeded(t, M, K, ne, nu, shared)
    while True:
        ids = np.stack([rng.choice(ne, nu, replace=False) for _ in range(n_tok)]).astype(np.int32)
        ids[5, 0] = -1
        ids[n_tok - 2, nu - 1] = ne
        tiles = mmid_tiles(ids, ne, M)
        if tiles >= MIN_UNITS * sms:
            break
        n_tok *= 2
    print(f"  SMs {sms}: {ne} experts x {M} x {K}, top-{nu}, {n_tok} tokens: {tiles} tiles on {sms} CTAs, {tiles / sms:.2f} tiles per CTA")
    n_b1 = 1 if shared else nu
    W = rand_blocks(rng, t, ne * M, K)
    b = rng.standard_normal((n_tok, n_b1, K)).astype(np.float32)
    rb = row_bytes(t, K)
    Wd = dev(np.concatenate([repack_rows_np(t, W, K).reshape(-1), np.zeros(64, np.uint8)]))
    bss, bts = K + 8, n_b1 * (K + 8) + 4                       # activation strides wider than the data (multiples of 4 floats)
    bh = np.full((n_tok, bts), np.nan, np.float32)
    for s in range(n_b1):
        bh[:, s * bss:s * bss + K] = b[:, s]
    bd, idd = dev(bh), dev(ids)
    dss, dts = M + 19, nu * (M + 19) + 7                        # output strides wider than the data
    ws = torch.zeros(max(L.b200_mul_mat_id_workspace(t, M, K, ne, nu, n_tok), 1), dtype=torch.uint8, device="cuda")
    assert L.b200_mul_mat_id_workspace(t, M, K, ne, nu, n_tok) > 0       # the grouped path
    rows_mask = np.zeros(dts * n_tok, bool)                     # the (token, slot) rows; everything else is padding
    for tt in range(n_tok):
        for s in range(nu):
            rows_mask[tt * dts + s * dss:tt * dts + s * dss + M] = True
    init = np.where(rows_mask, np.float32(np.nan), SENT).astype(np.float32)

    def run():
        dst = dev(init)
        b200.check(L.b200_mul_mat_id2(t, b200.p(Wd), M * rb, b200.p(bd), bts, bss, n_b1, b200.p(idd), nu, b200.p(dst), dts, dss,
                                      M, K, ne, nu, n_tok, b200.p(ws), b200.stream()))
        torch.cuda.synchronize()
        return dst.cpu().numpy()

    out = run()
    assert out.tobytes() == run().tobytes(), "two runs differ"
    got = out[rows_mask].reshape(n_tok, nu, M)
    assert (out[~rows_mask].view(np.uint32) == SENT.view(np.uint32)).all(), "a store landed outside the (token, slot) rows"
    valid = (ids >= 0) & (ids < ne)
    assert np.isnan(got[~valid]).all(), "rows of out-of-range ids were written"
    assert np.isfinite(got[valid]).all(), "rows left unwritten"
    # bit for bit the dense tile kernel on each expert's gathered columns (padded with zero columns to 128)
    for e in range(ne):
        pairs = [(tt, s) for tt in range(n_tok) for s in range(nu) if ids[tt, s] == e]
        nn = max(len(pairs), TILE)
        X = np.zeros((nn, K), np.float32)
        for j, (tt, s) in enumerate(pairs):
            X[j] = b[tt, s % n_b1]
        xd = dev(X)
        dst = torch.full((nn, M), float("nan"), dtype=torch.float32, device="cuda")
        wse = torch.zeros(L.b200_mul_mat_q_workspace(t, M, K, nn), dtype=torch.uint8, device="cuda")
        b200.check(L.b200_mul_mat_q(t, C.c_void_p(Wd.data_ptr() + e * M * rb), b200.p(xd), K, b200.p(dst), M, M, K, nn, b200.p(wse),
                                    b200.stream()))
        torch.cuda.synchronize()
        dense = dst.cpu().numpy()[:len(pairs)]
        assert dense.tobytes() == np.stack([got[tt, s] for tt, s in pairs]).tobytes(), (e, len(pairs))
    # the oracle on a token sample (the first and last tokens, the ones with out-of-range ids, and random ones)
    samp = sorted(set([0, 5, n_tok - 2, n_tok - 1] + list(rng.choice(n_tok, 28, replace=False))))
    ids_s = np.ascontiguousarray(ids[samp])
    b_s = np.ascontiguousarray(b[samp])
    want = np.full((len(samp), nu, M), np.nan, np.float32)
    oracle().orc_mul_mat_id(t, ptr(W), ptr(b_s), ptr(ids_s), ptr(want), M, K, ne, nu, len(samp), n_b1, nu)
    v = valid[samp]
    g, w = got[samp][v], want[v]
    err = float(np.abs(g - w).max() / np.abs(w).max())
    assert err <= 2e-5, err
