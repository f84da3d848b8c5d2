"""GPU parity tests: every CUDA kernel, called through the C-ABI (include/b200_ops.h), against the
CPU oracle (oracle/liboracle.so, pinned to the reference by test_oracle_*.py) on the same seeded
inputs.  Integer/byte results must be bit-exact; f32 results within the stated tolerance
(BASELINE.json north_star: logits within 1e-3 relative; we hold ops to <= 2e-5 of the output scale).
"""
import ctypes as C

import numpy as np
import pytest

from refutil import (F16, F32, Q4_0, Q5_0, Q4_K, Q5_K, Q6_K, Q8_0, Q8_K, ACT_TYPE, WEIGHT_TYPES, nmse, oracle, orc_dequant,
                     orc_mul_mat, orc_quantize_act, ptr, rand_blocks, row_bytes)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


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


def padded_weights(b200, t, W):
    """device copy of weight rows (+16 bytes slack), repacked for the kernel"""
    m = W.shape[0]
    flat = np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)])
    d = dev(flat)
    k = W.shape[1] // row_bytes(t, 256) * 256 if t in (Q4_K, Q5_K, Q6_K) else W.shape[1] // row_bytes(t, 32) * 32
    b200.check(b200.lib.b200_repack_rows(t, b200.p(d), m, k, b200.stream()))
    return d


def act_from_oracle(kind, xq, k):
    """oracle blocks (q8_K / q8_0 rows) -> our SoA act buffer bytes, per column"""
    L = load_ops().lib
    n = xq.shape[0]
    colb = L.b200_act_col_bytes(kind, k); doff = L.b200_act_d_offset(kind, k); boff = L.b200_act_bsum_offset(kind, k)
    out = np.zeros((n, colb), np.uint8)
    for c in range(n):
        if kind == 0:
            blk = xq[c].reshape(k // 256, 292)
            out[c, :k] = blk[:, 4:260].reshape(-1)
            out[c, doff:doff + 4 * (k // 256)] = blk[:, 0:4].reshape(-1)
            out[c, boff:boff + 2 * (k // 16)] = blk[:, 260:292].reshape(-1)
        else:
            blk = xq[c].reshape(k // 32, 34)
            out[c, :k] = blk[:, 2:34].reshape(-1)
            d = blk[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
            out[c, doff:doff + 4 * (k // 32)] = d.view(np.uint8)
            bs = blk[:, 2:34].view(np.int8).astype(np.int32).sum(axis=1).astype(np.int16)
            out[c, boff:boff + 2 * (k // 32)] = bs.view(np.uint8)
    return out


def load_ops():
    from conftest import load_pkg
    return load_pkg().ops


# ------------------------------------------------------------------ a2: activation quantisation
@pytest.mark.parametrize("wtype", [Q4_K, Q4_0])
@pytest.mark.parametrize("k,n", [(256, 1), (4096, 3), (14336, 2)])
def test_quantize_act_bit_exact(b200, wtype, k, n):
    rng = np.random.default_rng(k + n)
    x = (rng.standard_normal((n, k)) * rng.uniform(0.01, 30)).astype(np.float32)
    x[0, :256] = 0.0                                    # all-zero block
    if k >= 512:
        x[-1, 256:512] = np.float32(1.5) * rng.choice([-1, 1], 256)   # ties on |x|: first-index rule
    kind = b200.lib.b200_act_kind_for(wtype)
    want = act_from_oracle(kind, orc_quantize_act(wtype, x), k)
    act = torch.zeros(n * b200.act_col_bytes(kind, k), dtype=torch.uint8, device="cuda")
    b200.check(b200.lib.b200_quantize_act(kind, b200.p(dev(x)), k, b200.p(act), k, n, b200.stream()))
    got = act.cpu().numpy().reshape(n, -1)
    assert np.array_equal(got, want)


# ------------------------------------------------------------------ a1: repack
@pytest.mark.parametrize("t", WEIGHT_TYPES)
def test_repack_roundtrip(b200, t):
    rng = np.random.default_rng(t)
    k, m = 2048, 7
    W = rand_blocks(rng, t, m, k)
    d = dev(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)]))
    b200.check(b200.lib.b200_repack_rows(t, b200.p(d), m, k, b200.stream()))
    rep = d.cpu().numpy()[:W.size].reshape(m, -1)
    if b200.lib.b200_type_is_repacked(t):
        assert not np.array_equal(rep, W)
        assert np.array_equal(np.sort(rep, axis=1), np.sort(W, axis=1))       # a permutation inside each row
        nb = k // (32 if t in (Q4_0, Q8_0) else 256)
        if t == Q4_0:
            assert np.array_equal(rep[:, :nb * 16].reshape(m, nb, 16), W.reshape(m, nb, 18)[:, :, 2:])
            assert np.array_equal(rep[:, nb * 16:].reshape(m, nb, 2), W.reshape(m, nb, 18)[:, :, :2])
        if t == Q6_K:
            assert np.array_equal(rep[:, nb * 208:].reshape(m, nb, 2), W.reshape(m, nb, 210)[:, :, 208:])
    else:
        assert np.array_equal(rep, W)
    b200.check(b200.lib.b200_unpack_rows(t, b200.p(d), m, k, b200.stream()))
    assert np.array_equal(d.cpu().numpy()[:W.size].reshape(m, -1), W)


# ------------------------------------------------------------------ a3: decode matvec
def run_mmvq(b200, t, W, x, m, k, n, bias=None, resid=None):
    kind = b200.lib.b200_act_kind_for(t)
    act = torch.zeros(n * b200.act_col_bytes(kind, k), dtype=torch.uint8, device="cuda")
    b200.check(b200.lib.b200_quantize_act(kind, b200.p(dev(x)), k, b200.p(act), k, n, b200.stream()))
    Wd = padded_weights(b200, t, W)
    dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
    b = dev(bias) if bias is not None else None
    r = dev(resid) if resid is not None else None
    b200.check(b200.lib.b200_mul_mat_vec_q(t, b200.p(Wd), b200.p(act), b200.p(dst), m, b200.p(b), b200.p(r), m, k, n, b200.stream()))
    return dst.cpu().numpy()


@pytest.mark.parametrize("t", WEIGHT_TYPES)
@pytest.mark.parametrize("m,k,n", [(64, 2048, 1), (33, 4096, 1), (128, 4096, 2), (16, 2048, 3), (40, 4096, 4),
                                   (24, 2048, 5), (24, 2048, 7), (64, 14336, 8), (1, 2048, 1)])
def test_mmvq_vs_oracle(b200, t, m, k, n):
    rng = np.random.default_rng(1000 * t + m + k + n)
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    want = orc_mul_mat(t, W, x, m, n, k)
    got = run_mmvq(b200, t, W, x, m, k, n)
    scale = np.abs(want).max()
    assert np.isfinite(got).all()
    assert np.abs(got - want).max() <= 2e-5 * scale, (np.abs(got - want).max(), scale)
    assert nmse(got, want) < 1e-10


@pytest.mark.parametrize("t", [Q4_K, Q8_0])
def test_mmvq_bias_residual(b200, t):
    rng = np.random.default_rng(7)
    m, k, n = 96, 2048, 2
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    bias = rng.standard_normal(m).astype(np.float32); resid = rng.standard_normal((n, m)).astype(np.float32)
    want = orc_mul_mat(t, W, x, m, n, k) + bias[None, :] + resid
    got = run_mmvq(b200, t, W, x, m, k, n, bias, resid)
    assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max()


def test_mmvq_multi_mixed_types(b200):
    rng = np.random.default_rng(11)
    k, n = 4096, 1
    specs = [(Q4_K, 64), (Q4_K, 17), (Q6_K, 16)]
    x = rng.standard_normal((n, k)).astype(np.float32)
    act = torch.zeros(n * b200.act_col_bytes(0, k), dtype=torch.uint8, device="cuda")
    b200.check(b200.lib.b200_quantize_act(0, b200.p(dev(x)), k, b200.p(act), k, n, b200.stream()))
    descs = (b200.MmvDesc * len(specs))()
    keep, wants, dsts = [], [], []
    for i, (t, m) in enumerate(specs):
        W = rand_blocks(rng, t, m, k)
        wants.append(orc_mul_mat(t, W, x, m, n, k))
        Wd = padded_weights(b200, t, W); dst = torch.zeros((n, m), dtype=torch.float32, device="cuda")
        keep.append(Wd); dsts.append(dst)
        descs[i].W = Wd.data_ptr(); descs[i].dst = dst.data_ptr(); descs[i].bias = None; descs[i].m = m; descs[i].type = t
    b200.check(b200.lib.b200_mul_mat_vec_q_multi(descs, len(specs), b200.p(act), None, k, n, b200.stream()))
    for want, dst in zip(wants, dsts):
        assert np.abs(dst.cpu().numpy() - want).max() <= 2e-5 * np.abs(want).max()


@pytest.mark.parametrize("tg,tu", [(Q4_K, Q4_K), (Q4_0, Q4_0), (Q4_K, Q6_K)])
def test_mmvq_swiglu(b200, tg, tu):
    rng = np.random.default_rng(13)
    m, k, n = 96, 2048, 2
    Wg, Wu = rand_blocks(rng, tg, m, k), rand_blocks(rng, tu, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    g, u = orc_mul_mat(tg, Wg, x, m, n, k), orc_mul_mat(tu, Wu, x, m, n, k)
    want = np.zeros_like(g); oracle().orc_swiglu(ptr(g), ptr(u), ptr(want), g.size)
    acts = [None, None]
    for t in {tg, tu}:
        kind = b200.lib.b200_act_kind_for(t)
        a = torch.zeros(n * b200.act_col_bytes(kind, k), dtype=torch.uint8, device="cuda")
        b200.check(b200.lib.b200_quantize_act(kind, b200.p(dev(x)), k, b200.p(a), k, n, b200.stream()))
        acts[kind] = a
    dst = torch.zeros((n, m), dtype=torch.float32, device="cuda")
    Wgd, Wud = padded_weights(b200, tg, Wg), padded_weights(b200, tu, Wu)
    b200.check(b200.lib.b200_mul_mat_vec_q_swiglu(tg, b200.p(Wgd), tu, b200.p(Wud), b200.p(acts[0]), b200.p(acts[1]), b200.p(dst), m, k, n, b200.stream()))
    assert np.abs(dst.cpu().numpy() - want).max() <= 3e-5 * max(np.abs(want).max(), 1e-6)


@pytest.mark.parametrize("t,src,k", [(Q4_K, 2, 4096), (Q6_K, 2, 4096), (Q8_0, 2, 4096), (Q4_K, 1, 4096), (Q4_0, 1, 4096), (Q4_K, 1, 14336), (Q6_K, 1, 14336)])
def test_mmvq_fused_activation_prologue(b200, t, src, k):
    """rms_norm * w + quantise (act_source 2) or quantise only (1) inside the matvec kernel == oracle composition"""
    rng = np.random.default_rng(31 + t + src)
    m, n = 80, (2 if k == 4096 else 1)
    W = rand_blocks(rng, t, m, k)
    x = (rng.standard_normal((n, k)) * 2).astype(np.float32); w = (1 + 0.1 * rng.standard_normal(k)).astype(np.float32)
    resid = rng.standard_normal((n, m)).astype(np.float32)
    xin = x
    if src == 2:
        xin = np.zeros_like(x); oracle().orc_rms_norm(ptr(x), ptr(w), ptr(xin), k, n, 1e-5)
    want = orc_mul_mat(t, W, xin, m, n, k) + resid
    L = b200.MmvLaunch()
    Wd = padded_weights(b200, t, W); dst = torch.zeros((n, m), dtype=torch.float32, device="cuda")
    xd, wd, rd = dev(x), dev(w), dev(resid)
    L.n_mats = 1; L.k = k; L.ncols = n; L.act_source = src; L.eps = 1e-5
    L.mats[0].W = Wd.data_ptr(); L.mats[0].dst = dst.data_ptr(); L.mats[0].m = m; L.mats[0].type = t
    L.residual[0] = rd.data_ptr(); L.x = xd.data_ptr(); L.x_col_stride = k; L.norm_w = wd.data_ptr() if src == 2 else None
    b200.check(b200.lib.b200_mul_mat_vec_q_launch(C.byref(L), b200.stream()))
    got = dst.cpu().numpy()
    assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max(), np.abs(got - want).max()


def test_mmvq_rejects_bad_shapes(b200):
    d = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    assert b200.lib.b200_mul_mat_vec_q(Q4_K, b200.p(d), b200.p(d), b200.p(d), 8, None, None, 8, 100, 1, b200.stream()) < 0
    assert b200.lib.b200_mul_mat_vec_q(Q4_K, b200.p(d), b200.p(d), b200.p(d), 8, None, None, 8, 256, 9, b200.stream()) < 0
    assert b200.lib.b200_mul_mat_vec_q(3, b200.p(d), b200.p(d), b200.p(d), 8, None, None, 8, 256, 1, b200.stream()) < 0
    assert b"" != b200.lib.b200_last_error()


# ------------------------------------------------------------------ a4 (round 1: column groups)
@pytest.mark.parametrize("t", [Q4_K, Q6_K, Q8_0])
def test_mul_mat_q_batched(b200, t):
    rng = np.random.default_rng(17)
    m, k, n = 48, 2048, 19
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    want = orc_mul_mat(t, W, x, m, n, k)
    ws = torch.zeros(b200.lib.b200_mul_mat_q_workspace(t, m, k, n), dtype=torch.uint8, device="cuda")
    dst = torch.zeros((n, m), dtype=torch.float32, device="cuda")
    Wd = padded_weights(b200, t, W)
    b200.check(b200.lib.b200_mul_mat_q(t, b200.p(Wd), b200.p(dev(x)), k, b200.p(dst), m, m, k, n, b200.p(ws), b200.stream()))
    assert np.abs(dst.cpu().numpy() - want).max() <= 2e-5 * np.abs(want).max()


# ------------------------------------------------------------------ a5: rms_norm
@pytest.mark.parametrize("ncols,nrows,with_w", [(4096, 3, True), (2048, 1, False), (8192, 2, True), (64, 5, True)])
def test_rms_norm(b200, ncols, nrows, with_w):
    rng = np.random.default_rng(ncols + nrows)
    x = rng.standard_normal((nrows, ncols)).astype(np.float32) * 3
    w = (1 + 0.1 * rng.standard_normal(ncols)).astype(np.float32) if with_w else None
    want = np.zeros_like(x); oracle().orc_rms_norm(ptr(x), ptr(w), ptr(want), ncols, nrows, 1e-5)
    y = torch.zeros((nrows, ncols), dtype=torch.float32, device="cuda")
    wd = dev(w) if with_w else None
    b200.check(b200.lib.b200_rms_norm(b200.p(dev(x)), b200.p(wd), b200.p(y), ncols, nrows, ncols, ncols, 1e-5, b200.stream()))
    got = y.cpu().numpy()
    # same operation order as the oracle; only the double-precision sum order differs
    assert np.abs(got - want).max() <= 2e-7 * np.abs(want).max()


def test_rms_norm_quantize_fused(b200):
    rng = np.random.default_rng(5)
    k, n = 4096, 2
    x = rng.standard_normal((n, k)).astype(np.float32); w = (1 + 0.1 * rng.standard_normal(k)).astype(np.float32)
    y = np.zeros_like(x); oracle().orc_rms_norm(ptr(x), ptr(w), ptr(y), k, n, 1e-5)
    act0 = torch.zeros(n * b200.act_col_bytes(0, k), dtype=torch.uint8, device="cuda")
    act1 = torch.zeros(n * b200.act_col_bytes(1, k), dtype=torch.uint8, device="cuda")
    yd = torch.zeros((n, k), dtype=torch.float32, device="cuda")
    b200.check(b200.lib.b200_rms_norm_quantize(b200.p(dev(x)), b200.p(dev(w)), b200.p(yd), b200.p(act0), 0, b200.p(act1), 1, k, n, 1e-5, b200.stream()))
    ygot = yd.cpu().numpy()
    assert np.abs(ygot - y).max() <= 2e-7 * np.abs(y).max()
    # quantisation of the kernel's own f32 output must be bit-exact
    assert np.array_equal(act0.cpu().numpy().reshape(n, -1), act_from_oracle(0, orc_quantize_act(Q4_K, ygot), k))
    assert np.array_equal(act1.cpu().numpy().reshape(n, -1), act_from_oracle(1, orc_quantize_act(Q4_0, ygot), k))


# ------------------------------------------------------------------ a6: rope
ROPE_CASES = [
    dict(mode=0, ff=False, ext=0.0, fs=1.0, hd=128, nd=128, base=500000.0),
    dict(mode=2, ff=False, ext=0.0, fs=1.0, hd=128, nd=128, base=1000000.0),
    dict(mode=0, ff=True, ext=0.0, fs=1.0, hd=128, nd=128, base=500000.0),
    dict(mode=2, ff=True, ext=1.0, fs=0.25, hd=128, nd=128, base=10000.0),
    dict(mode=0, ff=False, ext=0.0, fs=1.0, hd=64, nd=64, base=10000.0),
    dict(mode=2, ff=False, ext=0.0, fs=1.0, hd=128, nd=64, base=10000.0),
]


def rope_params(b200, c):
    return b200.RopeParams(n_dims=c["nd"], mode=c["mode"], n_ctx_orig=8192, freq_base=c["base"], freq_scale=c["fs"],
                           ext_factor=c["ext"], attn_factor=1.0, beta_fast=32.0, beta_slow=1.0)


@pytest.mark.parametrize("c", ROPE_CASES)
def test_rope(b200, c):
    rng = np.random.default_rng(3)
    hd, nh, nt = c["hd"], 8, 6
    x = rng.standard_normal((nt, nh, hd)).astype(np.float32)
    pos = np.array([0, 1, 77, 4095, 8191, 31999], np.int32)
    ff = rng.uniform(1, 8, hd // 2).astype(np.float32) if c["ff"] else None
    want = np.zeros_like(x)
    oracle().orc_rope(ptr(x), ptr(want), ptr(pos), ptr(ff), hd, nh, nt, c["nd"], c["mode"], 8192, c["base"], c["fs"], c["ext"], 1.0, 32.0, 1.0)
    y = torch.zeros((nt, nh, hd), dtype=torch.float32, device="cuda")
    prm = rope_params(b200, c)
    b200.check(b200.lib.b200_rope(b200.p(dev(x)), b200.p(y), b200.p(dev(pos)), b200.p(dev(ff)) if c["ff"] else None,
                                  hd, nh, nt, hd, nh * hd, hd, nh * hd, C.byref(prm), b200.stream()))
    # theta is bit-identical; sinf/cosf differ from glibc by <= 2 ulp of a value <= 1
    assert np.abs(y.cpu().numpy() - want).max() <= 2e-6 * max(1.0, np.abs(want).max())


# ------------------------------------------------------------------ a7: set_rows
@pytest.mark.parametrize("dt", [F16, Q8_0, F32])
def test_set_rows_bit_exact(b200, dt):
    rng = np.random.default_rng(dt)
    nc, nr, tot = 1024, 5, 32
    src = (rng.standard_normal((nr, nc)) * 4).astype(np.float32); src[1, :32] = 0
    ids = np.array([5, 0, 31, 9, 17], np.int64)
    stride = {F16: nc * 2, Q8_0: nc // 32 * 34, F32: nc * 4}[dt]
    cache = rng.integers(0, 255, (tot, stride), dtype=np.uint8)
    want = cache.copy(); oracle().orc_set_rows(ptr(src), ptr(ids), ptr(want), dt, nc, nr, stride)
    cd = dev(cache)
    b200.check(b200.lib.b200_set_rows(b200.p(dev(src)), nc, b200.p(dev(ids)), b200.p(cd), dt, stride, nc, nr, b200.stream()))
    assert np.array_equal(cd.cpu().numpy(), want)


@pytest.mark.parametrize("kvt", [F16, Q8_0])
def test_rope_kv_store(b200, kvt):
    rng = np.random.default_rng(23)
    hd, nh, nhkv, nt, tot = 128, 8, 2, 3, 16
    c = ROPE_CASES[0]
    q = rng.standard_normal((nt, nh, hd)).astype(np.float32); k = rng.standard_normal((nt, nhkv, hd)).astype(np.float32)
    v = rng.standard_normal((nt, nhkv, hd)).astype(np.float32)
    pos = np.array([3, 4, 900], np.int32); ids = np.array([3, 4, 12], np.int64)
    qw, kw = np.zeros_like(q), np.zeros_like(k)
    for src, dst, h in ((q, qw, nh), (k, kw, nhkv)):
        oracle().orc_rope(ptr(src), ptr(dst), ptr(pos), None, hd, h, nt, 128, 0, 8192, c["base"], 1.0, 0.0, 1.0, 32.0, 1.0)
    stride = row_bytes(kvt, nhkv * hd)
    kc0 = rng.integers(0, 255, (tot, stride), dtype=np.uint8); vc0 = rng.integers(0, 255, (tot, stride), dtype=np.uint8)
    qd, kcd, vcd = dev(q), dev(kc0), dev(vc0)
    prm = rope_params(b200, c)
    b200.check(b200.lib.b200_rope_kv_store(b200.p(qd), b200.p(dev(k)), b200.p(dev(v)), b200.p(dev(pos)), None, b200.p(dev(ids)),
                                           b200.p(kcd), b200.p(vcd), kvt, stride, hd, nh, nhkv, nt, C.byref(prm), b200.stream()))
    qg = qd.cpu().numpy()
    assert np.abs(qg - qw).max() <= 2e-6 * np.abs(qw).max()
    # cache rows: convert the kernel's own roped K (recomputed here from the oracle within 2 ulp) —
    # compare dequantised values instead of bytes for K, bytes for V (no rope on V)
    vwant = vc0.copy(); oracle().orc_set_rows(ptr(v.reshape(nt, -1)), ptr(ids), ptr(vwant), kvt, nhkv * hd, nt, stride)
    assert np.array_equal(vcd.cpu().numpy(), vwant)
    kwant = kc0.copy(); oracle().orc_set_rows(ptr(kw.reshape(nt, -1)), ptr(ids), ptr(kwant), kvt, nhkv * hd, nt, stride)
    kg = kcd.cpu().numpy()
    untouched = np.setdiff1d(np.arange(tot), ids)
    assert np.array_equal(kg[untouched], kc0[untouched])
    a = orc_dequant(kvt, kg[ids], nt, nhkv * hd); b = orc_dequant(kvt, kwant[ids], nt, nhkv * hd)
    assert np.abs(a - b).max() <= (2e-3 if kvt == F16 else 4e-2) * np.abs(b).max()   # one quantisation step at most


# ------------------------------------------------------------------ a8: flash attention
@pytest.mark.parametrize("kvt", [F16, Q8_0])
@pytest.mark.parametrize("dk,nh,nhkv,nt,nkv", [(128, 32, 8, 1, 512), (128, 8, 1, 1, 256), (64, 32, 4, 1, 256), (128, 8, 2, 3, 1024),
                                               (128, 4, 4, 2, 256), (64, 6, 3, 1, 4096)])
def test_flash_attn(b200, kvt, dk, nh, nhkv, nt, nkv):
    rng = np.random.default_rng(dk + nh + nt + nkv + kvt)
    kvsize = nkv + 64
    q = rng.standard_normal((nt, nh, dk)).astype(np.float32)
    kf = rng.standard_normal((kvsize, nhkv * dk)).astype(np.float32); vf = rng.standard_normal((kvsize, nhkv * dk)).astype(np.float32)
    rb_row = row_bytes(kvt, nhkv * dk); rb_head = row_bytes(kvt, dk)
    kc = np.zeros((kvsize, rb_row), np.uint8); vc = np.zeros((kvsize, rb_row), np.uint8)
    ids = np.arange(kvsize, dtype=np.int64)
    oracle().orc_set_rows(ptr(kf), ptr(ids), ptr(kc), kvt, nhkv * dk, kvsize, rb_row)
    oracle().orc_set_rows(ptr(vf), ptr(ids), ptr(vc), kvt, nhkv * dk, kvsize, rb_row)
    npad = (nt + 63) // 64 * 64
    mask = np.full((npad, nkv), -np.inf, np.float32)
    for t in range(nt):
        mask[t, :nkv - 40 - nt + t + 1] = 0
    mask16 = mask.astype(np.float16)
    scale = 1.0 / np.sqrt(dk)
    want = np.zeros((nt, nh, dk), np.float32)
    oracle().orc_flash_attn_ext(ptr(q), nh * dk * 4, dk * 4, ptr(kc), rb_row, rb_head, ptr(vc), rb_row, rb_head, ptr(mask16), ptr(want),
                                kvt, dk, dk, nh, nhkv, nt, nkv, scale, 0.0, 0.0)
    ws = torch.zeros(max(16, b200.lib.b200_flash_attn_workspace(dk, nh, nt, nkv)), dtype=torch.uint8, device="cuda")
    dst = torch.full((nt, nh, dk), float("nan"), dtype=torch.float32, device="cuda")
    b200.check(b200.lib.b200_flash_attn_ext(b200.p(dev(q)), nh * dk, dk, b200.p(dev(kc)), rb_row, rb_head, b200.p(dev(vc)), rb_row, rb_head,
                                            b200.p(dev(mask16.view(np.uint16))), nkv, b200.p(dst), kvt, dk, dk, nh, nhkv, nt, nkv,
                                            scale, 0.0, 0.0, b200.p(ws), b200.stream()))
    got = dst.cpu().numpy()
    assert np.isfinite(got).all()
    if kvt == Q8_0:
        # integer K.Q block sums are identical to the oracle's; V accumulates in f32 on both sides
        assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max(), np.abs(got - want).max()
        assert nmse(got, want) < 1e-9
    else:
        # F16 V: the oracle accumulates V in fp16 (ops.cpp:8278-8340) — its rounding noise grows with n_kv and
        # dwarfs ours, so the tight check is against an f64 evaluation of the same f16-rounded Q/K/V, and the
        # oracle only has to agree to fp16-accumulator accuracy.
        q16 = q.astype(np.float16).astype(np.float64)
        kk = orc_dequant(F16, kc[:nkv], nkv, nhkv * dk).astype(np.float64); vv = orc_dequant(F16, vc[:nkv], nkv, nhkv * dk).astype(np.float64)
        truth = np.zeros((nt, nh, dk))
        for t in range(nt):
            for h in range(nh):
                hk = h // (nh // nhkv)
                s = (kk[:, hk * dk:(hk + 1) * dk] @ q16[t, h]) * scale + mask16[t].astype(np.float64)
                p = np.exp(s - s.max()); truth[t, h] = (p[:, None] * vv[:, hk * dk:(hk + 1) * dk]).sum(0) / p.sum()
        sc = np.abs(truth).max()
        err_gpu, err_orc = np.abs(got - truth).max(), np.abs(want - truth).max()
        assert err_gpu <= 2e-5 * sc, (err_gpu, sc)
        assert err_gpu <= err_orc, (err_gpu, err_orc)
        assert np.abs(got - want).max() <= 5e-2 * sc, (np.abs(got - want).max(), sc)


@pytest.mark.parametrize("kvt", [F16, Q8_0])
@pytest.mark.parametrize("hd,nh,nhkv,nkv,pos,mode", [(128, 32, 8, 768, 517, 0), (128, 8, 2, 256, 3, 2), (64, 32, 4, 256, 255, 0), (128, 4, 4, 1024, 600, 2)])
def test_rope_kv_flash_attn_equals_separate_kernels(b200, kvt, hd, nh, nhkv, nkv, pos, mode):
    """the fused decode launch (rope q/k, KV store, attention) against b200_rope_kv_store2 + b200_flash_attn_ext, which are
    each checked against the oracle above: identical cache bytes, identical roped Q, identical attention output"""
    rng = np.random.default_rng(hd + nh + nkv + kvt + mode)
    tot = nkv + 8
    q = rng.standard_normal((1, nh, hd)).astype(np.float32); k = rng.standard_normal((1, nhkv, hd)).astype(np.float32)
    v = rng.standard_normal((1, nhkv, hd)).astype(np.float32)
    rb_row = row_bytes(kvt, nhkv * hd); rb_head = row_bytes(kvt, hd)
    kf = rng.standard_normal((tot, nhkv * hd)).astype(np.float32); vf = rng.standard_normal((tot, nhkv * hd)).astype(np.float32)
    kc = np.zeros((tot, rb_row), np.uint8); vc = np.zeros((tot, rb_row), np.uint8)
    ids_all = np.arange(tot, dtype=np.int64)
    oracle().orc_set_rows(ptr(kf), ptr(ids_all), ptr(kc), kvt, nhkv * hd, tot, rb_row)
    oracle().orc_set_rows(ptr(vf), ptr(ids_all), ptr(vc), kvt, nhkv * hd, tot, rb_row)
    mask = np.full((64, nkv), -np.inf, np.float32); mask[0, :pos + 1] = 0
    mask16 = mask.astype(np.float16).view(np.uint16)
    posd, idsd = dev(np.array([pos], np.int32)), dev(np.array([pos], np.int64))
    c = dict(ROPE_CASES[0]); prm = rope_params(b200, c); prm.mode = mode; prm.n_dims = hd
    scale = 1.0 / np.sqrt(hd)
    wsb = max(16, b200.lib.b200_flash_attn_workspace(hd, nh, 1, nkv))
    # reference: two launches
    q1 = dev(q); qr1 = torch.zeros_like(q1); kc1, vc1 = dev(kc), dev(vc); ws1 = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    d1 = torch.full((1, nh, hd), float("nan"), dtype=torch.float32, device="cuda")
    b200.check(b200.lib.b200_rope_kv_store2(b200.p(q1), b200.p(qr1), b200.p(dev(k)), b200.p(dev(v)), b200.p(posd), None, b200.p(idsd), b200.p(idsd),
                                            b200.p(kc1), b200.p(vc1), kvt, rb_row, rb_row, hd, nh, nhkv, 1, C.byref(prm), b200.stream()))
    b200.check(b200.lib.b200_flash_attn_ext(b200.p(qr1), nh * hd, hd, b200.p(kc1), rb_row, rb_head, b200.p(vc1), rb_row, rb_head, b200.p(dev(mask16)), nkv,
                                            b200.p(d1), kvt, hd, hd, nh, nhkv, 1, nkv, scale, 0.0, 0.0, b200.p(ws1), b200.stream()))
    # fused: one launch
    q2 = dev(q); qr2 = torch.zeros_like(q2); kc2, vc2 = dev(kc), dev(vc); ws2 = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    d2 = torch.full((1, nh, hd), float("nan"), dtype=torch.float32, device="cuda")
    b200.check(b200.lib.b200_rope_kv_flash_attn(b200.p(q2), b200.p(qr2), b200.p(dev(k)), b200.p(dev(v)), b200.p(posd), None, b200.p(idsd), b200.p(idsd),
                                                b200.p(kc2), b200.p(vc2), kvt, rb_row, rb_head, rb_row, rb_head, b200.p(dev(mask16)), b200.p(d2),
                                                hd, nh, nhkv, nkv, C.byref(prm), scale, 0.0, 0.0, b200.p(ws2), b200.stream()))
    torch.cuda.synchronize()
    assert torch.equal(kc1, kc2) and torch.equal(vc1, vc2)
    assert torch.equal(qr1, qr2)
    assert torch.isfinite(d2).all() and torch.equal(d1, d2)


def test_flash_attn_f16_closer_to_f64_than_oracle(b200):
    """With F16 V the oracle accumulates in fp16; our f32 accumulation must be at least as close to an
    f64 evaluation of the same attention (same f16-rounded Q, K, V) as the oracle is."""
    rng = np.random.default_rng(99)
    dk, nh, nhkv, nt, nkv = 128, 8, 2, 1, 1024
    q = rng.standard_normal((nt, nh, dk)).astype(np.float32)
    kf = rng.standard_normal((nkv, nhkv * dk)).astype(np.float32); vf = rng.standard_normal((nkv, nhkv * dk)).astype(np.float32)
    k16, v16 = kf.astype(np.float16), vf.astype(np.float16)
    scale = 1.0 / np.sqrt(dk)
    q16 = q.astype(np.float16).astype(np.float64)
    truth = np.zeros((nt, nh, dk))
    for h in range(nh):
        kk = k16[:, (h // 4) * dk:(h // 4 + 1) * dk].astype(np.float64); vv = v16[:, (h // 4) * dk:(h // 4 + 1) * dk].astype(np.float64)
        s = (kk @ q16[0, h]) * scale
        p = np.exp(s - s.max()); truth[0, h] = (p[:, None] * vv).sum(0) / p.sum()
    rb_row, rb_head = nhkv * dk * 2, dk * 2
    kc, vc = k16.view(np.uint8).reshape(nkv, -1), v16.view(np.uint8).reshape(nkv, -1)
    want = np.zeros((nt, nh, dk), np.float32)
    oracle().orc_flash_attn_ext(ptr(q), nh * dk * 4, dk * 4, ptr(kc), rb_row, rb_head, ptr(vc), rb_row, rb_head, None, ptr(want),
                                F16, dk, dk, nh, nhkv, nt, nkv, scale, 0.0, 0.0)
    ws = torch.zeros(b200.lib.b200_flash_attn_workspace(dk, nh, nt, nkv), dtype=torch.uint8, device="cuda")
    dst = torch.zeros((nt, nh, dk), dtype=torch.float32, device="cuda")
    b200.check(b200.lib.b200_flash_attn_ext(b200.p(dev(q)), nh * dk, dk, b200.p(dev(kc)), rb_row, rb_head, b200.p(dev(vc)), rb_row, rb_head,
                                            None, 0, b200.p(dst), F16, dk, dk, nh, nhkv, nt, nkv, scale, 0.0, 0.0, b200.p(ws), b200.stream()))
    err_gpu = np.abs(dst.cpu().numpy() - truth).max(); err_orc = np.abs(want - truth).max()
    assert err_gpu <= err_orc and err_gpu <= 1e-5 * np.abs(truth).max() * 10, (err_gpu, err_orc)


# ------------------------------------------------------------------ a9: glue
def test_glue_ops(b200):
    rng = np.random.default_rng(29)
    a = rng.standard_normal((6, 1024)).astype(np.float32); b = rng.standard_normal((2, 1024)).astype(np.float32)
    for name, fn in (("b200_add", np.add), ("b200_mul", np.multiply)):
        y = torch.zeros((6, 1024), dtype=torch.float32, device="cuda")
        b200.check(getattr(b200.lib, name)(b200.p(dev(a)), b200.p(dev(b)), b200.p(y), 1024, 6, 2, b200.stream()))
        assert np.array_equal(y.cpu().numpy(), fn(a, np.tile(b, (3, 1))))
    g = (rng.standard_normal(4096) * 4).astype(np.float32); u = rng.standard_normal(4096).astype(np.float32)
    want = np.zeros_like(g); oracle().orc_swiglu(ptr(g), ptr(u), ptr(want), g.size)
    y = torch.zeros(4096, dtype=torch.float32, device="cuda")
    b200.check(b200.lib.b200_swiglu(b200.p(dev(g)), b200.p(dev(u)), b200.p(y), 4096, b200.stream()))
    assert np.abs(y.cpu().numpy() - want).max() <= 2e-6 * np.abs(want).max()
    src = rng.standard_normal((10, 512)).astype(np.float32); ids = np.array([9, 0, 3], np.int32)
    y = torch.zeros((3, 512), dtype=torch.float32, device="cuda")
    b200.check(b200.lib.b200_get_rows_f32(b200.p(dev(src)), 512, b200.p(dev(ids)), b200.p(y), 512, 3, b200.stream()))
    assert np.array_equal(y.cpu().numpy(), src[ids])
    x = (rng.standard_normal(1003) * 100).astype(np.float32)
    h = torch.zeros(1003, dtype=torch.float16, device="cuda")
    b200.check(b200.lib.b200_cpy_f32_f16(b200.p(dev(x)), b200.p(h), 1003, b200.stream()))
    assert np.array_equal(h.cpu().numpy().view(np.uint16), x.astype(np.float16).view(np.uint16))
    lg = rng.standard_normal((2, 128256)).astype(np.float32); lg[1, 777] = 50; lg[1, 90000] = 50
    idx = torch.zeros(2, dtype=torch.int32, device="cuda")
    b200.check(b200.lib.b200_argmax_f32(b200.p(dev(lg)), b200.p(idx), 128256, 2, b200.stream()))
    assert idx.cpu().numpy().tolist() == [int(lg[0].argmax()), 777]
    assert b200.lib.b200_kernel_launches() > 0


# ------------------------------------------------------------------ a4: batched MUL_MAT on the tensor cores (wgmma, mmq_tc.cu)
@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K])
@pytest.mark.parametrize("m,k,n", [(128, 2048, 128), (256, 4096, 40), (48, 2048, 19), (384, 2048, 300), (1024, 4096, 512)])
def test_mul_mat_q_tensor_core_vs_oracle(b200, t, m, k, n):
    """the wgmma tile kernel against the C oracle (ggml_vec_dot_q*_K_q8_K restated): the integer sums are exact, so only the
    f32 summation order over super-blocks differs — same bound as the matvec"""
    rng = np.random.default_rng(1000 + m + n)
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    x[n // 2, :256] = 0.0                                       # an all-zero q8_K block (d = 0)
    want = orc_mul_mat(t, W, x, m, n, k)
    ws = torch.zeros(b200.lib.b200_mul_mat_q_workspace(t, m, k, n), dtype=torch.uint8, device="cuda")
    dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
    Wd = padded_weights(b200, t, W)
    b200.check(b200.lib.b200_mul_mat_q(t, b200.p(Wd), b200.p(dev(x)), k, b200.p(dst), m, m, k, n, b200.p(ws), b200.stream()))
    got = dst.cpu().numpy()
    assert np.isfinite(got).all()
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err <= 2e-5, err


def test_mul_mat_q_tensor_core_baseline_shape(b200):
    """BASELINE config 3 shape: ffn_down of Llama-3-8B (m 4096, k 14336) against a 512-token ubatch; NMSE vs the oracle on a row sample"""
    rng = np.random.default_rng(5)
    t, m, k, n = Q4_K, 4096, 14336, 512
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    ws = torch.zeros(b200.lib.b200_mul_mat_q_workspace(t, m, k, n), dtype=torch.uint8, device="cuda")
    dst = torch.zeros((n, m), dtype=torch.float32, device="cuda")
    Wd = padded_weights(b200, t, W)
    b200.check(b200.lib.b200_mul_mat_q(t, b200.p(Wd), b200.p(dev(x)), k, b200.p(dst), m, m, k, n, b200.p(ws), b200.stream()))
    got = dst.cpu().numpy()
    rows = np.concatenate([np.arange(0, 64), np.arange(2000, 2064), np.arange(m - 64, m)])
    want = orc_mul_mat(t, W[rows], x, len(rows), n, k)
    d = (got[:, rows] - want).astype(np.float64)
    nmse = float((d * d).sum() / (want.astype(np.float64) ** 2).sum())
    assert nmse < 1e-10, nmse


@pytest.mark.parametrize("kvt", [F16, Q8_0])
@pytest.mark.parametrize("hd,nh,nhkv", [(128, 32, 8), (64, 32, 4)])
def test_fused_decode_attention_vs_oracle_at_depth(b200, kvt, hd, nh, nhkv):
    """the launch every decode token runs (rope q/k + KV store + split-KV attention, b200_rope_kv_flash_attn2) DIRECTLY against the
    C oracle (rope -> set_rows -> flash_attn_ext) at n_kv = 4096, position 4000; both rope-table modes (layer 0 computes and
    stores the per-token table, the other layers load it) must give the same bits"""
    rng = np.random.default_rng(7 + hd + kvt)
    nkv, pos = 4096, 4000
    q = rng.standard_normal((1, nh, hd)).astype(np.float32); k = rng.standard_normal((1, nhkv, hd)).astype(np.float32)
    v = rng.standard_normal((1, nhkv, hd)).astype(np.float32)
    rb_row = row_bytes(kvt, nhkv * hd); rb_head = row_bytes(kvt, hd)
    kf = rng.standard_normal((nkv, nhkv * hd)).astype(np.float32); vf = rng.standard_normal((nkv, nhkv * hd)).astype(np.float32)
    kc = np.zeros((nkv, rb_row), np.uint8); vc = np.zeros((nkv, rb_row), np.uint8)
    ids_all = np.arange(nkv, dtype=np.int64)
    oracle().orc_set_rows(ptr(kf), ptr(ids_all), ptr(kc), kvt, nhkv * hd, nkv, rb_row)
    oracle().orc_set_rows(ptr(vf), ptr(ids_all), ptr(vc), kvt, nhkv * hd, nkv, rb_row)
    mask = np.full((64, nkv), -np.inf, np.float32); mask[0, :pos + 1] = 0
    mask16 = mask.astype(np.float16).view(np.uint16)
    c = dict(ROPE_CASES[0]); prm = rope_params(b200, c); prm.mode = 0; prm.n_dims = hd
    scale = 1.0 / np.sqrt(hd)
    # oracle: rope(q), rope(k) -> cell pos, v -> cell pos, attention over the cache
    posn = np.array([pos], np.int32)
    qr = np.zeros_like(q); kr = np.zeros_like(k)
    oracle().orc_rope(ptr(q), ptr(qr), ptr(posn), None, hd, nh, 1, hd, 0, 8192, c["base"], c["fs"], c["ext"], 1.0, 32.0, 1.0)
    oracle().orc_rope(ptr(k), ptr(kr), ptr(posn), None, hd, nhkv, 1, hd, 0, 8192, c["base"], c["fs"], c["ext"], 1.0, 32.0, 1.0)
    kco, vco = kc.copy(), vc.copy()
    one = np.array([pos], np.int64)
    oracle().orc_set_rows(ptr(kr.reshape(1, -1)), ptr(one), ptr(kco), kvt, nhkv * hd, 1, rb_row)
    oracle().orc_set_rows(ptr(v.reshape(1, -1)), ptr(one), ptr(vco), kvt, nhkv * hd, 1, rb_row)
    want = np.zeros((1, nh, hd), np.float32)
    oracle().orc_flash_attn_ext(ptr(qr), nh * hd * 4, hd * 4, ptr(kco), rb_row, rb_head, ptr(vco), rb_row, rb_head, ptr(mask16), ptr(want),
                                kvt, hd, hd, nh, nhkv, 1, nkv, scale, 0.0, 0.0)
    posd, idsd = dev(posn), dev(one)
    wsb = max(16, b200.lib.b200_flash_attn_workspace(hd, nh, 1, nkv))
    tab = torch.zeros(2 * hd, dtype=torch.float32, device="cuda")
    outs = []
    for mode in (0, 1, None):                                    # compute + store the table, reuse it, no shared table at all
        q2 = dev(q); qr2 = torch.zeros_like(q2); kc2, vc2 = dev(kc), dev(vc); ws2 = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        d2 = torch.full((1, nh, hd), float("nan"), dtype=torch.float32, device="cuda")
        b200.check(b200.lib.b200_rope_kv_flash_attn2(b200.p(q2), b200.p(qr2), b200.p(dev(k)), b200.p(dev(v)), b200.p(posd), None, b200.p(idsd), b200.p(idsd),
                                                     b200.p(kc2), b200.p(vc2), kvt, rb_row, rb_head, rb_row, rb_head, b200.p(dev(mask16)), b200.p(d2),
                                                     hd, nh, nhkv, nkv, C.byref(prm), scale, 0.0, 0.0, b200.p(ws2), b200.p(tab) if mode is not None else None, mode or 0, b200.stream()))
        torch.cuda.synchronize()
        assert np.array_equal(kc2.cpu().numpy(), kco) and np.array_equal(vc2.cpu().numpy(), vco)          # cache bytes: bit-exact
        assert np.abs(qr2.cpu().numpy() - qr).max() <= 2e-6 * np.abs(qr).max()
        outs.append(d2.cpu().numpy())
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])
    if kvt == Q8_0:
        assert np.abs(outs[0] - want).max() <= 2e-5 * np.abs(want).max()
    else:
        # F16 V: the oracle accumulates V in fp16 (ops.cpp:8278-8340) — over 4000 positions that costs it ~1e-2; judge both against an
        # f64 evaluation of the same attention on the same f16-rounded Q / K / V
        K16 = kco.view(np.float16).reshape(nkv, nhkv, hd).astype(np.float64); V16 = vco.view(np.float16).reshape(nkv, nhkv, hd).astype(np.float64)
        q16 = qr.astype(np.float16).astype(np.float64)
        truth = np.zeros((1, nh, hd))
        for h in range(nh):
            sc = (K16[:pos + 1, h // (nh // nhkv)] @ q16[0, h]) * scale
            pr = np.exp(sc - sc.max()); truth[0, h] = (pr[:, None] * V16[:pos + 1, h // (nh // nhkv)]).sum(0) / pr.sum()
        err_gpu = np.abs(outs[0] - truth).max(); err_orc = np.abs(want - truth).max()
        assert err_gpu <= err_orc and err_gpu <= 2e-5 * np.abs(truth).max(), (err_gpu, err_orc)


# ------------------------------------------------------------------ a8: multi-token attention on the tensor cores (fattn_tc.cu)
@pytest.mark.parametrize("kvt", [F16, Q8_0])
@pytest.mark.parametrize("nh,nhkv,nt,nkv,past", [(8, 2, 128, 256, 100), (4, 4, 200, 768, 512), (32, 8, 512, 1024, 512), (8, 1, 33, 512, 300), (4, 2, 512, 4096, 3584)])
def test_flash_attn_tensor_core(b200, kvt, nh, nhkv, nt, nkv, past):
    """prefill-shaped FLASH_ATTN_EXT (>= 16 tokens, head 128): wgmma S = Q K^T and O = P V with f16 operands, f32 softmax.
    Checked against an f64 evaluation of the same attention on the cache's own (f16-rounded / de-quantised) K, V and the f16-rounded
    Q; f16 P and f16 d*q de-quantisation bound the deviation to ~1e-3 relative (the reference's CUDA path rounds the same way);
    the CPU oracle (f32 P; fp16 accumulation for F16 V) must agree to its own accuracy.  Causal mask with `past` cached positions,
    cache padding beyond, ragged token counts, GQA."""
    dk = 128
    rng = np.random.default_rng(nh + nt + nkv + kvt)
    q = rng.standard_normal((nt, nh, dk)).astype(np.float32)
    kf = rng.standard_normal((nkv, nhkv * dk)).astype(np.float32); vf = rng.standard_normal((nkv, nhkv * dk)).astype(np.float32)
    rb_row = row_bytes(kvt, nhkv * dk); rb_head = row_bytes(kvt, dk)
    kc = np.zeros((nkv, rb_row), np.uint8); vc = np.zeros((nkv, rb_row), np.uint8)
    ids = np.arange(nkv, dtype=np.int64)
    oracle().orc_set_rows(ptr(kf), ptr(ids), ptr(kc), kvt, nhkv * dk, nkv, rb_row)
    oracle().orc_set_rows(ptr(vf), ptr(ids), ptr(vc), kvt, nhkv * dk, nkv, rb_row)
    npad = (nt + 63) // 64 * 64
    mask = np.full((npad, nkv), -np.inf, np.float32)
    for t in range(nt):
        mask[t, :min(nkv, past + t + 1)] = 0                      # causal: token t sees the cached positions and the batch up to itself
    mask16 = mask.astype(np.float16)
    scale = 1.0 / np.sqrt(dk)
    want = np.zeros((nt, nh, dk), np.float32)
    oracle().orc_flash_attn_ext(ptr(q), nh * dk * 4, dk * 4, ptr(kc), rb_row, rb_head, ptr(vc), rb_row, rb_head, ptr(mask16), ptr(want),
                                kvt, dk, dk, nh, nhkv, nt, nkv, scale, 0.0, 0.0)
    ws = torch.zeros(max(16, b200.lib.b200_flash_attn_workspace(dk, nh, nt, nkv)), dtype=torch.uint8, device="cuda")
    dst = torch.full((nt, nh, dk), float("nan"), dtype=torch.float32, device="cuda")
    qd, kd, vd, md = dev(q), dev(kc), dev(vc), dev(mask16.view(np.uint16))     # named: a temporary's block would be recycled by the next allocation
    b200.check(b200.lib.b200_flash_attn_ext(b200.p(qd), nh * dk, dk, b200.p(kd), rb_row, rb_head, b200.p(vd), rb_row, rb_head,
                                            b200.p(md), nkv, b200.p(dst), kvt, dk, dk, nh, nhkv, nt, nkv,
                                            scale, 0.0, 0.0, b200.p(ws), b200.stream()))
    got = dst.cpu().numpy()
    assert np.isfinite(got).all()
    Kd = orc_dequant(kvt, kc, nkv, nhkv * dk).astype(np.float64).reshape(nkv, nhkv, dk)
    Vd = orc_dequant(kvt, vc, nkv, nhkv * dk).astype(np.float64).reshape(nkv, nhkv, dk)
    q16 = q.astype(np.float16).astype(np.float64)
    truth = np.zeros((nt, nh, dk))
    for h in range(nh):
        hk = h // (nh // nhkv)
        s = (q16[:, h] @ Kd[:, hk].T) * scale + mask[:nt].astype(np.float64)
        p = np.exp(s - s.max(axis=1, keepdims=True))
        truth[:, h] = (p @ Vd[:, hk]) / p.sum(axis=1, keepdims=True)
    err = np.abs(got - truth).max() / np.abs(truth).max()
    assert err <= 2e-3, err                                       # observed: 8e-5 .. 5e-4
    assert nmse(got, truth) < 1e-6, nmse(got, truth)
    # vs the CPU oracle, which is the noisier side in both modes: its F16-V path accumulates in fp16 (ops.cpp:8278-8340) and
    # its Q8_0-K path quantises the query row to int8 first (ops.cpp:8210-8222) where the tensor-core kernel keeps f16 queries
    assert nmse(got, want) < (1e-3 if kvt == F16 else 1e-4), nmse(got, want)
    assert nmse(got, truth) <= nmse(want, truth)


# ------------------------------------------------------------------ rows that are not a multiple of 256 elements (Qwen2-72B ffn_down)
@pytest.mark.parametrize("t", [Q5_0, Q8_0, Q4_0])
@pytest.mark.parametrize("m,k,n", [(48, 29568, 1), (16, 29568, 4), (8, 96, 2), (40, 29568, 19)])
def test_mul_mat_padded_rows(b200, t, m, k, n):
    """k % 256 != 0 for the 32-element block types: the reference quantiser falls back to Q5_0 / Q8_0 for Qwen2-72B's ffn_down
    (n_ff = 29568, llama-quant.cpp:442-470).  Weights go through b200_repack_rows_padded (zero blocks up to the next multiple of
    256), the activation prologue zero-fills past k_valid; decode matvec (fused in-kernel quantisation) and the batched path;
    the inverse conversion restores the ggml bytes exactly."""
    rng = np.random.default_rng(t * 100 + m + n)
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    want = orc_mul_mat(t, W, x, m, n, k)
    kp = b200.lib.b200_padded_k(t, k)
    assert kp % 256 == 0 and kp >= k
    src = dev(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)]))
    Wd = torch.zeros(m * row_bytes(t, kp) + 64, dtype=torch.uint8, device="cuda")
    b200.check(b200.lib.b200_repack_rows_padded(t, b200.p(src), b200.p(Wd), m, k, 0, b200.stream()))
    back = torch.zeros_like(src)
    b200.check(b200.lib.b200_repack_rows_padded(t, b200.p(Wd), b200.p(back), m, k, 1, b200.stream()))
    torch.cuda.synchronize()
    assert torch.equal(back[:W.size], src[:W.size])
    xd = dev(x)
    dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
    if n <= 8:
        L = b200.MmvLaunch()
        L.n_mats = 1; L.k = kp; L.k_valid = k; L.ncols = n; L.act_source = 1; L.x = xd.data_ptr(); L.x_col_stride = k
        L.mats[0].W = Wd.data_ptr(); L.mats[0].dst = dst.data_ptr(); L.mats[0].m = m; L.mats[0].type = t
        b200.check(b200.lib.b200_mul_mat_vec_q_launch(C.byref(L), b200.stream()))
    else:
        ws = torch.zeros(b200.lib.b200_mul_mat_q_workspace(t, m, kp, n), dtype=torch.uint8, device="cuda")
        b200.check(b200.lib.b200_mul_mat_q2(t, b200.p(Wd), b200.p(xd), k, b200.p(dst), m, m, kp, k, n, b200.p(ws), b200.stream()))
    got = dst.cpu().numpy()
    assert np.isfinite(got).all()
    assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max(), np.abs(got - want).max() / np.abs(want).max()
