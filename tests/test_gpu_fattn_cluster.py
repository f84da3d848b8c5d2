"""Split-KV decode attention (fattn.cu) at the shapes that exercise its cluster merge: the KV splits of one (token, head tile) are
the CTAs of one thread-block cluster and merge through distributed shared memory.  Cases: whole splits (and whole cluster members)
masked, n_kv not a multiple of the split length, a single split (cluster of 1), a long cache (16 splits of many chunks), 3-token
batches, both GQA tile widths G (1 and 2 query heads per CTA) and both KV types — against the CPU oracle at test_flash_attn's tolerances.  Every
case runs twice and must give bit-identical outputs: the merge reads its peers in a fixed order."""
import ctypes as C

import numpy as np
import pytest

from refutil import F16, Q8_0, nmse, oracle, orc_dequant, ptr, row_bytes

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

_KEEP = []


@pytest.fixture(autouse=True)
def _keep_alive():
    yield
    torch.cuda.synchronize()
    _KEEP.clear()


def dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    _KEEP.append(t)
    return t


def check_against_oracle(got, want, kvt, q, kc, vc, mask16, dk, nh, nhkv, nt, nkv, scale):
    """test_flash_attn's acceptance: Q8_0 within 2e-5 of the oracle; F16 within 2e-5 of an f64 evaluation and no further from it than
    the oracle (which accumulates V in fp16)"""
    assert np.isfinite(got).all()
    if kvt == Q8_0:
        assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max(), np.abs(got - want).max()
        assert nmse(got, want) < 1e-9
        return
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
@pytest.mark.parametrize("dk,nh,nhkv,nt,nkv,seen", [
    (128, 32, 8, 1, 768, 40),        # 16 splits of 48: splits 1..15 see nothing
    (128, 8, 2, 1, 1000, 1000),      # n_kv not a multiple of the split length (16 x 64 covers 1024)
    (128, 32, 8, 1, 32, 32),         # one split: a cluster of 1
    (128, 32, 8, 1, 8192, 8100),     # 16 splits of 512: sixteen chunks each
    (128, 32, 8, 3, 768, 600),       # 3-token batch
    (64, 8, 4, 3, 1024, 70),         # 3 tokens, head 64, most splits masked
    (128, 16, 8, 1, 640, 640),       # G = 2
    (128, 8, 8, 1, 512, 300),        # G = 1
    (64, 6, 6, 1, 200, 200),         # G = 1, head 64, a last split shorter than a chunk
])
def test_flash_attn_cluster_merge(b200, kvt, dk, nh, nhkv, nt, nkv, seen):
    rng = np.random.default_rng(dk + nh + nhkv + nt + nkv + seen + kvt)
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
        mask[t, :seen - nt + t + 1] = 0                             # causal: token t sees `seen - nt + t + 1` positions
    mask16 = mask.astype(np.float16)
    scale = 1.0 / np.sqrt(dk)
    want = np.zeros((nt, nh, dk), np.float32)
    oracle().orc_flash_attn_ext(ptr(q), nh * dk * 4, dk * 4, ptr(kc), rb_row, rb_head, ptr(vc), rb_row, rb_head, ptr(mask16), ptr(want),
                                kvt, dk, dk, nh, nhkv, nt, nkv, scale, 0.0, 0.0)
    qd, kd, vd, md = dev(q), dev(kc), dev(vc), dev(mask16.view(np.uint16))
    outs = []
    for _ in range(2):
        dst = torch.full((nt, nh, dk), float("nan"), dtype=torch.float32, device="cuda")
        b200.check(b200.lib.b200_flash_attn_ext(b200.p(qd), nh * dk, dk, b200.p(kd), rb_row, rb_head, b200.p(vd), rb_row, rb_head,
                                                b200.p(md), nkv, b200.p(dst), kvt, dk, dk, nh, nhkv, nt, nkv, scale, 0.0, 0.0, None, b200.stream()))
        outs.append(dst.cpu().numpy())
    assert np.array_equal(outs[0], outs[1])
    check_against_oracle(outs[0], want, kvt, q, kc, vc, mask16, dk, nh, nhkv, nt, nkv, scale)


@pytest.mark.parametrize("kvt", [F16, Q8_0])
@pytest.mark.parametrize("hd,nh,nhkv,nkv,pos", [(128, 32, 8, 768, 20), (128, 32, 8, 8192, 5000), (64, 16, 8, 512, 3)])
def test_fused_decode_attention_cluster_merge(b200, kvt, hd, nh, nhkv, nkv, pos):
    """the fused decode launch (rope q / k, KV store, attention) with the shared cos/sin table computed (mode 0) and loaded (mode 1,
    the instance every layer after the first runs, which reads the mask before the previous kernel has finished): a token far below
    n_kv, so that whole splits are masked.  Both modes, each twice, bit-identical; checked against the oracle's rope + set_rows +
    attention."""
    rng = np.random.default_rng(hd + nh + nkv + pos + kvt)
    q = rng.standard_normal((1, nh, hd)).astype(np.float32); k = rng.standard_normal((1, nhkv, hd)).astype(np.float32)
    v = rng.standard_normal((1, nhkv, hd)).astype(np.float32)
    rb_row = row_bytes(kvt, nhkv * hd); rb_head = row_bytes(kvt, hd)
    kf = rng.standard_normal((nkv, nhkv * hd)).astype(np.float32); vf = rng.standard_normal((nkv, nhkv * hd)).astype(np.float32)
    kc = np.zeros((nkv, rb_row), np.uint8); vc = np.zeros((nkv, rb_row), np.uint8)
    ids_all = np.arange(nkv, dtype=np.int64)
    oracle().orc_set_rows(ptr(kf), ptr(ids_all), ptr(kc), kvt, nhkv * hd, nkv, rb_row)
    oracle().orc_set_rows(ptr(vf), ptr(ids_all), ptr(vc), kvt, nhkv * hd, nkv, rb_row)
    mask = np.full((64, nkv), -np.inf, np.float32); mask[0, :pos + 1] = 0
    mask16 = mask.astype(np.float16)
    base = 500000.0
    prm = b200.RopeParams(n_dims=hd, mode=0, n_ctx_orig=8192, freq_base=base, freq_scale=1.0, ext_factor=0.0, attn_factor=1.0,
                          beta_fast=32.0, beta_slow=1.0)
    scale = 1.0 / np.sqrt(hd)
    posn = np.array([pos], np.int32); one = np.array([pos], np.int64)
    qr = np.zeros_like(q); kr = np.zeros_like(k)
    oracle().orc_rope(ptr(q), ptr(qr), ptr(posn), None, hd, nh, 1, hd, 0, 8192, base, 1.0, 0.0, 1.0, 32.0, 1.0)
    oracle().orc_rope(ptr(k), ptr(kr), ptr(posn), None, hd, nhkv, 1, hd, 0, 8192, base, 1.0, 0.0, 1.0, 32.0, 1.0)
    kco, vco = kc.copy(), vc.copy()
    oracle().orc_set_rows(ptr(kr.reshape(1, -1)), ptr(one), ptr(kco), kvt, nhkv * hd, 1, rb_row)
    oracle().orc_set_rows(ptr(v.reshape(1, -1)), ptr(one), ptr(vco), kvt, nhkv * hd, 1, rb_row)
    want = np.zeros((1, nh, hd), np.float32)
    oracle().orc_flash_attn_ext(ptr(qr), nh * hd * 4, hd * 4, ptr(kco), rb_row, rb_head, ptr(vco), rb_row, rb_head, ptr(mask16), ptr(want),
                                kvt, hd, hd, nh, nhkv, 1, nkv, scale, 0.0, 0.0)
    posd, idsd, md, kd, vd = dev(posn), dev(one), dev(mask16.view(np.uint16)), dev(k), dev(v)
    tab = torch.zeros(2 * hd, dtype=torch.float32, device="cuda")
    outs = []
    for mode in (0, 0, 1, 1):
        q2 = dev(q); qr2 = torch.zeros_like(q2); kc2, vc2 = dev(kc), dev(vc)
        d2 = torch.full((1, nh, hd), float("nan"), dtype=torch.float32, device="cuda")
        b200.check(b200.lib.b200_rope_kv_flash_attn2(b200.p(q2), b200.p(qr2), b200.p(kd), b200.p(vd), b200.p(posd), None, b200.p(idsd), b200.p(idsd),
                                                     b200.p(kc2), b200.p(vc2), kvt, rb_row, rb_head, rb_row, rb_head, b200.p(md), b200.p(d2),
                                                     hd, nh, nhkv, nkv, C.byref(prm), scale, 0.0, 0.0, None, b200.p(tab), mode, b200.stream()))
        torch.cuda.synchronize()
        assert np.array_equal(kc2.cpu().numpy(), kco) and np.array_equal(vc2.cpu().numpy(), vco)
        outs.append(d2.cpu().numpy())
    for o in outs[1:]:
        assert np.array_equal(outs[0], o)
    check_against_oracle(outs[0], want, kvt, qr, kco, vco, mask16, hd, nh, nhkv, 1, nkv, scale)
