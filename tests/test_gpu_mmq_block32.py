"""GPU: the batched MUL_MAT on Q4_0 / Q5_0 / Q8_0 weights on the tensor cores (int8 wgmma, csrc/mmq_tc32.cu) against the C oracle:
through the C-ABI (b200_mul_mat_q / _q2, padded rows included), through the graph executor, and through libllama.  The block
sums are exact and each block is folded with the oracle's roundings, so ops are held to <= 2e-5 of the output maximum."""
import os

import numpy as np
import pytest

from refutil import F32, Q4_0, Q5_0, Q8_0, have_ref, orc_mul_mat, rand_blocks, ref_quantize_weights, row_bytes

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

TYPES = [Q4_0, Q5_0, Q8_0]
MIN_COLS = 49           # T32_MIN_COLS of mmq.cu: fewer columns stream through the matvec in groups of 8


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def device_weights(b200, t, W, k):
    """native ggml rows -> the library's row layout (repacked; padded with zero blocks when k is not a multiple of 256)"""
    m = W.shape[0]
    kp = b200.lib.b200_padded_k(t, k)
    src = dev(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)]))
    if kp == k:
        b200.check(b200.lib.b200_repack_rows(t, b200.p(src), m, k, b200.stream()))
        return src, kp
    Wd = torch.zeros(m * row_bytes(t, kp) + 64, dtype=torch.uint8, device="cuda")
    b200.check(b200.lib.b200_repack_rows_padded(t, b200.p(src), b200.p(Wd), m, k, 0, b200.stream()))
    torch.cuda.synchronize()
    return Wd, kp


def mul_mat(b200, t, W, x, m, k, n):
    """b200_mul_mat_q2 run twice on NaN-filled outputs: the two results must be the same bits"""
    Wd, kp = device_weights(b200, t, W, k)
    xd = dev(x)
    ws = torch.zeros(b200.lib.b200_mul_mat_q_workspace(t, m, kp, n), dtype=torch.uint8, device="cuda")
    outs = []
    for _ in range(2):
        dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
        b200.check(b200.lib.b200_mul_mat_q2(t, b200.p(Wd), b200.p(xd), k, b200.p(dst), m, m, kp, k, n, b200.p(ws), b200.stream()))
        torch.cuda.synchronize()
        outs.append(dst.cpu().numpy())
    assert np.isfinite(outs[0]).all()
    assert np.array_equal(outs[0], outs[1])
    return outs[0]


def rel_err(got, want):
    return float(np.abs(got - want).max() / np.abs(want).max())


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("m,k,n", [(128, 2048, 128), (256, 4096, 40), (48, 2048, 19), (384, 2048, 300), (1024, 4096, 512)])
def test_block32_vs_oracle(b200, t, m, k, n):
    rng = np.random.default_rng(2000 + m + n + t)
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    x[n // 2, :256] = 0.0                                       # all-zero q8_0 blocks (d = 0)
    err = rel_err(mul_mat(b200, t, W, x, m, k, n), orc_mul_mat(t, W, x, m, n, k))
    assert err <= 2e-5, err


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("n", [MIN_COLS - 1, MIN_COLS, MIN_COLS + 1])
def test_block32_around_the_switch_over(b200, t, n):
    """one column below the tensor-core threshold (column groups through the matvec), at it, and above it"""
    rng = np.random.default_rng(31 + n + t)
    m, k = 200, 1024
    W = rand_blocks(rng, t, m, k)
    x = (rng.standard_normal((n, k)) * 3).astype(np.float32)
    err = rel_err(mul_mat(b200, t, W, x, m, k, n), orc_mul_mat(t, W, x, m, n, k))
    assert err <= 2e-5, err


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("m,k,n", [(40, 29568, 19), (136, 29568, 128), (24, 29568, 300), (8, 96, 64)])
def test_block32_padded_rows(b200, t, m, k, n):
    """k % 256 != 0 (Qwen2-72B ffn_down: 29568 -> 29696): zero weight blocks against zero activations with d = 0, so the sums are
    those of the unpadded rows"""
    rng = np.random.default_rng(t * 100 + m + n)
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    err = rel_err(mul_mat(b200, t, W, x, m, k, n), orc_mul_mat(t, W, x, m, n, k))
    assert err <= 2e-5, err


def test_block32_baseline_shape(b200):
    """BASELINE config 5 shape: ffn_down of Llama-3-8B at Q8_0 (m 4096, k 14336) against a 512-token ubatch; NMSE on a row sample"""
    rng = np.random.default_rng(5)
    t, m, k, n = Q8_0, 4096, 14336, 512
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    got = mul_mat(b200, t, W, x, m, k, n)
    rows = np.concatenate([np.arange(0, 64), np.arange(2000, 2064), np.arange(m - 64, m)])
    want = orc_mul_mat(t, W[rows], x, len(rows), n, k)
    d = (got[:, rows] - want).astype(np.float64)
    nmse = float((d * d).sum() / (want.astype(np.float64) ** 2).sum())
    assert nmse < 1e-10, nmse


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (reference quantiser) not present")
@pytest.mark.parametrize("t", TYPES)
def test_block32_reference_quantised_weights(b200, t):
    """weights quantised by the reference quantiser from N(0, 0.02^2): real f16 block scales, not random bit patterns"""
    rng = np.random.default_rng(77 + t)
    m, k, n = 256, 4096, 200
    W = ref_quantize_weights(t, (rng.standard_normal((m, k)) * 0.02).astype(np.float32))
    x = rng.standard_normal((n, k)).astype(np.float32)
    err = rel_err(mul_mat(b200, t, W, x, m, k, n), orc_mul_mat(t, W, x, m, n, k))
    assert err <= 2e-5, err


def test_block32_through_the_executor():
    """MUL_MAT nodes with a 300-column activation on a Q8_0 and a padded Q5_0 matrix, run directly, then captured in a CUDA graph and replayed"""
    import importlib
    from conftest import load_pkg
    load_pkg()
    G = importlib.import_module("llama_box_b200.graph"); M = importlib.import_module("llama_box_b200.model")
    rng = np.random.default_rng(9)
    n = 300
    cases = [(Q8_0, 384, 2048), (Q5_0, 136, 29568)]
    nl = G.NodeList(); keep = []; outs = []
    for t, m, k in cases:
        W = rand_blocks(rng, t, m, k)
        x = rng.standard_normal((n, k)).astype(np.float32)
        wd = M.Weights(t, m, k, blocks=W); xd = dev(x)
        dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
        nl.add(G.OP_MUL_MAT, G.T(dst.data_ptr(), F32, [m, n]), [wd.t, G.T(xd.data_ptr(), F32, [k, n])])
        keep += [wd, xd]; outs.append((dst, orc_mul_mat(t, W, x, m, n, k)))
    nodes = nl.build()
    ex = G.Executor(0)
    side = torch.cuda.Stream()                                   # the legacy default stream cannot be captured
    graph = torch.cuda.CUDAGraph()

    def check(what):
        torch.cuda.synchronize()
        for dst, want in outs:
            got = dst.cpu().numpy()
            assert np.isfinite(got).all(), what
            assert rel_err(got, want) <= 2e-5, what
            dst.fill_(float("nan"))
        torch.cuda.synchronize()
    with torch.cuda.stream(side):
        ex.compute(nodes, G.EXEC_FUSION)                         # sizes the workspace: nothing may allocate during capture
    check("direct")
    with torch.cuda.graph(graph, stream=side):
        ex.compute(nodes, G.EXEC_FUSION)
    for rep in range(2):
        graph.replay()
        check(f"replay {rep}")
    ex.close()


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (reference build) not present")
@pytest.mark.parametrize("config,ftype,kv", [("llama3-8b", "Q8_0", "q8_0"), ("tinyllama-1.1b", "Q4_0", "f16")])
def test_block32_prompt_through_libllama(tmp_path, tmp_path_factory, config, ftype, kv):
    """a 600-token prompt (a full 512-token ubatch + an 88-token one, both on the tensor-core path) and a few decode steps through
    the unmodified libllama, as close to ggml-cpu as ggml-cpu's own builds are to each other (tests/test_gpu_product.py)"""
    import test_gpu_product as P
    gguf = P.model_file(tmp_path_factory, config, ftype, 2)
    try:
        kw = dict(kv=kv, verify=1, prompt_len=600, gen=9)
        cpu = P.drv(gguf, str(tmp_path / "cpu"), False, **kw)
        others = P.cpu_builds(tmp_path, tmp_path_factory, gguf, **kw)
        gpu = P.drv(gguf, str(tmp_path / "gpu"), True, **kw)
        P.assert_within_reference_self_consistency(gpu, cpu, others, f"{config} {ftype} kv={kv} prompt=600")
    finally:
        P._models.pop((config, ftype, 2), None)
        os.remove(gguf)
