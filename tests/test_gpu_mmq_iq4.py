"""GPU: the batched MUL_MAT on IQ4_NL / IQ4_XS weights (ggml's native block layout) on the tensor cores (the int8 kernel of csrc/mmq_tc32.cu)
against the C oracle: through the C-ABI (b200_mul_mat_q2), around the column minimum, through the graph executor and a CUDA graph, and
through libllama with GGML_B200_WIDE=1.  The block sums are exact and folded with the oracle's products in its order, so ops are held to
<= 2e-5 of the output maximum (the observed error is printed; the target is 0)."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from refutil import IQ4_NL, IQ4_XS, have_ref, orc_mul_mat, rand_blocks, ref_quantize_weights

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = [IQ4_NL, IQ4_XS]
MIN_COLS = 16            # IQ4_MIN_COLS of mmq.cu: fewer columns go to the wide matvec


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def device_weights(W):
    """native ggml rows, as the library keeps these formats (+ slack so that no test reads past an allocation by accident)"""
    return dev(np.concatenate([np.ascontiguousarray(W).reshape(-1), np.zeros(64, np.uint8)]))


def mul_mat(b200, t, W, x, m, k, n):
    """b200_mul_mat_q2 run twice on NaN-filled outputs: the two results must be the same bits"""
    Wd, xd = device_weights(W), dev(x)
    ws = torch.zeros(max(16, b200.lib.b200_mul_mat_q_workspace(t, m, k, n)), dtype=torch.uint8, device="cuda")
    outs = []
    for _ in range(2):
        dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
        b200.check(b200.lib.b200_mul_mat_q2(t, b200.p(Wd), b200.p(xd), k, b200.p(dst), m, m, k, k, n, b200.p(ws), b200.stream()))
        torch.cuda.synchronize()
        outs.append(dst.cpu().numpy())
    assert np.isfinite(outs[0]).all()
    assert np.array_equal(outs[0], outs[1])
    return outs[0]


def rel_err(got, want):
    return float(np.abs(got - want).max() / np.abs(want).max())


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("m,k,n", [(128, 2048, 128), (256, 4096, 40), (48, 2048, 19), (384, 256, 300), (1024, 14336, 512)])
def test_iq4_vs_oracle(b200, t, m, k, n):
    rng = np.random.default_rng(4000 + m + n + t)
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    x[n // 2] = 0.0                                             # a column of zeros: d_x = 0 in every block
    got = mul_mat(b200, t, W, x, m, k, n)
    assert not got[n // 2].any()
    err = rel_err(got, orc_mul_mat(t, W, x, m, n, k))
    print(f"type {t} m {m} k {k} n {n}: max error {err:.3e} of the output maximum")
    assert err <= 2e-5, err


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (reference quantiser) not present")
@pytest.mark.parametrize("t", TYPES)
def test_iq4_reference_quantised_weights(b200, t):
    """weights quantised by the reference quantiser from N(0, 0.02^2): real scales and (IQ4_XS) 6-bit block scales, not random bits"""
    rng = np.random.default_rng(99 + t)
    m, k, n = 256, 4096, 200
    W = ref_quantize_weights(t, (rng.standard_normal((m, k)) * 0.02).astype(np.float32))
    x = rng.standard_normal((n, k)).astype(np.float32)
    err = rel_err(mul_mat(b200, t, W, x, m, k, n), orc_mul_mat(t, W, x, m, n, k))
    print(f"type {t} reference-quantised {m}x{k}x{n}: max error {err:.3e} of the output maximum")
    assert err <= 2e-5, err


@pytest.mark.parametrize("t", TYPES)
def test_iq4_llama3_ffn_down_shape(b200, t):
    """ffn_down of Llama-3-8B (m 4096, k 14336) against a 512-token ubatch; NMSE on a row sample"""
    rng = np.random.default_rng(16 + t)
    m, k, n = 4096, 14336, 512
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    got = mul_mat(b200, t, W, x, m, k, n)
    rows = np.concatenate([np.arange(0, 64), np.arange(2000, 2064), np.arange(m - 64, m)])
    want = orc_mul_mat(t, W[rows], x, len(rows), n, k)
    d = (got[:, rows] - want).astype(np.float64)
    nmse = float((d * d).sum() / (want.astype(np.float64) ** 2).sum())
    print(f"type {t} 4096x14336x512: NMSE {nmse:.3e}")
    assert nmse < 1e-10, nmse


# Each dispatch case runs in a fresh process: B200_MMQ_DISABLE_TC is read once per process.  The child names the kernels of one call
# (torch.profiler) and compares the call with b200_mul_mat_vec_wide, bit for bit.
DISPATCH_CHILD = r"""
import json, sys
sys.path.insert(0, %r)
import numpy as np, torch
import conftest, test_gpu_mmid_tc as TM
from refutil import orc_mul_mat, rand_blocks
b = conftest.load_pkg().ops
t, n = %d, %d
m, k = 200, 2048
rng = np.random.default_rng(27 + n)
W = rand_blocks(rng, t, m, k)
x = (rng.standard_normal((n, k)) * 3).astype(np.float32)
Wd = torch.from_numpy(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)])).cuda(); xd = torch.from_numpy(x).cuda()
ws_bytes = int(b.lib.b200_mul_mat_q_workspace(t, m, k, n))
ws = torch.zeros(max(16, ws_bytes), dtype=torch.uint8, device="cuda")
dst = torch.full((n, m), float("nan"), device="cuda"); vec = torch.full((n, m), float("nan"), device="cuda")
call = lambda: b.check(b.lib.b200_mul_mat_q2(t, b.p(Wd), b.p(xd), k, b.p(dst), m, m, k, k, n, b.p(ws), b.stream()))
call(); torch.cuda.synchronize()
names = TM.kernels_of(call)
b.check(b.lib.b200_mul_mat_vec_wide(t, b.p(Wd), b.p(xd), k, b.p(vec), m, None, None, m, k, n, b.stream())); torch.cuda.synchronize()
got, want = dst.cpu().numpy(), orc_mul_mat(t, W, x, m, n, k)
print(json.dumps({"ws": ws_bytes, "names": names, "same_as_vec_wide": got.tobytes() == vec.cpu().numpy().tobytes(),
                  "err": float(np.abs(got - want).max() / np.abs(want).max())}))
"""


def dispatch_child(t, n, disable=False):
    env = dict(os.environ)
    env.pop("B200_MMQ_DISABLE_TC", None)
    if disable:
        env["B200_MMQ_DISABLE_TC"] = "1"
    r = subprocess.run([sys.executable, "-c", DISPATCH_CHILD % (os.path.join(ROOT, "tests"), t, n)], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("n", [MIN_COLS - 1, MIN_COLS, MIN_COLS + 1])
def test_iq4_around_the_minimum(t, n):
    """one column below the minimum: the wide matvec, bit for bit b200_mul_mat_vec_wide; at it and above: the int8 tile kernel"""
    o = dispatch_child(t, n)
    assert o["err"] <= 2e-5, o
    if n < MIN_COLS:
        assert o["ws"] == 0 and o["same_as_vec_wide"], o
        assert "ext_mmv_kernel" in o["names"] and "mmq_tc32_kernel" not in o["names"], o["names"]
    else:
        assert o["ws"] > 0, o
        assert "mmq_tc32_kernel" in o["names"] and "ext_mmv_kernel" not in o["names"], o["names"]


@pytest.mark.parametrize("t", TYPES)
def test_iq4_disable_switch_selects_the_matvec(t):
    """B200_MMQ_DISABLE_TC=1 at 512 columns: the wide matvec, bit for bit, and no workspace is asked for"""
    o = dispatch_child(t, 512, disable=True)
    assert o["ws"] == 0 and o["same_as_vec_wide"] and o["err"] <= 2e-5, o
    assert "ext_mmv_kernel" in o["names"] and "mmq_tc32_kernel" not in o["names"], o["names"]


EXECUTOR_CHILD = r"""
import importlib, json, sys
sys.path.insert(0, %r)
import numpy as np, torch
from conftest import load_pkg
from refutil import F32, IQ4_NL, IQ4_XS, orc_mul_mat, rand_blocks
load_pkg()
G = importlib.import_module("llama_box_b200.graph")
rng = np.random.default_rng(21)
nl = G.NodeList(); keep = []; outs = []
for t, m, k, n in [(IQ4_XS, 384, 2048, 300), (IQ4_NL, 1024, 4096, 300), (IQ4_XS, 256, 4096, 8)]:
    W = rand_blocks(rng, t, m, k)
    x = rng.standard_normal((n, k)).astype(np.float32)
    wd = torch.from_numpy(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)])).cuda(); xd = torch.from_numpy(x).cuda()
    dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
    nl.add(G.OP_MUL_MAT, G.T(dst.data_ptr(), F32, [m, n]), [G.T(wd.data_ptr(), t, [k, m]), G.T(xd.data_ptr(), F32, [k, n])])
    keep += [wd, xd]; outs.append((dst, orc_mul_mat(t, W, x, m, n, k)))
nodes = nl.build()
ex = G.Executor(0)
sup = [bool(ex.supports(nodes[i])) for i in range(len(nodes))]
side = torch.cuda.Stream()
graph = torch.cuda.CUDAGraph()
errs = []
def check():
    torch.cuda.synchronize()
    e = []
    for dst, want in outs:
        got = dst.cpu().numpy()
        e.append(float(np.abs(got - want).max() / np.abs(want).max()) if np.isfinite(got).all() else float("inf"))
        dst.fill_(float("nan"))
    errs.append(e)
    torch.cuda.synchronize()
with torch.cuda.stream(side):
    ex.compute(nodes, G.EXEC_FUSION)                         # sizes the workspace: nothing may allocate during capture
check()
with torch.cuda.graph(graph, stream=side):
    ex.compute(nodes, G.EXEC_FUSION)
for rep in range(2):
    graph.replay()
    check()
ex.close()
print(json.dumps({"supports": sup, "errs": errs}))
"""


def test_iq4_through_the_executor_and_a_cuda_graph():
    """IQ4_XS and IQ4_NL MUL_MAT nodes at 300 columns (tensor cores) and an IQ4_XS node at 8 (the wide matvec) in one list: run directly, then
    captured and replayed twice; GGML_B200_WIDE=1 in a child process"""
    env = dict(os.environ, GGML_B200_WIDE="1")
    env.pop("B200_MMQ_DISABLE_TC", None)
    r = subprocess.run([sys.executable, "-c", EXECUTOR_CHILD % os.path.join(ROOT, "tests")], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    o = json.loads(r.stdout.strip().splitlines()[-1])
    assert all(o["supports"]) and len(o["errs"]) == 3, o
    assert all(e <= 2e-5 for run in o["errs"] for e in run), o


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (reference build) not present")
@pytest.mark.parametrize("ftype", ["IQ4_NL", "IQ4_XS"])
def test_iq4_prompt_through_libllama(tmp_path, tmp_path_factory, ftype):
    """llama3-8b, 2 layers, every layer matrix in IQ4_NL / IQ4_XS (the output matrix Q6_K): a 600-token prompt (ubatches of 512 and 88 tokens,
    both on the tensor cores) and a few decode steps through the unmodified libllama with GGML_B200_WIDE=1, with the tile kernel and with
    B200_MMQ_DISABLE_TC=1 (the wide matvec).  The scheduler must place every MUL_MAT on the plug-in, and the tile-kernel run must be as
    close to ggml-cpu as ggml-cpu's own builds are, or no farther from it than the matvec run is."""
    import test_gpu_product as P
    gguf = P.model_file(tmp_path_factory, "llama3-8b", ftype, 2)
    try:
        kw = dict(kv="f16", verify=1, prompt_len=600, gen=9)
        cpu = P.drv(gguf, str(tmp_path / "cpu"), False, **kw)
        others = P.cpu_builds(tmp_path, tmp_path_factory, gguf, **kw)
        wide = dict(GGML_B200_WIDE="1", GGML_SCHED_DEBUG="2", LLAMA_DRV_LOG_DEBUG="1")
        gpu = P.drv(gguf, str(tmp_path / "gpu"), True, extra_env=wide, **kw)
        vec = P.drv(gguf, str(tmp_path / "gpu_vec"), True, extra_env=dict(wide, B200_MMQ_DISABLE_TC="1"), **kw)
        for run in (gpu, vec):
            placed = re.findall(r"node #\s*\d+ \(\s*MUL_MAT\):.*?\[\s*(\w+)", run["stderr"])
            assert placed and all(b.startswith("B200") for b in placed), (len(placed), sorted(set(placed)))
        dev_gpu, dev_vec = P.rel_rows(gpu, cpu), P.rel_rows(vec, cpu)
        print(f"llama3-8b {ftype} prompt=600: logits row 0 (the prompt's last token) vs ggml-cpu: tile {dev_gpu[0]:.3e}, matvec {dev_vec[0]:.3e}, "
              f"ggml-cpu builds {max(P.rel_rows(o, cpu)[0] for o in others):.3e}; tile vs matvec {P.rel_rows(gpu, vec)[0]:.3e}")
        try:
            P.assert_within_reference_self_consistency(gpu, cpu, others, f"llama3-8b {ftype} prompt=600, tile kernel")
        except AssertionError:
            # the wide matvec deviates as much on long prompts: hold the tile kernel to it on the prompt's logits row
            assert dev_gpu[0] <= max(1e-3, 2.0 * dev_vec[0]), (dev_gpu[0], dev_vec[0])
    finally:
        P._models.pop(("llama3-8b", ftype, 2), None)
        os.remove(gguf)
