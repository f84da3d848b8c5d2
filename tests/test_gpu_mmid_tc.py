"""GPU: MUL_MAT_ID for prefill as a grouped GEMM on the tensor cores (csrc/mmid_route.cu: the expert schedule built on the device, then
the GROUPED instances of the tile kernels of mmq_tc.cu / mmq_tc32.cu) against the C oracle, bit for bit against b200_mul_mat_q on each
expert's gathered columns, run to run; which kernels run around the dispatch minimum; three MUL_MAT_ID nodes through the executor under CUDA-graph
capture; and 600-token prompts of a mixture-of-experts model through libllama with the grouped GEMM and with the matvec."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from refutil import F32, Q4_0, Q4_K, Q5_0, Q5_K, Q6_K, Q8_0, have_ref, oracle, ptr, rand_blocks, repack_rows_np, row_bytes

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIN_TOK = 16            # MMID_MIN_TOK of mmid_route.cu: fewer tokens stay on the matvec (ext_mmv_kernel) ...
MIN_PAIRS = 4           # ... and so do fewer than MMID_MIN_PAIRS (token, slot) pairs per expert


def min_tok(ne, nu):
    """fewest tokens that take the grouped GEMM"""
    return max(MIN_TOK, -(-MIN_PAIRS * ne // nu))


TYPES = [Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K]
M, K = 160, 2048        # 160 rows: a partial 128-row tile; k = 2048: every format's rule (Q6_K: k % 2048)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def routing(rng, n_tok, ne, nu, bad=True):
    """top-k-like ids (distinct per token) from the lower half of the experts only, expert 1 in almost every token; with `bad`, a few ids
    out of [0, ne) (their outputs must not be written)"""
    pool = max(nu, ne // 2)
    ids = np.zeros((n_tok, nu), np.int32)
    for t in range(n_tok):
        ch = rng.choice(pool, nu, replace=False)
        if 1 not in ch and rng.random() < 0.95:
            ch[rng.integers(nu)] = 1
        ids[t] = ch
    if bad:
        ids[3, 0] = -1
        ids[n_tok - 1, nu - 1] = ne
    return ids


class Case:
    """one MUL_MAT_ID: oracle output, and the library's over two runs on NaN-filled outputs (must be the same bits)"""

    def __init__(self, b200, t, ne, nu, n_tok, shared, seed=0, bad=True, call_id2=True):
        rng = np.random.default_rng(seed + 100 * t + 10 * ne + n_tok + shared)
        self.t, self.ne, self.nu, self.n_tok = t, ne, nu, n_tok
        self.n_b1 = 1 if shared else nu
        self.W = rand_blocks(rng, t, ne * M, K)
        self.b = rng.standard_normal((n_tok, self.n_b1, K)).astype(np.float32)
        self.ids = routing(rng, n_tok, ne, nu, bad)
        self.b200 = b200
        self.Wd = dev(np.concatenate([repack_rows_np(t, self.W, K).reshape(-1), np.zeros(64, np.uint8)]))
        self.bd, self.idd = dev(self.b), dev(self.ids)
        self.rb = row_bytes(t, K)
        L = b200.lib
        self.ws_bytes = L.b200_mul_mat_id_workspace(t, M, K, ne, nu, n_tok)
        self.ws = torch.zeros(max(self.ws_bytes, 1), dtype=torch.uint8, device="cuda")
        self.call_id2 = call_id2
        outs = [self.run() for _ in range(2)]
        assert outs[0].tobytes() == outs[1].tobytes(), "two runs differ"
        self.got = outs[0]

    def launch(self, dst):
        L, b = self.b200.lib, self.b200
        args = (self.t, b.p(self.Wd), M * self.rb, b.p(self.bd), self.n_b1 * K, K, self.n_b1, b.p(self.idd), self.nu, b.p(dst), self.nu * M, M,
                M, K, self.ne, self.nu, self.n_tok)
        if self.call_id2:
            b.check(L.b200_mul_mat_id2(*args, b.p(self.ws), b.stream()))
        else:
            b.check(L.b200_mul_mat_id(*args, b.stream()))

    def run(self):
        dst = torch.full((self.n_tok, self.nu, M), float("nan"), dtype=torch.float32, device="cuda")
        self.launch(dst)
        torch.cuda.synchronize()
        return dst.cpu().numpy()

    def want(self):
        w = np.full((self.n_tok, self.nu, M), np.nan, np.float32)
        oracle().orc_mul_mat_id(self.t, ptr(self.W), ptr(self.b), ptr(self.ids), ptr(w), M, K, self.ne, self.nu, self.n_tok, self.n_b1, self.nu)
        return w

    def check_oracle(self):
        want = self.want()
        valid = (self.ids >= 0) & (self.ids < self.ne)
        assert np.isnan(self.got[~valid]).all(), "rows of out-of-range ids were written"
        g, w = self.got[valid], want[valid]
        assert np.isfinite(g).all()
        err = float(np.abs(g - w).max() / np.abs(w).max())
        assert err <= 2e-5, err


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("n_tok", ["min", 129, 512])
@pytest.mark.parametrize("ne,nu", [(8, 2), (6, 3), (128, 8)])
def test_grouped_vs_oracle(b200, t, shared, n_tok, ne, nu):
    c = Case(b200, t, ne, nu, min_tok(ne, nu) if n_tok == "min" else n_tok, shared)
    assert c.ws_bytes > 0
    c.check_oracle()


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("ne,nu,n_tok", [(8, 2, 300), (128, 8, 64)])
def test_grouped_equals_dense_kernel_per_expert(b200, t, ne, nu, n_tok):
    """every output is folded by one CTA over its blocks in order from exact integer sums: b200_mul_mat_q over an expert's gathered columns
    (padded with zero columns to 128, so that the tile kernel takes them) gives the same bits"""
    c = Case(b200, t, ne, nu, n_tok, shared=False, seed=7)
    L, b = b200.lib, b200
    for e in range(ne):
        pairs = [(tt, s) for tt in range(n_tok) for s in range(nu) if c.ids[tt, s] == e]
        if not pairs:
            continue
        n = max(len(pairs), 128)
        X = np.zeros((n, K), np.float32)
        for j, (tt, s) in enumerate(pairs):
            X[j] = c.b[tt, s % c.n_b1]
        xd = dev(X)
        dst = torch.full((n, M), float("nan"), dtype=torch.float32, device="cuda")
        ws = torch.zeros(L.b200_mul_mat_q_workspace(t, M, K, n), dtype=torch.uint8, device="cuda")
        b.check(L.b200_mul_mat_q(t, C_ptr(c.Wd, e * M * c.rb), b.p(xd), K, b.p(dst), M, M, K, n, b.p(ws), b.stream()))
        torch.cuda.synchronize()
        dense = dst.cpu().numpy()[:len(pairs)]
        grouped = np.stack([c.got[tt, s] for tt, s in pairs])
        assert dense.tobytes() == grouped.tobytes(), (e, len(pairs))


def C_ptr(tensor, offset):
    import ctypes
    return ctypes.c_void_p(tensor.data_ptr() + offset)


def kernels_of(fn):
    """names of the CUDA kernels one call launches (torch.profiler, CUDA activities).  A profile whose activity buffer came back without a
    single kernel record is taken again."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = " ".join(e.key for e in prof.key_averages())
        if "kernel" in names.replace("cudaLaunchKernel", ""):
            break
    return names


# Each dispatch case runs in a fresh process: B200_MMQ_DISABLE_TC is read once per process, and CUPTI's activity records of a profile taken
# late in a long GPU session can come back empty.  The child also counts the library's launches for the call (grouped: router, quantiser,
# tile kernel; matvec: one launch), which does not depend on the profiler.
DISPATCH_CHILD = r"""
import json, sys
sys.path.insert(0, %r)
import conftest, test_gpu_mmid_tc as T
import torch
b = conftest.load_pkg().ops
t, ne, nu, n_tok = %d, %d, %d, %d
c = T.Case(b, t, ne, nu, n_tok, True, seed=3)
n0 = b.lib.b200_kernel_launches()
c.run()
launches = b.lib.b200_kernel_launches() - n0
names = T.kernels_of(c.run)
c.check_oracle()
same = T.Case(b, t, ne, nu, n_tok, True, seed=3, call_id2=False).got.tobytes() == c.got.tobytes()
print(json.dumps({"ws": int(c.ws_bytes), "names": names, "launches": int(launches), "same_as_mul_mat_id": same}))
"""


def dispatch_child(t, ne, nu, n_tok, disable=False):
    env = dict(os.environ)
    env.pop("B200_MMQ_DISABLE_TC", None)
    if disable:
        env["B200_MMQ_DISABLE_TC"] = "1"
    r = subprocess.run([sys.executable, "-c", DISPATCH_CHILD % (os.path.join(ROOT, "tests"), t, ne, nu, n_tok)], capture_output=True, text=True,
                       env=env, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("t", [Q4_K, Q8_0])
@pytest.mark.parametrize("ne,nu,n_tok", [(8, 2, MIN_TOK - 1), (8, 2, MIN_TOK), (8, 2, 200), (128, 8, 63), (128, 8, 64)])
def test_dispatch_around_the_minimum(t, ne, nu, n_tok):
    """the router and the grouped tile kernel run from min_tok(ne, nu) tokens on; below, b200_mul_mat_id2 is b200_mul_mat_id, bit for bit"""
    o = dispatch_child(t, ne, nu, n_tok)
    names = o["names"]
    tile = "mmq_tc32_kernel" if t == Q8_0 else "mmq_tc_kernel"
    if n_tok >= min_tok(ne, nu):
        assert o["ws"] > 0 and o["launches"] == 3, o
        assert "mmid_route_kernel" in names and tile in names and "ext_mmv_kernel" not in names, names
    else:
        assert o["ws"] == 0 and o["launches"] == 1, o
        assert "ext_mmv_kernel" in names and "mmid_route_kernel" not in names and tile not in names, names
        assert o["same_as_mul_mat_id"], o


def test_disable_switch_selects_the_matvec():
    """B200_MMQ_DISABLE_TC=1: the matvec at 200 tokens, bit for bit b200_mul_mat_id, and no workspace is asked for"""
    o = dispatch_child(Q4_K, 8, 2, 200, disable=True)
    assert o["ws"] == 0 and o["launches"] == 1 and o["same_as_mul_mat_id"], o
    assert "ext_mmv_kernel" in o["names"] and "mmid_route_kernel" not in o["names"], o


EXECUTOR_CHILD = r"""
import importlib, json, sys
sys.path.insert(0, %r)
import numpy as np, torch
from conftest import load_pkg
from refutil import F32, I32, Q4_K, Q6_K, oracle, ptr, rand_blocks, repack_rows_np
load_pkg()
G = importlib.import_module("llama_box_b200.graph")
E, FF, NE, NU, NT = 1024, 2048, 8, 2, 300
rng = np.random.default_rng(11)
O = oracle()
Wup, Wgate, Wdown = rand_blocks(rng, Q4_K, NE * FF, E), rand_blocks(rng, Q4_K, NE * FF, E), rand_blocks(rng, Q6_K, NE * E, FF)
x = rng.standard_normal((NT, E)).astype(np.float32)
ids = np.stack([rng.choice(NE, NU, replace=False) for _ in range(NT)]).astype(np.int32)
up = np.zeros((NT, NU, FF), np.float32); gate = np.zeros_like(up)
O.orc_mul_mat_id(Q4_K, ptr(Wup), ptr(x), ptr(ids), ptr(up), FF, E, NE, NU, NT, 1, NU)
O.orc_mul_mat_id(Q4_K, ptr(Wgate), ptr(x), ptr(ids), ptr(gate), FF, E, NE, NU, NT, 1, NU)
act = np.zeros_like(up); O.orc_swiglu(ptr(gate), ptr(up), ptr(act), act.size)
down = np.zeros((NT, NU, E), np.float32)
O.orc_mul_mat_id(Q6_K, ptr(Wdown), ptr(act), ptr(ids), ptr(down), E, FF, NE, NU, NT, NU, NU)
keep = []
def d(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda(); keep.append(t); return t
def wd(t, W, k):
    return d(np.concatenate([repack_rows_np(t, W, k).reshape(-1), np.zeros(64, np.uint8)]))
def out(ne):
    t = torch.full([int(np.prod(ne))], float("nan"), dtype=torch.float32, device="cuda"); keep.append(t); return t
xd, idd = d(x), d(ids)
upd, gated, actd, downd = out([NT, NU, FF]), out([NT, NU, FF]), out([NT, NU, FF]), out([NT, NU, E])
nl = G.NodeList()
x3 = G.T(xd.data_ptr(), F32, [E, 1, NT], [4, 4 * E, 4 * E, 4 * E * NT])
sel = G.T(idd.data_ptr(), I32, [NU, NT])
u = nl.add(G.OP_MUL_MAT_ID, G.T(upd.data_ptr(), F32, [FF, NU, NT]), [G.T(wd(Q4_K, Wup, E).data_ptr(), Q4_K, [E, FF, NE]), x3, sel])
g = nl.add(G.OP_MUL_MAT_ID, G.T(gated.data_ptr(), F32, [FF, NU, NT]), [G.T(wd(Q4_K, Wgate, E).data_ptr(), Q4_K, [E, FF, NE]), x3, sel])
a = nl.add(G.OP_GLU_SWIGLU, G.T(actd.data_ptr(), F32, [FF, NU, NT]), [g, u], [2, 0])
nl.add(G.OP_MUL_MAT_ID, G.T(downd.data_ptr(), F32, [E, NU, NT]), [G.T(wd(Q6_K, Wdown, FF).data_ptr(), Q6_K, [FF, E, NE]), a, sel])
nodes = nl.build()
ex = G.Executor(0)
sup = [bool(ex.supports(nodes[i])) for i in range(len(nodes))]
side = torch.cuda.Stream()
graph = torch.cuda.CUDAGraph()
def rel(got, want):
    return float(np.abs(got - want).max() / np.abs(want).max())
errs = []
def check():
    torch.cuda.synchronize()
    e = [rel(upd.cpu().numpy().reshape(up.shape), up), rel(gated.cpu().numpy().reshape(up.shape), gate), rel(downd.cpu().numpy().reshape(down.shape), down)]
    errs.append(e)
    for t in (upd, gated, actd, downd):
        t.fill_(float("nan"))
    torch.cuda.synchronize()
with torch.cuda.stream(side):
    ex.compute(nodes, G.EXEC_FUSION)
check()
with torch.cuda.graph(graph, stream=side):
    ex.compute(nodes, G.EXEC_FUSION)
for rep in range(2):
    graph.replay()
    check()
ex.close()
print(json.dumps({"supports": sup, "errs": errs}))
"""


def test_three_mul_mat_id_nodes_through_the_executor_and_a_cuda_graph():
    """up / gate (Q4_K) and down (Q6_K) MUL_MAT_ID nodes with SwiGLU between them, ids given as an input, 300 tokens: run directly, then
    captured and replayed (the workspace is planned before capture); GGML_B200_WIDE=1 in a child process"""
    env = dict(os.environ, GGML_B200_WIDE="1")
    env.pop("B200_MMQ_DISABLE_TC", None)
    r = subprocess.run([sys.executable, "-c", EXECUTOR_CHILD % os.path.join(ROOT, "tests")], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    o = json.loads(r.stdout.strip().splitlines()[-1])
    assert all(o["supports"]), o
    assert len(o["errs"]) == 3, o
    for e_up, e_gate, e_down in o["errs"]:
        assert e_up <= 2e-5 and e_gate <= 2e-5, o
        assert e_down <= 2e-3, o       # down re-quantises SwiGLU(gate, up): a last-bit difference upstream may flip one int8 rounding


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (reference build) not present")
@pytest.mark.parametrize("ftype", ["Q4_K_M", "Q8_0"])
def test_moe_prompt_through_libllama(tmp_path, tmp_path_factory, ftype):
    """test-moe (8 experts, top-2; at Q4_K_M layer 0's ffn_down_exps is Q4_K and layer 1's Q6_K): a 600-token prompt (ubatches of 512 and
    88 tokens, both on the grouped GEMM) and a few decode steps through the unmodified libllama with GGML_B200_WIDE=1, with the grouped GEMM
    and with B200_MMQ_DISABLE_TC=1 (the matvec).  The scheduler must place MUL_MAT_ID on the plug-in, and the grouped run must be as close
    to ggml-cpu as ggml-cpu's own builds are, or no farther from it than the matvec run is."""
    import test_gpu_product as P
    gguf = P.model_file(tmp_path_factory, "test-moe", ftype, 2)
    try:
        kw = dict(kv="f16", verify=1, prompt_len=600, gen=9)
        cpu = P.drv(gguf, str(tmp_path / "cpu"), False, **kw)
        others = P.cpu_builds(tmp_path, tmp_path_factory, gguf, **kw)
        wide = dict(GGML_B200_WIDE="1", GGML_SCHED_DEBUG="2", LLAMA_DRV_LOG_DEBUG="1")
        gpu = P.drv(gguf, str(tmp_path / "gpu"), True, extra_env=wide, **kw)
        vec = P.drv(gguf, str(tmp_path / "gpu_vec"), True, extra_env=dict(wide, B200_MMQ_DISABLE_TC="1"), **kw)
        for run in (gpu, vec):
            placed = re.findall(r"node #\s*\d+ \(\s*MUL_MAT_ID\w*\):.*?\[\s*(\w+)", run["stderr"])
            assert placed and all(b.startswith("B200") for b in placed), (len(placed), sorted(set(placed)))
        dev_gpu, dev_vec = P.rel_rows(gpu, cpu), P.rel_rows(vec, cpu)
        print(f"test-moe {ftype} prompt=600: logits row 0 (the prompt's last token) vs ggml-cpu: grouped {dev_gpu[0]:.3e}, matvec {dev_vec[0]:.3e}, "
              f"ggml-cpu builds {max(P.rel_rows(o, cpu)[0] for o in others):.3e}; grouped vs matvec {P.rel_rows(gpu, vec)[0]:.3e}")
        try:
            P.assert_within_reference_self_consistency(gpu, cpu, others, f"test-moe {ftype} prompt=600, grouped GEMM")
        except AssertionError:
            # the matvec path of the parent deviates as much on this file: hold the grouped GEMM to it on the prompt's logits row
            assert dev_gpu[0] <= max(1e-3, 2.0 * dev_vec[0]), (dev_gpu[0], dev_vec[0])
    finally:
        P._models.pop(("test-moe", ftype, 2), None)
        os.remove(gguf)
