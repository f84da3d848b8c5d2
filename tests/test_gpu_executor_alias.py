"""The graph executor's fusions over recycled buffers, layer by layer against the oracle.

The executor decides what fuses by reasoning about buffer addresses (hoisting a projection, grouping Q/K/V, eliding a norm
into a matvec prologue, folding a residual ADD into an epilogue).  libllama's graph allocator (ggml-alloc.c) reuses freed
buffers and puts ADD / MUL / RMS_NORM / ROPE results in place over their parent, so every list the plug-in hands over
aliases.  A wrong guard does not crash: a fused launch reads a buffer a later node already overwrote, and a few rows are
wrong.  Here SyntheticLlama's node lists are placed in one arena by three policies:
  fresh    every intermediate its own buffer (the control);
  gallocr  the reference allocator's rules: in place over the parent when the op can work in place, the parent is the
           arena's, not an output, this node is its last reader and the layouts match; otherwise the best fit from the
           free list; a buffer is freed after its last reader; a view keeps its parent alive;
  tight    the same legality, but each result takes the LOWEST free block that fits, so inputs are overwritten by the
           first node that may legally land on them.
Each layer runs with hidden_in set to the oracle's input for that layer and KV cells before the current position holding
the same oracle-written bytes on both sides; its output, its new KV rows and (last layer) its logits are compared with
tests/oracle_model.OracleLlama.  Between policies and execution modes the comparisons are bitwise or at 2e-5.

The CPU part (allocator, planned launch counts) runs without a GPU."""
import collections
import difflib
import functools
import os
import subprocess
import sys
import tempfile
import types as pytypes

import numpy as np
import pytest

from oracle_model import OracleLlama, causal_mask, make_host_weights
from refutil import F16, Q8_0, oracle, ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALIGN = 128                 # the plug-in's buffer alignment (ggml_backend_b200_buffer_type_get_alignment)
POLICIES = ("fresh", "gallocr", "tight")


def mods():
    import importlib
    from conftest import load_pkg
    load_pkg()
    return importlib.import_module("llama_box_b200.graph"), importlib.import_module("llama_box_b200.model")


# ---------------------------------------------------------------------------------------------------------- allocator
def nbytes(t):
    es = {0: 4, 1: 2, 26: 4, 27: 8}[t.type]
    return es + sum((t.ne[i] - 1) * t.nb[i] for i in range(4))


class Arena:
    """placement hook for SyntheticLlama.build: every intermediate goes into one arena at ALIGN-byte offsets.
    mark_output(items) may name intermediates to flag OUTPUT first (they are then never freed nor reused)."""

    def __init__(self, policy, device="cuda", mark_output=None):
        assert policy in POLICIES
        self.policy, self.device, self.mark_output = policy, device, mark_output

    def __call__(self, nl, fixed):
        G, _ = mods()
        inplace_ops = (G.OP_ADD, G.OP_MUL, G.OP_RMS_NORM, G.OP_ROPE, G.OP_SCALE, G.OP_SOFT_MAX)    # ggml_op_can_inplace, of the ops here
        self.nl, items = nl, nl.items
        if self.mark_output:
            for t in self.mark_output(items):
                t.flags |= G.FLAG_OUTPUT
        fixed_ids = {t.id for t in fixed}
        root = {}                                        # tensor id -> the arena tensor whose storage it is (itself, or a view's parent)
        for op, dst, srcs, _ in items:
            if op == G.OP_NONE:
                if srcs[0].id in root:
                    root[dst.id] = root[srcs[0].id]
            elif op != G.OP_SET_ROWS and dst.id not in fixed_ids:
                root[dst.id] = dst
        readers = collections.Counter(root[s.id].id for op, _, srcs, _ in items if op != G.OP_NONE for s in srcs if s is not None and s.id in root)
        self.block, self.inplace = {}, {}                # root id -> (offset, size); in-place result id -> parent id
        free, live, handed_over = [], {}, set()
        top = [0, 0]                                     # current end, high-water mark

        def alloc(size):
            fits = [b for b in free if b[1] >= size]
            if fits:
                b = min(fits, key=lambda b: (b[1], b[0])) if self.policy == "gallocr" else min(fits)
                free.remove(b)
                if b[1] > size:
                    free.append((b[0] + size, b[1] - size))
                return (b[0], size)
            off = top[0]; top[0] += size; top[1] = max(top[1], top[0])
            return (off, size)

        def release(off, size):
            free.append((off, size)); free.sort()
            merged = []
            for b in free:
                if merged and merged[-1][0] + merged[-1][1] == b[0]:
                    merged[-1] = (merged[-1][0], merged[-1][1] + b[1])
                else:
                    merged.append(b)
            if merged and merged[-1][0] + merged[-1][1] == top[0]:
                top[0] = merged.pop()[0]
            free[:] = merged

        for op, dst, srcs, _ in items:
            if op == G.OP_NONE:
                continue
            if root.get(dst.id) is dst:
                size = (nbytes(dst) + ALIGN - 1) // ALIGN * ALIGN
                blk = None
                if self.policy != "fresh" and op in inplace_ops:
                    for s in srcs:
                        p = root.get(s.id) if s is not None else None
                        if p is None or p.flags & G.FLAG_OUTPUT or readers[p.id] != 1 or p.id in handed_over:
                            continue
                        if s.ptr != p.ptr or s.type != dst.type or s.ne != dst.ne or s.nb != dst.nb or self.block[p.id][1] < size:
                            continue
                        blk = self.block[p.id]; self.inplace[dst.id] = p.id; handed_over.add(p.id)
                        del live[p.id]
                        break
                if blk is None:
                    blk = alloc(size)
                for other, ob in live.items():       # self-check: a result never lands on a live buffer
                    assert blk[0] + blk[1] <= ob[0] or ob[0] + ob[1] <= blk[0], (op, dst.id, other)
                self.block[dst.id] = blk; live[dst.id] = blk
            for s in srcs:
                if s is None or s.id not in root:
                    continue
                p = root[s.id]; readers[p.id] -= 1
                if readers[p.id] == 0 and self.policy != "fresh" and not p.flags & G.FLAG_OUTPUT and p.id not in handed_over:
                    release(*live.pop(p.id))
        self.size = top[1] + ALIGN
        if self.device == "cpu":
            base = 1 << 40
        else:
            import torch
            self.buf = torch.empty(self.size, dtype=torch.uint8, device=self.device)
            base = (self.buf.data_ptr() + ALIGN - 1) // ALIGN * ALIGN
        self.base = base
        old = {}
        for op, dst, srcs, _ in items:
            for t in [dst] + [s for s in srcs if s is not None]:
                old.setdefault(id(t), t.ptr)
        for op, dst, srcs, _ in items:
            if op == G.OP_NONE and srcs[0].id in root:
                dst.ptr = srcs[0].ptr + old[id(dst)] - old[id(srcs[0])]
            elif root.get(dst.id) is dst:
                dst.ptr = base + self.block[dst.id][0]

    def span(self, t):
        return (t.ptr - self.base, t.ptr - self.base + nbytes(t))


def overlap(a, b):
    return a[0] < b[1] and b[0] < a[1]


# ---------------------------------------------------------------------------------------------------------- models
BASE = dict(n_embd=2048, n_head=16, n_head_kv=4, head_dim=128, n_ff=4096, n_vocab=4096, n_layer=2, rope_base=500000.0, rope_mode=0, eps=1e-5, qkv_bias=False)
CASES = {
    # name: config changes, weight mix, KV cache type
    "q4km": (dict(), "Q4_K_M", F16),
    "q4_0": (dict(), "Q4_0", F16),
    "q8_0": (dict(), "Q8_0", Q8_0),
    "qwen2": (dict(qkv_bias=True, rope_mode=2, rope_base=1000000.0, eps=1e-6), "Q4_K_M", F16),
    "llama31": (dict(rope_freqs=True), "Q4_K_M", F16),               # rope frequency factors (Llama-3.1's rope_freqs)
    "partial": (dict(rope_n_dims=64), "Q4_0", F16),                   # partial rotary, n_dims = head_dim / 2
    "hd64": (dict(n_head=32, n_head_kv=4, head_dim=64), "Q4_K_M", F16),   # 64-wide heads at TinyLlama's 32 / 4 grouping
}


def case_cfg(name):
    ch, ftype, kv = CASES[name]
    cfg = dict(BASE); cfg.update(ch)
    return cfg, ftype, kv


def host_model(G, M, cfg, ftype="Q4_K_M", kv=F16, layer_range=(0, 2), first=False, last=False, n_ctx=1024):
    """SyntheticLlama's node lists over fake weight and cache addresses and host-side io buffers: what the dry-run planner needs"""
    m = object.__new__(M.SyntheticLlama)
    m.device = "cpu"
    m.c, m.n_ctx, m.kv_type, m.ftype, m.first, m.last, m.n_seq = dict(cfg), n_ctx, kv, ftype, first, last, 1
    m.layer_ids, m.bufs, m.rope_ff, m.tok_embd = list(range(*layer_range)), {}, None, None
    E, H, HK, D, FF, V = cfg["n_embd"], cfg["n_head"], cfg["n_head_kv"], cfg["head_dim"], cfg["n_ff"], cfg["n_vocab"]
    mix, out_t = M.type_mix(ftype, cfg["n_layer"], FF)
    nxt = [1 << 36]

    def addr(nbytes):
        a = nxt[0]; nxt[0] += (nbytes + 0xfffff) & ~0xfffff
        return pytypes.SimpleNamespace(data_ptr=lambda a=a: a)

    def W(t, rows, k):
        return pytypes.SimpleNamespace(t=G.T(addr(rows * G.row_size(t, k)).data_ptr(), t, [k, rows]))
    m.layers = []
    for i in m.layer_ids:
        t = mix[i]
        ly = dict(attn_norm=addr(4 * E), ffn_norm=addr(4 * E), wq=W(t["wq"], H * D, E), wk=W(t["wk"], HK * D, E), wv=W(t["wv"], HK * D, E),
                  wo=W(t["wo"], E, H * D), gate=W(t["gate"], FF, E), up=W(t["up"], FF, E), down=W(t["down"], E, FF))
        if cfg["qkv_bias"]:
            ly.update(bq=addr(4 * H * D), bk=addr(4 * HK * D), bv=addr(4 * HK * D))
        ly["k_caches"] = [addr(n_ctx * G.row_size(kv, HK * D))]; ly["v_caches"] = [addr(n_ctx * G.row_size(kv, HK * D))]
        m.layers.append(ly)
    m.output_norm = addr(4 * E) if last else None
    m.output = W(out_t, V, E) if last else None
    if cfg.get("rope_freqs"):
        import torch
        m.rope_ff = torch.ones(cfg.get("rope_n_dims", D) // 2)
    return m


def named(items, model):
    """the intermediates of each layer by role, found through the weights they are computed from"""
    G, _ = mods()
    out = []
    by_src = collections.defaultdict(list)
    for op, dst, srcs, _ in items:
        for s in srcs:
            if s is not None:
                by_src[s.id].append((op, dst, srcs))

    def after(t, op):
        for o, d, s in by_src[t.id]:
            if o == G.OP_NONE:
                r = after(d, op)
                if r is not None:
                    return r
            elif o == op:
                return d
        return None
    for ly in model.layers:
        mm = {k: next(d for op, d, s, _ in items if op == G.OP_MUL_MAT and s[0].ptr == ly[k].t.ptr) for k in ("wq", "wk", "wv", "wo", "gate", "up", "down")}
        nrm = next(d for op, d, s, _ in items if op == G.OP_MUL and s[1].ptr == ly["attn_norm"].data_ptr())
        fnrm = next(d for op, d, s, _ in items if op == G.OP_MUL and s[1].ptr == ly["ffn_norm"].data_ptr())
        q = after(mm["wq"], G.OP_ADD) or mm["wq"]
        r = dict(mm, normw=nrm, fnormw=fnrm, q=q, qr=after(q, G.OP_ROPE),
                 l_out=after(mm["down"], G.OP_ADD), att=next(d for op, d, s, _ in items if op == G.OP_FLASH_ATTN_EXT),
                 ffn_inp=after(mm["wo"], G.OP_ADD) or after(after(mm["wo"], G.OP_GET_ROWS), G.OP_ADD))
        r["h"] = next(d for op, d, s, _ in items if op == G.OP_GLU_SWIGLU and s[0] is mm["gate"])
        r["norm"] = next(s[0] for op, d, s, _ in items if op == G.OP_MUL and d is nrm)
        r["fnorm"] = next(s[0] for op, d, s, _ in items if op == G.OP_MUL and d is fnrm)
        out.append(r)
    return out


# ---------------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("n_tok", [1, 3, 40])
@pytest.mark.parametrize("case", ["q4km", "qwen2"])
def test_gallocr_lists_alias_like_the_reference_allocator(case, n_tok):
    G, M = mods()
    cfg, ftype, kv = case_cfg(case)
    model = host_model(G, M, cfg, ftype, kv)
    sizes = {}
    for policy in POLICIES:
        a = Arena(policy, "cpu")
        model.build(n_tok, 512, place=a)
        sizes[policy] = a.size
        if policy == "fresh":
            assert not a.inplace
            continue
        for il, t in enumerate(named(a.nl.items, model)):
            sp = {k: a.span(v) for k, v in t.items()}
            # the un-roped Q's buffer is taken by its ROPE in place, or reused for K or V
            assert sp["qr"] == sp["q"] or overlap(sp["q"], sp["wk"]) or overlap(sp["q"], sp["wv"]), (policy, il)
            # ffn_inp in place over wo's output, the norm-weight MULs in place over their RMS_NORM
            assert a.inplace.get(t["ffn_inp"].id) == t["wo"].id, (policy, il)
            assert a.inplace.get(t["normw"].id) == t["norm"].id and a.inplace.get(t["fnormw"].id) == t["fnorm"].id, (policy, il)
            # down / the layer output land on a buffer an earlier fused launch of the same layer read
            read = [sp[k] for k in ("normw", "fnormw", "att", "qr", "wo", "gate", "up")]
            assert any(overlap(sp["down"], r) or overlap(sp["l_out"], r) for r in read), (policy, il)
    assert max(sizes["tight"], sizes["gallocr"]) < sizes["fresh"], sizes


@pytest.mark.parametrize("case", list(CASES))
def test_recycled_decode_layers_keep_the_fused_launch_count(case):
    """without this the GPU comparisons below could pass by quietly not fusing"""
    G, M = mods()
    cfg, ftype, kv = case_cfg(case)
    model = host_model(G, M, cfg, ftype, kv)
    counts = {}
    for policy in POLICIES:
        nodes, _ = model.build(1, 512, place=Arena(policy, "cpu"))
        counts[policy] = G.plan(nodes, G.EXEC_FUSION)
    # norm in the prologue | QKV | rope + KV store + attention | wo + residual | gate/up + SwiGLU | down + residual, + the mask cast;
    # in the fresh list nothing overwrites the last layer's normalised FFN input, so it is also materialised (a caller may read it)
    assert counts == {"fresh": 5 * 2 + 2, "gallocr": 5 * 2 + 1, "tight": 5 * 2 + 1}, counts


# ---------------------------------------------------------------------------------------------------------- GPU harness
FLAGSETS = {"fused": 2, "fused+graphs": 2 | 1, "mega": 2 | 4, "mega+mmv": 2 | 4 | 8}      # EXEC_FUSION, |CUDA_GRAPHS, |MEGAKERNEL, |MEGA_MMV
# bounds on max|gpu - oracle| / max|oracle| of one layer, measured on an H100 80GB HBM3 (700 W): (what, KV cache type) -> bound.
# With an F16 cache the oracle accumulates V in fp16 (ggml-cpu/ops.cpp), which dominates: observed hidden 3.6e-3, logits 8.3e-3,
# new KV rows 6.1e-4 (f16 rounding of the roped K).  With a Q8_0 cache: hidden 4.1e-7, logits 3.4e-7, KV rows bit-identical
# (the KV bound is one Q8_0 step, 1/127 of a block's maximum).  The whole-model bar of test_gpu_executor.py is 3e-2 / 1e-3.
BOUNDS = {("hidden", F16): 6e-3, ("logits", F16): 1.2e-2, ("kv", F16): 1e-3, ("hidden", Q8_0): 2e-6, ("logits", Q8_0): 2e-6, ("kv", Q8_0): 8e-3}
MODES_TOL = 2e-5            # between execution modes and between placements that plan differently (fused vs plain: observed 0)
MEGA_TOL = 1e-4             # the persistent kernel's attention phase splits the KV range its own way: 7.2e-5 observed at n_kv = 512


def rel(a, b):
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def kv_rows(cache, kv_type, rows):
    """dequantised rows of a KV cache image (uint8 [n_ctx, row bytes])"""
    r = np.ascontiguousarray(cache[rows])
    if kv_type == F16:
        return r.view(np.float16).astype(np.float32)
    b = r.reshape(len(rows), -1, 34)
    d = b[:, :, :2].copy().view(np.float16).astype(np.float32)
    return (d * b[:, :, 2:].view(np.int8).astype(np.float32)).reshape(len(rows), -1)


@functools.lru_cache(maxsize=None)
def host_weights(case):
    _, M = mods()
    cfg, ftype, kv = case_cfg(case)
    mix, out_t = M.type_mix(ftype, cfg["n_layer"], cfg["n_ff"])
    hw, types = make_host_weights(cfg, mix, out_t)
    if cfg.get("rope_freqs"):
        hw["rope_freqs"] = np.linspace(1.0, 8.0, cfg.get("rope_n_dims", cfg["head_dim"]) // 2).astype(np.float32)
    return hw, types


class Problem:
    """one ubatch of one case: inputs, oracle results per layer, and the KV bytes both sides start from"""

    def __init__(self, case, n_tok, pos0, n_out, seed=0):
        cfg, ftype, kv = case_cfg(case)
        self.case, self.cfg, self.ftype, self.kv = case, cfg, ftype, kv
        self.n_tok, self.pos0, self.n_ctx = n_tok, pos0, 1024
        self.n_kv = max(256, (pos0 + n_tok + 255) // 256 * 256)
        hw, types = host_weights(case)
        self.hw = hw
        rng = np.random.default_rng(seed + 1000 * pos0 + n_tok)
        orc = OracleLlama(cfg, hw, types, self.n_ctx, kv, hw.get("rope_freqs"))
        HKD = cfg["n_head_kv"] * cfg["head_dim"]
        for il in range(cfg["n_layer"]):                    # the cells before the current position: oracle-written bytes
            if pos0:
                ids = np.arange(pos0, dtype=np.int64)
                for c in (orc.kc[il], orc.vc[il]):
                    rows = rng.standard_normal((pos0, HKD)).astype(np.float32)
                    oracle().orc_set_rows(ptr(rows), ptr(ids), ptr(c), kv, HKD, pos0, orc.kvrow)
        self.kc0 = [c.copy() for c in orc.kc]; self.vc0 = [c.copy() for c in orc.vc]
        self.tokens = rng.integers(0, cfg["n_vocab"], n_tok).astype(np.int32)
        self.pos = np.arange(pos0, pos0 + n_tok, dtype=np.int32); self.kv_idx = self.pos.astype(np.int64)
        self.mask = causal_mask(n_tok, self.n_kv, pos0)
        self.out_ids = np.array(sorted({n_tok - 1, 0, n_tok // 2})[-n_out:] if n_out > 1 else [n_tok - 1], np.int32)
        assert len(self.out_ids) == n_out
        m16 = self.mask.astype(np.float16).view(np.uint16)
        x = np.ascontiguousarray(hw["token_embd"][self.tokens])
        self.x_in, self.want = [], []
        for il in range(cfg["n_layer"]):
            last = il == cfg["n_layer"] - 1
            self.x_in.append(x)
            x = orc.layer(il, x, self.pos, self.kv_idx, self.n_kv, m16, self.out_ids if last else None)
            self.want.append(orc.logits(x) if last else x)
        self.kc1 = orc.kc; self.vc1 = orc.vc

    def model(self, il):
        _, M = mods()
        last = il == self.cfg["n_layer"] - 1
        return M.SyntheticLlama(self.cfg, self.ftype, n_ctx=self.n_ctx, kv_type=self.kv, host_weights=self.hw, layer_range=(il, il + 1), first=False, last=last)


class LayerRun:
    """one layer's list under one placement, run on the GPU"""

    def __init__(self, prob, il, model, policy, mark_output=None):
        import torch
        self.torch, self.prob, self.il, self.model = torch, prob, il, model
        self.last = il == prob.cfg["n_layer"] - 1
        self.arena = Arena(policy, mark_output=mark_output)
        self.nodes, self.io = model.build(prob.n_tok, prob.n_kv, n_out=len(prob.out_ids), place=self.arena)
        self.side = torch.cuda.Stream()

    def run(self, ex, flags, nodes=None, inputs=None):
        torch, p, io, ly = self.torch, self.prob, self.io, self.model.layers[0]
        x_in, pos, mask = inputs if inputs is not None else (p.x_in[self.il], p.pos, p.mask)
        self.arena.buf.fill_(0xff)                       # NaN: every intermediate must be written before it is read
        io["hidden_in"].copy_(torch.from_numpy(x_in)); io["pos"].copy_(torch.from_numpy(pos)); io["kv_idx"].copy_(torch.from_numpy(pos.astype(np.int64)))
        io["mask"].copy_(torch.from_numpy(mask)); io["out_ids"].copy_(torch.from_numpy(p.out_ids))
        ly["k_cache"].copy_(torch.from_numpy(p.kc0[self.il].reshape(-1))); ly["v_cache"].copy_(torch.from_numpy(p.vc0[self.il].reshape(-1)))
        torch.cuda.synchronize()
        with torch.cuda.stream(self.side):
            ex.compute(self.nodes if nodes is None else nodes, flags)
        torch.cuda.synchronize()
        out = (io["logits"] if self.last else io["hidden_out"]).cpu().numpy().copy()
        shape = p.kc0[self.il].shape
        return dict(out=out, k=ly["k_cache"].cpu().numpy().reshape(shape), v=ly["v_cache"].cpu().numpy().reshape(shape))


def same_bits(a, b):
    return all(np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)) for k in ("out", "k", "v"))


PLAN_CHILD = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1] + "/tests")
from conftest import load_pkg
load_pkg()
import llama_box_b200.graph as G
data = open(sys.argv[2], "rb").read()
nodes = (G.Node * (len(data) // C.sizeof(G.Node))).from_buffer_copy(data)
sys.exit(0 if G.plan(nodes, int(sys.argv[3])) >= 0 else 1)
"""


def plan_trace(nodes, flags):
    """the launches the planner issues for this list, as B200_PLAN_DEBUG prints them (read once per process: a child)"""
    with tempfile.NamedTemporaryFile(suffix=".nodes") as f:
        f.write(bytes(nodes)); f.flush()
        r = subprocess.run([sys.executable, "-c", PLAN_CHILD, ROOT, f.name, str(flags)], env=dict(os.environ, B200_PLAN_DEBUG="1"),
                           capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return [ln.split(":", 1)[1].strip() for ln in r.stderr.splitlines() if ln.startswith("plan ")]


def fusion_change(nodes_a, nodes_b, flags):
    d = difflib.unified_diff(plan_trace(nodes_a, flags), plan_trace(nodes_b, flags), lineterm="", n=0)
    return "; ".join(ln for ln in d if ln[:1] in "+-" and ln[:3] not in ("+++", "---"))


# ---------------------------------------------------------------------------------------------------------- GPU tests
SHAPES = {   # case -> [(n_tok, pos0, n_out)]: decode at 0 / 255 / 256 (n_kv grows) / 700, verify batches of 3 and 8, prefill ubatches
    "q4km": [(1, 0, 1), (1, 255, 1), (1, 256, 1), (1, 700, 1), (3, 97, 3), (8, 500, 1), (40, 0, 1), (200, 300, 3)],
    "q4_0": [(1, 256, 1), (3, 97, 3), (40, 0, 1)],
    # (no prefill: these random Q8_0 weights give attention scores of std ~100, where the prefill attention's f16 Q and ggml-cpu's
    #  Q8_0-quantised Q legitimately disagree by 10%; the Q4_0 case covers the block-32 prefill GEMM)
    "q8_0": [(1, 255, 1), (1, 0, 1), (8, 500, 1)],
    "qwen2": [(1, 700, 1), (3, 97, 3)],
    "llama31": [(1, 256, 1), (8, 500, 1), (40, 0, 1)],
    "partial": [(1, 0, 1), (3, 97, 3)],
    "hd64": [(1, 256, 1), (8, 500, 1), (40, 0, 1)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("case,n_tok,pos0,n_out", [(c, *s) for c, ss in SHAPES.items() for s in ss])
def test_layers_over_recycled_buffers_match_the_oracle(case, n_tok, pos0, n_out):
    pytest.importorskip("torch")
    G, _ = mods()
    prob = Problem(case, n_tok, pos0, n_out)
    flagsets = {k: v for k, v in FLAGSETS.items() if k != "mega+mmv" or prob.ftype == "Q4_K_M"}
    errors = []
    for il in range(prob.cfg["n_layer"]):
        last = il == prob.cfg["n_layer"] - 1
        model = prob.model(il)
        runs = {p: LayerRun(prob, il, model, p) for p in POLICIES}
        res = {}
        for p, lr in runs.items():
            for name, flags in [("plain", 0)] + list(flagsets.items()):
                ex = G.Executor(0)
                a, b = lr.run(ex, flags), lr.run(ex, flags)
                ex.close()
                if not same_bits(a, b):
                    errors.append(f"layer {il} {p} {name}: two runs differ")
                res[p, name] = a
                # against the oracle: this layer's output (or logits) and its new KV rows; the other cells are untouched
                what = "logits" if last else "hidden"
                e = rel(a["out"], prob.want[il])
                ek = max(rel(kv_rows(a[c], prob.kv, prob.kv_idx), kv_rows(w[il], prob.kv, prob.kv_idx)) for c, w in (("k", prob.kc1), ("v", prob.vc1)))
                print(f"METRIC {case} n={n_tok} pos={pos0} layer={il} {p} {name} {what}={e:.3e} kv={ek:.3e}")
                if not e <= BOUNDS[what, prob.kv]:
                    errors.append(f"layer {il} {p} {name}: {what} {e:.3e} > {BOUNDS[what, prob.kv]:.0e}")
                if not ek <= BOUNDS["kv", prob.kv]:
                    errors.append(f"layer {il} {p} {name}: new KV rows {ek:.3e} > {BOUNDS['kv', prob.kv]:.0e}")
                untouched = np.ones(prob.n_ctx, bool); untouched[prob.kv_idx] = False
                if not (np.array_equal(a["k"][untouched], prob.kc0[il][untouched]) and np.array_equal(a["v"][untouched], prob.vc0[il][untouched])):
                    errors.append(f"layer {il} {p} {name}: KV cells outside the ubatch changed")
        # one launch per node: the placement cannot matter
        for p in ("gallocr", "tight"):
            if not same_bits(res[p, "plain"], res["fresh", "plain"]):
                errors.append(f"layer {il} {p} plain: differs from fresh")
        for name, flags in flagsets.items():
            for p in ("gallocr", "tight"):
                a, f = res[p, name], res["fresh", name]
                na, nf = G.plan(runs[p].nodes, flags), G.plan(runs["fresh"].nodes, flags)
                if na == nf:
                    if not same_bits(a, f):
                        errors.append(f"layer {il} {p} {name}: same plan ({na} launches) as fresh but different bits (out {rel(a['out'], f['out']):.2e})")
                else:
                    change = fusion_change(runs["fresh"].nodes, runs[p].nodes, flags)
                    print(f"PLAN {case} n={n_tok} layer={il} {p} {name}: fresh {nf} -> {na}: {change}")
                    e = max(rel(a["out"], f["out"]), max(rel(kv_rows(a[c], prob.kv, prob.kv_idx), kv_rows(f[c], prob.kv, prob.kv_idx)) for c in "kv"))
                    if not e <= MODES_TOL:
                        errors.append(f"layer {il} {p} {name}: plans differ from fresh ({change}) and outputs by {e:.2e}")
            for p in POLICIES:                           # fused against one launch per node, same list
                a, b = res[p, name], res[p, "plain"]
                e = rel(a["out"], b["out"])
                kv_same = np.array_equal(a["k"], b["k"]) and np.array_equal(a["v"], b["v"])
                print(f"MODES {case} n={n_tok} pos={pos0} layer={il} {p} {name} vs plain: out={e:.3e} kv_bytes_equal={kv_same}")
                if not e <= (MEGA_TOL if name.startswith("mega") else MODES_TOL):
                    errors.append(f"layer {il} {p} {name}: {e:.2e} from plain")
                if name == "mega+mmv" and prob.kv == F16:
                    # the persistent kernel's matvec phase computes K / V with its own summation order: one f16 step at most
                    for c in "kv":
                        x, y = (kv_rows(r[c], F16, prob.kv_idx) for r in (a, b))
                        if not (np.abs(x - y) <= 2.0 ** -10 * np.maximum(np.abs(x), np.abs(y))).all():
                            errors.append(f"layer {il} {p} {name}: {c} cache rows differ from plain by more than one f16 step")
                elif not kv_same:
                    errors.append(f"layer {il} {p} {name}: KV bytes differ from plain")
        del runs, model
    assert not errors, "\n".join(errors)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_graph_replay_with_new_inputs_equals_eager(policy):
    """a captured decode layer replayed with new tokens, positions and mask gives the bits of an eager run"""
    pytest.importorskip("torch")
    G, _ = mods()
    prob = Problem("q4km", 1, 300, 1)
    rng = np.random.default_rng(5)
    for il in range(prob.cfg["n_layer"]):
        model = prob.model(il)
        lr = LayerRun(prob, il, model, policy)
        steps = [(rng.standard_normal((1, prob.cfg["n_embd"])).astype(np.float32), np.array([300 + s], np.int32), causal_mask(1, prob.n_kv, 300 + s)) for s in range(4)]
        flags = G.EXEC_FUSION | G.EXEC_CUDA_GRAPHS
        ex, eager = G.Executor(0), G.Executor(0)
        for s, inp in enumerate(steps):
            got = lr.run(ex, flags, inputs=inp)
            want = lr.run(eager, G.EXEC_FUSION, inputs=inp)
            assert same_bits(got, want), (il, s)
        assert ex.captures == 1 and ex.replays == len(steps) - 2, (ex.captures, ex.replays)
        ex.close(); eager.close()


@pytest.mark.gpu
@pytest.mark.parametrize("first", ["flagged", "unflagged"])
def test_output_flag_is_part_of_the_captured_graph(first):
    """two lists that differ only in the OUTPUT flag of the un-roped Q: the flagged one must leave Q in its buffer, whichever
    list was captured first (the fused attention block never writes Q when nobody reads it)"""
    pytest.importorskip("torch")
    G, _ = mods()
    prob = Problem("q4km", 1, 300, 1)
    model = prob.model(0)
    mm_q = lambda items: [next(d for op, d, s, _ in items if op == G.OP_MUL_MAT)]    # noqa: E731  (the first projection is Q's)
    lr = LayerRun(prob, 0, model, "gallocr", mark_output=mm_q)
    q = mm_q(lr.arena.nl.items)[0]
    flagged = lr.nodes
    q.flags = 0
    unflagged = lr.arena.nl.build()
    q.flags = G.FLAG_OUTPUT
    qlen = 4 * prob.cfg["n_head"] * prob.cfg["head_dim"]

    def q_of():
        off = q.ptr - lr.arena.buf.data_ptr()
        return lr.arena.buf[off:off + qlen].cpu().numpy().copy()
    eager = G.Executor(0)
    want_f = lr.run(eager, G.EXEC_FUSION, nodes=flagged); want_q = q_of()
    want_u = lr.run(eager, G.EXEC_FUSION, nodes=unflagged)
    assert np.isfinite(want_q.view(np.float32)).all()
    flags = G.EXEC_FUSION | G.EXEC_CUDA_GRAPHS
    ex = G.Executor(0)
    order = [flagged, unflagged] if first == "flagged" else [unflagged, flagged]
    for nodes in [order[0], order[0], order[1], order[1], order[0]]:       # eager, capture, then the other list, twice, and back
        got = lr.run(ex, flags, nodes=nodes)
        if nodes is flagged:
            assert same_bits(got, want_f) and np.array_equal(q_of(), want_q)
        else:
            assert same_bits(got, want_u)
    ex.close(); eager.close()
