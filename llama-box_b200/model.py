"""Synthetic Llama / Qwen2-shaped model resident in HBM + the decode / prefill node lists that
libllama would hand to the backend (llm_build_llama, /root/reference/llama.cpp/src/llama-model.cpp:
5968-6122; build_attn / build_ffn / build_norm in llama-graph.cpp; KV views in
llama-kv-cache-unified.cpp:1056-1190).  Measurement / test harness for the graph executor: no
weights ship with the reference and there is no network, so weights are random *valid* GGUF blocks
(or caller-provided blocks for parity tests).  Shapes follow SURVEY.md §8.
"""
import math

import numpy as np
import torch

from . import graph as G
from . import ops

CONFIGS = {
    # name: n_embd, n_head, n_head_kv, head_dim, n_ff, n_vocab, n_layer, rope_base, rope_mode, eps, qkv_bias
    "llama3-8b": dict(n_embd=4096, n_head=32, n_head_kv=8, head_dim=128, n_ff=14336, n_vocab=128256, n_layer=32, rope_base=500000.0, rope_mode=0, eps=1e-5, qkv_bias=False),
    "tinyllama-1.1b": dict(n_embd=2048, n_head=32, n_head_kv=4, head_dim=64, n_ff=5632, n_vocab=32000, n_layer=22, rope_base=10000.0, rope_mode=0, eps=1e-5, qkv_bias=False),
    "qwen2-72b": dict(n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=29568, n_vocab=152064, n_layer=80, rope_base=1000000.0, rope_mode=2, eps=1e-6, qkv_bias=True),
    "test-small": dict(n_embd=2048, n_head=16, n_head_kv=4, head_dim=128, n_ff=4096, n_vocab=4096, n_layer=2, rope_base=500000.0, rope_mode=0, eps=1e-5, qkv_bias=False),
}


def use_more_bits(i, n):
    # llama-quant.cpp:185-186
    return i < n // 8 or i >= 7 * n // 8 or (i - n // 8) % 3 == 2


def type_mix(ftype, n_layer, n_ff=0, is_70b=False):
    """per-layer tensor types of a GGUF quantisation mix (llama-quant.cpp:203-227,302-364), with the reference's fallback for rows that
    are not a multiple of 256 (llama-quant.cpp:442-470: Q4_K -> Q5_0, Q6_K -> Q8_0 — Qwen2-72B's ffn_down) and the 70B attn_v bump"""
    out = []
    for i in range(n_layer):
        if ftype == "Q4_K_M":
            hi = G.Q6_K if use_more_bits(i, n_layer) else G.Q4_K
            v = hi if hi == G.Q6_K or not is_70b else G.Q5_K
            down = hi if n_ff % 256 == 0 else (G.Q8_0 if hi == G.Q6_K else G.Q5_0)
            out.append(dict(wq=G.Q4_K, wk=G.Q4_K, wv=v, wo=G.Q4_K, gate=G.Q4_K, up=G.Q4_K, down=down))
        elif ftype == "Q4_0":
            out.append({k: G.Q4_0 for k in ("wq", "wk", "wv", "wo", "gate", "up", "down")})
        elif ftype == "Q8_0":
            out.append({k: G.Q8_0 for k in ("wq", "wk", "wv", "wo", "gate", "up", "down")})
        else:
            raise ValueError(ftype)
    return out, (G.Q8_0 if ftype == "Q8_0" else G.Q6_K)      # output.weight


def rand_blocks_gpu(gen, t, nrows, k):
    """random valid blocks generated on the device (bench-size tensors); same scale policy as tests/refutil.rand_blocks"""
    bb = ops.lib.b200_block_bytes(t); be = ops.lib.b200_block_elems(t)
    nb = nrows * (k // be)
    raw = torch.randint(0, 256, (nb, bb), dtype=torch.uint8, device="cuda", generator=gen)

    def scales(lo, hi, signed):
        v = torch.rand(nb, device="cuda", generator=gen) * (hi - lo) + lo
        if signed:
            v = v * (torch.randint(0, 2, (nb,), device="cuda", generator=gen) * 2 - 1)
        return v.to(torch.float16).view(torch.uint8).reshape(nb, 2)
    if t in (G.Q4_0, G.Q5_0, G.Q8_0):
        raw[:, 0:2] = scales(1e-3, 2e-3 if t == G.Q8_0 else (1e-2 if t == G.Q5_0 else 2e-2), True)
    elif t in (G.Q4_K, G.Q5_K):
        raw[:, 0:2] = scales(1e-4, 1e-3, False); raw[:, 2:4] = scales(1e-4, 1e-3, False)
    elif t == G.Q6_K:
        raw[:, 208:210] = scales(1e-5, 2e-4, True)
    return raw.reshape(-1)


class Weights:
    """one weight matrix in HBM: ggml blocks, repacked for the kernels, +64 B slack"""

    def __init__(self, t, m, k, blocks=None, gen=None):
        self.type, self.m, self.k = t, m, k
        nbytes = m * ops.row_bytes(t, k)
        kp = ops.lib.b200_padded_k(t, k)
        native = rand_blocks_gpu(gen, t, m, k) if blocks is None else torch.from_numpy(np.ascontiguousarray(blocks).reshape(-1)).cuda()
        if kp != k:                                       # rows not a multiple of 256 elements: private padded layout (b200_ops.h)
            self.buf = torch.zeros(m * ops.row_bytes(t, kp) + 64, dtype=torch.uint8, device="cuda")
            ops.check(ops.lib.b200_repack_rows_padded(t, ops.p(native), ops.p(self.buf), m, k, 0, ops.stream()))
            torch.cuda.synchronize()
        else:
            self.buf = torch.zeros(nbytes + 64, dtype=torch.uint8, device="cuda")
            self.buf[:nbytes] = native
            ops.check(ops.lib.b200_repack_rows(t, ops.p(self.buf), m, k, ops.stream()))
        self.t = G.T(self.buf.data_ptr(), t, [k, m])
        self.nbytes = nbytes


class SyntheticLlama:
    device = "cuda"                 # where the io buffers of build() live

    def __init__(self, cfg, ftype="Q4_K_M", n_ctx=4096, kv_type=G.F16, seed=1234, host_weights=None, n_layer=None,
                 layer_range=None, first=True, last=True, n_seq=1):
        c = dict(CONFIGS[cfg]) if isinstance(cfg, str) else dict(cfg)
        if n_layer:
            c["n_layer"] = n_layer
        self.c, self.n_ctx, self.kv_type, self.ftype = c, n_ctx, kv_type, ftype
        self.first, self.last, self.n_seq = first, last, n_seq
        lo, hi = layer_range if layer_range else (0, c["n_layer"])
        self.layer_ids = list(range(lo, hi))
        gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
        E, H, HK, D, FF, V, L = c["n_embd"], c["n_head"], c["n_head_kv"], c["head_dim"], c["n_ff"], c["n_vocab"], c["n_layer"]
        mix, out_t = type_mix(ftype, L, FF, c.get("n_embd") == 8192 and L == 80)
        hw = host_weights or {}

        def W(name, t, m, k):
            return Weights(t, m, k, hw.get(name), gen)

        def vec(name, n, mean):
            if name in hw:
                return torch.from_numpy(hw[name]).cuda()
            return (mean + 0.01 * torch.randn(n, device="cuda", generator=gen)).float()
        self.layers = []
        for i in self.layer_ids:
            t = mix[i]
            ly = dict(attn_norm=vec(f"blk.{i}.attn_norm", E, 1.0), ffn_norm=vec(f"blk.{i}.ffn_norm", E, 1.0),
                      wq=W(f"blk.{i}.attn_q", t["wq"], H * D, E), wk=W(f"blk.{i}.attn_k", t["wk"], HK * D, E), wv=W(f"blk.{i}.attn_v", t["wv"], HK * D, E),
                      wo=W(f"blk.{i}.attn_output", t["wo"], E, H * D), gate=W(f"blk.{i}.ffn_gate", t["gate"], FF, E), up=W(f"blk.{i}.ffn_up", t["up"], FF, E),
                      down=W(f"blk.{i}.ffn_down", t["down"], E, FF))
            if c["qkv_bias"]:
                ly.update(bq=vec(f"blk.{i}.bq", H * D, 0.0), bk=vec(f"blk.{i}.bk", HK * D, 0.0), bv=vec(f"blk.{i}.bv", HK * D, 0.0))
            kvrow = G.row_size(kv_type, HK * D)
            ly["k_caches"] = [torch.zeros(n_ctx * kvrow, dtype=torch.uint8, device="cuda") for _ in range(n_seq)]
            ly["v_caches"] = [torch.zeros(n_ctx * kvrow, dtype=torch.uint8, device="cuda") for _ in range(n_seq)]
            ly["k_cache"], ly["v_cache"] = ly["k_caches"][0], ly["v_caches"][0]
            self.layers.append(ly)
        self.output_norm = vec("output_norm", E, 1.0) if last else None
        self.output = W("output", out_t, V, E) if last else None
        self.tok_embd = None
        if first:
            self.tok_embd = torch.from_numpy(hw["token_embd"]).cuda() if "token_embd" in hw else (0.02 * torch.randn((V, E), device="cuda", generator=gen)).float()
        self.rope_ff = torch.from_numpy(hw["rope_freqs"]).cuda() if "rope_freqs" in hw else None
        self.bufs = {}

    # ---- bytes the decode step must stream from HBM (SURVEY.md §8d): weights + norms + KV
    def streamed_weight_bytes(self):
        b = (self.output.nbytes + self.output_norm.numel() * 4) if self.last else 0
        for ly in self.layers:
            b += sum(ly[k].nbytes for k in ("wq", "wk", "wv", "wo", "gate", "up", "down")) + 2 * ly["attn_norm"].numel() * 4
        return b

    def kv_bytes_per_pos(self):
        return 2 * len(self.layers) * G.row_size(self.kv_type, self.c["n_head_kv"] * self.c["head_dim"])

    def _buf(self, name, shape, dtype=torch.float32):
        key = (name, tuple(shape), dtype)
        if key not in self.bufs:
            self.bufs[key] = torch.zeros(shape, dtype=dtype, device=self.device)
        return self.bufs[key]

    def build(self, n_tok, n_kv, want_all_logits=False, seq=0, skip_attention=False, n_out=1, place=None):
        """node list for one ubatch of n_tok tokens attending to n_kv cache positions (n_kv % 256 == 0 with -fa).
        skip_attention (bench roofline leg only): leave out ROPE / SET_ROWS / FLASH_ATTN_EXT and feed the Q projection
        straight into wo, so that the list holds exactly the step's matvec launches with their in-situ prologues
        (rms_norm + quantise inside the kernel, residual epilogues, lm_head) and nothing else.
        Inputs (device buffers the caller fills): tokens i32[n_tok], pos i32[n_tok], kv_idx i64[n_tok],
        mask f32[n_kv, pad64(n_tok)] (cast to f16 by a CPY node like llama-graph.cpp:1424), out_ids i32[n_out]
        (n_out rows of logits unless want_all_logits).
        place: optional placement hook, called as place(nl, fixed) before the list is built.  It may move every
        intermediate (the dst of a compute node other than SET_ROWS, and the views of it) to addresses of its choosing,
        the way a graph allocator recycles buffers; `fixed` are the results the caller reads from io (hidden_out,
        logits) and must stay put.  Without it every intermediate has a buffer of its own."""
        c = self.c
        E, H, HK, D, FF, V = c["n_embd"], c["n_head"], c["n_head_kv"], c["head_dim"], c["n_ff"], c["n_vocab"]
        nl = G.NodeList()
        npad = (n_tok + 63) // 64 * 64
        n_out = n_tok if want_all_logits else n_out
        io = dict(tokens=self._buf("tokens", [n_tok], torch.int32), pos=self._buf("pos", [n_tok], torch.int32), kv_idx=self._buf("kv_idx", [n_tok], torch.int64),
                  mask=self._buf("mask", [npad, n_kv]), out_ids=self._buf("out_ids", [n_out], torch.int32), logits=self._buf("logits", [n_out, V]),
                  hidden_in=self._buf("hidden_in", [n_tok, E]), hidden_out=self._buf("hidden_out", [n_tok, E]))
        f = lambda name, ne, dt=torch.float32: self._buf(name + f"@{n_tok}", list(reversed(ne)), dt)  # noqa: E731
        tT = lambda ten, t, ne: G.T(ten.data_ptr(), t, ne)  # noqa: E731
        pos_t, idx_t = tT(io["pos"], G.I32, [n_tok]), tT(io["kv_idx"], G.I64, [n_tok])
        mask32 = tT(io["mask"], G.F32, [n_kv, npad]); mask16 = tT(f("mask16", [n_kv, npad], torch.float16), G.F16, [n_kv, npad])
        nl.add(G.OP_CPY, mask16, [mask32])
        # token embedding lookup: the reference runs it on the CPU (input layer, llama-model.cpp:1960-1962) and
        # uploads [n_embd, n_tok] f32; the resident-in-HBM harness gathers from an f32 table instead
        if self.first:
            inpL = nl.add(G.OP_GET_ROWS, tT(f("inp_embd", [E, n_tok]), G.F32, [E, n_tok]), [tT(self.tok_embd, G.F32, [E, V]), tT(io["tokens"], G.I32, [n_tok])])
        else:
            inpL = tT(io["hidden_in"], G.F32, [E, n_tok])          # handed over by the previous pipeline stage
        n_dims = c.get("rope_n_dims", D)                        # partial rotary: the first n_dims of each head
        rope_params = [0, n_dims, c["rope_mode"], 0, 8192, G.f32_bits(c["rope_base"]), G.f32_bits(1.0), G.f32_bits(0.0), G.f32_bits(1.0), G.f32_bits(32.0), G.f32_bits(1.0)]
        ff_t = tT(self.rope_ff, G.F32, [self.rope_ff.numel()]) if self.rope_ff is not None else None
        kvrow = G.row_size(self.kv_type, HK * D); kvhead = G.row_size(self.kv_type, D)
        for il, ly in enumerate(self.layers):
            last = self.last and il == len(self.layers) - 1
            wT = lambda v, n=E: tT(v, G.F32, [n])  # noqa: E731
            # attn_norm
            t1 = nl.add(G.OP_RMS_NORM, tT(f(f"norm{il % 2}", [E, n_tok]), G.F32, [E, n_tok]), [inpL], [G.f32_bits(c["eps"])])
            cur = nl.add(G.OP_MUL, tT(f(f"normw{il % 2}", [E, n_tok]), G.F32, [E, n_tok]), [t1, wT(ly["attn_norm"])])
            # Q, rope; K, rope; V  (llama-model.cpp:6004-6043)
            q = nl.add(G.OP_MUL_MAT, tT(f("q", [H * D, n_tok]), G.F32, [H * D, n_tok]), [ly["wq"].t, cur])
            if c["qkv_bias"]:
                q = nl.add(G.OP_ADD, tT(f("qb", [H * D, n_tok]), G.F32, [H * D, n_tok]), [q, wT(ly["bq"], H * D)])
            q3 = nl.view_op(q.reshape([D, H, n_tok]), q)
            srcs = [q3, pos_t] + ([ff_t] if ff_t else [])
            if not skip_attention:
                qr = nl.add(G.OP_ROPE, tT(f("qr", [D, H, n_tok]), G.F32, [D, H, n_tok]), srcs, rope_params)
            k = nl.add(G.OP_MUL_MAT, tT(f("k", [HK * D, n_tok]), G.F32, [HK * D, n_tok]), [ly["wk"].t, cur])
            if c["qkv_bias"]:
                k = nl.add(G.OP_ADD, tT(f("kb", [HK * D, n_tok]), G.F32, [HK * D, n_tok]), [k, wT(ly["bk"], HK * D)])
            k3 = nl.view_op(k.reshape([D, HK, n_tok]), k)
            srcs = [k3, pos_t] + ([ff_t] if ff_t else [])
            if not skip_attention:
                kr = nl.add(G.OP_ROPE, tT(f("kr", [D, HK, n_tok]), G.F32, [D, HK, n_tok]), srcs, rope_params)
            v = nl.add(G.OP_MUL_MAT, tT(f("v", [HK * D, n_tok]), G.F32, [HK * D, n_tok]), [ly["wv"].t, cur])
            if c["qkv_bias"]:
                v = nl.add(G.OP_ADD, tT(f("vb", [HK * D, n_tok]), G.F32, [HK * D, n_tok]), [v, wT(ly["bv"], HK * D)])
            if skip_attention:
                assert H * D == E
                att2 = q
            else:
                # KV store (llama-kv-cache-unified.cpp:1103-1160)
                kc = G.T(ly["k_caches"][seq].data_ptr(), self.kv_type, [HK * D, self.n_ctx]); vc = G.T(ly["v_caches"][seq].data_ptr(), self.kv_type, [HK * D, self.n_ctx])
                k2 = nl.view_op(kr.reshape([HK * D, n_tok]), kr)
                nl.add(G.OP_SET_ROWS, kc, [k2, idx_t])
                nl.add(G.OP_SET_ROWS, vc, [v, idx_t])
                # attention (llama-graph.cpp:1236-1265; views llama-kv-cache-unified.cpp:1056-1101)
                qp = nl.view_op(qr.view([D, n_tok, H], [4, 4 * D * H, 4 * D, 4 * D * H * n_tok]), qr)
                kv = nl.view_op(kc.view([D, n_kv, HK], [G.ELEM_SIZE.get(self.kv_type, 34), kvrow, kvhead, kvrow * n_kv]), kc)
                vv = nl.view_op(vc.view([D, n_kv, HK], [G.ELEM_SIZE.get(self.kv_type, 34), kvrow, kvhead, kvrow * n_kv]), vc)
                att = nl.add(G.OP_FLASH_ATTN_EXT, tT(f("att", [D, H, n_tok]), G.F32, [D, H, n_tok]), [qp, kv, vv, mask16],
                             [G.f32_bits(1.0 / math.sqrt(D)), G.f32_bits(0.0), G.f32_bits(0.0), 10])
                att2 = nl.view_op(att.reshape([H * D, n_tok]), att)
            cur = nl.add(G.OP_MUL_MAT, tT(f("wo", [E, n_tok]), G.F32, [E, n_tok]), [ly["wo"].t, att2])
            inpSA, nt = inpL, n_tok
            if last and not want_all_logits:
                oid = tT(io["out_ids"], G.I32, [n_out])
                cur = nl.add(G.OP_GET_ROWS, tT(f("wo_sel", [E, n_out]), G.F32, [E, n_out]), [cur, oid])
                inpSA = nl.add(G.OP_GET_ROWS, tT(f("sa_sel", [E, n_out]), G.F32, [E, n_out]), [inpSA, oid])
                nt = n_out
            ffn_inp = nl.add(G.OP_ADD, tT(f(f"ffn_inp{il % 2}", [E, nt]), G.F32, [E, nt]), [cur, inpSA])
            t1 = nl.add(G.OP_RMS_NORM, tT(f("fnorm", [E, nt]), G.F32, [E, nt]), [ffn_inp], [G.f32_bits(c["eps"])])
            cur = nl.add(G.OP_MUL, tT(f("fnormw", [E, nt]), G.F32, [E, nt]), [t1, wT(ly["ffn_norm"])])
            up = nl.add(G.OP_MUL_MAT, tT(f("up", [FF, nt]), G.F32, [FF, nt]), [ly["up"].t, cur])
            gate = nl.add(G.OP_MUL_MAT, tT(f("gate", [FF, nt]), G.F32, [FF, nt]), [ly["gate"].t, cur])
            h = nl.add(G.OP_GLU_SWIGLU, tT(f("h", [FF, nt]), G.F32, [FF, nt]), [gate, up], [2, 0])
            dn = nl.add(G.OP_MUL_MAT, tT(f("down", [E, nt]), G.F32, [E, nt]), [ly["down"].t, h])
            final_stage_out = (not self.last) and il == len(self.layers) - 1
            l_out = tT(io["hidden_out"], G.F32, [E, nt]) if final_stage_out else tT(f(f"l_out{il % 2}", [E, nt]), G.F32, [E, nt])
            inpL = nl.add(G.OP_ADD, l_out, [dn, ffn_inp])
        if not self.last:
            if place is not None:
                place(nl, [inpL])
            return nl.build(), io
        nt = n_out
        t1 = nl.add(G.OP_RMS_NORM, tT(f("onorm", [E, nt]), G.F32, [E, nt]), [inpL], [G.f32_bits(c["eps"])])
        cur = nl.add(G.OP_MUL, tT(f("onormw", [E, nt]), G.F32, [E, nt]), [t1, tT(self.output_norm, G.F32, [E])])
        logits = tT(io["logits"], G.F32, [V, nt])
        logits.flags = G.FLAG_OUTPUT                           # libllama flags t_logits (llama-context.cpp graph outputs)
        nl.add(G.OP_MUL_MAT, logits, [self.output.t, cur])
        if place is not None:
            place(nl, [logits])
        return nl.build(), io
