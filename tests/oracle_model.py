"""CPU forward pass of a Llama-shaped model composed ONLY of oracle ops (oracle/liboracle.so), in the
node order of llm_build_llama (/root/reference/llama.cpp/src/llama-model.cpp:5968-6122).  Test
infrastructure: the checker for the graph executor (tests/test_gpu_executor.py) and for smoke()."""
import math

import numpy as np

from refutil import F16, Q8_0, oracle, orc_mul_mat, ptr, rand_blocks, row_bytes

MIX_KEYS = ("wq", "wk", "wv", "wo", "gate", "up", "down")


def make_host_weights(cfg, mix, out_type, seed=7, scale_mul=0.25):
    """random valid blocks + norm/bias/embedding vectors, keyed like llama_box_b200.model.SyntheticLlama"""
    rng = np.random.default_rng(seed)
    E, H, HK, D, FF, V, L = cfg["n_embd"], cfg["n_head"], cfg["n_head_kv"], cfg["head_dim"], cfg["n_ff"], cfg["n_vocab"], cfg["n_layer"]
    hw, types = {}, {}
    shapes = dict(wq=(H * D, E), wk=(HK * D, E), wv=(HK * D, E), wo=(E, H * D), gate=(FF, E), up=(FF, E), down=(E, FF))
    names = dict(wq="attn_q", wk="attn_k", wv="attn_v", wo="attn_output", gate="ffn_gate", up="ffn_up", down="ffn_down")
    for i in range(L):
        for k in MIX_KEYS:
            m, kk = shapes[k]
            hw[f"blk.{i}.{names[k]}"] = rand_blocks(rng, mix[i][k], m, kk, scale_mul); types[f"blk.{i}.{names[k]}"] = (mix[i][k], m, kk)
        hw[f"blk.{i}.attn_norm"] = (1 + 0.05 * rng.standard_normal(E)).astype(np.float32)
        hw[f"blk.{i}.ffn_norm"] = (1 + 0.05 * rng.standard_normal(E)).astype(np.float32)
        if cfg.get("qkv_bias"):
            hw[f"blk.{i}.bq"] = (0.1 * rng.standard_normal(H * D)).astype(np.float32)
            hw[f"blk.{i}.bk"] = (0.1 * rng.standard_normal(HK * D)).astype(np.float32)
            hw[f"blk.{i}.bv"] = (0.1 * rng.standard_normal(HK * D)).astype(np.float32)
    hw["output_norm"] = (1 + 0.05 * rng.standard_normal(E)).astype(np.float32)
    hw["output"] = rand_blocks(rng, out_type, V, E); types["output"] = (out_type, V, E)
    hw["token_embd"] = (0.5 * rng.standard_normal((V, E))).astype(np.float32)
    return hw, types


class OracleLlama:
    def __init__(self, cfg, hw, types, n_ctx, kv_type=F16, rope_ff=None):
        self.c, self.hw, self.types, self.n_ctx, self.kv_type, self.ff = cfg, hw, types, n_ctx, kv_type, rope_ff
        HK, D = cfg["n_head_kv"], cfg["head_dim"]
        self.kvrow = row_bytes(kv_type, HK * D)
        self.kc = [np.zeros((n_ctx, self.kvrow), np.uint8) for _ in range(cfg["n_layer"])]
        self.vc = [np.zeros((n_ctx, self.kvrow), np.uint8) for _ in range(cfg["n_layer"])]

    def mm(self, name, x):
        t, m, k = self.types[name]
        return orc_mul_mat(t, self.hw[name], x, m, x.shape[0], k)

    def norm(self, x, w):
        y = np.zeros_like(x); oracle().orc_rms_norm(ptr(x), ptr(w), ptr(y), x.shape[1], x.shape[0], self.c["eps"])
        return y

    def rope(self, x, pos, nh):
        c = self.c; D = c["head_dim"]; n = x.shape[0]
        y = np.zeros_like(x)
        oracle().orc_rope(ptr(x), ptr(y), ptr(pos), ptr(self.ff), D, nh, n, c.get("rope_n_dims", D), c["rope_mode"], 8192, c["rope_base"], 1.0, 0.0, 1.0, 32.0, 1.0)
        return y

    def forward(self, tokens, pos, kv_idx, n_kv, mask16, trace=None):
        """tokens i32[n], pos i32[n], kv_idx i64[n], mask16 uint16 [npad, n_kv] -> logits of the last token [V]"""
        x = np.ascontiguousarray(self.hw["token_embd"][tokens])
        for il in range(self.c["n_layer"]):
            x = self.layer(il, x, pos, kv_idx, n_kv, mask16, [len(tokens) - 1] if il == self.c["n_layer"] - 1 else None, trace)
        return self.logits(x)[0]

    def logits(self, x):
        """output norm + output matrix of the rows x [n_out, n_embd] -> [n_out, V]"""
        return self.mm("output", self.norm(x, self.hw["output_norm"]))

    def layer(self, il, x, pos, kv_idx, n_kv, mask16, out_ids=None, trace=None):
        """one layer on x [n, n_embd]: stores the new K / V rows in this layer's cache and returns the layer's output,
        of the rows out_ids only if given (the last layer's output-row selection, llama-model.cpp:6054-6058)"""
        c = self.c
        H, HK, D = c["n_head"], c["n_head_kv"], c["head_dim"]
        n = x.shape[0]
        cur = self.norm(x, self.hw[f"blk.{il}.attn_norm"])
        q, k, v = self.mm(f"blk.{il}.attn_q", cur), self.mm(f"blk.{il}.attn_k", cur), self.mm(f"blk.{il}.attn_v", cur)
        if c.get("qkv_bias"):
            q = q + self.hw[f"blk.{il}.bq"]; k = k + self.hw[f"blk.{il}.bk"]; v = v + self.hw[f"blk.{il}.bv"]
        q_pre = q
        q = self.rope(np.ascontiguousarray(q), pos, H); k = self.rope(np.ascontiguousarray(k), pos, HK)
        oracle().orc_set_rows(ptr(k), ptr(kv_idx), ptr(self.kc[il]), self.kv_type, HK * D, n, self.kvrow)
        oracle().orc_set_rows(ptr(np.ascontiguousarray(v)), ptr(kv_idx), ptr(self.vc[il]), self.kv_type, HK * D, n, self.kvrow)
        att = np.zeros((n, H * D), np.float32)
        hb = row_bytes(self.kv_type, D)
        oracle().orc_flash_attn_ext(ptr(q), H * D * 4, D * 4, ptr(self.kc[il]), self.kvrow, hb, ptr(self.vc[il]), self.kvrow, hb, ptr(mask16), ptr(att),
                                    self.kv_type, D, D, H, HK, n, n_kv, 1.0 / math.sqrt(D), 0.0, 0.0)
        o = self.mm(f"blk.{il}.attn_output", att)
        if trace is not None and il == 0:
            trace.update(normw0=cur, q=q_pre, qr=q, kr=k, v=v, att=att, wo=o)
        if out_ids is not None:
            o, x = o[list(out_ids)], x[list(out_ids)]
        ffn_inp = o + x
        cur = self.norm(ffn_inp, self.hw[f"blk.{il}.ffn_norm"])
        up, gate = self.mm(f"blk.{il}.ffn_up", cur), self.mm(f"blk.{il}.ffn_gate", cur)
        h = np.zeros_like(gate); oracle().orc_swiglu(ptr(gate), ptr(up), ptr(h), gate.size)
        dn = self.mm(f"blk.{il}.ffn_down", h)
        if trace is not None and il == 0:
            trace.update(ffn_inp0=ffn_inp, fnormw=cur, up=up, gate=gate, h=h, down=dn)
        return dn + ffn_inp


def causal_mask(n_tok, n_kv, pos0):
    """mask rows as llama_kv_cache_unified::set_input_kq_mask builds them: 0 for cells <= token position, -inf otherwise"""
    npad = (n_tok + 63) // 64 * 64
    m = np.full((npad, n_kv), -np.inf, np.float32)
    for t in range(n_tok):
        m[t, :pos0 + t + 1] = 0
    return m
