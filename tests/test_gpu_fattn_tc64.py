"""GPU: multi-token FLASH_ATTN_EXT with 64-wide heads (TinyLlama, Llama-3.2-1B, Qwen2.5-0.5B) on the tensor cores (csrc/fattn_tc.cu,
the D = 64 instance) against an f64 evaluation and the C oracle: F16 and Q8_0 caches, the head groupings of those models, ragged token
counts around the dispatch minimum, causal and block-diagonal masks, fully masked padding rows, softcap; which kernel ran; run-to-run bit
identity; and 600-token prompts through libllama with the tensor cores on and off."""
import os

import numpy as np
import pytest

from refutil import F16, Q8_0, have_ref, nmse, oracle, orc_dequant, ptr, row_bytes

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

D = 64
MIN_TOK = 40            # FT_MIN_TOK_D64 of fattn_tc.cu: fewer tokens of a 64-wide head stay on the vector kernel


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def causal(nt, nkv, past):
    """token t sees the cached positions and the batch up to itself; rows padded to 64 as libllama pads them"""
    mask = np.full(((nt + 63) // 64 * 64, nkv), -np.inf, np.float32)
    for t in range(nt):
        mask[t, :min(nkv, past + t + 1)] = 0
    return mask


class Case:
    """one attention call: cache rows written by the oracle's set_rows, `extra` rows of 0xff bytes (f16 NaN, q8_0 d = NaN) after the
    n_kv cells that the kernel must never read; the library's output of two runs on NaN-filled buffers, the oracle's, and f64"""

    def __init__(self, b200, kvt, nh, nhkv, nt, nkv, mask, softcap=0.0, extra=16, seed=0):
        rng = np.random.default_rng(seed + 10 * nh + nt + nkv + kvt)
        q = rng.standard_normal((nt, nh, D)).astype(np.float32)
        kf = rng.standard_normal((nkv, nhkv * D)).astype(np.float32); vf = rng.standard_normal((nkv, nhkv * D)).astype(np.float32)
        rb_row, rb_head = row_bytes(kvt, nhkv * D), row_bytes(kvt, D)
        kc = np.zeros((nkv, rb_row), np.uint8); vc = np.zeros((nkv, rb_row), np.uint8)
        ids = np.arange(nkv, dtype=np.int64)
        oracle().orc_set_rows(ptr(kf), ptr(ids), ptr(kc), kvt, nhkv * D, nkv, rb_row)
        oracle().orc_set_rows(ptr(vf), ptr(ids), ptr(vc), kvt, nhkv * D, nkv, rb_row)
        mask16 = mask.astype(np.float16)
        scale = 1.0 / np.sqrt(D)
        self.want = np.zeros((nt, nh, D), np.float32)
        oracle().orc_flash_attn_ext(ptr(q), nh * D * 4, D * 4, ptr(kc), rb_row, rb_head, ptr(vc), rb_row, rb_head, ptr(mask16), ptr(self.want),
                                    kvt, D, D, nh, nhkv, nt, nkv, scale, 0.0, softcap)
        junk = np.full((extra, rb_row), 0xff, np.uint8)
        qd, kd, vd, md = dev(q), dev(np.concatenate([kc, junk])), dev(np.concatenate([vc, junk])), dev(mask16.view(np.uint16))

        def call(dst):
            b200.check(b200.lib.b200_flash_attn_ext(b200.p(qd), nh * D, D, b200.p(kd), rb_row, rb_head, b200.p(vd), rb_row, rb_head,
                                                    b200.p(md), nkv, b200.p(dst), kvt, D, D, nh, nhkv, nt, nkv, scale, 0.0, softcap, None, b200.stream()))
        self.call = lambda: call(torch.full((nt, nh, D), float("nan"), dtype=torch.float32, device="cuda"))
        outs = []
        for _ in range(2):
            dst = torch.full((nt, nh, D), float("nan"), dtype=torch.float32, device="cuda")
            call(dst)
            torch.cuda.synchronize()
            outs.append(dst.cpu().numpy())
        assert outs[0].tobytes() == outs[1].tobytes(), "two runs differ"
        self.got = outs[0]
        Kd = orc_dequant(kvt, kc, nkv, nhkv * D).astype(np.float64).reshape(nkv, nhkv, D)
        Vd = orc_dequant(kvt, vc, nkv, nhkv * D).astype(np.float64).reshape(nkv, nhkv, D)
        q16 = q.astype(np.float16).astype(np.float64)
        m64 = mask16[:nt].astype(np.float64)
        self.live = np.isfinite(m64).any(axis=1)                 # rows with at least one visible position
        self.truth = np.zeros((nt, nh, D))
        for h in range(nh):
            hk = h // (nh // nhkv)
            s = (q16[self.live, h] @ Kd[:, hk].T) * scale
            if softcap:
                s = softcap * np.tanh(s / softcap)
            s = s + m64[self.live]
            p = np.exp(s - s.max(axis=1, keepdims=True))
            self.truth[self.live, h] = (p @ Vd[:, hk]) / p.sum(axis=1, keepdims=True)
        self.kvt = kvt

    def check(self):
        """the bounds of test_flash_attn_tensor_core (tests/test_gpu_ops.py) on the rows that see at least one position"""
        assert np.isfinite(self.got).all()
        g, w, t = self.got[self.live], self.want[self.live], self.truth[self.live]
        err = np.abs(g - t).max() / np.abs(t).max()
        assert err <= 2e-3, err
        assert nmse(g, t) < 1e-6, nmse(g, t)
        assert nmse(g, w) < (1e-3 if self.kvt == F16 else 1e-4), nmse(g, w)
        assert nmse(g, t) <= nmse(w, t), (nmse(g, t), nmse(w, t))


def kernels_of(fn):
    """names of the CUDA kernels one call launches (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.key for e in prof.key_averages())


SHAPES = [  # n_head, n_head_kv, n_tok, n_kv, past
    (32, 4, MIN_TOK, 512, 300),                # TinyLlama, at the minimum; cells past + n_tok .. n_kv - 1 are cache padding
    (32, 4, MIN_TOK + 1, 1024, 700),
    (32, 8, 97, 512, 0),                       # Llama-3.2-1B, a fresh prompt
    (14, 2, 200, 768, 512),                    # Qwen2.5-0.5B: 7 query heads per KV head
    (14, 2, 45, 1000, 900),                    # n_kv not a multiple of the 128-position block
    (4, 4, 512, 1024, 512),
    (32, 4, 512, 2048, 1536),
    (4, 4, 512, 8192, 7680),
]


@pytest.mark.parametrize("kvt", [F16, Q8_0])
@pytest.mark.parametrize("nh,nhkv,nt,nkv,past", SHAPES)
def test_head64_vs_oracle(b200, kvt, nh, nhkv, nt, nkv, past):
    Case(b200, kvt, nh, nhkv, nt, nkv, causal(nt, nkv, past)).check()


@pytest.mark.parametrize("kvt", [F16, Q8_0])
def test_head64_block_diagonal_mask(b200, kvt):
    """two sequences in one ubatch: tokens 0..89 continue sequence 0 (cells 0..389), tokens 90..199 start sequence 1 (cells 512..621)"""
    nt, nkv = 200, 768
    mask = np.full((256, nkv), -np.inf, np.float32)
    for t in range(90):
        mask[t, :300 + t + 1] = 0
    for t in range(90, nt):
        mask[t, 512:512 + t - 90 + 1] = 0
    Case(b200, kvt, 32, 4, nt, nkv, mask).check()


@pytest.mark.parametrize("kvt", [F16, Q8_0])
def test_head64_fully_masked_rows(b200, kvt):
    """the last rows of the batch see no position at all (padding tokens): their output is finite, the others are exact"""
    nt, nkv = 48, 512
    mask = causal(nt, nkv, 200)
    mask[40:nt] = -np.inf
    c = Case(b200, kvt, 32, 4, nt, nkv, mask)
    assert np.isfinite(c.got[40:]).all()
    c.check()


def test_head64_softcap(b200):
    Case(b200, F16, 32, 4, 200, 1024, causal(200, 1024, 600), softcap=5.0).check()


@pytest.mark.parametrize("nt", [MIN_TOK - 1, MIN_TOK, 200])
def test_head64_runs_on_the_tensor_cores_from_the_minimum(b200, nt):
    """fattn_tc_kernel runs from MIN_TOK query tokens on; below that the vector kernel does (speculative verify batches)"""
    c = Case(b200, F16, 32, 4, nt, 1024, causal(nt, 1024, 600))
    names = kernels_of(c.call)
    assert ("fattn_tc_kernel" in names) == (nt >= MIN_TOK), names
    assert "fattn_vec_kernel" in names or nt >= MIN_TOK, names
    c.check()


@pytest.mark.skipif(not have_ref(), reason="oracle/_ref (reference build) not present")
@pytest.mark.parametrize("kv", ["f16", "q8_0"])
def test_head64_prompt_through_libllama(tmp_path, tmp_path_factory, kv):
    """TinyLlama Q4_0, 2 layers: a 600-token prompt (a 512-token ubatch and an 88-token one, both on the tensor-core attention) and a
    few decode steps through the unmodified libllama, as close to ggml-cpu as ggml-cpu's own builds are to each other; the same
    with B200_FATTN_DISABLE_TC=1 (the vector kernel) in the driver's process"""
    import test_gpu_product as P
    gguf = P.model_file(tmp_path_factory, "tinyllama-1.1b", "Q4_0", 2)
    try:
        kw = dict(kv=kv, verify=1, prompt_len=600, gen=9)
        cpu = P.drv(gguf, str(tmp_path / "cpu"), False, **kw)
        others = P.cpu_builds(tmp_path, tmp_path_factory, gguf, **kw)
        gpu = P.drv(gguf, str(tmp_path / "gpu"), True, **kw)
        P.assert_within_reference_self_consistency(gpu, cpu, others, f"tinyllama Q4_0 kv={kv} prompt=600")
        vec = P.drv(gguf, str(tmp_path / "gpu_vec"), True, extra_env=dict(B200_FATTN_DISABLE_TC="1"), **kw)
        P.assert_within_reference_self_consistency(vec, cpu, others, f"tinyllama Q4_0 kv={kv} prompt=600, vector attention")
    finally:
        P._models.pop(("tinyllama-1.1b", "Q4_0", 2), None)
        os.remove(gguf)
