#!/usr/bin/env python3
"""Kernel-level timing of the batched MUL_MAT (b200_mul_mat_q, wgmma path) on the Llama-3-8B matmul shapes at a 512-token
ubatch: CUDA events on the launching stream, 20 repetitions after 3 warm-ups, weights of all shapes (> L2) cycled between reps."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import load_pkg  # noqa: E402
import importlib  # noqa: E402

b = load_pkg().ops
M = importlib.import_module("llama_box_b200.model"); G = importlib.import_module("llama_box_b200.graph")
n = int(sys.argv[1]) if len(sys.argv) > 1 else 512
gen = torch.Generator(device="cuda"); gen.manual_seed(1)
shapes = [("wq/wo 4096x4096 Q4_K", G.Q4_K, 4096, 4096), ("wk/wv 1024x4096 Q4_K", G.Q4_K, 1024, 4096), ("gate/up 14336x4096 Q4_K", G.Q4_K, 14336, 4096),
          ("down 4096x14336 Q4_K", G.Q4_K, 4096, 14336), ("down 4096x14336 Q6_K", G.Q6_K, 4096, 14336), ("output 128256x4096 Q6_K", G.Q6_K, 128256, 4096)]
out = []
st = torch.cuda.Stream()
for name, t, m, k in shapes:
    W = M.Weights(t, m, k, gen=gen)
    x = torch.randn(n, k, device="cuda")
    ws = torch.zeros(b.lib.b200_mul_mat_q_workspace(t, m, k, n), dtype=torch.uint8, device="cuda")
    dst = torch.zeros(n, m, device="cuda")
    with torch.cuda.stream(st):
        for _ in range(3):
            b.check(b.lib.b200_mul_mat_q(t, b.p(W.buf), b.p(x), k, b.p(dst), m, m, k, n, b.p(ws), torch.cuda.current_stream().cuda_stream))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 20
        st.synchronize(); e0.record(st)
        for _ in range(reps):
            b.check(b.lib.b200_mul_mat_q(t, b.p(W.buf), b.p(x), k, b.p(dst), m, m, k, n, b.p(ws), torch.cuda.current_stream().cuda_stream))
        e1.record(st); st.synchronize()
    ms = e0.elapsed_time(e1) / reps
    fl = 2.0 * m * k * n
    out.append({"shape": name, "n_tokens": n, "ms": ms, "tflops_useful": fl / ms / 1e9, "weight_GBps": m * b.row_bytes(t, k) / ms / 1e6})
    print(out[-1])
    del W, x, ws, dst
print(json.dumps(out))
