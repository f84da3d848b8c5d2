#!/usr/bin/env python3
"""Bring-up aid for fattn_tc.cu: one multi-token attention shape against an f64 evaluation; error statistics per query tile / head.

    fattn_probe.py f16|q8_0 n_head n_head_kv n_tok n_kv past [head_size, default 128]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import load_pkg  # noqa: E402
from refutil import F16, Q8_0, oracle, orc_dequant, ptr, row_bytes  # noqa: E402

b = load_pkg().ops
kvt = {"f16": F16, "q8_0": Q8_0}[sys.argv[1]]
nh, nhkv, nt, nkv, past = (int(v) for v in sys.argv[2:7])
dk = int(sys.argv[7]) if len(sys.argv) > 7 else 128
rng = np.random.default_rng(1)
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
    mask[t, :min(nkv, past + t + 1)] = 0
mask16 = mask.astype(np.float16)
scale = 1.0 / np.sqrt(dk)
dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
ws = torch.zeros(max(16, b.lib.b200_flash_attn_workspace(dk, nh, nt, nkv)), dtype=torch.uint8, device="cuda")
dst = torch.full((nt, nh, dk), float("nan"), dtype=torch.float32, device="cuda")
qd, kd, vd, md = dev(q), dev(kc), dev(vc), dev(mask16.view(np.uint16))       # keep them alive: a temporary's block is recycled by the next allocation
b.check(b.lib.b200_flash_attn_ext(b.p(qd), nh * dk, dk, b.p(kd), rb_row, rb_head, b.p(vd), rb_row, rb_head,
                                  b.p(md), nkv, b.p(dst), kvt, dk, dk, nh, nhkv, nt, nkv, scale, 0.0, 0.0, b.p(ws), b.stream()))
torch.cuda.synchronize()
got = dst.cpu().numpy()
Kd = orc_dequant(kvt, kc, nkv, nhkv * dk).astype(np.float64).reshape(nkv, nhkv, dk)
Vd = orc_dequant(kvt, vc, nkv, nhkv * dk).astype(np.float64).reshape(nkv, nhkv, dk)
q16 = q.astype(np.float16).astype(np.float64)
truth = np.zeros((nt, nh, dk))
for h in range(nh):
    hk = h // (nh // nhkv)
    s = (q16[:, h] @ Kd[:, hk].T) * scale + mask[:nt].astype(np.float64)
    p = np.exp(s - s.max(axis=1, keepdims=True))
    truth[:, h] = (p @ Vd[:, hk]) / p.sum(axis=1, keepdims=True)
err = np.abs(got - truth) / np.abs(truth).max()
print(f"{sys.argv[1]} D={dk} nh={nh} nhkv={nhkv} nt={nt} nkv={nkv} past={past}: finite {np.isfinite(got).mean():.3f} max err {np.nanmax(err):.3e}")
for t0 in range(0, nt, 128):
    e = err[t0:t0 + 128]
    print(f"  q tile {t0 // 128}: max err {np.nanmax(e):.2e}; per head", " ".join(f"{np.nanmax(e[:, h]):.1e}" for h in range(min(nh, 8))), "| worst rows", np.argsort(-np.nanmax(e, axis=(1, 2)))[:5] + t0)
