#!/usr/bin/env python3
"""Bring-up aid for the wgmma batched MUL_MAT (mmq_tc.cu, mmq_tc32.cu): one shape, error statistics against the C oracle, sample values."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import load_pkg  # noqa: E402
from refutil import Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K, orc_mul_mat, rand_blocks  # noqa: E402

b = load_pkg().ops
T = {"q4_K": Q4_K, "q5_K": Q5_K, "q6_K": Q6_K, "q4_0": Q4_0, "q5_0": Q5_0, "q8_0": Q8_0}[sys.argv[1] if len(sys.argv) > 1 else "q4_K"]
m, k, n = (int(v) for v in (sys.argv[2:5] if len(sys.argv) > 4 else (128, 2048, 128)))
rng = np.random.default_rng(3)
W = rand_blocks(rng, T, m, k)
x = rng.standard_normal((n, k)).astype(np.float32)
want = orc_mul_mat(T, W, x, m, n, k)
Wd = torch.from_numpy(np.concatenate([W.reshape(-1), np.zeros(64, np.uint8)])).cuda()
b.check(b.lib.b200_repack_rows(T, b.p(Wd), m, k, b.stream()))
ws = torch.zeros(b.lib.b200_mul_mat_q_workspace(T, m, k, n), dtype=torch.uint8, device="cuda")
dst = torch.full((n, m), float("nan"), dtype=torch.float32, device="cuda")
xd = torch.from_numpy(x).cuda()
b.check(b.lib.b200_mul_mat_q(T, b.p(Wd), b.p(xd), k, b.p(dst), m, m, k, n, b.p(ws), b.stream()))
torch.cuda.synchronize()
got = dst.cpu().numpy()
err = np.abs(got - want) / np.abs(want).max()
print(f"type {sys.argv[1] if len(sys.argv) > 1 else 'q4_K'} m={m} k={k} n={n}: finite {np.isfinite(got).mean():.3f}  max err {np.nanmax(err):.3e}  frac<1e-5 {(err < 1e-5).mean():.4f}")
print(" got ", got[0, :6], "\n want", want[0, :6])
if np.nanmax(err) > 1e-4:
    bad = np.argwhere(~(err < 1e-5))
    print(" first bad (n, r):", bad[:8].tolist(), " bad rows", sorted(set(bad[:, 1].tolist()))[:16], " bad cols", sorted(set(bad[:, 0].tolist()))[:16])
