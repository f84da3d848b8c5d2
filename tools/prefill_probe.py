#!/usr/bin/env python3
"""Prefill tok/s through the product path (libllama + libggml-b200.so, in-process) on a synthetic GGUF (--config / --ftype,
default Llama-3-8B Q4_K_M): a 4096-token prompt in 512-token ubatches (BASELINE config 3) and the first 512-token ubatch alone;
F16 and Q8_0 KV.  B200_MMQ_DISABLE_TC=1 in the environment times the column-group arm of the batched MUL_MAT.
Q2_K / Q3_K_M / IQ4_NL / IQ4_XS files (--ftype) run on the device with GGML_B200_WIDE=1 in the environment; their column-group arm is
the wide matvec."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from drvutil import Drv  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--config", default="llama3-8b"); ap.add_argument("--ftype", default="Q4_K_M")
args = ap.parse_args()
path = f"/dev/shm/b200_bench_{args.config}_{args.ftype}.gguf"
if not os.path.exists(path):
    subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "make_gguf.py"), "--config", args.config, "--ftype", args.ftype, "--out", path], check=True, capture_output=True)
rng = np.random.default_rng(1)
for kv in ("f16", "q8_0"):
    d = Drv(path, ctx=8192, ubatch=512, ctk=kv, ctv=kv)
    toks = rng.integers(0, d.n_vocab, size=4096).tolist()
    d.decode(toks[:512]); d.logits(); d.reset()
    res = {}
    for n in (512, 4096):
        t0 = time.perf_counter()
        for i in range(0, n, 2048):
            d.decode(toks[i:min(n, i + 2048)])
        d.logits()
        res[n] = n / (time.perf_counter() - t0)
        d.reset()
    print(f"{args.config} {args.ftype} (batched MUL_MAT: {'column groups' if os.environ.get('B200_MMQ_DISABLE_TC') else 'tensor cores'}) kv {kv}: pp512 {res[512]:.0f} tok/s, pp4096 {res[4096]:.0f} tok/s  (tc attention {'off' if os.environ.get('B200_FATTN_DISABLE_TC') else 'on'})")
    d.close()
