#!/usr/bin/env python3
"""First timing of the wide path (llama-box_b200/csrc/mmvq_ext.cu) — NOT yet run on hardware (DESIGN.md §9): b200_mul_mat_vec_wide per format on the
Llama-3-8B matmul shapes (decode column and an 8-column verify batch) and b200_mul_mat_id on a Mixtral-8x7B-shaped expert stack.  CUDA events on the
launching stream, 20 repetitions after 3 warm-ups, a fresh weight buffer per shape (> L2 for the big ones).  Prints one JSON line per case:
GB/s of weight bytes against MEASURED_PEAKS.json's HBM figure.
    python tools/wide_bench.py [ncols]"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import load_pkg  # noqa: E402

b = load_pkg().ops
L = b.lib
ncols = int(sys.argv[1]) if len(sys.argv) > 1 else 1
peak = 3350.0                      # H100 SXM data sheet (HBM3), unless MEASURED_PEAKS.json has a measured value
try:
    peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:  # noqa: BLE001
    pass
NAMES = {2: "q4_0", 3: "q4_1", 6: "q5_0", 7: "q5_1", 8: "q8_0", 10: "q2_K", 11: "q3_K", 12: "q4_K", 13: "q5_K", 14: "q6_K", 20: "iq4_nl", 23: "iq4_xs", 39: "mxfp4"}
st = torch.cuda.Stream()


def timed(fn, reps=20):
    with torch.cuda.stream(st):
        for _ in range(3):
            fn(torch.cuda.current_stream().cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st.synchronize(); e0.record(st)
        for _ in range(reps):
            fn(torch.cuda.current_stream().cuda_stream)
        e1.record(st); st.synchronize()
    return e0.elapsed_time(e1) / reps


def rand_weights(nbytes):
    """random bytes are valid blocks for timing purposes (values may be inf / nan: only the time is read)"""
    return torch.randint(0, 255, (nbytes + 64,), dtype=torch.uint8, device="cuda")


for t in sorted(NAMES):
    for m, k in ((4096, 4096), (14336, 4096), (4096, 14336)):
        if not L.b200_wide_shape_supported(t, k):
            continue
        rb = L.b200_wide_row_bytes(t, k)
        W = rand_weights(m * rb); x = torch.randn(ncols, k, device="cuda"); dst = torch.zeros(ncols, m, device="cuda")
        ms = timed(lambda s: b.check(L.b200_mul_mat_vec_wide(t, b.p(W), b.p(x), k, b.p(dst), m, None, None, m, k, ncols, s)))
        print(json.dumps({"op": "mul_mat_vec_wide", "type": NAMES[t], "m": m, "k": k, "ncols": ncols, "us": round(ms * 1e3, 2), "weight_GBps": round(m * rb / ms / 1e6, 1),
                          "frac_of_hbm_peak": round(m * rb / ms / 1e6 / peak, 3)}))
        del W, x, dst
# Mixtral-8x7B expert stack: 8 experts, 2 used, up/gate 14336x4096
for t in (12, 14, 3):
    m, k, ne, nu, nt = 14336, 4096, 8, 2, ncols
    rb = L.b200_wide_row_bytes(t, k)
    W = rand_weights(ne * m * rb); xb = torch.randn(nt, 1, k, device="cuda"); dst = torch.zeros(nt, nu, m, device="cuda")
    ids = torch.from_numpy(np.stack([np.random.default_rng(i).permutation(ne)[:nu] for i in range(nt)]).astype(np.int32)).cuda()
    ms = timed(lambda s: b.check(L.b200_mul_mat_id(t, b.p(W), m * rb, b.p(xb), k, k, 1, b.p(ids), nu, b.p(dst), nu * m, m, m, k, ne, nu, nt, s)))
    print(json.dumps({"op": "mul_mat_id", "type": NAMES[t], "m": m, "k": k, "n_expert": ne, "n_used": nu, "n_tok": nt, "us": round(ms * 1e3, 2),
                      "weight_GBps_streamed": round(min(nt * nu, ne) * m * rb / ms / 1e6, 1)}))
    del W, xb, dst, ids
