#!/usr/bin/env python3
"""First timing of the wide path (llama-box_b200/csrc/mmvq_ext.cu) — NOT yet run on hardware (DESIGN.md §9): b200_mul_mat_vec_wide per format on the
Llama-3-8B matmul shapes (decode column and an 8-column verify batch) and b200_mul_mat_id on a Mixtral-8x7B-shaped expert stack.  CUDA events on the
launching stream, 20 repetitions after 3 warm-ups, a fresh weight buffer per shape (> L2 for the big ones).  Prints one JSON line per case:
GB/s of weight bytes against MEASURED_PEAKS.json's HBM figure.
    python tools/wide_bench.py [ncols]

--mmid: prefill MUL_MAT_ID (b200_mul_mat_id2) in two arms, the grouped tensor-core GEMM and B200_MMQ_DISABLE_TC=1 (the matvec), as alternating
child processes (the switch is read once per process) timed with CUDA events, on a Mixtral-8x7B stack (4096 / 14336, 8 experts, top-2: up
Q4_K, down Q6_K) and a fine-grained one (2048 / 768, 128 experts, top-8: up Q4_K, down Q8_0).  Prints per case and arm ms and useful
TFLOP/s (2 m k N, N = n_tok * n_used), and the largest difference between the arms' outputs relative to the output maximum.
    python tools/wide_bench.py --mmid [--n-tok 512 ...] [--sweep] [--shapes NAME ...] [--rounds 2] [--lib PATH]
--sweep times 8 ... 128 tokens, where MMID_MIN_TOK / MMID_MIN_PAIRS are placed; give --lib a build with -DMMID_MIN_TOK=9 -DMMID_MIN_PAIRS=0
so that the grouped arm runs at every count (the default build sends the small counts to the matvec in both arms)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

NAMES = {2: "q4_0", 3: "q4_1", 6: "q5_0", 7: "q5_1", 8: "q8_0", 10: "q2_K", 11: "q3_K", 12: "q4_K", 13: "q5_K", 14: "q6_K", 20: "iq4_nl", 23: "iq4_xs", 39: "mxfp4"}
# (name, m, k, n_expert, n_used, type, shared activation)
MMID_SHAPES = [("mixtral_up", 14336, 4096, 8, 2, 12, True), ("mixtral_down", 4096, 14336, 8, 2, 14, False),
               ("finegrained_up", 768, 2048, 128, 8, 12, True), ("finegrained_down", 2048, 768, 128, 8, 8, False)]


def mmid_parent(argv):
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--mmid", action="store_true")
    ap.add_argument("--n-tok", type=int, nargs="*", default=[512])
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--shapes", nargs="*", default=[s[0] for s in MMID_SHAPES])
    a = ap.parse_args(argv)
    toks = [8, 12, 16, 24, 32, 48, 64, 96, 128] if a.sweep else a.n_tok
    tmp = tempfile.mkdtemp()
    for name, m, k, ne, nu, t, shared in [s for s in MMID_SHAPES if s[0] in a.shapes]:
        for nt in toks:
            res = {"tc": [], "mv": []}
            for r in range(a.rounds):
                for arm in (("tc", "mv") if r % 2 == 0 else ("mv", "tc")):
                    env = dict(os.environ)
                    env.pop("B200_MMQ_DISABLE_TC", None)
                    if arm == "mv":
                        env["B200_MMQ_DISABLE_TC"] = "1"
                    if a.lib:
                        env["B200_OPS_LIB"] = a.lib
                    out = os.path.join(tmp, f"{arm}.npy")
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--mmid-child", name, str(nt), out], env=env, capture_output=True, text=True)
                    if p.returncode != 0:
                        sys.stderr.write(p.stderr[-3000:])
                        raise SystemExit(f"child failed: {name} {nt} {arm}")
                    res[arm].append(json.loads(p.stdout.strip().splitlines()[-1]))
            o_tc, o_mv = np.load(os.path.join(tmp, "tc.npy")), np.load(os.path.join(tmp, "mv.npy"))
            diff = float(np.abs(o_tc - o_mv).max() / np.abs(o_mv).max())
            flop = 2.0 * m * k * nt * nu
            line = {"op": "mul_mat_id", "shape": name, "type": NAMES[t], "m": m, "k": k, "n_expert": ne, "n_used": nu, "n_tok": nt}
            for arm in ("tc", "mv"):
                ms = min(x["ms"] for x in res[arm])
                line[arm + "_ms"] = round(ms, 4); line[arm + "_tflops"] = round(flop / ms / 1e9, 2); line[arm + "_workspace"] = res[arm][0]["workspace"]
            line["speedup"] = round(line["mv_ms"] / line["tc_ms"], 2)
            line["max_rel_diff"] = diff
            print(json.dumps(line), flush=True)


def mmid_child(name, nt, out):
    import torch
    from conftest import load_pkg
    b = load_pkg().ops
    L = b.lib
    _, m, k, ne, nu, t, shared = [s for s in MMID_SHAPES if s[0] == name][0]
    rb = L.b200_row_bytes(t, k)
    g = torch.Generator(device="cuda").manual_seed(1)
    # random bytes with bit 14 of every 16-bit word cleared: every f16 scale is finite and below 2, so both arms' outputs compare
    W = (torch.randint(-32768, 32767, ((ne * m * rb + 64) // 2,), dtype=torch.int16, device="cuda", generator=g) & ~0x4000).view(torch.uint8)
    n_b1 = 1 if shared else nu
    x = torch.randn(nt, n_b1, k, device="cuda", generator=g)
    ids = torch.stack([torch.randperm(ne, device="cuda", generator=g)[:nu] for _ in range(nt)]).to(torch.int32).contiguous()
    dst = torch.zeros(nt, nu, m, device="cuda")
    wsb = L.b200_mul_mat_id_workspace(t, m, k, ne, nu, nt)
    ws = torch.zeros(max(wsb, 256), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream()

    def call():
        b.check(L.b200_mul_mat_id2(t, b.p(W), m * rb, b.p(x), n_b1 * k, k, n_b1, b.p(ids), nu, b.p(dst), nu * m, m, m, k, ne, nu, nt, b.p(ws), st.cuda_stream))
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    reps = 20
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        call()
    e1.record(st)
    torch.cuda.synchronize()
    np.save(out, dst.cpu().numpy())
    print(json.dumps({"ms": e0.elapsed_time(e1) / reps, "workspace": int(wsb)}))


if len(sys.argv) > 1 and sys.argv[1] == "--mmid-child":
    mmid_child(sys.argv[2], int(sys.argv[3]), sys.argv[4])
    raise SystemExit(0)
if len(sys.argv) > 1 and sys.argv[1] == "--mmid":
    mmid_parent(sys.argv[1:])
    raise SystemExit(0)

import torch  # noqa: E402
from conftest import load_pkg  # noqa: E402

b = load_pkg().ops
L = b.lib
ncols = int(sys.argv[1]) if len(sys.argv) > 1 else 1
peak = 3350.0                      # H100 SXM data sheet (HBM3), unless MEASURED_PEAKS.json has a measured value
try:
    peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:  # noqa: BLE001
    pass
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
