#!/usr/bin/env python3
"""Kernel-level timing of the batched MUL_MAT (b200_mul_mat_q2) on the matmul shapes of the BASELINE models: CUDA events on the
launching stream, 20 repetitions after 3 warm-ups.

    mmq_bench.py [--cols 512] [--family kquant|block32|q2q3|iq4|all]  one arm, the shapes at one column count
    mmq_bench.py --sweep 9,16,32,64,128 --family block32          column sweep on the 8B shapes (where the tensor cores start to win)
    mmq_bench.py --arms [--reps 3] ...                            both arms (tensor cores / column groups through the matvec,
                                                                  B200_MMQ_DISABLE_TC=1) as alternating child processes, the median
                                                                  of each, their ratio, and the largest difference of their outputs

q2q3: Q2_K and Q3_K (the wide path's formats) on the Llama-3-8B and Llama-3-70B projection shapes, weights in ggml's native block layout
(the layout the library keeps for them); their other arm is the wide matvec (b200_mul_mat_vec_wide, one pass per column group).
iq4: IQ4_NL and IQ4_XS on the same shapes, likewise in native layout, on the int8 kernel (mmq_tc32.cu) against the wide matvec.

Useful TFLOP/s = 2 m k n / time; the share of peak is against the data sheet's dense rate of the pipe the kernel uses (int8 1979 TOPS
for the block-32 and IQ4 formats, f16 989 TFLOP/s for the K-quants; H100 SXM at 700 W)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def shapes(G, family):
    kq = [("wq/wo 4096x4096 Q4_K", G.Q4_K, 4096, 4096), ("wk/wv 1024x4096 Q4_K", G.Q4_K, 1024, 4096), ("gate/up 14336x4096 Q4_K", G.Q4_K, 14336, 4096),
          ("down 4096x14336 Q4_K", G.Q4_K, 4096, 14336), ("down 4096x14336 Q6_K", G.Q6_K, 4096, 14336), ("output 128256x4096 Q6_K", G.Q6_K, 128256, 4096)]
    b32 = [("wq/wo 4096x4096 Q8_0", G.Q8_0, 4096, 4096), ("wk/wv 1024x4096 Q8_0", G.Q8_0, 1024, 4096), ("gate/up 14336x4096 Q8_0", G.Q8_0, 14336, 4096),
           ("down 4096x14336 Q8_0", G.Q8_0, 4096, 14336), ("output 128256x4096 Q8_0", G.Q8_0, 128256, 4096),
           ("tinyllama 2048x2048 Q4_0", G.Q4_0, 2048, 2048), ("tinyllama gate/up 5632x2048 Q4_0", G.Q4_0, 5632, 2048), ("tinyllama down 2048x5632 Q4_0", G.Q4_0, 2048, 5632),
           ("qwen2-72b down 8192x29568 Q5_0", G.Q5_0, 8192, 29568), ("qwen2-72b down 8192x29568 Q8_0", G.Q8_0, 8192, 29568)]
    llama = [("8b wq/wo 4096x4096", 4096, 4096), ("8b wk/wv 1024x4096", 1024, 4096), ("8b gate/up 14336x4096", 14336, 4096),
             ("8b down 4096x14336", 4096, 14336), ("70b wq/wo 8192x8192", 8192, 8192), ("70b wk/wv 1024x8192", 1024, 8192),
             ("70b gate/up 28672x8192", 28672, 8192), ("70b down 8192x28672", 8192, 28672)]
    q23 = [(f"{name} {tn}", t, m, k) for name, m, k in llama for tn, t in (("Q2_K", G.Q2_K), ("Q3_K", G.Q3_K))]
    iq4 = [(f"{name} {tn}", t, m, k) for name, m, k in llama for tn, t in (("IQ4_NL", G.IQ4_NL), ("IQ4_XS", G.IQ4_XS))]
    return {"kquant": kq, "block32": b32, "q2q3": q23, "iq4": iq4, "all": kq + b32 + q23 + iq4}[family]


class NativeWeights:
    """random valid blocks in ggml's own layout (model.Weights repacks, and knows only the tuned formats)"""
    def __init__(self, b, t, m, k):
        import numpy as np
        import torch
        from refutil import rand_blocks
        self.buf = torch.from_numpy(np.concatenate([rand_blocks(np.random.default_rng(1), t, m, k).reshape(-1), np.zeros(64, np.uint8)])).cuda()
        self.row_bytes = b.lib.b200_wide_row_bytes(t, k)


def worker(args):
    import importlib
    import numpy as np
    import torch
    from conftest import load_pkg
    b = load_pkg().ops
    M = importlib.import_module("llama_box_b200.model"); G = importlib.import_module("llama_box_b200.graph")
    cols = [int(c) for c in args.sweep.split(",")] if args.sweep else [args.cols]
    todo = shapes(G, args.family)
    if args.sweep:
        todo = [s for s in todo if "4096" in s[0] and "output" not in s[0]]
    out = []
    st = torch.cuda.Stream()
    for name, t, m, k in todo:
        gen = torch.Generator(device="cuda"); gen.manual_seed(1)
        native = t in (G.Q2_K, G.Q3_K, G.IQ4_NL, G.IQ4_XS)
        W = NativeWeights(b, t, m, k) if native else M.Weights(t, m, k, gen=gen)
        kp = k if native else b.lib.b200_padded_k(t, k)
        rb = W.row_bytes if native else b.row_bytes(t, kp)
        for n in cols:
            x = torch.randn(n, k, device="cuda", generator=gen)
            ws = torch.zeros(b.lib.b200_mul_mat_q_workspace(t, m, kp, n), dtype=torch.uint8, device="cuda")
            dst = torch.zeros(n, m, device="cuda")
            call = lambda: b.check(b.lib.b200_mul_mat_q2(t, b.p(W.buf), b.p(x), k, b.p(dst), m, m, kp, k, n, b.p(ws), torch.cuda.current_stream().cuda_stream))  # noqa: E731
            with torch.cuda.stream(st):
                for _ in range(3):
                    call()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                reps = 20
                st.synchronize(); e0.record(st)
                for _ in range(reps):
                    call()
                e1.record(st); st.synchronize()
            ms = e0.elapsed_time(e1) / reps
            peak = 1979.0 if t in (G.Q4_0, G.Q5_0, G.Q8_0, G.IQ4_NL, G.IQ4_XS) else 989.0
            tf = 2.0 * m * k * n / ms / 1e9
            out.append({"shape": name, "n_tokens": n, "ms": ms, "tflops_useful": tf, "share_of_pipe_peak": tf / peak, "weight_GBps_per_pass": m * rb / ms / 1e6})
            if args.dump:
                np.save(os.path.join(args.dump, f"{len(out) - 1}.npy"), dst[:, :: max(1, m // 256)].cpu().numpy())
            del x, ws, dst
        del W
    print(json.dumps(out))


def arms(args):
    import numpy as np
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout.strip()
    print(card.replace("\n", " | "))
    base = [sys.executable, os.path.abspath(__file__), "--worker", "--family", args.family, "--cols", str(args.cols)] + (["--sweep", args.sweep] if args.sweep else [])
    runs = {"tc": [], "groups": []}
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(args.reps):
            for arm in ("tc", "groups"):
                env = dict(os.environ)
                env.pop("B200_MMQ_DISABLE_TC", None)
                if arm == "groups":
                    env["B200_MMQ_DISABLE_TC"] = "1"
                d = os.path.join(tmp, arm); os.makedirs(d, exist_ok=True)
                r = subprocess.run(base + ["--dump", d], capture_output=True, text=True, env=env)
                if r.returncode != 0:
                    sys.exit(r.stdout[-2000:] + r.stderr[-2000:])
                runs[arm].append(json.loads(r.stdout.strip().splitlines()[-1]))
        res = []
        for i, row in enumerate(runs["tc"][0]):
            tc = statistics.median(r[i]["ms"] for r in runs["tc"]); gr = statistics.median(r[i]["ms"] for r in runs["groups"])
            a, g = np.load(os.path.join(tmp, "tc", f"{i}.npy")), np.load(os.path.join(tmp, "groups", f"{i}.npy"))
            fl = row["tflops_useful"] * row["ms"]
            res.append({"shape": row["shape"], "n_tokens": row["n_tokens"], "tc_ms": round(tc, 4), "tc_ms_all": [round(r[i]["ms"], 4) for r in runs["tc"]],
                        "groups_ms": round(gr, 4), "groups_ms_all": [round(r[i]["ms"], 4) for r in runs["groups"]], "speedup": round(gr / tc, 2),
                        "tc_tflops_useful": round(fl / tc, 1), "tc_share_of_pipe_peak": round(row["share_of_pipe_peak"] * row["ms"] / tc, 3),
                        "groups_weight_GBps": round(row["weight_GBps_per_pass"] * row["ms"] / gr * ((row["n_tokens"] + 7) // 8), 0),
                        "arms_max_rel_diff": float(np.abs(a - g).max() / np.abs(g).max())})
            print(res[-1])
    print(json.dumps({"card": card, "results": res}))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cols", type=int, default=512); ap.add_argument("--sweep", default=""); ap.add_argument("--family", default="all", choices=["kquant", "block32", "q2q3", "iq4", "all"])
    ap.add_argument("--arms", action="store_true"); ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--worker", action="store_true"); ap.add_argument("--dump", default="")
    a = ap.parse_args()
    arms(a) if a.arms else worker(a)
