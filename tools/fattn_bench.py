#!/usr/bin/env python3
"""Kernel-level timing of the multi-token FLASH_ATTN_EXT (b200_flash_attn_ext) at prefill shapes: TinyLlama (32 query heads, 4 KV heads,
head 64) and Llama-3-8B (32 / 8, head 128), F16 and Q8_0 caches, causal mask with `past` cached positions.  CUDA events on the launching
stream around 20 calls after 3 warm-ups; the calls are queued behind a device sleep, so the window times the kernels, not the enqueue.

    fattn_bench.py                        one arm, the prefill shapes (n_tok 512, n_kv 512 .. 8192)
    fattn_bench.py --sweep                the token sweep (n_tok 8 .. 64, n_kv 512 / 2048) that places the head-64 minimum
    fattn_bench.py --arms [--reps 3] ...  both arms, the tensor-core kernel and the vector kernel (B200_FATTN_DISABLE_TC=1), as
                                          alternating child processes: the median of each, their ratio and the largest difference
                                          of their outputs

Below the head-64 minimum the dispatch chooses the vector kernel in both arms; a sweep under it needs a library built with a lower
FT_MIN_TOK_D64 (fattn_tc.cu), which B200_OPS_LIB selects.  Each row says which kernel ran (torch.profiler, one call).  Useful TFLOP/s = 4 n_head D
(visible query / position pairs) / time; the share is of the H100 SXM data sheet's dense f16 rate, 989 TFLOP/s at 700 W."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
F16, Q8_0 = 1, 8
PEAK_F16 = 989.0
TINY, L8B = ("tinyllama", 32, 4, 64), ("llama3-8b", 32, 8, 128)


def cases(sweep):
    """(model, n_head, n_head_kv, D, kv type, n_tok, n_kv, past): the batch is the last n_tok positions of n_kv"""
    out = []
    for kvt in (F16, Q8_0):
        if sweep:
            for nkv in (512, 2048):
                for nt in (8, 12, 16, 24, 32, 40, 48, 64):
                    out.append(TINY + (kvt, nt, nkv, nkv - nt))
        else:
            for nkv in (512, 2048, 4096, 8192):
                out.append(TINY + (kvt, 512, nkv, nkv - 512))
            out.append(L8B + (kvt, 512, 4096, 3584))
    return out


def visible_pairs(nt, nkv, past):
    return sum(min(nkv, past + t + 1) for t in range(nt))


def worker(args):
    import numpy as np
    import torch
    from conftest import load_pkg
    b = load_pkg().ops
    out = []
    st = torch.cuda.Stream()
    for model, nh, nhkv, d, kvt, nt, nkv, past in cases(args.sweep):
        gen = torch.Generator(device="cuda"); gen.manual_seed(nt * 7 + nkv + kvt)
        q = torch.randn(nt, nh, d, device="cuda", generator=gen)
        if kvt == F16:
            rb_row, rb_head = nhkv * d * 2, d * 2
            k = torch.randn(nkv, nhkv * d, device="cuda", generator=gen).half()
            v = torch.randn(nkv, nhkv * d, device="cuda", generator=gen).half()
        else:                                                   # q8_0 blocks: f16 d in [0.01, 0.03), int8 quants
            rb_row, rb_head = nhkv * d // 32 * 34, d // 32 * 34

            def q8():
                blk = torch.randint(-127, 128, (nkv, nhkv * d // 32, 34), device="cuda", generator=gen, dtype=torch.int32).to(torch.int8).view(torch.uint8)
                dd = (0.01 + 0.02 * torch.rand(nkv, nhkv * d // 32, device="cuda", generator=gen)).half()
                blk[:, :, 0:2] = dd.view(torch.uint8).view(nkv, nhkv * d // 32, 2)
                return blk.contiguous()
            k, v = q8(), q8()
        rows = torch.arange((nt + 63) // 64 * 64, device="cuda")[:, None]          # rows padded to 64 as libllama pads them
        mask = torch.where(torch.arange(nkv, device="cuda")[None, :] <= past + rows, 0.0, float("-inf")).half()
        dst = torch.full((nt, nh, d), float("nan"), device="cuda")
        scale = 1.0 / d ** 0.5

        def call():
            b.check(b.lib.b200_flash_attn_ext(b.p(q), nh * d, d, b.p(k), rb_row, rb_head, b.p(v), rb_row, rb_head, b.p(mask), nkv, b.p(dst),
                                              kvt, d, d, nh, nhkv, nt, nkv, scale, 0.0, 0.0, None, torch.cuda.current_stream().cuda_stream))
        with torch.cuda.stream(st):
            for _ in range(3):
                call()
            st.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                call()
                st.synchronize()
            names = {e.key for e in prof.key_averages() if "fattn" in e.key}
            kernel = "tc" if any("fattn_tc_kernel" in n for n in names) else "vec" if any("fattn_vec_kernel" in n for n in names) else ",".join(sorted(names))
            reps = 20
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(40_000_000)                       # ~20 ms: the calls below are queued before the first one starts
            e0.record(st)
            for _ in range(reps):
                call()
            e1.record(st); st.synchronize()
        ms = e0.elapsed_time(e1) / reps
        tf = 4.0 * nh * d * visible_pairs(nt, nkv, past) / ms / 1e9
        kvn = "f16" if kvt == F16 else "q8_0"
        out.append({"shape": f"{model} {nh}/{nhkv} D{d} {kvn}", "n_tok": nt, "n_kv": nkv, "past": past, "kernel": kernel, "ms": ms,
                    "tflops_useful": tf, "share_of_f16_peak": tf / PEAK_F16})
        if args.dump:
            np.save(os.path.join(args.dump, f"{len(out) - 1}.npy"), dst.cpu().numpy())
        del q, k, v, mask, dst
    print(json.dumps(out))


def arms(args):
    import numpy as np
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout.strip()
    print(card.replace("\n", " | "))
    base = [sys.executable, os.path.abspath(__file__), "--worker"] + (["--sweep"] if args.sweep else [])
    runs = {"tc": [], "vec": []}
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(args.reps):
            for arm in ("tc", "vec"):
                env = dict(os.environ)
                env.pop("B200_FATTN_DISABLE_TC", None)
                if arm == "vec":
                    env["B200_FATTN_DISABLE_TC"] = "1"
                dd = os.path.join(tmp, arm); os.makedirs(dd, exist_ok=True)
                r = subprocess.run(base + ["--dump", dd], capture_output=True, text=True, env=env)
                if r.returncode != 0:
                    sys.exit(r.stdout[-2000:] + r.stderr[-2000:])
                runs[arm].append(json.loads(r.stdout.strip().splitlines()[-1]))
        res = []
        for i, row in enumerate(runs["tc"][0]):
            tc = statistics.median(r[i]["ms"] for r in runs["tc"]); vec = statistics.median(r[i]["ms"] for r in runs["vec"])
            a, g = np.load(os.path.join(tmp, "tc", f"{i}.npy")), np.load(os.path.join(tmp, "vec", f"{i}.npy"))
            fl = row["tflops_useful"] * row["ms"]
            res.append({"shape": row["shape"], "n_tok": row["n_tok"], "n_kv": row["n_kv"], "past": row["past"],
                        "kernels": row["kernel"] + "/" + runs["vec"][0][i]["kernel"],
                        "tc_ms": round(tc, 4), "tc_ms_all": [round(r[i]["ms"], 4) for r in runs["tc"]],
                        "vec_ms": round(vec, 4), "vec_ms_all": [round(r[i]["ms"], 4) for r in runs["vec"]], "speedup": round(vec / tc, 2),
                        "tc_tflops_useful": round(fl / tc, 1), "tc_share_of_f16_peak": round(fl / tc / PEAK_F16, 3),
                        "vec_tflops_useful": round(fl / vec, 1),
                        "arms_max_rel_diff": float(np.abs(a - g).max() / np.abs(g).max())})
            print(res[-1])
    print(json.dumps({"card": card, "results": res}))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--arms", action="store_true"); ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--worker", action="store_true"); ap.add_argument("--dump", default="")
    a = ap.parse_args()
    arms(a) if a.arms else worker(a)
