#!/usr/bin/env python3
"""In-kernel timeline of one decode token (B200_TRACE, common.cuh): which part of every matvec / attention launch is spent waiting
for the previous kernel, rebuilding activations, waiting for the first ring slot, computing.  Runs bench.py's device-resident leg
(CUDA graph + PDL, the configuration `value` is measured in), drops the trace of the warm-up tokens and prints the last token.
usage: tools/trace_decode.py [bench.py flags, e.g. --n-past 512 --kv f16] > gpurun_out/r2_trace_decode.txt"""
import ctypes as C
import os
import sys

os.environ["B200_TRACE"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402

WORDS = 12


def dump(ops, fn):
    buf = (C.c_ulonglong * (4096 * WORDS))()
    f = getattr(ops.lib, fn)
    f.restype = C.c_int
    n = f(buf, 4096)
    return [[int(buf[i * WORDS + j]) for j in range(WORDS)] for i in range(n)]


def main():
    import importlib
    import torch
    from conftest import load_pkg
    args = bench.parse()
    pkg = load_pkg()
    G = importlib.import_module("llama_box_b200.graph"); M = importlib.import_module("llama_box_b200.model")
    ops = pkg.ops
    torch.cuda.set_device(0)
    kvt = G.F16 if args.kv == "f16" else G.Q8_0
    model = M.SyntheticLlama(args.model, args.ftype, n_ctx=args.ctx, kv_type=kvt, n_layer=args.layers or None)
    ex = G.Executor(0)
    flags = (0 if args.no_graphs else G.EXEC_CUDA_GRAPHS) | (0 if args.no_fusion else G.EXEC_FUSION)
    stream = torch.cuda.Stream()
    bench.device_resident_leg(args, model, ex, ops, G, stream, flags, args.n_past, 10, 6, 0, clocks=False)
    dump(ops, "b200_mmv_trace_dump"); dump(ops, "b200_fa_trace_dump")              # discard
    res = bench.device_resident_leg(args, model, ex, ops, G, stream, flags, args.n_past + 20, 2, 0, 0, clocks=False)
    mm = dump(ops, "b200_mmv_trace_dump"); fa = dump(ops, "b200_fa_trace_dump")
    print(f"# {args.model} {args.ftype} kv={args.kv} n_past~{args.n_past + 20}; 2 traced tokens at {res['ms_per_step']:.3f} ms/token; records: mmvq {len(mm)}, attention {len(fa)}")
    recs = []
    for r in mm:
        cta = r[8] >> 48; pairs = (r[8] >> 16) & 0xffffffff; typ = (r[8] >> 8) & 0xff; nm = r[8] & 0xff
        recs.append(("mmvq", r, f"cta {cta:3d} units {pairs:6d} type {typ:2d} mats {nm} k {r[9]}"))
    for r in fa:
        recs.append(("attn", r, f"split {r[8] >> 48:2d}/{r[8] & 0xffff} n_kv {(r[8] >> 16) & 0xffffffff}"))
    recs.sort(key=lambda x: x[1][0])
    t0 = recs[0][1][0]
    # SM clock per ns from the longest record
    best = max(recs, key=lambda x: x[1][11] - x[1][0])[1]
    ghz = (best[10] - best[1]) / max(1, best[11] - best[0])
    print(f"# SM clock ~{ghz:.3f} GHz (clock64 / globaltimer over the longest record); times in us; columns = deltas between consecutive stamps")
    print("# mmvq: entry->primed | ->prev kernel done (griddepcontrol.wait) | ->activations ready | ->warp0 first slot | ->warp0 done | ->CTA done")
    print("# attn: entry->K/V requested | ->QKV done (wait) | ->rope+stage | ->positions done | ->cluster's partials published | ->slice merged | ->exit")
    last_end = None
    for kind, r, info in recs:
        c = [r[1], r[2], r[3], r[4], r[5], r[6]] + ([r[7]] if kind == "attn" else []) + [r[10]]
        d = [(c[i + 1] - c[i]) / ghz / 1e3 if c[i + 1] and c[i] else float("nan") for i in range(len(c) - 1)]
        start = (r[0] - t0) / 1e3; end = (r[11] - t0) / 1e3
        gap = "" if last_end is None else f" (start {start - last_end:+6.2f} vs prev end)"
        print(f"{start:9.2f} {kind} dur {end - start:6.2f} | " + " ".join(f"{x:6.2f}" for x in d) + f" | {info}{gap}")
        last_end = end


if __name__ == "__main__":
    main()
