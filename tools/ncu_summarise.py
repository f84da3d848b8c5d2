#!/usr/bin/env python3
"""Turn the round's `ncu --set full` captures (r2_*.ncu-rep, produced by tools/profile_r2.sh on the GPU) into the
evidence under profiles/ (git-ignored, per machine): one TSV per capture with the metrics the roofline discussion uses, the launch-list summary,
and profiles/r2_kernel_traffic.json (DRAM bytes per algorithmic byte of the matvec launches — what bench.py's roofline.traffic
reads instead of a hard-coded constant).  Runs here (no GPU): `ncu -i <rep> --page raw --csv`."""
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "gpurun_out")
OUT = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "profiles")

METRICS = [
    ("duration_us", "gpu__time_duration.sum", 1e-3),
    ("dram_read_MB", "dram__bytes_read.sum", 1e-6),
    ("dram_write_MB", "dram__bytes_write.sum", 1e-6),
    ("dram_pct_of_peak", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", 1),
    ("sm_pct_of_peak", "sm__throughput.avg.pct_of_peak_sustained_elapsed", 1),
    ("tensor_pipe_pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 1),
    ("tensor_subpipe_hmma_pct", "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", 1),
    ("issue_active_pct", "sm__inst_issued.avg.pct_of_peak_sustained_active", 1),
    ("warps_active_pct", "sm__warps_active.avg.pct_of_peak_sustained_active", 1),
    ("regs_per_thread", "launch__registers_per_thread", 1),
    ("grid", "launch__grid_size", 1),
    ("block", "launch__block_size", 1),
    ("smem_dyn_KB", "launch__shared_mem_per_block_dynamic", 1e-3),
    ("stall_long_scoreboard", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", 1),
    ("stall_barrier", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", 1),
    ("stall_short_scoreboard", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", 1),
    ("stall_mio_throttle", "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", 1),
    ("stall_wait", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", 1),
    ("stall_sleeping", "smsp__average_warps_issue_stalled_sleeping_per_issue_active.ratio", 1),
    ("stall_membar", "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio", 1),
    ("smem_bank_conflicts_ld", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_ld.sum", 1),
    ("smem_bank_conflicts_st", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_st.sum", 1),
    ("l2_hit_pct", "lts__t_sector_hit_rate.pct", 1),
]


def raw_rows(rep):
    r = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True)
    rows = list(csv.reader(io.StringIO(r.stdout)))
    if len(rows) < 3:
        return [], []
    hdr = rows[0]
    global UNITS
    UNITS = dict(zip(hdr, rows[1]))                        # rows[1] = units
    return hdr, rows[2:]


UNITS = {}
TO_BASE = {"nsecond": 1e-9, "ns": 1e-9, "usecond": 1e-6, "us": 1e-6, "msecond": 1e-3, "ms": 1e-3, "second": 1.0, "s": 1.0,
           "byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}


def num(s):
    try:
        return float(s.replace(",", ""))
    except ValueError:
        return None


def summarise(rep, name):
    hdr, rows = raw_rows(rep)
    if not rows:
        print("no data in", rep); return []
    col = {h: i for i, h in enumerate(hdr)}
    out = []
    for r in rows:
        d = {"kernel": r[col["Kernel Name"]][:60]}
        for key, metric, scale in METRICS:
            if metric in col:
                v = num(r[col[metric]])
                u = TO_BASE.get(UNITS.get(metric, ""), None)
                if v is not None and u is not None:        # times -> us, bytes -> MB whatever unit ncu chose for this capture
                    v = v * u * (1e6 if "second" in UNITS[metric] or UNITS[metric] in ("ns", "us", "ms", "s") else 1e-6) / scale * scale
                    d[key] = round(v, 3)
                else:
                    d[key] = None if v is None else round(v * scale, 3)
        out.append(d)
    path = os.path.join(OUT, name + ".tsv")
    keys = ["kernel"] + [k for k, _, _ in METRICS]
    with open(path, "w") as f:
        f.write("# ncu --set full --clock-control none (tools/profile_r2.sh), one row per profiled launch; from " + os.path.basename(rep) + "\n")
        f.write("\t".join(keys) + "\n")
        for d in out:
            f.write("\t".join("" if d.get(k) is None else str(d.get(k)) for k in keys) + "\n")
    print("wrote", path, len(out), "launches")
    return out


def launch_list(csv_path, name):
    if not os.path.exists(csv_path):
        return
    rows = [r for r in csv.reader(open(csv_path)) if len(r) > 5]
    hdr = None
    agg = {}
    total = 0.0
    for r in rows:
        if "Kernel Name" in r:
            hdr = {h: i for i, h in enumerate(r)}; continue
        if hdr is None or r[hdr["Metric Name"]] != "gpu__time_duration.sum":
            continue
        k = r[hdr["Kernel Name"]].split("(")[0][:48]
        v = num(r[hdr["Metric Value"]]) or 0.0
        unit = r[hdr["Metric Unit"]]
        us = v * {"ns": 1e-3, "us": 1.0, "ms": 1e3, "nsecond": 1e-3, "usecond": 1.0, "msecond": 1e3}.get(unit, 1e-3)
        a = agg.setdefault(k, [0, 0.0]); a[0] += 1; a[1] += us; total += us
    with open(os.path.join(OUT, name + ".txt"), "w") as f:
        f.write("# ncu launch list of ~2 decode tokens (gpu__time_duration.sum, --clock-control none; cold-cache, serialised: SHARES, not absolutes)\n")
        f.write(f"{'kernel':50s} {'launches':>8s} {'avg us':>9s} {'share':>7s}\n")
        for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"{k:50s} {n:8d} {us / n:9.2f} {100 * us / total:6.1f}%\n")
    print("wrote launch summary", name)


def main():
    os.makedirs(OUT, exist_ok=True)
    traffic = {}
    for fn in sorted(os.listdir(SRC)):
        if fn.startswith("r2_") and fn.endswith(".ncu-rep"):
            rows = summarise(os.path.join(SRC, fn), fn[:-8])
            if fn == "r2_mmvq.ncu-rep" and rows:
                # algorithmic bytes of the in-situ matvec launches of Llama-3-8B Q4_K_M (weights only), matched by size
                MB = 1e6
                expected = {"qkv q4_K": 6144 * 4096 * 0.5625 / MB, "qkv v=q6_K": (5120 * 0.5625 + 1024 * 0.8203125) * 4096 / MB, "wo": 4096 * 4096 * 0.5625 / MB,
                            "gate+up": 2 * 14336 * 4096 * 0.5625 / MB, "down q4_K": 4096 * 14336 * 0.5625 / MB, "down q6_K": 4096 * 14336 * 0.8203125 / MB}
                dram = alg = 0.0
                inst = []
                for d in rows:
                    rd = (d.get("dram_read_MB") or 0) + (d.get("dram_write_MB") or 0)
                    nm, ex = min(expected.items(), key=lambda kv: abs(kv[1] - (d.get("dram_read_MB") or 0)))
                    dram += rd; alg += ex
                    inst.append({"instance": nm, "algorithmic_MB": round(ex, 3), "dram_MB": round(rd, 3), "duration_us": d.get("duration_us")})
                traffic = {"source": "profiles/r2_mmvq.tsv (ncu --set full, dram__bytes_read.sum + dram__bytes_write.sum of 8 consecutive in-situ matvec launches = 2 layers)",
                           "dram_bytes_per_algorithmic_byte": dram / alg if alg else None, "launches": inst}
    launch_list(os.path.join(ROOT, "gpurun_out", "r2_launches_decode.csv"), "r2_launches_decode_summary")
    if traffic.get("dram_bytes_per_algorithmic_byte"):
        wbytes = 4616331264                                # matvec weight bytes of one Llama-3-8B Q4_K_M token (bench.py bytes_per_token)
        traffic["mmvq_per_token_dram_bytes"] = int(wbytes * traffic["dram_bytes_per_algorithmic_byte"])
        json.dump(traffic, open(os.path.join(OUT, "r2_kernel_traffic.json"), "w"), indent=1)
        print("wrote r2_kernel_traffic.json: ratio", traffic["dram_bytes_per_algorithmic_byte"])


if __name__ == "__main__":
    sys.exit(main())
