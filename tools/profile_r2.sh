#!/bin/bash
# Round-2 profiling pass (run under gpurun, ONE GPU): ncu launch list of a decode step + `--set full` captures of the kernels
# VERDICT r1 asked for.  Outputs land in gpurun_out/; tools/ncu_summarise.py turns the .ncu-rep files into profiles/r2_*.
set -u
mkdir -p gpurun_out /tmp/prof
B="python bench.py --no-e2e --no-cpu-baseline --no-extras --no-graphs"
NCU="ncu --clock-control none"
# 1. every launch of ~2 decode tokens with its device time (cold cache, serialised: shares, not absolutes)
$NCU --metrics gpu__time_duration.sum -k regex:'mmvq|fattn|mk_kernel|argmax|cpy|get_rows|rms_norm|bin_bcast' -s 340 -c 340 --csv --log-file gpurun_out/r2_launches_decode.csv $B --steps 2 --warmup 2 > /dev/null 2>&1
# 2. --set full: attention kernel, F16 KV at n_kv 768 and 4096, Q8_0 KV at 768 and 4096
$NCU --set full --import-source on -k regex:fattn_vec -s 40 -c 2 -f -o /tmp/prof/r2_fattn_f16_768 $B --steps 2 --warmup 2 --n-past 600 > /dev/null 2>&1
$NCU --set full --import-source on -k regex:fattn_vec -s 40 -c 2 -f -o /tmp/prof/r2_fattn_f16_4096 $B --steps 2 --warmup 2 --n-past 3900 > /dev/null 2>&1
$NCU --set full --import-source on -k regex:fattn_vec -s 40 -c 2 -f -o /tmp/prof/r2_fattn_q8_768 $B --steps 2 --warmup 2 --n-past 600 --kv q8_0 > /dev/null 2>&1
$NCU --set full --import-source on -k regex:fattn_vec -s 40 -c 2 -f -o /tmp/prof/r2_fattn_q8_4096 $B --steps 2 --warmup 2 --n-past 3900 --kv q8_0 > /dev/null 2>&1
# 3. --set full: the matvec launches of one layer in situ (QKV, wo, gate/up, down), the lm_head launch (persistent kernel) and argmax
$NCU --set full --import-source on -k regex:mmvq_kernel -s 64 -c 8 -f -o /tmp/prof/r2_mmvq $B --steps 2 --warmup 2 > /dev/null 2>&1
$NCU --set full --import-source on -k regex:'mk_kernel|argmax' -s 2 -c 2 -f -o /tmp/prof/r2_lmhead_argmax $B --steps 2 --warmup 2 > /dev/null 2>&1
# 4. --set full: the wgmma prefill GEMM (ffn_up shape 14336 x 4096, 512 tokens) + its activation quantiser
$NCU --set full --import-source on -k regex:'mmq_tc|quantize_mmq' -c 4 -f -o /tmp/prof/r2_mmq_tc python tools/mmq_probe.py q4_K 14336 4096 512 > gpurun_out/r2_mmq_tc_probe.log 2>&1
$NCU --set full --import-source on -k regex:'mmq_tc' -c 1 -f -o /tmp/prof/r2_mmq_tc_q6k python tools/mmq_probe.py q6_K 4096 14336 512 >> gpurun_out/r2_mmq_tc_probe.log 2>&1
# 5. --set full: the wgmma multi-token attention (32 heads / 8 KV heads, 512-token ubatch at depth 3584 -> n_kv 4096), F16 and Q8_0 cache
$NCU --set full --import-source on -k regex:fattn_tc -c 1 -f -o /tmp/prof/r2_fattn_tc_f16 python tools/fattn_probe.py f16 32 8 512 4096 3584 > gpurun_out/r2_fattn_tc_probe.log 2>&1
$NCU --set full --import-source on -k regex:fattn_tc -c 1 -f -o /tmp/prof/r2_fattn_tc_q8 python tools/fattn_probe.py q8_0 32 8 512 4096 3584 >> gpurun_out/r2_fattn_tc_probe.log 2>&1
ls -la /tmp/prof/*.ncu-rep
# the .ncu-rep files stay on the box (gpurun_out/ is capped at 64 MiB): summarise them here
python tools/ncu_summarise.py /tmp/prof gpurun_out/profiles
# per-source-line stall samples of the GEMM kernel (top lines)
for f in r2_mmq_tc r2_mmq_tc_q6k r2_fattn_tc_f16; do ncu -i /tmp/prof/$f.ncu-rep --page source --csv -k regex:'mmq_tc|fattn_tc' 2>/dev/null | python tools/ncu_source_top.py > gpurun_out/profiles/${f}_source_top.txt; done
ncu -i /tmp/prof/r2_fattn_f16_768.ncu-rep --page source --csv 2>/dev/null | python tools/ncu_source_top.py > gpurun_out/profiles/r2_fattn_f16_768_source_top.txt
