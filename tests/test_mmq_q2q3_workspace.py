"""CPU: prefill on Q2_K / Q3_K weights goes to the K-quant tensor-core kernel (csrc/mmq_tc.cu).  b200_mul_mat_q_workspace asks for that
kernel's activation image where it takes the call and for nothing otherwise (the wide matvec it falls back to quantises the columns
itself), and the executor's dry run plans one b200_mul_mat_q2 call per batched Q2_K / Q3_K MUL_MAT when the wide path is switched on."""
import json
import os
import subprocess
import sys

import pytest

from refutil import Q2_K, Q3_K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLS = [1, 8, 9, 31, 32, 33, 127, 128, 129, 300, 512, 2048]
MIN_COLS = 9            # TC_MIN_COLS of mmq.cu


def image_k(k, n):
    nt = (n + 127) // 128
    return nt * (k // 64) * 16384 + nt * (k // 256) * 4608


@pytest.mark.parametrize("t", [Q2_K, Q3_K])
def test_workspace_is_the_k_quant_image_or_nothing(b200, t):
    L = b200.lib
    for k in [256, 2048, 4096, 8192, 14336, 28672]:
        for n in COLS:
            assert L.b200_mul_mat_q_workspace(t, 4096, k, n) == (image_k(k, n) if n >= MIN_COLS else 0), (k, n)
    for k, n in [(100, 512), (4096 + 32, 512), (0, 512), (4096, 0)]:
        assert L.b200_mul_mat_q_workspace(t, 4096, k, n) == 0, (k, n)


def test_no_act_kind_for_the_wide_k_quants(b200):
    """the two formats have no act-buffer matvec: b200_act_kind_for stays unsupported for them"""
    assert b200.lib.b200_act_kind_for(Q2_K) < 0 and b200.lib.b200_act_kind_for(Q3_K) < 0


CHILD = r"""
import importlib, json, sys
sys.path.insert(0, %r)
from conftest import load_pkg
load_pkg()
G = importlib.import_module("llama_box_b200.graph")
base = [0x10000000]
def buf(n):
    p = base[0]; base[0] += (n + 0xfffff) & ~0xfffff; return p
nl = G.NodeList()
for t, m, k, n in %r:
    x = G.T(buf(4 * k * n), G.F32, [k, n])
    w = G.T(buf(G.row_size(t, k) * m), t, [k, m])
    nl.add(G.OP_MUL_MAT, G.T(buf(4 * m * n), G.F32, [m, n]), [w, x])
nodes = nl.build()
print(json.dumps({"supports": [int(G._lib.b200_executor_supports(nodes[i])) for i in range(len(nodes))], "plan": G.plan(nodes, G.EXEC_FUSION)}))
"""


def dry_run(cases):
    env = dict(os.environ, GGML_B200_WIDE="1", B200_PLAN_DEBUG="1")
    r = subprocess.run([sys.executable, "-c", CHILD % (os.path.join(ROOT, "tests"), cases)], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, r.stderr[-2000:]
    calls = [ln.split(":", 1)[1].strip() for ln in r.stderr.splitlines() if ln.startswith("plan ")]
    return json.loads(r.stdout.strip().splitlines()[-1]), calls


def test_executor_plans_the_tile_kernel_for_512_columns():
    o, calls = dry_run([(Q3_K, 4096, 4096, 512), (Q2_K, 14336, 4096, 512)])
    assert all(o["supports"]) and o["plan"] == 2, (o, calls)
    assert len(calls) == 2 and all(c.startswith("b200_mul_mat_q2(") for c in calls), calls


def test_executor_keeps_the_matvec_below_the_minimum():
    """decode, 2-8-token verify batches: the wide matvec as before"""
    o, calls = dry_run([(Q3_K, 4096, 4096, 1), (Q2_K, 4096, 4096, 8), (Q3_K, 1024, 4096, 9)])
    assert all(o["supports"]) and o["plan"] == 3, (o, calls)
    assert calls[0].startswith("b200_mul_mat_vec_wide(") and calls[1].startswith("b200_mul_mat_vec_wide("), calls
    assert calls[2].startswith("b200_mul_mat_q2("), calls
