"""CPU: b200_mul_mat_id_workspace — the grouped MUL_MAT_ID's schedule (column-tile count, per-expert counts, tile -> expert table, column map)
and the tile kernel's activation image sized for the upper bound of column tiles, floor(N / 128) + min(n_expert, N) with N = n_tok * n_used;
0 (the matvec) below MMID_MIN_TOK tokens or MMID_MIN_PAIRS pairs per expert, for the wide-only formats and for rows the tile kernels do not
take; and a dry run of a prefill-sized Mixtral-style block through the executor."""
import pytest

from refutil import Q4_0, Q4_K, Q5_0, Q5_K, Q6_K, Q8_0

MIN_TOK = 16            # MMID_MIN_TOK of csrc/mmid_route.cu
MIN_PAIRS = 4           # MMID_MIN_PAIRS: (token, slot) pairs per expert on average
WIDE_ONLY = [3, 7, 10, 11, 20, 23, 39]


def up256(x):
    return (x + 255) // 256 * 256


def image(t, k, n):
    nt = (n + 127) // 128
    if t in (Q4_0, Q5_0, Q8_0):
        return nt * (k // 128) * (8 * 2048 + 4 * 512)
    return nt * (k // 64) * 16384 + nt * (k // 256) * (4096 + 512)


def expected(t, k, ne, nu, n_tok):
    n = n_tok * nu
    if n_tok < MIN_TOK or n < MIN_PAIRS * ne:
        return 0
    ub = n // 128 + min(ne, n)
    route = up256(up256(up256(16 + 4 * ne) + 4 * ub) + 4 * 128 * ub)
    return route + image(t, k, 128 * ub)


@pytest.mark.parametrize("t", [Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K])
def test_workspace_covers_the_bound(b200, t):
    L = b200.lib
    for k in (2048, 4096, 14336):
        for ne, nu in ((8, 2), (6, 3), (128, 8), (64, 6)):
            for n_tok in (MIN_TOK, 17, 42, 43, 63, 64, 129, 512, 4096):
                assert L.b200_mul_mat_id_workspace(t, 4096, k, ne, nu, n_tok) == expected(t, k, ne, nu, n_tok), (k, ne, nu, n_tok)
    assert L.b200_mul_mat_id_workspace(t, 4096, 4096, 8, 2, MIN_TOK) > 0                 # Mixtral: from the minimum on
    assert L.b200_mul_mat_id_workspace(t, 4096, 2048, 128, 8, 63) == 0                   # 128 experts, top-8: from 64 tokens
    assert L.b200_mul_mat_id_workspace(t, 4096, 2048, 128, 8, 64) > 0


@pytest.mark.parametrize("t", [Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K])
def test_no_workspace_below_the_minimum(b200, t):
    """decode and the 2-8-token verify batches keep the matvec and its bits"""
    L = b200.lib
    for n_tok in range(1, MIN_TOK):
        assert L.b200_mul_mat_id_workspace(t, 4096, 4096, 8, 2, n_tok) == 0
    assert MIN_TOK >= 9


def test_no_workspace_where_the_tile_kernels_do_not_go(b200):
    L = b200.lib
    for t in WIDE_ONLY:
        assert L.b200_mul_mat_id_workspace(t, 4096, 4096, 8, 2, 512) == 0, t
    assert L.b200_mul_mat_id_workspace(Q6_K, 4096, 1536, 8, 2, 512) == 0        # Q6_K rows: k % 2048
    assert L.b200_mul_mat_id_workspace(Q4_K, 4096, 4000, 8, 2, 512) == 0
    assert L.b200_mul_mat_id_workspace(Q4_K, 0, 4096, 8, 2, 512) == 0
    assert L.b200_mul_mat_id_workspace(Q4_K, 4096, 4096, 0, 2, 512) == 0


def test_executor_dry_run_of_a_prefill_block():
    """the Mixtral-style block of tests/moe_graph.py at 512 tokens, GGML_B200_WIDE=1: every node is taken and the plan is the same 15 C-ABI
    calls as for decode (each MUL_MAT_ID is one call, whichever kernels it launches)"""
    from test_wide_plan import run_child
    for wtype in (3, 23):
        o = run_child(True, 512, wtype)
        assert o["wide"] == 1 and all(o["supports"]) and o["plan"] == 15, o
