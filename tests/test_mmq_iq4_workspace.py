"""CPU: prefill on IQ4_NL / IQ4_XS weights goes to the int8 tensor-core kernel (csrc/mmq_tc32.cu).  b200_mul_mat_q_workspace asks for that
kernel's activation image where it takes the call and for nothing otherwise (the wide matvec it falls back to quantises the columns
itself), MUL_MAT_ID stays on the matvec, and the executor's dry run plans one b200_mul_mat_q2 call per batched IQ4_NL / IQ4_XS MUL_MAT when
the wide path is switched on."""
import pytest

from refutil import IQ4_NL, IQ4_XS
from test_mmq_q2q3_workspace import COLS, dry_run

MIN_COLS = 16            # IQ4_MIN_COLS of mmq.cu


def image32(k, n):
    """the block-32 image: per 128-token tile and 128-k stage, 16 KB of int8 and 4 x 128 f32 block scales"""
    return (n + 127) // 128 * (k // 128) * (8 * 2048 + 4 * 512)


@pytest.mark.parametrize("t", [IQ4_NL, IQ4_XS])
def test_workspace_is_the_int8_image_or_nothing(b200, t):
    L = b200.lib
    for k in [256, 2048, 4096, 14336, 28672]:
        for n in COLS:
            assert L.b200_mul_mat_q_workspace(t, 4096, k, n) == (image32(k, n) if n >= MIN_COLS else 0), (k, n)
    for k, n in [(100, 512), (4096 + 32, 512), (2048 + 128, 512), (0, 512), (4096, 0)]:
        assert L.b200_mul_mat_q_workspace(t, 4096, k, n) == 0, (k, n)


@pytest.mark.parametrize("t", [IQ4_NL, IQ4_XS])
def test_no_act_kind_and_no_grouped_workspace(b200, t):
    """no act-buffer matvec for these formats, and MUL_MAT_ID stays on the wide matvec"""
    assert b200.lib.b200_act_kind_for(t) < 0
    for n_tok in (16, 512, 4096):
        assert b200.lib.b200_mul_mat_id_workspace(t, 4096, 4096, 8, 2, n_tok) == 0


def test_executor_plans_the_tile_kernel_for_512_columns():
    o, calls = dry_run([(IQ4_NL, 4096, 4096, 512), (IQ4_XS, 14336, 4096, 512), (IQ4_XS, 4096, 14336, 512)])
    assert all(o["supports"]) and o["plan"] == 3, (o, calls)
    assert len(calls) == 3 and all(c.startswith("b200_mul_mat_q2(") for c in calls), calls


def test_executor_keeps_the_matvec_below_the_minimum():
    """decode, 2-8-token verify batches, and IQ4_NL rows that are not a multiple of 256: the wide matvec as before"""
    o, calls = dry_run([(IQ4_NL, 4096, 4096, 1), (IQ4_XS, 4096, 4096, 8), (IQ4_NL, 1024, 4096, 1), (IQ4_XS, 1024, 4096, 8),
                        (IQ4_NL, 4096, 4096 + 32, 512)])
    assert all(o["supports"]) and o["plan"] == 5, (o, calls)
    assert all(c.startswith("b200_mul_mat_vec_wide(") for c in calls), calls
