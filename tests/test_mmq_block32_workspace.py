"""CPU: b200_mul_mat_q_workspace for the 32-element block formats covers both users of the buffer — the q8_0 act columns of the
column-group path and the tensor-core kernel's activation image (csrc/mmq_tc32.cu: per 128-token tile and 128-k stage, 16 KB of
int8 plus 2 KB of f32 block scales) — and is what it was for the K-quants."""
import pytest

from refutil import Q4_0, Q4_K, Q5_0, Q5_K, Q6_K, Q8_0

COLS = [1, 8, 9, 31, 32, 33, 127, 128, 129, 300, 512, 2048]


def image32(k, n):
    return (n + 127) // 128 * (k // 128) * (8 * 2048 + 4 * 512)


def image_k(k, n):
    nt = (n + 127) // 128
    return nt * (k // 64) * 16384 + nt * (k // 256) * (4096 + 512)


@pytest.mark.parametrize("t", [Q4_0, Q5_0, Q8_0])
def test_workspace_covers_act_columns_and_image(b200, t):
    L = b200.lib
    for k in [256, 2048, 4096, 14336, L.b200_padded_k(t, 29568), L.b200_padded_k(t, 96)]:
        assert k % 256 == 0
        for n in COLS:
            ws = L.b200_mul_mat_q_workspace(t, 4096, k, n)
            vec = n * L.b200_act_col_bytes(1, k)
            assert ws >= vec
            assert ws in (vec, max(vec, image32(k, n)))          # the image only where the tensor-core path takes the shape
            if n >= 128:
                assert ws >= image32(k, n)
    assert L.b200_mul_mat_q_workspace(t, 4096, 100, 16) == 0 and L.b200_mul_mat_q_workspace(t, 4096, 256, 0) == 0


@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K])
def test_workspace_of_the_k_quants_is_unchanged(b200, t):
    L = b200.lib
    for k in [256, 2048, 4096, 14336]:
        for n in COLS:
            vec = n * L.b200_act_col_bytes(0, k)
            tc = n >= 9 and (t != Q6_K or k % 2048 == 0)
            assert L.b200_mul_mat_q_workspace(t, 4096, k, n) == (max(vec, image_k(k, n)) if tc else vec)
