"""CPU: the stage load and unpack the int8 tile kernel (csrc/mmq_tc32.cu) runs on IQ4_NL / IQ4_XS weights in ggml's native block layout, and
the q8_K arithmetic of its IQ4_XS activation image — csrc/mmq_wide32.cuh compiled with g++ (tests/hostsim/iq4sim.cpp) — against the C
oracle, which tests/test_oracle_vs_ref.py pins to the unmodified reference.  The IQ4_NL load is also run under AddressSanitizer on rows
held in allocations of exactly their size: no stage reads a byte past its row."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from refutil import IQ4_NL, IQ4_XS, ROOT, have_ref, orc_dequant, orc_quantize_act, ptr, rand_blocks, ref_quantize_weights, row_bytes

SRC = os.path.join(ROOT, "tests", "hostsim", "iq4sim.cpp")
KV = np.array([-127, -104, -83, -65, -49, -35, -22, -10, 1, 13, 25, 38, 53, 69, 89, 113], np.int32)


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("iq4sim") / "libiq4sim.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-DXF_CHECK_ALIGN", "-x", "c++", SRC, "-o", so])
    L = C.CDLL(so)
    L.sim_iq4_unpack_row.restype = C.c_long
    L.sim_iq4_unpack_row.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    L.sim_q8k_column.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    return L


def numpy_ints(t, row, k):
    """the block integers and scales straight from the layout: kvalues_iq4nl[nibble], d, and (IQ4_XS) ls - 32 per sub-block"""
    if t == IQ4_NL:
        b = row.reshape(k // 32, 18)
        d = b[:, 0:2].copy().view(np.uint16).reshape(-1)
        qs = b[:, 2:]
        ls = None
    else:
        b = row.reshape(k // 256, 136)
        d = np.repeat(b[:, 0:2].copy().view(np.uint16).reshape(-1), 8)
        sh = b[:, 2:4].copy().view(np.uint16).reshape(-1).astype(np.int32)
        ib = np.arange(8)
        ls = ((b[:, 4 + ib // 2].astype(np.int32) >> (4 * (ib % 2))) & 15) | (((sh[:, None] >> (2 * ib)) & 3) << 4)
        ls = ls.reshape(-1) - 32
        qs = b[:, 8:].reshape(k // 32, 16)
    q = np.concatenate([KV[qs & 15], KV[qs >> 4]], axis=1).reshape(-1)
    return q, d, ls


def weights(t, k, kind, rng, m=6):
    if kind == "random":
        return rand_blocks(rng, t, m, k)
    return ref_quantize_weights(t, (rng.standard_normal((m, k)) * 0.02).astype(np.float32))


@pytest.mark.parametrize("t", [IQ4_NL, IQ4_XS])
@pytest.mark.parametrize("k", [256, 512, 4096])
@pytest.mark.parametrize("kind", ["random", "reference"])
def test_stage_unpack_matches_the_oracle(sim, t, k, kind):
    if kind == "reference" and not have_ref():
        pytest.skip("oracle/_ref (reference quantiser) not present")
    rng = np.random.default_rng(100 * t + k + (kind == "reference"))
    W = weights(t, k, kind, rng)
    deq = orc_dequant(t, W, W.shape[0], k)
    f16 = lambda h: h.view(np.float16).astype(np.float32)        # noqa: E731
    for i in range(W.shape[0]):
        row = np.ascontiguousarray(W[i])
        q = np.zeros(k, np.int8); sc = np.zeros(k // 32, np.uint32)
        assert sim.sim_iq4_unpack_row(t, ptr(row), k, ptr(q), ptr(sc)) == 0            # every load aligned
        wq, wd, wls = numpy_ints(t, row, k)
        assert np.array_equal(q.astype(np.int32), wq), (t, k, i)
        assert np.array_equal((sc & 0xffff).astype(np.uint16), wd), (t, k, i)
        dw = f16((sc & 0xffff).astype(np.uint16))
        if t == IQ4_NL:
            rec = np.repeat(dw, 32) * q.astype(np.float32)                                  # d * kvalues[nibble], as the oracle de-quantises
        else:
            ls = (sc >> 16).astype(np.uint16).view(np.int16).astype(np.int32)
            assert np.array_equal(ls, wls), (t, k, i)
            rec = np.repeat((dw * ls.astype(np.float32)).astype(np.float32), 32) * q.astype(np.float32)
        assert np.array_equal(rec.astype(np.float32), deq[i]), (t, k, i)


def test_q8k_arithmetic_of_the_iq4_xs_image_is_the_oracles(sim):
    """the q8_K quantiser of the IQ4_XS activation image: its 8-element arithmetic after the warp's first-largest-|x| reduction gives the
    oracle's bytes (ties for the largest |x|, a zero super-block, values on rounding ties and across 12 decades)"""
    rng = np.random.default_rng(7)
    k = 256 * 64
    x = (rng.standard_normal(k) * 10.0 ** rng.uniform(-6, 6, k // 256).repeat(256)).astype(np.float32)
    x[:256] = 0.0
    x[256:512] = 1.0; x[300] = -1.0                                   # every |x| ties; the first (positive) one is the max
    x[512:768] = np.arange(256, dtype=np.float32) - 127.0           # iscale * x on integers and halves
    x[768:1024] = rng.integers(-254, 255, 256).astype(np.float32) / 2.0
    x[1024] = -8.0; x[1025:1280] = np.clip(x[1025:1280], -8.0, 8.0); x[1100] = 8.0   # a negative first maximum
    want = orc_quantize_act(IQ4_XS, x[None, :])[0].reshape(k // 256, 292)
    q = np.zeros(k, np.int8); d = np.zeros(k // 256, np.float32)
    sim.sim_q8k_column(ptr(x), k, ptr(q), ptr(d))
    assert np.array_equal(d.view(np.uint32), want[:, 0:4].copy().view(np.uint32).reshape(-1))
    assert np.array_equal(q.reshape(k // 256, 256), want[:, 4:260].view(np.int8))


@pytest.mark.skipif(shutil.which("g++") is None, reason="no g++")
@pytest.mark.parametrize("k", [256, 512, 4096])
def test_iq4_nl_stage_loads_stay_inside_the_row(tmp_path, k):
    """AddressSanitizer: every stage of IQ4_NL rows (the format whose stages are not whole blocks) and IQ4_XS rows, each row in a heap
    allocation of exactly its size, is loaded and unpacked without a read past the allocation"""
    exe = str(tmp_path / "iq4sim")
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address", "-fno-omit-frame-pointer", "-ffp-contract=off", "-DXF_CHECK_ALIGN",
                        "-DIQ4SIM_MAIN", "-x", "c++", SRC, "-o", exe], capture_output=True, text=True)
    if r.returncode != 0 and "asan" in r.stderr.lower():
        pytest.skip("AddressSanitizer runtime not available: " + r.stderr[-300:])
    assert r.returncode == 0, r.stderr[-2000:]
    for t in (IQ4_NL, IQ4_XS):
        assert row_bytes(t, k) % 8 == 0
        o = subprocess.run([exe, str(t), str(k), "64", str(k + t)], capture_output=True, text=True,
                           env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0"))
        assert o.returncode == 0 and o.stdout.startswith("ok") and "misaligned 0" in o.stdout, (o.stdout, o.stderr[-3000:])
