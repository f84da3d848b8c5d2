"""ctypes mirror of include/b200_graph.h + a small builder for ggml-style node lists.

Host-side mirror of the reference's graph IR for this path (ggml/include/ggml.h:613-645): ne[] in
elements, nb[] in bytes, ops in the order llm_build_llama emits them
(/root/reference/llama.cpp/src/llama-model.cpp:5968-6122).
"""
import ctypes as C

from . import ops

F32, F16, Q4_0, Q5_0, Q8_0, Q4_K, Q5_K, Q6_K, I32, I64 = 0, 1, 2, 6, 8, 12, 13, 14, 26, 27
Q4_1, Q5_1, Q2_K, Q3_K, IQ4_NL, IQ4_XS, MXFP4 = 3, 7, 10, 11, 20, 23, 39      # the wide path's formats (b200_ops.h)
OP_NONE, OP_MUL_MAT, OP_RMS_NORM, OP_MUL, OP_ADD, OP_ROPE, OP_SET_ROWS, OP_FLASH_ATTN_EXT, OP_GLU_SWIGLU, OP_GET_ROWS, OP_CPY, OP_MUL_MAT_ID, OP_SOFT_MAX, OP_ARGSORT, OP_SUM_ROWS, OP_DIV, OP_CONT, OP_SCALE, OP_UNARY = range(19)
EXEC_CUDA_GRAPHS, EXEC_FUSION, EXEC_MEGAKERNEL, EXEC_MEGA_MMV = 1, 2, 4, 8
FLAG_OUTPUT = 2                     # B200_TENSOR_FLAG_OUTPUT (== GGML_TENSOR_FLAG_OUTPUT): the caller reads this tensor
MAX_SRC = 6
ELEM_SIZE = {F32: 4, F16: 2, I32: 4, I64: 8}


class Tensor(C.Structure):
    _fields_ = [("id", C.c_uint64), ("data", C.c_void_p), ("type", C.c_int32), ("flags", C.c_int32), ("ne", C.c_int64 * 4), ("nb", C.c_int64 * 4)]


class Node(C.Structure):
    _fields_ = [("op", C.c_int32), ("n_src", C.c_int32), ("dst", Tensor), ("src", Tensor * MAX_SRC), ("op_params", C.c_int32 * 16)]


_lib = ops.lib
_lib.b200_executor_create.restype = C.c_void_p; _lib.b200_executor_create.argtypes = [C.c_int]
_lib.b200_executor_free.restype = None; _lib.b200_executor_free.argtypes = [C.c_void_p]
_lib.b200_executor_supports.restype = C.c_int; _lib.b200_executor_supports.argtypes = [C.POINTER(Node)]
_lib.b200_executor_plan.restype = C.c_int64; _lib.b200_executor_plan.argtypes = [C.POINTER(Node), C.c_int, C.c_int]
_lib.b200_executor_compute.restype = C.c_int; _lib.b200_executor_compute.argtypes = [C.c_void_p, C.POINTER(Node), C.c_int, C.c_void_p, C.c_int]
for _n in ("b200_executor_last_kernels", "b200_executor_graph_captures", "b200_executor_graph_replays", "b200_executor_mk_launches", "b200_executor_mk_phases"):
    getattr(_lib, _n).restype = C.c_int64; getattr(_lib, _n).argtypes = [C.c_void_p]
_lib.b200_executor_wide_enabled.restype = C.c_int; _lib.b200_executor_wide_enabled.argtypes = []
GRAPH_SYMBOLS = ["b200_executor_wide_enabled", "b200_executor_plan", "b200_executor_create", "b200_executor_free", "b200_executor_supports", "b200_executor_compute",
                 "b200_executor_last_kernels", "b200_executor_graph_captures", "b200_executor_graph_replays", "b200_executor_mk_launches", "b200_executor_mk_phases"]

_next_id = [1]


def row_size(t, ne0):
    if t in ELEM_SIZE:
        return ELEM_SIZE[t] * ne0
    rb = ops.row_bytes(t, ne0)
    return rb if rb > 0 else ops.lib.b200_wide_row_bytes(t, ne0)


class T:
    """a tensor handle: device pointer + ggml-style shape/strides (contiguous unless nb given)"""

    def __init__(self, ptr, type_, ne, nb=None, tid=None):
        ne = list(ne) + [1] * (4 - len(ne))
        if nb is None:
            nb = [ELEM_SIZE.get(type_, ops.lib.b200_block_bytes(type_) or 1), row_size(type_, ne[0]), 0, 0]
            nb[2] = nb[1] * ne[1]; nb[3] = nb[2] * ne[2]
        self.ptr, self.type, self.ne, self.nb = int(ptr), type_, ne, list(nb)
        self.flags = 0
        if tid is None:
            tid = _next_id[0]; _next_id[0] += 1
        self.id = tid

    def view(self, ne, nb, offset=0):
        """a view sharing storage (new identity, like ggml_view_*/ggml_reshape/ggml_permute results)"""
        return T(self.ptr + offset, self.type, ne, nb)

    def reshape(self, ne):
        return T(self.ptr, self.type, ne)

    def fill(self, ct):
        ct.id, ct.data, ct.type, ct.flags = self.id, self.ptr, self.type, self.flags
        for i in range(4):
            ct.ne[i] = self.ne[i]; ct.nb[i] = self.nb[i]


def f32_bits(x):
    return C.c_int32.from_buffer_copy(C.c_float(x)).value


class NodeList:
    def __init__(self):
        self.items = []

    def add(self, op, dst, srcs, params=None):
        self.items.append((op, dst, list(srcs), list(params or [])))
        return dst

    def view_op(self, dst, src):
        """RESHAPE / VIEW / PERMUTE: recorded like ggml records them (op NONE, one src)"""
        return self.add(OP_NONE, dst, [src])

    def build(self):
        arr = (Node * len(self.items))()
        for n, (op, dst, srcs, params) in zip(arr, self.items):
            n.op, n.n_src = op, len(srcs)
            dst.fill(n.dst)
            for i, s in enumerate(srcs):
                if s is not None:
                    s.fill(n.src[i])
            for i, p in enumerate(params):
                n.op_params[i] = p
        return arr


def plan(nodes, flags=EXEC_CUDA_GRAPHS | EXEC_FUSION):
    """launches the executor would issue for this node list (dry run, no device)"""
    return int(_lib.b200_executor_plan(nodes, len(nodes), flags))


class Executor:
    def __init__(self, device=0):
        self.h = _lib.b200_executor_create(device)
        if not self.h:
            raise ops.B200Error(_lib.b200_last_error().decode())

    def compute(self, nodes, flags=EXEC_CUDA_GRAPHS | EXEC_FUSION, stream=None):
        ops.check(_lib.b200_executor_compute(self.h, nodes, len(nodes), stream if stream is not None else ops.stream(), flags))

    def supports(self, node):
        return bool(_lib.b200_executor_supports(C.byref(node)))

    @property
    def last_kernels(self):
        return _lib.b200_executor_last_kernels(self.h)

    @property
    def captures(self):
        return _lib.b200_executor_graph_captures(self.h)

    @property
    def replays(self):
        return _lib.b200_executor_graph_replays(self.h)

    @property
    def mk_launches(self):
        return _lib.b200_executor_mk_launches(self.h)

    @property
    def mk_phases(self):
        return _lib.b200_executor_mk_phases(self.h)

    def close(self):
        if self.h:
            _lib.b200_executor_free(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
