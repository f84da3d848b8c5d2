"""llama-box_b200 — H100-native (sm_90a) kernels for the GGUF-quantised decode/prefill hot path
of gpustack/llama-box, behind a C-ABI (include/b200_ops.h) and a ggml backend plug-in
(include/ggml_b200.h).  This Python package is the host-side binding used by tests/ and bench.py;
the product is the two shared libraries.  There is no CPU fallback: importing `ops` without the
built CUDA library raises.
"""
from . import ops  # noqa: F401
