"""Every CUDA object of an engine has an owner that frees it: buffers, pinned words, streams, events, graph
executables and peer mappings are acquired and released only inside the owner types at the top of lwse_engine.cu,
and lwse_destroy frees nothing by name (the member destructors do).  Source checks; the GPU side is
test_gpu_engine_lifetime.py."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "lws_b200", "csrc", "lwse_engine.cu")).read()
OWNERS, REST = SRC.split("\nstruct lwse_engine {", 1)


def _body(src, signature):
    """The text of the function that starts at ``signature``, up to its closing brace at column 0."""
    i = src.index(signature)
    return src[i: src.index("\n}\n", i)]


def _code(text):
    return re.sub(r"//[^\n]*", "", text)


def test_no_raw_handle_members():
    engine = _code(REST[: REST.index("\n};\n")])
    for t in ("cudaStream_t", "cudaEvent_t", "cudaGraphExec_t"):
        assert not re.search(rf"\b{t}\b", engine), t


def test_acquire_and_release_only_in_the_owners():
    rest = _code(REST)
    for call in ("cudaMalloc(", "cudaHostAlloc", "cudaMallocHost", "cudaFree", "cudaStreamCreate", "cudaEventCreate",
                 "cudaStreamDestroy", "cudaEventDestroy", "cudaGraphExecDestroy", "cudaIpcCloseMemHandle"):
        assert call not in rest, call
    # (and the owners do acquire and release them)
    for call in ("cudaMalloc(", "cudaHostAlloc", "cudaFree(", "cudaFreeHost", "cudaStreamCreate", "cudaEventCreate",
                 "cudaStreamDestroy", "cudaEventDestroy", "cudaGraphExecDestroy", "cudaIpcCloseMemHandle"):
        assert call in OWNERS, call


def test_destroy_frees_nothing_by_name():
    assert "release(" not in _body(SRC, "LWSE_API void lwse_destroy(")
