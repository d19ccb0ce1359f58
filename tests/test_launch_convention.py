"""Every kernel launcher reports one result: the kernels it enqueued (>= 0), or the CUDA error it met, negated
(lwse_launch.cuh).  A kernel file turns a launch into that result only through ``launch_result``; a launcher that
calls another passes the callee's result through; the engine counts it in ``count_launch``.  Source checks; the
counts themselves are pinned on the GPU by test_gpu_launch_counts.py and test_gpu_drain_launches.py."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lws_b200", "csrc")
SOURCES = {os.path.relpath(p, CSRC): open(p).read()
           for p in sorted(glob.glob(os.path.join(CSRC, "**", "*"), recursive=True))
           if p.endswith((".cu", ".cuh", ".hpp"))}


def _code(text):
    return re.sub(r"//[^\n]*", "", text)


def _launchers():
    """{name: body} of every launcher a kernel file defines: the functions at column 0 named launch_*."""
    out = {}
    for name, src in SOURCES.items():
        if not name.endswith("_kernels.cu"):
            continue
        for m in re.finditer(r"^(?:static )?int (launch_\w+)\(", src, re.M):
            body = src[src.index("{", m.end()): src.index("\n}\n", m.end())]
            out[f"{name}:{m.group(1)}"] = _code(body)
    return out


def test_no_error_out_parameter():
    for name, src in SOURCES.items():
        assert not re.search(r"\bcuda_err\b", src), name


def test_launchers_pass_errors_through():
    launchers = _launchers()
    assert len(launchers) >= 50
    for name, body in launchers.items():
        assert "return -1;" not in body, name


def test_one_result_helper_and_one_grid_for():
    code = {name: _code(src) for name, src in SOURCES.items()}
    assert not any("launched_or_fail" in src for src in code.values())
    grid_for = [name for name, src in code.items() for _ in re.finditer(r"\bunsigned grid_for\(", src)]
    assert grid_for == ["lwse_device.cuh"]


def test_last_error_read_only_in_launch_result():
    """cudaGetLastError's value is read in launch_result alone; every other call only clears the error state."""
    reads = [(name, line.strip()) for name, src in SOURCES.items() for line in _code(src).splitlines()
             if "cudaGetLastError" in line and line.strip() != "(void)cudaGetLastError();"]
    assert reads == [("lwse_launch.cuh", "const cudaError_t e = cudaGetLastError();")]
    launch = SOURCES["lwse_launch.cuh"]
    helper = launch[launch.index("inline int launch_result("):]
    assert "cudaGetLastError" in helper[: helper.index("\n}\n")]
