"""What ptxas made of the tensor-core mainloops (no GPU needed): the compiled library's SASS and the build's ptxas report.

The convolution and the screened-correlation kernels hand every ring stage back with an mbarrier arrive right after
the wgmma.wait_group that retires the stage's reads.  A cluster-scope release on that arrive is lowered to a
MEMBAR.ALL.GPU per call, a full memory fence on every k-block between one group of HGMMAs and the next.  These tests
keep such a fence out of that path, and keep ptxas from serializing the wgmma pipeline or spilling in the kernels the
480p benchmark runs.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200", "csrc")
BUILD = os.path.join(CSRC, "build")
KERNELS = ("conv_tc_kernel", "corr_screen_kernel")


def _cuda_tool(name):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cand = os.path.join(os.path.dirname(nvcc), name)
    path = cand if os.path.exists(cand) else shutil.which(name)
    assert path, f"{name} not found (CUDA toolkit next to {nvcc} or on PATH)"
    return path


@pytest.fixture(scope="module")
def built():
    subprocess.run(["make", "-C", CSRC, "-j8"], check=True, capture_output=True)


def _sass_functions(obj):
    """{mangled name: [(address, instruction)]} of every kernel in a relocatable object."""
    out = subprocess.run([_cuda_tool("cuobjdump"), "-sass", obj], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", out)[1:]:
        name, body = chunk.split("\n", 1)
        ins = []
        for line in body.split("\n"):
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
            if m:
                ins.append((int(m.group(1), 16), m.group(2)))
        funcs[name.strip()] = ins
    return funcs


def _fences_before_release(ins):
    """GPU-scope fences between the last HGMMA of a group (gsb0) and the stage-release arrive that follows it."""
    bad = []
    for i, (_, op) in enumerate(ins):
        if not (op.startswith("HGMMA") and "gsb0" in op):
            continue
        for addr, op2 in ins[i + 1:]:
            if "SYNCS.ARRIVE" in op2 or op2.startswith("HGMMA"):
                break
            if re.search(r"MEMBAR\.\w+\.GPU", op2):
                bad.append(hex(addr))
    return bad


@pytest.mark.parametrize("src,kernel", [("conv_tc", "conv_tc_kernel"), ("corr_tc", "corr_screen_kernel")])
def test_no_gpu_fence_in_wgmma_mainloop(built, src, kernel):
    funcs = {n: i for n, i in _sass_functions(os.path.join(BUILD, src + ".o")).items() if kernel in n}
    assert funcs, f"no {kernel} instantiation in {src}.o"
    for name, ins in funcs.items():
        assert any(op.startswith("HGMMA") for _, op in ins), name
        bad = _fences_before_release(ins)
        assert not bad, f"{name}: MEMBAR.*.GPU between HGMMA and the stage release at {bad}"


def _ptxas_report(src):
    """{mangled name: (spill store bytes, [serialization reasons])} from the build's ptxas -v log."""
    log = open(os.path.join(BUILD, src + ".ptxas.log")).read()
    serial = re.findall(r"serialized due to (.*?) in the function '(\S+)'", log)
    rep, cur = {}, None
    for line in log.split("\n"):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur:
            rep[cur] = (int(m.group(1)), [r for r, f in serial if f == cur])
    return rep


@pytest.mark.parametrize("src", ["conv_tc", "corr_tc"])
def test_no_wgmma_serialization_or_spills(built, src):
    rep = {n: v for n, v in _ptxas_report(src).items() if any(k in n for k in KERNELS)}
    assert rep, f"no tensor-core kernel in the ptxas report of {src}"
    for name, (spill, serial) in rep.items():
        assert not serial, f"{name}: wgmma serialized ({serial})"
        # the benchmark runs the plain convolution tiles, not the row-shared ones (last template argument RS)
        if "conv_tc_kernel" in name:
            rs = re.search(r"conv_tc_kernelI(?:Li\d+E){3}Lb[01]ELb([01])E", name)
            assert rs, name
            if rs.group(1) == "1":
                continue
        assert spill == 0, f"{name}: {spill} bytes of spill stores"
