"""The wgmma kernels of the layer GEMM and the Res2Net chain must compile to asynchronous MMAs.

ptxas serialises every wgmma of a kernel -- each MMA then waits for the previous one to retire -- when the MMA issue
sits on a path it cannot prove uniform (C7520, e.g. a K-step loop with a runtime trip count), or when the kernel
contains a function call anywhere (C7510, e.g. a printf), and says so only as an informational line.  This test
compiles both sources exactly as the Makefile's ptxas-info target does (flags and all, into a temporary directory),
fails on any such line that names one of the kernels, and checks in the SASS that every layer-kernel instance issues
several HGMMA per WARPGROUP.DEPBAR, as it does when a stage's MMAs run back to back.  Needs nvcc, not a GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "asv_subtools_b200", "csrc")
SOURCES = {"tdnn_gemm.cu": "tdnn_gemm_bf16x3_kernel", "res2net.cu": "res2net_chain_kernel"}
SERIALISED = re.compile(r"\((C7510|C7519|C7520)\)")
# every instantiation of the layer kernel: BLOCK_N 32 / 64 / 128, fused pooling, trial histogram, swish
LAYER_INSTANCES = 8


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


NVCC = _nvcc()
pytestmark = pytest.mark.skipif(NVCC is None or shutil.which("make") is None, reason="needs nvcc and make")


def _ptxas_commands():
    """The nvcc command lines of `make ptxas-info` for SOURCES, as make expands them."""
    out = subprocess.run(["make", "-s", "-n", "-C", CSRC, "NVCC=" + NVCC, "ptxas-info"], check=True,
                         capture_output=True, text=True).stdout
    cmds = {}
    for line in out.splitlines():
        for src in SOURCES:
            if re.search(r"-c\s+" + re.escape(src) + r"\s", line + " "):
                cmds[src] = line
    assert set(cmds) == set(SOURCES), "make ptxas-info no longer compiles " + ", ".join(set(SOURCES) - set(cmds))
    return cmds


@pytest.fixture(scope="module")
def compiled():
    """{source: (ptxas log, SASS text)}, both sources compiled concurrently."""
    tmp = tempfile.mkdtemp(prefix="xvb_wgmma_")
    try:
        procs = {}
        for src, cmd in _ptxas_commands().items():
            obj = os.path.join(tmp, src + ".o")
            assert "/dev/null" in cmd
            procs[src] = (obj, subprocess.Popen(cmd.replace("/dev/null", obj), shell=True, cwd=CSRC, text=True,
                                                stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
        res = {}
        for src, (obj, p) in procs.items():
            log = p.communicate()[0]
            assert p.returncode == 0, log[-4000:]
            cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
            sass = subprocess.run([cuobjdump, "-sass", obj], check=True, capture_output=True, text=True).stdout
            res[src] = (log, sass)
        return res
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


@pytest.mark.parametrize("src", sorted(SOURCES))
def test_no_serialised_wgmma(compiled, src):
    log = compiled[src][0]
    kernel = SOURCES[src]
    assert kernel in log, "ptxas -v printed nothing about " + kernel
    bad = [ln for ln in log.splitlines() if SERIALISED.search(ln) and kernel in ln]
    assert not bad, "\n".join(bad)


def _sass_counts(sass, kernel):
    """{function: (HGMMA count, WARPGROUP.DEPBAR count)} for the functions whose name contains `kernel`."""
    counts, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if kernel in m.group(1) else None
            if cur:
                counts[cur] = [0, 0]
            continue
        if cur:
            counts[cur][0] += bool(re.search(r"\bHGMMA\.", line))
            counts[cur][1] += bool(re.search(r"\bWARPGROUP\.DEPBAR\b", line))
    return counts


def test_layer_kernel_mmas_run_back_to_back(compiled):
    counts = _sass_counts(compiled["tdnn_gemm.cu"][1], SOURCES["tdnn_gemm.cu"])
    assert len(counts) == LAYER_INSTANCES, sorted(counts)
    for fn, (hgmma, depbar) in counts.items():
        # a full stage is 12 MMAs (4 K steps x 3 products) under one wait; serialised code waits after each MMA
        assert hgmma >= 12 and depbar < hgmma, (fn, hgmma, depbar)


def test_res2net_chain_mmas_run_back_to_back(compiled):
    counts = _sass_counts(compiled["res2net.cu"][1], SOURCES["res2net.cu"])
    assert len(counts) == 1, sorted(counts)
    for fn, (hgmma, depbar) in counts.items():
        assert hgmma >= 12 and depbar < hgmma, (fn, hgmma, depbar)
