"""Speaker retrieval on the CPU: the top-k file writer and the mAP of score/retrieve.py and score/metrics.py against
the reference's own trans_score_format.py / cal_mAP.py output (tests/golden/retrieval.npz), the ctypes prototypes of
the retrieval entry points against include/xvb200.h, and csrc/retrieval.cu built for sm_90a without spills or stack."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "retrieval.npz")


def _golden():
    z = np.load(GOLDEN)
    return z, [str(k) for k in z["enroll_keys"]], [str(k) for k in z["test_keys"]]


def _stable_topk(s, k):
    """Score descending, index ascending: nlargest(keep='first') over a score file in trials order."""
    return np.stack([np.lexsort((np.arange(r.size), -r))[:k] for r in s])


def test_writer_reproduces_trans_score_format():
    from asv_subtools_b200.score.retrieve import format_topk
    z, ek, tk = _golden()
    text = format_topk(ek, tk, _stable_topk(z["scores64"], 10))
    assert text.encode("utf-8") == bytes(z["top10"])
    assert not text.endswith("\n") and text.count("\n") == len(ek) - 1
    # the golden has exact ties inside the top-10 lists (duplicated test vectors): the lower test index comes first
    s = z["scores64"]
    idx = _stable_topk(s, 10)
    assert sum(int(np.sum(np.diff(s[i, idx[i]]) == 0)) for i in range(len(ek))) > 0


def test_writer_skips_empty_slots_and_sorts_speakers():
    from asv_subtools_b200.score.retrieve import format_topk
    text = format_topk(["b", "a", "c"], ["u0", "u1"], np.array([[1, 0, -1], [0, -1, -1], [1, -1, -1]]))
    assert text == "a u0\nb u1 u0\nc u1"


def test_map_equals_cal_map_on_the_golden():
    from asv_subtools_b200.score import metrics
    z, _, _ = _golden()
    top = bytes(z["top10"]).decode("utf-8").splitlines(True)
    meta = bytes(z["meta"]).decode("utf-8").splitlines(True)
    assert "mAP=%.3f" % metrics.retrieval_map(top, meta) == str(z["map_line"])


def test_map_quirks():
    from asv_subtools_b200.score import metrics
    meta = ["pool/u1.wav s1-a-01\n", "pool/u2a.wav s1-b-02\n", "wav/u3.wav s2-x\n", "pool/u4.wav s2-y\n"]
    # every position adds hits-so-far / i, hit or not; the sum is divided by 10 whatever the list length
    assert metrics.retrieval_map(["s1 u1 u9 u1"], meta) == pytest.approx((1 / 1 + 1 / 2 + 2 / 3) / 10, abs=0)
    # strip('.wav') is a character-set strip: u2a loses its 'a' and never matches; "wav/u3.wav" -> "/u3" -> "u3"
    assert metrics.retrieval_map(["s1 u2a"], meta) == 0.0
    assert metrics.retrieval_map(["s2 u3"], meta) == pytest.approx(0.1, abs=0)
    # the mean is over the lines of the top-k file
    assert metrics.retrieval_map(["s1 u1", "s2 u9"], meta) == pytest.approx(0.05, abs=0)
    with pytest.raises(KeyError):
        metrics.retrieval_map(["s3 u1"], meta)


def test_map_files_roundtrip(tmp_path):
    from asv_subtools_b200.score import metrics
    z, _, _ = _golden()
    (tmp_path / "top").write_bytes(bytes(z["top10"]))
    (tmp_path / "meta").write_bytes(bytes(z["meta"]))
    assert "mAP=%.3f" % metrics.retrieval_map_files(str(tmp_path / "top"), str(tmp_path / "meta")) == str(z["map_line"])


# ------------------------------------------------------------------------------------------------ C ABI
_CTYPES = {"const float*": C.c_void_p, "float*": C.c_void_p, "int64_t*": C.c_void_p, "uint64_t*": C.c_void_p,
           "void*": C.c_void_p, "int64_t": C.c_int64, "int": C.c_int}


def _header_prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "xvb200.h")).read(), flags=re.S)
    m = re.search(r"\b(int|int64_t)\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    args = []
    for a in m.group(2).split(","):
        a = " ".join(a.split())
        args.append(_CTYPES[re.sub(r"\s*\b\w+$", "", a).replace(" *", "*")])
    return {"int": C.c_int, "int64_t": C.c_int64}[m.group(1)], args


@pytest.mark.parametrize("name", ["xvb_topk_merge", "xvb_retrieve_topk_slab_bytes", "xvb_retrieve_topk"])
def test_ctypes_prototypes_match_the_header(name):
    from asv_subtools_b200 import _lib
    res, args = _lib.SIGNATURES[name]
    assert (res, args) == _header_prototype(name), name


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="needs nvcc")
def test_retrieval_builds_for_sm90a_without_spills(tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    src = os.path.join(ROOT, "asv_subtools_b200", "csrc", "retrieval.cu")
    obj = str(tmp_path / "retrieval.o")
    flags = ["-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-c", src, "-o", obj], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    for want in ("xvb_topk_merge", "xvb_retrieve_topk_slab_bytes", "xvb_retrieve_topk"):
        assert re.search(r"\bT\s+" + want + r"\b", syms), want
    seen = 0
    for block in re.split(r"(?=ptxas info\s+: Compiling entry function)", r.stderr):
        if "Compiling entry function" not in block:
            continue
        seen += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block
    assert seen == 3, r.stderr[-3000:]
