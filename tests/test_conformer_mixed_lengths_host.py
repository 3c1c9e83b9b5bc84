"""CPU checks of masked Conformer batches: both Conformer extractors take lengths, the blueprint's chunk rule is the
reference's 300-frame rule and pipeline/extract_embeddings.py --mixed-lengths cuts with it, the blueprint's refusals of
a masked batch it cannot run come before any device work, and csrc/conformer.cu / csrc/ecapa.cu build for sm_90a with
the masked entries and without spills or stack."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import conformer_oracle as co  # noqa: E402
from asv_subtools_b200.model import transformer_xvector as tx  # noqa: E402
from asv_subtools_b200.pipeline import extract_embeddings as ee  # noqa: E402

FRAMES = [7, 299, 300, 301, 599, 600, 650, 899, 29999, 100000]


def test_both_conformer_extractors_take_lengths():
    assert tx.ConformerExtractor.TAKES_LENGTHS is True
    assert tx.NativeConformerExtractor.TAKES_LENGTHS is True


@pytest.fixture(scope="module")
def small_model():
    kwargs, fdim = co.CASES["small"][:2]
    return tx.TransformerXvector(fdim, 10, training=False, extracted_embedding="near", **kwargs).eval()


@pytest.mark.parametrize("frames", FRAMES)
def test_chunk_sizes_is_the_chunk_plan(small_model, frames):
    assert small_model.chunk_sizes(frames) == tx.chunk_plan(frames)[0] == co.chunk_plan(frames)[0]


def test_pipeline_cuts_conformer_utterances_by_chunk_sizes(small_model):
    for frames in FRAMES:
        assert ee.model_chunk_lengths(small_model, frames) == small_model.chunk_sizes(frames), frames
    assert ee.model_chunk_lengths(small_model, 1799) == [299] * 5 + [304]
    assert ee.model_chunk_lengths(small_model, 650) == [216, 216, 218]
    # the maxChunk rule of the other models would have left 650 frames whole
    assert ee.chunk_lengths(650) == [650]


def test_blueprint_refuses_a_masked_batch_it_cannot_run(small_model):
    """Every refusal comes before the model touches a device (the model here lives on the CPU)."""
    m = small_model
    x = np.zeros((4, 50, 23), np.float32)
    for lens, bad in (([50, 6, 7, 50], r"lengths\[1\]=6 outside \[7, T=50\]"), ([50, 50, 51, 7], r"lengths\[2\]=51"),
                      ([0, 7, 7, 7], r"lengths\[0\]=0"), ([7, 7, 7, -7], r"lengths\[3\]=-7")):
        with pytest.raises(ValueError, match=bad):
            m.extract_embedding_batch(x, lengths=lens)
    # 20 005 frames subsample to T' = 5000, past the positional tables
    with pytest.raises(ValueError, match="5000 subsampled frames"):
        m.extract_embedding_batch(np.zeros((1, 20005, 23), np.float32), lengths=[20005])
    with pytest.raises(ValueError, match="4 entries for a batch of 2"):
        m.extract_embedding_batch(np.zeros((2, 50, 23), np.float32), lengths=[50, 50, 50, 50])
    with pytest.raises(ValueError, match="feature dim 23"):
        m.extract_embedding_batch(np.zeros((2, 50, 80), np.float32), lengths=[50, 20])
    with pytest.raises(TypeError, match="float32"):
        m.extract_embedding_batch(np.zeros((2, 50, 23), np.float64), lengths=[50, 20])


def test_only_instances_built_by_init_take_lengths():
    cls = tx.TransformerXvector
    with pytest.raises(NotImplementedError, match="TransformerXvector"):
        cls.extract_embedding_batch(cls.__new__(cls), np.zeros((2, 50, 80), np.float32), lengths=[50, 20])


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _ptxas(src, tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    obj = str(tmp_path / (os.path.basename(src) + ".o"))
    flags = ["-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-c", src, "-o", obj], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    blocks = {}
    for block in re.split(r"(?=ptxas info\s+: Compiling entry function)", r.stderr):
        m = re.search(r"Compiling entry function '(\S+)'", block)
        if m:
            blocks[m.group(1)] = block
    return syms, blocks


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="needs nvcc")
def test_masked_kernels_build_for_sm90a_without_spills(tmp_path):
    """The three kernels with a masked mode keep their registers (head 32, attention at most 40, attentive pooling
    at most 64), with no stack and no spills."""
    csrc = os.path.join(ROOT, "asv_subtools_b200", "csrc")
    want = {"subsample_head_kernel": 32, "rope_attention_kernelILi32": 40, "rope_attention_kernelILi64": 40,
            "rope_attention_kernelILi128": 40, "attn_stats_pool_kernel": 64}
    seen = set()
    for src, entries in (("conformer.cu", ("xvb_subsample_head_lengths", "xvb_rope_attention_lengths")),
                         ("ecapa.cu", ("xvb_attn_stats_pool_lengths",))):
        syms, blocks = _ptxas(os.path.join(csrc, src), tmp_path)
        for e in entries:
            assert re.search(r"\bT\s+" + e + r"\b", syms), e
        for name, block in blocks.items():
            for k, regs in want.items():
                if re.search(r"\d" + k + r"(E|\b)", name):
                    seen.add(k)
                    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block
                    used = int(re.search(r"Used (\d+) registers", block).group(1))
                    assert used <= regs, (k, used)
    assert seen == set(want), seen
