"""CPU checks of masked CAM++ batches: both CAM++ extractors take lengths, the blueprint's refusals of a masked batch it
cannot run, the chunk rule of pipeline/extract_embeddings.py --mixed-lengths (the model's own rule where it has one),
and csrc/campplus.cu built for sm_90a with the masked gate entry and without spills or stack."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from asv_subtools_b200.model import campplus_xvector as cx  # noqa: E402
from asv_subtools_b200.pipeline import extract_embeddings as ee  # noqa: E402


def test_both_campplus_extractors_take_lengths():
    assert cx.CamPPExtractor.TAKES_LENGTHS is True
    assert cx.NativeCamPPExtractor.TAKES_LENGTHS is True


@pytest.fixture(scope="module")
def small_model():
    return cx.CamPPXvector(40, 10, embd_dim=192, init_channels=64, growth_rate=32, bn_size=2).eval()


def test_blueprint_refuses_a_masked_batch_it_cannot_run(small_model):
    """Every refusal comes before the model touches a device."""
    m = small_model
    x = np.zeros((4, 50, 40), np.float32)
    for lens, bad in (([50, 2, 3, 50], r"lengths\[1\]=2 outside \[3, T=50\]"), ([50, 50, 51, 3], r"lengths\[2\]=51"),
                      ([0, 3, 3, 3], r"lengths\[0\]=0"), ([3, 3, 3, -7], r"lengths\[3\]=-7")):
        with pytest.raises(ValueError, match=bad):
            m.extract_embedding_batch(x, lengths=lens)
    with pytest.raises(ValueError, match="T <= 4000, got T=4001"):
        m.extract_embedding_batch(np.zeros((2, 4001, 40), np.float32), lengths=[4001, 300])
    with pytest.raises(ValueError, match="4 entries for a batch of 2|2 entries"):
        m.extract_embedding_batch(np.zeros((2, 50, 40), np.float32), lengths=[50, 50, 50, 50])
    with pytest.raises(ValueError, match="feature dim 40"):
        m.extract_embedding_batch(np.zeros((2, 50, 80), np.float32), lengths=[50, 20])
    with pytest.raises(TypeError, match="float32"):
        m.extract_embedding_batch(np.zeros((2, 50, 40), np.float64), lengths=[50, 20])


def test_only_instances_built_by_init_take_lengths():
    """egrecho's EcapaXvector borrows the extraction methods, and an object init never built has no configuration:
    both refuse a masked batch with NotImplementedError naming their class."""
    from asv_subtools_b200.model.egrecho_ecapa_xvector import EcapaXvector
    for cls in (cx.CamPPXvector, EcapaXvector):
        with pytest.raises(NotImplementedError, match=cls.__name__):
            cls.extract_embedding_batch(cls.__new__(cls), np.zeros((2, 50, 80), np.float32), lengths=[50, 20])


def test_pipeline_cuts_by_the_models_own_chunk_rule(small_model):
    from asv_subtools_b200.model.xvector import Xvector
    assert ee.model_chunk_lengths(small_model, 9000) == [4000, 2500, 2500]
    assert ee.model_chunk_lengths(small_model, 4001) == [2001, 2000]
    assert ee.model_chunk_lengths(small_model, 4000) == [4000]
    assert ee.model_chunk_lengths(small_model, 2) == [2]
    xv = Xvector(23, 10, training=False, extracted_embedding="far")
    for frames in (2, 9000, 10000, 10001, 25000):
        assert ee.model_chunk_lengths(xv, frames) == ee.chunk_lengths(frames), frames
    assert ee.model_chunk_lengths(xv, 9000) == [9000]


class _Recorder:
    """A model for extract_stream_mixed that records every masked batch; its chunk rule is CAM++'s, or none."""

    def __init__(self, campplus):
        if campplus:
            self.chunk_sizes = lambda frames: cx.chunk_sizes(frames)
        self.batches = []

    def extract_embedding_batch(self, x, lengths):
        self.batches.append(list(lengths))
        return torch.ones(len(lengths), 3)


@pytest.mark.parametrize("campplus, want", [(True, [4000, 2500, 2500, 700]), (False, [700, 9000])])
def test_extract_stream_mixed_batches_the_models_chunks(campplus, want):
    model, out = _Recorder(campplus), {}
    feats = [("a", np.zeros((9000, 4), np.float32)), ("b", np.zeros((700, 4), np.float32))]
    utts, batches, _, _ = ee.extract_stream_mixed(model, iter(feats), lambda k, v: out.setdefault(k, v), batch_size=8,
                                                  log=lambda *_: None)
    assert utts == 2 and batches == len(model.batches)
    assert sorted(n for b in model.batches for n in b) == sorted(want)
    assert sorted(out) == ["a", "b"] and all(np.allclose(v, 1.0) for v in out.values())


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="needs nvcc")
def test_campplus_kernels_build_for_sm90a_without_spills(tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    src = os.path.join(ROOT, "asv_subtools_b200", "csrc", "campplus.cu")
    obj = str(tmp_path / "campplus.o")
    flags = ["-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-c", src, "-o", obj], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
    for want in ("xvb_cam_gate", "xvb_cam_gate_lengths", "xvb_bn_relu_planes"):
        assert re.search(r"\bT\s+" + want + r"\b", syms), want
    kernels = 0
    for block in re.split(r"(?=ptxas info\s+: Compiling entry function)", r.stderr):
        if "Compiling entry function" not in block:
            continue
        kernels += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block
    assert kernels == 2, r.stderr[-3000:]
