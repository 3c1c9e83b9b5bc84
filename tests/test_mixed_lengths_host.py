"""Batch rule of --mixed-lengths (pipeline/extract_embeddings.py plan_mixed_batches, the same rule as xvb-extract's),
the chunk rule it runs after, the ctypes mirror of xvb_tdnn_args_t.lengths and the integration script's switch.
CPU only."""
import os
import subprocess

import numpy as np
import pytest

from asv_subtools_b200.pipeline.extract_embeddings import Batcher, chunk_lengths, plan_mixed_batches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check_plan(lengths, batch):
    plan = plan_mixed_batches(lengths, batch)
    flat = [i for b in plan for i in b]
    assert sorted(flat) == list(range(len(lengths)))                 # every item exactly once
    for b in plan:
        assert 1 <= len(b) <= batch
        lens = [lengths[i] for i in b]
        assert lens == sorted(lens)
        tmax = max(lens)
        assert 8 * (len(b) * tmax - sum(lens)) <= len(b) * tmax      # padding <= 1/8 of the batch
    ordered = [lengths[i] for i in flat]
    assert ordered == sorted(ordered)                                # ascending, batches consecutive
    return plan


@pytest.mark.parametrize("seed,n,batch", [(0, 4000, 256), (1, 1000, 64), (2, 300, 7), (3, 50, 1)])
def test_mixed_batches_on_a_seeded_length_spread(seed, n, batch):
    rng = np.random.RandomState(seed)
    lengths = [int(v) for v in rng.randint(1, 3000, n)] + [1, 1, 2, 3, 10000]
    plan = _check_plan(lengths, batch)
    if batch == 256:          # a dense spread puts most items in full batches (short ones pad too much to share)
        assert sum(len(b) for b in plan if len(b) == batch) >= 0.75 * len(lengths)


def test_mixed_batches_grow_with_a_log_spread():
    rng = np.random.RandomState(7)
    lengths = [int(v) for v in np.exp(rng.uniform(0, np.log(12000), 2000))]
    plan = _check_plan(lengths, 256)
    assert len(plan) < len(set(lengths))                             # fewer batches than equal-length buckets


def _batcher_buckets(lengths, batch):
    bt = Batcher(batch, length=lambda i: lengths[i])
    out = []
    for i in range(len(lengths)):
        out += [[k for k, _ in b] for b in bt.add(i, i)]
    return out + [[k for k, _ in b] for b in bt.flush()]


@pytest.mark.parametrize("n,batch", [(1, 256), (256, 256), (600, 256), (10, 3), (5, 1)])
def test_equal_lengths_give_the_equal_length_buckets(n, batch):
    lengths = [200] * n
    assert plan_mixed_batches(lengths, batch) == _batcher_buckets(lengths, batch)


def test_lengths_too_far_apart_to_share_a_batch_stay_in_their_buckets():
    rng = np.random.RandomState(5)
    lengths = [int(v) for v in rng.choice([100, 200, 400, 800], 700)]   # any mix of two pads more than 1/8
    got = sorted(tuple(b) for b in plan_mixed_batches(lengths, 64))
    assert got == sorted(tuple(b) for b in _batcher_buckets(lengths, 64))


def test_empty_and_single():
    assert plan_mixed_batches([], 4) == []
    assert plan_mixed_batches([7], 4) == [[0]]


@pytest.mark.parametrize("frames", [1, 2, 9999, 10000, 10001, 12000, 20001, 35000])
def test_chunk_lengths_is_the_max_chunk_rule(frames):
    lens = chunk_lengths(frames)
    num_split = (frames + 9999) // 10000
    assert len(lens) == num_split and sum(lens) == frames
    assert all(l == frames // num_split for l in lens[:-1]) and max(lens) <= 10000 + num_split


def test_tdnn_args_mirror_ends_with_lengths():
    import ctypes as C
    from asv_subtools_b200._lib import TdnnArgs
    names = [f[0] for f in TdnnArgs._fields_]
    assert names[-2:] == ["groups", "lengths"] and TdnnArgs.lengths.size == C.sizeof(C.c_void_p)


def test_integration_switch_passes_the_flag(tmp_path):
    old = "python3 subtools/pytorch/pipeline/onestep/extract_embeddings.py"
    job = tmp_path / "extract_xvectors_for_pytorch.sh"
    job.write_text("#!/bin/bash\n{} --use-gpu=true m f o\n".format(old))
    for value, want in (("1", True), ("", False), ("0", False)):
        env = dict(os.environ, XVB200_DRYRUN="1", XVB200_REF=str(job), XVB200_MIXED_LENGTHS=value)
        r = subprocess.run(["bash", os.path.join(ROOT, "integration/extract_xvectors_b200.sh"), "m", "d", "o"],
                           capture_output=True, text=True, env=env, cwd=str(tmp_path))
        lines = [l for l in r.stdout.splitlines() if l.startswith(">")]
        assert r.returncode == 0 and len(lines) == 1, r.stdout + r.stderr
        assert ("--mixed-lengths" in lines[0]) == want
