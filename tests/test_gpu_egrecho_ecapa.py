"""egrecho's ECAPA-TDNN on the GPU: the native ECAPA-TDNN handle in its chained form and the op-by-op twin against the
reference's golden embeddings and each other, batch rows against per-utterance calls, shard calls, XVBG0001 model files
and bin/xvb-extract."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import egrecho_ecapa_oracle as eo  # noqa: E402
from asv_subtools_b200.model import ecapa_tdnn_xvector as etx  # noqa: E402
from asv_subtools_b200.model import egrecho_ecapa_xvector as eg  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "egrecho_ecapa.npz"))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
DEV = torch.device("cuda", 0)


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cosine(a, b):
    a, b = np.asarray(a, dtype=np.float64).reshape(len(a), -1), np.asarray(b, dtype=np.float64).reshape(len(b), -1)
    return float(np.min(np.sum(a * b, 1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1)))


def _model(case, pos="near"):
    config, _, _, _, seed, _ = eo.CASES[case]
    m = eg.EcapaXvector(config["inputs_dim"], 10, extracted_embedding=pos, **eo.blueprint_kwargs(config))
    m.load_state_dict(eo.seeded_state_dict(GOLD["keys_" + case], seed), strict=True)
    return m.to(DEV).eval()


SHORT = [(c, p, t) for c, (_, frames, _, positions, _, _) in eo.CASES.items() for p in positions for t in frames]
LONG = [(c, p, t) for c, (_, _, long_frames, positions, _, _) in eo.CASES.items() for p in positions for t in long_frames]


@pytest.mark.parametrize("case,pos,t", SHORT)
def test_native_and_twin_match_golden_and_each_other(case, pos, t):
    m = _model(case, pos)
    fseed = eo.CASES[case][5]
    feats = eo.utterances(2, t, m.inputs_dim, fseed + t).to(DEV)
    want = GOLD["{}_{}_T{}".format(case, pos, t)]
    twin = etx.EcapaExtractor(m, DEV).extract(feats).cpu().numpy()
    outs = [twin]
    if m.channels in etx.NATIVE_CHANNELS:
        assert isinstance(m.extractor(), etx.NativeEcapaExtractor)
        nat = m.extractor().extract(feats).cpu().numpy()
        assert np.array_equal(nat, twin), (case, pos, t)
        outs.append(nat)
    else:
        assert isinstance(m.extractor(), etx.EcapaExtractor)
    for got in outs:
        assert rel(got, want) <= 1e-4 and cosine(got, want) >= 1 - 1e-6, (case, pos, t, rel(got, want))


@pytest.mark.parametrize("case,pos,t", LONG)
def test_chunk_rule_matches_extract_embedding(case, pos, t):
    m = _model(case, pos)
    feats = eo.utterances(2, t, m.inputs_dim, eo.CASES[case][5] + t)
    got = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(2)])
    want = GOLD["{}_{}_T{}".format(case, pos, t)]
    assert rel(got, want) <= 1e-4 and cosine(got, want) >= 1 - 1e-6, rel(got, want)
    batch = m.extract_embedding_batch(feats).cpu().numpy()
    assert np.array_equal(batch, got)


@pytest.mark.parametrize("case", ["c512", "c1024"])
def test_native_equals_twin_and_batch_rows_equal_single_calls(case):
    """Native handle and twin bit for bit at every batch and length; a batch row equals the utterance extracted alone
    bit for bit (each kernel's per-row arithmetic does not depend on the batch)."""
    m = _model(case)
    nat, twin = m.extractor(), etx.EcapaExtractor(m, DEV)
    g = torch.Generator().manual_seed(11)
    for B in (1, 3, 64):
        for T in (1, 2, 5, 37, 300):
            x = torch.randn(B, T, 80, generator=g).to(DEV)
            a, b = nat.extract(x), twin.extract(x)
            assert torch.equal(a, b), (case, B, T)
            if B == 3:
                for i in range(B):
                    assert torch.equal(nat.extract(x[i:i + 1].contiguous())[0], a[i]), (case, T, i)


def test_shard_calls_on_two_lanes_equal_per_batch_calls():
    m = _model("c1024")
    ex = m.extractor()
    feats = eo.utterances(160, 120, 80, 77).to(DEV)
    shard = ex.extract_shard(feats, batch=64)
    per = torch.cat([ex.extract(feats[i:i + 64].contiguous()) for i in range(0, 160, 64)])
    torch.cuda.synchronize()
    assert torch.equal(shard, per)
    host = np.empty((160, 192), dtype=np.float32)
    pinned = feats.cpu().pin_memory()
    ex.extract_shard_host(pinned.data_ptr(), 160, 120, host.ctypes.data, batch=64)
    assert np.array_equal(host, per.cpu().numpy())


def test_xvbg0001_round_trip_layout_and_rejections(tmp_path):
    from asv_subtools_b200 import _lib
    m = _model("mqmha")
    ex = m.extractor()
    path = str(tmp_path / "eg.xvbm")
    ex.save(path)
    raw = open(path, "rb").read()
    # magic | feat_dim, channels, mfa_dim, att_hidden, embed_dim, n_layers | the pooling record | residual form
    assert raw[:8] == b"XVBG0001"
    head = struct.unpack("<14i", raw[8:64])
    recs = eg.native_records(m)
    assert head == (80, 512, 1536, 128 * 4 * 2, 192, len(recs), 4, 2, 128, 1, 1, 1, 1, 1)
    name_len = struct.unpack("<i", raw[64:68])[0]
    assert raw[68:68 + name_len] == b"layer1"
    feats = eo.utterances(3, 90, 80, 9).to(DEV)
    loaded = etx.NativeEcapaExtractor.load(path)
    assert torch.equal(loaded.extract(feats), ex.extract(feats))
    again = str(tmp_path / "again.xvbm")
    loaded.save(again)
    assert open(again, "rb").read() == raw
    for name, data in (("trunc", raw[:len(raw) // 2]), ("trunc_header", raw[:60]), ("magic", b"XVBG0002" + raw[8:]),
                       ("form", raw[:60] + struct.pack("<i", 2) + raw[64:])):
        bad = str(tmp_path / name)
        open(bad, "wb").write(data)
        with pytest.raises(_lib.XvbError):
            etx.NativeEcapaExtractor.load(bad)


def test_xvb_extract_runs_an_xvbg0001_file(tmp_path):
    from asv_subtools_b200 import kaldi_io
    from asv_subtools_b200.pipeline import extract_embeddings
    m = _model("c512")
    model = str(tmp_path / "c512.xvbm")
    m.extractor().save(model)
    lens = {"a": 9000, "b": 4001, "c": 300, "d": 300, "e": 37}
    feats = {k: eo.utterances(1, t, 80, 600 + i)[0].numpy() for i, (k, t) in enumerate(lens.items())}
    feats["g"] = eo.utterances(2, 9000, 80, eo.CASES["c512"][5] + 9000)[1].numpy()
    ark = str(tmp_path / "feats.ark")
    with open(ark, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    out = str(tmp_path / "xv.ark")
    run = subprocess.run([BIN, "--batch", "4", model, ark, "ark:" + out], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    assert rel(got["g"][None], GOLD["c512_near_T9000"][1:]) <= 1e-4
    # the Python CLI over the same blueprint and the backbone weights of a checkpoint
    params = str(tmp_path / "final.params")
    torch.save({"ecapa." + k: v for k, v in m.state_dict().items()}, params)
    py_out = str(tmp_path / "py.ark")
    blueprint = os.path.join(ROOT, "asv_subtools_b200", "model", "egrecho_ecapa_xvector.py")
    extract_embeddings.main(["--model-blueprint", blueprint, "--model-creation", "EcapaXvector(80,10)", "--use-gpu", "true",
                             params, "ark:" + ark, "ark:" + py_out])
    py = dict(kaldi_io.read_vec_flt_ark(py_out))
    for k, v in feats.items():
        want = m.extract_embedding(v).numpy()
        assert rel(got[k], want) <= 1e-5, k
        assert rel(py[k], want) <= 1e-5, k
        with torch.no_grad():
            ref = eo.extract_embedding(eo.seeded_state_dict(GOLD["keys_c512"], eo.CASES["c512"][4]),
                                       torch.from_numpy(v)[None], eo.CASES["c512"][0])[0].numpy()
        assert rel(got[k], ref) <= 1e-4, k
    run = subprocess.run([BIN, "--mixed-lengths", model, ark, "ark:" + out], capture_output=True, text=True, timeout=300)
    assert run.returncode == 1 and "ERROR" in run.stderr
