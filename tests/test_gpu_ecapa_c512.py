"""ECAPA-TDNN C512 (Res2Net scale 8 x width 64) on the GPU: the native handle (xvb_ecapa_t over the width-64 chain kernel)
and the op-by-op Python twin against the reference's golden embeddings (tests/golden/ecapa512.npz), handle == twin bit
for bit, XVBE model files, the shard calls, a C512 and a C1024 handle sharing one device, bin/xvb-extract and the
Python CLI on a C512 model, and the twin's fallback for a channel count the chain kernel does not take."""
import copy
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

import ecapa512_cases as c5
from oracle import nnet as onn

pytestmark = pytest.mark.gpu
EMB_TOL = 1e-4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cos(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)))


def _model(case, pos, native, monkeypatch):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    monkeypatch.setenv("XVB_ECAPA_NATIVE", native)
    kw, spec, seed = c5.CASES[case][:3]
    m = ECAPA_TDNN(80, 10, training=False, extracted_embedding=pos, **copy.deepcopy(kw))
    m.load_state_dict(onn.make_state_dict(spec, seed), strict=True)
    m.cuda().eval()
    assert type(m.extractor()).__name__ == ("NativeEcapaExtractor" if native == "1" else "EcapaExtractor")
    return m


@pytest.mark.parametrize("native", ["1", "0"])
@pytest.mark.parametrize("case", sorted(c5.CASES))
def test_c512_matches_reference_golden(golden, monkeypatch, case, native):
    g = golden("ecapa512")
    _, _, _, positions, frames, _ = c5.CASES[case]
    for pos in positions:
        m = _model(case, pos, native, monkeypatch)
        for t in frames:
            key = "{}_{}_T{}".format(case, pos, t)
            want = g[key]
            feats = c5.utterances(case, t)
            got = np.stack([m.extract_embedding(f).numpy() for f in feats])       # the maxChunk rule for T = 10 050
            if t <= 10000:
                batch = m.extract_embedding_batch(feats).cpu().numpy()
                assert rel(batch, want) <= EMB_TOL, key
            for i in range(len(feats)):
                assert rel(got[i], want[i]) <= EMB_TOL, (key, i)
                assert cos(got[i], want[i]) >= 1 - 1e-6, (key, i)
        m.invalidate()


def test_c512_handle_equals_twin_bit_for_bit(monkeypatch):
    feats = {(B, T): torch.from_numpy(onn.synthetic_feats(B, T, 80, 7000 + 10 * B + T)).cuda()
             for B in (1, 3, 64) for T in (2, 37, 128, 129, 300)}
    for case, pos in (("canon", "near"), ("canon", "near_affine"), ("fc1", "far"), ("fc1", "near_affine"), ("fc1", "near"),
                      ("mqmha", "near")):
        outs = {}
        for native in ("1", "0"):
            m = _model(case, pos, native, monkeypatch)
            ex = m.extractor()
            outs[native] = {k: ex.extract(x).clone() for k, x in feats.items()}
            m.invalidate()
        for k in feats:
            assert torch.equal(outs["1"][k], outs["0"][k]), (case, pos, k)
            assert torch.isfinite(outs["1"][k]).all(), (case, pos, k)


def test_c512_twin_per_scale_gemms_agree_with_chain(monkeypatch):
    feats = torch.from_numpy(onn.synthetic_feats(5, 150, 80, 7100)).cuda()
    outs = {}
    for mode in ("chain", "gemm"):
        monkeypatch.setenv("XVB_ECAPA_RES2NET", mode)
        m = _model("canon", "near", "0", monkeypatch)
        assert m.extractor().chain == (mode == "chain")
        outs[mode] = m.extractor().extract(feats).cpu().numpy()
        m.invalidate()
    assert rel(outs["gemm"], outs["chain"]) <= 1e-5


def test_c512_model_files_round_trip_and_bad_channels_are_refused(tmp_path, monkeypatch):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import NativeEcapaExtractor
    feats = torch.from_numpy(onn.synthetic_feats(6, 93, 80, 7200)).cuda()
    for case, magic in (("canon", b"XVBE0001"), ("mqmha", b"XVBE0002")):
        m = _model(case, "near", "1", monkeypatch)
        ex = m.extractor()
        path = str(tmp_path / "{}.xvbm".format(case))
        ex.save(path)
        raw = open(path, "rb").read()
        assert raw[:8] == magic and struct.unpack("<6i", raw[8:32])[:2] == (80, 512)
        ex2 = NativeEcapaExtractor.load(path)
        assert ex2.feat_dim == 80 and ex2.embed_dim == 192
        assert torch.equal(ex2.extract(feats), ex.extract(feats)), case
        ex2.close()
        m.invalidate()
        bad = str(tmp_path / "{}_768.xvbm".format(case))
        with open(bad, "wb") as f:
            f.write(raw[:12] + struct.pack("<i", 768) + raw[16:])
        with pytest.raises(RuntimeError, match="768"):
            NativeEcapaExtractor.load(bad)


@pytest.mark.parametrize("lanes", ["0", "1"])
def test_c512_shard_calls_equal_per_batch_extraction(monkeypatch, lanes):
    m = _model("canon", "near", "1", monkeypatch)
    ex = m.extractor()
    n, t = 11, 47
    feats = torch.from_numpy(onn.synthetic_feats(n, t, 80, 7300)).cuda()
    want = torch.cat([ex.extract(feats[i:i + 4]).clone() for i in range(0, n, 4)])         # batches of 4, 4, 3
    monkeypatch.setenv("XVB_LANES", lanes)
    assert torch.equal(ex.extract_shard(feats, 4), want)
    assert torch.equal(ex.extract_shard(feats, 4), want)                                    # lanes reused
    assert torch.equal(ex.extract_shard(feats[:8], 4), want[:8])
    assert np.array_equal(ex.extract_host(feats[:4].cpu().numpy()), want[:4].cpu().numpy())
    host = torch.empty(n, t, 80, dtype=torch.float32, pin_memory=True)
    host.copy_(feats)
    out = torch.empty(n, ex.embed_dim, dtype=torch.float32, pin_memory=True)
    ex.extract_shard_host(host.data_ptr(), n, t, out.data_ptr(), 4)
    assert torch.equal(out, want.cpu())


def test_c512_and_c1024_handles_alternate_on_one_device(monkeypatch):
    """Both handles draw on the device's one shared workspace; alternating them (the C1024 call grows it, the C512 call
    reuses it) must give the bits of fresh handles."""
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    monkeypatch.setenv("XVB_ECAPA_NATIVE", "1")

    def c1024():
        m = ECAPA_TDNN(80, 10, **dict(copy.deepcopy(c5.CANON), training=False, extracted_embedding="near",
                                      ecapa_params=dict(c5.CANON["ecapa_params"], channels=1024)))
        m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80), 201), strict=True)
        return m.cuda().eval()

    small = [torch.from_numpy(onn.synthetic_feats(3, 61, 80, 7400 + i)).cuda() for i in range(2)]
    big = [torch.from_numpy(onn.synthetic_feats(9, 211, 80, 7410 + i)).cuda() for i in range(2)]
    fresh = {}
    for name, make in (("c512", lambda: _model("canon", "near", "1", monkeypatch)), ("c1024", c1024)):
        for i in range(2):
            for which, x in (("small", small[i]), ("big", big[i])):
                m = make()
                fresh[name, which, i] = m.extractor().extract(x).clone()
                m.invalidate()
    a, b = _model("canon", "near", "1", monkeypatch).extractor(), c1024().extractor()
    for i in range(2):
        for which, x in (("small", small[i]), ("big", big[i])):
            assert torch.equal(a.extract(x), fresh["c512", which, i]), (which, i)
            assert torch.equal(b.extract(x), fresh["c1024", which, i]), (which, i)
        assert torch.equal(a.extract(big[i]), fresh["c512", "big", i])


def test_xvb_extract_and_python_cli_on_a_c512_model_file(tmp_path, monkeypatch):
    """XVBE0001 C512 file -> bin/xvb-extract without Python: one utterance longer than --max-chunk (three chunks), all
    against the oracle; and the Python CLI on a reference-style model dir (--blueprint-dir) gives the same vectors as the
    binary at the default chunk size."""
    from asv_subtools_b200 import kaldi_io
    m = _model("canon", "near", "1", monkeypatch)
    kw, spec, seed = c5.CASES["canon"][:3]
    sd = onn.make_state_dict(spec, seed)
    model = str(tmp_path / "ecapa512.xvbm")
    m.extractor().save(model)
    lengths = [120, 120, 75, 450, 2]                        # 450 > --max-chunk 200: chunks of 150
    feats = {"e{}".format(i): onn.synthetic_feats(1, t, 80, 7500 + i)[0] for i, t in enumerate(lengths)}
    ark = str(tmp_path / "feats.ark")
    with open(ark, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    out = str(tmp_path / "bin200.ark")
    run = subprocess.run([BIN, "--batch", "2", "--max-chunk", "200", model, ark, "ark:" + out], capture_output=True,
                         text=True, timeout=600)
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(got) == sorted(feats)
    for k, v in feats.items():
        want = onn.extract_embedding(lambda x: onn.ecapa_forward(sd, x, "near"), v, max_chunk=200).numpy()
        assert got[k].shape == (192,) and rel(got[k], want) <= EMB_TOL, k
    out = str(tmp_path / "bin.ark")
    run = subprocess.run([BIN, "--batch", "2", model, ark, "ark:" + out], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout + run.stderr
    binary = dict(kaldi_io.read_vec_flt_ark(out))
    torch.save(sd, str(tmp_path / "final.params"))
    creation = "ECAPA_TDNN(80,10,training=False,extracted_embedding='near',{})".format(
        ",".join("{}={!r}".format(k, v) for k, v in kw.items()))
    (tmp_path / "nnet.config").write_text('model_blueprint;subtools/pytorch/model/ecapa_tdnn_xvector.py\nmodel_creation;"{}"\n'
                                          .format(creation.replace('"', '""')))
    cli = str(tmp_path / "cli.ark")
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--nnet-config",
                        str(tmp_path / "nnet.config"), "--blueprint-dir", os.path.join(ROOT, "asv_subtools_b200", "model"),
                        "--batch-size", "2", str(tmp_path / "final.params"), "ark:" + ark, "ark:" + cli],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    py = dict(kaldi_io.read_vec_flt_ark(cli))
    assert sorted(py) == sorted(feats)
    for k, v in feats.items():
        assert rel(py[k], binary[k]) <= 1e-5, k
        want = onn.extract_embedding(lambda x: onn.ecapa_forward(sd, x, "near"), v).numpy()
        assert rel(py[k], want) <= EMB_TOL, k


def test_c256_runs_on_the_twin_and_matches_the_oracle(monkeypatch):
    """Width 32 (C = 256) is not a chain-kernel instance: build_extractor keeps the Python twin, whose Res2Net blocks run
    as the chunk copy + per-scale GEMMs."""
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    monkeypatch.setenv("XVB_ECAPA_NATIVE", "1")
    kw = copy.deepcopy(c5.CANON)
    kw["ecapa_params"]["channels"] = 256
    sd = onn.make_state_dict(onn.ecapa_spec(80, channels=256), 256)
    m = ECAPA_TDNN(80, 10, training=False, extracted_embedding="near", **kw)
    m.load_state_dict(sd, strict=True)
    m.cuda().eval()
    assert type(m.extractor()).__name__ == "EcapaExtractor"
    feats = onn.synthetic_feats(3, 140, 80, 7600)
    got = m.extract_embedding_batch(feats).cpu().numpy()
    with torch.no_grad():
        ref = onn.ecapa_forward(sd, torch.from_numpy(feats).transpose(1, 2), "near").squeeze(2).numpy()
    for i in range(3):
        assert rel(got[i], ref[i]) <= EMB_TOL, i
