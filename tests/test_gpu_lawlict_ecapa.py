"""The ECAPA-TDNN of pytorch/model/ecapa-tdnn-xvector.py (the runEcapaXvector.py launcher's model) on the GPU: the
native ECAPA-TDNN handle with the attention without global context and the op-by-op twin against the reference's golden
embeddings and each other, batch rows against per-utterance calls, shard calls, XVBE0003 model files, bin/xvb-extract and
the Python CLI on a launcher model directory."""
import ctypes
import importlib.util
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
import ecapa512_cases as c5  # noqa: E402
import lawlict_ecapa_oracle as lo  # noqa: E402
from asv_subtools_b200.model import ecapa_tdnn_xvector as etx  # noqa: E402
from oracle import nnet as onn  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "lawlict_ecapa.npz"))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
BLUEPRINT = os.path.join(ROOT, "asv_subtools_b200", "model", "ecapa-tdnn-xvector.py")
DEV = torch.device("cuda", 0)


def _load_blueprint():
    spec = importlib.util.spec_from_file_location("lawlict_ecapa_blueprint", BLUEPRINT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


bp = _load_blueprint()


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cosine(a, b):
    a, b = np.asarray(a, dtype=np.float64).reshape(len(a), -1), np.asarray(b, dtype=np.float64).reshape(len(b), -1)
    return float(np.min(np.sum(a * b, 1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1)))


def _model(case, pos="near"):
    inputs_dim, kw = lo.CASES[case][:2]
    m = bp.ECAPA_TDNN(inputs_dim, 1211, **dict(kw, extracted_embedding=pos))
    m.load_state_dict(lo.state_dict(case), strict=True)
    return m.to(DEV).eval()


def _dense(channels):
    """ECAPA_TDNN (ecapa_tdnn_xvector.py) of the same width, with the default attentive pooling."""
    kw = dict(c5.CANON, ecapa_params=dict(c5.CANON["ecapa_params"], channels=channels))
    m = etx.ECAPA_TDNN(80, 10, **kw)
    m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80, channels=channels), 201), strict=True)
    return m.to(DEV).eval()


SHORT = [(c, p, t) for c, (_, _, short, _, poss, _, _) in lo.CASES.items() for p in poss for t in short]
LONG = [(c, p, t) for c, (_, _, _, long, poss, _, _) in lo.CASES.items() for p in poss for t in long]


@pytest.mark.parametrize("case,pos,t", SHORT)
def test_native_and_twin_match_golden_and_each_other(case, pos, t):
    m = _model(case, pos)
    feats = torch.from_numpy(lo.utterances(case, t)).to(DEV)
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
    feats = lo.utterances(case, t)
    got = np.stack([m.extract_embedding(f).numpy() for f in feats])
    want = GOLD["{}_{}_T{}".format(case, pos, t)]
    assert rel(got, want) <= 1e-4 and cosine(got, want) >= 1 - 1e-6, rel(got, want)


@pytest.mark.parametrize("case", ["launcher", "c1024"])
def test_native_equals_twin_batch_rows_and_launches(case):
    """Native handle and twin bit for bit at every batch and length; a batch row equals the utterance extracted alone bit
    for bit; the handle issues two launches fewer than ECAPA_TDNN's of the same width (no global statistics pass, no
    att_gs), one fewer at T = 1."""
    m = _model(case)
    nat, twin = m.extractor(), etx.EcapaExtractor(m, DEV)
    dense = _dense(m.channels).extractor()
    g = torch.Generator().manual_seed(12)
    for B in (1, 3, 64):
        for T in (1, 2, 5, 37, 300):
            x = torch.randn(B, T, 80, generator=g).to(DEV)
            a, b = nat.extract(x), twin.extract(x)
            assert torch.equal(a, b), (case, B, T)
            dense.extract(x)
            # at T = 1 att_x, which has no per-utterance bias, takes the layer kernel's split-K path: one reduction more
            fewer = 1 if T == 1 else 2
            assert nat.last_launches == dense.last_launches - fewer, (B, T, nat.last_launches, dense.last_launches)
            if B == 3:
                for i in range(B):
                    assert torch.equal(nat.extract(x[i:i + 1].contiguous())[0], a[i]), (case, T, i)


def test_shard_calls_on_two_lanes_equal_per_batch_calls():
    m = _model("launcher")
    ex = m.extractor()
    feats = torch.from_numpy(onn.synthetic_feats(160, 120, 80, 78)).to(DEV)
    shard = ex.extract_shard(feats, batch=64)
    per = torch.cat([ex.extract(feats[i:i + 64].contiguous()) for i in range(0, 160, 64)])
    torch.cuda.synchronize()
    assert torch.equal(shard, per)
    host = np.empty((160, 192), dtype=np.float32)
    pinned = feats.cpu().pin_memory()
    ex.extract_shard_host(pinned.data_ptr(), 160, 120, host.ctypes.data, batch=64)
    assert np.array_equal(host, per.cpu().numpy())


def test_xvbe0003_round_trip_layout_and_rejections(tmp_path):
    from asv_subtools_b200 import _lib
    m = _model("fc1", "near")
    ex = m.extractor()
    path = str(tmp_path / "lawlict.xvbm")
    ex.save(path)
    raw = open(path, "rb").read()
    # magic | feat_dim, channels, mfa_dim, att_hidden, embed_dim, n_layers | global_context | f32 floor
    assert raw[:8] == b"XVBE0003"
    head = struct.unpack("<7i", raw[8:36])
    recs = bp.native_records(m)
    assert head == (80, 512, 1536, 128, 192, len(recs), 0)
    assert struct.unpack("<f", raw[36:40])[0] == np.float32(1e-9)
    name_len = struct.unpack("<i", raw[40:44])[0]
    assert raw[44:44 + name_len] == b"layer1"
    feats = torch.from_numpy(onn.synthetic_feats(3, 90, 80, 10)).to(DEV)
    loaded = etx.NativeEcapaExtractor.load(path)
    assert torch.equal(loaded.extract(feats), ex.extract(feats))
    again = str(tmp_path / "again.xvbm")
    loaded.save(again)
    assert open(again, "rb").read() == raw
    default_floor = struct.pack("<if", 1, 1e-5)
    for name, data in (("trunc", raw[:len(raw) // 2]), ("trunc_header", raw[:38]), ("magic", b"XVBE0004" + raw[8:]),
                       ("form", raw[:32] + struct.pack("<i", 2) + raw[36:]),
                       ("floor", raw[:36] + struct.pack("<f", 0.0) + raw[40:]),
                       ("default", raw[:32] + default_floor + raw[40:]),
                       ("global", raw[:32] + struct.pack("<i", 1) + raw[36:])):   # global context without att_gs
        bad = str(tmp_path / name)
        open(bad, "wb").write(data)
        with pytest.raises(_lib.XvbError):
            etx.NativeEcapaExtractor.load(bad)
    # the dense model still writes XVBE0001
    dense = str(tmp_path / "dense.xvbm")
    _dense(512).extractor().save(dense)
    assert open(dense, "rb").read(8) == b"XVBE0001"


def test_set_attention_refusals():
    """set_attention is refused after set_mqmha, set_chained or a set_layer, and set_mqmha / set_chained after it;
    finalize refuses an att_gs record without global context."""
    from asv_subtools_b200 import _lib
    lib = _lib.lib

    def fresh():
        h = ctypes.c_void_p()
        assert lib.xvb_ecapa_create(ctypes.byref(h), 80, 512, 1536, 512, 192) == 0
        return h

    for first, second in ((lambda h: lib.xvb_ecapa_set_mqmha(h, 2, 2, 128, 0, 2, 1, 1),
                           lambda h: lib.xvb_ecapa_set_attention(h, 0, 1e-9)),
                          (lambda h: lib.xvb_ecapa_set_chained(h, 1), lambda h: lib.xvb_ecapa_set_attention(h, 0, 1e-9)),
                          (lambda h: lib.xvb_ecapa_set_attention(h, 0, 1e-9),
                           lambda h: lib.xvb_ecapa_set_mqmha(h, 2, 2, 128, 0, 2, 1, 1)),
                          (lambda h: lib.xvb_ecapa_set_attention(h, 0, 1e-9), lambda h: lib.xvb_ecapa_set_chained(h, 1))):
        h = fresh()
        try:
            assert first(h) == 0
            assert second(h) != 0
        finally:
            lib.xvb_ecapa_destroy(h)
    h = fresh()
    try:
        for gc, floor in ((2, 1e-9), (0, 0.0), (0, 1.5)):
            assert lib.xvb_ecapa_set_attention(h, gc, floor) != 0
    finally:
        lib.xvb_ecapa_destroy(h)

    m = _model("launcher")
    recs = bp.native_records(m)
    extra = ("att_gs", np.zeros((128, 3072, 1), np.float32), np.zeros(128, np.float32), [0], None, None, False)
    m.native_records = lambda: recs + [extra]
    with pytest.raises(_lib.XvbError, match="att_gs"):
        etx.NativeEcapaExtractor(m, DEV)


def test_xvb_extract_and_python_cli_on_a_launcher_model(tmp_path):
    """XVBE0003 file -> bin/xvb-extract, including an utterance past the default --max-chunk 10000, against the oracle;
    --mixed-lengths refuses the file; the Python CLI on an nnet.config naming subtools/pytorch/model/ecapa-tdnn-xvector.py
    with the launcher's creation string (--blueprint-dir) gives the same vectors."""
    from asv_subtools_b200 import kaldi_io
    m = _model("launcher")
    model = str(tmp_path / "launcher.xvbm")
    m.extractor().save(model)
    lens = {"a": 300, "b": 300, "c": 37, "d": 1, "e": 129}
    feats = {k: onn.synthetic_feats(1, t, 80, 700 + i)[0] for i, (k, t) in enumerate(lens.items())}
    feats["long"] = lo.utterances("launcher", 10050)[0]
    ark = str(tmp_path / "feats.ark")
    with open(ark, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    out = str(tmp_path / "xv.ark")
    run = subprocess.run([BIN, "--batch", "4", model, ark, "ark:" + out], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(got) == sorted(feats)
    assert rel(got["long"][None], GOLD["launcher_near_T10050"]) <= 1e-4
    sd = lo.state_dict("launcher")
    for k, v in feats.items():
        want = lo.extract_embedding(sd, v, lo.LAUNCHER).numpy()
        assert got[k].shape == (192,) and rel(got[k], want) <= 1e-4, k
        assert rel(got[k], m.extract_embedding(v).numpy()) <= 1e-5, k
    run = subprocess.run([BIN, "--mixed-lengths", model, ark, "ark:" + out], capture_output=True, text=True, timeout=300)
    assert run.returncode == 1 and "ERROR" in run.stderr
    torch.save(dict(sd, **{"loss.weight": torch.zeros(1211, 192, 1)}), str(tmp_path / "final.params"))
    creation = lo.creation_string(dict(lo.LAUNCHER, training=True))
    (tmp_path / "nnet.config").write_text('model_blueprint;subtools/pytorch/model/ecapa-tdnn-xvector.py\nmodel_creation;"{}"\n'
                                          .format(creation.replace('"', '""')))
    cli = str(tmp_path / "cli.ark")
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--nnet-config",
                        str(tmp_path / "nnet.config"), "--blueprint-dir", os.path.join(ROOT, "asv_subtools_b200", "model"),
                        "--batch-size", "2", str(tmp_path / "final.params"), "ark:" + ark, "ark:" + cli],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    py = dict(kaldi_io.read_vec_flt_ark(cli))
    assert sorted(py) == sorted(feats)
    for k in feats:
        assert rel(py[k], got[k]) <= 1e-5, k
