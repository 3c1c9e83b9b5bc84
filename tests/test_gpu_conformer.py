"""Conformer x-vector on the GPU: each new kernel against torch fp32, the swish epilogue, the unpadded conv, the reference's
golden embeddings through the blueprint, batch vs per-utterance calls (one chunk and several) and the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conformer_oracle as co
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLUEPRINT = os.path.join(ROOT, "asv_subtools_b200", "model", "transformer_xvector.py")


@pytest.fixture(scope="module")
def ops():
    from asv_subtools_b200 import ops as o
    return o


@pytest.fixture(autouse=True)
def _no_tf32():
    """The torch references below run in fp32 (or float64), never TF32."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _t(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x


@pytest.mark.parametrize("C", [128, 256, 1536, 3072])
@pytest.mark.parametrize("mode", ["plain", "residual", "table_second_swish", "noaffine_tanh"])
def test_layer_norm_vs_torch(ops, C, mode):
    from asv_subtools_b200._lib import ACT_SWISH, ACT_TANH
    torch.manual_seed(C)
    B, T = 3, 37
    x = torch.randn(B, T, C, device="cuda") * 3 + 0.5
    ln = lambda z, *a: F.layer_norm(z.double(), (C,), *[None if t is None else t.double() for t in a], 1e-5)  # noqa: E731
    g, b = 1 + 0.1 * torch.randn(C, device="cuda"), 0.1 * torch.randn(C, device="cuda")
    g2, b2 = 1 + 0.1 * torch.randn(C, device="cuda"), 0.1 * torch.randn(C, device="cuda")
    d = torch.randn(B, T, 2 * C, device="cuda")[..., :C]        # a view with pitch 2C
    tab = torch.randn(T, C, device="cuda")
    y = ops.SplitPlanes.empty((B, T, C), "cuda")
    yf = torch.empty(B, T, C, device="cuda")
    r = x.clone()
    if mode == "plain":
        ops.layer_norm(r, g, b, y=y, y_f32=yf)
        v, ref = x, ln(x, g, b)
    elif mode == "residual":
        ops.layer_norm(r, g, b, delta=d, delta_scale=0.5, x_out=r, y=y, y_f32=yf)
        v = x + 0.5 * d
        ref = ln(v, g, b)
    elif mode == "table_second_swish":
        ops.layer_norm(r, g, b, table=tab, delta=d, x_out=r, second=(g2, b2), act=ACT_SWISH, y=y, y_f32=yf)
        v = ln(x + tab + d, g, b)
        ref = F.silu(ln(v.float(), g2, b2))
    else:
        ops.layer_norm(r, act=ACT_TANH, y=y, y_f32=yf)
        v, ref = x, torch.tanh(ln(x, None, None))
    assert rel(_t(yf), _t(ref)) <= 2e-6, rel(_t(yf), _t(ref))
    assert rel(_t(y.float()), _t(ref)) <= 3e-5
    assert rel(_t(r), _t(v)) <= 1e-6


def _attn_ref(qkv, H, dk, rope, rope_v, mult):
    B, T, _ = qkv.shape
    D = H * dk
    q, k, v = (qkv[..., i * D:(i + 1) * D].reshape(B, T, H, dk).transpose(1, 2).double() for i in range(3))
    if rope is not None:
        r = rope.double()
        q, k = co._rotary(q, r), co._rotary(k, r)
        if rope_v:
            v = co._rotary(v, r)
    s = torch.matmul(q, k.transpose(-2, -1)) / np.sqrt(dk) * mult
    return torch.matmul(torch.softmax(s, -1), v).transpose(1, 2).reshape(B, T, D)


@pytest.mark.parametrize("T", [1, 8, 74, 98, 240])
@pytest.mark.parametrize("norm", ["softmax", "softmax_plus"])
@pytest.mark.parametrize("rot", ["rope_v", "rope", "none"])
def test_rope_attention_vs_torch(ops, T, norm, rot):
    from asv_subtools_b200.model.transformer_xvector import rotary_table, softmax_plus_multiplier
    torch.manual_seed(T)
    B, H, dk = 3, 4, 64
    qkv = torch.randn(B, T, 3 * H * dk, device="cuda") * 2
    rope = rotary_table(dk)[:T].cuda() if rot != "none" else None
    mult = softmax_plus_multiplier(T, torch.tensor(5.7)) if norm == "softmax_plus" else 1.0
    y = ops.SplitPlanes.empty((B, T, H * dk), "cuda")
    ops.rope_attention(qkv, H, dk, y, rope=rope, rope_v=rot == "rope_v", score_mult=mult)
    ref = _attn_ref(qkv, H, dk, rope, rot == "rope_v", mult)
    assert rel(_t(y.float()), _t(ref)) <= 1e-5, rel(_t(y.float()), _t(ref))


@pytest.mark.parametrize("dk", [32, 128])
def test_rope_attention_other_head_sizes(ops, dk):
    from asv_subtools_b200.model.transformer_xvector import rotary_table
    torch.manual_seed(dk)
    B, T, H = 2, 41, 2
    qkv = torch.randn(B, T, 3 * H * dk + 8, device="cuda")[..., :3 * H * dk]    # row pitch > 3 H dk
    rope = rotary_table(dk)[:T].cuda()
    y = ops.SplitPlanes.empty((B, T, H * dk), "cuda")
    ops.rope_attention(qkv, H, dk, y, rope=rope, rope_v=True)
    assert rel(_t(y.float()), _t(_attn_ref(qkv, H, dk, rope, True, 1.0))) <= 1e-5


@pytest.mark.parametrize("C,K,T,bn,act", [(256, 15, 74, False, "swish"), (128, 15, 8, True, "relu"), (256, 15, 1, False, "swish"),
                                          (512, 31, 40, False, "swish"), (128, 3, 17, True, "swish")])
def test_conv_module_vs_torch(ops, C, K, T, bn, act):
    from asv_subtools_b200._lib import ACT_RELU, ACT_SWISH
    torch.manual_seed(C + K + T)
    B = 3
    x = torch.randn(B, T, 2 * C, device="cuda")
    w, b = torch.randn(C, K, device="cuda") / np.sqrt(K), 0.1 * torch.randn(C, device="cuda")
    na, nb = 1 + 0.1 * torch.randn(C, device="cuda"), 0.1 * torch.randn(C, device="cuda")
    y = ops.SplitPlanes.empty((B, T, C), "cuda")
    ops.conv_module(x, w, b, na, nb, y, batch_norm=bn, act=ACT_SWISH if act == "swish" else ACT_RELU)
    z = F.conv1d(F.glu(x.transpose(1, 2).double(), dim=1), w.unsqueeze(1).double(), b.double(), padding=K // 2, groups=C)
    na, nb = na.double(), nb.double()
    z = z * na[:, None] + nb[:, None] if bn else F.layer_norm(z.transpose(1, 2), (C,), na, nb, 1e-5).transpose(1, 2)
    ref = (F.silu(z) if act == "swish" else F.relu(z)).transpose(1, 2)
    assert rel(_t(y.float()), _t(ref)) <= 3e-5, rel(_t(y.float()), _t(ref))


@pytest.mark.parametrize("T,F_,C", [(300, 80, 256), (7, 80, 256), (150, 23, 128), (9, 3, 16)])
def test_subsample_head_vs_torch(ops, T, F_, C):
    torch.manual_seed(T)
    B = 2
    x = torch.randn(B, T, F_, device="cuda")
    w, b = torch.randn(C, 1, 3, 3, device="cuda") / 3, 0.1 * torch.randn(C, device="cuda")
    y = ops.SplitPlanes.empty((B, (T - 1) // 2, (F_ - 1) // 2, C), "cuda")
    ops.subsample_head(x, w, b, y)
    ref = F.relu(F.conv2d(x.unsqueeze(1).double(), w.double(), b.double(), stride=2)).permute(0, 2, 3, 1)
    assert rel(_t(y.float()), _t(ref)) <= 3e-5, rel(_t(y.float()), _t(ref))


@pytest.mark.parametrize("T,F_,C,stride", [(149, 39, 256, 2), (3, 3, 256, 2), (74, 11, 128, 2), (12, 10, 64, 2),
                                           (20, 9, 32, 1)])
def test_unpadded_conv_vs_torch(ops, T, F_, C, stride):
    torch.manual_seed(T + C)
    B = 3
    x = torch.relu(torch.randn(B, T, F_, C, device="cuda"))
    w = torch.randn(C, C, 3, 3, device="cuda") / np.sqrt(9 * C)       # (Cout, Cin, kf, kt): the kernel's tap order
    bias = 0.1 * torch.randn(C, device="cuda")
    xp = ops.split_f32(x.contiguous())
    xf = xp.float()
    To, Fo = (T - 3) // stride + 1, (F_ - 3) // stride + 1
    y = ops.SplitPlanes.empty((B, To, Fo, C), "cuda")
    yv = torch.empty(B, To, Fo, C, device="cuda")
    ops.conv2d(xp, ops.pack_conv2d_weight(w), C, 3, stride, torch.ones(C, device="cuda"), bias, relu=True, y=y, y_f32=yv,
               valid=True)
    # the reference convolves (B, C, F, T) layout here: H = F (kf), W = T (kt)
    ref = F.relu(F.conv2d(xf.permute(0, 3, 2, 1).double(), w.double(), bias.double(), stride=stride)).permute(0, 3, 2, 1)
    assert ref.shape == yv.shape
    assert rel(_t(yv), _t(ref)) <= 3e-5, rel(_t(yv), _t(ref))
    assert rel(_t(y.float()), _t(ref)) <= 3e-5


def test_unpadded_conv_writes_nothing_past_its_outputs(ops):
    """Outputs a padded conv would add at the far edges (T - 1 odd) are not written."""
    B, T, F_, C = 2, 10, 8, 64
    x = ops.split_f32(torch.randn(B, T, F_, C, device="cuda").contiguous())
    w = ops.pack_conv2d_weight(torch.randn(C, C, 3, 3, device="cuda") / 30)
    To, Fo = (T - 3) // 2 + 1, (F_ - 3) // 2 + 1
    buf = torch.full((B * To * Fo * C + 4096,), 7.0, device="cuda")
    ops.conv2d(x, w, C, 3, 2, torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), relu=True,
               y_f32=buf[:B * To * Fo * C].view(B, To, Fo, C), valid=True)
    assert bool((buf[B * To * Fo * C:] == 7.0).all())


@pytest.mark.parametrize("bn", [False, True])
def test_swish_epilogue_vs_torch(ops, bn):
    torch.manual_seed(5)
    B, T, cin, cout = 3, 74, 256, 512
    x = torch.randn(B, T, cin, device="cuda")
    w = torch.randn(cout, cin, device="cuda") / 16
    b = torch.randn(cout, device="cuda")
    s, t = (1 + 0.1 * torch.randn(cout, device="cuda"), 0.1 * torch.randn(cout, device="cuda")) if bn else (None, None)
    xp = ops.split_f32(x)
    y = torch.empty(B, T, cout, device="cuda")
    ops.tdnn_affine_ex(xp, ops.pack_tdnn_weight(w.unsqueeze(-1).contiguous(), [0]), cout, [0], bias=b, bn_scale=s,
                       bn_shift=t, swish=True, y_f32=y)
    ref = F.silu(xp.float().double() @ w.T.double() + b.double())
    if bn:
        ref = ref * s.double() + t.double()
    assert rel(_t(y), _t(ref)) <= 3e-5, rel(_t(y), _t(ref))


def _model(case, pos):
    from asv_subtools_b200.model.transformer_xvector import TransformerXvector
    kwargs, fdim, _, _, seed, _ = co.CASES[case]
    m = TransformerXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(co.seeded_state_dict(np.load(os.path.join(ROOT, "tests", "golden", "conformer.npz"))["keys_" + case],
                                           seed), strict=True)
    return m.cuda().eval()


GOLDEN_CASES = [(case, pos, t) for case, (_, _, frames, positions, _, _) in sorted(co.CASES.items())
                for pos in positions for t in frames]


@pytest.mark.parametrize("case,pos,t", GOLDEN_CASES)
def test_embeddings_match_reference_golden(golden, case, pos, t):
    _, fdim, _, _, _, fseed = co.CASES[case]
    feats = onn.synthetic_feats(2, t, fdim, fseed + t)
    ref = golden("conformer")["{}_{}_T{}".format(case, pos, t)]
    got = np.stack([_model(case, pos).extract_embedding(feats[i]).numpy() for i in range(2)])
    cos = np.sum(got * ref, 1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
    print("conformer {} {} T={}: rel {:.3e}, 1 - cos {:.3e}".format(case, pos, t, rel(got, ref), 1 - cos.min()))
    assert rel(got, ref) <= 1e-4 and cos.min() >= 1 - 1e-6, (case, pos, t, rel(got, ref), cos)


def test_batch_equals_single_utterance_calls():
    m = _model("launcher", "near")
    feats = onn.synthetic_feats(64, 300, 80, 77)
    batch = m.extract_embedding_batch(feats).cpu().numpy()
    single = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(64)])
    print("conformer batch vs single: rel {:.3e}".format(rel(batch, single)))
    assert rel(batch, single) <= 2e-6


@pytest.mark.parametrize("case,t", [("launcher", 899), ("small", 650), ("rotv", 1211)])
def test_multi_chunk_batch_equals_single_utterance_calls(case, t):
    _, fdim, _, positions, _, _ = co.CASES[case]
    m = _model(case, positions[-1])
    feats = onn.synthetic_feats(5, t, fdim, 31)
    batch = m.extract_embedding_batch(feats).cpu().numpy()
    single = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(5)])
    print("conformer multi-chunk batch vs single ({}, T={}): rel {:.3e}".format(case, t, rel(batch, single)))
    assert rel(batch, single) <= 2e-6


def test_extract_embeddings_cli_with_blueprint_dir(tmp_path):
    """A reference-style model dir (nnet.config naming the reference's transformer_xvector.py and a launcher-style
    creation string) extracts through the CLI with --blueprint-dir: one FV per key, equal to the per-utterance
    embeddings, which point the same way as the torch restatement's."""
    from asv_subtools_b200 import kaldi_io
    from asv_subtools_b200.pipeline.extract_embeddings import create_model_from_py
    creation = co.creation(co.LAUNCHER, 80, "near").replace("training=False", "training=True", 1)
    keys = np.load(os.path.join(ROOT, "tests", "golden", "conformer.npz"))["keys_launcher"]
    sd = co.seeded_state_dict(keys, 401)
    torch.save(sd, str(tmp_path / "final.params"))
    (tmp_path / "nnet.config").write_text('model_blueprint;subtools/pytorch/model/transformer_xvector.py\nmodel_creation;"{}"\n'
                                          .format(creation.replace('"', '""')))
    rng = np.random.RandomState(12)
    feats = {"utt{}".format(i): rng.standard_normal((t, 80)).astype(np.float32) for i, t in enumerate([50, 50, 23, 7, 620])}
    with open(tmp_path / "feats.ark", "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = str(tmp_path / "dir.ark")
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--nnet-config",
                        str(tmp_path / "nnet.config"), "--blueprint-dir", os.path.join(ROOT, "asv_subtools_b200", "model"),
                        "--batch-size", "4", str(tmp_path / "final.params"), "ark:" + str(tmp_path / "feats.ark"), "ark:" + out],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(got) == sorted(feats) and open(out, "rb").read().count(b"FV ") == len(feats)
    m = create_model_from_py(BLUEPRINT, creation)
    m.load_state_dict(sd, strict=False)
    m.cuda().eval()
    cfg = co.config(co.LAUNCHER)
    for k, v in feats.items():
        one = m.extract_embedding(v).numpy()
        ref = co.extract(sd, v, cfg, "near").numpy()
        assert rel(got[k], one) <= 1e-6, k
        assert np.dot(one, ref) / (np.linalg.norm(one) * np.linalg.norm(ref)) >= 1 - 1e-6, k
