"""ResNet x-vector on the H100: the 2-D conv kernel, the head conv and the SE scaling against torch-CPU, then whole
embeddings against the reference's golden outputs (tests/golden/resnet.npz), the batched call and the extraction CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resnet_oracle as ro
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLUEPRINT = os.path.join(ROOT, "asv_subtools_b200", "model", "resnet_xvector.py")
# pytorch/launcher/runResnetXvector_online.py:221-275, rewritten with training=False and extracted_embedding="near"
ONLINE_CREATION = (
    'ResNetXvector(80,1211,aug_dropout=0.0,tail_dropout=0.0,training=False,extracted_embedding="near",'
    'resnet_params={"head_conv":True,"head_conv_params":{"kernel_size":3,"stride":1,"padding":1},"head_maxpool":False,'
    '"head_maxpool_params":{"kernel_size":3,"stride":2,"padding":1},"block":"BasicBlock","layers":[3,4,6,3],'
    '"planes":[32,64,128,256],"use_se":True,"se_ratio":4,"convXd":2,"norm_layer_params":{"momentum":0.5,"affine":True},'
    '"full_pre_activation":False,"zero_init_residual":False},pooling="statistics",pooling_params={"num_head":16,'
    '"share":True,"affine_layers":1,"hidden_size":64,"context":[0],"stddev":True,"temperature":False,"fixed":True},'
    'fc1=False,fc1_params={"nonlinearity":"relu","nonlinearity_params":{"inplace":True},"bn-relu":False,"bn":True,'
    '"bn_params":{"momentum":0.5,"affine":False,"track_running_stats":True}},fc2_params={"nonlinearity":"",'
    '"nonlinearity_params":{"inplace":True},"bn-relu":False,"bn":True,"bn_params":{"momentum":0.5,"affine":False,'
    '"track_running_stats":True}},margin_loss=True,margin_loss_params={"method":"am","m":0.2,"feature_normalize":True,'
    '"s":30,"mhe_loss":False,"mhe_w":0.01},use_step=True,step_params={"margin_warm":False,"margin_warm_conf":'
    '{"start_epoch":1,"end_epoch":1,"offset_margin":-0.0,"init_lambda":1.0},"T":None,"m":True,"lambda_0":0,'
    '"lambda_b":1000,"alpha":5,"gamma":1e-4,"s":False,"s_tuple":(30,12),"s_list":None,"t":False,"t_tuple":(0.5,1.2),'
    '"p":False,"p_tuple":(0.5,0.1)})')


@pytest.fixture(scope="module")
def ops():
    from asv_subtools_b200 import ops as o
    return o


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def planes_of(ops, x):
    """fp32 CUDA (..., C) -> SplitPlanes and the fp32 values the planes hold (what the kernel multiplies)."""
    p = ops.split_f32(x.contiguous())
    return p, p.float()


def ref_conv(xv, w, stride, k):
    """F.conv2d in float64 on the (B, T, F, C) layout: the reference's (B, C, F, T) convolution."""
    x = xv.double().cpu().permute(0, 3, 2, 1)
    y = F.conv2d(x, w.double().cpu(), stride=stride, padding=k // 2)
    return y.permute(0, 3, 2, 1)


# (Cin, Cout, k, stride, F, T, B): output F' in {80, 40, 23, 12, 10, 3}, T in {1, 2, 7, 200}, B in {1, 5, 64}
CONV_CASES = [
    (32, 32, 3, 1, 80, 200, 5),
    (32, 64, 3, 2, 80, 7, 64),
    (32, 64, 1, 2, 80, 7, 64),
    (64, 128, 3, 1, 23, 2, 5),
    (64, 128, 3, 2, 23, 200, 1),
    (64, 128, 1, 2, 23, 200, 1),
    (128, 256, 3, 2, 20, 1, 64),
    (128, 256, 1, 2, 6, 7, 5),
    (128, 256, 3, 1, 3, 200, 5),
    (32, 32, 3, 1, 12, 1, 1),
    (64, 128, 3, 2, 45, 7, 5),
]


@pytest.mark.parametrize("cin, cout, k, stride, fdim, t, b", CONV_CASES)
def test_conv2d_kernel_vs_torch(ops, cin, cout, k, stride, fdim, t, b):
    g = torch.Generator().manual_seed(cin * 1000 + fdim + t)
    x = torch.randn(b, t, fdim, cin, generator=g).cuda()
    w = (torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5).cuda()
    xp, xv = planes_of(ops, x)
    to, fo = (t - 1) // stride + 1, (fdim - 1) // stride + 1
    y = ops.SplitPlanes.empty((b, to, fo, cout), "cuda")
    yf = torch.empty(b, to, fo, cout, device="cuda")
    ops.conv2d(xp, ops.pack_conv2d_weight(w), cout, k, stride, y=y, y_f32=yf)
    ref = ref_conv(xv, w, stride, k)
    assert tuple(ref.shape) == (b, to, fo, cout)
    assert rel(yf.cpu(), ref) <= 3e-5
    assert rel(y.float().cpu(), ref) <= 3e-5


@pytest.mark.parametrize("relu", [False, True])
def test_conv2d_epilogues_bn_residual_relu_second_output(ops, relu):
    """y = [relu](conv * scale + shift + res); y2 = relu(y * scale2 + shift2) (the pre-activation hand-over)."""
    g = torch.Generator().manual_seed(7)
    b, t, fdim, cin, cout = 5, 37, 23, 64, 128
    x = torch.randn(b, t, fdim, cin, generator=g).cuda()
    w = (torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5).cuda()
    res = torch.randn(b, 19, 12, cout, generator=g).cuda()
    sc, sh, sc2, sh2 = (torch.rand(cout, generator=g).cuda() + 0.5, 0.1 * torch.randn(cout, generator=g).cuda(),
                        torch.rand(cout, generator=g).cuda() + 0.5, 0.3 * torch.randn(cout, generator=g).cuda())
    xp, xv = planes_of(ops, x)
    rp, rv = planes_of(ops, res)
    y, y2 = ops.SplitPlanes.empty((b, 19, 12, cout), "cuda"), ops.SplitPlanes.empty((b, 19, 12, cout), "cuda")
    yf = torch.empty(b, 19, 12, cout, device="cuda")
    ops.conv2d(xp, ops.pack_conv2d_weight(w), cout, 3, 2, sc, sh, res=rp, relu=relu, y=y, y_f32=yf, scale2=sc2, shift2=sh2, y2=y2)
    ref = ref_conv(xv, w, 2, 3) * sc.double().cpu() + sh.double().cpu() + rv.double().cpu()
    if relu:
        ref = ref.clamp(min=0)
    ref2 = (ref * sc2.double().cpu() + sh2.double().cpu()).clamp(min=0)
    assert rel(yf.cpu(), ref) <= 3e-5 and rel(y.float().cpu(), ref) <= 3e-5
    assert rel(y2.float().cpu(), ref2) <= 3e-5


def test_head_conv_vs_oracle(ops):
    g = torch.Generator().manual_seed(3)
    b, t, fdim = 3, 41, 23
    x = torch.randn(b, t, fdim, generator=g)
    w = torch.randn(32, 1, 3, 3, generator=g) * 0.5
    sc, sh, sc2, sh2 = torch.rand(32, generator=g) + 0.5, 0.1 * torch.randn(32, generator=g), \
        torch.rand(32, generator=g) + 0.5, 0.2 * torch.randn(32, generator=g)
    y, y2 = ops.SplitPlanes.empty((b, t, fdim, 32), "cuda"), ops.SplitPlanes.empty((b, t, fdim, 32), "cuda")
    ops.conv2d_head(x.cuda(), w.cuda(), sc.cuda(), sh.cuda(), y, sc2.cuda(), sh2.cuda(), y2)
    ref = F.relu(F.conv2d(x.double().transpose(1, 2).unsqueeze(1), w.double(), padding=1) * sc.double()[:, None, None] +
                 sh.double()[:, None, None]).permute(0, 3, 2, 1)
    assert rel(y.float().cpu(), ref) <= 1e-5
    assert rel(y2.float().cpu(), (ref * sc2.double() + sh2.double()).clamp(min=0)) <= 1e-5


@pytest.mark.parametrize("relu", [False, True])
def test_se_residual_vs_oracle(ops, relu):
    g = torch.Generator().manual_seed(5)
    b, t, fdim, c = 4, 9, 10, 64
    z, ident = torch.randn(b, t, fdim, c, generator=g).cuda(), torch.randn(b, t, fdim, c, generator=g).cuda()
    gate = torch.rand(b, c, generator=g).cuda()
    sc2, sh2 = torch.rand(c, generator=g).cuda() + 0.5, 0.2 * torch.randn(c, generator=g).cuda()
    zp, zv = planes_of(ops, z)
    ip, iv = planes_of(ops, ident)
    y, y2 = ops.SplitPlanes.empty((b, t, fdim, c), "cuda"), ops.SplitPlanes.empty((b, t, fdim, c), "cuda")
    yf = torch.empty(b, t, fdim, c, device="cuda")
    ops.se_residual(zp, gate, ip, relu=relu, y=y, y_f32=yf, scale2=sc2, shift2=sh2, y2=y2)
    ref = zv * gate[:, None, None, :] + iv
    if relu:
        ref = ref.clamp(min=0)
    assert torch.equal(yf, ref)                                     # the reference's rounding: mul, then add
    assert rel(y.float().cpu(), ref.cpu()) <= 1e-5
    assert rel(y2.float().cpu(), (ref * sc2 + sh2).clamp(min=0).cpu()) <= 1e-5


def _model(case, pos):
    from asv_subtools_b200.model.resnet_xvector import ResNetXvector
    kwargs, fdim, _, _, seed, _ = ro.CASES[case]
    m = ResNetXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed), strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("case, pos", [(c, p) for c in sorted(ro.CASES) for p in ro.CASES[c][3]])
def test_embeddings_match_reference_golden(golden, case, pos):
    g = golden("resnet")
    _, fdim, frames, _, _, fseed = ro.CASES[case]
    m = _model(case, pos)
    for t in frames:
        feats = onn.synthetic_feats(2, t, fdim, fseed + t)
        ref = g["{}_{}_T{}".format(case, pos, t)]
        got = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(2)])
        cos = np.sum(got * ref, 1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
        print("resnet {} {} T={}: rel {:.3e}, 1 - cos {:.3e}".format(case, pos, t, rel(got, ref), 1 - cos.min()))
        assert rel(got, ref) <= 1e-4 and cos.min() >= 1 - 1e-6, (case, pos, t, rel(got, ref), cos)


def test_batch_equals_single_utterance_calls():
    """extract_embedding_batch on 64 x 200 frames equals 64 extract_embedding calls to rounding, not bit for bit: the conv
    kernel's tile shape (utterances x frames x bins per tile, N width) follows the batch size, which can move the last
    bit (measured on an H100: max |delta| ~1e-6 on embedding entries of magnitude ~4)."""
    m = _model("online", "near")
    feats = onn.synthetic_feats(64, 200, 80, 77)
    batch = m.extract_embedding_batch(feats).cpu().numpy()
    single = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(64)])
    assert rel(batch, single) <= 1e-6


def test_extract_embeddings_cli_with_online_creation_and_blueprint_dir(tmp_path):
    """A reference-style model dir (nnet.config naming the reference's resnet_xvector.py and the online launcher's
    creation string) extracts through the CLI with --blueprint-dir, and --model-blueprint / --model-creation gives the
    same vectors: one FV per key, equal to the per-utterance embeddings."""
    from asv_subtools_b200 import kaldi_io
    from asv_subtools_b200.pipeline.extract_embeddings import create_model_from_py
    sd = onn.make_state_dict(ro.resnet_spec(80, ro.ONLINE), 301)
    torch.save(sd, str(tmp_path / "final.params"))
    (tmp_path / "nnet.config").write_text('model_blueprint;subtools/pytorch/model/resnet_xvector.py\nmodel_creation;"{}"\n'
                                          .format(ONLINE_CREATION.replace('"', '""')))
    rng = np.random.RandomState(11)
    feats = {"utt{}".format(i): rng.standard_normal((t, 80)).astype(np.float32) for i, t in enumerate([50, 50, 23, 1, 120])}
    with open(tmp_path / "feats.ark", "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    env = dict(os.environ, PYTHONPATH=ROOT)
    outs = {}
    for name, flags in (("dir", ["--nnet-config", str(tmp_path / "nnet.config"), "--blueprint-dir",
                                 os.path.join(ROOT, "asv_subtools_b200", "model")]),
                        ("bp", ["--model-blueprint", BLUEPRINT, "--model-creation", ONLINE_CREATION])):
        out = str(tmp_path / (name + ".ark"))
        r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings"] + flags +
                           ["--batch-size", "4", str(tmp_path / "final.params"), "ark:" + str(tmp_path / "feats.ark"),
                            "ark:" + out], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        outs[name] = dict(kaldi_io.read_vec_flt_ark(out))
        raw = open(out, "rb").read()
        assert raw.count(b"FV ") == len(feats)
    m = create_model_from_py(BLUEPRINT, ONLINE_CREATION)
    m.load_state_dict(sd, strict=False)
    m.cuda().eval()
    for k, v in feats.items():
        one = m.extract_embedding(v).numpy()
        with torch.no_grad():
            ref = ro.resnet_forward(sd, torch.from_numpy(v).T.unsqueeze(0), "near", ro.ONLINE).squeeze().numpy()
        for name in outs:
            assert sorted(outs[name]) == sorted(feats)
            assert rel(outs[name][k], one) <= 1e-6, (name, k)
        assert rel(one, ref) <= 1e-4, k
