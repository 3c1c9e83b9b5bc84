"""Masked batches of utterances of different lengths on the CAM++ x-vector (xvb_campp_extract_lengths and its op-by-op
twin CamPPExtractor): the masked CAM gate against float64 and against the unmasked gate of each utterance alone; every
row of a masked batch bit for bit its solo extraction, on the handle and the twin, handle == twin; what lies past an
utterance's end is never read, and the twin's workspace holds zeros there; all lengths equal to T is the unmasked call;
the frame budget; alternating masked and equal-length calls; bad lengths; the goldens packed into masked batches; and
xvb-extract / pipeline/extract_embeddings.py with --mixed-lengths on a CAM++ model.  Needs an H100 (`-m gpu`)."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import campplus_oracle as co  # noqa: E402
from asv_subtools_b200 import kaldi_io, ops  # noqa: E402
from asv_subtools_b200.model.campplus_xvector import (SEG_LEN, CamPPExtractor, CamPPXvector,  # noqa: E402
                                                      NativeCamPPExtractor, chunk_sizes)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(HERE)
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
GOLDEN = np.load(os.path.join(HERE, "golden", "campplus.npz"))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cosines(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.sum(a * b, -1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))


_MODELS = {}


def _sd(case):
    return co.seeded_state_dict(GOLDEN["keys_" + case], co.CASES[case][3])


def _model(case):
    if case not in _MODELS:
        kw = dict(co.CASES[case][0])
        m = CamPPXvector(kw.pop("inputs_dim"), 10, **kw)
        m.load_state_dict(_sd(case), strict=True)
        _MODELS[case] = m.cuda().eval()
    return _MODELS[case]


def _extractors(case="default"):
    """(handle, twin) on one model, each built directly so that the environment switch is not involved."""
    m = _model(case)
    return NativeCamPPExtractor(m), CamPPExtractor(m, torch.device("cuda"))


def _padded(rows, T, fill=0.0):
    x = np.full((len(rows), T, rows[0].shape[1]), fill, dtype=np.float32)
    for i, r in enumerate(rows):
        x[i, :r.shape[0]] = r
    return torch.from_numpy(x).cuda()


def _utterances(lens, fdim, seed):
    return [co.utterances(1, t, fdim, seed + i)[0].numpy() for i, t in enumerate(lens)]


# ------------------------------------------------------------------ 1. the masked gate against float64 and solo calls
def test_cam_gate_lengths_vs_float64_and_solo_calls():
    lens = [1, 2, 99, 100, 101, 150, 199, 200, 201, 2000]
    B, T, Cc, R, G = len(lens), 2000, 128, 64, 32
    nseg = (T + SEG_LEN - 1) // SEG_LEN
    g = torch.Generator().manual_seed(11)
    x = torch.relu(torch.randn(B, T, Cc, generator=g)).cuda()
    h = ops.split_f32(x)
    for b, L in enumerate(lens):       # poison what lies past each end, in both planes
        h.hi[b, L:] = float("nan")
        h.lo[b, L:] = float("nan")
    w1, b1 = (torch.randn(R, Cc, generator=g) / Cc ** 0.5).cuda(), (torch.randn(R, generator=g) * 0.1).cuda()
    w2, b2 = (torch.randn(G, R, generator=g) / R ** 0.5).cuda(), (torch.randn(G, generator=g) * 0.1).cuda()
    buf = torch.full(((B * nseg + 1) * G,), 7.0, device="cuda")    # one spare fenced row after the gate
    out = buf[:B * nseg * G].view(B, nseg, G)
    d_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ops.cam_gate(h, w1, b1, w2, b2, seg_len=SEG_LEN, out=out, lengths=d_lens)
    assert torch.equal(buf[B * nseg * G:], torch.full((G,), 7.0, device="cuda"))
    hv = ops.SplitPlanes(h.hi.clone(), h.lo.clone(), Cc)
    for b, L in enumerate(lens):
        hv.hi[b, L:] = 0
        hv.lo[b, L:] = 0
    hf = hv.float().double().cpu()
    W1, B1, W2, B2 = (t.double().cpu() for t in (w1, b1, w2, b2))
    got = out.cpu()
    for b, L in enumerate(lens):
        ns = (L + SEG_LEN - 1) // SEG_LEN
        u = hf[b, :L]
        ctx = torch.stack([u.mean(0) + u[s * SEG_LEN:(s + 1) * SEG_LEN].mean(0) for s in range(ns)])
        want = torch.sigmoid(torch.relu(ctx @ W1.T + B1) @ W2.T + B2)
        assert rel(got[b, :ns], want) <= 1e-5, (L, rel(got[b, :ns], want))
        assert torch.count_nonzero(got[b, ns:]) == 0, L
        # the unmasked gate of the utterance alone, T = L
        solo = ops.cam_gate(ops.SplitPlanes(h.hi[b:b + 1, :L].contiguous(), h.lo[b:b + 1, :L].contiguous(), Cc), w1, b1, w2,
                            b2, seg_len=SEG_LEN)
        assert torch.equal(got[b:b + 1, :ns], solo.cpu()), L
    with pytest.raises(RuntimeError, match="xvb_cam_gate_lengths: null lengths"):
        from asv_subtools_b200._lib import check, lib
        check(lib.xvb_cam_gate_lengths(h.hi.data_ptr(), h.lo.data_ptr(), Cc, B, T, Cc, SEG_LEN, w1.data_ptr(), b1.data_ptr(),
                                       R, w2.data_ptr(), b2.data_ptr(), G, None, out.data_ptr(), None),
              "xvb_cam_gate_lengths")


# ------------------------------------------------------------------ 2. rows against solo extraction, handle == twin
MIXED = [3, 4, 5, 199, 200, 201, 255, 256, 257, 300, 600]


def _mixed_lengths(n, seed):
    rng = np.random.RandomState(seed)
    lens = MIXED + [int(v) for v in rng.randint(3, 601, n - len(MIXED))]
    rng.shuffle(lens)
    return lens


def test_rows_equal_solo_extraction_on_handle_and_twin():
    native, twin = _extractors()
    lens = _mixed_lengths(64, 5)
    utts = _utterances(lens, 80, 3000)
    x = _padded(utts, max(lens))
    with torch.no_grad():
        got_n = native.extract(x, lengths=lens).clone()
        n_launch = native.last_launches
        got_t = twin.extract(x, lengths=lens).clone()
        assert twin.last_launches == n_launch
        assert torch.equal(got_n, got_t), (got_n - got_t).abs().max().item()
        for i, u in enumerate(utts):
            xs = torch.from_numpy(u[None]).cuda()
            solo_n, solo_t = native.extract(xs), twin.extract(xs)
            assert torch.equal(got_n[i], solo_n[0]), (i, lens[i], (got_n[i] - solo_n[0]).abs().max().item())
            assert torch.equal(got_t[i], solo_t[0]), (i, lens[i])


# ------------------------------------------------------------------ 3. padding is never read; the twin's zeros
def test_padding_is_never_read_and_the_twin_workspace_is_zero_past_each_end():
    native, twin = _extractors()
    lens = _mixed_lengths(19, 9)[:19]
    utts = _utterances(lens, 80, 4000)
    T = max(lens) + 7
    with torch.no_grad():
        want = native.extract(_padded(utts, T), lengths=lens).clone()
        for fill in (float("nan"), 1e30, -1e30):
            assert torch.equal(native.extract(_padded(utts, T, fill), lengths=lens), want), fill
            assert torch.equal(twin.extract(_padded(utts, T, fill), lengths=lens), want), fill
        torch.cuda.synchronize()
    ws = twin._ws
    L = torch.tensor(lens)
    L2 = (L + 1) // 2
    T2 = (T + 1) // 2
    nseg = (L2 + SEG_LEN - 1) // SEG_LEN

    def zero_past(t, ends, name, offset=0):
        t = t.cpu()
        for b, e in enumerate(ends.tolist()):
            assert torch.count_nonzero(t[b, offset + e:]) == 0, (name, b, e)

    planes = {k: v for k, v in ws.items() if isinstance(v, ops.SplitPlanes)}
    for name in [k for k in planes if k[0] in "xaosc"]:          # the FCM head, (B, T, F, 32)
        zero_past(planes[name].hi, L, name)
        zero_past(planes[name].lo, L, name)
    for p in (ws["pad"].hi, ws["pad"].lo):                           # (B, T + 4, row): 2 zero frames, then L frames
        zero_past(p, L, "pad", offset=2)
        assert torch.count_nonzero(p[:, :2].cpu()) == 0
    for name, p in [("buf%d" % i, q) for i, q in enumerate(ws["bufs"])] + [("h", ws["h"]), ("z", ws["z"])]:
        assert p.hi.shape[1] == T2
        zero_past(p.hi, L2, name)
        zero_past(p.lo, L2, name)
    zero_past(ws["pool_in"], L2, "pool_in")
    zero_past(ws["gate"], nseg, "gate")


# ------------------------------------------------------------------ 4. the unmasked path, the frame budget, refusals
@pytest.mark.parametrize("case", sorted(co.CASES))
def test_all_lengths_equal_T_is_the_unmasked_call(case):
    native, twin = _extractors(case)
    fdim = co.CASES[case][0]["inputs_dim"]
    with torch.no_grad():
        for b in (1, 3, 64):
            for t in (3, 37, 201):
                x = co.utterances(b, t, fdim, 10 * b + t).cuda()
                want = native.extract(x).clone()
                assert torch.equal(native.extract(x, lengths=[t] * b), want), (case, b, t)
                assert torch.equal(twin.extract(x, lengths=[t] * b), want), (case, b, t)


def test_masked_call_over_the_frame_budget_equals_per_utterance_calls():
    """40 utterances padded to 4000 frames run as groups of 9 (the 128 * 300 frame budget)."""
    native, _ = _extractors()
    rng = np.random.RandomState(17)
    lens = [4000, 3, 3999, 2001] + [int(v) for v in rng.randint(3, 4001, 36)]
    utts = _utterances(lens, 80, 5000)
    with torch.no_grad():
        whole = native.extract(_padded(utts, 4000), lengths=lens)
        for i, u in enumerate(utts):
            assert torch.equal(whole[i], native.extract(torch.from_numpy(u[None]).cuda())[0]), (i, lens[i])


def test_masked_and_equal_length_calls_alternate_on_one_workspace():
    native, twin = _extractors()
    a = co.utterances(8, 300, 80, 61).cuda()
    lens = [300, 3, 150, 299, 201, 4, 100, 77]
    utts = _utterances(lens, 80, 62)
    with torch.no_grad():
        for ex in (native, twin):
            plain = ex.extract(a).clone()
            masked = ex.extract(_padded(utts, 300), lengths=lens).clone()
            assert torch.equal(ex.extract(a), plain)
            assert torch.equal(ex.extract(_padded(utts, 300), lengths=lens), masked)
            small = co.utterances(3, 37, 80, 63).cuda()
            want = ex.extract(small).clone()
            ex.extract(_padded(utts, 300), lengths=lens)
            assert torch.equal(ex.extract(small), want)


def test_bad_lengths_are_refused_by_the_c_entry_and_python():
    native, twin = _extractors("small")
    x = torch.zeros(4, 30, 40, device="cuda")
    for lens, bad in (([30, 2, 5, 3], r"lengths\[1\]=2"), ([30, 30, 31, 3], r"lengths\[2\]=31"),
                      ([0, 3, 3, 3], r"lengths\[0\]=0")):
        with pytest.raises(RuntimeError, match="xvb_campp_extract_lengths: " + bad):
            native.extract(x, lengths=lens)
        with pytest.raises(ValueError, match=bad):
            twin.extract(x, lengths=lens)
    emb = torch.full((4, native.embed_dim), 7.0, device="cuda")
    arr = (C.c_int32 * 4)(5, 6, 2, 7)
    assert native._fn("extract_lengths")(native._h, C.c_void_p(x.data_ptr()), arr, 4, 30, C.c_void_p(emb.data_ptr()),
                                         native._stream()) == -1   # XVB_EINVAL, nothing launched
    assert native._fn("extract_lengths")(native._h, C.c_void_p(x.data_ptr()), None, 4, 30, C.c_void_p(emb.data_ptr()),
                                         native._stream()) == -1
    torch.cuda.synchronize()
    assert torch.equal(emb, torch.full_like(emb, 7.0))


# ------------------------------------------------------------------ 5. goldens packed into masked batches
@pytest.mark.parametrize("case", sorted(co.CASES))
def test_goldens_in_masked_batches(case):
    cfg, frames, long_frames, _, fseed = co.CASES[case]
    fdim = cfg["inputs_dim"]
    native, twin = _extractors(case)
    rows, want = [], []
    for t in frames:
        rows += list(co.utterances(2, t, fdim, fseed + t).numpy())
        want.append(GOLDEN["{}_T{}".format(case, t)])
    filler = _utterances([5, 333, 41], fdim, 70)
    T = max(r.shape[0] for r in rows + filler)
    batch = filler[:2] + rows + filler[2:]
    lens = [r.shape[0] for r in batch]
    ref = np.concatenate(want)
    for ex in (native, twin):
        got = ex.extract(_padded(batch, T), lengths=lens).cpu().numpy()[2:2 + len(rows)]
        assert rel(got, ref) <= 1e-4 and cosines(got, ref).min() >= 1 - 1e-6, (case, rel(got, ref))
    # utterances past the 4000-frame chunk: their chunks in one masked batch, combined as extract_embedding does
    for t in long_frames:
        x = co.utterances(2, t, fdim, fseed + t).numpy()
        chunks, owner = [], []
        for i in range(2):
            off = 0
            for s in chunk_sizes(t):
                chunks.append(x[i, off:off + s])
                owner.append(i)
                off += s
        emb = native.extract(_padded(chunks, max(c.shape[0] for c in chunks)), lengths=[c.shape[0] for c in chunks]).cpu()
        got = np.zeros((2, emb.shape[1]), np.float32)
        for e, c, i in zip(emb.numpy(), chunks, owner):
            got[i] += np.float32(c.shape[0]) * e
        got /= np.float32(t)
        ref = GOLDEN["{}_T{}".format(case, t)]
        assert rel(got, ref) <= 1e-4 and cosines(got, ref).min() >= 1 - 1e-6, (case, t, rel(got, ref))


# ------------------------------------------------------------------ 6. xvb-extract and the Python CLI
def _write_ark(path, feats):
    with open(path, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, np.ascontiguousarray(v, dtype=np.float32), key=k)


def test_cli_mixed_lengths_on_a_campplus_model(tmp_path):
    m = _model("default")
    sd = _sd("default")
    model = str(tmp_path / "campplus.xvbm")
    NativeCamPPExtractor(m).save(model)
    assert open(model, "rb").read(8) == b"XVBP0001"
    rng = np.random.RandomState(2027)
    lens = [3, 4, 4001, 9000, 4000, 200, 201] + [int(v) for v in rng.randint(3, 2500, 25)]
    feats = {"u{:02d}".format(i): co.utterances(1, t, 80, 7000 + i)[0].numpy() for i, t in enumerate(lens)}
    ark = str(tmp_path / "feats.ark")
    _write_ark(ark, feats)
    runs = {}
    for name, flag in (("mixed", ["--mixed-lengths"]), ("plain", [])):
        out = str(tmp_path / (name + ".ark"))
        r = subprocess.run([BIN, "--batch", "16"] + flag + [model, "ark:" + ark, "ark:" + out], capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        runs[name] = (dict(kaldi_io.read_vec_flt_ark(out)), r.stderr)
    got, summary = runs["mixed"]
    assert sorted(got) == sorted(feats)
    s = re.search(r"(\d+) masked batches, (\d+) padded frames \(([0-9.]+) of (\d+) batch frames\)", summary)
    assert s, summary
    assert int(s.group(1)) < len(feats) + 3 and float(s.group(3)) <= 0.125
    for k in feats:
        assert rel(got[k], runs["plain"][0][k]) <= 1e-6, (k, rel(got[k], runs["plain"][0][k]))
    with torch.no_grad():
        for k in ("u00", "u01", "u02", "u03", "u05", "u11"):
            ref = co.extract_embedding(sd, torch.from_numpy(feats[k][None])).numpy()[0]
            assert rel(got[k], ref) <= 1e-4, (k, rel(got[k], ref))

    torch.save(sd, str(tmp_path / "final.params"))
    out = str(tmp_path / "py.ark")
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--mixed-lengths",
                        "--model-blueprint", os.path.join(ROOT, "asv_subtools_b200", "model", "campplus_xvector.py"),
                        "--model-creation", "CamPPXvector(80, 10)", "--batch-size", "16",
                        str(tmp_path / "final.params"), "ark:" + ark, "ark:" + out],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    py = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(py) == sorted(feats) and "masked batches" in r.stderr
    for k in feats:
        assert rel(py[k], got[k]) <= 1e-6, (k, rel(py[k], got[k]))

    short = str(tmp_path / "short.ark")
    _write_ark(short, {"a": feats["u05"], "s": co.utterances(1, 2, 80, 9)[0].numpy()})
    r = subprocess.run([BIN, "--mixed-lengths", model, "ark:" + short, "ark:" + str(tmp_path / "s.ark")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 1 and "ERROR" in r.stderr and "lengths" in r.stderr, r.stdout + r.stderr
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--mixed-lengths",
                        "--model-blueprint", os.path.join(ROOT, "asv_subtools_b200", "model", "campplus_xvector.py"),
                        "--model-creation", "CamPPXvector(80, 10)", str(tmp_path / "final.params"), "ark:" + short,
                        "ark:" + str(tmp_path / "s2.ark")],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=900)
    assert r.returncode == 1 and "at least 3 frames" in r.stderr, r.stdout + r.stderr

