"""ECAPA-TDNN C512 on the CPU: the oracle replays the reference's golden embeddings (tests/golden/ecapa512.npz), the
blueprint's C512 state_dict has the reference's layout and parameter count, and the width-64 float64 machinery behind
test_gpu_res2net_w64_edges.py passes the checks test_ecapa_exact_host.py applies at width 128."""
import numpy as np
import pytest
import torch

import ecapa512_cases as c5
import gemm_exact as gx
import res2net_w64_exact as rx

SM_COUNTS = (132, 114, 78)   # H100 SXM, H100 PCIe, and a smaller part
W = rx.W


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


@pytest.mark.parametrize("key", c5.keys())
def test_oracle_replays_c512_golden(golden, key):
    g = golden("ecapa512")
    case, rest = next((c, key[len(c) + 1:]) for c in sorted(c5.CASES, key=len, reverse=True) if key.startswith(c + "_"))
    pos, t = rest.rsplit("_T", 1)
    want = g[key]
    got = c5.oracle(case, pos, c5.utterances(case, int(t)))
    assert got.shape == want.shape
    assert rel(got, want) < 1e-5, key


def test_blueprint_c512_state_dict_is_the_reference_layout(golden):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    g = golden("ecapa512")
    m = ECAPA_TDNN(80, 10, training=False, extracted_embedding="near", **c5.CANON)
    sd = m.state_dict()
    mine = [(k, tuple(v.shape)) for k, v in sd.items()]
    spec = [(k, tuple(s)) for k, s, _ in c5.CANON_SPEC]
    assert mine == spec
    ref = [(k, tuple(int(d) for d in s.split(",") if d)) for k, s in (e.rsplit(":", 1) for e in g["keys_canon"])]
    assert mine == ref
    params = sum(v.numel() for k, v in sd.items() if not k.endswith(("running_mean", "running_var", "num_batches_tracked")))
    assert params == c5.PARAMS == int(g["params_canon"])
    assert m.layer2.res2net_block.width == W and m.layer2.res2net_block.scale == 8
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in c5.onn.make_state_dict(c5.CANON_SPEC, 1).items()},
                      strict=True)


def test_blueprint_picks_the_native_extractor_for_512_and_1024(monkeypatch):
    from asv_subtools_b200.model import ecapa_tdnn_xvector as mod
    assert mod.NATIVE_CHANNELS == (512, 1024) and mod.CHAIN_WIDTHS == (64, 128)
    picked = {}
    monkeypatch.setattr(mod, "NativeEcapaExtractor", lambda m, dev: "native")
    monkeypatch.setattr(mod, "EcapaExtractor", lambda m, dev: "twin")
    for ch in (256, 512, 768, 1024):
        m = mod.ECAPA_TDNN(80, 10, training=False, ecapa_params={"channels": ch})
        m.device_for_extraction = lambda: "cpu"
        for native in ("1", "0"):
            monkeypatch.setenv("XVB_ECAPA_NATIVE", native)
            picked[ch, native] = m.build_extractor()
    assert picked == {(256, "1"): "twin", (512, "1"): "native", (768, "1"): "twin", (1024, "1"): "native",
                      (256, "0"): "twin", (512, "0"): "twin", (768, "0"): "twin", (1024, "0"): "twin"}


# ------------------------------------------------------------------------------------------------ width-64 chain reference
@pytest.mark.parametrize("sms", SM_COUNTS)
def test_w64_catalogue_covers_the_edges(sms):
    cases = rx.res2net_cases(sms).values()
    rnd = sms * rx.CTAS_PER_SM
    assert {1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257} <= {c["T"] for c in cases}
    assert any(c["B"] == 1 and -(-c["T"] // 128) >= 20 for c in cases)
    assert {1, 2, 3, 4, 5} <= {c["d"] for c in cases}
    assert any(c["d"] == c["T"] - 1 for c in cases) and any(c["d"] == c["T"] and c["T"] > 1 for c in cases)
    assert any(c["d"] > c["T"] for c in cases) and any(c["d"] > 128 and c["T"] > c["d"] for c in cases)
    assert {2, 3, 4, 8, 12, 16} <= {c["scale"] for c in cases}
    assert {1, rnd - 1, rnd, rnd + 1, 2 * rnd + 1} <= {c["B"] for c in cases}
    assert any(c["B"] > 2 * rnd and c["T"] > 128 for c in cases)
    assert any(c.get("layers") and c["B"] > rnd for c in cases) and any(c.get("layers") and c["T"] > 128 for c in cases)
    for c in cases:
        assert c["C"] == W * c["scale"]
        assert c["ldx"] % 8 == 0 and c["ldy"] % 8 == 0 and c["ldx"] != c["ldy"]
        assert c["ldx"] >= c["x_c0"] + c["C"] + 8 and c["ldy"] >= c["y_c0"] + c["C"] + 8


def test_w64_cover_planes_cover_every_k_position():
    for sms in SM_COUNTS:
        for name, case in rx.res2net_cases(sms).items():
            d = rx.make_res2net(case, 3)
            S = case["scale"] - 1
            assert d["w_hi"].shape == d["w_lo"].shape == (S * W, 3 * W)
            for plane in (d["w_hi"], d["w_lo"]):
                assert set(np.unique(plane)) == {-1.0, 0.0, 1.0}, name
                for st in range(S):
                    p = plane[st * W:(st + 1) * W]
                    assert np.all((p != 0).any(axis=0)), "{} step {}: a K position feeds no output row".format(name, st)
            for key in ("bias", "shift"):
                assert np.all(d[key] / gx.GRID == np.round(d[key] / gx.GRID)) and d[key].shape == (S * W,)
            assert set(np.unique(d["scale"])) <= {-1.0, 1.0}
            if S > 1:
                b = d["bias"].reshape(S, W)
                assert all(not np.array_equal(b[0], b[i]) for i in range(1, S)), name


def test_w64_cases_are_exact():
    for sms in SM_COUNTS:
        for name, case in rx.res2net_cases(sms).items():
            d = rx.make_res2net(case, 11)
            yh, yl = rx.res2net_reference(case, d)
            assert yh.shape == (case["B"], case["T"], case["C"]), name
            assert np.array_equal(yh[..., :W], d["x"][0][..., :W]) and np.array_equal(yl[..., :W], d["x"][1][..., :W])
            assert np.all(np.isfinite(yh)) and np.all(np.isfinite(yl))
            assert np.array_equal(gx.bf16_round(yh), yh) and np.array_equal(gx.bf16_round(yl), yl)
            assert np.all(yl / gx.GRID == np.round(yl / gx.GRID)), name
            if case["T"] * case["B"] >= 100:
                assert (yl[..., W:] != 0).mean() > 0.05, name


def test_w64_reference_against_plain_chunk_chain():
    case = dict(rx.res2net_cases(132)["scale4"], B=2, T=40, d=3)
    d = rx.make_res2net(case, 5)
    yh, yl = rx.res2net_reference(case, d)
    hx, lx = (a.astype(np.float64) for a in d["x"])
    T, dil = case["T"], case["d"]

    def conv(a, w):           # a (B, T, 64), w (64, 192) tap-major -> (B, T, 64)
        out = np.zeros(a.shape[:2] + (W,))
        for tap, off in enumerate((-dil, 0, dil)):
            for t in range(T):
                if 0 <= t + off < T:
                    out[:, t] += a[:, t + off] @ w[:, tap * W:(tap + 1) * W].T
        return out

    for st in range(case["scale"] - 1):
        r, k = slice(st * W, (st + 1) * W), slice((st + 1) * W, (st + 2) * W)
        wh, wl = d["w_hi"][r].astype(np.float64), d["w_lo"][r].astype(np.float64)
        acc = conv(hx[..., k] + lx[..., k], wh) + conv(hx[..., k], wl)
        if st:
            ph, pl = yh[..., r].astype(np.float64), yl[..., r].astype(np.float64)
            acc += conv(ph + pl, wh) + conv(ph, wl)
        v = np.maximum(acc + d["bias"][r], 0) * d["scale"][r] + d["shift"][r]
        h, lo = gx.split_bf16(v.astype(np.float32))
        assert np.array_equal(yh[..., k], h) and np.array_equal(yl[..., k], lo), st


@pytest.mark.parametrize("name", ["T129", "T65", "scale3", "scale16", "d_T-1"])
def test_w64_every_product_term_of_both_sources_matters(name):
    case = rx.res2net_cases(132)[name]
    d = rx.make_res2net(case, 7)
    full = rx.res2net_reference(case, d)
    for src in ("x", "y"):
        for term in ("hh", "lh", "hl"):
            try:
                got = rx.res2net_reference(case, d, drop=((src, term),))
            except AssertionError:
                continue      # the dropped term left the exact range: it certainly changed the output
            assert not (np.array_equal(got[0], full[0]) and np.array_equal(got[1], full[1])), (name, src, term)
