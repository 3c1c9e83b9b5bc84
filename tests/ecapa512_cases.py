"""ECAPA-TDNN C512 (ecapa_params={"channels": 512}: Res2Net scale 8 x width 64, 6 538 112 parameters): the creation
kwargs and golden cases shared by tests/golden/make_golden_ecapa512.py, test_ecapa_c512_host.py and
test_gpu_ecapa_c512.py.  Every case is (kwargs, state_dict spec, state_dict seed, positions, frame counts, feature seed);
its golden key is "<case>_<pos>_T<frames>", two utterances per key (one for the chunked T = 10 050)."""
import copy

import ecapa_mqmha_oracle as mo
from oracle import nnet as onn

C = 512
PARAMS = 6538112          # ECAPA_TDNN(80, 10, ecapa_params={"channels": 512}) without the loss layer

_BN = {"momentum": 0.5, "affine": True, "track_running_stats": True}
_ECAPA = {"channels": C, "embd_dim": 192, "mfa_conv": 1536, "bn_params": _BN}
# the canonical launcher recipe (runEcapaXvector_online.py:221-263) at 512 channels: fc2 without ReLU, BN without affine
CANON = dict(ecapa_params=_ECAPA, pooling="ecpa-attentive",
             pooling_params={"hidden_size": 128, "time_attention": True, "stddev": True}, fc1=False,
             fc2_params={"nonlinearity": "", "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                         "bn_params": {"momentum": 0.5, "affine": False, "track_running_stats": True}})
# fc1=True with the blueprint's fc defaults (ReLU, affine BN), as make_golden_ecapa_fc1.py
FC1 = dict(ecapa_params={"channels": C}, fc1=True)
# the roadmap launcher's MQMHA pooling at 512 channels
MQMHA = copy.deepcopy(mo.ROADMAP_KW)
MQMHA["ecapa_params"]["channels"] = C

CANON_SPEC = onn.ecapa_spec(80, channels=C)
CASES = {
    "canon": (CANON, CANON_SPEC, 511, ("near", "near_affine"), (300, 200, 129, 37, 2), 5110),
    "canon_long": (CANON, CANON_SPEC, 511, ("near",), (10050,), 5120),     # two chunks of the maxChunk = 10000 rule
    "fc1": (FC1, onn.ecapa_spec(80, channels=C, fc1=True, fc2_bn_affine=True), 513, ("far", "near_affine", "near"), (120,),
            5130),
    "mqmha": (MQMHA, mo.ecapa_mqmha_spec(MQMHA), 514, ("near",), (300,), 5140),
}


def utterances(case, frames):
    """(n, frames, 80) float32 features of a case: two utterances, one for the chunked length."""
    return onn.synthetic_feats(1 if frames > 10000 else 2, frames, 80, CASES[case][5] + frames)


def keys():
    """Every golden key, in a stable order."""
    return ["{}_{}_T{}".format(case, pos, t) for case, (_, _, _, poss, ts, _) in CASES.items() for pos in poss for t in ts]


def oracle(case, pos, feats):
    """The torch-CPU oracle (oracle.nnet / ecapa_mqmha_oracle) through the maxChunk rule: (n, 192) float64."""
    import numpy as np
    kw, spec, seed, _, _, _ = CASES[case]
    sd = onn.make_state_dict(spec, seed)
    if case == "mqmha":
        fwd = lambda x: mo.ecapa_mqmha_forward(sd, x, kw, pos)  # noqa: E731
    else:
        fc1 = kw.get("fc1", False)          # the fc1 case keeps the blueprint's fc2 defaults: ReLU, affine BN
        fwd = lambda x: onn.ecapa_forward(sd, x, pos, fc2_relu=fc1, fc1=fc1)  # noqa: E731
    return np.stack([onn.extract_embedding(fwd, f).double().numpy() for f in feats])
