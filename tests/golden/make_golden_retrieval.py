"""Golden data for speaker retrieval (tests/test_retrieval_host.py, tests/test_gpu_retrieval.py): runs the reference's
own recipe/cnsrc/sr/trans_score_format.py and cal_mAP.py, unmodified, on seeded vectors.  Build machine only (needs
the reference tree and pandas):  python tests/golden/make_golden_retrieval.py <reference root>

  * 12 enrolled speakers (ids "id1xxxx", written in shuffled order) and 150 test utterances in 32 dimensions.  Test
    utterances are speaker centres plus noise; 20 of them are exact copies of others, so exact ties occur inside
    top-10 lists.
  * Scores are cosine in float64 of the stored float32 vectors, written with repr() into an all-pairs file in trials
    order (getTrials.sh 1: for each test utterance, every enrolled speaker in sorted order).
  * The seed is the first one at which every speaker's 11 best scores that are not exact copies differ by more than
    1e-4, so a float32 GPU ranking must reproduce the file byte for byte.
  * The test metadata has cal_mAP.py's edge cases: utterance names ending in 'a', 'v' or 'w' (strip('.wav') eats
    them, so they never count as hits), a directory made only of those characters, and lines for utterances outside
    the test set."""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# trans_score_format.py reads row['spk-id'] from the frame groupby('spk-id').apply(...) returns.  pandas < 3 passes
# each group to the function with its grouping column; pandas 3 leaves that column out.  This runs the script
# unmodified with the older behaviour restored for groupby.apply: each group, key column included, in sorted key order.
PANDAS2_APPLY = """
import runpy, sys
import pandas as pd
from pandas.core.groupby.generic import DataFrameGroupBy
def apply(self, func, *args, **kwargs):
    keys, parts = zip(*[(k, func(g, *args, **kwargs)) for k, g in self])
    return pd.concat(parts, keys=keys)
DataFrameGroupBy.apply = apply
sys.argv = sys.argv[1:]
runpy.run_path(sys.argv[0], run_name="__main__")
"""
M, N, D, DUP = 12, 150, 32, 20


def make(seed):
    rng = np.random.RandomState(seed)
    spk = ["id1{:04d}".format(i) for i in rng.choice(9000, M, replace=False)]
    centres = rng.randn(M, D)
    enroll = (centres + 0.3 * rng.randn(M, D)).astype(np.float32)
    owner = rng.randint(0, M, N - DUP)
    test = (centres[owner] + 0.9 * rng.randn(N - DUP, D)).astype(np.float32)
    src = rng.choice(N - DUP, DUP, replace=False)
    test = np.concatenate([test, test[src]])
    owner = np.concatenate([owner, owner[src]])
    perm = rng.permutation(N)
    test, owner = test[perm], owner[perm]
    suffix = ["", "", "", "", "a", "v", "w"]
    utt = ["u{:04d}{}".format(i, suffix[rng.randint(len(suffix))]) for i in range(N)]
    order = rng.permutation(M)                         # the enroll ark is not in sorted order
    return [spk[i] for i in order], enroll[order], utt, test, owner, spk


def scores64(enroll, test):
    e = enroll.astype(np.float64)
    t = test.astype(np.float64)
    e /= np.linalg.norm(e, axis=1, keepdims=True)
    t /= np.linalg.norm(t, axis=1, keepdims=True)
    return e @ t.T


def separated(s, test):
    _, first = np.unique(test, axis=0, return_index=True)
    for row in s:
        top = np.sort(row[np.sort(first)])[::-1][:11]
        if np.min(np.diff(-top)) <= 1e-4:
            return False
    return True


def main(ref):
    for seed in range(1000):
        spk_keys, enroll, utt, test, owner, spk = make(seed)
        s = scores64(enroll, test)
        if separated(s, test):
            break
    sr = os.path.join(ref, "recipe", "cnsrc", "sr")
    with tempfile.TemporaryDirectory() as tmp:
        score_file = os.path.join(tmp, "cosine.score")
        row = {k: i for i, k in enumerate(spk_keys)}
        with open(score_file, "w") as f:
            for j, u in enumerate(utt):
                for k in sorted(spk_keys):
                    f.write("{} {} {}\n".format(k, u, repr(float(s[row[k], j]))))
        top_file = score_file + ".top10"
        subprocess.check_call([sys.executable, "-c", PANDAS2_APPLY, os.path.join(sr, "trans_score_format.py"), score_file,
                               top_file])
        top10 = open(top_file, "rb").read()
        rng = np.random.RandomState(seed + 1)
        dirs = ["pool", "wav", "test/pool"]
        lines = []
        for j, u in enumerate(utt):
            d = dirs[rng.randint(len(dirs))] if j % 5 == 0 else "pool"
            lines.append("{}/{}.wav {}-speech-01-{:03d}".format(d, u, spk[owner[j]], j))
        for j in range(5):                             # utterances outside the test set
            lines.append("pool/x{:03d}.wav {}-interview-02-{:03d}".format(j, spk[j % M], j))
        order_meta = rng.permutation(len(lines))
        meta = "".join(lines[i] + "\n" for i in order_meta)
        meta_file = os.path.join(tmp, "test.meta")
        open(meta_file, "w").write(meta)
        out = subprocess.run([sys.executable, os.path.join(sr, "cal_mAP.py"), top_file, meta_file], capture_output=True,
                             text=True, check=True).stdout
    ties = sum(int(np.sum(np.diff(np.sort(r)) == 0)) for r in s)
    np.savez_compressed(os.path.join(HERE, "retrieval.npz"), seed=seed, enroll=enroll, enroll_keys=np.array(spk_keys),
                        test=test, test_keys=np.array(utt), scores64=s, top10=np.frombuffer(top10, dtype=np.uint8),
                        meta=np.frombuffer(meta.encode(), dtype=np.uint8), map_line=np.array(out.strip()))
    print("seed", seed, "exact ties", ties, out.strip(), "top10 bytes", len(top10))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: make_golden_retrieval.py <reference root>")
    main(sys.argv[1])
