"""Speaker retrieval, task 2 of the CN-Celeb recipe (recipe/cnsrc/sr/run-cnsrc_sr.sh stage 4), in one command:
    python -m asv_subtools_b200.score.retrieve [--top 10] [--norm] [--submean F]
        [--plda MODEL [--num-utts F] [--smoothing S]]
        <enroll.ark|scp> <test.ark|scp> <out.top10> [--test-meta META]
writes the file trans_score_format.py makes from the all-pairs score file of getTrials.sh 1 + scoreSets_sr.sh --
every enrolled speaker (sorted, pandas' groupby order) followed by its `--top` best test utterances, best first,
lines joined by '\\n' with no trailing newline -- without writing or ranking the N_spk x N_test score lines.
Equal scores rank by position in the test ark (nlargest(keep='first') over trials in test-ark order).
Scores are cosine (`score="cosine"`), or with --plda the Kaldi-style PLDA LLR of score.sh `plda` (length-normalised
in the PLDA space; --num-utts: the `spk n` ark ivector-mean writes; --smoothing: ivector-copy-plda's, score.sh's
$plda_smoothing).  --test-meta prints cal_mAP.py's mAP=%.3f."""
import argparse
import sys
import traceback

import numpy as np
import torch

from .. import kaldi_io, ops
from . import backend, metrics


def format_topk(enroll_keys, test_keys, idx):
    """The top-k file of trans_score_format.py: speakers in sorted order, `spk utt1 ... uttk` per line, joined by
    '\\n' without a trailing one.  idx (M, k) int64 rows of test indices in the order of `enroll_keys`, -1 = empty."""
    idx = np.asarray(idx)
    row = {k: i for i, k in enumerate(enroll_keys)}
    lines = []
    for spk in sorted(row):
        lines.append(" ".join([spk] + [test_keys[j] for j in idx[row[spk]] if j >= 0]))
    return "\n".join(lines)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("enroll")
    ap.add_argument("test")
    ap.add_argument("out_top")
    ap.add_argument("--top", type=int, default=10, help="utterances kept per speaker (1..256)")
    ap.add_argument("--submean", default=None, help="global mean vector file (ivector-mean output)")
    ap.add_argument("--norm", action="store_true", help="length-normalise both sides (ivector-normalize-length)")
    ap.add_argument("--plda", default=None, help="PLDA model (Kaldi text or .ori vectors): score by PLDA LLR")
    ap.add_argument("--num-utts", default=None, help="`spk n` ark of enroll utterance counts (with --plda)")
    ap.add_argument("--smoothing", type=float, default=0.0,
                    help="within-class covariance smoothing of the PLDA model (ivector-copy-plda --smoothing, with --plda)")
    ap.add_argument("--test-meta", default=None, help="test metadata: print the mAP of cal_mAP.py")
    args = ap.parse_args(argv)
    try:
        ek, e = backend.load_vectors(args.enroll)
        tk, t = backend.load_vectors(args.test)
        mean = None
        if args.submean:
            mean = torch.from_numpy(np.asarray(kaldi_io.read_vec_flt(args.submean), dtype=np.float32)).cuda()
        e = backend.preprocess(e, mean, args.norm)
        t = backend.preprocess(t, mean, args.norm)
        row = col = None
        if args.plda:
            from .plda import read_num_utts
            from .plda_train import PLDA
            try:
                model = PLDA.read_trans(args.plda)
            except (ValueError, UnicodeDecodeError):
                model = PLDA.read_ori(args.plda)
            if args.smoothing:
                model.smooth_within_class_covariance(args.smoothing)
            n = None
            if args.num_utts:
                table = read_num_utts(args.num_utts)
                n = np.array([table[k] for k in ek], dtype=np.float32)
            e, row, t, col = model._operands(model.transform_ivectors(e, n), n, model.transform_ivectors(t, None))
        elif args.num_utts or args.smoothing:
            raise ValueError("--num-utts and --smoothing need --plda")
        _, idx = ops.retrieve_topk(e, t, args.top, row_bias=row, col_bias=col)
        text = format_topk(ek, tk, idx.cpu().numpy())
        with open(args.out_top, "w", encoding="utf-8") as f:
            f.write(text)
        if args.test_meta:
            print("mAP=%.3f" % metrics.retrieval_map_files(args.out_top, args.test_meta))
    except BaseException as err:  # same contract as the reference CLIs: traceback, exit 1
        if not isinstance(err, KeyboardInterrupt):
            traceback.print_exc()
        sys.exit(1)


if __name__ == "__main__":
    main()
