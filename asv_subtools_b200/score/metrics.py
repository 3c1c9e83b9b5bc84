"""EER / minDCF in the three definitions the reference carries (SURVEY Appendix B.12); vectorised
NumPy on the host (a sort plus cumulative counts).  Same results as the reference scripts on the
same scores (tests/test_metrics.py replays the golden values).

  bosaris : computeEER-like-Bosaris.py:50-107   (average of the two points nearest the crossing)
  det     : subtools2/egrecho/score/binary_metrics.py:11-120 (linear interpolation on the DET curve)
  kaldi   : Kaldi compute-eer as called by computeEER.sh:21-22 (step rule)
"""
import numpy as np


def _as_arrays(scores, labels):
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    lab = np.asarray(labels).reshape(-1)
    if lab.dtype.kind in "US":
        lab = (lab == "target")
    lab = lab.astype(bool)
    if s.shape != lab.shape:
        raise ValueError("scores and labels differ in length")
    if not lab.any() or lab.all():
        raise ValueError("need both target and nontarget trials")
    return s, lab


def eer_bosaris(scores, labels):
    """Thresholds walk upward through the sorted scores (ties: nontargets first, as the reference's
    list sort orders [score, label] pairs); FR counts targets at or below the threshold, FA counts
    nontargets above it; at the first point with FAR <= FRR the nearer of {this, previous} point
    gives EER = (FAR+FRR)/2."""
    s, lab = _as_arrays(scores, labels)
    order = np.lexsort((lab, s))
    s, lab = s[order], lab[order]
    n_tar, n_non = int(lab.sum()), int((~lab).sum())
    frr = np.cumsum(lab) / n_tar
    far = (n_non - np.cumsum(~lab)) / n_non
    idx = int(np.argmax(far <= frr))
    now = abs(far[idx] - frr[idx])
    prev = abs(far[idx - 1] - frr[idx - 1]) if idx > 0 else np.inf
    if now <= prev:
        return float((far[idx] + frr[idx]) / 2), float(s[idx])
    return float((far[idx - 1] + frr[idx - 1]) / 2), float(s[idx - 1])


def det_curve(scores, labels):
    s, lab = _as_arrays(scores, labels)
    desc = np.argsort(s, kind="mergesort")[::-1]
    s, lab = s[desc], lab[desc]
    edges = np.r_[np.where(np.diff(s))[0], s.size - 1]
    tps = np.cumsum(lab)[edges].astype(np.float64)
    fps = 1 + edges - tps
    thr = s[edges]
    fns = tps[-1] - tps
    first = fps.searchsorted(fps[0], side="right") - 1 if fps.searchsorted(fps[0], side="right") > 0 else None
    last = tps.searchsorted(tps[-1]) + 1
    sl = slice(first, last)
    return fps[sl][::-1] / fps[-1], fns[sl][::-1] / tps[-1], thr[sl][::-1]


def eer_det(scores, labels):
    fpr, fnr, thr = det_curve(scores, labels)
    i0 = np.flatnonzero(fnr - fpr <= 0)[-1]
    i1 = np.flatnonzero(fnr - fpr > 0)[0]
    d0, d1 = fnr[i0] - fpr[i0], fnr[i1] - fpr[i1]
    w = abs(d0) / (d1 - d0)
    return float(fnr[i0] + w * (fnr[i1] - fnr[i0])), float(thr[i0] + w * (thr[i1] - thr[i0]))


def min_dcf(scores, labels, p_target=0.01, c_miss=1.0, c_fa=1.0):
    fpr, fnr, _ = det_curve(scores, labels)
    return float(np.min(c_miss * fnr * p_target + c_fa * fpr * (1 - p_target)) / min(c_miss * p_target, c_fa * (1 - p_target)))


def eer_kaldi(scores, labels):
    s, lab = _as_arrays(scores, labels)
    tar, non = np.sort(s[lab]), np.sort(s[~lab])
    nt, nn = tar.size, non.size
    i = np.arange(nt)
    ni = np.clip(nn - 1 - (nn * i // nt), 0, nn - 1)
    hit = np.flatnonzero(non[ni] < tar)
    k = int(hit[0]) if hit.size else nt - 1
    return k / nt, float(tar[k])


METHODS = {"bosaris": eer_bosaris, "det": eer_det, "kaldi": eer_kaldi}


def retrieval_map(top_lines, meta_lines):
    """mAP of a speaker-retrieval top-k file, computed exactly as recipe/cnsrc/sr/cal_mAP.py does, quirks included.
    `top_lines`: the lines of the top-k file (`spk utt1 ... uttk`); `meta_lines`: the lines of the test metadata
    (`<dir>/<utt>.wav <spk>-<...> ...`).  Returns the float cal_mAP.py prints as "mAP=%.3f"."""
    targets = {}
    for line in meta_lines:
        fields = line.strip("\n").split(" ")
        spk = fields[1].split("-")[0]                 # the speaker is field 2 up to its first '-'
        # strip('.wav') removes any of the characters '.', 'w', 'a', 'v' from both ends (a character set, not a
        # suffix): "pool/utt13a.wav" -> "pool/utt13", "wav/abc.wav" -> "/abc"; then the part after the first '/'
        # is the utterance, so an utterance whose name ends in one of those characters never counts as a hit
        utt = fields[0].strip(".wav").split("/")[1]
        targets.setdefault(spk, set()).add(utt)
    total, rows = 0.0, 0
    for line in top_lines:
        fields = line.strip("\n").split(" ")
        rows += 1
        if fields[0] not in targets:
            raise KeyError("speaker {} of the top-k file is not in the test metadata".format(fields[0]))
        mine = targets[fields[0]]
        hits, score = 0, 0.0
        for i in range(1, len(fields)):
            if fields[i] in mine:
                hits += 1
            score += hits / i                          # every position adds precision@i, hit or not
        score /= 10                                    # the constant 10 of the recipe, whatever the list length
        total += score
    if rows == 0:
        raise ValueError("empty top-k file")
    return total / rows


def retrieval_map_files(top_path, meta_path):
    with open(meta_path, encoding="utf-8") as f:
        meta = f.readlines()
    with open(top_path, encoding="utf-8") as f:
        top = f.readlines()
    return retrieval_map(top, meta)
