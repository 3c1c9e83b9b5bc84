#!/bin/bash
# Speaker retrieval for recipe/cnsrc/sr/run-cnsrc_sr.sh stage 4.  The reference has no shell function for this step
# (it runs getTrials.sh 1, scoreSets_sr.sh and trans_score_format.py), so this is a new one rather than a shadow and
# lives outside score_b200.sh, whose functions each replace a reference function of the same name.  Source it, then:
#
#     retrieve <enroll.ark|scp> <test.ark|scp> <out.top10> [test.meta]
#
# The vectors are the processed ones (enroll `mean-...-norm`, test `...-norm`).  Writes trans_score_format.py's
# .top10 file; with test.meta also prints cal_mAP.py's mAP.  retrieve_top (default 10) sets the list length.
#
#   XVB200_ROOT    repo root (default: the directory above this file)
#   XVB200_PYTHON  interpreter (default: python3)

XVB200_ROOT=${XVB200_ROOT:-$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)}
XVB200_PYTHON=${XVB200_PYTHON:-python3}

function retrieve(){
	local meta=()
	[ -n "$4" ] && meta=(--test-meta "$4")
	PYTHONPATH="$XVB200_ROOT${PYTHONPATH:+:$PYTHONPATH}" $XVB200_PYTHON -m asv_subtools_b200.score.retrieve \
		--top "${retrieve_top:-10}" "$1" "$2" "$3" "${meta[@]}" || exit 1
	return 0
}
