#!/bin/bash
# Batched B200 extraction behind the reference's own job script.
#
#   integration/extract_xvectors_b200.sh [options of extract_xvectors_for_pytorch.sh] <model-dir> <data-dir> <output-dir>
#
# Run from the recipe directory, where `subtools/` is the reference checkout, exactly like
# subtools/pytorch/pipeline/extract_xvectors_for_pytorch.sh.  That script hard-codes its extractor
# (`python3 subtools/pytorch/pipeline/onestep/extract_embeddings.py`, lines 128-141); this wrapper runs the reference
# script UNMODIFIED except for that one command, rewritten on the fly (nothing of the reference is copied or patched on
# disk) to the batched CLI twin with the same flags and positionals:
#
#   python -m asv_subtools_b200.pipeline.extract_embeddings --batch-size $XVB200_BATCH --blueprint-dir <repo>/asv_subtools_b200/model
#
# --blueprint-dir makes the CLI take the B200 blueprint of the same file name (xvector.py, ecapa_tdnn_xvector.py, ...)
# instead of the path stored in <model-dir>/config/nnet.config, so a reference model directory works as it is: same
# creation string, same final.params.  Everything else -- data splitting, the apply-cmvn-sliding / select-voiced-frames
# feature pipes, copy-vector on the output, the ERROR grep over the logs, xvector.scp concatenation -- is the reference's.
#
#   XVB200_ROOT    repo root (default: the directory above this file)      XVB200_PYTHON  interpreter (default: python3)
#   XVB200_BATCH   utterances per batch (default 256)                      XVB200_REF     the reference script to wrap
#   XVB200_DRYRUN  non-empty: print the rewritten command lines and exit
#   XVB200_MIXED_LENGTHS  1: add --mixed-lengths (batches of utterances of different lengths, at most 1/8 padding;
#                  TDNN x-vector models with statistics or attention pooling other than LDE, F-TDNN, ResNet
#                  x-vector, Conformer and CAM++ models only)

set -e
XVB200_ROOT=${XVB200_ROOT:-$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)}
XVB200_PYTHON=${XVB200_PYTHON:-python3}
XVB200_BATCH=${XVB200_BATCH:-256}
mixed=""
[ "${XVB200_MIXED_LENGTHS:-}" = "1" ] && mixed=" --mixed-lengths"
XVB200_REF=${XVB200_REF:-subtools/pytorch/pipeline/extract_xvectors_for_pytorch.sh}

[ ! -f "$XVB200_REF" ] && echo "[exit] $XVB200_REF not found: run from the recipe directory (or set XVB200_REF)" && exit 1

old="python3 subtools/pytorch/pipeline/onestep/extract_embeddings.py"
new="env PYTHONPATH=$XVB200_ROOT\${PYTHONPATH:+:\$PYTHONPATH} $XVB200_PYTHON -m asv_subtools_b200.pipeline.extract_embeddings --batch-size $XVB200_BATCH$mixed --blueprint-dir $XVB200_ROOT/asv_subtools_b200/model"
grep -q "$old" "$XVB200_REF" || { echo "[exit] $XVB200_REF does not call '$old' any more: nothing to swap"; exit 1; }

tmp=$(mktemp /tmp/extract_xvectors_b200.XXXXXX.sh)
trap 'rm -f "$tmp"' EXIT
sed "s#$old#$new#g" "$XVB200_REF" > "$tmp"
if [ -n "$XVB200_DRYRUN" ]; then        # show what would run instead of the reference's extractor lines
	diff "$XVB200_REF" "$tmp" | grep '^>' || true
	exit 0
fi
# the batched path is a GPU path: default to --use-gpu true unless the caller says otherwise
case " $* " in *" --use-gpu"*) bash "$tmp" "$@";; *) bash "$tmp" --use-gpu true "$@";; esac
