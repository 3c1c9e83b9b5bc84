# -*- coding:utf-8 -*-
"""Batched embedding extractor -- CLI twin of pytorch/pipeline/onestep/extract_embeddings.py.

Same positionals and flags (extract_embeddings.py:17-45):

    python -m asv_subtools_b200.pipeline.extract_embeddings [--nnet-config F | --model-blueprint P
        --model-creation S] [--use-gpu true] [--gpu-id ID] <model-path> <feats-rspecifier> <vectors-wspecifier>

What differs from the reference loop (:73-83, one utterance per iteration): utterances are read
from the ark stream, bucketed by frame count, and every bucket is extracted in ONE call of
`extract_embedding_batch()` (equal-length utterances need no padding, exactly like
splitDataByLength.sh-balanced jobs); utterances longer than maxChunk fall back to the
per-utterance `extract_embedding()` with the reference's chunk rule.  One `FV` vector is written per
input key (bucket order).  `--shard i/n` keeps every n-th utterance (one process per GPU without
pre-splitting the scp).

`--mixed-lengths` (models whose extractor takes lengths: the TDNN x-vector family with statistics pooling or an attention
pooling other than LDE -- attentive, multi-head, multi-resolution, xi-vector --, the F-TDNN x-vector, the ResNet x-vector,
the Conformer x-vector and CAM++): the model's chunk rule cuts every utterance first (the maxChunk rule, or the model's own
`chunk_sizes` where it has one: the Conformer's 300-frame rule, CAM++'s 4000-frame egrecho rule), and the chunks are batched across lengths instead of by exact frame count (`plan_mixed_batches`); a batch runs as one masked
call, `extract_embedding_batch(x, lengths)`, and each utterance's embedding is sum(len_i * emb_i) / frames over its
chunks, as `bin/xvb-extract --mixed-lengths` does.  The pooling merge order depends on the batch shape, so the vectors
differ from the default mode's at the rounding level.
"""
import argparse
import os
import sys
import traceback

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200 import kaldi_io  # noqa: E402

MAX_CHUNK = 10000


def read_nnet_config(path):
    """`;`-separated two-row CSV written by utils.write_nnet_config (utils.py:189-202)."""
    vals = {}
    with open(path) as f:
        for line in f:
            line = line.rstrip("\n")
            if ";" in line:
                k, v = line.split(";", 1)
                vals[k.strip()] = v.strip().strip('"').replace('""', '"')
    return vals["model_blueprint"], vals["model_creation"]


def create_model_from_py(model_blueprint, model_creation):
    """Import a blueprint by path and evaluate the creation string (utils.py:163-186)."""
    if not os.path.exists(model_blueprint):
        raise TypeError("Expected {} to exist.".format(model_blueprint))
    sys.path.insert(0, os.path.dirname(os.path.abspath(model_blueprint)))
    module = __import__(os.path.basename(model_blueprint).split(".")[0])
    return eval("module.{0}".format(model_creation), {"module": module})


class Batcher:
    """Buckets (key, feats) by frame count; yields full buckets, and everything at flush()."""

    def __init__(self, batch_size, max_pending_frames=4_000_000, length=None):
        """`length(item)`: the bucketing key (default: rows of the item); `max_pending_frames` bounds what is held
        back waiting for a bucket to fill (in units of that key), after which everything pending is flushed."""
        self.batch_size, self.max_pending = batch_size, max_pending_frames
        self.buckets, self.pending = {}, 0
        self.length = length or (lambda a: a.shape[0])

    def add(self, key, feats):
        t = self.length(feats)
        b = self.buckets.setdefault(t, [])
        b.append((key, feats))
        self.pending += t
        if len(b) >= self.batch_size:
            self.pending -= t * len(b)
            yield self.buckets.pop(t)
        elif self.pending > self.max_pending:
            yield from self.flush()

    def flush(self):
        for t in sorted(self.buckets):
            yield self.buckets[t]
        self.buckets, self.pending = {}, 0


def plan_mixed_batches(lengths, batch_size):
    """The batch rule of --mixed-lengths (the same as xvb-extract's): items in ascending length (ties in arrival order),
    each batch up to `batch_size` consecutive items whose padded frames n * max(len) - sum(len) are at most 1/8 of
    n * max(len).  Returns lists of indices into `lengths`.  Equal lengths give the equal-length buckets: runs of
    batch_size items in arrival order, then the remainder."""
    order = sorted(range(len(lengths)), key=lambda i: lengths[i])
    batches, i = [], 0
    while i < len(order):
        j, total = i + 1, lengths[order[i]]
        while j < len(order) and j - i < batch_size:
            n, tmax = j - i + 1, lengths[order[j]]
            if 8 * (n * tmax - (total + tmax)) > n * tmax:
                break
            total += tmax
            j += 1
        batches.append(order[i:j])
        i = j
    return batches


def chunk_lengths(frames, max_chunk=MAX_CHUNK):
    """The maxChunk rule of framework.py:29-39: ceil(frames / max_chunk) chunks of frames // num_split frames, the last
    one taking the remainder."""
    num_split = (frames + max_chunk - 1) // max_chunk
    split = frames // num_split
    return [split] * (num_split - 1) + [frames - split * (num_split - 1)]


def model_chunk_lengths(model, frames):
    """The chunks --mixed-lengths cuts a `frames`-long utterance into for `model`: its own rule when the blueprint has
    one (`model.chunk_sizes(frames)`, e.g. the Conformer's 300-frame rule or CAM++'s 4000-frame egrecho rule), else the
    maxChunk rule (chunk_lengths)."""
    own = getattr(model, "chunk_sizes", None)
    return list(own(frames)) if own is not None else chunk_lengths(frames)


def extract_stream_mixed(model, reader, writer, batch_size=256, shard=(0, 1), log=print, max_pending_frames=4_000_000):
    """--mixed-lengths form of extract_stream.  Returns (utterances, batches, padded frames, batch frames)."""
    utts, items = [], []              # utts: [key, frames, chunks pending, sum(len_i * emb_i)]; items: (utt, chunk)
    stats = [0, 0, 0]
    pending = [0]

    def run():
        lens = [c.shape[0] for _, c in items]
        for idx in plan_mixed_batches(lens, batch_size):
            tmax = max(lens[i] for i in idx)
            x = np.zeros((len(idx), tmax, items[idx[0]][1].shape[1]), dtype=np.float32)
            for r, i in enumerate(idx):
                x[r, :lens[i]] = items[i][1]
            emb = model.extract_embedding_batch(x, lengths=[lens[i] for i in idx]).cpu().numpy()
            stats[0] += 1
            stats[1] += len(idx) * tmax - sum(lens[i] for i in idx)
            stats[2] += len(idx) * tmax
            for r, i in enumerate(idx):
                u = utts[items[i][0]]
                u[3] = u[3] + np.float32(lens[i]) * emb[r]
                u[2] -= 1
                if u[2] == 0:
                    writer(u[0], u[3] / np.float32(u[1]))
                    u[3] = None
        items.clear()
        pending[0] = 0

    count = 0
    for i, (key, feats) in enumerate(reader):
        if i % shard[1] != shard[0]:
            continue
        log("Process utterance for key {0}".format(key))
        feats = np.ascontiguousarray(feats)
        if feats.dtype != np.float32:
            raise TypeError("features of {} are {}, the extractor takes float32 (FM/CM) matrices".format(key, feats.dtype))
        count += 1
        lens = model_chunk_lengths(model, feats.shape[0])
        utts.append([key, feats.shape[0], len(lens), np.float32(0)])
        off = 0
        for n in lens:
            items.append((len(utts) - 1, feats[off:off + n]))
            off += n
        pending[0] += feats.shape[0]
        if pending[0] > max_pending_frames:
            run()
    run()
    return count, stats[0], stats[1], stats[2]


def extract_stream(model, reader, writer, batch_size=256, shard=(0, 1), log=print):
    """reader yields (key, (T,F) float32 ndarray); writer(key, 1-D float32 ndarray)."""
    batcher = Batcher(batch_size)
    count = 0

    def run(bucket):
        t = bucket[0][1].shape[0]
        if t > MAX_CHUNK:
            for key, feats in bucket:
                writer(key, model.extract_embedding(feats).numpy())
            return
        x = np.stack([f for _, f in bucket])
        emb = model.extract_embedding_batch(x).cpu().numpy()
        for (key, _), e in zip(bucket, emb):
            writer(key, e)

    for i, (key, feats) in enumerate(reader):
        if i % shard[1] != shard[0]:
            continue
        log("Process utterance for key {0}".format(key))
        feats = np.ascontiguousarray(feats)
        if feats.dtype != np.float32:
            raise TypeError("features of {} are {}, the extractor takes float32 (FM/CM) matrices".format(key, feats.dtype))
        count += 1
        for bucket in batcher.add(key, feats):
            run(bucket)
    for bucket in batcher.flush():
        run(bucket)
    return count


def main(argv=None):
    ap = argparse.ArgumentParser(description="Extract embeddings from a piece of feats.scp or pipeline (B200)")
    ap.add_argument("--nnet-config", type=str, default="")
    ap.add_argument("--model-blueprint", type=str, default=None)
    ap.add_argument("--model-creation", type=str, default=None)
    ap.add_argument("--use-gpu", type=str, default="true", choices=["true", "false"])
    ap.add_argument("--gpu-id", type=str, default="")
    ap.add_argument("--batch-size", type=int, default=256)
    ap.add_argument("--shard", type=str, default="0/1", help="i/n: keep utterances with index %% n == i")
    ap.add_argument("--mixed-lengths", action="store_true",
                    help="batch utterances of different lengths (padding at most 1/8 of a batch); TDNN x-vector models with "
                         "statistics or attention pooling (not LDE), F-TDNN, ResNet x-vector, Conformer and CAM++ models only")
    ap.add_argument("--blueprint-dir", type=str, default="",
                    help="take the blueprint of the same file name from this directory (asv_subtools_b200/model) instead of "
                         "the path stored in nnet.config, so a reference model dir is used as it is")
    ap.add_argument("model_path", metavar="model-path")
    ap.add_argument("feats_rspecifier", metavar="feats-rspecifier")
    ap.add_argument("vectors_wspecifier", metavar="vectors-wspecifier")
    print(" ".join(sys.argv))
    args = ap.parse_args(argv)
    try:
        if args.nnet_config != "":
            blueprint, creation = read_nnet_config(args.nnet_config)
        elif args.model_blueprint is not None and args.model_creation is not None:
            blueprint, creation = args.model_blueprint, args.model_creation
        else:
            raise ValueError("Expected nnet_config or (model_blueprint, model_creation) to exist.")
        if args.blueprint_dir:
            swapped = os.path.join(args.blueprint_dir, os.path.basename(blueprint))
            if not os.path.exists(swapped):
                raise FileNotFoundError("no B200 blueprint named {} in {}".format(os.path.basename(blueprint), args.blueprint_dir))
            blueprint = swapped
        if args.use_gpu != "true":
            raise RuntimeError("asv_subtools_b200 has no CPU path: run with --use-gpu true on an H100")
        model = create_model_from_py(blueprint, creation)
        model.load_state_dict(torch.load(args.model_path, map_location="cpu"), strict=False)
        torch.cuda.set_device(int(args.gpu_id.split(",")[0]) if args.gpu_id != "" else 0)
        model.cuda().eval()
        i, n = (int(v) for v in args.shard.split("/"))
        if args.mixed_lengths:
            ex = model.extractor()
            if not getattr(ex, "TAKES_LENGTHS", False):
                print("ERROR: --mixed-lengths needs a TDNN x-vector model with statistics or attention pooling (not LDE), an "
                      "F-TDNN, a ResNet x-vector, a Conformer or a CAM++ model; {} runs on {}".format(type(model).__name__,
                                                                                                     type(ex).__name__),
                      file=sys.stderr)
                sys.exit(1)
        # native ark reader (csrc/ark_io.cpp): the reference's byte-at-a-time key loop is the wall at GPU rates
        with kaldi_io.open_or_fd(args.vectors_wspecifier, "wb") as w:
            reader = kaldi_io.read_mat_ark_native(args.feats_rspecifier)
            write = lambda k, v: kaldi_io.write_vec_flt(w, v, key=k)  # noqa: E731
            if args.mixed_lengths:
                utts, batches, padded, total = extract_stream_mixed(model, reader, write, batch_size=args.batch_size,
                                                                    shard=(i, n))
                print("extract_embeddings: {} utterances, {} masked batches, {} padded frames ({:.4f} of {} batch frames)"
                      .format(utts, batches, padded, padded / max(total, 1), total), file=sys.stderr)
            else:
                extract_stream(model, reader, write, batch_size=args.batch_size, shard=(i, n))
    except SystemExit:
        raise
    except BaseException as err:
        if not isinstance(err, KeyboardInterrupt):
            traceback.print_exc()
        sys.exit(1)


if __name__ == "__main__":
    main()
