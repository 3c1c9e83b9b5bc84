"""The XVBM0002 layout (a TDNN x-vector with an attention or xi-vector pooling, asv_subtools_b200/csrc/model_file.cpp)
written from host arrays, independently of the library's writer."""
import struct

import numpy as np

RELU, BN = 1, 2
POOL_ATTENTION, POOL_XI_POSTMEAN, POOL_XI_POSTDIST = 1, 2, 3


def tap_record(w, b, s, t, ctx, relu):
    """One tap record: i32 Cout, Cin, ntaps, tot_context, flags, has_bias, has_bn | i32 ctx | f32 w, bias?, scale?, shift?"""
    w = np.ascontiguousarray(w, dtype=np.float32)
    flags = (RELU if relu else 0) | (BN if s is not None else 0)
    out = struct.pack("<7i", w.shape[0], w.shape[1], len(ctx), w.shape[2], flags, b is not None, s is not None)
    out += struct.pack("<{}i".format(len(ctx)), *ctx) + w.tobytes()
    for v in (b, s, t):
        if v is not None:
            out += np.ascontiguousarray(v, dtype=np.float32).tobytes()
    return out


def xvbm2(feat_dim, eps, kind, pooled, gdiv, unweighted, prior, frames, attention, segments):
    """magic | i32 feat_dim | f32 eps | i32 n_frame, n_segment | i32 kind, pooled, gdiv, unweighted, n_attention
    | f32 prior_logprec[pooled], prior_mean[pooled] (xi-vector kinds) | frame, attention and segment tap records.
    Each layer: (w (Cout, Cin, tot), bias, scale, shift, context, relu), None where absent."""
    out = b"XVBM0002" + struct.pack("<ifii", feat_dim, eps, len(frames), len(segments))
    out += struct.pack("<5i", kind, pooled, gdiv, 1 if unweighted else 0, len(attention))
    if prior is not None:
        out += b"".join(np.ascontiguousarray(p, dtype=np.float32).reshape(-1).tobytes() for p in prior)
    return out + b"".join(tap_record(*layer) for layer in list(frames) + list(attention) + list(segments))
