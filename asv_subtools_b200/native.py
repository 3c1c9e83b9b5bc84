"""Python handles over the native whole-model extractors of the C library: the TDNN (xvb_extractor_*, ops.Extractor),
ECAPA-TDNN (xvb_ecapa_*), ResNet (xvb_resnet_*), RepVGG / RepSPK (xvb_repvgg_*), Conformer (xvb_conformer_*) and CAM++
(xvb_campp_*) x-vectors.  NativeExtractor holds the part they share: create, set_layer per record and finalize (or load
a model file), save, extract and close; ShardExtractor adds the host-buffer and whole-shard calls of the TDNN, ECAPA-TDNN
and ResNet handles."""
import ctypes as C

import numpy as np
import torch


def _cuda_f32(feats, feat_dim):
    if not (isinstance(feats, torch.Tensor) and feats.is_cuda and feats.dtype == torch.float32 and feats.is_contiguous()):
        raise TypeError("feats must be a contiguous CUDA float32 tensor")
    if feats.shape[2] != feat_dim:
        raise ValueError("expected feature dim {}, got {}".format(feat_dim, feats.shape[2]))
    return feats


def host_lengths(lengths, b):
    """The lengths argument of a masked extract call ((B,) sequence, ndarray or tensor) as a contiguous host int32 array
    of B entries; out-of-range values stay out of range (clipped to int32) for the library's check to name them."""
    if isinstance(lengths, torch.Tensor):
        lengths = lengths.cpu().numpy()
    lens = np.ascontiguousarray(np.asarray(lengths, dtype=np.int64).reshape(-1))
    if lens.shape[0] != b:
        raise ValueError("lengths has {} entries for a batch of {}".format(lens.shape[0], b))
    return np.clip(lens, -2 ** 31, 2 ** 31 - 1).astype(np.int32)


def device_lengths(lengths, b, t, device):
    """The lengths of a masked batch of the Python launch sequences, checked on the host: ValueError naming the first
    entry outside [1, t]; None when every entry equals t (the unmasked sequence runs), else a device int32 (B,) tensor."""
    lens = host_lengths(lengths, b)
    bad = np.flatnonzero((lens < 1) | (lens > t))
    if bad.size:
        raise ValueError("lengths[{}]={} outside [1, T={}]".format(bad[0], lens[bad[0]], t))
    if (lens == t).all():
        return None
    return torch.from_numpy(lens).pin_memory().to(device, non_blocking=True)   # no host wait on the stream


class NativeExtractor:
    """xvb_<PREFIX>_t: packed weights, workspace and the whole launch sequence in the C library, on the device that is
    current when it is built from a model `m` (or loaded from a model file at `path`).

    A family sets PREFIX and supplies `_create_args(m)`, the arguments of xvb_<PREFIX>_create after the handle,
    `_configure(m)`, any call between create and the first set_layer, and `_layers(m)`, which yields
    (name, shape, (w, b, scale, shift), flags) per record, `shape` being the set_layer arguments between the name and
    the arrays.

    TAKES_LENGTHS: the handle has xvb_<PREFIX>_extract_lengths, and extract() takes `lengths` (a masked batch of
    utterances of different lengths).  extract_embedding_batch and the --mixed-lengths CLIs ask this of any extractor."""

    PREFIX = None
    TAKES_LENGTHS = False

    def __init__(self, m=None, device=None, path=None):
        from asv_subtools_b200._lib import check, lib
        self._lib, self._check = lib, check
        self._h = C.c_void_p()
        with torch.cuda.device(device if device is not None else torch.cuda.current_device()):
            if path is not None:
                self._call("load", C.byref(self._h), str(path).encode())
            else:
                self._call("create", C.byref(self._h), *self._create_args(m))
                self._configure(m)
                for name, shape, arrays, flags in self._layers(m):
                    arrs = [None if a is None else np.ascontiguousarray(a, dtype=np.float32) for a in arrays]
                    ptr = [None if a is None else a.ctypes.data_as(C.c_void_p) for a in arrs]
                    self._call("set_layer", self._h, name.encode(), *shape, *ptr, flags)
                self._call("finalize", self._h)
        self.feat_dim = self._fn("feat_dim")(self._h)
        self.embed_dim = self._fn("embed_dim")(self._h)

    def _configure(self, m):
        pass

    def _fn(self, name):
        return getattr(self._lib, "xvb_{}_{}".format(self.PREFIX, name))

    def _call(self, name, *args):
        self._check(self._fn(name)(*args), "xvb_{}_{}".format(self.PREFIX, name))

    @classmethod
    def load(cls, path):
        return cls(path=path)

    def save(self, path):
        """Write the model file that load() and bin/xvb-extract read."""
        self._call("save", self._h, str(path).encode())

    @property
    def last_launches(self):
        return self._fn("last_launches")(self._h)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _input(self, feats):
        return _cuda_f32(feats, self.feat_dim)

    def extract(self, feats, lengths=None):
        """feats (B, T, F) fp32 CUDA (one chunk per utterance) -> (B, embed_dim) fp32 CUDA, asynchronous on the current
        stream.  lengths (B,) host ints, 1 <= lengths[b] <= T (TAKES_LENGTHS families): a batch of utterances of
        different lengths, row b being feats[b, :lengths[b]] extracted alone; the frames past them are never read."""
        feats = self._input(feats)
        B, T, _ = feats.shape
        emb = torch.empty(B, self.embed_dim, dtype=torch.float32, device=feats.device)
        if lengths is None:
            self._call("extract", self._h, C.c_void_p(feats.data_ptr()), B, T, C.c_void_p(emb.data_ptr()), self._stream())
            return emb
        if not self.TAKES_LENGTHS:
            raise NotImplementedError("{}: extract(lengths=...) is not supported by this family".format(type(self).__name__))
        lens = host_lengths(lengths, B)
        self._call("extract_lengths", self._h, C.c_void_p(feats.data_ptr()), lens.ctypes.data_as(C.c_void_p), B, T,
                   C.c_void_p(emb.data_ptr()), self._stream())
        return emb

    def close(self):
        h, self._h = self._h, None
        if h:
            self._fn("destroy")(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShardExtractor(NativeExtractor):
    """A handle with xvb_<PREFIX>_extract_host, _extract_shard, _extract_shard_host and (where the family has it)
    _set_gather; `batch` is the default batch of the shard calls."""

    batch = 128

    def extract_host(self, feats_np):
        """feats (B, T, F) float32 host array -> (B, D) float32 host array (H2D + D2H + one sync inside the call)."""
        feats_np = np.ascontiguousarray(feats_np, dtype=np.float32)
        b, t, f = feats_np.shape
        if f != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, f))
        emb = np.empty((b, self.embed_dim), dtype=np.float32)
        self._call("extract_host", self._h, feats_np.ctypes.data_as(C.c_void_p), b, t, emb.ctypes.data_as(C.c_void_p),
                   self._stream())
        return emb

    def extract_shard(self, feats, batch=None, out=None):
        """feats (N, T, F) fp32 CUDA -> (N, D) fp32 CUDA (`out` if given): the whole shard in `batch`-utterance batches,
        one C call (extract_embeddings.py:73-83's loop), asynchronous on the current stream."""
        n, t, _ = self._input(feats).shape
        if out is None:
            out = torch.empty(n, self.embed_dim, dtype=torch.float32, device=feats.device)
        elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.dtype == torch.float32 and out.is_contiguous()):
            raise TypeError("out must be a contiguous CUDA float32 tensor")
        elif tuple(out.shape) != (n, self.embed_dim):
            raise ValueError("out must be ({}, {})".format(n, self.embed_dim))
        self._call("extract_shard", self._h, C.c_void_p(feats.data_ptr()), n, t, int(batch or self.batch),
                   C.c_void_p(out.data_ptr()), self._stream())
        return out

    def extract_shard_host(self, feats_ptr, n, t, emb_ptr, batch=None):
        """Pinned host feats (n, t, F) in, host embeddings (n, D) out; the copies overlap the stack."""
        self._call("extract_shard_host", self._h, C.c_void_p(feats_ptr), int(n), int(t), int(batch or self.batch),
                   C.c_void_p(emb_ptr), self._stream())

    def set_gather(self, pointers, ntables, row0, ld):
        """Replicated-table form of the shard calls (parallel.PeerTable.attach): every batch's embeddings also go to
        `ntables` table copies at row0 + row; ntables = 0 turns it off."""
        self._call("set_gather", self._h, pointers, int(ntables), int(row0), int(ld))
