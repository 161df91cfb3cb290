"""Stored results of the reference's own CUDA extension for the reference-parity tests.

The parity tests compare this repository's ops with the unmodified reference extension (deployment/kvquant quant_cuda,
compiled by oracle/build_ref.py into oracle/_ref/) on seeded inputs.  The reference is not part of this repository,
so what it returned on those inputs is stored under tests/golden/ref_<test module>.npz and the tests compare against
that.  With the extension built, a run with KVQ_REF_GOLDEN_OUT=<dir> compares against the live reference instead
and re-records the files into <dir>:

    KVQ_REF_GOLDEN_OUT=/tmp/golden python -m pytest -m gpu tests/test_gpu_vs_reference.py ...

What is stored per result:
  * exact(): results compared bit for bit (packed codes, index arrays, element-wise fp32 outputs) as SHA-256 digests
    of their bytes, dtype and shape;
  * rows(): toleranced float results [R, n] as a fixed, seeded sample of `cols` columns of every row plus the largest
    magnitude of every full row (the scale the tolerances are relative to).
"""
import hashlib
import os
import sys
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _np(x):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().contiguous().numpy()
    return np.ascontiguousarray(x)


def digest(x):
    a = _np(x)
    h = hashlib.sha256()
    h.update(("%s %s|" % (a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8)


class RefGolden:
    def __init__(self, name):
        self.name = name
        self.out_dir = os.environ.get("KVQ_REF_GOLDEN_OUT") or None
        self.ref = None
        if self.out_dir:
            sys.path.insert(0, os.path.join(ROOT, "oracle"))
            import build_ref
            self.ref = build_ref.load()
            if self.ref is None:
                raise RuntimeError("KVQ_REF_GOLDEN_OUT is set but oracle/_ref/quant_cuda_ref.so is not built")
            self.data = {}
        else:
            with np.load(os.path.join(GOLDEN, "ref_%s.npz" % name)) as f:
                self.data = dict(f)

    @property
    def recording(self):
        return self.out_dir is not None

    def save(self):
        if self.recording:
            os.makedirs(self.out_dir, exist_ok=True)
            np.savez_compressed(os.path.join(self.out_dir, "ref_%s.npz" % self.name), **self.data)

    def value(self, key, ref_fn=None):
        """A small array stored whole (flags, counters)."""
        if self.recording:
            self.data[key] = _np(ref_fn())
        return self.data[key]

    def exact(self, key, ours, ref_fn=None):
        """Assert `ours` equals the reference result bit for bit (recording: ref_fn() is run and compared live)."""
        if self.recording:
            r = ref_fn()
            assert np.array_equal(_np(ours), _np(r)) and _np(ours).dtype == _np(r).dtype, key
            self.data[key + "#sha"] = digest(r)
        assert np.array_equal(digest(ours), self.data[key + "#sha"]), "%s differs from the reference" % key

    def rows(self, key, ours, ref_fn=None, cols=32):
        """(ours_sample, ref_sample, ref_row_max) as float64 tensors on the CPU for a toleranced comparison of a float
        result viewed as [R, n]: the same seeded `cols` columns of every row (all columns when n <= cols), and the
        largest |ref| over each full row."""
        a = _np(ours).astype(np.float64)
        a = a.reshape(-1, a.shape[-1]) if a.ndim > 1 else a.reshape(1, -1)
        if self.recording:
            r = _np(ref_fn()).astype(np.float64).reshape(a.shape)
            n = r.shape[1]
            rng = np.random.default_rng(zlib.crc32(("%s/%s" % (self.name, key)).encode()))
            idx = np.arange(n) if n <= cols else np.sort(rng.choice(n, cols, replace=False))
            self.data[key + "#idx"] = idx.astype(np.int32)
            self.data[key + "#val"] = r[:, idx].astype(np.float32)
            self.data[key + "#max"] = np.abs(r).max(axis=1).astype(np.float32)
        idx = self.data[key + "#idx"]
        return (torch.from_numpy(a[:, idx]), torch.from_numpy(self.data[key + "#val"].astype(np.float64)),
                torch.from_numpy(self.data[key + "#max"].astype(np.float64)))


def rel_rows(a, b, bmax):
    """max |a-b| over the sample relative to the largest |ref| of the whole result, and the same per row relative to
    that row's own largest |ref| (a wrong small element cannot hide behind a large one in another row)."""
    d = (a - b).abs()
    return (d.max() / bmax.max().clamp_min(1e-30)).item(), (d.amax(dim=1) / bmax.clamp_min(1e-30)).max().item()
