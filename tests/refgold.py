"""What the unmodified reference extension computed on a given test input, kept as golden data
(tests/golden/refgold_<name>.npz), so that the comparisons with the reference run on any machine.

Small arrays are stored whole.  A large one is stored as the SHA-1 of its bytes (bit-exact comparisons), the largest
magnitude (the scale of a gradient tolerance) and a fixed, seeded sample of its elements (tolerance comparisons).

Regenerating, where the reference extension is built (oracle/_ref/_refC.so, `python oracle/build_ref.py`):

    GSR_REF_RECORD=<dir> python -m pytest -m gpu tests      # then copy <dir>/refgold_*.npz to tests/golden/

In that mode `reference()` runs the reference live, writes what it returned to <dir> and the test compares against
exactly what was written."""
import hashlib
import os

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WHOLE = 4096     # arrays up to this many elements are stored whole
NSAMPLE = 4096   # sampled elements of a larger array


def _np(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def _sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def sample_index(n):
    """The fixed sample of a flattened array of n elements (all of them when n <= WHOLE)."""
    if n <= WHOLE:
        return np.arange(n)
    return np.sort(np.random.RandomState(n % (2 ** 31)).choice(n, NSAMPLE, replace=False))


class Ref:
    def __init__(self, store):
        self.s = store

    def names(self):
        return sorted(k for k in self.s if ":" not in k)

    def scalar(self, key):
        return self.s[key].item()

    def array(self, key):
        """The whole array (only for arrays stored whole)."""
        assert key + ":sha" not in self.s, f"{key} is stored as a sample"
        return self.s[key]

    def assert_equal(self, key, x, what=""):
        """x is bit-identical to the reference's array `key`."""
        a = _np(x)
        assert tuple(a.shape) == tuple(self.s[key + ":shape"]), (what or key, a.shape, self.s[key + ":shape"])
        if key + ":sha" not in self.s:
            assert np.array_equal(a, self.s[key]), f"{what or key} not bit-identical to the reference"
            return
        if _sha(a) != str(self.s[key + ":sha"]):
            mine = a.reshape(-1)[sample_index(a.size)]
            bad = int((mine != self.s[key]).sum())
            raise AssertionError(f"{what or key} not bit-identical to the reference ({bad}/{mine.size} sampled elements differ)")

    def pair(self, key, x):
        """(x's elements, the reference's elements, the reference's largest magnitude) on the stored positions."""
        a = _np(x)
        assert tuple(a.shape) == tuple(self.s[key + ":shape"]), (key, a.shape, self.s[key + ":shape"])
        return a.reshape(-1)[sample_index(a.size)], self.s[key].reshape(-1), float(self.s[key + ":absmax"])


def _pack(vals):
    store = {}
    for k, v in vals.items():
        a = _np(v)
        if a.ndim == 0 or k.startswith("seg_"):  # scalars and the list segments of reference_tile_segments: whole
            store[k] = a
            continue
        store[k + ":shape"] = np.asarray(a.shape, np.int64)
        store[k + ":absmax"] = np.asarray(np.abs(a.astype(np.float64)).max() if a.size else 0.0)
        if a.size <= WHOLE:
            store[k] = a
        else:
            store[k + ":sha"] = np.asarray(_sha(a))
            store[k] = a.reshape(-1)[sample_index(a.size)]
    return store


def reference(name, compute):
    """Ref over the reference's results for test input `name`.  compute() -> {key: tensor / array / scalar} runs the
    reference extension; it is called only when recording."""
    out = os.environ.get("GSR_REF_RECORD")
    if out:
        from oracle import ref_driver
        assert ref_driver.available(), "GSR_REF_RECORD needs the reference extension (python oracle/build_ref.py)"
        store = _pack(compute())
        os.makedirs(out, exist_ok=True)
        np.savez_compressed(os.path.join(out, f"refgold_{name}.npz"), **store)
        return Ref(store)
    path = os.path.join(GOLD, f"refgold_{name}.npz")
    assert os.path.exists(path), f"{path} missing: regenerate it (see tests/refgold.py)"
    return Ref(dict(np.load(path)))
