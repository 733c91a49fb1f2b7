"""Generate tests/golden/create_datasets.npz from the UNMODIFIED reference ``create_datasets.py`` -- TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_create

``create_datasets.py`` imports h5py and tqdm (neither installed here, no network).  Stand-ins are placed in sys.modules:
``h5py.File(name, mode)`` is a context manager that in read mode returns a seeded synthetic raw file (``train`` / ``test``
``images`` and ``timestamps``, from ``raw_files()`` below) and in write mode an in-memory file whose ``create_group`` /
``create_dataset`` / ``resize`` / ``__setitem__`` record what is written; ``special_dtype(vlen=str)`` is ``object`` and
``tqdm`` passes its iterable through.  The reference's ``create_dataset`` then runs unmodified.  Its ``ROOT_DIR`` paths
are only dictionary keys, so nothing is written under the reference.

Stored per case: the parameters, the base name of the file the reference writes, and each split's ``images``; and the raw
frames of every synthetic file.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np

REF = os.environ.get("SMAAT_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "create_datasets.npz")

SIZE = 12                                          # num_pixels 144: 0.2 -> 28.8, 0.29 -> 41.76, 0.5 -> 72
COUNTS = (0, 28, 29, 41, 42, 71, 72, 73, 144)      # rain pixels per frame around those bounds
DRY_COUNTS = (0, 5, 28)                           # below 28.8: no frame qualifies at 0.2
# raw file -> (train frames, test frames, counts the test frames draw from)
RAW = {"mixed": (40, 30, COUNTS), "dry_test": (30, 24, DRY_COUNTS)}
# case -> (raw file, input_length, image_ahead, rain_amount_thresh)
CASES = {
    "l12_a6_t20": ("mixed", 12, 6, 0.2),
    "l12_a6_t50": ("mixed", 12, 6, 0.5),
    "l4_a2_t29": ("mixed", 4, 2, 0.29),            # int(0.29 * 100) == 28 in the file name
    "dry_l4_a2_t20": ("dry_test", 4, 2, 0.2),      # no test frame qualifies: a (0, seq, H, W) dataset
}

_u32 = lambda v: np.uint32(v).view(np.float32)     # noqa: E731
# values counted by `> 0`: ordinary, the smallest and largest positive denormals, the largest finite, +inf
RAIN = np.array([0.25, 1.0, _u32(0x00000001), _u32(0x007fffff), _u32(0x7f7fffff), np.inf], np.float32)
# values not counted: +0, -0, negatives, negative denormals, -inf, quiet / signalling NaNs of either sign with payloads
DRY = np.array([0.0, 0.0, 0.0, -0.0, -0.5, _u32(0x80000001), _u32(0x807fffff), -np.inf, _u32(0x7fc00001), _u32(0xffc01234),
                _u32(0x7f800001), _u32(0xff800002)], np.float32)


def _frames(rng, n, counts):
    """n SIZE x SIZE frames, each with a rain-pixel count drawn from `counts`, values from the RAIN / DRY palettes."""
    out = np.empty((n, SIZE * SIZE), np.float32)
    for f in range(n):
        c = int(rng.choice(counts))
        pos = rng.permutation(SIZE * SIZE)
        out[f] = DRY[rng.integers(0, len(DRY), SIZE * SIZE)]
        out[f, pos[:c]] = RAIN[rng.integers(0, len(RAIN), c)]
    return out.reshape(n, SIZE, SIZE)


def raw_files():
    """{raw file: {split: (n, 12, 12) float32 frames}}, seeded."""
    rng = np.random.default_rng(20261019)
    res = {}
    for name, (n_train, n_test, test_counts) in RAW.items():
        res[name] = {"train": _frames(rng, n_train, COUNTS), "test": _frames(rng, n_test, test_counts)}
    return res


class _Dataset:
    def __init__(self, shape, dtype):
        self.data = np.zeros(shape, dtype=dtype)

    def resize(self, size, axis=0):
        assert axis == 0
        new = np.zeros((size,) + self.data.shape[1:], dtype=self.data.dtype)
        k = min(size, self.data.shape[0])
        new[:k] = self.data[:k]
        self.data = new

    def __setitem__(self, idx, value):
        self.data[idx] = value


class _Group(dict):
    def create_dataset(self, name, shape, maxshape=None, dtype=None, compression=None, compression_opts=None):
        self[name] = _Dataset(shape, dtype)
        return self[name]


class _WriteFile(dict):
    def create_group(self, name):
        self[name] = _Group()
        return self[name]


def _stand_ins(state):
    h5 = types.ModuleType("h5py")

    class File:
        def __init__(self, name, mode="r", **kw):
            if mode == "r":
                self.obj = state["raw"]
            else:
                self.obj = state["written"].setdefault(os.path.basename(str(name)), _WriteFile())

        def __enter__(self):
            return self.obj

        def __exit__(self, *exc):
            return False

    h5.File = File
    h5.special_dtype = lambda vlen=None: object
    tq = types.ModuleType("tqdm")
    tq.tqdm = lambda it, **kw: it
    return h5, tq


def main():
    raws = raw_files()
    state = {"raw": None, "written": {}}
    sys.modules["h5py"], sys.modules["tqdm"] = _stand_ins(state)
    sys.path.insert(0, REF)
    import create_datasets as ref  # noqa: E402

    res = {}
    for name, frames in raws.items():
        for split, a in frames.items():
            res[f"raw/{name}/{split}"] = a
    for case, (raw, L, A, t) in CASES.items():
        fr = raws[raw]
        state["raw"] = {sp: {"images": fr[sp], "timestamps": np.array([[f"{sp}-{i:06d}"] for i in range(len(fr[sp]))], object)}
                        for sp in ("train", "test")}
        state["written"] = {}
        ref.create_dataset(input_length=L, image_ahead=A, rain_amount_thresh=t)
        (fname, f), = state["written"].items()
        res[f"{case}/raw"] = np.str_(raw)
        res[f"{case}/params"] = np.array([L, A, t], np.float64)
        res[f"{case}/file"] = np.str_(fname)
        for sp in ("train", "test"):
            res[f"{case}/{sp}"] = f[sp]["images"].data
        print(case, fname, {sp: f[sp]["images"].data.shape for sp in ("train", "test")})
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
