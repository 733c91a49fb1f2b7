"""-m gpu: the rain-pixel count (smaat_rain_pixels_fwd through ops.rain_pixel_counts) against numpy's `np.sum(frame > 0)`,
exactly, on both load paths and at every position of a 16-byte vector; and create_datasets end to end against the
unmodified reference's datasets (tests/golden/create_datasets.npz) and the host restatement at 288 x 288."""
import os

import numpy as np
import pytest
import torch

from smaat_unet_b200 import create_datasets as CD
from smaat_unet_b200 import ops

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "create_datasets.npz"))
CASES = sorted({k.split("/")[0] for k in GOLD.files if not k.startswith("raw/")})

_u32 = lambda v: np.uint32(v).view(np.float32)     # noqa: E731
EDGES = np.array([0.0, -0.0, np.nan, -np.nan, _u32(0x7fc00001), _u32(0xffc01234), _u32(0x7f800001), _u32(0xff800001),
                  _u32(0x00000001), _u32(0x007fffff), _u32(0x80000001), _u32(0x807fffff), np.inf, -np.inf, 1.0, -1.0,
                  _u32(0x7f7fffff), _u32(0xff7fffff)], np.float32)


def _numpy_counts(frames):
    return np.sum(frames > 0, axis=(1, 2))


def _device_counts(frames, offset=0):
    """Counts of (N, H, W) frames placed `offset` floats into a device buffer (offset 1: no 16-byte alignment)."""
    n = frames.size
    buf = torch.empty(n + offset, device="cuda", dtype=torch.float32)
    buf[offset:].copy_(torch.from_numpy(np.ascontiguousarray(frames).ravel()))
    got = ops.rain_pixel_counts(buf[offset:].view(frames.shape))
    assert got.dtype == torch.int32 and got.shape == (frames.shape[0],)
    return got.cpu().numpy()


def _rainy(rng, n, H, W):
    """Frames with a spread of rain fractions: each pixel rains with the frame's own probability."""
    p = rng.random(n, dtype=np.float32)[:, None, None]
    v = rng.random((n, H, W), dtype=np.float32)
    return np.where(v < p, v + np.float32(0.01), np.float32(0) - v).astype(np.float32)


@pytest.mark.parametrize("offset", [0, 1])
def test_counts_288(offset):
    frames = _rainy(np.random.default_rng(1), 64, 288, 288)
    assert np.array_equal(_device_counts(frames, offset), _numpy_counts(frames))


@pytest.mark.parametrize("shape", [(9, 17, 17), (1, 17, 17), (1, 288, 288), (1, 1, 1), (3, 1, 3), (600, 12, 12)])
def test_counts_odd_planes_and_single_frames(shape):
    frames = _rainy(np.random.default_rng(2), *shape)
    for off in (0, 1, 2, 3):
        assert np.array_equal(_device_counts(frames, off), _numpy_counts(frames)), (shape, off)


def test_counts_edge_values_at_every_vector_position():
    """Frame (value, lane): a 4 x 8 frame of -1 with `value` at every pixel p with p % 4 == lane (16-byte loads) --
    and the same frames starting one float off alignment (4-byte loads)."""
    frames = []
    for v in EDGES:
        for lane in range(4):
            f = np.full(32, -1.0, np.float32)
            f[lane::4] = v
            frames.append(f.reshape(4, 8))
    frames = np.stack(frames)
    want = _numpy_counts(frames)
    assert set(want.tolist()) == {0, 8}
    for off in (0, 1):
        assert np.array_equal(_device_counts(frames, off), want)
    # counted are exactly the positive denormals, the positive normals and +inf
    assert sorted(EDGES[EDGES > 0].view(np.uint32).tolist()) == [0x00000001, 0x007fffff, 0x3f800000, 0x7f7fffff, 0x7f800000]


@pytest.mark.parametrize("case", CASES)
def test_create_datasets_matches_reference(case, tmp_path):
    L, A, t = GOLD[f"{case}/params"].tolist()
    raw = str(GOLD[f"{case}/raw"])
    prefix = str(tmp_path / "frames")
    for sp in ("train", "test"):
        np.save(f"{prefix}_{sp}.npy", GOLD[f"raw/{raw}/{sp}"])
    files = CD.create_datasets(prefix, str(tmp_path / "out"), int(L), int(A), (t,), chunk=5)   # windows span chunks
    stem = os.path.splitext(str(GOLD[f"{case}/file"]))[0]
    for sp in ("train", "test"):
        assert os.path.basename(files[t][sp]) == f"{stem}_{sp}.npy"
        got, want = np.load(files[t][sp]), GOLD[f"{case}/{sp}"]
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_scan_matches_numpy_across_chunk_sizes():
    frames = GOLD["raw/mixed/train"]
    for chunk in (1, 3, 7, 40, 1000):
        assert np.array_equal(CD.scan_rain_pixels(frames, chunk), _numpy_counts(frames)), chunk


def test_create_datasets_288_matches_host_restatement(tmp_path):
    """Every shard holds, in ascending i, the windows frames[i - 18 : i] of the frames whose numpy count passes."""
    rng = np.random.default_rng(3)
    prefix = str(tmp_path / "frames")
    for sp, n in (("train", 60), ("test", 40)):
        np.save(f"{prefix}_{sp}.npy", _rainy(rng, n, 288, 288))
    files = CD.create_datasets(prefix, str(tmp_path / "out"), 12, 6, (0.2, 0.5), chunk=16)
    for sp in ("train", "test"):
        frames = np.load(f"{prefix}_{sp}.npy")
        counts = _numpy_counts(frames)
        for t in (0.2, 0.5):
            idx = [i for i in range(18, frames.shape[0]) if int(counts[i]) >= 288 * 288 * t]
            got = np.load(files[t][sp], mmap_mode="r")
            assert 0 < len(idx) < frames.shape[0] - 18 and got.shape == (len(idx), 18, 288, 288)
            for k, i in enumerate(idx):
                assert np.array_equal(np.asarray(got[k]).view(np.uint32), frames[i - 18:i].view(np.uint32))
