"""CPU checks of the precipitation dataset builder (smaat_unet_b200.create_datasets) against the unmodified reference's
create_datasets.py (tests/golden/create_datasets.npz, oracle/make_golden_create.py): selection and writing fed numpy's
rain-pixel counts, the file names, the refusal of non-square frames, the shards read back through
precipitation_maps_oversampled_shard, and the C entry point's argument checks."""
import ctypes
import os

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from smaat_unet_b200 import create_datasets as CD
from smaat_unet_b200 import ops
from smaat_unet_b200.data import precipitation_maps_oversampled_shard

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "create_datasets.npz"))
CASES = sorted({k.split("/")[0] for k in GOLD.files if not k.startswith("raw/")})
SPLITS = ("train", "test")


def _case(case):
    L, A, t = GOLD[f"{case}/params"].tolist()
    return str(GOLD[f"{case}/raw"]), int(L), int(A), t


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _numpy_counts(frames):
    return np.sum(frames > 0, axis=(1, 2))


def test_golden_covers_the_edges():
    frames = GOLD["raw/mixed/train"]
    counts = set(_numpy_counts(np.concatenate([GOLD["raw/mixed/train"], GOLD["raw/mixed/test"]])).tolist())
    assert {0, 28, 29, 41, 42, 71, 72, 73, 144} <= counts
    b = set(_bits(frames).ravel().tolist())
    assert {0x00000001, 0x80000000, 0x80000001, 0x7f800000, 0xff800000, 0x7fc00001, 0xffc01234, 0x7f800001} <= b
    assert GOLD["dry_l4_a2_t20/test"].shape == (0, 6, 12, 12)


@pytest.mark.parametrize("case", CASES)
def test_host_selection_and_writing_match_reference(case, tmp_path):
    raw, L, A, t = _case(case)
    for sp in SPLITS:
        frames = GOLD[f"raw/{raw}/{sp}"]
        res, nbytes = CD.write_split(frames, _numpy_counts(frames), str(tmp_path), sp, L, A, (t,))
        path, n = res[t]
        stem = os.path.splitext(str(GOLD[f"{case}/file"]))[0]
        assert os.path.basename(path) == f"{stem}_{sp}.npy"
        got, want = np.load(path), GOLD[f"{case}/{sp}"]
        assert got.dtype == np.float32 and got.shape == want.shape and n == want.shape[0]
        assert np.array_equal(_bits(got), _bits(want))
        assert nbytes == want.nbytes


def test_every_threshold_from_one_pass(tmp_path):
    """0.2 and 0.5 written in one call give the reference's two separate runs."""
    frames = GOLD["raw/mixed/train"]
    res, _ = CD.write_split(frames, _numpy_counts(frames), str(tmp_path), "train", 12, 6, (0.2, 0.5))
    for t, case in ((0.2, "l12_a6_t20"), (0.5, "l12_a6_t50")):
        assert np.array_equal(_bits(np.load(res[t][0])), _bits(GOLD[f"{case}/train"]))


def test_file_name_formula():
    assert CD.dataset_file_name(4, 2, 0.29, "test") == "train_test_2016-2019_input-length_4_img-ahead_2_rain-threshold_28_test.npy"
    assert CD.dataset_file_name(12, 6, 0.5, "train") == "train_test_2016-2019_input-length_12_img-ahead_6_rain-threshold_50_train.npy"


def test_selection_window_ends_before_the_tested_frame():
    """Frame i passes the test and the window is images[i - seq : i]: its target is frame i - 1; num_pixels is H * H."""
    counts = np.zeros(10, np.int64)
    counts[7] = 29                       # 0.2 * 144 = 28.8
    assert CD.select_indices(counts, 2, 1, 0.2, 12).tolist() == [7]
    counts[7] = 28
    assert CD.select_indices(counts, 2, 1, 0.2, 12).tolist() == []
    counts[:] = 144
    assert CD.select_indices(counts, 2, 1, 0.2, 12).tolist() == list(range(3, 10))


def _write_frames(prefix, shapes):
    for sp, shape in shapes.items():
        np.save(f"{prefix}_{sp}.npy", np.ones(shape, np.float32))


@pytest.mark.parametrize("shapes", [{"train": (30, 12, 10), "test": (30, 12, 10)},
                                    {"train": (30, 12, 12), "test": (30, 10, 12)},
                                    {"train": (30, 12, 12), "test": (30, 10, 10)}])
def test_non_square_or_mismatched_frames_raise_before_writing(tmp_path, shapes):
    prefix = str(tmp_path / "frames")
    _write_frames(prefix, shapes)
    out = tmp_path / "out"
    with pytest.raises(ValueError):
        CD.create_datasets(prefix, str(out), 4, 2)
    assert not out.exists()


@pytest.mark.parametrize("case", ["l12_a6_t20", "l4_a2_t29"])
def test_oversampled_shard_reads_written_samples(case, tmp_path):
    raw, L, A, t = _case(case)
    frames = GOLD[f"raw/{raw}/train"]
    res, _ = CD.write_split(frames, _numpy_counts(frames), str(tmp_path), "train", L, A, (t,))
    ds = precipitation_maps_oversampled_shard(res[t][0], L, A, train=True)
    want = GOLD[f"{case}/train"]
    assert len(ds) == want.shape[0] > 0
    for i in range(len(ds)):
        x, y = ds[i]
        assert np.array_equal(_bits(x), _bits(want[i, :L])) and np.array_equal(_bits(y), _bits(want[i, -1]))


def test_rain_pixels_refuses_bad_arguments():
    lib = S._lib.load()
    fake = ctypes.c_void_p(256)              # never dereferenced: the checks run before any launch
    for args in ((None, 1, 4, fake, None), (fake, 1, 4, None, None), (fake, 0, 4, fake, None), (fake, -1, 4, fake, None),
                 (fake, 1, 0, fake, None), (fake, 1, 1 << 31, fake, None)):
        assert lib.smaat_rain_pixels_fwd(*args) == -1
        assert b"rain_pixels" in lib.smaat_last_error()


def test_rain_pixel_counts_has_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.rain_pixel_counts(torch.zeros(2, 4, 4))


def test_thresholds_sharing_a_file_name_raise_before_writing(tmp_path):
    prefix = str(tmp_path / "frames")
    _write_frames(prefix, {"train": (30, 12, 12), "test": (30, 12, 12)})
    with pytest.raises(ValueError, match="share a file name"):
        CD.create_datasets(prefix, str(tmp_path / "out"), 4, 2, (0.2, 0.205))
    assert not (tmp_path / "out").exists()


def test_command_line_defaults():
    a = CD.parse_args(["--frames-prefix", "p", "--out-dir", "o"])
    assert (a.input_length, a.image_ahead, a.thresholds, a.splits, a.chunk) == (12, 6, [0.2, 0.5], ["train", "test"], 256)
