"""CPU checks of the VOC input path: the host-side draws and the CPU restatement of the reference's augmentations against the
golden outputs of the unmodified reference (tests/golden/voc_augment.npz, oracle/make_golden_voc.py), the one-off shard
conversion, and the loader's uint8 batches with their augmentation rows."""
import os
import random

import numpy as np
import pytest
import torch

from smaat_unet_b200 import data as D

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voc_augment.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _aug_cases(g):
    for si in range(2):
        for k in range(int(g[f"aug/{si}/n"])):
            yield f"aug/{si}/{k}"


def _write_shard(prefix, imgs, masks):
    np.save(f"{prefix}_images.npy", np.ascontiguousarray(imgs, np.uint8))
    np.save(f"{prefix}_masks.npy", np.ascontiguousarray(masks, np.uint8))


def test_fixture_covers_every_combination(gold):
    for si in range(2):
        got = {tuple(gold[f"aug/{si}/{k}/choice"]) for k in range(int(gold[f"aug/{si}/n"]))}
        assert got == {(f, r, b) for f in (0, 1) for r in (-1, 0, 1) for b in (-1, 0, 1)}


def test_draws_and_cpu_augmentation_reproduce_reference(gold):
    for p in _aug_cases(gold):
        choice = D.voc_segmentation_shard.draw_augmentation(random.Random(int(gold[p + "/seed"])))
        assert choice == tuple(int(v) for v in gold[p + "/choice"]), p
        img, mask = D.voc_augment_u8(gold[p + "/img"], gold[p + "/mask"], choice)
        np.testing.assert_array_equal(img, gold[p + "/out_img"], err_msg=p)
        np.testing.assert_array_equal(mask, gold[p + "/out_mask"], err_msg=p)


def test_draw_count_follows_reference_conditions():
    class Counting(random.Random):
        n = 0

        def random(self):
            Counting.n += 1
            return super().random()

    counts = set()
    rng = Counting(5)
    for _ in range(200):
        Counting.n = 0
        D.voc_segmentation_shard.draw_augmentation(rng)
        counts.add(Counting.n)
    assert counts == {3, 4, 5}


def test_shard_getitem_matches_reference_getitem(gold, tmp_path):
    for i in range(2):
        p = f"item/{i}"
        _write_shard(tmp_path / "voc", gold[p + "/img_u8"][None], gold[p + "/mask_u8"][None])
        ds = D.voc_segmentation_shard(tmp_path / "voc", augmentations=True, seed=int(gold[p + "/seed"]))
        assert len(ds) == 1
        x, y = ds[0]
        assert x.dtype == torch.float32 and y.dtype == torch.int64
        np.testing.assert_array_equal(x.numpy().view(np.int32), gold[p + "/x"].view(np.int32), err_msg=p)
        np.testing.assert_array_equal(y.numpy(), gold[p + "/y"], err_msg=p)
        assert (gold[p + "/mask_u8"] == 255).any() and gold[p + "/choice"][1] != 0


def test_shard_without_augmentations_only_normalises(gold, tmp_path):
    p = "item/0"
    _write_shard(tmp_path / "voc", gold[p + "/img_u8"][None], gold[p + "/mask_u8"][None])
    x, y = D.voc_segmentation_shard(tmp_path / "voc")[0]
    ref = (torch.from_numpy(gold[p + "/img_u8"]).permute(2, 0, 1).float() / 255 - torch.tensor(D.VOC_MEAN)[:, None, None]) \
        / torch.tensor(D.VOC_STD)[:, None, None]
    assert torch.equal(x, ref)
    t = torch.from_numpy(gold[p + "/mask_u8"]).long()
    t[t == 255] = 0
    assert torch.equal(y, t)


@pytest.mark.parametrize("hw", [(1, 40000), (40000, 1), (1, 1), (2, 3), (37, 29)])
def test_rotation_source_matches_pil(hw):
    Image = pytest.importorskip("PIL.Image")
    h, w = hw
    rng = np.random.default_rng(h * 7 + w)
    m = rng.integers(0, 256, (h, w), dtype=np.uint8)
    for deg in (10, -10):
        ref = np.asarray(Image.fromarray(m).rotate(deg, Image.NEAREST, False, None, fillcolor=0))
        got = D.voc_augment_u8(np.repeat(m[..., None], 3, 2), m, (0, 1 if deg > 0 else -1, 0))[1]
        np.testing.assert_array_equal(got, ref)


def test_convert_voc_equals_reference_transformations(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    transforms = pytest.importorskip("torchvision.transforms")
    voc = tmp_path / "VOC2012"
    for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation"):
        (voc / d).mkdir(parents=True)
    rng = np.random.default_rng(3)
    names = ["b", "a", "c"]                     # split-file order, not sorted
    for n, (h, w) in zip(names, [(300, 400), (260, 333), (224, 224)]):
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(voc / "JPEGImages" / f"{n}.jpg")
        Image.fromarray(rng.integers(0, 21, (h, w), dtype=np.uint8), mode="P").save(voc / "SegmentationClass" / f"{n}.png")
    (voc / "ImageSets" / "Segmentation" / "train.txt").write_text("\n".join(names) + "\n")
    pi, pm = D.convert_voc(tmp_path, "train", str(tmp_path / "shard"))
    imgs, masks = np.load(pi), np.load(pm)
    assert imgs.shape == (3, 224, 224, 3) and masks.shape == (3, 224, 224) and imgs.dtype == masks.dtype == np.uint8
    tf = transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224)])
    for i, n in enumerate(names):
        np.testing.assert_array_equal(imgs[i], np.asarray(tf(Image.open(voc / "JPEGImages" / f"{n}.jpg").convert("RGB"))))
        np.testing.assert_array_equal(masks[i], np.asarray(tf(Image.open(voc / "SegmentationClass" / f"{n}.png"))))
    assert len(D.voc_segmentation_shard(tmp_path / "shard")) == 3


def _small_shard(tmp_path, n=13, h=5, w=7):
    rng = np.random.default_rng(11)
    imgs = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    masks = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
    _write_shard(tmp_path / "s", imgs, masks)
    return imgs, masks


def _epoch(loader):
    out = []
    for b in loader:
        out.append(tuple(t.clone() for t in b))
    return out


def test_loader_carries_uint8_batches_and_aug_rows(tmp_path):
    imgs, masks = _small_shard(tmp_path)
    ds = D.voc_segmentation_shard(tmp_path / "s", augmentations=True)
    loader = D.PinnedBatchLoader(ds, 4, shuffle=True, seed=2, drop_last=False, pin_memory=False)
    batches = _epoch(loader)
    assert [b[0].shape[0] for b in batches] == [4, 4, 4, 1]
    rng = loader.augmentation_rng()
    order = loader.epoch_indices()
    for bi, (x, y, aug) in enumerate(batches):
        assert x.dtype == torch.uint8 and y.dtype == torch.uint8 and aug.dtype == torch.int8
        assert aug.shape == (x.shape[0], 3)
        for j in range(x.shape[0]):
            i = order[bi * 4 + j]
            assert np.array_equal(x[j].numpy(), imgs[i]) and np.array_equal(y[j].numpy(), masks[i])
            assert tuple(aug[j].tolist()) == ds.draw_augmentation(rng)
    plain = D.PinnedBatchLoader(D.voc_segmentation_shard(tmp_path / "s"), 4, pin_memory=False)
    assert all(len(b) == 2 and b[0].dtype == torch.uint8 for b in _epoch(plain))


def test_loader_aug_rows_are_deterministic_per_epoch_and_rank(tmp_path):
    _small_shard(tmp_path, n=16)

    def run(epoch, rank, world=2):
        ds = D.voc_segmentation_shard(tmp_path / "s", augmentations=True)
        ld = D.PinnedBatchLoader(ds, 4, shuffle=True, seed=9, rank=rank, world=world, pin_memory=False)
        ld.set_epoch(epoch)
        return ld.epoch_indices(), torch.cat([b[2] for b in _epoch(ld)])

    i0, a0 = run(0, 0)
    i1, a1 = run(0, 1)
    assert sorted(i0 + i1) == list(range(16)) and not set(i0) & set(i1)
    j0, b0 = run(0, 0)
    assert i0 == j0 and torch.equal(a0, b0)                   # same seed, epoch and rank: same order and choices
    assert not torch.equal(a0, a1)                            # ranks draw from their own generators
    k0, c0 = run(1, 0)
    assert not torch.equal(a0, c0)                            # so do epochs


def test_voc_shard_rejects_bad_layout(tmp_path):
    _write_shard(tmp_path / "bad", np.zeros((2, 4, 4, 3), np.uint8), np.zeros((2, 4, 5), np.uint8))
    with pytest.raises(ValueError):
        D.voc_segmentation_shard(tmp_path / "bad")
