"""Generate tests/golden/voc_augment.npz from the UNMODIFIED reference VOC dataset -- TEST INFRASTRUCTURE ONLY.

    SMAAT_REFERENCE=/path/to/SmaAt-UNet python -m oracle.make_golden_voc

Needs PIL and torchvision.  `utils/dataset_VOC.py` imports matplotlib for a plotting helper the dataset never calls; when
matplotlib is missing, an empty stand-in module is placed in sys.modules.  Two parts:

  * aug/<size>/<k>: `VOCSegmentation.apply_augmentations` called directly on seeded uint8 RGB images and P-mode masks at odd,
    non-square sizes, after `random.seed(seed)`.  Seeds are chosen so that all 18 (flip, rotation, brightness) combinations
    occur; which one a seed gave is recorded by wrapping the module's `TF.hflip` / `TF.rotate` / `TF.adjust_brightness`
    (the calls go through unchanged).  Stored: inputs, seed, recorded choice, augmented uint8 outputs.
  * item/<k>: `VOCSegmentation.__getitem__` with the training script's transformations (Resize(256) + CenterCrop(224),
    train_SmaAtUNet.py:149) and augmentations on, over a synthetic JPEG / P-mode PNG tree, after `random.seed(seed)`.
    Stored: the post-transformation uint8 image and mask (decoded in this process), seed, choice, and the returned fp32
    image and int64 target.  The masks carry 255 borders and the seeds rotate, so fill enters the frame.
"""
from __future__ import annotations

import os
import random
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

REF = os.environ.get("SMAAT_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "voc_augment.npz")
SIZES = ((29, 37), (48, 31))          # (H, W): PIL sizes 37x29 and 31x48
ITEM_SEEDS = 2


def _palette_mask(rng, h, w, block=1):
    from PIL import Image
    m = rng.integers(0, 21, (-(-h // block), -(-w // block)), dtype=np.uint8).repeat(block, 0).repeat(block, 1)[:h, :w].copy()
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = 255              # VOC's "void" border
    m[h // 3: h // 3 + 2, :] = 255
    im = Image.fromarray(m, mode="P")
    im.putpalette(list(rng.integers(0, 256, 768, dtype=np.uint8)))
    return im


class _Spy:
    """Stands in for the module's `TF`: records which augmentation ran, then calls torchvision's function."""

    def __init__(self, tf):
        self.tf, self.calls = tf, []

    def hflip(self, img):
        self.calls.append(("flip", 1))
        return self.tf.hflip(img)

    def rotate(self, img, angle, *a, **k):
        self.calls.append(("rot", 1 if angle > 0 else -1))
        return self.tf.rotate(img, angle, *a, **k)

    def adjust_brightness(self, img, f):
        self.calls.append(("bright", 1 if f > 1 else -1))
        return self.tf.adjust_brightness(img, f)

    def choice(self):
        d = dict(self.calls)                                    # image and mask calls carry the same value
        return np.array([d.get("flip", 0), d.get("rot", 0), d.get("bright", 0)], dtype=np.int8)


def main():
    from PIL import Image
    from torchvision import transforms

    if "matplotlib" not in sys.modules:
        try:
            import matplotlib.pyplot  # noqa: F401
        except ImportError:
            mpl = types.ModuleType("matplotlib")
            mpl.pyplot = types.ModuleType("matplotlib.pyplot")
            sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot
    sys.path.insert(0, REF)
    from utils import dataset_VOC as D  # noqa: E402
    spy = _Spy(D.TF)
    D.TF = spy
    res = {}
    rng = np.random.default_rng(20261017)
    ds = D.VOCSegmentation.__new__(D.VOCSegmentation)         # apply_augmentations reads no instance state
    for si, (h, w) in enumerate(SIZES):
        seen, seed, k = set(), 0, 0
        while len(seen) < 18:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            mask = _palette_mask(rng, h, w)
            while True:                                        # next seed that gives a combination not seen yet
                spy.calls.clear()
                random.seed(seed)
                ai, am = ds.apply_augmentations(Image.fromarray(img), mask)
                seed += 1
                c = tuple(spy.choice())
                if c not in seen:
                    break
            seen.add(c)
            p = f"aug/{si}/{k}"
            res[p + "/img"], res[p + "/mask"] = img, np.asarray(mask)
            res[p + "/seed"], res[p + "/choice"] = np.int64(seed - 1), spy.choice()
            res[p + "/out_img"], res[p + "/out_mask"] = np.asarray(ai), np.asarray(am)
            k += 1
        res[f"aug/{si}/n"] = np.int64(k)
    tf = transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224)])
    with tempfile.TemporaryDirectory() as tmp:
        voc = Path(tmp) / "VOC2012"
        for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation"):
            (voc / d).mkdir(parents=True)
        names = []
        for i, (h, w) in enumerate(((300, 400), (333, 260))):
            yy, xx = np.mgrid[0:h, 0:w]
            img = np.stack([(xx * 255 // w), (yy * 255 // h), ((xx + yy) * 7) % 256], -1).astype(np.uint8)
            Image.fromarray(img).save(voc / "JPEGImages" / f"s{i}.jpg", quality=90)
            _palette_mask(rng, h, w, block=24).save(voc / "SegmentationClass" / f"s{i}.png")
            names.append(f"s{i}")
        (voc / "ImageSets" / "Segmentation" / "train.txt").write_text("\n".join(names) + "\n")
        vds = D.VOCSegmentation(Path(tmp), image_set="train", transformations=tf, augmentations=True)
        seed = 0
        for i in range(len(names)):
            while True:                                        # a seed that rotates (and, for the first, flips and brightens)
                spy.calls.clear()
                random.seed(seed)
                x, t = vds[i]
                c = spy.choice()
                seed += 1
                if c[1] != 0 and (i > 0 or (c[0] == 1 and c[2] == 1)) and (i == 0 or c[2] == -1):
                    break
            p = f"item/{i}"
            res[p + "/img_u8"] = np.asarray(tf(Image.open(vds.images[i]).convert("RGB")))
            res[p + "/mask_u8"] = np.asarray(tf(Image.open(vds.masks[i])))
            res[p + "/seed"], res[p + "/choice"] = np.int64(seed - 1), c
            res[p + "/x"], res[p + "/y"] = x.numpy(), t.numpy()
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, len(res), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
