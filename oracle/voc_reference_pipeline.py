"""The reference's VOC training input pipeline, restated for timing -- MEASUREMENT INFRASTRUCTURE ONLY.

What `VOCSegmentation.__getitem__` does per sample when train_SmaAtUNet.py:149-173 builds it (transformations
Resize(256) + CenterCrop(224), augmentations on, DataLoader num_workers=0): decode the JPEG and the PNG with PIL, run the
transformations on both, the random hflip / +-10 degree rotation / x1.2 or x0.8 brightness (utils/dataset_VOC.py:150-168,
the same module-level `random` draws), ToTensor + Normalize(ImageNet mean / std), and `target[target == 255] = 0`.
tools/bench_voc_input.py times it where the reference tree is not available.  Needs PIL and torchvision.
"""
from __future__ import annotations

import os
import random

import numpy as np
import torch
from torch.utils.data import Dataset


class VOCReferencePipeline(Dataset):
    def __init__(self, root, image_set="train", augmentations=True):
        from torchvision import transforms
        voc = os.path.join(os.fspath(root), "VOC2012")
        with open(os.path.join(voc, "ImageSets", "Segmentation", image_set + ".txt")) as f:
            names = [n.strip() for n in f]
        self.images = [os.path.join(voc, "JPEGImages", n + ".jpg") for n in names]
        self.masks = [os.path.join(voc, "SegmentationClass", n + ".png") for n in names]
        self.crop = transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224)])
        self.to_tensor = transforms.Compose([transforms.ToTensor(),
                                             transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
        self.augmentations = augmentations

    def __len__(self):
        return len(self.images)

    @staticmethod
    def augment(img, mask):
        import torchvision.transforms.functional as TF
        if random.random() > 0.5:
            img, mask = TF.hflip(img), TF.hflip(mask)
        if random.random() > 0.5:
            deg = -10 if random.random() > 0.5 else 10
            img, mask = TF.rotate(img, deg), TF.rotate(mask, deg)
        if random.random() > 0.5:
            img = TF.adjust_brightness(img, 1.2 - 0.4 if random.random() > 0.5 else 1.2)
        return img, mask

    def __getitem__(self, index):
        from PIL import Image
        img = self.crop(Image.open(self.images[index]).convert("RGB"))
        mask = self.crop(Image.open(self.masks[index]))
        if self.augmentations:
            img, mask = self.augment(img, mask)
        target = torch.from_numpy(np.array(mask)).long()
        target[target == 255] = 0
        return self.to_tensor(img), target
