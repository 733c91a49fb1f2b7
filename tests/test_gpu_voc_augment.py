"""-m gpu: the VOC input kernel (smaat_voc_augment_fwd through ops.voc_augment) against the unmodified reference's outputs
(tests/golden/voc_augment.npz) and the CPU restatement in data.py, bit for bit, and a TrainSession fed uint8 batches through
ops.VOCNormalize against a twin session fed the CPU path's fp32 / int64 batches."""
import itertools
import os

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from smaat_unet_b200 import data as D
from smaat_unet_b200 import ops
from smaat_unet_b200.train import TrainSession

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voc_augment.npz")
COMBOS = list(itertools.product((0, 1), (-1, 0, 1), (-1, 0, 1)))


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


def _cpu_batch(imgs, masks, augs):
    """The reference's samples through the CPU restatement: (B, 3, H, W) fp32, (B, H, W) int64."""
    xs, ys = [], []
    for img, mask, a in zip(imgs, masks, augs):
        x, y = D.voc_normalize_u8(*D.voc_augment_u8(img, mask, tuple(int(v) for v in a)))
        xs.append(x)
        ys.append(y)
    return torch.stack(xs), torch.stack(ys)


def _run(imgs, masks, augs, **kw):
    aug = None if augs is None else torch.as_tensor(np.asarray(augs), dtype=torch.int8).cuda()
    return ops.voc_augment(torch.from_numpy(np.ascontiguousarray(imgs)).cuda(), torch.from_numpy(np.ascontiguousarray(masks)).cuda(),
                           aug, **kw)


def _assert_same(got, want):
    (gx, gy), (wx, wy) = got, want
    assert gx.shape == wx.shape and gx.dtype == torch.float32 and gy.dtype == torch.int64
    assert torch.equal(_bits(gx), _bits(wx)), "image differs"
    assert torch.equal(gy.cpu(), wy), "target differs"


def test_kernel_reproduces_reference_augmentations():
    g = np.load(GOLD)
    for si in range(2):
        keys = [f"aug/{si}/{k}" for k in range(int(g[f"aug/{si}/n"]))]
        imgs, masks = np.stack([g[k + "/img"] for k in keys]), np.stack([g[k + "/mask"] for k in keys])
        augs = np.stack([g[k + "/choice"] for k in keys])
        # the reference's uint8 results, normalised: v -> (v / 255 - m) / s is one-to-one, so equal fp32 means equal uint8
        want = torch.stack([D.voc_normalize_u8(g[k + "/out_img"], g[k + "/out_mask"])[0] for k in keys])
        want_y = torch.stack([torch.from_numpy(np.where(g[k + "/out_mask"] == 255, 0, g[k + "/out_mask"]).astype(np.int64))
                              for k in keys])
        _assert_same(_run(imgs, masks, augs), (want, want_y))


def test_kernel_reproduces_reference_getitem():
    g = np.load(GOLD)
    for i in range(2):
        p = f"item/{i}"
        got = _run(g[p + "/img_u8"][None], g[p + "/mask_u8"][None], g[p + "/choice"][None])
        _assert_same(got, (torch.from_numpy(g[p + "/x"])[None], torch.from_numpy(g[p + "/y"])[None]))


@pytest.mark.parametrize("hw", [(1, 1), (1, 9), (9, 1), (2, 3), (31, 33), (13, 250), (227, 221), (224, 224)])
def test_mixed_batches_at_odd_sizes(hw):
    h, w = hw
    rng = np.random.default_rng(h * 1000 + w)
    order = rng.permutation(len(COMBOS))
    augs = np.array([COMBOS[i] for i in order], dtype=np.int8)
    imgs = rng.integers(0, 256, (len(augs), h, w, 3), dtype=np.uint8)
    masks = rng.integers(0, 256, (len(augs), h, w), dtype=np.uint8)
    masks[:, ::2] = 255
    _assert_same(_run(imgs, masks, augs), _cpu_batch(imgs, masks, augs))


@pytest.mark.parametrize("hw", [(1, 40000), (40000, 1)])
def test_double_precision_walk(hw):
    """Sizes whose corners map outside PIL's fixed-point range: PIL walks the rows in doubles."""
    h, w = hw
    rng = np.random.default_rng(7)
    augs = np.array([(0, 1, 0), (1, -1, 1), (0, -1, -1)], dtype=np.int8)
    imgs = rng.integers(0, 256, (3, h, w, 3), dtype=np.uint8)
    masks = rng.integers(0, 256, (3, h, w), dtype=np.uint8)
    _assert_same(_run(imgs, masks, augs), _cpu_batch(imgs, masks, augs))


def test_no_augmentation_and_strided_outputs():
    rng = np.random.default_rng(3)
    B, H, W = 5, 17, 23
    imgs = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    masks = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
    want = _cpu_batch(imgs, masks, np.zeros((B, 3), np.int8))
    _assert_same(_run(imgs, masks, None), want)
    bx = torch.full((B, 5, H, W), -7.0, device="cuda")
    by = torch.full((B, 2, H, W), -7, device="cuda", dtype=torch.int64)
    augs = np.array([COMBOS[i] for i in (17, 3, 9, 0, 12)], dtype=np.int8)
    x, y = _run(imgs, masks, augs, out_x=bx[:, 1:4], out_y=by[:, 1])
    assert x.data_ptr() == bx[:, 1:4].data_ptr() and y.data_ptr() == by[:, 1].data_ptr()
    _assert_same((bx[:, 1:4], by[:, 1]), _cpu_batch(imgs, masks, augs))
    assert (bx[:, 0] == -7).all() and (bx[:, 4] == -7).all() and (by[:, 0] == -7).all()
    mean, std = (0.5, 0.25, 0.125), (0.3, 0.2, 0.1)
    x, _ = _run(imgs, masks, augs, mean=mean, std=std)
    want = torch.stack([D.voc_normalize_u8(D.voc_augment_u8(i, m, tuple(a))[0], m, mean, std)[0] for i, m, a in zip(imgs, masks, augs)])
    assert torch.equal(_bits(x), _bits(want))


def test_bad_arguments_raise():
    x = torch.zeros(2, 4, 4, 3, dtype=torch.uint8, device="cuda")
    y = torch.zeros(2, 4, 4, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        ops.voc_augment(x.float(), y)
    with pytest.raises(ValueError):
        ops.voc_augment(x, y[:1])
    with pytest.raises(ValueError):
        ops.voc_augment(x, y, torch.zeros(2, 3, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError):
        ops.voc_augment(x, y, out_x=torch.empty(2, 4, 4, 3, device="cuda"))


def _voc_shard(tmp_path, n, seed=0):
    rng = np.random.default_rng(seed)
    imgs = rng.integers(0, 256, (n, 224, 224, 3), dtype=np.uint8)
    masks = rng.integers(0, 21, (n, 224, 224), dtype=np.uint8)
    masks[:, :8] = 255
    masks[:, :, -5:] = 255
    np.save(tmp_path / "voc_images.npy", imgs)
    np.save(tmp_path / "voc_masks.npy", masks)
    return D.voc_segmentation_shard(tmp_path / "voc", augmentations=True)


def test_train_session_on_uint8_batches_matches_fp32_twin(tmp_path):
    """Two epochs of 11 samples at batch 8 (steps of 8 and 3 rows) from the pinned loader, guarded by last_h2d_event.  The
    static inputs the captured graphs read are bitwise those of the twin session fed the CPU path's fp32 / int64 batches.
    Each step starts the twin from the session's state; loss, gradient bucket and IoU counts then agree up to the order of
    the atomically merged sums in the BatchNorm statistics and the backward (the bound TrainSession's own two-phase check
    uses for that noise)."""
    ds = _voc_shard(tmp_path, 11)
    torch.manual_seed(0)
    m0 = S.SmaAt_UNet(3, 21)
    m1 = S.SmaAt_UNet(3, 21)
    m1.load_state_dict(m0.state_dict())
    sess = TrainSession(m0, 8, (3, 224, 224), loss="cross_entropy", input_transform=ops.VOCNormalize())
    twin = TrainSession(m1, 8, (3, 224, 224), loss="cross_entropy")
    loader = D.PinnedBatchLoader(ds, 8, shuffle=True, seed=4, drop_last=False)
    rows = []
    for epoch in range(2):
        loader.set_epoch(epoch)
        for x, y, aug in loader:
            assert x.is_pinned() and aug.is_pinned()
            xf, yf = _cpu_batch(x.numpy(), y.numpy(), aug.numpy())      # taken before the step: the slot is still ours
            with torch.no_grad():
                for a, b in zip([twin.flat_param, twin.exp_avg, twin.exp_avg_sq, twin.opt_step] + list(twin.model.buffers()),
                                [sess.flat_param, sess.exp_avg, sess.exp_avg_sq, sess.opt_step] + list(sess.model.buffers())):
                    a.copy_(b)
            ops.bump_weights_generation()
            loss = sess.step(x, y, aug=aug)
            loader.guard(sess.last_h2d_event())
            loss_t = twin.step(xf, yf)
            n = x.shape[0]
            rows.append(n)
            torch.cuda.synchronize()
            assert torch.equal(_bits(sess.x[:n]), _bits(twin.x[:n])) and torch.equal(sess.y[:n], twin.y[:n])
            assert torch.equal(_bits(sess.x[:n]), _bits(xf)) and torch.equal(sess.y[:n].cpu(), yf)
            assert abs(float(loss) - float(loss_t)) <= 1e-5 * abs(float(loss_t))
            scale = float(twin.flat_grad.abs().max())
            assert float((sess.flat_grad - twin.flat_grad).abs().max()) <= 1e-3 * scale
            a, b = sess.metrics.totals_snapshot().double(), twin.metrics.totals_snapshot().double()
            assert float((a - b).abs().sum()) <= 1e-4 * float(b.abs().sum())
    assert rows == [8, 3, 8, 3]


def test_train_session_input_checks():
    m = S.SmaAt_UNet(3, 21)
    with pytest.raises(ValueError):
        TrainSession(m, 2, (3, 32, 32), input_transform=ops.VOCNormalize())              # MSE: no class-index target
    sess = TrainSession(m, 2, (3, 32, 32), loss="cross_entropy", input_transform=ops.VOCNormalize())
    x = torch.zeros(2, 32, 32, 3, dtype=torch.uint8)
    y = torch.zeros(2, 32, 32, dtype=torch.uint8)
    with pytest.raises(ValueError):
        sess.step(x.float(), y)
    with pytest.raises(ValueError):
        sess.step(x, y, aug=torch.zeros(1, 3, dtype=torch.int8))
    sess.step(x.cuda(), y.cuda(), aug=torch.tensor([[1, 1, 1], [0, -1, -1]], dtype=torch.int8).cuda())
    want = _cpu_batch(x.numpy(), y.numpy(), [(1, 1, 1), (0, -1, -1)])
    _assert_same((sess.x, sess.y), want)
    plain = TrainSession(S.SmaAt_UNet(3, 21), 2, (3, 32, 32), loss="cross_entropy")
    with pytest.raises(TypeError):
        plain.step(x, y)
