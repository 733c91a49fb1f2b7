"""CPU-side checks of the serving heads: UNet / UNetAttention offer the serving forward InferenceSession looks up, and the
blocks refuse an unknown head before any CUDA call."""
import pytest
import torch

import smaat_unet_b200 as S


def test_dense_models_offer_the_serving_forward():
    for cls in (S.UNet, S.UNetAttention):
        for bilinear in (True, False):
            m = cls(3, 21, bilinear)
            for name in ("forward_serving", "forward_classes", "forward_probs"):
                assert callable(getattr(m, name, None)), f"{cls.__name__}.{name}"


def test_blocks_refuse_an_unknown_head_before_touching_a_tensor():
    # CPU tensors: a check that reached them would raise RuntimeError (no CPU fallback), not ValueError
    x, low, oc = torch.zeros(1, 64, 8, 8), torch.zeros(1, 128, 4, 4), S.OutConv(64, 3)
    calls = {"DoubleConv.run": lambda **kw: S.DoubleConv(64, 64).run(x, **kw),
             "DoubleConvDS.run": lambda **kw: S.DoubleConvDS(64, 64).run(x, **kw),
             "Up.forward": lambda **kw: S.Up(128, 64)(low, x, **kw),
             "UpDS.forward": lambda **kw: S.UpDS(128, 64)(low, x, **kw)}
    for call in calls.values():
        for head in ("class", "logit", "argmax", None):
            with pytest.raises(ValueError, match="head must be one of"):
                call(outconv=oc, head=head)
        for head in ("classes", "probs"):
            with pytest.raises(ValueError, match="needs the OutConv"):
                call(head=head)
