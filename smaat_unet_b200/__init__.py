"""smaat_unet_b200 -- H100 (sm_90a) implementation of the SmaAt-UNet forward hot path.

Drop-in ``nn.Module`` replacements for the reference's DS-conv blocks, dense UNet blocks and CBAM
(``modules``), the same model assemblies (``model.SmaAt_UNet``, ``model.UNetDS``, ``model.UNetDSAttention4CBAMs``, ``model.UNet``,
``model.UNetAttention``), a helper that rebinds the
reference's own classes (``patch_reference``), and the functional kernel wrappers (``ops``).
All arithmetic runs in ``libsmaat_b200.so`` (C ABI: ``include/smaat_b200.h``).
"""
from . import _lib, ops  # noqa: F401
from .data import (PinnedBatchLoader, convert_voc, precipitation_maps_classification_shard,  # noqa: F401
                   precipitation_maps_oversampled_shard, precipitation_maps_shard, voc_segmentation_shard)
from .metrics import PrecipitationMetrics, loss_func, step_loss  # noqa: F401
from .segmentation import ConfusionMatrix, CrossEntropyLoss, CrossEntropyLossWithOptions, IoU, ce_step, cross_entropy  # noqa: F401
from .model import SmaAt_UNet, UNet, UNetAttention, UNetDS, UNetDSAttention4CBAMs  # noqa: F401
from .modules import (CBAM, ChannelAttention, DepthwiseSeparableConv, DoubleConv, DoubleConvDS, Down, DownDS,  # noqa: F401
                      OutConv, SpatialAttention, Up, UpDS)
from .ops import get_pointwise_mode, set_fused_dsconv, set_pointwise_mode  # noqa: F401
from .patch import patch_reference  # noqa: F401

__all__ = ["SmaAt_UNet", "UNetDS", "UNetDSAttention4CBAMs", "UNet", "UNetAttention", "DoubleConv", "Down", "Up", "CBAM", "ChannelAttention", "SpatialAttention", "DepthwiseSeparableConv", "DoubleConvDS",
           "DownDS", "UpDS", "OutConv", "patch_reference", "PrecipitationMetrics", "loss_func", "step_loss", "CrossEntropyLoss", "CrossEntropyLossWithOptions", "ConfusionMatrix", "IoU", "ce_step", "cross_entropy", "set_pointwise_mode", "get_pointwise_mode", "ops"]
