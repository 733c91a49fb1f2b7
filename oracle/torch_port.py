"""torch-functional CPU port of the reference forward -- TEST INFRASTRUCTURE ONLY.

Same algorithm as ``oracle/smaat_oracle.py`` (and therefore as the reference
files it cites), written as pure functions over a reference-keyed state_dict
and dispatched to ``torch.nn.functional`` -- i.e. the same ATen/oneDNN CPU
kernels the reference's ``nn.Module``s run (SURVEY section 6: 90 % of the CPU
time is ``aten::mkldnn_convolution``).  Used for

* parity at sizes where the numpy oracle is too slow (full 288x288 frames), and
* the ``cpu_baseline`` / ``--impl reference`` arm of ``bench.py`` (kind "port":
  /root/reference does not exist on the GPU box, so the reference's own
  modules cannot be imported there).

It is pinned twice: against the golden fixtures (``tests/test_oracle_golden.py``)
and against the numpy oracle.  Never imported by the product package.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _bn(x, sd, p, training):
    # nn.BatchNorm2d defaults: eps 1e-5, momentum 0.1 (parts_ds.py:25,34; layers.py:120)
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        training=training, momentum=0.1, eps=1e-5)


def ds_conv(x, sd, p):
    # layers.py:47-50
    w = sd[p + ".depthwise.weight"]
    y = F.conv2d(x, w, sd[p + ".depthwise.bias"], padding=1, groups=x.shape[1])
    return F.conv2d(y, sd[p + ".pointwise.weight"], sd[p + ".pointwise.bias"])


def double_conv_ds(x, sd, p, training=False):
    # parts_ds.py:17-36
    y = F.relu(_bn(ds_conv(x, sd, p + ".double_conv.0"), sd, p + ".double_conv.1", training))
    return F.relu(_bn(ds_conv(y, sd, p + ".double_conv.3"), sd, p + ".double_conv.4", training))


def down_ds(x, sd, p, training=False):
    # parts_ds.py:47-53
    return double_conv_ds(F.max_pool2d(x, 2), sd, p + ".maxpool_conv.1", training)


def up_ds(x_low, x_skip, sd, p, training=False):
    # parts_ds.py:75-86 (bilinear branch; ConvTranspose2d branch :72-73 when the state_dict holds up.weight)
    if p + ".up.weight" in sd:
        up = F.conv_transpose2d(x_low, sd[p + ".up.weight"], sd[p + ".up.bias"], stride=2)
    else:
        up = F.interpolate(x_low, scale_factor=2, mode="bilinear", align_corners=True)
    dY, dX = x_skip.shape[2] - up.shape[2], x_skip.shape[3] - up.shape[3]
    up = F.pad(up, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])
    return double_conv_ds(torch.cat([x_skip, up], dim=1), sd, p + ".conv", training)


def cbam(x, sd, p, training=False):
    # layers.py:105-111, 122-129, 138-141
    ca = p + ".channel_att.MLP"

    def mlp(v):
        return F.linear(F.relu(F.linear(v, sd[ca + ".1.weight"], sd[ca + ".1.bias"])), sd[ca + ".3.weight"], sd[ca + ".3.bias"])

    # The max pools use the reference's ops (AdaptiveMaxPool2d(1), torch.max(dim=1)), not Tensor.amax: the forward values
    # agree, but on tied maxima (exact zeros after a ReLU are common) amax splits the gradient evenly among the ties while
    # these send all of it to one index, as the reference's backward does.
    s = torch.sigmoid(mlp(x.mean(dim=(2, 3))) + mlp(F.adaptive_max_pool2d(x, 1).flatten(1)))
    x = x * s[:, :, None, None]
    w = sd[p + ".spatial_att.conv.weight"]
    m = torch.cat([x.mean(dim=1, keepdim=True), torch.max(x, dim=1, keepdim=True)[0]], dim=1)
    a = _bn(F.conv2d(m, w, None, padding=w.shape[-1] // 2), sd, p + ".spatial_att.bn", training)
    return x * torch.sigmoid(a)


def smaat_unet_forward(x, sd, training=False, n_cbams=5):
    # SmaAt_UNet.py:41-57; n_cbams = 4 / 0: unet_precip_regression_lightning.py:193-208 / :104-117
    enc = [double_conv_ds(x, sd, "inc", training)]
    for i in range(1, 5):
        enc.append(down_ds(enc[-1], sd, f"down{i}", training))
    att = [cbam(e, sd, f"cbam{i + 1}", training) if i < n_cbams else e for i, e in enumerate(enc)]
    y = att[4]
    for i in range(1, 5):
        y = up_ds(y, att[4 - i], sd, f"up{i}", training)
    return F.conv2d(y, sd["outc.conv.weight"], sd["outc.conv.bias"])


def to_torch_sd(np_sd, dtype=torch.float32, device="cpu"):
    out = {}
    for k, v in np_sd.items():
        t = torch.as_tensor(v)
        out[k] = (t if t.dtype == torch.int64 else t.to(dtype)).to(device).clone()
    return out
