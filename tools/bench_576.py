"""BASELINE configs[4]: high-res 576x576 inference, batch 8, one GPU (same pixel count per step as 32 x 288^2)."""
import json, sys, torch
sys.path.insert(0, ".")
import smaat_unet_b200 as S
from smaat_unet_b200.engine import InferenceSession
for mode in ("tf32x3", "tf32"):
    S.set_pointwise_mode(mode)
    torch.manual_seed(0)
    model = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().eval()
    sess = InferenceSession(model, 8, (12, 576, 576))
    xs = [torch.rand(8, 12, 576, 576, device="cuda") for _ in range(2)]
    for i in range(5): sess.forward(xs[i % 2])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(20): sess.forward(xs[i % 2])
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    print(json.dumps({"workload": "configs[4]: SmaAt-UNet forward (eval), batch=8, 12->1ch 576x576, 1 GPU", "pointwise": mode,
                      "frames_per_s": 8 / (ms * 1e-3), "ms_per_step": ms, "launches_per_forward": int(sess.launches_per_forward)}))
