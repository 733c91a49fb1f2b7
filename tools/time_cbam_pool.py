"""A/B: CBAM channel-gate front end (global avg/max pool [+ 2x2 max-pool] + MLP + sigmoid) as ONE launch (last-arriving CTA runs the
MLP) vs pool kernel + MLP kernel, per SmaAt-UNet attention shape.  usage: python tools/time_cbam_pool.py"""
import sys, torch
sys.path.insert(0, ".")
from smaat_unet_b200 import ops
B = 32
for C, S in [(64, 288), (128, 144), (256, 72), (512, 36), (512, 18)]:
    x = torch.rand(B, C, S, S, device="cuda")
    hid = max(C // 16, 1)
    w1, b1 = torch.randn(hid, C, device="cuda") * 0.1, torch.randn(hid, device="cuda")
    w2, b2 = torch.randn(C, hid, device="cuda") * 0.1, torch.randn(C, device="cuda")
    poolable = S % 4 == 0
    def fused():
        return ops.cbam_pool_mlp(x, w1, b1, w2, b2, with_maxpool=True)
    def split():
        r = ops.cbam_pool_maxpool(x) if poolable else None
        avg, mx = (r[0], r[1]) if r is not None else ops.cbam_pool(x)
        return ops.cbam_mlp(avg, mx, w1, b1, w2, b2)
    res = {}
    for name, f in (("one launch", fused), ("pool + mlp", split)):
        for _ in range(3): f()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20): f()
        e1.record(); torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) / 20
    a = fused(); b = split()
    err = float((a[0] - b).abs().max())
    gb = (5 if poolable else 4) * B * C * S * S / 1e9
    print(f"C={C:4d} S={S:4d}: one launch {res['one launch'] * 1e3:7.1f} us ({gb / res['one launch']:6.0f} GB/s)   pool + mlp {res['pool + mlp'] * 1e3:7.1f} us   |sc diff| {err:.1e}")
