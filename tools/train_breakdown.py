"""Per-kernel breakdown of one eager training step (fwd + bwd + Adam, B=32, 12x288x288) from CUDA events around every
C-ABI launch (ops.profile).  usage: python tools/train_breakdown.py [batch]"""
import sys
import torch
sys.path.insert(0, ".")
import smaat_unet_b200 as S
from smaat_unet_b200 import ops
from smaat_unet_b200.train import TrainSession

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
torch.manual_seed(0)
model = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
sess = TrainSession(model, B, (12, 288, 288), lr=1e-3, use_graph=False)
x = torch.rand(B, 12, 288, 288, device="cuda")
y = torch.rand(B, 288, 288, device="cuda")
for _ in range(3):
    sess.step(x, y)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
with ops.profile() as prof:
    e0.record()
    sess.step(x, y)
    e1.record()
torch.cuda.synchronize()
tot = e0.elapsed_time(e1)
agg = prof.summary()
ksum = sum(a["ms"] for a in agg.values())
print(f"eager training step B={B}: {tot:.2f} ms wall on the stream (events), {ksum:.2f} ms inside {sum(a['launches'] for a in agg.values())} C-ABI launches")
print(f"{'kernel':40s} {'n':>4s} {'ms':>8s} {'share':>6s} {'GB/s':>7s} {'TF':>6s}")
for name, a in sorted(agg.items(), key=lambda kv: -kv[1]["ms"]):
    print(f"{name:40s} {a['launches']:4d} {a['ms']:8.3f} {100 * a['ms'] / ksum:5.1f}% {a['bytes'] / a['ms'] / 1e6:7.0f} {a['flops'] / a['ms'] / 1e9:6.1f}")
print("-- top 25 by shape")
for name, a in sorted(prof.summary(by_shape=True).items(), key=lambda kv: -kv[1]["ms"])[:25]:
    print(f"{name:48s} {a['launches']:4d} {a['ms']:8.3f} {a['bytes'] / a['ms'] / 1e6:7.0f} GB/s {a['flops'] / a['ms'] / 1e9:6.1f} TF")
