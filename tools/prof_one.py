"""Run one kernel shape a few times (for a profiler).  usage: prof_one.py dsconv|pw|dw <mode>"""
import sys, torch
sys.path.insert(0, ".")
import smaat_unet_b200 as S
from smaat_unet_b200 import ops
what, mode = sys.argv[1], (sys.argv[2] if len(sys.argv) > 2 else "tf32x3")
B, C, H, W, k, Cout = 32, 64, 288, 288, 2, 64
if len(sys.argv) > 3:
    C, H, Cout = int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]); W = H
torch.manual_seed(0)
x = torch.rand(B, C, H, W, device="cuda")
dw_w = torch.randn(k * C, 1, 3, 3, device="cuda"); dw_b = torch.randn(k * C, device="cuda")
pw_w = torch.randn(Cout, k * C, 1, 1, device="cuda") * 0.1
sc = torch.rand(Cout, device="cuda") + 0.5; sh = torch.randn(Cout, device="cuda")
split = ops.split_tf32(pw_w.view(Cout, -1))
for _ in range(3):
    if what == "dsconv":
        y = ops.dsconv(x, dw_w, dw_b, k, pw_w, sc, sh, True, mode=mode, w_split=split)
    elif what == "dw":
        y = ops.dw3x3(x, dw_w, dw_b, k)
    else:
        d = torch.rand(B, k * C, H, W, device="cuda")
        y = ops.pw1x1(d, pw_w, sc, sh, True, mode=mode, w_split=split)
torch.cuda.synchronize()
print("ok", tuple(y.shape))
