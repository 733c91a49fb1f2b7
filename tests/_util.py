"""Shared helpers for the GPU parity tests (oracle = checker, CUDA path = subject)."""
import numpy as np
import torch

# Tolerances (relative to max|reference|), stated per pointwise arithmetic mode:
#   fp32   : CUDA-core FFMA, exact fp32 products, fp32 accumulate
#   tf32x3 : wgmma 3xTF32 split; products carry ~2^-21 relative error
#   tf32   : wgmma single TF32 pass (10-bit mantissa inputs) -- what cuDNN gives the reference by default on a GPU
PW_TOL = {"fp32": 2e-5, "tf32x3": 3e-5, "tf32": 4e-3}
# end-to-end (18 pointwise layers + BN scaling) tolerances for the full network
NET_TOL = {"fp32": 1e-4, "tf32x3": 1e-4, "tf32": 2e-2}


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dtype).cuda()


def rel_err(got, ref):
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    denom = max(np.abs(ref).max(), 1e-30)
    return float(np.abs(got - ref).max() / denom)


def assert_close(got, ref, tol, what=""):
    e = rel_err(got, ref)
    assert np.isfinite(e) and e <= tol, f"{what}: max rel err {e:.3e} > tol {tol:.1e}"
    return e


def load_np_state_dict(module, np_sd, prefix=""):
    """Load a numpy (reference-keyed) state_dict into a module; strict."""
    sd = {}
    for k, v in np_sd.items():
        if prefix and not k.startswith(prefix):
            continue
        t = torch.as_tensor(np.asarray(v))
        sd[k[len(prefix):]] = t if t.dtype == torch.int64 else t.float()
    module.load_state_dict(sd, strict=True)
    return module
