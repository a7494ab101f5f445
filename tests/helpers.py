"""Shared helpers for the GPU parity tests: parameter ranges of the reference Processor
classes (modules.py:136-155, 179-186, 204-230), seeded inputs, oracle runs with gradients."""
import torch

SR = 44100


def eq_ranges(sr=SR):
    g, q = (-20.0, 20.0), (0.1, 6.0)
    hi = (sr // 2) - 1000
    fr = [(20, 2000), (80, 2000), (2000, 8000), (8000, 12000), (12000, hi), (4000, hi)]
    out = []
    for f in fr:
        out += [g, f, q]
    return out


COMP_RANGES = [(-60.0, 0.0), (1.0, 20.0), (5.0, 100.0), (5.0, 100.0), (0.0, 12.0), (0.0, 12.0)]
REVERB_RANGES = [(0.0, 1.0)] * 25


def denorm(p01, ranges, dtype=torch.float32):
    """(bs, P) in [0,1] -> list of P tensors (bs,), denormalised in fp32 like modules.py:13-14."""
    p01 = torch.as_tensor(p01).float()
    return [(p01[:, i] * (hi - lo) + lo).to(dtype) for i, (lo, hi) in enumerate(ranges)]


def run_with_grads(fn, x, params, dtype, device):
    """y, dx, [dparam] for loss = mean(y^2); tensors created on `device` in `dtype`."""
    xx = torch.as_tensor(x).to(device=device, dtype=dtype).clone().requires_grad_(True)
    pp = [torch.as_tensor(p).to(device=device, dtype=dtype).clone().requires_grad_(True) for p in params]
    y = fn(xx, pp)
    y.pow(2).mean().backward()
    return y.detach().cpu(), xx.grad.detach().cpu(), [None if p.grad is None else p.grad.detach().cpu() for p in pp]


def peak_err(a, b):
    """per-item max|a-b| / max|b| (SURVEY.md 8c)"""
    a = torch.as_tensor(a).double()
    b = torch.as_tensor(b).double()
    bs = b.shape[0]
    return (a - b).reshape(bs, -1).abs().amax(1) / b.reshape(bs, -1).abs().amax(1).clamp_min(1e-30)


def eq_kernel_instantiations(lib_path):
    """{(direction, table type, W, S)} of the eq_fwd_kernel / eq_bwd_kernel entry points in the library, read from
    its symbol table with cuobjdump; None where cuobjdump is not installed"""
    import os
    import re
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        return None
    out = subprocess.run([cuobjdump, "-symbols", lib_path], capture_output=True, text=True).stdout
    pat = re.compile(r"STO_ENTRY\s+\S*eq_(fwd|bwd)_kernelI(f|6float2)Li(\d+)ELi(\d+)E")
    return {(m[1], "float" if m[2] == "f" else "float2", int(m[3]), int(m[4])) for m in pat.finditer(out)}


# the EQ kernels dispatch_fwd / dispatch_bwd (biquad.cu) can launch: the backward has no W = 16, and its (8, 2) does
# not fit in shared memory (eight warps x eight units of 2 x 480 floats), so a request for it falls through to (8, 1)
EQ_INSTANTIATIONS = ({("fwd", c, w, s) for c in ("float", "float2") for w in (1, 2, 3, 4, 8, 16) for s in (1, 2)}
                     | {("bwd", c, w, s) for c in ("float", "float2") for w in (1, 2, 3, 4) for s in (1, 2)}
                     | {("bwd", c, 8, 1) for c in ("float", "float2")})


def param_grad_err(got, ref):
    """per-item |got-ref| / max_over_params|ref| for lists of (bs,) gradients (SURVEY.md 8c)."""
    keep = [i for i, r in enumerate(ref) if r is not None]
    g = torch.stack([torch.as_tensor(got[i]).double().reshape(-1) for i in keep], 1)
    r = torch.stack([torch.as_tensor(ref[i]).double().reshape(-1) for i in keep], 1)
    return ((g - r).abs() / r.abs().amax(1, keepdim=True).clamp_min(1e-30)).amax(1)
