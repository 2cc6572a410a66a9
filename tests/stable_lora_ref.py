"""fp32 torch restatement of the two stable-LoRA primitives (prims.lora_delta_merge / lora_delta_grad, csrc/lora_delta.cu),
written from the module contract: W_eff = W + scaling * view(B @ A) (Conv3d: the mean over the fourth axis of the
(out, in, 3, 3, 1) view), and the exact gradient of A and B through that view.  Used by the CPU wiring tests (patched into
prims next to oracle/ops_ref.py) and as the reference of the GPU kernel tests."""
import contextlib

import torch


def _logical_shape(w_phys, conv3d):
    Co, KH, KW, Ci = w_phys.shape
    return (Co, Ci, 3, 1, 1) if conv3d else (Co, Ci, KH, KW)


def delta_logical(A, B, scaling, shape, conv3d):
    """The delta in the logical (out, in, k, k) / (out, in, 3, 1, 1) layout, fp32."""
    ba = B.float() @ A.float()
    if conv3d:
        Co, Ci = shape[:2]
        return torch.mean(ba.view(Co, Ci, 3, 3, 1), dim=-2, keepdim=True) * scaling
    return ba.view(shape) * scaling


def to_phys(t):
    """(out, in, kh, kw) or (out, in, 3, 1, 1) -> [out, kh, kw, in] / [out, 3, 1, in]."""
    if t.dim() == 5:
        t = t.flatten(3)
    return t.permute(0, 2, 3, 1).contiguous()


def from_phys(t, conv3d):
    lg = t.permute(0, 3, 1, 2)
    return lg.unsqueeze(-1) if conv3d else lg


def merge_f32(base, A, B, scaling, conv3d):
    """fp32 W_eff in the physical layout (before the kernel's single bf16 rounding)."""
    return base.float() + to_phys(delta_logical(A, B, scaling, _logical_shape(base, conv3d), conv3d))


def lora_delta_merge(base, A, B, scaling, conv3d):
    from oracle import ops_ref
    return merge_f32(base, A, B, scaling, conv3d).to(ops_ref.BF)


@torch.enable_grad()
def lora_delta_grad(dw, A, B, scaling, conv3d, dA, dB):
    a = A.detach().float().requires_grad_(True)
    b = B.detach().float().requires_grad_(True)
    d = delta_logical(a, b, scaling, _logical_shape(dw, conv3d), conv3d)
    ga, gb = torch.autograd.grad(d, (a, b), from_phys(dw.float(), conv3d))
    dA += ga
    dB += gb


@contextlib.contextmanager
def patched_prims():
    """oracle/ops_ref.py's emulated primitives plus the two above (tests only)."""
    from helpers import emulated_prims
    from t2v_b200 import prims
    saved = {n: getattr(prims, n) for n in ("lora_delta_merge", "lora_delta_grad")}
    with emulated_prims():
        prims.lora_delta_merge, prims.lora_delta_grad = lora_delta_merge, lora_delta_grad
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(prims, n, f)
