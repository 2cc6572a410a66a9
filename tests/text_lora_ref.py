"""fp32 torch restatement of the text-LoRA primitive prims.gelu_bwd (csrc/elementwise.cu gelu_bwd_kernel), written from its
contract: dx = dy * d/dx gelu(x), the exact erf GELU or CLIP's quick_gelu x * sigmoid(1.702 x), rounded once to bf16.
Used by the CPU tests (patched into prims next to oracle/ops_ref.py) and as the reference of the GPU kernel test."""
import contextlib

import torch


def gelu_grad_f32(x, quick=False):
    x = x.float()
    if quick:
        s = torch.sigmoid(1.702 * x)
        return s + 1.702 * x * s * (1 - s)
    return 0.5 * (1 + torch.erf(x * 0.5 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


def gelu_bwd(x, dy, quick=False):
    from oracle import ops_ref
    return (dy.float() * gelu_grad_f32(x, quick)).to(ops_ref.BF)   # bf16, or fp32 when a test switches the emulation to fp32


@contextlib.contextmanager
def emulated():
    """oracle/ops_ref.py's emulated primitives plus gelu_bwd (tests only)."""
    from helpers import emulated_prims
    from t2v_b200 import prims
    saved = prims.gelu_bwd
    with emulated_prims():
        prims.gelu_bwd = gelu_bwd
        try:
            yield
        finally:
            prims.gelu_bwd = saved
