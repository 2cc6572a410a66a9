"""fp32 torch restatement of csrc/optim.cu adamw8bit_chunks_kernel, in the kernel's order of operations (tests only).

`emulated()` extends helpers.emulated_prims() with it, so optim.AdamW8bit runs on CPU tensors."""
import contextlib

import torch

from helpers import emulated_prims

QBLOCK = 256


def _adamw(p, g, m, v, hp):
    """csrc/optim.cu adamw_one on fp32 tensors; hp: the 8 fp32 0-dim tensors of one hyper-parameter row. Returns (m, v)."""
    lr, b1, b2, eps, wd, bc1, bc2s, gscale = hp
    g = g * gscale
    p.mul_(1.0 - lr * wd)
    m = b1 * m + (1.0 - b1) * g
    v = b2 * v + (1.0 - b2) * g * g
    denom = v.sqrt() / bc2s + eps
    p.sub_((lr / bc1) * (m / denom))
    return m, v


def quantize(x, absmax, qmap):
    """Nearest-entry code of x / absmax: the smallest i with x / absmax <= 0.5f * (map[i] + map[i+1]); the code of 0.0 where
    absmax is 0."""
    mids = (qmap[:-1] + qmap[1:]) * 0.5
    zero = int((qmap == 0).nonzero()[0, 0])
    safe = torch.where(absmax == 0, torch.ones_like(absmax), absmax)
    codes = torch.searchsorted(mids, (x / safe).contiguous())
    return torch.where(absmax == 0, torch.full_like(codes, zero), codes).to(torch.uint8)


@torch.no_grad()
def adamw8bit_chunks(p, g, shadow, n_shadow, chunks, hp_row, qmaps, m32, v32, code_m, code_v, absmax_m, absmax_v, zero_grad=True,
                     g_bf16=None):
    hp = list(hp_row.float().unbind(0))
    map_m, map_v = qmaps[:256], qmaps[256:]
    for off, n, soff, bits in chunks.tolist():
        sl = slice(off, off + n)
        ss = slice(soff, soff + n)
        gs = g[sl] if g_bf16 is None else g_bf16[sl].float()
        if bits == 32:
            m32[ss], v32[ss] = _adamw(p[sl], gs, m32[ss], v32[ss], hp)
        else:
            nb = (n + QBLOCK - 1) // QBLOCK
            bs = slice(soff // QBLOCK, soff // QBLOCK + nb)
            expand = lambda a: a.repeat_interleave(QBLOCK)[:n]   # noqa: E731
            m = map_m[code_m[ss].long()] * expand(absmax_m[bs])
            v = map_v[code_v[ss].long()] * expand(absmax_v[bs])
            m, v = _adamw(p[sl], gs, m, v, hp)
            for x, qmap, codes, absmax in ((m, map_m, code_m, absmax_m), (v, map_v, code_v, absmax_v)):
                padded = torch.zeros(nb * QBLOCK, dtype=x.dtype, device=x.device)
                padded[:n] = x.abs()
                absmax[bs] = padded.view(nb, QBLOCK).amax(1)
                codes[ss] = quantize(x, expand(absmax[bs]), qmap)
        if shadow is not None and off < n_shadow:
            shadow[sl].copy_(p[sl])
        if zero_grad:
            g[sl].zero_()


@contextlib.contextmanager
def emulated():
    """helpers.emulated_prims() plus this restatement of prims.adamw8bit_chunks."""
    from t2v_b200 import prims
    with emulated_prims():
        saved = prims.adamw8bit_chunks
        prims.adamw8bit_chunks = adamw8bit_chunks
        try:
            yield
        finally:
            prims.adamw8bit_chunks = saved
