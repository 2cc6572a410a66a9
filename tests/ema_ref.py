"""fp32 torch restatement of the weight EMA of csrc/optim.cu (`use_ema`): diffusers' `EMAModel` with its default arguments
(tests only).

`emulated()` extends adamw8bit_ref.emulated() with the three EMA primitives, so optim.FusedAdamW / AdamW8bit with an
`ema_decay` run on CPU tensors."""
import contextlib

import numpy as np
import torch

import adamw8bit_ref


def decay(k, ema_decay):
    """d_k for the step count k >= 1 after this step's increment, in fp64: 0 at k = 1, else min(ema_decay, k / (9 + k)).
    ema_decay is rounded to fp32 first, as the kernels receive it."""
    if k <= 1:
        return 0.0
    return min(float(np.float32(ema_decay)), k / (9.0 + k))


def one_minus_decay(k, ema_decay):
    """1 - d_k, rounded to fp32 (the factor EMAModel.step multiplies an fp32 tensor by)."""
    return torch.tensor(1.0 - decay(k, ema_decay), dtype=torch.float32)


def ema_step(s, p, omd):
    """EMAModel.step on one tensor: s -= (1 - d) * (s - p), in place."""
    s.sub_(omd * (s - p))


def _lerp(p, ema, rows, step, ema_decay):
    omd = one_minus_decay(int(step[0]), ema_decay)
    for off, n, e in rows:
        ema_step(ema[e:e + n], p[off:off + n], omd)


@torch.no_grad()
def adamw_ema_chunks(p, g, m, v, shadow, n_shadow, chunks, hp_row, ema, step, ema_decay, zero_grad=True, g_bf16=None):
    from oracle import ops_ref
    ops_ref.adamw_chunks(p, g, m, v, shadow, n_shadow, chunks[:, :2], hp_row, zero_grad, g_bf16)
    _lerp(p, ema, chunks[:, [0, 1, 2]].tolist(), step, ema_decay)


@torch.no_grad()
def adamw8bit_ema_chunks(p, g, shadow, n_shadow, chunks, hp_row, qmaps, m32, v32, code_m, code_v, absmax_m, absmax_v, ema, step, ema_decay,
                         zero_grad=True, g_bf16=None):
    adamw8bit_ref.adamw8bit_chunks(p, g, shadow, n_shadow, chunks[:, :4], hp_row, qmaps, m32, v32, code_m, code_v, absmax_m, absmax_v,
                                   zero_grad, g_bf16)
    _lerp(p, ema, chunks[:, [0, 1, 4]].tolist(), step, ema_decay)


@torch.no_grad()
def ema_swap_chunks(p, ema, shadow, n_shadow, rows):
    for off, n, e in rows.tolist():
        held = p[off:off + n].clone()
        p[off:off + n].copy_(ema[e:e + n])
        ema[e:e + n].copy_(held)
        if shadow is not None and off < n_shadow:
            shadow[off:off + n].copy_(p[off:off + n])


@contextlib.contextmanager
def emulated():
    """adamw8bit_ref.emulated() plus this restatement of the EMA primitives."""
    from t2v_b200 import prims
    names = ("adamw_ema_chunks", "adamw8bit_ema_chunks", "ema_swap_chunks")
    with adamw8bit_ref.emulated():
        saved = {n: getattr(prims, n) for n in names}
        for n in names:
            setattr(prims, n, globals()[n])
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(prims, n, f)
