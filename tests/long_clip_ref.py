"""fp32 restatement of the long-clip temporal attention primitives (prims.attn_long_fwd / attn_long_bwd, tests only), next
to oracle/ops_ref.py whose attn_small_fwd / bwd restate the short path with the same strided sequence addressing.

The backward is written the way attn_long_bwd computes it - P from the forward's logsumexp, delta = rowsum(dO o O) from the
forward's output - so a test that checks it against autograd also checks that those two saved tensors carry what the
kernel needs."""
import contextlib

import torch

from oracle import ops_ref


def attn_long_fwd(q, k, v, o, lse, addr):
    """o = softmax(q k^T / sqrt(D)) v per (sequence, head); lse [nseq, heads, L] = logsumexp of the scaled scores."""
    D = addr[-1]
    Q, K, V = (ops_ref._seq_view(t, addr, False).float() for t in (q, k, v))
    S = Q @ K.transpose(-1, -2) * D ** -0.5
    ops_ref._seq_view(o, addr, True).copy_((torch.softmax(S, -1) @ V).to(o.dtype))
    lse.copy_(torch.logsumexp(S, -1).reshape(lse.shape))
    return o, lse


def attn_long_bwd(q, k, v, o, do, lse, dq, dk, dv, addr):
    D = addr[-1]
    scale = D ** -0.5
    Q, K, V = (ops_ref._seq_view(t, addr, False).float() for t in (q, k, v))
    O, dO = (ops_ref._seq_view(t, addr, True).float() for t in (o, do))
    P = torch.exp(Q @ K.transpose(-1, -2) * scale - lse.float().reshape(Q.shape[:-1]).unsqueeze(-1))
    delta = (dO * O).sum(-1, keepdim=True)
    dS = P * (dO @ V.transpose(-1, -2) - delta) * scale
    for g, dst in ((dS @ K, dq), (dS.transpose(-1, -2) @ Q, dk), (P.transpose(-1, -2) @ dO, dv)):
        ops_ref._seq_view(dst, addr, False).copy_(g.to(dst.dtype))
    return dq, dk, dv


PRIMS = ("attn_long_fwd", "attn_long_bwd")


@contextlib.contextmanager
def emulated_prims():
    """helpers.emulated_prims() plus the two primitives above: temporal attention of any clip length on the CPU."""
    from helpers import emulated_prims as base
    from t2v_b200 import prims
    saved = {n: getattr(prims, n) for n in PRIMS}
    with base():
        for n in PRIMS:
            setattr(prims, n, globals()[n])
        try:
            yield
        finally:
            for n, fn in saved.items():
                setattr(prims, n, fn)
