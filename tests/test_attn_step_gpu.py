"""Every attention launch of tests/golden/attn_launches.json (the cfg-2, 320x576, image-batch and long-clip UNet steps, the
text-encoder LoRA step, the VAE encode, and attn_long at L = 256) run through the prims entry points (ops for the unfused
composite) in the step's layout (row pitches, fused [.., 3C] / [.., 2C] column slices, SeqAddr strides) and checked element by
element against a float64 reference (tests/attn_check.py).

  forward:   o (and lse for flash / attn_long);
  backward:  dq, dk, dv from the kernel's own forward o and lse, into gradient buffers preset to NaN: every element the launch
             owns must be written (the whole [.., 3C] / [.., 2C] buffer when the step fuses the projections), and guard
             elements before and after each buffer must stay NaN;
  flash_attn_bwd: t2v_flash_attn_bwd_splits must return the census value for this device's SM count (132 or 114).
Outputs written without atomics (all but dk / dv of a flash backward that splits the query range) must be reproduced bit for
bit by a second call.  Each check prints one ATTNCHECK line: max (|y - r| - 2^-8 |r|) / m and the relative L2 error."""
import math

import pytest
import torch

import attn_check as A

pytestmark = pytest.mark.gpu

LAUNCHES = A.launches()
GUARD = 4096   # sentinel elements before and after every output buffer
DEV = "cuda"


def _report(lid, res):
    for name, (ratio, l2) in res.items():
        print(f"ATTNCHECK {lid} {name} ratio={ratio:.3e} l2={l2:.3e}")


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _same(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), f"{what}: a second call changed the output"


class Guarded:
    """A NaN-filled tensor with GUARD NaN elements on each side in the same allocation."""

    def __init__(self, shape, dtype):
        n = math.prod(shape)
        self.flat = torch.full((n + 2 * GUARD,), math.nan, dtype=dtype, device=DEV)
        self.t = self.flat[GUARD:GUARD + n].view(shape)

    def assert_owned(self, what):
        assert not bool(torch.isnan(self.t).any()), f"{what}: {int(torch.isnan(self.t).sum())} elements of the buffer not written"
        assert bool(torch.isnan(self.flat[:GUARD]).all() and torch.isnan(self.flat[-GUARD:]).all()), \
            f"{what}: an element outside the buffer was written"


def _inputs(r):
    Z, Lq, Lk, D, heads, causal = A.geometry(r)
    inp = A.make_inputs(r, DEV)
    lay = A.layout(r, DEV)
    for n, c in (("q", "Q"), ("k", "K"), ("v", "V"), ("do", "dO")):
        A.scatter(r, inp[c], lay[n], heads, D)
    for b in lay["buffers"] + [lay["do"]]:
        assert not bool(torch.isnan(b).any()), "the input layout is not covered by the canonical problems"
    return inp, lay


def _grad_buffers(r):
    """Guarded NaN gradient buffers in the step's layout: dq / dk / dv views and the Guarded owners."""
    Z, Lq, Lk, D, heads, _ = A.geometry(r)
    C = heads * D
    if A.is_temporal(r):
        lead_q = lead_k = (r["rows"],)
    else:
        lead_q, lead_k = (r["Nb"], Lq), (r["Nb"], Lk)
    if r["fused"] == "qkv":
        g = Guarded(lead_q + (3 * C,), torch.bfloat16)
        return (g.t[..., :C], g.t[..., C:2 * C], g.t[..., 2 * C:]), [g]
    if r["fused"] == "kv":
        gq, gkv = Guarded(lead_q + (C,), torch.bfloat16), Guarded(lead_k + (2 * C,), torch.bfloat16)
        return (gq.t, gkv.t[..., :C], gkv.t[..., C:]), [gq, gkv]
    gs = [Guarded(lead_q + (C,), torch.bfloat16), Guarded(lead_k + (C,), torch.bfloat16), Guarded(lead_k + (C,), torch.bfloat16)]
    return tuple(g.t for g in gs), gs


def _canon(r, t, heads, D):
    return A.gather(r, t, heads, D)


def _flash(r, lid):
    from t2v_b200 import native, prims
    Z, Lq, Lk, D, heads, _ = A.geometry(r)
    inp, lay = _inputs(r)
    q, k, v, do = lay["q"], lay["k"], lay["v"], lay["do"]
    o, lse = prims.flash_attn_fwd(q, k, v, heads)
    if r["kind"] == "flash_attn_fwd":
        res = A.check_outputs(r, inp, {"o": _canon(r, o, heads, D), "lse": lse.reshape(Z, Lq)}, lid)
        o2, lse2 = prims.flash_attn_fwd(q, k, v, heads)
        _same(o, o2, f"{lid} o")
        _same(lse, lse2, f"{lid} lse")
        return res
    (dq, dk, dv), owners = _grad_buffers(r)
    prims.flash_attn_bwd(q, k, v, o, do, lse, heads, dq, dk, dv)
    for g in owners:
        g.assert_owned(lid)
    res = A.check_outputs(r, inp, {n: _canon(r, t, heads, D) for n, t in (("dq", dq), ("dk", dk), ("dv", dv))}, lid)
    first = [t.clone() for t in (dq, dk, dv)]
    prims.flash_attn_bwd(q, k, v, o, do, lse, heads, dq, dk, dv)
    splits = native.lib().t2v_flash_attn_bwd_splits(r["Nb"], heads, Lq, Lk)
    for name, a, b in zip(("dq", "dk", "dv"), first, (dq, dk, dv)):
        if name == "dq" or splits == 1:
            _same(a, b, f"{lid} {name}")
    _report(lid, res)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if f"splits_{sms}" not in r:
        pytest.skip(f"{lid}: the census pins the dK/dV split count for 132 and 114 SMs; this device has {sms}")
    assert splits == r[f"splits_{sms}"], f"{lid}: t2v_flash_attn_bwd_splits = {splits}, census {r[f'splits_{sms}']} on {sms} SMs"
    return {}


def _temporal(r, lid):
    from t2v_b200 import prims
    Z, Lq, Lk, D, heads, _ = A.geometry(r)
    addr = tuple(r["addr"])
    inp, lay = _inputs(r)
    q, k, v, do = lay["q"], lay["k"], lay["v"], lay["do"]
    long = A.family(r) == "long"
    nseq, L = addr[0], addr[8]

    def fwd():
        go = Guarded((r["rows"], heads * D), torch.bfloat16)
        gl = Guarded((nseq, heads, L), torch.float32) if long else None
        if long:
            prims.attn_long_fwd(q, k, v, go.t, gl.t, addr)
        else:
            prims.attn_small_fwd(q, k, v, go.t, addr)
        return go, gl

    go, gl = fwd()
    if r["kind"].endswith("fwd"):
        go.assert_owned(f"{lid} o")
        outs = {"o": _canon(r, go.t, heads, D)}
        if long:
            gl.assert_owned(f"{lid} lse")
            outs["lse"] = gl.t.reshape(Z, L)
        res = A.check_outputs(r, inp, outs, lid)
        go2, gl2 = fwd()
        _same(go.t, go2.t, f"{lid} o")
        if long:
            _same(gl.t, gl2.t, f"{lid} lse")
        return res

    def bwd():
        (dq, dk, dv), owners = _grad_buffers(r)
        if long:
            prims.attn_long_bwd(q, k, v, go.t, do, gl.t, dq, dk, dv, addr)
        else:
            prims.attn_small_bwd(q, k, v, do, dq, dk, dv, addr)
        return (dq, dk, dv), owners

    grads, owners = bwd()
    for g in owners:
        g.assert_owned(lid)
    res = A.check_outputs(r, inp, {n: _canon(r, t, heads, D) for n, t in zip(("dq", "dk", "dv"), grads)}, lid)
    grads2, _ = bwd()
    for name, a, b in zip(("dq", "dk", "dv"), grads, grads2):
        _same(a, b, f"{lid} {name}")
    return res


def _composite(r, lid):
    from t2v_b200 import ops
    Z, Lq, Lk, D, heads, causal = A.geometry(r)
    inp, lay = _inputs(r)
    q, k, v, do = lay["q"], lay["k"], lay["v"], lay["do"]

    def fwd():
        if causal:
            return ops.causal_attention_fwd(q, k, v, heads)
        assert not ops._use_flash(q, heads), "this launch runs the fused kernel, not the composite"
        return ops._attn_core_fwd(q, k, v, heads)

    o, p = fwd()
    res = A.check_outputs(r, inp, {"o": _canon(r, o, heads, D)}, lid)
    o2, p2 = fwd()
    _same(o, o2, f"{lid} o")
    if r["bwd"]:
        def bwd():
            (dq, dk, dv), owners = _grad_buffers(r)
            ops._attn_core_bwd(q, k, v, p, do, dq, dk, dv, heads)
            return (dq, dk, dv), owners

        grads, owners = bwd()
        for g in owners:
            g.assert_owned(lid)
        res.update(A.check_outputs(r, inp, {n: _canon(r, t, heads, D) for n, t in zip(("dq", "dk", "dv"), grads)}, lid))
        grads2, _ = bwd()
        for name, a, b in zip(("dq", "dk", "dv"), grads, grads2):
            _same(a, b, f"{lid} {name}")
    return res


@pytest.mark.parametrize("r", LAUNCHES, ids=[A.launch_id(r) for r in LAUNCHES])
def test_step_attention(r):
    lid = A.launch_id(r)
    fam = A.family(r)
    run = _flash if fam == "flash" else _composite if fam == "composite" else _temporal
    _report(lid, run(r, lid))
    torch.cuda.empty_cache()
