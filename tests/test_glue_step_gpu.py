"""Every glue-kernel launch of tests/golden/glue_launches.json (the training steps, the text-encoder steps, the VAE encode, the
data-side resize, and the synthetic launches), run through the prims entry points in the step's layout and checked element by
element against a float64 reference (tests/glue_check.py).

Every output buffer is NaN-filled with GUARD NaN elements on each side in the same allocation: the buffers a launch writes into
(colsum / colsum_f32 / embed_tokens_bwd accumulators preset to nonzero values, the dst of the casts) are made that way here, and
the buffers the prims allocate themselves are handed out that way by a torch.empty / torch.empty_like that prims sees for the
duration of the call.  Every element of the output must be written (or keep its preset) and every guard must stay NaN.  The
padded channels 4..7 (3..7 for the resized frames) of every [.., 8] tensor must come back zero, and each ragged-batch slice must
equal the single-clip resize bit for bit.  Each check prints one GLUECHECK line: max (|y - r| - 2^-8 |r|) / m and the relative
L2 error.  test_gelu_sweep runs both GELU forms over x in [-20, 20]; test_timestep_sweep the embedding of every t in [0, 999]
at dim 320; test_cast_tails both casts at lengths that leave a tail after the last 8-element vector."""
import math
import types

import pytest
import torch

import glue_check as G

pytestmark = pytest.mark.gpu

LAUNCHES = G.launches()
GUARD = 4096
DEV = "cuda"


def _report(lid, res):
    for name, (ratio, l2) in res.items():
        print(f"GLUECHECK {lid} {name} ratio={ratio:.3e} l2={l2:.3e}")


class Guarded:
    """A NaN-filled tensor with GUARD NaN elements on each side in the same allocation."""

    def __init__(self, shape, dtype):
        n = math.prod(shape)
        self.flat = torch.full((n + 2 * GUARD,), math.nan, dtype=dtype, device=DEV)
        self.t = self.flat[GUARD:GUARD + n].view(tuple(shape))

    def assert_guards(self, what):
        assert bool(torch.isnan(self.flat[:GUARD]).all() and torch.isnan(self.flat[-GUARD:]).all()), \
            f"{what}: an element outside the buffer was written"

    def assert_written(self, what):
        assert not bool(torch.isnan(self.t).any()), f"{what}: {int(torch.isnan(self.t).sum())} elements of the buffer not written"
        self.assert_guards(what)


class _GuardedTorch(types.ModuleType):
    """torch as prims sees it during one call: empty / empty_like hand out Guarded floating-point buffers."""

    def __init__(self):
        super().__init__("torch")
        self.made = []

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *shape, device=None, dtype=None, **kw):
        shape = tuple(shape[0]) if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)) else shape
        dtype = dtype or torch.float32
        if not dtype.is_floating_point:
            return torch.empty(shape, device=device, dtype=dtype, **kw)
        g = Guarded(shape, dtype)
        self.made.append(g)
        return g.t

    def empty_like(self, x, **kw):
        return self.empty(tuple(x.shape), device=x.device, dtype=kw.get("dtype", x.dtype))


def _guarded_call(fn, *args, **kw):
    """fn(*args, **kw) with prims allocating Guarded outputs; returns (result, the Guarded buffers)."""
    from t2v_b200 import prims
    shim = _GuardedTorch()
    saved = prims.torch
    prims.torch = shim
    try:
        out = fn(*args, **kw)
    finally:
        prims.torch = saved
    return out, shim.made


def _full(t, n):
    """The device copy of a drawn pattern repeated to n elements."""
    t = t.to(DEV).reshape(-1)
    return t if t.numel() == n else t.repeat(-(-n // t.numel()))[:n].contiguous()


def _preset(t):
    g = Guarded(tuple(t.shape), t.dtype)
    g.t.copy_(t.to(DEV))
    return g


def run(r, inp):
    """Launches `r` on the GPU; returns ({output: tensor}, [Guarded buffers to check])."""
    from t2v_b200 import prims
    k = r["kind"]
    d = {n: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for n, v in inp.items()}
    if k == "latents_to_nhwc8":
        y, gs = _guarded_call(prims.latents_to_nhwc8, d["x0"], d.get("noise"), d.get("abar"), d.get("t"))
        return {"y": y}, gs
    if k == "nhwc8_to_latents":
        y, gs = _guarded_call(prims.nhwc8_to_latents, d["x"], r["B"], r["C"], r["F"])
        return {"out": y}, gs
    if k in ("mse_loss_fwd", "mse_loss_bwd"):
        args = (d["pred"], d["noise"]) + ((d["gout"],) if k.endswith("bwd") else ())
        y, gs = _guarded_call(getattr(prims, k), *args)
        return {"loss" if k.endswith("fwd") else "dpred": y}, gs
    if k in ("velocity_mse_loss_fwd", "velocity_mse_loss_bwd"):
        args = (d["pred"], d["x0"], d["noise"], d["abar"], d["t"]) + ((d["gout"],) if k.endswith("bwd") else ())
        y, gs = _guarded_call(getattr(prims, k), *args)
        return {"loss" if k.endswith("fwd") else "dpred": y}, gs
    if k == "timestep_embedding":
        y, gs = _guarded_call(prims.timestep_embedding, d["t"], r["dim"])
        return {"y": y}, gs
    if k == "colsum":
        out = _preset(inp["preset"])
        prims.colsum(d["x"], out.t, r["S"], r["P"], r["C"])
        return {"out": out.t}, [out]
    if k == "colsum_f32":
        out = _preset(inp["preset"])
        prims.colsum_f32(d["x"], out.t)
        return {"out": out.t}, [out]
    if k == "upsample_nearest_fwd":
        y, gs = _guarded_call(prims.upsample_nearest_fwd, d["x"], (r["Ho"], r["Wo"]))
        return {"y": y}, gs
    if k == "upsample_nearest_bwd":
        y, gs = _guarded_call(prims.upsample_nearest_bwd, d["dy"], (r["H"], r["W"]))
        return {"dx": y}, gs
    if k == "concat_channels":
        y, gs = _guarded_call(prims.concat_channels, d["a"], d["b"])
        return {"y": y}, gs
    if k == "split_channels":
        (a, b), gs = _guarded_call(prims.split_channels, d["g"], r["Ca"])
        return {"a": a, "b": b}, gs
    if k in ("add_bf16", "add_f32"):
        ts = [_full(inp[n], r["n"]) for n in ("a", "b", "c") if n in inp]
        y, gs = _guarded_call(getattr(prims, k), *ts)
        return {"y": y}, gs
    if k == "scale_bf16":
        y, gs = _guarded_call(prims.scale_bf16, _full(inp["a"], r["n"]), r["alpha"])
        return {"y": y}, gs
    if k == "cast_f32_bf16":
        src = _full(inp["src"], r["n"])
        if r["into"]:
            dst = Guarded((r["n"],), torch.bfloat16)
            prims.cast_f32_bf16(src, dst.t)
            return {"y": dst.t}, [dst]
        y, gs = _guarded_call(prims.cast_f32_bf16, src)
        return {"y": y}, gs
    if k == "cast_bf16_f32":
        dst = Guarded((r["n"],), torch.float32)
        prims.cast_bf16_f32(_full(inp["src"], r["n"]), dst.t)
        return {"y": dst.t}, [dst]
    if k == "dropout_scale_add":
        y, gs = _guarded_call(prims.dropout_scale_add, d["x"], d.get("base"), r["p"], r["scale"], inp["seed"], d["epoch"])
        return {"y": y}, gs
    if k == "embed_tokens":
        y, gs = _guarded_call(prims.embed_tokens, d["ids"], d["tok"], d["pos"])
        return {"y": y}, gs
    if k == "embed_tokens_bwd":
        dtok = _preset(inp["dtok"]) if r["dtok"] else None
        dpos = _preset(inp["dpos"]) if r["dpos"] else None
        prims.embed_tokens_bwd(d["ids"], d["dy"], dtok.t if dtok else None, dpos.t if dpos else None, r["vocab"])
        out = {}
        if dtok:
            out["dtok"] = dtok.t
        if dpos:
            out["dpos"] = dpos.t
        return out, [g for g in (dtok, dpos) if g is not None]
    if k == "gelu_bf16":
        y, gs = _guarded_call(prims.gelu_bf16, d["x"], bool(r["quick"]))
        return {"y": y}, gs
    if k == "gelu_bwd":
        y, gs = _guarded_call(prims.gelu_bwd, d["x"], d["dy"], bool(r["quick"]))
        return {"dx": y}, gs
    if k == "vae_sample":
        y, gs = _guarded_call(prims.vae_sample, d["moments"], d["eps"], r["B"], r["F"], r["scale"])
        return {"z": y}, gs
    if k == "frames_u8_to_nhwc8":
        y, gs = _guarded_call(prims.frames_u8_to_nhwc8, d["frames"], (r["h"], r["w"]))
        return {"y": y}, gs
    if k == "frames_u8_to_nhwc8_ragged":
        y, gs = _guarded_call(prims.frames_u8_to_nhwc8_ragged, d["packed"], inp["table"], (r["h"], r["w"]))
        return {"y": y}, gs
    raise KeyError(k)


@pytest.mark.parametrize("r", LAUNCHES, ids=[G.launch_id(r) for r in LAUNCHES])
def test_step_glue(r):
    lid = G.launch_id(r)
    inp = G.make_inputs(r)
    out, guarded = run(r, inp)
    torch.cuda.synchronize()
    for i, g in enumerate(guarded):
        g.assert_written(f"{lid} buffer {i}")
    _report(lid, G.check_outputs(r, inp, out, lid))
    if r["kind"] == "frames_u8_to_nhwc8_ragged":
        from t2v_b200 import prims
        f0 = 0
        for i, c in enumerate(inp["clips"]):
            one = prims.frames_u8_to_nhwc8(c.to(DEV), (r["h"], r["w"]))
            assert torch.equal(out["y"][f0:f0 + c.shape[0]].view(torch.int16), one.view(torch.int16)), f"{lid}: clip {i} differs from its own resize"
            f0 += c.shape[0]


def test_gelu_sweep():
    """Both GELU forms and their derivatives over x in [-20, 20]."""
    n = 8192
    x = torch.linspace(-20, 20, n).bfloat16()
    dy = torch.linspace(-1, 1.5, n).flip(0).bfloat16()
    for quick in (0, 1):
        for kind in ("gelu_bf16", "gelu_bwd"):
            r = {"kind": kind, "n": n, "quick": quick}
            inp = {"x": x, "dy": dy} if kind == "gelu_bwd" else {"x": x}
            out, guarded = run(r, inp)
            for g in guarded:
                g.assert_written(f"sweep-{kind}-q{quick}")
            _report(f"sweep-{kind}-q{quick}", G.check_outputs(r, inp, out, f"sweep-{kind}-q{quick}"))


def test_timestep_sweep():
    """timestep_embedding of every t in [0, 999] at dim 320."""
    r = {"kind": "timestep_embedding", "B": 1000, "dim": 320}
    inp = {"t": torch.arange(1000, dtype=torch.int64)}
    out, guarded = run(r, inp)
    for g in guarded:
        g.assert_written("sweep-timestep_embedding")
    _report("sweep-timestep_embedding", G.check_outputs(r, inp, out, "sweep-timestep_embedding"))


@pytest.mark.parametrize("n", [1, 7, 13, 1003, 65541])
def test_cast_tails(n):
    """Both casts where n % 8 != 0: the tail after the last vector is rounded (and widened) like the rest."""
    for kind, extra in (("cast_f32_bf16", {"into": 1}), ("cast_f32_bf16", {"into": 0}), ("cast_bf16_f32", {})):
        r = {"kind": kind, "n": n, **extra}
        inp = G.make_inputs(r)
        out, guarded = run(r, inp)
        for g in guarded:
            g.assert_written(f"{G.launch_id(r)}")
        G.check_outputs(r, inp, out, G.launch_id(r))
