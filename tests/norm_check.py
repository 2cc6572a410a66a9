"""Element-wise checks of the normalisation and activation entry points (prims.groupnorm_fwd / groupnorm_bwd, layernorm_fwd /
layernorm_bwd, geglu_fwd / geglu_bwd, silu_bf16 / silu_bf16_bwd / silu_f32_to_bf16 / silu_bwd_f32) against a float64 reference.
Shared by tests/test_norm_step_gpu.py (the kernels, at every launch of a cfg-2 training step: tests/golden/norm_launches.json)
and tests/test_norm_step_cpu.py (the same checks against the fp32 oracle and against deliberately broken outputs, without a GPU).

Reference r: the float64 result of the operation on the same bf16 / fp32 inputs.  Where a kernel output depends on earlier
outputs of the same launch, r is computed from the kernel's own values, so that a failure names its stage:
    GroupNorm forward  (a) stat = (mean, rstd)  against float64 statistics of x;
                       (b) ab = (a, b)          against a = gamma rstd, b = beta - mean a from the kernel's stat;
                       (c) y                    against SiLU(a x + b) (or a x + b) from the kernel's ab;
    GroupNorm backward dx, dgamma, dbeta        from x, dy, gamma and the kernel's stat and ab;
    LayerNorm          stat against x; y and the backward from the kernel's stat.
Magnitude m: the same expression on absolute values of every term (and of the group / row sums), so that it bounds what fp32
rounding of each intermediate can contribute.  With z = a x + b, SiLU(z) = z s(z), SiLU'(z) = s (1 + z (1 - s)):
    GroupNorm y       m = |SiLU'(z)| (|a x| + |b|) + |SiLU(z)|      (the fp32 rounding of z and an accurate s)
    SiLU derivative   m = |dy| (s (1 + |z|) + |SiLU''(z)| (|a x| + |b|))
    GEGLU             m = |h| (|gelu(g)| + |g|) and |h| |g| in the gradient: the fp32 cancellation in 1 + erff(g / sqrt 2)
                      for very negative g is admitted; it is conditioning, not a defect of the kernel.
Every element must satisfy
    bf16 output:   |y - r| <= 2^-8 |r| + eps m        (one round-to-nearest of an fp32 result)
    fp32 output:   |y - r| <= eps m
and the relative L2 error of a bf16 output must be at most 2^-8.  (No L2 bound in eps: m exceeds |r| by design where the
operation is ill-conditioned, e.g. rstd under a common mode, so 16 eps |r| would not follow from the element bound.)  A s(z) with an absolute error of 2^-12 (the hardware
tanh, 0.5 tanh(z / 2) + 0.5) is wrong by several bf16 ulps of SiLU(z) for z < -4 and is rejected; the per-kernel tests' metric
max|y - r| / max|r| < 1e-2 accepts it.  dgamma / dbeta accumulate into buffers preset to 1 and 3.

Inputs (seed = crc32 of the launch id, drawn on the CPU so that every device sees the same values): x with a per-group common
mode of up to 30 standard deviations (the E[x^2] - mean^2 cancellation), gamma ~ 1 + 0.5 N(0, 1), beta ~ 1.5 N(0, 1), SiLU
inputs ~ 3 N(0, 1), GEGLU gates ~ 3 N(0, 1); every SiLU launch must put at least 1% of its z below -4.

eps, per output: the next power of two at or above 4x the largest ratio (check()) measured in two runs over the step's launches,
with and without producer statistics (the sums use atomics, so the ratios vary), and the sweep of test_norm_step_gpu.py, on one NVIDIA H100 80GB HBM3 at a 700 W power limit
(1980 MHz max SM clock).  Where no error beyond one bf16 rounding was measured (ratio 0), eps = 2^-22, four fp32 unit
roundoffs.  The ratios measured with the hardware-tanh sigmoid the GroupNorm kernels used before are in brackets: its forward
failed at every GroupNorm+SiLU launch (worst in the census: z = -13.616, y = -1.5855e-05, r = -1.6621e-05; in the sweep
z = -16.015, y = -0, r = -1.7748e-06), and its backward ratios exceed these eps too."""
import json
import math
import os
import zlib

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
LAUNCHES = os.path.join(HERE, "golden", "norm_launches.json")

U_BF16 = 2.0 ** -8
EPS = {                                   # measured max ratio (kernel, launch)
    "gn.mean": 2.0 ** -20,       # 1.32e-07  groupnorm_fwd 1x16384x320, fps 4, own sums
    "gn.rstd": 2.0 ** -20,       # 1.44e-07  groupnorm_fwd 1x1024x1280
    "gn.a": 2.0 ** -22,          # 5.95e-08  groupnorm_fwd 16x64x1920, own sums
    "gn.b": 2.0 ** -21,          # 1.11e-07  groupnorm_fwd 16x256x1280, own sums
    "gn.y": 2.0 ** -22,          # 0
    "gn.dx": 2.0 ** -24,         # 7.71e-09  groupnorm_bwd 16x1024x960 silu       [tanh sigmoid: 2.70e-06]
    "gn.dgamma": 2.0 ** -21,     # 1.16e-07  groupnorm_bwd 1x1024x1280            [tanh sigmoid: 1.46e-06]
    "gn.dbeta": 2.0 ** -20,      # 2.36e-07  groupnorm_bwd 1x16384x320            [tanh sigmoid: 4.78e-06]
    "ln.mean": 2.0 ** -21,       # 1.17e-07  layernorm_fwd 4096x640
    "ln.rstd": 2.0 ** -21,       # 6.27e-08  layernorm_fwd 16384x320
    "ln.y": 2.0 ** -25,          # 4.13e-09  layernorm_fwd 16384x320
    "ln.dx": 2.0 ** -26,         # 2.61e-09  layernorm_bwd 16384x320
    "ln.dgamma": 2.0 ** -26,     # 2.96e-09  layernorm_bwd 256x1280
    "ln.dbeta": 2.0 ** -19,      # 2.49e-07  layernorm_bwd 16384x320
    "geglu.y": 2.0 ** -23,       # 2.37e-08  geglu_fwd 256x5120
    "geglu.dproj": 2.0 ** -23,   # 2.37e-08  geglu_bwd 16384x2048
    "silu.y": 2.0 ** -22,        # 0
    "silu.dx": 2.0 ** -20,       # 1.58e-07  silu_bwd_f32, sweep
}
SILU_TAIL = (-4.0, 0.01)   # every SiLU launch: at least 1% of its z below -4


def launches():
    with open(LAUNCHES) as f:
        return json.load(f)


def launch_id(r):
    k = r["kind"]
    if k.startswith("groupnorm"):
        s = f'{k}-{r["S"]}x{r["P"]}x{r["C"]}-g{r["G"]}' + ("-silu" if r["silu"] else "")
        if k == "groupnorm_fwd":
            s += f'-eps{r["eps"]:g}'
            if r["stats"]:
                s += f'-st{r["stats"]}x{r["frames"]}' + (f'-c0_{r["C0"]}' if r["C0"] != r["C"] else "")
        else:
            s += "-add" * r["add"] + "-dg" * r["dgamma"] + "-db" * r["dbeta"]
        return s
    if k.startswith("layernorm"):
        s = f'{k}-{r["rows"]}x{r["C"]}'
        return s + (f'-eps{r["eps"]:g}' if k == "layernorm_fwd" else "-add" * r["add"] + "-dg" * r["dgamma"] + "-db" * r["dbeta"])
    if k.startswith("geglu"):
        return f'{k}-{r["M"]}x{r["I"]}'
    return f'{k}-{"x".join(map(str, r["shape"]))}' + ("" if r.get("apply", 1) else "-cast")


# ---------------------------------------------------------------------------------------------- inputs
def _gen(r):
    return torch.Generator().manual_seed(zlib.crc32(launch_id(r).encode()))


def _common_mode(g, lead, C, groups):
    """[*lead, C] fp32: per group a common mode of U(-30, 30) standard deviations, per channel an offset of 0.5 N(0, 1) and
    a spread of 0.5 + U(0, 1)."""
    ratio = (torch.rand(groups, generator=g) * 2 - 1) * 30
    mu = ratio.repeat_interleave(C // groups) + 0.5 * torch.randn(C, generator=g)
    sd = 0.5 + torch.rand(C, generator=g)
    return torch.randn(*lead, C, generator=g) * sd + mu


def _affine(g, C):
    return 1 + 0.5 * torch.randn(C, generator=g), 1.5 * torch.randn(C, generator=g)


def make_inputs(r, device):
    g = _gen(r)
    k = r["kind"]
    out = {}
    if k.startswith("groupnorm"):
        S, P, C, G = r["S"], r["P"], r["C"], r["G"]
        out["x"] = _common_mode(g, (S, P), C, G).bfloat16()
        out["gamma"], out["beta"] = _affine(g, C)
        if k == "groupnorm_bwd":
            out["dy"] = (torch.randn(S, P, C, generator=g) + 0.25).bfloat16()
            if r["add"]:
                out["add"] = torch.randn(S, P, C, generator=g).bfloat16()
    elif k.startswith("layernorm"):
        rows, C = r["rows"], r["C"]
        x = torch.randn(rows, C, generator=g) * (0.5 + torch.rand(C, generator=g))
        out["x"] = (x + (torch.rand(rows, 1, generator=g) * 2 - 1) * 30).bfloat16()
        out["gamma"], out["beta"] = _affine(g, C)
        if k == "layernorm_bwd":
            out["dy"] = (torch.randn(rows, C, generator=g) + 0.25).bfloat16()
            if r["add"]:
                out["add"] = torch.randn(rows, C, generator=g).bfloat16()
    elif k.startswith("geglu"):
        M, I = r["M"], r["I"]
        out["proj"] = torch.cat([2 * torch.randn(M, I, generator=g), 3 * torch.randn(M, I, generator=g)], 1).bfloat16()
        if k == "geglu_bwd":
            out["dout"] = torch.randn(M, I, generator=g).bfloat16()
    else:
        x = 3 * torch.randn(*r["shape"], generator=g)
        f32 = k in ("silu_f32_to_bf16", "silu_bwd_f32")
        out["x"] = x if f32 else x.bfloat16()
        if k.endswith("bwd") or k == "silu_bwd_f32":
            dy = torch.randn(*r["shape"], generator=g) + 0.25
            out["dy"] = dy if f32 else dy.bfloat16()
    return {n: t.to(device) for n, t in out.items()}


def producer_stats(x, r, channel_stats):
    """The per-frame sums the step hands groupnorm_fwd for launch `r` (None when it hands none): `channel_stats` ([S, P, C] bf16
    -> [S, C, 2] fp32) over the frames = S * fps slots of x, one source per channel range [0, C0) and [C0, C)."""
    if not r["stats"]:
        return None
    S, P, C = x.shape
    xf = x.reshape(r["frames"], S * P // r["frames"], C)
    if r["stats"] == 1:
        return [channel_stats(xf)]
    return [channel_stats(xf[..., :r["C0"]].contiguous()), channel_stats(xf[..., r["C0"]:].contiguous())]


# ---------------------------------------------------------------------------------------------- float64 pieces
def _sig(z):
    return torch.sigmoid(z)


def silu_terms(z, zmag):
    """(SiLU(z), m of the forward, SiLU'(z), m of the derivative per unit |dy|) with zmag = |a x| + |b| bounding the rounding
    of z."""
    s = _sig(z)
    d1 = s * (1 + z * (1 - s))
    d2 = s * (1 - s) * (2 + z * (1 - 2 * s))
    return z * s, d1.abs() * zmag + (z * s).abs(), d1, s * (1 + z.abs()) + d2.abs() * zmag


def _gelu(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def _gelu_grad(x):
    phi = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * phi, phi


# ---------------------------------------------------------------------------------------------- references
def gn_stat_reference(x, G, eps):
    """{mean, rstd}: (r, m) of the [S, G] group statistics of x [S, P, C]; the sums are fp32 (any order), the variance is
    E[x^2] - mean^2, so the rstd bound scales with E[x^2] / (var + eps)."""
    S, P, C = x.shape
    xd = x.double().view(S, P, G, C // G)
    mean = xd.mean(dim=(1, 3))
    var = (xd - mean[:, None, :, None]).pow(2).mean(dim=(1, 3))
    rstd = 1 / torch.sqrt(var + eps)
    ex2 = xd.pow(2).mean(dim=(1, 3))
    return {"mean": (mean, xd.abs().mean(dim=(1, 3))), "rstd": (rstd, rstd * (1 + ex2 / (var + eps)))}


def gn_ab_reference(stat, gamma, beta, G):
    """{a, b}: (r, m) of [S, C] from the kernel's stat."""
    C = gamma.numel()
    mean = stat[..., 0].double().repeat_interleave(C // G, dim=1)
    rstd = stat[..., 1].double().repeat_interleave(C // G, dim=1)
    a = gamma.double() * rstd
    return {"a": (a, a.abs()), "b": (beta.double() - mean * a, beta.double().abs() + (mean * a).abs())}


def gn_y_reference(x, ab, silu):
    """(r, m) of y from the kernel's ab [S, C, 2]."""
    a, b = ab[..., 0].double()[:, None, :], ab[..., 1].double()[:, None, :]
    xd = x.double()
    z = a * xd + b
    zmag = (a * xd).abs() + b.abs()
    if not silu:
        return z, zmag
    y, m, _, _ = silu_terms(z, zmag)
    return y, m


def _norm_bwd(dz, mdz, gamma, xh, xm, rstd, n, group):
    """dx = rstd (gamma dz - T0 / n - xhat T1 / n) with T0 = sum gamma dz, T1 = sum gamma dz xhat over each normalisation group
    (`group` sums a [.., C] tensor over the group and broadcasts it back); m from |.| of every term and of the sums."""
    gd, gm = gamma * dz, gamma.abs() * mdz
    T0, T1 = group(gd), group(gd * xh)
    A0, A1 = group(gm), group(gm * xm)
    dx = rstd * (gd - T0 / n - xh * T1 / n)
    m = rstd * (gm + (A0 + T0.abs()) / n + xm * (A1 + T1.abs()) / n)
    return dx, m


def gn_bwd_reference(x, dy, gamma, stat, ab, G, silu, add=None):
    """{dx, dgamma, dbeta}: (r, m) from the kernel's stat and ab; dgamma / dbeta accumulate into 1 and 3."""
    S, P, C = x.shape
    cpg = C // G
    xd, dyd, gd = x.double(), dy.double(), gamma.double()
    mean = stat[..., 0].double().repeat_interleave(cpg, dim=1)[:, None, :]
    rstd = stat[..., 1].double().repeat_interleave(cpg, dim=1)[:, None, :]
    xh = (xd - mean) * rstd
    xm = (xd.abs() + mean.abs()) * rstd
    if silu:
        a, b = ab[..., 0].double()[:, None, :], ab[..., 1].double()[:, None, :]
        z = a * xd + b
        _, _, d1, md1 = silu_terms(z, (a * xd).abs() + b.abs())
        dz, mdz = dyd * d1, dyd.abs() * md1
    else:
        dz, mdz = dyd, dyd.abs()

    def group(t):
        return t.view(S, P, G, cpg).sum(dim=(1, 3), keepdim=True).expand(S, P, G, cpg).reshape(S, P, C)

    dx, m = _norm_bwd(dz, mdz, gd, xh, xm, rstd, P * cpg, group)
    if add is not None:
        dx, m = dx + add.double(), m + add.double().abs()
    return {"dx": (dx, m), "dgamma": (1 + (dz * xh).sum(dim=(0, 1)), 1 + (mdz * xm).sum(dim=(0, 1))),
            "dbeta": (3 + dz.sum(dim=(0, 1)), 3 + mdz.sum(dim=(0, 1)))}


def ln_stat_reference(x, eps):
    xd = x.double()
    mean = xd.mean(-1)
    var = (xd - mean[:, None]).pow(2).mean(-1)
    rstd = 1 / torch.sqrt(var + eps)
    return {"mean": (mean, xd.abs().mean(-1)), "rstd": (rstd, rstd * (1 + xd.pow(2).mean(-1) / (var + eps)))}


def ln_y_reference(x, gamma, beta, stat):
    xd, gd, bd = x.double(), gamma.double(), beta.double()
    mean, rstd = stat[:, :1].double(), stat[:, 1:].double()
    return (xd - mean) * rstd * gd + bd, (xd.abs() + mean.abs()) * rstd * gd.abs() + bd.abs()


def ln_bwd_reference(x, dy, gamma, stat, add=None):
    xd, dyd, gd = x.double(), dy.double(), gamma.double()
    mean, rstd = stat[:, :1].double(), stat[:, 1:].double()
    xh = (xd - mean) * rstd
    xm = (xd.abs() + mean.abs()) * rstd
    dx, m = _norm_bwd(dyd, dyd.abs(), gd, xh, xm, rstd, x.shape[1], lambda t: t.sum(-1, keepdim=True))
    if add is not None:
        dx, m = dx + add.double(), m + add.double().abs()
    return {"dx": (dx, m), "dgamma": (1 + (dyd * xh).sum(0), 1 + (dyd.abs() * xm).sum(0)),
            "dbeta": (3 + dyd.sum(0), 3 + dyd.abs().sum(0))}


def geglu_reference(proj, dout=None):
    h, g = proj.double().chunk(2, dim=-1)
    gl = _gelu(g)
    if dout is None:
        return h * gl, h.abs() * (gl.abs() + g.abs())
    d = dout.double()
    gg, phi = _gelu_grad(g)
    dh, mh = d * gl, d.abs() * (gl.abs() + g.abs())
    dg, mg = d * h * gg, (d * h).abs() * (gg.abs() + 1 + g.abs() * phi * (1 + g * g))
    return torch.cat([dh, dg], -1), torch.cat([mh, mg], -1)


def silu_reference(x, dy=None, apply=True):
    z = x.double()
    if not apply:
        return z, z.abs()
    y, m, d1, md1 = silu_terms(z, z.abs())
    if dy is None:
        return y, m
    return dy.double() * d1, dy.double().abs() * md1


# ---------------------------------------------------------------------------------------------- checks
def _coords(flat, shape):
    out = []
    for n in reversed(shape):
        out.append(flat % n)
        flat //= n
    return "(" + ", ".join(map(str, reversed(out))) + ")"


def check(y, r, m, key, rounded, what, z=None):
    """Asserts the per-element bound and the L2 bound of `y` against the float64 reference `r` with magnitude `m` (eps EPS[key]).
    Returns (ratio, relative L2 error): ratio = max |y - r| / m, for bf16 output max (|y - r| - 2^-8 |r|) / m (the error beyond
    a round-to-nearest of r, which the eps term has to cover).  `z`: the SiLU input, quoted with the worst element."""
    assert tuple(y.shape) == tuple(r.shape), (what, tuple(y.shape), tuple(r.shape))
    eps = EPS[key]
    yd = y.double()
    err = (yd - r).abs()
    bound = eps * m + (U_BF16 * r.abs() if rounded else 0.0)
    ok = err <= bound                          # NaN compares false
    l2 = float((yd - r).norm() / r.norm().clamp_min(1e-300))
    excess = (err - U_BF16 * r.abs()).clamp_min(0) if rounded else err
    ratio = float(torch.where(m > 0, excess / m.clamp_min(1e-300), torch.where(excess > 0, math.inf, 0.0)).nan_to_num(nan=math.inf).max())
    if not bool(ok.all()):
        score = torch.where(ok, torch.full_like(err, -1.0), (err - bound) / bound.clamp_min(1e-300)).nan_to_num(nan=math.inf)
        i = int(score.flatten().argmax())
        yv, rv, mv, bv = (float(t.flatten()[i]) for t in (yd, r, m, bound))
        zt = f"z={float(z.flatten()[i])!r} " if z is not None else ""
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of bound; worst at {_coords(i, tuple(y.shape))}: "
                             f"{zt}y={yv!r} r={rv!r} m={mv!r} |y-r|={abs(yv - rv)!r} > bound {bv!r}; rel L2 {l2:.3e}")
    assert not rounded or l2 <= U_BF16, f"{what}: relative L2 error {l2:.3e} > {U_BF16:.3e}"
    return ratio, l2


def _z(x, ab):
    return ab[..., 0].double()[:, None, :] * x.double() + ab[..., 1].double()[:, None, :]


def assert_silu_tail(z, what):
    lim, frac = SILU_TAIL
    got = float((z < lim).double().mean())
    assert got >= frac, f"{what}: only {got:.2%} of z below {lim} (the inputs must exercise the negative tail of SiLU)"


def check_gn_fwd(r, inp, y, stat, ab, what):
    """Stages (a) stat, (b) ab, (c) y of a GroupNorm forward; returns {output: (ratio, l2)}."""
    x = inp["x"]
    res = {}
    for name, (ref, m) in gn_stat_reference(x, r["G"], r["eps"]).items():
        res[name] = check(stat[..., ["mean", "rstd"].index(name)], ref, m, f"gn.{name}", False, f"{what} stat {name}")
    for name, (ref, m) in gn_ab_reference(stat, inp["gamma"], inp["beta"], r["G"]).items():
        res[name] = check(ab[..., ["a", "b"].index(name)], ref, m, f"gn.{name}", False, f"{what} ab {name}")
    z = _z(x, ab)
    if r["silu"]:
        assert_silu_tail(z, what)
    ref, m = gn_y_reference(x, ab, r["silu"])
    res["y"] = check(y, ref, m, "gn.y", True, f"{what} y", z if r["silu"] else None)
    return res


def check_gn_bwd(r, inp, stat, ab, dx, dgamma, dbeta, what):
    z = _z(inp["x"], ab)
    if r["silu"]:
        assert_silu_tail(z, what)
    ref = gn_bwd_reference(inp["x"], inp["dy"], inp["gamma"], stat, ab, r["G"], r["silu"], inp.get("add"))
    out = {"dx": dx, "dgamma": dgamma, "dbeta": dbeta}
    return {n: check(out[n], rv, m, f"gn.{n}", n == "dx", f"{what} {n}", z if (n == "dx" and r["silu"]) else None)
            for n, (rv, m) in ref.items() if out[n] is not None}


def check_ln_fwd(r, inp, y, stat, what):
    res = {}
    for name, (ref, m) in ln_stat_reference(inp["x"], r["eps"]).items():
        res[name] = check(stat[:, ["mean", "rstd"].index(name)], ref, m, f"ln.{name}", False, f"{what} stat {name}")
    ref, m = ln_y_reference(inp["x"], inp["gamma"], inp["beta"], stat)
    res["y"] = check(y, ref, m, "ln.y", True, f"{what} y")
    return res


def check_ln_bwd(r, inp, stat, dx, dgamma, dbeta, what):
    ref = ln_bwd_reference(inp["x"], inp["dy"], inp["gamma"], stat, inp.get("add"))
    out = {"dx": dx, "dgamma": dgamma, "dbeta": dbeta}
    return {n: check(out[n], rv, m, f"ln.{n}", n == "dx", f"{what} {n}") for n, (rv, m) in ref.items() if out[n] is not None}


def check_geglu(r, inp, out, what):
    ref, m = geglu_reference(inp["proj"], inp.get("dout"))
    key = "geglu.dproj" if r["kind"] == "geglu_bwd" else "geglu.y"
    return {key.split(".")[1]: check(out, ref, m, key, True, f"{what} {key.split('.')[1]}")}


def check_silu(r, inp, out, what):
    k = r["kind"]
    apply = r.get("apply", 1)
    if apply:
        assert_silu_tail(inp["x"].double(), what)
    bwd = k in ("silu_bf16_bwd", "silu_bwd_f32")
    ref, m = silu_reference(inp["x"], inp.get("dy") if bwd else None, apply)
    name = "dx" if bwd else "y"
    return {name: check(out, ref, m, f"silu.{name}", k != "silu_bwd_f32", f"{what} {name}", inp["x"].double())}


def old_metric(y, r):
    """max|y - r| / max|r|: the per-kernel tests' tolerance metric (they accept < 1e-2 for bf16 output)."""
    return float((y.double() - r).abs().max() / r.abs().max())
