"""Every GroupNorm, LayerNorm, GEGLU and SiLU launch of a cfg-2 training step (tests/golden/norm_launches.json), run through the
prims entry points with the statistics configuration the step uses and checked element by element against a float64
reference (tests/norm_check.py).

  groupnorm_fwd: with the producer sums the step passes (prims.channel_stats per frame slot, split at C0 where the step passes
                 two sources), and again without them (the kernel computes its own sums);
  groupnorm_bwd: from the kernel's own forward stat / ab, dgamma = 1 and dbeta = 3 accumulated;
  layernorm_bwd: from the kernel's own forward stat, dgamma = 1 and dbeta = 3 accumulated.
Outputs written without atomics (the forward y of every kernel given the same sums, and the element-wise backward kernels) must
be reproduced bit for bit by a second call.  Each check prints one NORMCHECK line: max |y - r| / m and the relative L2 error.
test_silu_sweep runs every SiLU path over z in [-20, 20]."""
import pytest
import torch

import norm_check as N

pytestmark = pytest.mark.gpu

LAUNCHES = N.launches()


def _report(lid, res):
    for name, (ratio, l2) in res.items():
        print(f"NORMCHECK {lid} {name} ratio={ratio:.3e} l2={l2:.3e}")


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _same(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), f"{what}: a second call changed the output"


def _gn_fwd(r, inp, lid):
    from t2v_b200 import prims
    x, gamma, beta = inp["x"], inp["gamma"], inp["beta"]
    stats = N.producer_stats(x, r, prims.channel_stats)
    fps = r["fps"] if stats else 1

    def run(st):
        return prims.groupnorm_fwd(x, gamma, beta, r["G"], r["eps"], r["silu"], st, fps if st else 1)

    y, stat, ab = run(stats)
    res = N.check_gn_fwd(r, inp, y, stat, ab, lid)
    if stats:
        _same(y, run(stats)[0], f"{lid} y")
        y0, stat0, ab0 = run(None)
        res.update({f"{k}_ownsums": v for k, v in N.check_gn_fwd(r, inp, y0, stat0, ab0, f"{lid} (own sums)").items()})
    return res


def _gn_bwd(r, inp, lid):
    from t2v_b200 import prims
    C = r["C"]
    x, gamma = inp["x"], inp["gamma"]
    _, stat, ab = prims.groupnorm_fwd(x, gamma, inp["beta"], r["G"], 1e-5, r["silu"])
    dg = torch.ones(C, device="cuda") if r["dgamma"] else None
    db = torch.full((C,), 3.0, device="cuda") if r["dbeta"] else None
    dx = prims.groupnorm_bwd(inp["dy"], x, gamma, stat, ab, r["G"], r["silu"], inp.get("add"), dg, db)
    return N.check_gn_bwd(r, inp, stat, ab, dx, dg, db, lid)


def _ln_fwd(r, inp, lid):
    from t2v_b200 import prims
    y, stat = prims.layernorm_fwd(inp["x"], inp["gamma"], inp["beta"], r["eps"])
    res = N.check_ln_fwd(r, inp, y, stat, lid)
    _same(y, prims.layernorm_fwd(inp["x"], inp["gamma"], inp["beta"], r["eps"])[0], f"{lid} y")
    return res


def _ln_bwd(r, inp, lid):
    from t2v_b200 import prims
    C = r["C"]
    _, stat = prims.layernorm_fwd(inp["x"], inp["gamma"], inp["beta"], 1e-5)
    dg = torch.ones(C, device="cuda") if r["dgamma"] else None
    db = torch.full((C,), 3.0, device="cuda") if r["dbeta"] else None
    dx = prims.layernorm_bwd(inp["dy"], inp["x"], inp["gamma"], stat, inp.get("add"), dg, db)
    res = N.check_ln_bwd(r, inp, stat, dx, dg, db, lid)
    _same(dx, prims.layernorm_bwd(inp["dy"], inp["x"], inp["gamma"], stat, inp.get("add")), f"{lid} dx")
    return res


def _elementwise(r, inp, lid):
    from t2v_b200 import prims
    k = r["kind"]
    if k == "geglu_fwd":
        run = lambda: prims.geglu_fwd(inp["proj"])   # noqa: E731
    elif k == "geglu_bwd":
        run = lambda: prims.geglu_bwd(inp["proj"], inp["dout"])   # noqa: E731
    elif k == "silu_f32_to_bf16":
        run = lambda: prims.silu_f32_to_bf16(inp["x"], bool(r["apply"]))   # noqa: E731
    elif k in ("silu_bf16_bwd", "silu_bwd_f32"):
        run = lambda: getattr(prims, k)(inp["x"], inp["dy"])   # noqa: E731
    else:
        run = lambda: prims.silu_bf16(inp["x"])   # noqa: E731
    out = run()
    res = (N.check_geglu if k.startswith("geglu") else N.check_silu)(r, inp, out, lid)
    _same(out, run(), f"{lid} output")
    return res


RUN = {"groupnorm_fwd": _gn_fwd, "groupnorm_bwd": _gn_bwd, "layernorm_fwd": _ln_fwd, "layernorm_bwd": _ln_bwd}


@pytest.mark.parametrize("r", LAUNCHES, ids=[N.launch_id(r) for r in LAUNCHES])
def test_step_norm(r):
    lid = N.launch_id(r)
    inp = N.make_inputs(r, "cuda")
    _report(lid, RUN.get(r["kind"], _elementwise)(r, inp, lid))


def test_silu_sweep():
    """z over [-20, 20] through every SiLU path: the element-wise kernels directly, GroupNorm through gamma (x spans [-1, 1]
    in every channel, so a = gamma rstd maps it onto [-20, 20] and b ~ 0)."""
    n = 8192
    z = torch.linspace(-20, 20, n, device="cuda")
    dy = torch.linspace(-1, 1.5, n, device="cuda").flip(0)
    cases = [({"kind": "silu_bf16", "shape": [n]}, {"x": z.bfloat16()}),
             ({"kind": "silu_bf16_bwd", "shape": [n]}, {"x": z.bfloat16(), "dy": dy.bfloat16()}),
             ({"kind": "silu_f32_to_bf16", "shape": [n], "apply": 1}, {"x": z}),
             ({"kind": "silu_bwd_f32", "shape": [n]}, {"x": z, "dy": dy})]
    for r, inp in cases:
        _report(f"sweep-{r['kind']}", _elementwise(r, inp, f"sweep-{r['kind']}"))
    from t2v_b200 import prims
    S, P, C, G = 1, n, 64, 32
    x = torch.linspace(-1, 1, P, device="cuda")[None, :, None].expand(S, P, C).contiguous().bfloat16()
    gamma = torch.full((C,), 20 * (1 / 3) ** 0.5, device="cuda")
    beta = torch.zeros(C, device="cuda")
    r = {"kind": "groupnorm_fwd", "S": S, "P": P, "C": C, "G": G, "eps": 1e-5, "silu": 1}
    inp = {"x": x, "gamma": gamma, "beta": beta, "dy": dy.bfloat16()[None, :, None].expand(S, P, C).contiguous()}
    y, stat, ab = prims.groupnorm_fwd(x, gamma, beta, G, 1e-5, 1)
    _report("sweep-groupnorm_fwd", N.check_gn_fwd(r, inp, y, stat, ab, "sweep-groupnorm_fwd"))
    dg, db = torch.ones(C, device="cuda"), torch.full((C,), 3.0, device="cuda")
    dx = prims.groupnorm_bwd(inp["dy"], x, gamma, stat, ab, G, 1, None, dg, db)
    _report("sweep-groupnorm_bwd", N.check_gn_bwd(r, inp, stat, ab, dx, dg, db, "sweep-groupnorm_bwd"))
