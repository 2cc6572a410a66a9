"""The checks of tests/norm_check.py have teeth, shown without a GPU.  The fp32 oracle (oracle/ops_ref.py: fp32 math, one rounding
to bf16, an accurate sigmoid) stands in for the kernels on step launches small enough for the CPU; the checks must accept its
output with the eps constants the GPU test uses, and must reject outputs broken the way a defect of the kernels would break
them.  The old max|y - r| / max|r| < 1e-2 metric accepts a sigmoid built on an 11-bit tanh."""
import json

import pytest
import torch
import torch.nn.functional as F

import norm_check as N
from oracle import ops_ref as O

# step launches the CPU checks in seconds (the first two GroupNorms are the ones with a two-source split and fps = 4 slots)
CASES = {
    "gn_fwd_two_sources": dict(kind="groupnorm_fwd", S=16, P=16, C=2560, G=32, eps=1e-5, silu=1, stats=2, frames=16, C0=1280, fps=1),
    "gn_fwd_per_clip": dict(kind="groupnorm_fwd", S=1, P=16384, C=320, G=32, eps=1e-5, silu=1, stats=1, frames=4, C0=320, fps=4),
    "gn_fwd_c320": dict(kind="groupnorm_fwd", S=16, P=256, C=320, G=32, eps=1e-5, silu=1, stats=1, frames=16, C0=320, fps=1),
    "gn_bwd_silu": dict(kind="groupnorm_bwd", S=16, P=16, C=1280, G=32, silu=1, add=0, dgamma=1, dbeta=1),
    "ln_fwd": dict(kind="layernorm_fwd", rows=256, C=1280, eps=1e-5),
    "ln_bwd": dict(kind="layernorm_bwd", rows=256, C=1280, add=0, dgamma=1, dbeta=1),
    "geglu_fwd": dict(kind="geglu_fwd", M=256, I=5120),
    "geglu_bwd": dict(kind="geglu_bwd", M=256, I=5120),
    "silu_bf16": dict(kind="silu_bf16", shape=[1, 1280]),
    "silu_bf16_bwd": dict(kind="silu_bf16_bwd", shape=[1, 1280]),
    "silu_cast": dict(kind="silu_f32_to_bf16", shape=[1, 1, 1, 320], apply=0),
}

_CACHE = {}


def _launch(name):
    want = CASES[name]
    for r in N.launches():
        if r == want:
            return r
    raise AssertionError(f"{name} is not a launch of tests/golden/norm_launches.json")


def _case(name):
    """(launch, inputs, oracle outputs) of a named launch, computed once."""
    if name not in _CACHE:
        r = _launch(name)
        inp = N.make_inputs(r, "cpu")
        k = r["kind"]
        if k == "groupnorm_fwd":
            st = N.producer_stats(inp["x"], r, O.channel_stats)
            y, stat, ab = O.groupnorm_fwd(inp["x"], inp["gamma"], inp["beta"], r["G"], r["eps"], r["silu"], st, r["fps"])
            out = {"y": y, "stat": stat, "ab": ab, "sums": st}
        elif k == "groupnorm_bwd":
            _, stat, ab = O.groupnorm_fwd(inp["x"], inp["gamma"], inp["beta"], r["G"], 1e-5, r["silu"])
            dg, db = torch.ones(r["C"]), torch.full((r["C"],), 3.0)
            dx = O.groupnorm_bwd(inp["dy"], inp["x"], inp["gamma"], stat, ab, r["G"], r["silu"], None, dg, db)
            out = {"stat": stat, "ab": ab, "dx": dx, "dgamma": dg, "dbeta": db}
        elif k == "layernorm_fwd":
            y, stat = O.layernorm_fwd(inp["x"], inp["gamma"], inp["beta"], r["eps"])
            out = {"y": y, "stat": stat}
        elif k == "layernorm_bwd":
            _, stat = O.layernorm_fwd(inp["x"], inp["gamma"], inp["beta"], 1e-5)
            dg, db = torch.ones(r["C"]), torch.full((r["C"],), 3.0)
            out = {"stat": stat, "dx": O.layernorm_bwd(inp["dy"], inp["x"], inp["gamma"], stat, None, dg, db), "dgamma": dg, "dbeta": db}
        elif k == "geglu_fwd":
            out = {"out": O.geglu_fwd(inp["proj"])}
        elif k == "geglu_bwd":
            out = {"out": O.geglu_bwd(inp["proj"], inp["dout"])}
        elif k == "silu_f32_to_bf16":
            out = {"out": O.silu_f32_to_bf16(inp["x"], bool(r["apply"]))}
        elif k == "silu_bf16_bwd":
            out = {"out": O.silu_bf16_bwd(inp["x"], inp["dy"])}
        else:
            out = {"out": O.silu_bf16(inp["x"])}
        _CACHE[name] = (r, inp, out)
    return _CACHE[name]


def _check(name, out):
    """Every check the GPU test applies to the step's launch of `name`, on `out`."""
    r, inp, _ = _case(name)
    k = r["kind"]
    if k == "groupnorm_fwd":
        return N.check_gn_fwd(r, inp, out["y"], out["stat"], out["ab"], name)
    if k == "groupnorm_bwd":
        return N.check_gn_bwd(r, inp, out["stat"], out["ab"], out["dx"], out["dgamma"], out["dbeta"], name)
    if k == "layernorm_fwd":
        return N.check_ln_fwd(r, inp, out["y"], out["stat"], name)
    if k == "layernorm_bwd":
        return N.check_ln_bwd(r, inp, out["stat"], out["dx"], out["dgamma"], out["dbeta"], name)
    return (N.check_geglu if k.startswith("geglu") else N.check_silu)(r, inp, out["out"], name)


# ---------------------------------------------------------------------------------------------- census
COUNTS = {"groupnorm_fwd": 26, "groupnorm_bwd": 26, "layernorm_fwd": 5, "layernorm_bwd": 5, "geglu_fwd": 5, "geglu_bwd": 5,
          "silu_bf16": 1, "silu_bf16_bwd": 1, "silu_f32_to_bf16": 3, "silu_bwd_f32": 0}


def test_census_matches_gpu_parametrization():
    recs = N.launches()
    assert {k: sum(r["kind"] == k for r in recs) for k in COUNTS} == COUNTS
    assert len(recs) == sum(COUNTS.values())
    assert len({N.launch_id(r) for r in recs}) == len(recs)
    import test_norm_step_gpu as G
    (mark,) = [m for m in G.test_step_norm.pytestmark if m.name == "parametrize"]
    assert mark.args[1] == recs


def test_census_reproduced_by_generator():
    """The full-size cfg-2 step on the CPU over the oracle (GEMMs replaced by allocators) makes exactly the recorded launches."""
    import sys
    sys.path.insert(0, N.HERE + "/golden")
    import make_norm_launches as M
    assert json.loads(json.dumps(M.step_launches())) == N.launches()


# ---------------------------------------------------------------------------------------------- the oracle passes
@pytest.mark.parametrize("name", list(CASES))
def test_oracle_output_passes(name):
    _check(name, _case(name)[2])


def test_oracle_own_sums_pass():
    """The same GroupNorm without producer sums (the kernel's fallback computes its own)."""
    r, inp, _ = _case("gn_fwd_two_sources")
    y, stat, ab = O.groupnorm_fwd(inp["x"], inp["gamma"], inp["beta"], r["G"], r["eps"], r["silu"])
    N.check_gn_fwd(r, inp, y, stat, ab, "own sums")


def test_silu_sweep_oracle_passes():
    z = torch.linspace(-20, 20, 8192)
    dy = torch.linspace(-1, 1.5, 8192).flip(0)
    for r, inp, out in (({"kind": "silu_bf16", "shape": [8192]}, {"x": z.bfloat16()}, O.silu_bf16(z.bfloat16())),
                        ({"kind": "silu_bwd_f32", "shape": [8192]}, {"x": z, "dy": dy}, O.silu_bwd_f32(z, dy)),
                        ({"kind": "silu_f32_to_bf16", "shape": [8192], "apply": 1}, {"x": z}, O.silu_f32_to_bf16(z))):
        N.check_silu(r, inp, out, r["kind"])


# ---------------------------------------------------------------------------------------------- broken outputs are rejected
def sigmoid_tanh11(z):
    """0.5 tanh(z / 2) + 0.5 with tanh rounded to 11 significant bits: the error of the hardware tanh (tanh.approx.f32)."""
    m, e = torch.frexp(torch.tanh(0.5 * z))
    return 0.5 * torch.ldexp(torch.round(m * 2048) / 2048, e) + 0.5


def _z32(x, ab):
    return ab[..., 0][:, None, :] * x.float() + ab[..., 1][:, None, :]


def _gn_bwd_f32(name, sigmoid=torch.sigmoid, drop_z_term=False):
    """The oracle's GroupNorm backward in fp32 with the SiLU derivative built on `sigmoid` (optionally without z (1 - s))."""
    r, inp, out = _case(name)
    x, gamma, stat, ab = inp["x"], inp["gamma"], out["stat"], out["ab"]
    S, P, C = x.shape
    G, cpg = r["G"], C // r["G"]
    mean, rstd = (stat[..., i].repeat_interleave(cpg, dim=1)[:, None, :] for i in (0, 1))
    xh = (x.float() - mean) * rstd
    z = _z32(x, ab)
    s = sigmoid(z)
    dz = inp["dy"].float() * (s if drop_z_term else s * (1 + z * (1 - s)))
    dxh = (dz * gamma).view(S, P, G, cpg)
    xg = xh.view(S, P, G, cpg)
    dx = rstd.view(S, 1, G, cpg) * (dxh - dxh.mean(dim=(1, 3), keepdim=True) - xg * (dxh * xg).mean(dim=(1, 3), keepdim=True))
    return {"stat": stat, "ab": ab, "dx": dx.view(S, P, C).bfloat16(), "dgamma": 1 + (dz * xh).sum(dim=(0, 1)),
            "dbeta": 3 + dz.sum(dim=(0, 1))}


def _gn_fwd_tanh_sigmoid():
    _, inp, out = _case("gn_fwd_c320")
    z = _z32(inp["x"], out["ab"])
    return dict(out, y=(z * sigmoid_tanh11(z)).bfloat16())


def _gn_group_from_vector_start():
    """Every channel takes the statistics of the group of its 8-channel vector's first channel (C = 320: 10 channels per group,
    so channels 10..15 of vector 1 read group 0)."""
    r, inp, out = _case("gn_fwd_c320")
    C, cpg = r["C"], r["C"] // r["G"]
    grp = (torch.arange(C) // 8 * 8) // cpg
    mean, rstd = out["stat"][..., 0][:, grp], out["stat"][..., 1][:, grp]
    a = rstd * inp["gamma"]
    ab = torch.stack([a, inp["beta"] - mean * a], -1)
    return dict(out, ab=ab, y=F.silu(_z32(inp["x"], ab)).bfloat16())


def _gn_tail_unnormalised():
    """The last 5 pixels of the last sample (the ragged end of its last chunk) keep x."""
    _, inp, out = _case("gn_fwd_c320")
    y = out["y"].clone()
    y[-1, -5:] = inp["x"][-1, -5:]
    return dict(out, y=y)


def _gn_with_sums(name, sums):
    r, inp, out = _case(name)
    y, stat, ab = O.groupnorm_fwd(inp["x"], inp["gamma"], inp["beta"], r["G"], r["eps"], r["silu"], sums, r["fps"])
    return {"y": y, "stat": stat, "ab": ab}


def _gn_one_slot():
    """A per-clip norm (4 frame slots per sample) that sums slot 0 only."""
    r, _, out = _case("gn_fwd_per_clip")
    st = out["sums"][0].clone()
    st.view(r["S"], r["fps"], r["C"], 2)[:, 1:] = 0
    return _gn_with_sums("gn_fwd_per_clip", [st])


def _gn_split_off_by_8():
    """The second source read from channel C0 + 8 on (the split at the concatenation misplaced by one vector)."""
    _, _, out = _case("gn_fwd_two_sources")
    s0, s1 = out["sums"]
    return _gn_with_sums("gn_fwd_two_sources", [s0, torch.cat([s1[:, 8:], torch.zeros_like(s1[:, :8])], 1)])


def _dparams(how):
    r, inp, out = _case("gn_bwd_silu")
    dg, db = (torch.ones(r["C"]), torch.full((r["C"],), 3.0)) if how == "twice" else (torch.zeros(r["C"]), torch.zeros(r["C"]))
    for _ in range(2 if how == "twice" else 1):
        O.groupnorm_bwd(inp["dy"], inp["x"], inp["gamma"], out["stat"], out["ab"], r["G"], r["silu"], None, dg, db)
    return dict(out, dgamma=dg, dbeta=db)


MUTATIONS = {
    "sigmoid_tanh11_fwd": ("gn_fwd_c320", _gn_fwd_tanh_sigmoid),
    "sigmoid_tanh11_bwd": ("gn_bwd_silu", lambda: _gn_bwd_f32("gn_bwd_silu", sigmoid_tanh11)),
    "group_from_vector_start": ("gn_fwd_c320", _gn_group_from_vector_start),
    "tail_pixels_unnormalised": ("gn_fwd_c320", _gn_tail_unnormalised),
    "per_clip_one_slot": ("gn_fwd_per_clip", _gn_one_slot),
    "two_source_split_off_by_8": ("gn_fwd_two_sources", _gn_split_off_by_8),
    "dparams_added_twice": ("gn_bwd_silu", lambda: _dparams("twice")),
    "dparams_overwritten": ("gn_bwd_silu", lambda: _dparams("overwritten")),
    "silu_derivative_z_term_dropped": ("gn_bwd_silu", lambda: _gn_bwd_f32("gn_bwd_silu", drop_z_term=True)),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_rejected(mutation):
    name, make = MUTATIONS[mutation]
    with pytest.raises(AssertionError, match="out of bound"):
        _check(name, make())


def test_fp32_bwd_restatement_passes():
    """The fp32 backward the sigmoid mutations are built from passes with an accurate sigmoid: the mutations fail for the
    sigmoid alone."""
    _check("gn_bwd_silu", _gn_bwd_f32("gn_bwd_silu"))


def test_tanh_sigmoid_rejected_and_missed_by_old_metric():
    """The sigmoid of the hardware tanh stays below 1e-2 of max|y| (forward) and max|dx| (backward), so the per-kernel
    tests' metric accepts it, though it is wrong by several bf16 ulps where z < -4."""
    _, inp, out = _case("gn_fwd_c320")
    y = _gn_fwd_tanh_sigmoid()["y"]
    r_y, _ = N.gn_y_reference(inp["x"], out["ab"], 1)
    assert N.old_metric(y, r_y) < 1e-2
    r, inp, out = _case("gn_bwd_silu")
    dx = _gn_bwd_f32("gn_bwd_silu", sigmoid_tanh11)["dx"]
    r_dx = N.gn_bwd_reference(inp["x"], inp["dy"], inp["gamma"], out["stat"], out["ab"], r["G"], 1)["dx"][0]
    assert N.old_metric(dx, r_dx) < 1e-2
    with pytest.raises(AssertionError, match="out of bound"):
        _check("gn_fwd_c320", _gn_fwd_tanh_sigmoid())
