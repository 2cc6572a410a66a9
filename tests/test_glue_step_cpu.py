"""The checks of tests/glue_check.py have teeth, shown without a GPU.  An fp32 restatement of each glue kernel (oracle/ops_ref.py
where it states the operation, local ones for gelu_bwd, embed_tokens_bwd, the velocity loss and the ragged resize, which it does
not) stands in for the kernels on census launches small enough for the CPU: the checks must accept it with the eps the GPU test
uses, and reject outputs broken the way a defect of the kernels would break them.  OLD_METRIC_ACCEPTS pins which of those the
per-kernel tests' max|y - r| / max|r| < 1e-2 metric would let through."""
import json
import math
import sys

import pytest
import torch

import glue_check as G

# ---------------------------------------------------------------------------------------------- census
COUNTS = {"latents_to_nhwc8": 6, "nhwc8_to_latents": 1, "mse_loss_fwd": 5, "mse_loss_bwd": 5, "velocity_mse_loss_fwd": 2,
          "velocity_mse_loss_bwd": 2, "timestep_embedding": 3, "colsum": 25, "colsum_f32": 9, "upsample_nearest_fwd": 15,
          "upsample_nearest_bwd": 15, "concat_channels": 32, "split_channels": 32, "add_bf16": 43, "add_f32": 1, "scale_bf16": 1,
          "cast_f32_bf16": 20, "cast_bf16_f32": 1, "dropout_scale_add": 4, "embed_tokens": 1, "embed_tokens_bwd": 2, "gelu_bf16": 2,
          "gelu_bwd": 2, "vae_sample": 3, "frames_u8_to_nhwc8": 2, "frames_u8_to_nhwc8_ragged": 1}


def _golden():
    sys.path.insert(0, G.HERE + "/golden")
    import make_glue_launches as M
    return M


def test_census_matches_gpu_parametrization():
    recs = G.launches()
    assert {k: sum(r["kind"] == k for r in recs) for k in COUNTS} == COUNTS
    assert len(recs) == sum(COUNTS.values())
    assert set(COUNTS) == set(_golden().KINDS)
    assert len({G.launch_id(r) for r in recs}) == len(recs)
    import test_glue_step_gpu as GPU
    (mark,) = [m for m in GPU.test_step_glue.pytestmark if m.name == "parametrize"]
    assert mark.args[1] == recs


def test_census_covers_the_edges():
    """colsum past the first column block and with row-bias segments, add_noise and the velocity at B = 4, an embed_tokens_bwd
    whose prompt repeats an id into both tables, both GELU forms, dropout forward with a base and backward without, both cast
    forms, and a ragged resize of two source sizes."""
    recs = G.launches()
    assert any(r["kind"] == "colsum" and r["blocks"] > 1 for r in recs)
    assert any(r["kind"] == "colsum" and r["S"] > 1 for r in recs)
    assert any(r["kind"] == "colsum_f32" and r["S"] > 1 for r in recs)
    for kind in ("latents_to_nhwc8", "velocity_mse_loss_fwd", "velocity_mse_loss_bwd", "timestep_embedding"):
        assert any(r["kind"] == kind and r["B"] == 4 for r in recs), kind
    assert any(r["kind"] == "latents_to_nhwc8" and not r["noise"] for r in recs)
    bwd = [r for r in recs if r["kind"] == "embed_tokens_bwd" and r["dtok"] and r["dpos"]]
    assert bwd and all(len(set(G.make_inputs(r)["ids"][0].tolist())) < r["L"] for r in bwd)
    for kind in ("gelu_bf16", "gelu_bwd"):
        assert {r["quick"] for r in recs if r["kind"] == kind} == {0, 1}, kind
    assert {r["base"] for r in recs if r["kind"] == "dropout_scale_add" and r["p"] > 0} == {0, 1}
    assert {r["into"] for r in recs if r["kind"] == "cast_f32_bf16"} == {0, 1}
    assert any(r["kind"] == "add_bf16" and r["inputs"] == 3 for r in recs)
    assert any(r["kind"] == "frames_u8_to_nhwc8_ragged" and len({tuple(c[1:]) for c in r["clips"]}) > 1 for r in recs)
    synth = [r for r in recs if r.get("synthetic")]
    assert {r["kind"] for r in synth} == {"colsum", "nhwc8_to_latents", "scale_bf16", "gelu_bf16", "gelu_bwd", "embed_tokens_bwd"}


def _module_functions(mod):
    return {n: v for n, v in vars(mod).items() if callable(v)}


def test_census_reproduced_by_generator():
    """The workloads on the meta device make exactly the recorded launches, and leave every prims / ops function, the dropout
    epochs and the CPU random state as they found them."""
    from t2v_b200 import ops, prims
    before = {m.__name__: _module_functions(m) for m in (prims, ops)}
    flash, epochs, rng = ops._Flash.enabled, dict(ops._epochs), torch.get_rng_state()
    assert json.loads(json.dumps(_golden().step_launches())) == G.launches()
    for m in (prims, ops):
        after = _module_functions(m)
        changed = sorted(n for n in before[m.__name__].keys() | after.keys() if before[m.__name__].get(n) is not after.get(n))
        assert not changed, f"the census left {m.__name__}.{changed} replaced"
    assert ops._Flash.enabled == flash
    assert ops._epochs.keys() == epochs.keys() and all(ops._epochs[k] is t for k, t in epochs.items())
    assert torch.equal(torch.get_rng_state(), rng), "the census moved the CPU random state"


# ---------------------------------------------------------------------------------------------- fp32 restatements
def velocity_f32(inp, shift=0):
    """The velocity in fp32 as the kernel forms it; `shift` reads abar[t - shift]."""
    a = inp["abar"][inp["t"] - shift].view(-1, 1, 1, 1, 1)
    return a.sqrt() * inp["noise"] - (1 - a).sqrt() * inp["x0"]


def _mse(pred, target, C, gout=None):
    B, C_, F, H, W = target.shape
    p = pred.float().view(B, F, H, W, 8)[..., :C].permute(0, 4, 1, 2, 3)
    e = p - target
    if gout is None:
        return (e * e).mean()
    from oracle import ops_ref
    return ops_ref.latents_to_nhwc8((2.0 * e / e.numel() * gout).contiguous())


def gelu_bwd_f32(x, dy, quick, tanh_form=False):
    xf = x.float()
    if tanh_form:
        c = math.sqrt(2 / math.pi)
        u = c * (xf + 0.044715 * xf ** 3)
        th = torch.tanh(u)
        g = 0.5 * (1 + th) + 0.5 * xf * (1 - th * th) * c * (1 + 3 * 0.044715 * xf * xf)
    else:
        import text_lora_ref
        g = text_lora_ref.gelu_grad_f32(xf, bool(quick))
    return (dy.float() * g).bfloat16()


def embed_bwd_f32(r, inp, every_row=False):
    """dtok / dpos accumulated in fp32; `every_row`: a repeated id's sum added once per row that holds it."""
    B, L, C, V = r["B"], r["L"], r["C"], r["vocab"]
    ids = inp["ids"].clamp(0, V - 1).flatten()
    dy = inp["dy"].float()
    out = {}
    if r["dtok"]:
        dtok = inp["dtok"].clone()
        acc = torch.zeros(V, C).index_add_(0, ids, dy)
        if every_row:
            for i in torch.unique(ids).tolist():
                dtok[i] += acc[i] * int((ids == i).sum())
        else:
            dtok += acc
        out["dtok"] = dtok
    if r["dpos"]:
        dpos = inp["dpos"].clone()
        dpos[:L] += dy.view(B, L, C).sum(0)
        out["dpos"] = dpos
    return out


def restate(r, inp):
    """The launch's outputs from fp32 restatements, as the GPU test's run() returns them."""
    from oracle import ops_ref as O
    k = r["kind"]
    if k == "latents_to_nhwc8":
        return {"y": O.latents_to_nhwc8(inp["x0"], inp.get("noise"), inp.get("abar"), inp.get("t"))}
    if k == "nhwc8_to_latents":
        return {"out": O.nhwc8_to_latents(inp["x"], r["B"], r["C"], r["F"])}
    if k in ("mse_loss_fwd", "mse_loss_bwd", "velocity_mse_loss_fwd", "velocity_mse_loss_bwd"):
        tgt = velocity_f32(inp) if k.startswith("velocity") else inp["noise"]
        if k.endswith("fwd"):
            return {"loss": _mse(inp["pred"], tgt, r["C"])}
        return {"dpred": _mse(inp["pred"], tgt, r["C"], inp["gout"])}
    if k == "timestep_embedding":
        return {"y": O.timestep_embedding(inp["t"], r["dim"])}
    if k == "colsum":
        out = inp["preset"].clone()
        O.colsum(inp["x"], out, r["S"], r["P"], r["C"])
        return {"out": out}
    if k == "colsum_f32":
        out = inp["preset"].clone()
        O.colsum_f32(inp["x"], out)
        return {"out": out}
    if k == "upsample_nearest_fwd":
        return {"y": O.upsample_nearest_fwd(inp["x"], (r["Ho"], r["Wo"]))}
    if k == "upsample_nearest_bwd":
        return {"dx": O.upsample_nearest_bwd(inp["dy"], (r["H"], r["W"]))}
    if k == "concat_channels":
        return {"y": O.concat_channels(inp["a"], inp["b"])}
    if k == "split_channels":
        a, b = O.split_channels(inp["g"], r["Ca"])
        return {"a": a, "b": b}
    if k == "add_bf16":
        return {"y": O.add_bf16(inp["a"], inp["b"], inp.get("c"))}
    if k == "add_f32":
        return {"y": O.add_f32(inp["a"], inp["b"])}
    if k == "scale_bf16":
        return {"y": O.scale_bf16(inp["a"], r["alpha"])}
    if k == "cast_f32_bf16":
        return {"y": O.cast_f32_bf16(inp["src"])}
    if k == "cast_bf16_f32":
        dst = torch.empty(inp["src"].shape)
        O.cast_bf16_f32(inp["src"], dst)
        return {"y": dst}
    if k == "dropout_scale_add":
        return {"y": O.dropout_scale_add(inp["x"], inp.get("base"), r["p"], r["scale"], inp["seed"], inp["epoch"])}
    if k == "embed_tokens":
        return {"y": O.embed_tokens(inp["ids"], inp["tok"], inp["pos"])}
    if k == "embed_tokens_bwd":
        return embed_bwd_f32(r, inp)
    if k == "gelu_bf16":
        return {"y": O.gelu_bf16(inp["x"], bool(r["quick"]))}
    if k == "gelu_bwd":
        return {"dx": gelu_bwd_f32(inp["x"], inp["dy"], r["quick"])}
    if k == "vae_sample":
        return {"z": O.vae_sample(inp["moments"], inp["eps"], r["B"], r["F"], r["scale"])}
    if k == "frames_u8_to_nhwc8":
        return {"y": O.frames_u8_to_nhwc8(inp["frames"], (r["h"], r["w"]))}
    if k == "frames_u8_to_nhwc8_ragged":
        return {"y": torch.cat([O.frames_u8_to_nhwc8(c, (r["h"], r["w"])) for c in inp["clips"]])}
    raise KeyError(k)


SMALL = 1 << 21   # elements of the largest tensor of a launch the CPU restates


def _size(r):
    if "n" in r:
        return r["n"]
    k = r["kind"]
    if k == "colsum":
        return r["S"] * r["P"] * r["C"]
    if k in ("embed_tokens", "embed_tokens_bwd"):
        return r["vocab"] * r["C"] if (k == "embed_tokens" or r["dtok"]) else r["L"] * r["C"]
    if k in ("frames_u8_to_nhwc8",):
        return r["F"] * r["H0"] * r["W0"] * 3
    if k == "frames_u8_to_nhwc8_ragged":
        return sum(F * H * W * 3 for F, H, W in r["clips"])
    if k.startswith("upsample"):
        return r["N"] * r["Ho"] * r["Wo"] * r["C"]
    if k in ("concat_channels",):
        return r["M"] * (r["Ca"] + r["Cb"])
    if k == "split_channels":
        return r["M"] * r["Ct"]
    if k == "colsum_f32":
        return r["S"] * r["C"]
    if k == "vae_sample":
        return r["B"] * r["F"] * r["h"] * r["w"] * 8
    if k == "timestep_embedding":
        return r["B"] * r["dim"]
    return r["B"] * r["F"] * r["H"] * r["W"] * 8


def _first_small(kind, pred=lambda r: True):
    """The smallest census launch of `kind` satisfying `pred`."""
    cands = [r for r in G.launches() if r["kind"] == kind and pred(r)]
    return min(cands, key=_size)


RESTATED = {}
for _k in COUNTS:
    _r = _first_small(_k)
    if _size(_r) <= 64 * SMALL or _k in ("embed_tokens", "embed_tokens_bwd"):
        RESTATED[G.launch_id(_r)] = _r

_CACHE = {}


def _case(r):
    lid = G.launch_id(r)
    if lid not in _CACHE:
        inp = G.make_inputs(r)
        _CACHE[lid] = (inp, G.reference(r, inp))
    return _CACHE[lid]


@pytest.mark.parametrize("lid", list(RESTATED))
def test_restated_kernels_pass(lid):
    r = RESTATED[lid]
    inp, ref = _case(r)
    G.check_outputs(r, inp, restate(r, inp), lid, ref)


def test_reference_mask_is_the_oracles():
    """keep_mask (numpy uint64) and oracle/ops_ref.py's int64 restatement of mix32 agree, epoch mixing included."""
    from oracle import ops_ref as O
    r = _first_small("dropout_scale_add")
    inp = G.make_inputs(r)
    y = O.dropout_scale_add(torch.ones(r["n"], dtype=torch.bfloat16), None, r["p"], r["scale"], inp["seed"], inp["epoch"])
    assert torch.equal(y != 0, G.keep_mask(r["n"], r["p"], inp["seed"], inp["epoch"]))


def test_resize_reference_is_torch_bilinear():
    r = _first_small("frames_u8_to_nhwc8")
    fr = G.make_inputs(r)["frames"][:1]
    v, _ = G.bilinear(fr, r["h"], r["w"])
    t = torch.nn.functional.interpolate(fr.permute(0, 3, 1, 2).double(), size=(r["h"], r["w"]), mode="bilinear", align_corners=False)
    assert torch.allclose(v, t.permute(0, 2, 3, 1) / 127.5 - 1, rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------------------------- broken outputs are rejected
def _mut_add_noise_t0():
    r = _first_small("latents_to_nhwc8", lambda r: r["noise"] and r["B"] == 4)
    inp, _ = _case(r)
    from oracle import ops_ref as O
    return r, {"y": O.latents_to_nhwc8(inp["x0"], inp["noise"], inp["abar"], inp["t"][:1].expand(r["B"]).contiguous())}


def _mut_velocity_tm1(kind):
    def make():
        r = _first_small(kind, lambda r: r["B"] == 1)
        inp, _ = _case(r)
        tgt = velocity_f32(inp, shift=1)
        if kind.endswith("fwd"):
            return r, {"loss": _mse(inp["pred"], tgt, r["C"])}
        return r, {"dpred": _mse(inp["pred"], tgt, r["C"], inp["gout"])}
    return make


def _colsum_case():
    return _first_small("colsum", lambda r: r["blocks"] > 1)


def _mut_colsum_last_row():
    """The last row of the last (ragged) chunk of each segment left out of the sum."""
    r = _first_small("colsum", lambda r: r["S"] > 1)
    inp, _ = _case(r)
    return r, {"out": inp["preset"] + inp["x"][:, :-1].float().sum(1)}


def _mut_colsum_block_early():
    """The last column block written 8 columns before its place."""
    r = _colsum_case()
    inp, _ = _case(r)
    out = inp["preset"].clone()
    s = inp["x"].float().sum(1)
    c0 = (r["blocks"] - 1) * 4096
    out[:, :c0] += s[:, :c0]
    out[:, c0 - 8:r["C"] - 8] += s[:, c0:]
    return r, {"out": out}


def _mut_add_two_roundings():
    r = _first_small("add_bf16", lambda r: r["inputs"] == 3)
    inp, _ = _case(r)
    return r, {"y": ((inp["a"].float() + inp["b"].float()).bfloat16().float() + inp["c"].float()).bfloat16()}


def _mut_gelu_tanh():
    r = _first_small("gelu_bwd", lambda r: not r["quick"])
    inp, _ = _case(r)
    return r, {"dx": gelu_bwd_f32(inp["x"], inp["dy"], 0, tanh_form=True)}


def _mut_embed_every_row():
    r = _first_small("embed_tokens_bwd", lambda r: r["dtok"] and r["dpos"])
    inp, _ = _case(r)
    return r, embed_bwd_f32(r, inp, every_row=True)


def _mut_cast_truncates():
    r = _first_small("cast_f32_bf16")
    inp, _ = _case(r)
    return r, {"y": (inp["src"].view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()}


def _mut_dropout_shift():
    """The backward's mask read one element late."""
    r = _first_small("dropout_scale_add", lambda r: not r["base"])
    inp, _ = _case(r)
    keep = G.keep_mask(r["n"] + 1, r["p"], inp["seed"], inp["epoch"])[1:]
    k = torch.tensor(r["scale"], dtype=torch.float32) / (1 - torch.tensor(r["p"], dtype=torch.float32))
    return r, {"y": torch.where(keep, inp["x"].float() * k, torch.zeros(())).bfloat16()}


def _mut_temb_shift():
    """Timesteps(downscale_freq_shift=1): f_i = exp(-ln(10000) i / (half - 1))."""
    r = _first_small("timestep_embedding")
    inp, _ = _case(r)
    half = r["dim"] // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / (half - 1))
    a = inp["t"][:, None].float() * f[None]
    return r, {"y": torch.cat([torch.cos(a), torch.sin(a)], -1).bfloat16()}


def _mut_resize_align_corners():
    r = _first_small("frames_u8_to_nhwc8")
    inp, _ = _case(r)
    v, _ = G.bilinear(inp["frames"], r["h"], r["w"], align_corners=True)
    y = torch.cat([v, torch.zeros(v.shape[:-1] + (5,), dtype=torch.float64)], -1)
    return r, {"y": y.bfloat16()}


MUTATIONS = {
    "add_noise_sample0_timestep": _mut_add_noise_t0,
    "velocity_abar_t_minus_1_loss": _mut_velocity_tm1("velocity_mse_loss_fwd"),
    "velocity_abar_t_minus_1_dpred": _mut_velocity_tm1("velocity_mse_loss_bwd"),
    "colsum_ragged_chunk_last_row_dropped": _mut_colsum_last_row,
    "colsum_last_block_8_columns_early": _mut_colsum_block_early,
    "add3_two_roundings": _mut_add_two_roundings,
    "gelu_bwd_tanh_form": _mut_gelu_tanh,
    "embed_bwd_repeated_id_every_row": _mut_embed_every_row,
    "cast_truncates": _mut_cast_truncates,
    "dropout_bwd_mask_shifted": _mut_dropout_shift,
    "timestep_freq_shift_1": _mut_temb_shift,
    "resize_align_corners": _mut_resize_align_corners,
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_rejected(mutation):
    r, out = MUTATIONS[mutation]()
    inp, ref = _case(r)
    with pytest.raises(AssertionError, match="out of bound|differ in bits"):
        G.check_outputs(r, inp, out, mutation, ref)


def _old_metric_accepts(mutation):
    r, out = MUTATIONS[mutation]()
    inp, ref = _case(r)
    got = G.split_outputs(r, out)
    if r["kind"] == "dropout_scale_add":
        ref_y = torch.where(ref["_keep"], torch.zeros(r["n"], dtype=torch.float64), 0.0)
        ref_y[ref["_keep"]] = ref["y"][0]
        return G.old_metric(got["y"], ref_y) < 1e-2
    if r["kind"] == "embed_tokens_bwd":
        full = inp["dtok"].double().clone()
        full[ref["_used"]] = ref["dtok"][0]
        return G.old_metric(got["dtok"], full) < 1e-2 and G.old_metric(got["dpos"], ref["dpos"][0]) < 1e-2
    return all(G.old_metric(got[n], v[0]) < 1e-2 for n, v in ref.items() if not n.startswith("_") and n in got)


OLD_METRIC_ACCEPTS = {"velocity_abar_t_minus_1_loss", "add3_two_roundings", "gelu_bwd_tanh_form", "cast_truncates"}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_old_metric(mutation):
    """The mutations the per-kernel tests' max-ratio metric would let through (OLD_METRIC_ACCEPTS) and the ones it catches."""
    assert _old_metric_accepts(mutation) == (mutation in OLD_METRIC_ACCEPTS)
