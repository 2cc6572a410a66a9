"""The checks of tests/attn_check.py have teeth, shown without a GPU.  An fp32 restatement of each attention kernel family (P and
dS rounded to bf16 where the kernels round them, the online softmax of flash_attn.cu / attn_long over 64-key tiles) stands in for
the kernels on census launches small enough for the CPU.  It is written here rather than taken from oracle/ops_ref.py, whose
attention functions are not what is checked: they compute one untiled fp32 softmax without the kernels' bf16 roundings, and
the mutations below need the tile structure (a skipped rescale, a dropped ragged tile, padded keys).  The census generator
does run the model code over oracle/ops_ref.py, on the meta device, to record the launches; the checks must accept it with the eps the GPU test uses, and reject
outputs broken the way a defect of the kernels would break them.  On these inputs the old max|y - r| / max|r| metric (< 1e-2,
1.5e-2 for gradients) also catches every mutation on at least one of its outputs (OLD_METRIC_ACCEPTS is empty), but not on each:
it accepts the lse of padded keys scored 0 (0.8 %), which the element bound rejects; and the restated kernels' own error (up
to 2.8e-3 m, P rounded to bf16) sits a factor of 4 under the fitted eps, where a 1e-2-of-max tolerance has no resolution."""
import json
import math
import sys

import pytest
import torch

import attn_check as A

LOG2E = 1.4426950408889634

# census launches the CPU checks in seconds
CASES = {
    "flash_fwd_ragged": dict(kind="flash_attn_fwd", Nb=1, Lq=256, Lk=77, heads=20, D=64, q_ld=1280, k_ld=2560, v_ld=2560, fused="kv",
                             o_ld=1280),
    "flash_fwd_45": dict(kind="flash_attn_fwd", Nb=16, Lq=45, Lk=45, heads=20, D=64, q_ld=1280, k_ld=1280, v_ld=1280, fused="none",
                         o_ld=1280),
    "flash_bwd_split": dict(kind="flash_attn_bwd", Nb=1, Lq=720, Lk=77, heads=20, D=64, q_ld=1280, k_ld=1280, v_ld=1280, fused="none",
                            o_ld=1280, do_ld=1280, dq_ld=1280, dk_ld=1280, dv_ld=1280, splits_132=3, splits_114=3),
    "flash_bwd_qkv": dict(kind="flash_attn_bwd", Nb=16, Lq=16, Lk=16, heads=20, D=64, q_ld=3840, k_ld=3840, v_ld=3840, fused="qkv",
                          o_ld=1280, do_ld=1280, dq_ld=3840, dk_ld=3840, dv_ld=3840, splits_132=1, splits_114=1),
    "small_fwd": dict(kind="attn_small_fwd", addr=[16, 16, 256, 1, 16, 3840, 1280, 20, 16, 64], rows=256, fused="qkv"),
    "small_fwd_2clips": dict(kind="attn_small_fwd", addr=[32, 16, 256, 1, 16, 3840, 1280, 20, 16, 64], rows=512, fused="qkv"),
    "small_bwd": dict(kind="attn_small_bwd", addr=[16, 16, 256, 1, 16, 3840, 1280, 20, 16, 64], rows=256, fused="qkv"),
    "long_fwd": dict(kind="attn_long_fwd", addr=[16, 16, 768, 1, 16, 3840, 1280, 20, 48, 64], rows=768, fused="qkv"),
    "long_bwd": dict(kind="attn_long_bwd", addr=[16, 16, 768, 1, 16, 3840, 1280, 20, 48, 64], rows=768, fused="qkv"),
    "clip_causal": dict(kind="composite", Nb=1, Lq=77, Lk=77, heads=16, D=64, q_ld=1024, k_ld=1024, v_ld=1024, fused="none", causal=77,
                        bwd=1, do_ld=1024, dq_ld=1024, dk_ld=1024, dv_ld=1024),
}


def _bf(t):
    return t.bfloat16().float()


# ---------------------------------------------------------------------------------------------- fp32 restatements
def online_fwd(inp, causal=False, skip_alpha_l=False, skip_alpha_o=False, pad_zero=False, drop_tail=False):
    """flash_attn.cu / attn_long forward: 64-key tiles, base-2 online softmax, l from the fp32 p, O += bf16(p) V; returns
    (o bf16, lse fp32 natural log).  Broken variants: the rescale alpha not applied to l or to O, padded keys scored 0 instead
    of -inf, the ragged last tile skipped."""
    Q, K, V = (inp[n].float() for n in ("Q", "K", "V"))
    Z, Lq, D = Q.shape
    Lk = K.shape[1]
    sc2 = D ** -0.5 * LOG2E
    m = torch.full((Z, Lq, 1), -math.inf)
    l = torch.zeros(Z, Lq, 1)
    o = torch.zeros(Z, Lq, D)
    ntiles = -(-Lk // A.TILE)
    for j in range(ntiles):
        if drop_tail and j == ntiles - 1 and Lk % A.TILE:
            break
        k0, k1 = j * A.TILE, min(Lk, (j + 1) * A.TILE)
        s = (Q @ K[:, k0:k1].transpose(1, 2)) * sc2
        v = V[:, k0:k1]
        if causal:
            s = s.masked_fill(torch.arange(k0, k1)[None, None, :] > torch.arange(Lq)[None, :, None], -math.inf)
        if pad_zero and k1 - k0 < A.TILE:
            s = torch.cat([s, torch.zeros(Z, Lq, A.TILE - (k1 - k0))], -1)
            v = torch.cat([v, torch.zeros(Z, A.TILE - (k1 - k0), D)], 1)
        mx = torch.maximum(m, s.max(-1, keepdim=True).values)
        alpha = torch.exp2(m - mx)
        p = torch.exp2(s - mx)
        l = (l if skip_alpha_l else l * alpha) + p.sum(-1, keepdim=True)
        o = (o if skip_alpha_o else o * alpha) + _bf(p) @ v
        m = mx
    return (o / l).bfloat16(), ((m + torch.log2(l)) / LOG2E).squeeze(-1)


def softmax_fwd(inp, causal=False, causal_shift=0):
    """attn_small / the composite: normalised P rounded to bf16 before P V.  `causal_shift` = 1 lets row i see key i + 1."""
    Q, K, V = (inp[n].float() for n in ("Q", "K", "V"))
    Z, Lq, D = Q.shape
    s = (Q @ K.transpose(1, 2)) * D ** -0.5
    if causal:
        s = s.masked_fill(torch.arange(K.shape[1])[None, None, :] > torch.arange(Lq)[None, :, None] + causal_shift, -math.inf)
    P = _bf(torch.softmax(s, -1))
    return (P @ V).bfloat16(), P


def lse_bwd(inp, o, lse, no_scale=False, delta_row_shift=0, drop_rows=None):
    """flash_attn.cu / attn_long backward from the forward's o and lse: P = exp(s - lse), delta = rowsum(dO o) from the bf16 o,
    dS = P (dP - delta) scale, dv = bf16(P)^T dO, dq = bf16(dS) K, dk = bf16(dS)^T Q.  Broken variants: dS without the scale,
    delta of a neighbouring row, the dk / dv partial of query rows `drop_rows` dropped."""
    Q, K, V, dO = (inp[n].float() for n in ("Q", "K", "V", "dO"))
    D = Q.shape[2]
    scale = D ** -0.5
    P = torch.exp((Q @ K.transpose(1, 2)) * scale - lse[..., None])
    delta = (dO * o.float()).sum(-1, keepdim=True)
    if delta_row_shift:
        delta = delta.roll(delta_row_shift, 1)
    dS = P * (dO @ V.transpose(1, 2) - delta) * (1.0 if no_scale else scale)
    Pk, dSk, dOk, Qk = _bf(P), _bf(dS), dO, Q
    if drop_rows is not None:
        keep = torch.ones(Q.shape[1], 1)
        keep[drop_rows] = 0
        Pk, dSk = Pk * keep, dSk * keep
    return {"dq": (_bf(dS) @ K).bfloat16(), "dk": (dSk.transpose(1, 2) @ Qk).bfloat16(), "dv": (Pk.transpose(1, 2) @ dOk).bfloat16()}


def prob_bwd(inp, P, composite):
    """attn_small (fp32 P, delta = rowsum(P dP)) and the composite (the stored bf16 P): dS rounded to bf16 before its GEMMs."""
    Q, K, V, dO = (inp[n].float() for n in ("Q", "K", "V", "dO"))
    scale = Q.shape[2] ** -0.5
    dP = dO @ V.transpose(1, 2)
    dS = _bf(P * (dP - (P * dP).sum(-1, keepdim=True)) * scale)
    return {"dq": (dS @ K).bfloat16(), "dk": (dS.transpose(1, 2) @ Q).bfloat16(), "dv": (_bf(P).transpose(1, 2) @ dO).bfloat16()}


_CACHE = {}


def _launch(name):
    want = CASES[name]
    assert want in A.launches(), f"{name} is not a launch of tests/golden/attn_launches.json"
    return want


def _case(name):
    """(launch, canonical inputs, restated kernel outputs, float64 reference), computed once."""
    if name not in _CACHE:
        r = _launch(name)
        inp = A.make_inputs(r)
        fam, causal = A.family(r), A.geometry(r)[5]
        if fam in ("flash", "long"):
            o, lse = online_fwd(inp)
            out = {"o": o, "lse": lse}
            if A.has_bwd(r):
                out = lse_bwd(inp, o, lse)
        else:
            o, P = softmax_fwd(inp, causal)
            out = {"o": o}
            if A.has_bwd(r):
                out = dict(prob_bwd(inp, P if fam == "composite" else torch.softmax(_scores(inp, causal), -1), fam == "composite"),
                           **({"o": o} if fam == "composite" else {}))
        _CACHE[name] = (r, inp, out, A.reference(inp, causal, A.has_bwd(r)))
    return _CACHE[name]


def _scores(inp, causal):
    Q, K = inp["Q"].float(), inp["K"].float()
    s = (Q @ K.transpose(1, 2)) * Q.shape[2] ** -0.5
    if causal:
        s = s.masked_fill(torch.arange(K.shape[1])[None, None, :] > torch.arange(Q.shape[1])[None, :, None], -math.inf)
    return s


def _check(name, out):
    r, inp, _, ref = _case(name)
    return A.check_outputs(r, inp, out, name, ref)


# ---------------------------------------------------------------------------------------------- census
COUNTS = {"flash_attn_fwd": 55, "flash_attn_bwd": 55, "attn_small_fwd": 20, "attn_small_bwd": 20, "attn_long_fwd": 11,
          "attn_long_bwd": 11, "composite": 2}


def _golden():
    sys.path.insert(0, A.HERE + "/golden")
    import make_attn_launches as M
    return M


def test_census_matches_gpu_parametrization():
    recs = A.launches()
    assert {k: sum(r["kind"] == k for r in recs) for k in COUNTS} == COUNTS
    assert len(recs) == sum(COUNTS.values())
    assert len({A.launch_id(r) for r in recs}) == len(recs)
    import test_attn_step_gpu as G
    (mark,) = [m for m in G.test_step_attention.pytestmark if m.name == "parametrize"]
    assert mark.args[1] == recs


def test_census_covers_the_edges():
    """A split flash backward on both SM counts, attn_long at its L = 256 limit, a causal composite, the VAE's d = 512
    composite, the ragged 320x576 lengths (self-attention at 2880, 720, 180 and 45 tokens, cross-attention of 16 x 45 = 720
    queries on 77 keys), and temporal sequences of a second clip (nseq > inner: the outer_rows term of SeqAddr)."""
    recs = A.launches()
    for kind in ("attn_small_fwd", "attn_small_bwd"):
        assert any(r["kind"] == kind and r["addr"][0] > r["addr"][1] for r in recs), kind
    assert any(r["kind"] == "flash_attn_bwd" and r["splits_132"] > 1 and r["splits_114"] > 1 for r in recs)
    assert any(r["kind"] == "flash_attn_bwd" and r["Nb"] == 4 and r["Lq"] == 4096 and r["Lk"] == 77 and r["splits_132"] > 1 for r in recs)
    assert any(r["kind"].startswith("attn_long") and r["addr"][8] == 256 for r in recs)
    assert any(r["kind"] == "composite" and r["causal"] == 77 and r["bwd"] for r in recs)
    assert any(r["kind"] == "composite" and r["D"] == 512 and not r["bwd"] for r in recs)
    for Lq, Lk in ((45, 45), (180, 180), (720, 720), (2880, 2880), (720, 77)):
        assert any(r["kind"] == "flash_attn_fwd" and r.get("Lq") == Lq and r.get("Lk") == Lk for r in recs), (Lq, Lk)


def _module_functions(mod):
    return {n: v for n, v in vars(mod).items() if callable(v)}


def test_census_reproduced_by_generator():
    """The workloads on the meta device over the oracle (GEMMs and attention prims replaced by allocators) make exactly the
    recorded launches, and leave every prims / ops function, the dropout epochs and the CPU random state as they found them:
    later tests in the same process run the real kernels on unchanged state."""
    from t2v_b200 import ops, prims
    before = {m.__name__: _module_functions(m) for m in (prims, ops)}
    flash, epochs, rng = ops._Flash.enabled, dict(ops._epochs), torch.get_rng_state()
    assert json.loads(json.dumps(_golden().step_launches())) == A.launches()
    for m in (prims, ops):
        after = _module_functions(m)
        changed = sorted(n for n in before[m.__name__].keys() | after.keys() if before[m.__name__].get(n) is not after.get(n))
        assert not changed, f"the census left {m.__name__}.{changed} replaced"
    assert ops._Flash.enabled == flash
    assert ops._epochs.keys() == epochs.keys() and all(ops._epochs[k] is t for k, t in epochs.items())
    assert torch.equal(torch.get_rng_state(), rng), "the census moved the CPU random state"


@pytest.mark.parametrize("args,want", [
    ((1, 5, 16384, 77), (27, 23)),     # cfg-2 cross-attention: 10 CTAs, 256 query blocks
    ((4, 5, 4096, 77), (7, 6)),        # 512^2 image batch: 40 CTAs
    ((4, 10, 1024, 77), (4, 3)),
    ((1, 20, 720, 77), (3, 3)),        # 320x576, 12 query blocks: capped at nqb / 4
    ((1, 20, 256, 77), (1, 1)),        # 4 query blocks: < 8, no split
    ((16, 5, 1024, 1024), (1, 1)),     # 1280 CTAs >= SM count
    ((2, 2, 512, 64), (2, 2)),         # 4 CTAs would take 66 / 57 splits; 8 query blocks cap them at 2
])
def test_splits_restatement_pinned(args, want):
    M = _golden()
    assert tuple(M.splits(*args, sms) for sms in (132, 114)) == want


# ---------------------------------------------------------------------------------------------- the restatements pass
@pytest.mark.parametrize("name", list(CASES))
def test_restated_kernels_pass(name):
    _check(name, _case(name)[2])


# ---------------------------------------------------------------------------------------------- broken outputs are rejected
def _fwd_variant(**kw):
    _, inp, _, _ = _case("flash_fwd_ragged")
    o, lse = online_fwd(inp, **kw)
    return {"o": o, "lse": lse}


def _lse_log2():
    return dict(_case("flash_fwd_ragged")[2], lse=_case("flash_fwd_ragged")[2]["lse"] * LOG2E)


def _bwd_variant(**kw):
    _, inp, _, _ = _case("flash_bwd_split")
    o, lse = online_fwd(inp)
    return lse_bwd(inp, o, lse, **kw)


def _split_dropped():
    """The second of the 3 query splits (blocks 4..7, rows 256..511) never reaches dk / dv."""
    r = _launch("flash_bwd_split")
    per = -(-(-(-r["Lq"] // 64)) // r["splits_132"]) * 64
    return _bwd_variant(drop_rows=slice(per, 2 * per))


def _head_shifted():
    """dk written into the fused [.., 3C] gradient one head (64 columns) to the right."""
    r, inp, out, _ = _case("flash_bwd_qkv")
    Z, Lq, Lk, D, heads, _ = A.geometry(r)
    C = heads * D
    g = torch.zeros(r["Nb"], Lq, 3 * C, dtype=torch.bfloat16)
    A.scatter(r, out["dq"], g[..., :C], heads, D)
    A.scatter(r, out["dv"], g[..., 2 * C:], heads, D)
    A.scatter(r, out["dk"], g[..., C + D:2 * C + D], heads, D)
    return {n: A.gather(r, g[..., i * C:(i + 1) * C], heads, D) for i, n in enumerate(("dq", "dk", "dv"))}


def _causal_off_by_one():
    _, inp, _, _ = _case("clip_causal")
    o, P = softmax_fwd(inp, True, causal_shift=1)
    return dict(prob_bwd(inp, P, True), o=o)


def _wrong_stride(name, field):
    """A temporal sequence walked with SeqAddr field `field` (4: the frame stride seq_rows, 2: the clip stride outer_rows) one
    token row short: the kernel reads and writes the wrong token rows."""
    r, inp, _, _ = _case(name)
    Z, Lq, Lk, D, heads, _ = A.geometry(r)
    bad = list(r["addr"])
    bad[field] -= 1
    lay = A.layout(r, "cpu", fill=0.0)
    for n, c in (("q", "Q"), ("k", "K"), ("v", "V")):
        A.scatter(r, inp[c], lay[n], heads, D)
    wrong = {c: A.gather(r, lay[n], heads, D, addr=bad) for n, c in (("q", "Q"), ("k", "K"), ("v", "V"))}
    o = torch.zeros(r["rows"], heads * D, dtype=torch.bfloat16)
    A.scatter(r, softmax_fwd(wrong)[0], o, heads, D, addr=bad)
    return {"o": A.gather(r, o, heads, D)}


MUTATIONS = {
    "ragged_tile_dropped": ("flash_fwd_ragged", lambda: _fwd_variant(drop_tail=True)),
    "padded_keys_score_0": ("flash_fwd_ragged", lambda: _fwd_variant(pad_zero=True)),
    "alpha_of_l_skipped": ("flash_fwd_ragged", lambda: _fwd_variant(skip_alpha_l=True)),
    "alpha_of_o_skipped": ("flash_fwd_ragged", lambda: _fwd_variant(skip_alpha_o=True)),
    "lse_in_log2_units": ("flash_fwd_ragged", _lse_log2),
    "ds_not_scaled": ("flash_bwd_split", lambda: _bwd_variant(no_scale=True)),
    "delta_of_wrong_row": ("flash_bwd_split", lambda: _bwd_variant(delta_row_shift=1)),
    "query_split_partial_dropped": ("flash_bwd_split", _split_dropped),
    "fused_gradient_one_head_right": ("flash_bwd_qkv", _head_shifted),
    "causal_mask_off_by_one": ("clip_causal", _causal_off_by_one),
    "temporal_wrong_frame_stride": ("small_fwd", lambda: _wrong_stride("small_fwd", 4)),
    "temporal_wrong_clip_stride": ("small_fwd_2clips", lambda: _wrong_stride("small_fwd_2clips", 2)),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_rejected(mutation):
    name, make = MUTATIONS[mutation]
    with pytest.raises(AssertionError, match="out of bound"):
        _check(name, make())


def _old_metric_accepts(mutation):
    """Whether every broken output of `mutation` stays below the old metric's tolerance."""
    name, make = MUTATIONS[mutation]
    _, _, _, ref = _case(name)
    return all(A.old_metric(y, ref[n][0]) < (1e-2 if n in ("o", "lse") else 1.5e-2) for n, y in make().items())


OLD_METRIC_ACCEPTS = set()


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_old_metric(mutation):
    """The mutations the per-kernel tests' max-ratio metric would let through (OLD_METRIC_ACCEPTS) and the ones it catches."""
    assert _old_metric_accepts(mutation) == (mutation in OLD_METRIC_ACCEPTS)
