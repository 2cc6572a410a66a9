"""The checks of tests/optim_check.py have teeth, shown without a GPU.  fp32 restatements of the optimizer, delta and compression
kernels stand in for the kernels on small census-shaped tables (the synthetic 8-bit launches of the census, and a table of more
rows than the 1,056-block grid with frozen gaps between them and rows past n_shadow): the checks must accept them with the eps
the GPU test uses, and reject outputs broken the way a defect of the kernels would break them.  OLD_METRIC_ACCEPTS pins which of
those the metrics of the per-kernel tests this census replaced (allclose at rtol 1e-5 / atol 1e-7 for fp32 outputs, codes off by
one on 0.01 % of elements, the merged weight at 2^-8 |r| + 1e-6 max |r|, the projected gradient at 2e-5 max |r|, and
max |y - r| / max |r| < 1e-2 for the compression) would let through."""
import json
import math
import sys

import pytest
import torch

import optim_check as C

# ---------------------------------------------------------------------------------------------- census
COUNTS = {"sqnorm_chunks": 9, "adamw_prepare": 2, "adamw_chunks": 6, "adamw8bit_chunks": 3, "adamw_ema_chunks": 2,
          "adamw8bit_ema_chunks": 4, "ema_swap_chunks": 3, "lora_delta_merge": 37, "lora_delta_grad": 37, "scale_cast_f32_bf16": 72}


def _golden():
    sys.path.insert(0, C.HERE + "/golden")
    import make_optim_launches as M
    return M


_RUN = []


def _workloads():
    """(records, tables) of the generator's workloads, run once."""
    if not _RUN:
        _RUN.append(_golden().run_workloads())
    return _RUN[0]


def test_census_matches_gpu_parametrization():
    recs = C.launches()
    assert {k: sum(r["kind"] == k for r in recs) for k in COUNTS} == COUNTS
    assert len(recs) == sum(COUNTS.values())
    assert set(COUNTS) == set(_golden().KINDS)
    assert len({C.launch_id(r) for r in recs}) == len(recs)
    import test_optim_step_gpu as GPU
    (mark,) = [m for m in GPU.test_step_optim.pytestmark if m.name == "parametrize"]
    assert mark.args[1] == recs


def test_census_reproduced_by_generator():
    """The workloads on the meta device make exactly the recorded launches, every recorded digest is that of a rebuilt table,
    and prims, the dropout epochs and the CPU random state are left as they were."""
    from t2v_b200 import prims
    before = {n: v for n, v in vars(prims).items() if callable(v)}
    rng = torch.get_rng_state()
    M = _golden()
    seen, tables = M.run_workloads()
    launches = seen + [r for r in M.synthetic()]
    assert json.loads(json.dumps(launches)) == C.launches()
    for r in C.launches():
        if "sha256" in r:
            assert M.digest(tables[r["sha256"]]) == r["sha256"]
    after = {n: v for n, v in vars(prims).items() if callable(v)}
    assert not sorted(n for n in before.keys() | after.keys() if before.get(n) is not after.get(n))
    assert torch.equal(torch.get_rng_state(), rng)


def test_census_covers_the_edges():
    recs = C.launches()
    _, tables = _workloads()
    upd = [r for r in recs if r["kind"] in _golden().UPDATE_KINDS]
    assert any(r["n_rows"] > _golden().GRID for r in upd), "no table with more rows than the grid"
    assert any(r["kind"] == "adamw_prepare" and r["n_sets"] == 2 for r in recs), "two hyper-parameter sets"
    # frozen elements around the rows: the arena keeps trainable tensors first, so a run's frozen elements follow its rows
    assert any(sum(tables[r["sha256"]][:, 1].tolist()) < r["total"] // 10 for r in upd if "sha256" in r), "frozen elements"
    for r in upd:
        if r.get("above_shadow"):
            t = C.table(r) if "rows" in r else tables[r["sha256"]]
            assert bool((t[:, 0] < r["n_shadow"]).any())
    assert any(r.get("above_shadow") for r in upd), "rows on both sides of n_shadow"
    assert {r["kind"] for r in upd if r.get("synthetic")} == {"adamw8bit_chunks", "adamw8bit_ema_chunks"}
    assert any(r["kind"] == "adamw8bit_chunks" and r["n_shadow"] < r["total"] for r in upd if r.get("synthetic"))
    assert any("ema" in r["kind"] and not r.get("synthetic") for r in upd), "EMA rows"
    assert all(r["rows8"] > 0 and r["rows32"] > 0 for r in upd if "8bit" in r["kind"] and "rows8" in r), "8-bit and fp32 rows"
    assert {r["g16"] for r in upd} == {0, 1} and {r["g16"] for r in recs if r["kind"] == "sqnorm_chunks"} == {0, 1}
    deltas = [r for r in recs if r["kind"] == "lora_delta_merge" and not r.get("synthetic")]
    assert {r["k"] for r in deltas} == {1, 3} and any(r["conv3d"] for r in deltas)
    assert {r["world"] for r in recs if r["kind"] == "scale_cast_f32_bf16"} == {2, 6, 8}
    assert max(r["n"] for r in recs if r["kind"] == "scale_cast_f32_bf16") == 1 << 26
    ragged = {n % 256 for n, bits in _golden().SYNTH_8BIT if bits == 8}
    assert {64, 128, 192} <= ragged


# ---------------------------------------------------------------------------------------------- fp32 restatements
def many_rows(kind, ema, g16):
    """1,100 rows of 64 elements with a frozen 64-element gap after each; the last 100 rows lie past n_shadow."""
    rows = [[128 * i, 64] + ([64 * i] if ema else []) for i in range(1100)]
    return {"kind": kind, "cols": 3 if ema else 2, "g16": g16, "hp": [1e-3, 0.9, 0.999, 1e-8, 1e-2], "n_rows": 1100,
            "total": 128 * 1100, "n_shadow": 128 * 1000, "n_state": 128 * 1100, "n_ema": 64 * 1100 if ema else 0, "rows": rows,
            **({"ema_decay": 0.9999} if ema else {})}


def _synth(kind):
    (r,) = [r for r in C.launches() if r["kind"] == kind and r.get("synthetic")]
    return r


def update_f32(r, tab, b, hp, k, mut=()):
    """The update kernels restated in fp32 (one rounding per operation) on the buffers of C.alloc_update; `mut` breaks it."""
    lr, b1, b2, eps, wd, bc1, sbc2, clip = hp.float().unbind()
    qmap = C.qmaps()
    mid_m, mid_v = 0.5 * (qmap[:255] + qmap[1:256]), 0.5 * (qmap[256:511] + qmap[257:512])
    zero_m = int((qmap[:256] == 0).nonzero()[0, 0])
    d = C.ema_d(k, r.get("ema_decay", 0.0))
    if "ema_decay_plus1" in mut and k > 1:
        d = min(float(torch.tensor(r["ema_decay"]).float()), (1 + k) / (10 + k))
    omd = torch.tensor(1.0 - d, dtype=torch.float64).float()
    eight, ema = "8bit" in r["kind"], "ema" in r["kind"]
    rows = tab[:1056] if "first_grid_rows_only" in mut else tab
    for row in rows.tolist():
        off, n = row[0], row[1]
        soff, bits = (row[2], row[3]) if eight else (off, 32)
        p = b["p"].t[off:off + n]
        g = b["g16"].t[off:off + n].float() if "g16" in b else b["g"].t[off:off + n].clone()
        if bits == 32:
            mb, vb = (b["m32"], b["v32"]) if eight else (b["m"], b["v"])
            m, v = mb.t[soff:soff + n].clone(), vb.t[soff:soff + n].clone()
        else:
            blk = torch.arange(n) // C.QBLOCK + soff // C.QBLOCK
            m = qmap[:256][b["qm"].t[soff:soff + n].long()] * b["am"].t[blk]
            v = qmap[256:][b["qv"].t[soff:soff + n].long()] * b["av"].t[blk]
            m_old, v_old = m.clone(), v.clone()
        gc = g * clip
        m1 = b1 * m + (1 - b1) * gc
        v1 = b2 * v + (1 - b2) * gc * gc
        den = (v1.sqrt() + eps) / sbc2 if "eps_before_bc2" in mut else v1.sqrt() / sbc2 + eps
        upd = (lr / bc1) * (m1 / den)
        p1 = (p - upd) * (1 - lr * wd) if "decay_after_step" in mut else p * (1 - lr * wd) - upd
        p.copy_(p1)
        if bits == 32:
            mb.t[soff:soff + n], vb.t[soff:soff + n] = m1, v1
        else:
            for x, x_old, qb, ab, md, zc in ((m1, m_old, "qm", "am", mid_m, zero_m), (v1, v_old, "qv", "av", mid_v, 0)):
                for j in range(0, n, C.QBLOCK):
                    xs = x[j:j + C.QBLOCK]
                    src = x_old[j:j + C.QBLOCK] if "absmax_old_moments" in mut else xs
                    am = src.abs().max()
                    b[ab].t[(soff + j) // C.QBLOCK] = am
                    code = torch.searchsorted(md, (xs / am).contiguous(), side="left").clamp(max=255) if am > 0 else torch.full_like(xs, zc, dtype=torch.long)
                    b[qb].t[soff + j:soff + j + xs.numel()] = code.to(torch.uint8)
        if off < r["n_shadow"]:
            b["shadow"].t[off:off + n] = p1.bfloat16()
        b["g"].t[off:off + n] = 0.0
        if ema:
            e = b["ema"].t[row[-1]:row[-1] + n]
            e.copy_(e - omd * (e - p1))


def _update_case(r, k, moments, mut=()):
    tab = C.table(r)
    b, P = C.alloc_update(r, tab, k, moments, "cpu")
    hp = C.hp_row(r["hp"], k - 1 if "bias_k_minus_1" in mut else k, C.CLIP if moments else 1.0)
    update_f32(r, tab, b, hp, k, mut)
    return r, tab, k, moments, b, P


UPDATE_CASES = {
    "adamw_many_rows": lambda: many_rows("adamw_chunks", False, 0),
    "adamw_ema_many_rows_g16": lambda: many_rows("adamw_ema_chunks", True, 1),
    "adamw8bit_synthetic": lambda: _synth("adamw8bit_chunks"),
    "adamw8bit_ema_synthetic_g16": lambda: _synth("adamw8bit_ema_chunks"),
}


@pytest.mark.parametrize("case", list(UPDATE_CASES))
@pytest.mark.parametrize("k,moments", C.STATES)
def test_restated_update_passes(case, k, moments):
    r, tab, k, moments, b, P = _update_case(UPDATE_CASES[case](), k, moments)
    C.check_update(r, tab, k, moments, b, P, case, "cpu")


def test_restated_swap_sqnorm_prepare_delta_cast_pass():
    from oracle import ops_ref as O
    r8 = _synth("adamw8bit_ema_chunks")
    rows = [[a[0], a[1], a[4]] for a in r8["rows"]]
    rs = {"kind": "ema_swap_chunks", "rows": rows, "total": r8["total"], "n_shadow": r8["n_shadow"], "n_ema": r8["n_ema"]}
    tab = C.table(rs)
    b, P = C.alloc_swap(rs, tab, "cpu")
    for swapped in (True, False):
        for a in rows:
            p, e = b["p"].t[a[0]:a[0] + a[1]], b["ema"].t[a[2]:a[2] + a[1]]
            tmp = p.clone()
            p.copy_(e)
            e.copy_(tmp)
            if a[0] < rs["n_shadow"]:
                b["shadow"].t[a[0]:a[0] + a[1]] = p.bfloat16()
        for buf in b.values():
            buf.covered.zero_()
        C.check_swap(rs, tab, b, P, "swap", "cpu", swapped)
    for g16 in (0, 1):
        rq = {"kind": "sqnorm_chunks", "rows": [a[:2] for a in r8["rows"]], "total": r8["total"], "g16": g16}
        tq = C.table(rq)
        buf, out, P = C.alloc_sqnorm(rq, tq, "cpu")
        for a in rq["rows"]:
            x = buf.t[a[0]:a[0] + a[1]].float()
            out[0] += float((x.double() ** 2).sum())
        C.check_sqnorm(rq, tq, buf, out, P, "sqnorm", "cpu")
    for n_sets in (1, 2):
        for k in (1, 2, 3, 10, 10 ** 4, 10 ** 6):
            for max_norm in (0.0, 1e6, 1.0):
                hp_in, hp, state, sq = _prepare_in(n_sets, k - 1)
                O.adamw_prepare(hp_in, hp, state, sq, max_norm)
                C.check_prepare(hp_in, hp, k - 1, state[0], torch.tensor(3.25), sq, max_norm, f"prepare k{k}")
    for r in _small_deltas():
        inp = C.delta_inputs(r, "cpu")
        C.check_delta(r, inp, _delta_f32(r, inp), C.launch_id(r))
    for world in (2, 6, 8):
        rc = {"kind": "scale_cast_f32_bf16", "n": 3 * C.PATTERN + 5, "world": world}
        x = C.cast_inputs(rc["n"], "cpu")
        y = (x.repeat(4)[:rc["n"]] * torch.tensor(1.0 / world, dtype=torch.float32)).bfloat16()
        C.check_cast(rc, x, y, "cast")


def _prepare_in(n_sets, k_before):
    hp_in = torch.tensor([[5e-6, 0.9, 0.999, 1e-8, 1e-2], [1e-5, 0.8, 0.99, 1e-6, 1e-4]][:n_sets], dtype=torch.float32)
    return hp_in, torch.zeros(n_sets, 8), torch.tensor([k_before], dtype=torch.int64), torch.tensor([3.25, -7.0], dtype=torch.float64)


def _small_deltas():
    """The smallest recorded and synthetic delta launches: Conv2d k = 1 and k = 3 and Conv3d, both kernels."""
    recs = [r for r in C.launches() if r["kind"].startswith("lora_delta")]
    out = []
    for kind in ("lora_delta_merge", "lora_delta_grad"):
        for sel in (lambda r: not r["conv3d"] and r["k"] == 1, lambda r: not r["conv3d"] and r["k"] == 3, lambda r: r["conv3d"]):
            out.append(min((r for r in recs if r["kind"] == kind and sel(r)), key=lambda r: r["Cout"] * r["Cin"] * r["r"]))
    return out


def _delta_f32(r, inp, no_third=False):
    import stable_lora_ref as R
    conv3d = bool(r["conv3d"])
    if r["kind"] == "lora_delta_merge":
        if no_third:
            co, ci = r["Cout"], r["Cin"]
            d = (inp["B"] @ inp["A"]).view(co, ci, 3, 3, 1).sum(-2) * r["scaling"]
            return {"merged": (inp["base"] + d.permute(0, 2, 3, 1)).bfloat16()}
        return {"merged": R.lora_delta_merge(inp["base"], inp["A"], inp["B"], r["scaling"], conv3d)}
    dA, dB = inp["dA"].clone(), inp["dB"].clone()
    R.lora_delta_grad(inp["dw"], inp["A"], inp["B"], r["scaling"], conv3d, dA, dB)
    return {"dA": dA, "dB": dB}


# ---------------------------------------------------------------------------------------------- broken outputs are rejected
UPDATE_MUTATIONS = {   # name: (case, k, moments)
    "first_grid_rows_only": ("adamw_many_rows", 1000, True),
    "decay_after_step": ("adamw_many_rows", 1000, True),
    "eps_before_bc2": ("adamw_many_rows", 1000, True),
    "bias_k_minus_1": ("adamw_many_rows", 1000, True),
    "absmax_old_moments": ("adamw8bit_synthetic", 1000, True),
    "ema_decay_plus1": ("adamw_ema_many_rows_g16", 1000, True),
}


def _mutated_update(name):
    case, k, moments = UPDATE_MUTATIONS[name]
    r = UPDATE_CASES[case]()
    return _update_case(r, k, moments, mut=(name,))


def _clip_mutant(name):
    """adamw_prepare's clip factor without the + 1e-6 (active clipping) or without the clamp to 1 (inactive)."""
    hp_in, hp, state, sq = _prepare_in(1, 9)
    max_norm = 1.0 if name == "clip_without_1e-6" else 1e6
    from oracle import ops_ref as O
    O.adamw_prepare(hp_in, hp, state, sq, max_norm)
    norm = math.sqrt(3.25)
    hp[0, 7] = float(torch.tensor(max_norm / norm if name == "clip_without_1e-6" else max_norm / (norm + 1e-6)).float())
    return hp_in, hp, state, sq, max_norm


def _conv3d_merge():
    (r,) = [x for x in _small_deltas() if x["kind"] == "lora_delta_merge" and x["conv3d"]]
    return r


MUTATIONS = list(UPDATE_MUTATIONS) + ["clip_without_1e-6", "clip_without_clamp", "conv3d_delta_without_third", "cast_truncates"]


def _run_mutation(name):
    """Runs the new check on the broken output; returns the old metric's verdict (True: it would accept the output)."""
    if name in UPDATE_MUTATIONS:
        r, tab, k, moments, b, P = _mutated_update(name)
        old = _old_update(r, tab, k, moments, b, P)
        with pytest.raises(AssertionError, match="out of bound|differ in bits|codes off"):
            C.check_update(r, tab, k, moments, b, P, name, "cpu")
        return old
    if name.startswith("clip"):
        hp_in, hp, state, sq, max_norm = _clip_mutant(name)
        with pytest.raises(AssertionError, match="within 1 ulp"):
            C.check_prepare(hp_in, hp, 9, state[0], torch.tensor(3.25), sq, max_norm, name)
        return _old_clip(hp)
    if name == "conv3d_delta_without_third":
        r = _conv3d_merge()
        inp = C.delta_inputs(r, "cpu")
        out = _delta_f32(r, inp, no_third=True)
        with pytest.raises(AssertionError, match="out of bound"):
            C.check_delta(r, inp, out, name)
        ref = C.delta_ref(r, inp)["merged"][0]
        err = (out["merged"].double() - ref).abs()
        return bool((err <= ref.abs() * 2.0 ** -8 + 1e-6 * ref.abs().max()).all())
    if name == "cast_truncates":
        rc = {"kind": "scale_cast_f32_bf16", "n": C.PATTERN, "world": 8}
        x = C.cast_inputs(rc["n"], "cpu")
        y = ((x * 0.125).view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()
        with pytest.raises(AssertionError, match="differ in bits"):
            C.check_cast(rc, x, y, name)
        r = x.double() / 8
        return float((y.double() - r).abs().max() / r.abs().max()) < 1e-2
    raise KeyError(name)


def _old_update(r, tab, k, moments, b, P):
    """The replaced tests' verdict: fp32 outputs allclose(rtol 1e-5, atol 1e-7) to the reference, codes within one of it on
    all but 0.01 % of elements, and the EMA bit for bit against EMAModel.step on the kernel's own p."""
    clean = _update_case(r, k, moments)[4]
    for n in b:
        y, ref = b[n].t, clean[n].t
        if y.dtype == torch.uint8:
            d = (y.long() - ref.long()).abs()
            if int(d.max()) > 1 or float((d == 0).double().mean()) < 0.9999:
                return False
        elif n in ("shadow", "g", "g16"):
            if not torch.equal(y.view(torch.int16 if y.dtype == torch.bfloat16 else torch.int32),
                               ref.view(torch.int16 if ref.dtype == torch.bfloat16 else torch.int32)):
                return False
        elif n == "ema":
            ok = True
            for row in tab.tolist():
                e0 = C.pat(P["ema"], torch.arange(row[-1], row[-1] + row[1]))
                want = C.ema_fp32(e0, b["p"].t[row[0]:row[0] + row[1]], k, r["ema_decay"])
                ok = ok and torch.equal(y[row[-1]:row[-1] + row[1]].view(torch.int32), want.view(torch.int32))
            if not ok:
                return False
        else:
            fin = ~(torch.isnan(ref))
            if not torch.allclose(y[fin], ref[fin], rtol=1e-5, atol=1e-7):
                return False
    return True


def _old_clip(hp):
    """The old end-to-end tests compared FusedAdamW's weights with torch at rtol 1e-5 / atol 1e-7: the clip factor scales the
    gradient of one update of lr 1e-3 on weights of magnitude 1."""
    good = 1.0 / (math.sqrt(3.25) + 1e-6)
    return abs(float(hp[0, 7]) - good) * 1e-3 <= 1e-7 + 1e-5


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_rejected(mutation):
    _run_mutation(mutation)


OLD_METRIC_ACCEPTS = {"clip_without_1e-6", "cast_truncates"}


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_old_metric(mutation):
    """The mutations the replaced tests' metrics would let through (OLD_METRIC_ACCEPTS) and the ones they catch."""
    assert _run_mutation(mutation) == (mutation in OLD_METRIC_ACCEPTS)
