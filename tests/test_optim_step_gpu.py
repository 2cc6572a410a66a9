"""Every launch of tests/golden/optim_launches.json (the optimizer, EMA, stable-LoRA delta and gradient-compression kernels of the
training steps, and the synthetic launches) run through the prims entry points at full size on the real chunk table, and checked
element by element against a float64 reference (tests/optim_check.py).  The table of a recorded launch is rebuilt on the CPU by
tests/golden/make_optim_launches.py and must match the recorded sha256.

Every buffer is SENTINEL-filled with guard elements on both sides; only the elements of the rows get inputs, and every other
element (frozen gaps, the shadow past n_shadow, the 8-bit block padding, the guards) must come back bit for bit.  Each update
launch runs twice: k = 1 from the zero state and k = 1000 from random moments with clipping.  sqnorm_chunks accumulates into a
nonzero preset; ema_swap_chunks is checked after one swap and after the swap back; test_prepare_sweep runs adamw_prepare over
k in {1, 2, 3, 10, 10^4, 10^6} with max_norm 0, inactive and active, for one and two hyper-parameter sets.  The float64
reference runs on the device in slabs of at most 2^25 elements, and every buffer is freed between launches.  Each check prints
one OPTIMCHECK line: the largest ratio |y - r| / m (bf16 outputs: (|y - r| - 2^-8 |r|) / m) and the relative L2 error."""
import gc

import pytest
import torch

import optim_check as C

pytestmark = pytest.mark.gpu

LAUNCHES = C.launches()
DEV = "cuda"


def _report(lid, res):
    for name, (ratio, l2) in res.items():
        print(f"OPTIMCHECK {lid} {name} ratio={ratio:.3e} l2={l2:.3e}")


@pytest.fixture(autouse=True)
def _free():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _update(r, tab, k, moments):
    from t2v_b200 import prims
    b, P = C.alloc_update(r, tab, k, moments, DEV)
    hp = C.hp_row(r["hp"], k, C.CLIP if moments else 1.0).to(DEV)
    step = torch.tensor([k], dtype=torch.int64, device=DEV)
    t = tab.to(DEV).contiguous()
    g16 = b["g16"].t if "g16" in b else None
    kind = r["kind"]
    if kind == "adamw_chunks":
        prims.adamw_chunks(b["p"].t, b["g"].t, b["m"].t, b["v"].t, b["shadow"].t, r["n_shadow"], t, hp, True, g16)
    elif kind == "adamw_ema_chunks":
        prims.adamw_ema_chunks(b["p"].t, b["g"].t, b["m"].t, b["v"].t, b["shadow"].t, r["n_shadow"], t, hp, b["ema"].t, step,
                               r["ema_decay"], True, g16)
    else:
        q = C.qmaps().to(DEV)
        args = (b["p"].t, b["g"].t, b["shadow"].t, r["n_shadow"], t, hp, q, b["m32"].t, b["v32"].t, b["qm"].t, b["qv"].t, b["am"].t,
                b["av"].t)
        if kind == "adamw8bit_chunks":
            prims.adamw8bit_chunks(*args, True, g16)
        else:
            prims.adamw8bit_ema_chunks(*args, b["ema"].t, step, r["ema_decay"], True, g16)
    torch.cuda.synchronize()
    lid = f"{C.launch_id(r)} k{k}"
    _report(lid, C.check_update(r, tab, k, moments, b, P, lid, DEV))


def _tab(r):
    return C.table(r)


@pytest.mark.parametrize("r", LAUNCHES, ids=[C.launch_id(r) for r in LAUNCHES])
def test_step_optim(r):
    from t2v_b200 import prims
    kind = r["kind"]
    lid = C.launch_id(r)
    if kind in ("adamw_chunks", "adamw_ema_chunks", "adamw8bit_chunks", "adamw8bit_ema_chunks"):
        tab = _tab(r)
        for k, moments in C.STATES:
            _update(r, tab, k, moments)
            gc.collect()
            torch.cuda.empty_cache()
    elif kind == "sqnorm_chunks":
        tab = _tab(r)
        buf, out, P = C.alloc_sqnorm(r, tab, DEV)
        t = tab.to(DEV).contiguous()
        if r["g16"]:
            g = torch.zeros(8, device=DEV)
            prims.sqnorm_chunks(g, t, out, buf.t)
        else:
            prims.sqnorm_chunks(buf.t, t, out)
        torch.cuda.synchronize()
        _report(lid, C.check_sqnorm(r, tab, buf, out, P, lid, DEV))
    elif kind == "ema_swap_chunks":
        tab = _tab(r)
        b, P = C.alloc_swap(r, tab, DEV)
        t = tab.to(DEV).contiguous()
        prims.ema_swap_chunks(b["p"].t, b["ema"].t, b["shadow"].t, r["n_shadow"], t)
        torch.cuda.synchronize()
        C.check_swap(r, tab, b, P, f"{lid} swapped", DEV, True)
        for buf in b.values():
            buf.covered.zero_()
        prims.ema_swap_chunks(b["p"].t, b["ema"].t, b["shadow"].t, r["n_shadow"], t)
        torch.cuda.synchronize()
        C.check_swap(r, tab, b, P, f"{lid} restored", DEV, False)
        _report(lid, {"swap": (0.0, 0.0)})
    elif kind == "adamw_prepare":
        _prepare(r["n_sets"], r["max_norm"], 3.25, 9, lid)
    elif kind in ("lora_delta_merge", "lora_delta_grad"):
        inp = C.delta_inputs(r, DEV)
        if kind == "lora_delta_merge":
            out = {"merged": prims.lora_delta_merge(inp["base"], inp["A"], inp["B"], r["scaling"], bool(r["conv3d"]))}
        else:
            dA, dB = inp["dA"].clone(), inp["dB"].clone()
            prims.lora_delta_grad(inp["dw"], inp["A"], inp["B"], r["scaling"], bool(r["conv3d"]), dA, dB)
            out = {"dA": dA, "dB": dB}
        torch.cuda.synchronize()
        _report(lid, C.check_delta(r, inp, out, lid))
    elif kind == "scale_cast_f32_bf16":
        n = r["n"]
        x = C.cast_inputs(n, DEV)
        src = C.Buf(n, torch.float32, DEV)
        src.t.copy_(x.repeat(-(-n // x.numel()))[:n])
        dst = C.Buf(n, torch.bfloat16, DEV)
        prims.scale_cast_f32_bf16(src.t, dst.t, 1.0 / r["world"])
        torch.cuda.synchronize()
        src.covered.fill_(True)
        dst.covered.fill_(True)
        src.assert_untouched(f"{lid} src")
        dst.assert_untouched(f"{lid} dst")
        assert torch.equal(src.t[:x.numel()], x), f"{lid}: src written"
        _report(lid, C.check_cast(r, x, dst.t, lid))
    else:
        raise KeyError(kind)


def _prepare(n_sets, max_norm, sq0, k_before, what):
    from t2v_b200 import prims
    hp_in = torch.tensor([[5e-6, 0.9, 0.999, 1e-8, 1e-2], [1e-5, 0.8, 0.99, 1e-6, 1e-4]][:n_sets], dtype=torch.float32)
    hp = torch.full((n_sets, 8), float("nan"), device=DEV)
    state = torch.tensor([k_before], dtype=torch.int64, device=DEV)
    sq = torch.tensor([sq0, -7.0], dtype=torch.float64, device=DEV)
    prims.adamw_prepare(hp_in.to(DEV), hp, state, sq, max_norm)
    torch.cuda.synchronize()
    C.check_prepare(hp_in, hp.cpu(), k_before, state.cpu()[0], torch.tensor(sq0), sq.cpu(), max_norm, what)
    print(f"OPTIMCHECK {what} prepare ratio=0.000e+00 l2=0.000e+00")


@pytest.mark.parametrize("n_sets", [1, 2])
def test_prepare_sweep(n_sets):
    """k in {1, 2, 3, 10, 10^4, 10^6}; max_norm 0 (off), 1e6 (inactive), 1.0 (active: the norm is sqrt(3.25))."""
    for k in (1, 2, 3, 10, 10 ** 4, 10 ** 6):
        for max_norm in (0.0, 1e6, 1.0):
            _prepare(n_sets, max_norm, 3.25, k - 1, f"prepare-sets{n_sets}-k{k}-max{max_norm}")
