"""EMA of the trained weights (`use_ema`, optim.FusedAdamW / AdamW8bit `ema_decay`) on CPU over the emulated primitives: the
decay sequence against diffusers' EMAModel formula, both optimizers against torch AdamW + the EMAModel restatement in
tests/ema_ref.py, no feedback into the training state, the compact layout, the swap round trip, `train.main` checkpoints and
its argument checks."""
import os
import shutil

import pytest
import torch

import ema_ref as ref


def _diffusers_decay(optimization_step, decay=0.9999):
    """EMAModel.get_decay with its defaults (update_after_step 0, use_ema_warmup False, min_decay 0), called after
    `optimization_step += 1`."""
    step = max(0, optimization_step - 0 - 1)
    if step <= 0:
        return 0.0
    cur = (1 + step) / (10 + step)
    return max(min(cur, decay), 0.0)


def test_decay_sequence():
    assert ref.decay(1, 0.9999) == 0.0 and ref.decay(2, 0.9999) == 2 / 11
    cap = float(torch.tensor(0.999, dtype=torch.float32))    # binds from k = 8,991 on
    prev = -1.0
    for k in range(1, 10001):
        d = ref.decay(k, 0.999)
        assert d == _diffusers_decay(k, cap), k
        assert d >= prev and d <= cap
        prev = d
    assert ref.decay(10000, 0.999) == cap and ref.decay(8990, 0.999) < cap
    assert ref.decay(10000, 0.9999) == 10000 / 10009


# ---------------------------------------------------------------------------------------------------- optimizers vs torch
def _net():
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(24, 40), torch.nn.Linear(40, 16, bias=False), torch.nn.LayerNorm(16), torch.nn.Linear(16, 8),
                              torch.nn.Linear(8, 640))    # last weight: 5,120 elements -> 8-bit moments in AdamW8bit
    net[1].weight.requires_grad_(False)
    return net


def _groups(m):
    return [dict(params=[p for n, p in m.named_parameters() if n.startswith("0.")], lr=3e-3),
            dict(params=[p for n, p in m.named_parameters() if not n.startswith("0.") and p.requires_grad], lr=1e-3, weight_decay=0.05)]


def _train(cls, ema_decay, steps=6, ref_net=None):
    """`steps` optimizer steps of cls on _net() with seeded gradients; with ref_net, torch AdamW + clipping + the EMAModel
    restatement run the same gradients.  Returns (net, arena, opt, reference EMA by parameter name)."""
    from t2v_b200.runtime import ParamArena
    net = _net()
    kw = dict(lr=1e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=1e-2)
    if ref_net is not None:
        ref_net.load_state_dict(net.state_dict())
        o_ref = torch.optim.AdamW(_groups(ref_net), **kw)
        ema = {n: p.detach().clone() for n, p in ref_net.named_parameters() if p.requires_grad}
    arena = ParamArena(net)
    opt = cls(arena, _groups(net), max_grad_norm=1.0, ema_decay=ema_decay, **kw)
    g = torch.Generator().manual_seed(1)
    for step in range(steps):
        for n, q in net.named_parameters():
            if q.requires_grad:
                grad = torch.randn(q.shape, generator=g) * (3.0 if step == 2 else 0.3)
                q.grad.copy_(grad)
                if ref_net is not None:
                    ref_net.get_parameter(n).grad = grad.clone()
        opt.step()
        if ref_net is not None:
            torch.nn.utils.clip_grad_norm_([p for p in ref_net.parameters() if p.grad is not None], 1.0)
            o_ref.step()
            omd = ref.one_minus_decay(step + 1, ema_decay)
            for n, p in ref_net.named_parameters():
                if p.requires_grad:
                    ref.ema_step(ema[n], p.detach(), omd)
    return net, arena, opt, (ema if ref_net is not None else None)


def _ema_of(opt, arena, p):
    """The optimizer's EMA of parameter p, read through ema_weights()."""
    with opt.ema_weights():
        return p.detach().clone()


@pytest.mark.parametrize("name", ["FusedAdamW", "AdamW8bit"])
def test_optimizer_ema_matches_torch_adamw_and_restatement(name):
    from t2v_b200 import optim
    cls = getattr(optim, name)
    ref_net = _net()
    with ref.emulated():
        net, arena, opt, ema_ref = _train(cls, 0.9, ref_net=ref_net)
        assert opt.steps == 6 and len(opt._sets) == 2
        frozen = net[1].weight.detach().clone()
        with opt.ema_weights():
            got = {n: p.detach().clone() for n, p in net.named_parameters()}
        assert torch.equal(net[1].weight, frozen) and torch.equal(got["1.weight"], frozen)   # a frozen parameter is its own EMA
    for n, e in ema_ref.items():
        if name == "AdamW8bit" and n == "4.weight":
            continue   # 8-bit moments: the weights themselves only follow torch up to quantisation
        assert torch.allclose(got[n], e, rtol=1e-5, atol=1e-7), (n, float((got[n] - e).abs().max()))


@pytest.mark.parametrize("name", ["FusedAdamW", "AdamW8bit"])
def test_ema_never_feeds_back(name):
    """Weights, moments, shadow and step count are bit-identical to the same run without an EMA; the EMA is saved and
    snapshotted with the rest of the state."""
    from t2v_b200 import optim
    cls = getattr(optim, name)
    with ref.emulated():
        _, arena_a, opt_a, _ = _train(cls, None)
        net_b, arena_b, opt_b, _ = _train(cls, 0.99)
    assert opt_a.ema is None and "ema" not in opt_a.state_dict()["fused"]
    assert torch.equal(arena_a.master, arena_b.master) and torch.equal(arena_a.shadow, arena_b.shadow)
    for (k, a), b in zip(opt_a._moments().items(), opt_b._moments().values()):
        assert torch.equal(a, b), k
    assert opt_a.steps == opt_b.steps == 6
    assert len(opt_b.state_tensors()) == len(opt_a.state_tensors()) + 1 and torch.equal(opt_b.state_dict()["fused"]["ema"], opt_b.ema)


def test_ema_tracks_each_step():
    from t2v_b200.optim import FusedAdamW
    from t2v_b200.runtime import ParamArena
    net = _net()
    trainable = [p for p in net.parameters() if p.requires_grad]
    with ref.emulated():
        arena = ParamArena(net)
        opt = FusedAdamW(arena, trainable, lr=1e-2, ema_decay=0.95)
        track = [p.detach().clone() for p in trainable]
        assert all(torch.equal(_ema_of(opt, arena, p), t) for p, t in zip(trainable, track))   # starts as a copy
        g = torch.Generator().manual_seed(2)
        for k in range(1, 30):
            arena.grad.copy_(torch.randn(arena.grad.numel(), generator=g))
            opt.step()
            omd = ref.one_minus_decay(k, 0.95)
            for p, t in zip(trainable, track):
                ref.ema_step(t, p.detach(), omd)
            if k == 1:   # d_1 = 0: the weights, up to the rounding of ema - (ema - p) that EMAModel.step has as well
                assert all(torch.allclose(t, p.detach(), rtol=1e-7, atol=1e-9) for p, t in zip(trainable, track))
        for p, t in zip(trainable, track):
            assert torch.equal(_ema_of(opt, arena, p), t)


def test_swap_round_trip_is_bitwise():
    from t2v_b200.optim import AdamW8bit
    with ref.emulated():
        net, arena, opt, _ = _train(AdamW8bit, 0.9)
        before = [t.clone() for t in (arena.master, arena.shadow, opt.ema)]
        with opt.ema_weights():
            swapped = arena.master.clone()
            assert torch.equal(arena.shadow[:arena.n_mat], swapped[:arena.n_mat].bfloat16())
        for a, b in zip(before, (arena.master, arena.shadow, opt.ema)):
            assert torch.equal(a, b)
    o = arena.offsets[[id(p) for p in arena.params].index(id(net[1].weight))]
    frozen = slice(o, o + net[1].weight.numel())
    assert not torch.equal(swapped, before[0]) and torch.equal(swapped[frozen], before[0][frozen])


def test_ema_is_compact_on_a_lora_model():
    from test_train_loop import TINY
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.optim import FusedAdamW
    from t2v_b200.runtime import ParamArena, _align
    from t2v_b200.utils.lora_handler import LoraHandler
    m = UNet3DConditionModel(**TINY)
    m.requires_grad_(False)
    handler = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    handler.add_lora_to_model(True, m, handler.unet_replace_modules, 0.0, "", r=4)
    trainable = [p for p in m.parameters() if p.requires_grad]
    with ref.emulated():
        arena = ParamArena(m)
        opt = FusedAdamW(arena, trainable, lr=1e-3, ema_decay=0.9999)
        assert opt.ema.numel() == sum(_align(p.numel()) for p in trainable) < arena.total // 10
        weights = [p.detach().clone() for p in trainable]
        with opt.ema_weights():   # the EMA starts as a copy of the weights
            assert all(torch.equal(p, w) for p, w in zip(trainable, weights))


# ---------------------------------------------------------------------------------------------------- train.main
def _lora_files(out, step):
    d = os.path.join(out, "lora")
    return os.path.join(d, f"{step}_unet.pt"), os.path.join(d, f"{step}_unet_ema.pt")


def _weights(d, sub):
    from safetensors.torch import load_file
    return load_file(os.path.join(d, sub, "diffusion_pytorch_model.safetensors"))


def _lora_unet(lora_path=""):
    """A fresh TINY UNet with the LoRA injection of test_train_loop._run, loading lora_path when given."""
    from test_train_loop import TINY
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.utils.lora_handler import LoraHandler
    m = UNet3DConditionModel(**TINY)
    m.requires_grad_(False)
    handler = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    handler.add_lora_to_model(True, m, handler.unet_replace_modules, 0.0, lora_path, r=4)
    return m


def test_train_main_writes_ema_checkpoints(tmp_path, capsys):
    from test_train_loop import _run
    from t2v_b200.utils.lora import extract_lora_ups_down
    with ref.emulated():
        r = _run(tmp_path / "ema", "cpu", True, capsys, use_ema=True, ema_decay=0.9)
        base = _run(tmp_path / "plain", "cpu", True, capsys)
    opt, unet = r["optimizer"], r["stepper"].unet
    assert opt.ema is not None and base["optimizer"].ema is None
    out, out_base = str(tmp_path / "ema" / "out_lora"), str(tmp_path / "plain" / "out_lora")
    with ref.emulated(), opt.ema_weights():
        want_sd = {k: v.clone() for k, v in unet.state_dict().items()}
        want_lora = [t.weight.detach().clone() for ud in extract_lora_ups_down(unet, ["UNet3DConditionModel"]) for t in ud]
    for d, step in ((out, 2), (os.path.join(out, "checkpoint-1"), 1)):
        assert os.path.isdir(os.path.join(d, "unet_ema")) and all(os.path.isfile(f) for f in _lora_files(d, step)), d
    # the final EMA files hold the optimizer's EMA
    fresh = _lora_unet()
    fresh.load_state_dict(_weights(out, "unet_ema"))   # a LoRA run saves the UNet with its injected LoRA layers
    got = fresh.state_dict()
    assert got.keys() == want_sd.keys() and all(torch.equal(got[k], want_sd[k]) for k in got)
    saved = torch.load(_lora_files(out, 2)[1])
    assert len(saved) == len(want_lora) and all(torch.equal(a, b) for a, b in zip(saved, want_lora))
    lora_dir = tmp_path / "ema_lora_only"
    lora_dir.mkdir()
    shutil.copy(_lora_files(out, 2)[1], lora_dir / "2_unet_ema.pt")
    fresh = _lora_unet(str(lora_dir))
    loaded = [t.weight.detach() for ud in extract_lora_ups_down(fresh, ["UNet3DConditionModel"]) for t in ud]
    assert all(torch.equal(a, b) for a, b in zip(loaded, want_lora))
    assert not all(torch.equal(a, b) for a, b in zip(saved, torch.load(_lora_files(out, 2)[0])))
    # the training weights are those of the same seeded run without an EMA
    for step, d, db in ((2, out, out_base), (1, os.path.join(out, "checkpoint-1"), os.path.join(out_base, "checkpoint-1"))):
        a, b = torch.load(_lora_files(d, step)[0]), torch.load(_lora_files(db, step)[0])
        assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))
        sa, sb = _weights(d, "unet"), _weights(db, "unet")
        assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sb)
    assert not os.path.exists(os.path.join(out_base, "unet_ema"))


@pytest.mark.parametrize("kw", [dict(fused_adamw=False), dict(ema_decay=1.5), dict(ema_decay=-0.1), dict(ema_decay=float("nan")),
                                dict(ema_decay=float("inf"))])
def test_train_main_rejects_bad_ema_arguments_before_loading(tmp_path, monkeypatch, kw):
    from t2v_b200 import train

    def no_load(*a, **k):
        raise AssertionError("the UNet must not load")
    monkeypatch.setattr(train.UNet3DConditionModel, "from_pretrained", no_load)
    with pytest.raises(ValueError):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "out"), use_ema=True, device="cpu", **kw)
