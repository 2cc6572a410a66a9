"""Blockwise 8-bit AdamW (optim.AdamW8bit, `use_8bit_adam`): the quantisation maps against a committed table, small tensors
against torch.optim.AdamW, one step from zero state against the stated quantisation rule, convergence, `train.main`, the
compact state size; on the GPU checkpoint round trips and the CUDA-graph step (the kernel's element-wise check at every launch
of the training steps is tests/test_optim_step_gpu.py)."""
import json
import os

import pytest
import torch

import adamw8bit_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adamw8bit_qmaps.json")
gpu = pytest.mark.gpu
DEVICES = ["cpu", pytest.param("cuda", marks=gpu)]


def _ctx(device):
    import contextlib
    return ref.emulated() if device == "cpu" else contextlib.nullcontext()


def test_quantisation_maps():
    from t2v_b200.optim import dynamic_map
    with open(GOLDEN) as f:
        gold = json.load(f)
    for signed, key in ((True, "signed"), (False, "unsigned")):
        q = dynamic_map(signed)
        assert q.dtype == torch.float32 and q.shape == (256,)
        assert bool((q[1:] > q[:-1]).all())
        assert 0.0 in q.tolist() and 1.0 in q.tolist()
        assert bool((q < 0).any()) == signed
        assert torch.equal(q, torch.tensor(gold[key], dtype=torch.float32)), key


# ---------------------------------------------------------------------------------------------------- small tensors vs torch
def _net(device):
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(24, 40), torch.nn.Linear(40, 16, bias=False), torch.nn.LayerNorm(16), torch.nn.Linear(16, 8),
                              torch.nn.Linear(8, 640))    # last weight: 5,120 elements -> 8-bit; every other tensor < 4,096
    net[1].weight.requires_grad_(False)
    return net.to(device)


@pytest.mark.parametrize("device", DEVICES)
def test_small_tensors_match_torch_adamw(device):
    from t2v_b200 import optim
    from t2v_b200.runtime import ParamArena
    ref_net, net = _net(device), _net(device)
    net.load_state_dict(ref_net.state_dict())
    groups = lambda m: [dict(params=[p for n, p in m.named_parameters() if n.startswith("0.")], lr=3e-3),  # noqa: E731
                        dict(params=[p for n, p in m.named_parameters() if not n.startswith("0.")], lr=1e-3, weight_decay=0.05)]
    o_ref = torch.optim.AdamW(groups(ref_net), lr=1e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=1e-2)
    with _ctx(device):
        arena = ParamArena(net)
        o8 = optim.AdamW8bit(arena, groups(net), lr=1e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
        assert len(o8._sets) == 2 and o8.covers_all_trainable()
        assert o8._layout[id(net[4].weight)][0] == 8 and all(o8._layout[id(p)][0] == 32 for p in net.parameters()
                                                             if p.requires_grad and p is not net[4].weight)
        g = torch.Generator().manual_seed(1)
        frozen = net[1].weight.detach().clone()
        w0 = net[4].weight.detach().clone()
        for step in range(5):
            for p, q in zip(ref_net.parameters(), net.parameters()):
                if p.requires_grad:
                    grad = torch.randn(p.shape, generator=g).to(device) * (3.0 if step == 2 else 0.3)
                    p.grad = grad.clone()
                    q.grad.copy_(grad)
            norm = torch.nn.utils.clip_grad_norm_([p for p in ref_net.parameters() if p.grad is not None], 1.0)
            o_ref.step()
            o8.step()
            assert abs(float(o8.last_grad_norm()) - float(norm)) < 1e-5 * float(norm) and o8.steps == step + 1
            assert float(arena.grad.abs().max()) == 0.0
    for (n, p), q in zip(ref_net.named_parameters(), net.parameters()):
        if p.numel() < 4096:
            assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), (n, float((p - q).abs().max()))
    assert torch.equal(net[1].weight, frozen)
    # the 8-bit tensor follows torch's trajectory up to the quantisation of its moments
    d_ref, d8 = ref_net[4].weight.detach() - w0, net[4].weight.detach() - w0
    assert float((d8 - d_ref).norm() / d_ref.norm()) < 0.1
    for p in net.parameters():
        if p.dim() >= 2 and p.requires_grad:
            assert torch.equal(p._t2v_shadow.reshape(-1).float(), p.detach().reshape(-1).bfloat16().float())


# ---------------------------------------------------------------------------------------------------- one step, zero state
def test_first_step_follows_the_quantisation_rule():
    from t2v_b200 import optim
    from t2v_b200.runtime import ParamArena
    torch.manual_seed(0)
    # 4,160 elements: 16 full blocks + a 64-element block; 65,792: two chunk rows (65,536 + 256)
    net = torch.nn.Sequential(torch.nn.Linear(65, 64, bias=False), torch.nn.Linear(257, 256, bias=False))
    b1, b2 = 0.9, 0.999
    with ref.emulated():
        arena = ParamArena(net)
        opt = optim.AdamW8bit(arena, net.parameters(), lr=1e-3, betas=(b1, b2), eps=1e-8, weight_decay=1e-2)
        assert opt._sets[0]["chunks"].shape == (3, 4)
        g = torch.Generator().manual_seed(2)
        grads = {}
        for p in net.parameters():
            grads[p] = torch.randn(p.shape, generator=g)
            grads[p].view(-1)[:256] = 0.0       # first block all zero
            p.grad.copy_(grads[p])
        opt.step()
    b1t, b2t = torch.tensor(b1, dtype=torch.float32), torch.tensor(b2, dtype=torch.float32)
    for p in net.parameters():
        assert torch.isfinite(p).all()
        bits, s = opt._layout[id(p)]
        assert bits == 8
        n = p.numel()
        nb = (n + 255) // 256
        gv = grads[p].reshape(-1)
        for x, qmap, codes, absmax in (((1 - b1t) * gv, opt.qmaps[:256], opt.code_m, opt.absmax_m),
                                       ((1 - b2t) * gv * gv, opt.qmaps[256:], opt.code_v, opt.absmax_v)):
            am = absmax[s // 256:s // 256 + nb]
            padded = torch.zeros(nb * 256)
            padded[:n] = x.abs()
            assert torch.allclose(am, padded.view(nb, 256).amax(1), rtol=1e-6, atol=0)
            assert float(am[0]) == 0.0 and int(codes[s]) == int((qmap == 0).nonzero()[0, 0])
            c = codes[s:s + n].long()
            gap = torch.maximum(qmap[(c + 1).clamp(max=255)] - qmap[c], qmap[c] - qmap[(c - 1).clamp(min=0)])
            a = am.repeat_interleave(256)[:n]
            err = (qmap[c] * a - x).abs()
            # half a map gap, plus fp32 rounding of x / absmax for moments that sit on a midpoint
            assert bool((err <= 0.5 * gap * a + 5e-7 * x.abs()).all()), float((err - 0.5 * gap * a).max())


# ---------------------------------------------------------------------------------------------------- convergence
def _least_squares(device, make_opt, steps=300):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(512, 128, generator=g).to(device)
    w_true = (torch.randn(64, 128, generator=g) / 128 ** 0.5).to(device)
    y = x @ w_true.t() + 0.01 * torch.randn(512, 64, generator=g).to(device)
    torch.manual_seed(4)
    lin = torch.nn.Linear(128, 64, bias=False).to(device)   # 8,192 elements: 8-bit moments
    opt = make_opt(lin)
    w = lin.weight
    for _ in range(steps):
        loss = ((x @ w.t() - y) ** 2).mean()
        (grad,) = torch.autograd.grad(loss, [w])
        if w.grad is None:
            w.grad = grad
        else:
            w.grad.copy_(grad)
        opt.step()
    return float(((x @ w.detach().t() - y) ** 2).mean())


@pytest.mark.parametrize("device", DEVICES)
def test_converges_like_torch_adamw(device):
    from t2v_b200 import optim
    from t2v_b200.runtime import ParamArena
    kw = dict(lr=3e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    base = _least_squares(device, lambda lin: torch.optim.AdamW(lin.parameters(), **kw))
    with _ctx(device):
        got = _least_squares(device, lambda lin: optim.AdamW8bit(ParamArena(lin), lin.parameters(), max_grad_norm=1.0, **kw))
    assert got <= 1.1 * base, (got, base)


# ---------------------------------------------------------------------------------------------------- train.main, state size
@pytest.mark.parametrize("lora", [False, True])
def test_train_main_8bit_cpu_emulated(tmp_path, capsys, lora):
    from test_train_loop import _run
    from t2v_b200.optim import AdamW8bit
    with ref.emulated():
        r = _run(tmp_path, "cpu", lora, capsys, use_8bit_adam=True)
    assert isinstance(r["optimizer"], AdamW8bit) and r["optimizer"].steps == 2


def test_train_main_8bit_rejects_torch_adamw(tmp_path):
    from t2v_b200 import train
    with pytest.raises(ValueError):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "out"), use_8bit_adam=True, fused_adamw=False,
                   device="cpu")


def test_state_is_compact():
    """Bytes of state = 2 per element of the 8-bit tensors (each padded to whole blocks) + 8 per block + 8 per element of the
    fp32 tensors; frozen parameters cost nothing."""
    from test_train_loop import TINY
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.optim import AdamW8bit
    from t2v_b200.runtime import ParamArena, _align
    m = UNet3DConditionModel(**TINY)
    m.requires_grad_(False)
    for n, p in m.named_parameters():
        if "attn1" in n or "attn2" in n:
            p.requires_grad_(True)
    trainable = [p for p in m.parameters() if p.requires_grad]
    with ref.emulated():
        opt = AdamW8bit(ParamArena(m), trainable, lr=1e-3)
    want, n8 = 0, 0
    for p in trainable:
        if p.numel() >= 4096:
            blocks = (_align(p.numel()) + 255) // 256
            want += 2 * 256 * blocks + 8 * blocks
            n8 += 1
        else:
            want += 8 * _align(p.numel())
    assert n8 > 0 and opt.state_bytes() == want
    assert want < 8 * sum(p.numel() for p in trainable) / 3


# ---------------------------------------------------------------------------------------------------- GPU: kernel cases (tests/test_ema_gpu.py)
def _kernel_case(seed):
    """Four tensors in a flat arena: 8-bit with a ragged 64-element last block, 8-bit over two chunk rows with a ragged
    320-element last row, a 32-bit one and 8-bit with a ragged 128-element block that has no bf16 shadow.  Two
    hyper-parameter sets: tensors {0, 2} and {1, 3}."""
    lens, bits = [4160, 65856, 1024, 4224], [8, 8, 32, 8]
    offs, soffs, off, s8, s32 = [], [], 0, 0, 0
    for n, b in zip(lens, bits):
        offs.append(off)
        off += n
        if b == 8:
            soffs.append(s8)
            s8 += (n + 255) // 256 * 256
        else:
            soffs.append(s32)
            s32 += n
    rows = [[], []]
    for i, (n, b) in enumerate(zip(lens, bits)):
        for lo in range(0, n, 65536):
            rows[i % 2].append((offs[i] + lo, min(65536, n - lo), soffs[i] + lo, b))
    g = torch.Generator().manual_seed(seed)
    st = {"p": torch.randn(off, generator=g), "shadow": torch.randn(off, generator=g).bfloat16(),
          "m32": torch.randn(s32, generator=g) * 1e-2, "v32": torch.rand(s32, generator=g) * 1e-4,
          "code_m": torch.randint(0, 256, (s8,), generator=g).to(torch.uint8), "code_v": torch.randint(0, 256, (s8,), generator=g).to(torch.uint8),
          "absmax_m": torch.rand(s8 // 256, generator=g) * 1e-2, "absmax_v": torch.rand(s8 // 256, generator=g) * 1e-4}
    st["absmax_m"][3] = 0.0    # a block whose previous absmax is 0 dequantises to 0
    mask8 = torch.zeros(s8, dtype=torch.bool)
    for n, b, s in zip(lens, bits, soffs):
        if b == 8:
            mask8[s:s + n] = True
    return st, [torch.tensor(r, dtype=torch.int64) for r in rows], offs[3], mask8, g


def _hp(step):
    out = []
    for lr, b1, b2, eps, wd, scale in ((1e-3, 0.9, 0.999, 1e-8, 1e-2, 0.7), (5e-4, 0.8, 0.99, 1e-6, 0.0, 1.0)):
        out.append(torch.tensor([lr, b1, b2, eps, wd, 1 - b1 ** step, (1 - b2 ** step) ** 0.5, scale], dtype=torch.float32))
    return out


# ---------------------------------------------------------------------------------------------------- GPU: checkpoint, train.main
def _round_trip_net():
    torch.manual_seed(6)
    return torch.nn.Sequential(torch.nn.Linear(96, 80), torch.nn.LayerNorm(80), torch.nn.Linear(80, 8)).cuda()   # 7,680 / 80 / 640


def _steps(opt, arena, first, count):
    for k in range(first, first + count):
        g = torch.Generator().manual_seed(100 + k)
        arena.grad.copy_(torch.randn(arena.grad.numel(), generator=g).cuda())
        opt.step()


@gpu
def test_state_dict_round_trip_is_bit_identical():
    """N steps, save, load into a fresh optimizer on a copy of the weights, M more steps == N + M steps without a break.
    No clipping: the gradient norm sums with atomics, the 8-bit update has none."""
    from t2v_b200.optim import AdamW8bit
    from t2v_b200.runtime import ParamArena
    kw = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    net_a = _round_trip_net()
    arena_a = ParamArena(net_a)
    opt_a = AdamW8bit(arena_a, net_a.parameters(), **kw)
    _steps(opt_a, arena_a, 0, 7)
    net_b = _round_trip_net()
    arena_b = ParamArena(net_b)
    opt_b = AdamW8bit(arena_b, net_b.parameters(), **kw)
    _steps(opt_b, arena_b, 0, 3)
    sd = opt_b.state_dict()
    sd["fused"] = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in sd["fused"].items()}
    net_c = _round_trip_net()
    arena_c = ParamArena(net_c)
    arena_c.master.copy_(arena_b.master)
    arena_c.refresh_shadow()
    opt_c = AdamW8bit(arena_c, net_c.parameters(), **kw)
    opt_c.load_state_dict(sd)
    assert opt_c.steps == 3
    _steps(opt_c, arena_c, 3, 4)
    torch.cuda.synchronize()
    assert torch.equal(arena_c.master, arena_a.master) and torch.equal(arena_c.shadow, arena_a.shadow)
    for (k, a), c in zip(opt_a._moments().items(), opt_c._moments().values()):
        assert torch.equal(a, c), k


@gpu
@pytest.mark.parametrize("lora", [False, True])
def test_train_main_8bit_gpu_graph(tmp_path, capsys, lora):
    from test_train_loop import _run
    from t2v_b200.optim import AdamW8bit
    r = _run(tmp_path, "cuda:0", lora, capsys, use_8bit_adam=True)
    assert isinstance(r["optimizer"], AdamW8bit)
    assert r["stepper"].use_graph and len(r["stepper"]._graphs) == 1
    assert r["optimizer"].steps == 2   # the capture's dry runs were undone from the snapshot
