"""Clips longer than 32 frames on the CPU: the fp32 restatement of attn_long (tests/long_clip_ref.py) against float64
autograd, the F <= 32 / F > 32 dispatch of ops.temporal_attention, a 40-frame UNet step against the oracle, and train.main
with 40 frames (and its refusal of 257) - all over emulated primitives."""
import os

import pytest
import torch

import long_clip_ref as LC
from helpers import rel_l2, seeded_state_dict

SMALL = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)


def _tokens(B, F, HW, heads, D, fused, dtype=torch.float32, seed=0):
    """q, k, v as strided views of frames-major tokens [B*F*HW, C] (column slices of one [rows, 3C] buffer when fused)."""
    g = torch.Generator().manual_seed(seed)
    C, rows = heads * D, B * F * HW
    if fused:
        qkv = torch.randn(rows, 3 * C, generator=g).to(dtype)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    else:
        qkv = None
        q, k, v = (torch.randn(rows, C, generator=g).to(dtype) for _ in range(3))
    do = torch.randn(rows, C, generator=g).to(dtype)
    return qkv, q, k, v, do


def _addr(B, F, HW, heads, D, fused):
    C = heads * D
    return (B * HW, HW, F * HW, 1, HW, 3 * C if fused else C, C, heads, F, D)


def _autograd64(q, k, v, do, B, F, HW, heads, D):
    """float64 attention along the frame axis by explicit permutes: tokens [B, F, HW, heads, D] -> [B, HW, heads, F, D]."""
    def seq(t):
        return t.double().reshape(B, F, HW, heads, D).permute(0, 2, 3, 1, 4).detach().requires_grad_(True)
    Q, K, V = seq(q), seq(k), seq(v)
    S = Q @ K.transpose(-1, -2) * D ** -0.5
    O = torch.softmax(S, -1) @ V
    dO = do.double().reshape(B, F, HW, heads, D).permute(0, 2, 3, 1, 4)
    gq, gk, gv = torch.autograd.grad(O, (Q, K, V), dO)
    back = lambda t: t.permute(0, 3, 1, 2, 4).reshape(B * F * HW, heads * D)
    return back(O), torch.logsumexp(S, -1).reshape(B * HW, heads, F), back(gq), back(gk), back(gv)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("L", [8, 48, 100])
def test_reference_matches_float64_autograd(L, fused):
    B, HW, heads, D = 2, 3, 2, 32
    _, q, k, v, do = _tokens(B, L, HW, heads, D, fused)
    addr = _addr(B, L, HW, heads, D, fused)
    o_ref, lse_ref, gq, gk, gv = _autograd64(q, k, v, do, B, L, HW, heads, D)
    o = torch.zeros_like(do)
    lse = torch.zeros(B * HW, heads, L)
    LC.attn_long_fwd(q, k, v, o, lse, addr)
    assert torch.allclose(o.double(), o_ref, rtol=0, atol=1e-5)
    assert torch.allclose(lse.double(), lse_ref, rtol=0, atol=1e-5)
    grads = torch.zeros(3, *q.shape) if not fused else torch.zeros(q.shape[0], 3 * q.shape[1])
    C = heads * D
    dq, dk, dv = (grads[i] for i in range(3)) if not fused else (grads[:, :C], grads[:, C:2 * C], grads[:, 2 * C:])
    LC.attn_long_bwd(q, k, v, o, do, lse, dq, dk, dv, addr)
    for got, exp in ((dq, gq), (dk, gk), (dv, gv)):
        assert torch.allclose(got.double(), exp, rtol=0, atol=1e-4 * exp.abs().max().item())


def _count_attention_calls():
    from t2v_b200 import prims
    calls = {n: 0 for n in ("attn_small_fwd", "attn_small_bwd", "attn_long_fwd", "attn_long_bwd")}
    for n in calls:
        fn = getattr(prims, n)

        def counted(*a, _n=n, _fn=fn):
            calls[_n] += 1
            return _fn(*a)
        setattr(prims, n, counted)
    return calls


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("F", [32, 48])
def test_temporal_attention_dispatch_by_frame_count(F, fused):
    """F <= 32 takes exactly the attn_small path; F = 48 only attn_long.  Values and gradients match float64 autograd."""
    from t2v_b200 import ops
    B, HW, heads, D = 2, 3, 2, 64
    qkv, q, k, v, do = _tokens(B, F, HW, heads, D, fused, seed=1)
    with LC.emulated_prims():
        calls = _count_attention_calls()
        if fused:
            x = qkv.clone().requires_grad_(True)
            o = ops.temporal_attention_fused(x, heads, B, F, HW)
            o.backward(do)
            C = heads * D
            got = (x.grad[:, :C], x.grad[:, C:2 * C], x.grad[:, 2 * C:])
        else:
            xs = [t.clone().requires_grad_(True) for t in (q, k, v)]
            o = ops.temporal_attention(*xs, heads, B, F, HW)
            o.backward(do)
            got = tuple(t.grad for t in xs)
    long = F > 32
    assert calls == {"attn_small_fwd": int(not long), "attn_small_bwd": int(not long),
                     "attn_long_fwd": int(long), "attn_long_bwd": int(long)}, calls
    o_ref, _, *g_ref = _autograd64(q, k, v, do, B, F, HW, heads, D)
    assert torch.allclose(o.detach().double(), o_ref, rtol=0, atol=1e-5)
    for a, b in zip(got, g_ref):
        assert torch.allclose(a.double(), b, rtol=0, atol=1e-4 * b.abs().max().item())


def test_small_unet_step_at_40_frames_matches_oracle():
    """step.finetune_loss at F = 40 (every temporal attention on attn_long) over emulated primitives against the oracle,
    with the bounds of tests/test_v_prediction_cpu.py (fp32 activations, bf16 weight shadows)."""
    from oracle import leaves as L
    from oracle import ops_ref
    from oracle import unet3d_ref as R
    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    sd = seeded_state_dict(m, 5)
    m.load_state_dict(sd)
    m.eval().requires_grad_(True)
    g = torch.Generator().manual_seed(11)
    lat = torch.randn(1, 4, 40, 8, 8, generator=g) * 0.18215 * 5
    noise = torch.randn(1, 4, 40, 8, 8, generator=g)
    t = torch.tensor([417])
    ehs = torch.randn(1, 5, 64, generator=g)
    abar = L.ddpm_alphas_cumprod()
    old = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        with LC.emulated_prims():
            calls = _count_attention_calls()
            loss = S.finetune_loss(m, lat, noise, t, ehs, abar)
            loss.backward()
    finally:
        ops_ref.BF = old
    assert calls["attn_long_fwd"] > 0 and calls["attn_long_bwd"] == calls["attn_long_fwd"], calls
    assert calls["attn_small_fwd"] == calls["attn_small_bwd"] == 0, calls
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    loss_r, _ = R.finetune_loss(p, R.full_config(**SMALL), lat, noise, t, ehs, abar)
    loss_r.backward()
    assert abs(loss.item() - loss_r.item()) <= 2e-2 * loss_r.item(), (loss.item(), loss_r.item())
    top = max(v.grad.norm().item() for v in p.values() if v.grad is not None)
    errs = sorted(rel_l2(q.grad, p[n].grad) for n, q in m.named_parameters()
                  if p[n].grad is not None and p[n].grad.norm().item() >= 1e-5 * top)
    assert len(errs) > 500 and errs[len(errs) // 2] < 4e-2 and errs[-1] < 0.15, (len(errs), errs[len(errs) // 2], errs[-5:])
    temporal = [rel_l2(q.grad, p[n].grad) for n, q in m.named_parameters() if "temp_attentions" in n and "to_q" in n]
    assert temporal and max(temporal) < 4e-2, temporal


def _pretrained_unet(root):
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    m.load_state_dict(seeded_state_dict(m, 0))
    m.save_pretrained(os.path.join(root, "unet"))
    return root


def run_long_training(tmp_path, device, frames=40, **extra):
    from t2v_b200 import train
    root = _pretrained_unet(str(tmp_path / "model"))
    kw = dict(pretrained_model_path=root, output_dir=str(tmp_path / "out"), dataset_types=["synthetic"],
              train_data=dict(n=2, n_sample_frames=frames, height=64, width=64), max_train_steps=2, learning_rate=1e-4,
              checkpointing_steps=10, seed=0, shuffle=False, device=device, eval_train=True, trainable_modules=["temp_attentions"],
              save_pretrained_model=False)
    kw.update(extra)
    return train.main(**kw)


def test_train_main_40_frames_cpu(tmp_path):
    with LC.emulated_prims():
        calls = _count_attention_calls()
        r = run_long_training(tmp_path, "cpu")
    assert r["steps"] == 2
    assert calls["attn_long_fwd"] > 0 and calls["attn_long_bwd"] > 0 and calls["attn_small_fwd"] == 0, calls


@pytest.mark.parametrize("section", ["train_data", "validation_data"])
def test_train_main_rejects_257_frames_before_loading_the_unet(tmp_path, section):
    """The pretrained folder has no unet/ at all: the ValueError must come first, not a missing-file error."""
    from t2v_b200 import train
    kw = dict(train_data=dict(n_sample_frames=257)) if section == "train_data" else dict(validation_data=dict(num_frames=257))
    with pytest.raises(ValueError, match="257"):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "out"), dataset_types=["synthetic"], device="cpu",
                   **kw)
