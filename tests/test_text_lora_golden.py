"""Text-encoder LoRA against the REFERENCE's own code (tests/golden/make_golden_text_lora.py): the reference's utils/lora.py on a
real transformers.CLIPTextModel and on the reference UNet, with the two-pass step of train.py:803-834 (F = 4: pass 0 on the
full clip with detached states, pass 1 on frame 1 with the trainable states; F = 1: one pass).  The H100-native side is
`step.DataParallelStep(text_encoder=)` with this repo's encoder, injector and UNet.  CPU: emulated primitives in fp32, at 1e-4.
GPU: the CUDA kernels, at the cloneofsimo tolerances of DESIGN §5 (loss 3e-3; >= 97 % of gradient tensors with cosine > 0.98)."""
import contextlib
import io
import os
import sys

import pytest
import torch

from helpers import cosine, seeded_state_dict
from oracle import ops_ref
from text_lora_ref import emulated

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLDEN)
DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


def test_injection_census_matches_reference():
    """The reference's injector on transformers' ViT-H text tower and this repo's injector on its own encoder wrap the same
    138 Linear layers, in the same order, with the same factor shapes."""
    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils import lora as mylora
    want = torch.load(os.path.join(GOLDEN, "text_lora_census_vith.pt"), weights_only=False)
    with torch.device("meta"), contextlib.redirect_stdout(io.StringIO()):
        m = CLIPTextModel()
        mylora.inject_trainable_lora_extended(m, {"CLIPEncoderLayer"}, r=16)
    got = [(n, tuple(w.lora_down.weight.shape), tuple(w.lora_up.weight.shape)) for n, w in m.named_modules()
           if isinstance(w, mylora.LoraInjectedLinear)]
    assert len(want) == 138 and got == [tuple(x) for x in want]


@contextlib.contextmanager
def _backend(device):
    if device == "cpu":
        old = ops_ref.BF
        ops_ref.BF = torch.float32
        try:
            with emulated():
                yield
        finally:
            ops_ref.BF = old
    else:
        yield


def _models(c, device):
    from make_golden_lora import seed_lora_
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils import lora as mylora
    unet = UNet3DConditionModel(**c["unet_cfg"])
    unet.load_state_dict(seeded_state_dict(unet, c["seeds"]["unet_base"]))
    unet.requires_grad_(False)
    te = CLIPTextModel(c["text_cfg"])
    te.load_state_dict(seeded_state_dict(te, c["seeds"]["text_base"]))
    with contextlib.redirect_stdout(io.StringIO()):
        mylora.inject_trainable_lora_extended(te, {"CLIPEncoderLayer"}, r=c["r_text"])
        mylora.inject_trainable_lora_extended(unet, {"UNet3DConditionModel"}, r=c["r_unet"])
    seed_lora_(te, c["seeds"]["text_lora"])
    seed_lora_(unet, c["seeds"]["unet_lora"])
    return unet.to(device).eval(), te.to(device).eval()


def _run_step(c, device, monkeypatch):
    from t2v_b200 import step as S
    unet, te = _models(c, device)
    losses, states = [], []
    finetune_loss, encode = S.finetune_loss, te.encode

    def record_loss(*a, **k):
        loss = finetune_loss(*a, **k)
        losses.append(loss.detach())
        return loss

    def record_states(ids):
        out = encode(ids)
        out.retain_grad()
        states.append(out)
        return out
    monkeypatch.setattr(S, "finetune_loss", record_loss)
    monkeypatch.setattr(te, "encode", record_states)
    with _backend(device):
        # the parameter arena keeps bf16 copies of the weights for the kernels, so the fp32 CPU check runs without it
        stepper = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device=device), passes=2, text_encoder=te, adopt=device != "cpu")
        total = stepper(c["latents"].to(device), c["noise"].to(device), c["timesteps"].to(device), c["prompt_ids"].to(device))
    return unet, te, total, losses, states[0]


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("frames", [4, 1])
def test_step_matches_reference(frames, device, monkeypatch):
    c = torch.load(os.path.join(GOLDEN, f"text_lora_step_f{frames}.pt"), weights_only=False)
    unet, te, total, losses, states = _run_step(c, device, monkeypatch)
    want = c["pass_losses"]
    assert len(losses) == len(want) == (2 if frames > 1 else 1)
    loss_tol = 1e-4 if device == "cpu" else 3e-3
    for got, ref in zip(losses, want):
        assert abs(got.item() - ref.item()) <= loss_tol * abs(ref.item()), (got.item(), ref.item())
    assert abs(total.item() - sum(x.item() for x in want)) <= loss_tol * sum(x.item() for x in want)
    states_grad = states.grad.float().cpu().view(c["states_grad"].shape)
    text = dict(te.named_parameters())
    unet_p = dict(unet.named_parameters())
    assert sorted(n for n, p in text.items() if p.grad is not None) == sorted(c["text_grads"])
    # LoRA tensors the reference gave no gradient (the temporal layers at F = 1) have none here either: the arena's gradient
    # views exist for every trainable tensor, so "none" means all zero
    for n, p in unet_p.items():
        if "lora" in n and n not in c["unet_grad_norms"]:
            assert p.grad is None or not p.grad.any(), n
    assert all(unet_p[n].grad is not None for n in c["unet_grad_norms"])
    pairs = [(states_grad, c["states_grad"])] + [(text[n].grad, g) for n, g in c["text_grads"].items()] \
        + [(unet_p[n].grad, g) for n, g in c["unet_grads"].items()]
    if device == "cpu":
        for got, ref in pairs:
            assert (got.float().cpu() - ref).norm() <= 1e-4 * ref.norm(), (got.norm(), ref.norm())
        top = max(c["unet_grad_norms"].values())
        for n, gn in c["unet_grad_norms"].items():
            assert abs(unet_p[n].grad.norm().item() - gn) <= 1e-4 * max(gn, 1e-3 * top), n
        for n, gn in c["text_grad_norms"].items():
            assert abs(text[n].grad.norm().item() - gn) <= 1e-4 * gn, n
    else:
        cos = [cosine(got.float().cpu(), ref) for got, ref in pairs]
        assert sum(x > 0.98 for x in cos) >= 0.97 * len(cos), sorted(cos)[:5]
        for n, gn in c["text_grad_norms"].items():
            assert abs(text[n].grad.norm().item() - gn) <= 5e-2 * gn, n
