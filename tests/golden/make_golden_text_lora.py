"""Generates tests/golden/text_lora_*.pt from the REFERENCE's own code: $T2V_REFERENCE_ROOT/utils/lora.py imported unmodified
(inject_trainable_lora_extended, LoraInjectedLinear) injected into a real `transformers.CLIPTextModel` and into the reference's
models/*.py UNet over oracle/diffusers_standin, and the two-pass step of the reference's train.py:803-834 restated line by line
with text_trainable = True.  fp32, CPU, eval mode (dropout is the identity; its mask is a torch RNG draw):
    T2V_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_golden_text_lora.py
Weights are not stored: the base weights come from helpers.seeded_state_dict and the LoRA factors from make_golden_lora.seed_lora_
(both keyed by parameter name, so the test rebuilds the same values on its own models)."""
import contextlib
import io
import os
import sys
import tempfile

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from helpers import seeded_state_dict  # noqa: E402
from make_golden_lora import ref_lora, seed_lora_  # noqa: E402
from oracle import leaves as L  # noqa: E402
from oracle.reference_import import import_reference_unet  # noqa: E402

UNET = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=128)
TEXT = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, max_position_embeddings=77,
            hidden_act="gelu", layer_norm_eps=1e-5)
R_UNET, R_TEXT, SEEDS = 8, 4, dict(unet_base=0, text_base=5, unet_lora=11, text_lora=13)
PROMPTS = ["a red ball rolls", "waves"]
VITH = dict(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23, num_attention_heads=16,
            max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5)


def prompt_ids():
    """The prompts through a real CLIPTokenizer (byte-level vocabulary of tests/test_pipeline_train.py), padded to 77 as
    the reference's get_prompt_ids pads them."""
    from transformers import CLIPTokenizer
    from test_pipeline_train import _tiny_tokenizer
    with tempfile.TemporaryDirectory() as d:
        nvocab = _tiny_tokenizer(d)
        tok = CLIPTokenizer.from_pretrained(d)
    ids = tok(PROMPTS, truncation=True, padding="max_length", max_length=tok.model_max_length, return_tensors="pt").input_ids
    return ids, nvocab


def census(ref):
    from transformers import CLIPTextConfig, CLIPTextModel
    with torch.device("meta"), contextlib.redirect_stdout(io.StringIO()):
        m = CLIPTextModel(CLIPTextConfig(**VITH))
        ref.inject_trainable_lora_extended(m, {"CLIPEncoderLayer"}, r=16)
    return [(n, tuple(w.lora_down.weight.shape), tuple(w.lora_up.weight.shape)) for n, w in m.named_modules()
            if isinstance(w, ref.LoraInjectedLinear)]


def case(ref, frames):
    from transformers import CLIPTextConfig, CLIPTextModel
    ids, nvocab = prompt_ids()
    te = CLIPTextModel(CLIPTextConfig(vocab_size=nvocab, **TEXT))
    te.load_state_dict({k: v for k, v in seeded_state_dict(te, SEEDS["text_base"]).items() if not k.endswith("position_ids")},
                       strict=False)
    te.requires_grad_(False)
    unet = import_reference_unet()(**UNET)
    unet.load_state_dict(seeded_state_dict(unet, SEEDS["unet_base"]))
    unet.requires_grad_(False)
    with contextlib.redirect_stdout(io.StringIO()):
        ref.inject_trainable_lora_extended(te, {"CLIPEncoderLayer"}, r=R_TEXT)
        ref.inject_trainable_lora_extended(unet, {"UNet3DConditionModel"}, r=R_UNET)
    seed_lora_(te, SEEDS["text_lora"])
    seed_lora_(unet, SEEDS["unet_lora"])
    te.eval()
    unet.eval()
    B = ids.shape[0]
    g = torch.Generator().manual_seed(17 + frames)
    latents = torch.randn(B, 4, frames, 16, 16, generator=g)
    noise = torch.randn(B, 4, frames, 16, 16, generator=g)
    timesteps = torch.tensor([211, 733])
    abar = L.ddpm_alphas_cumprod()
    noisy_latents = L.add_noise(latents, noise, timesteps, abar)
    target = noise                                       # prediction_type 'epsilon'
    encoder_hidden_states = te(ids)[0]
    encoder_hidden_states.retain_grad()
    # ---- reference train.py:803-834, text_trainable = True
    video_length = latents.shape[2]
    losses = []
    should_truncate_video = video_length > 1
    detached_encoder_state = encoder_hidden_states.clone().detach()
    trainable_encoder_state = encoder_hidden_states.clone()
    for i in range(2):
        should_detach = noisy_latents.shape[2] > 1 and i == 0
        if should_truncate_video and i == 1:
            noisy_latents = noisy_latents[:, :, 1, :, :].unsqueeze(2)
            target = target[:, :, 1, :, :].unsqueeze(2)
        ehs = detached_encoder_state if should_detach else trainable_encoder_state
        model_pred = unet(noisy_latents, timesteps, encoder_hidden_states=ehs).sample
        losses.append(F.mse_loss(model_pred.float(), target.float(), reduction="mean"))
        if video_length == 1 and i == 0:
            break
    loss = losses[0] if len(losses) == 1 else losses[0] + losses[1]
    # ----
    loss.backward()
    text_grads = {n: p.grad.detach().clone() for n, p in te.named_parameters() if "lora" in n}
    unet_grads = {n: p.grad for n, p in unet.named_parameters() if "lora" in n and p.grad is not None}
    small = [n for n in unet_grads if unet_grads[n].numel() <= 2048]
    keep = sorted(small, key=lambda n: -unet_grads[n].norm().item())[:24]
    return dict(unet_cfg=UNET, text_cfg=dict(TEXT, vocab_size=nvocab), r_unet=R_UNET, r_text=R_TEXT, seeds=SEEDS, prompt_ids=ids,
                latents=latents, noise=noise, timesteps=timesteps, pass_losses=[x.detach() for x in losses],
                states_grad=encoder_hidden_states.grad.detach().clone(),
                text_grads=text_grads, text_grad_norms={n: v.norm().item() for n, v in text_grads.items()},
                unet_grad_norms={n: v.norm().item() for n, v in unet_grads.items()},
                unet_grads={n: unet_grads[n].detach().clone() for n in keep},
                source="reference utils/lora.py on transformers.CLIPTextModel and the reference's models/*.py over "
                       "oracle/diffusers_standin; step restated from train.py:803-834; fp32 CPU, eval mode")


def main():
    torch.set_num_threads(8)
    ref = ref_lora()
    golden = os.path.join(ROOT, "tests", "golden")
    path = os.path.join(golden, "text_lora_census_vith.pt")
    torch.save(census(ref), path)
    print("census", os.path.getsize(path) // 1024, "KiB")
    for frames in (4, 1):
        path = os.path.join(golden, f"text_lora_step_f{frames}.pt")
        torch.save(case(ref, frames), path)
        print(path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
