"""Generates tests/golden/text_train_*.pt from the REFERENCE's own code: a real `transformers.CLIPTextModel` (tokenizer-padded
prompts, so the pad id repeats) and the reference's models/*.py UNet over oracle/diffusers_standin; for the combined case the
reference's utils/lora.py injects cloneofsimo LoRA into the text encoder, imported unmodified.  The reference's train.py does
not import without accelerate / diffusers, so these parts of it are restated line by line:
  * handle_trainable_modules (train.py:316-337) and create_optimizer_params / param_optim (:205-236), with the group order of
    :579-595 - UNet, text encoder, text LoRA - and the text groups built from extra_unet_params (:576, SURVEY H4);
  * the two-pass step of :803-834 with text_trainable = True;
  * the clip over list(unet.parameters()) + list(text_encoder.parameters()) (:863-875) and one torch.optim.AdamW step.
fp32, CPU, eval mode (dropout is the identity):
    T2V_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_golden_text_train.py
Weights are not stored: the base weights come from helpers.seeded_state_dict and the LoRA factors from make_golden_lora.seed_lora_."""
import contextlib
import io
import itertools
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from helpers import seeded_state_dict  # noqa: E402
from make_golden_lora import ref_lora, seed_lora_  # noqa: E402
from make_golden_text_lora import prompt_ids  # noqa: E402
from oracle import leaves as L  # noqa: E402
from oracle.reference_import import import_reference_unet  # noqa: E402

UNET = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)
TEXT = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, max_position_embeddings=77,
            hidden_act="gelu", layer_norm_eps=1e-5)
SEEDS = dict(unet_base=0, text_base=5, text_lora=13)
R_TEXT = 4
TRAINABLE_MODULES = ["attn2.to_out"]
HYPER = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0, extra_unet_params={"weight_decay": 0.25})
CASES = {"all": (["all"], False), "substring": (["layers.1.mlp", "final_layer_norm"], False), "all_lora": (["all"], True)}
# post-step weights stored for these names (token rows: the used ids and one unused row are checked by the test)
SAMPLE = ["text_model.embeddings.token_embedding.weight", "text_model.embeddings.position_embedding.weight",
          "text_model.encoder.layers.0.self_attn.q_proj.weight", "text_model.encoder.layers.1.mlp.fc1.weight",
          "text_model.encoder.layers.1.mlp.fc2.bias", "text_model.encoder.layers.1.layer_norm2.weight",
          "text_model.final_layer_norm.weight", "text_model.final_layer_norm.bias"]
UNET_SAMPLE = ["down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_out.0.weight",
               "up_blocks.3.attentions.2.transformer_blocks.0.attn2.to_out.0.bias"]


# ---- reference train.py:316-337 (handle_trainable_modules), :205-236 (create_optimizer_params, param_optim), restated
def handle_trainable_modules(model, trainable_modules=None, is_enabled=True, negation=None):
    acc = []
    unfrozen_params = 0
    if trainable_modules is not None:
        unlock_all = any([name == "all" for name in trainable_modules])
        if unlock_all:
            model.requires_grad_(True)
            unfrozen_params = len(list(model.parameters()))
        else:
            model.requires_grad_(False)
            for name, param in model.named_parameters():
                for tm in trainable_modules:
                    if all([tm in name, name not in acc, "lora" not in name]):
                        param.requires_grad_(is_enabled)
                        acc.append(name)
                        unfrozen_params += 1
    return unfrozen_params


def param_optim(model, condition, extra_params=None, is_lora=False, negation=None):
    extra_params = extra_params if len(extra_params.keys()) > 0 else None
    return {"model": model, "condition": condition, "extra_params": extra_params, "is_lora": is_lora, "negation": negation}


def create_optim_params(name="param", params=None, lr=5e-6, extra_params=None):
    params = {"name": name, "params": params, "lr": lr}
    if extra_params is not None:
        for k, v in extra_params.items():
            params[k] = v
    return params


def create_optimizer_params(model_list, lr):
    optimizer_params = []
    for optim in model_list:
        model, condition, extra_params, is_lora, negation = optim.values()
        if is_lora and condition and isinstance(model, list):
            params = create_optim_params(params=itertools.chain(*model), extra_params=extra_params)
            optimizer_params.append(params)
            continue
        if is_lora and condition and not isinstance(model, list):
            for n, p in model.named_parameters():
                if "lora" in n:
                    optimizer_params.append(create_optim_params(n, p, lr, extra_params))
            continue
        if condition:
            for n, p in model.named_parameters():
                should_negate = "lora" in n and not is_lora
                if should_negate:
                    continue
                optimizer_params.append(create_optim_params(n, p, lr, extra_params))
    return optimizer_params
# ----


def case(ref, frames, trainable_text_modules, use_text_lora):
    from transformers import CLIPTextConfig, CLIPTextModel
    ids, nvocab = prompt_ids()
    te = CLIPTextModel(CLIPTextConfig(vocab_size=nvocab, **TEXT))
    te.load_state_dict({k: v for k, v in seeded_state_dict(te, SEEDS["text_base"]).items() if not k.endswith("position_ids")},
                       strict=False)
    unet = import_reference_unet()(**UNET)
    unet.load_state_dict(seeded_state_dict(unet, SEEDS["unet_base"]))
    # freeze_models (train.py:542), then handle_trainable_modules on the UNet (:603)
    te.requires_grad_(False)
    unet.requires_grad_(False)
    text_lora_params = None
    if use_text_lora:
        with contextlib.redirect_stdout(io.StringIO()):
            text_lora_params, _ = ref.inject_trainable_lora_extended(te, {"CLIPEncoderLayer"}, r=R_TEXT)
        seed_lora_(te, SEEDS["text_lora"])
    handle_trainable_modules(unet, TRAINABLE_MODULES)
    lr, extra = HYPER["lr"], HYPER["extra_unet_params"]
    # train.py:574-595 (extra_text_encoder_params = extra_unet_params)
    optim_params = [param_optim(unet, True, extra_params=extra),
                    param_optim(te, True, extra_params=extra),
                    param_optim(text_lora_params, use_text_lora, is_lora=True, extra_params={**{"lr": lr}, **extra})]
    params = create_optimizer_params(optim_params, lr)
    optimizer = torch.optim.AdamW(params, lr=lr, betas=HYPER["betas"], weight_decay=HYPER["weight_decay"], eps=HYPER["eps"])
    groups = [(g.get("name"), len(g["params"]), g["lr"], g.get("weight_decay")) for g in optimizer.param_groups]
    # train.py:768-773: on the first step, before the encoder runs
    handle_trainable_modules(te, trainable_text_modules)
    census = sorted(n for n, p in te.named_parameters() if p.requires_grad)
    te.eval()
    unet.eval()
    B = ids.shape[0]
    g = torch.Generator().manual_seed(23 + frames)
    latents = torch.randn(B, 4, frames, 16, 16, generator=g)
    noise = torch.randn(B, 4, frames, 16, 16, generator=g)
    timesteps = torch.tensor([211, 733])
    abar = L.ddpm_alphas_cumprod()
    noisy_latents = L.add_noise(latents, noise, timesteps, abar)
    target = noise
    encoder_hidden_states = te(ids)[0]
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
    # ---- train.py:863-879
    loss.backward()
    text_grads = {n: p.grad.detach().clone() for n, p in te.named_parameters() if p.grad is not None}
    unet_grads = {n: p.grad.detach().clone() for n, p in unet.named_parameters() if p.grad is not None}
    params_to_clip = list(unet.parameters()) + list(te.parameters())
    total_norm = torch.nn.utils.clip_grad_norm_(params_to_clip, HYPER["max_grad_norm"])
    optimizer.step()
    after = {n: p.detach().clone() for n, p in te.named_parameters() if n in SAMPLE or "lora" in n and "layers.1.mlp.fc1" in n}
    for n in UNET_SAMPLE:
        after["unet." + n] = unet.get_parameter(n).detach().clone()
    return dict(unet_cfg=UNET, text_cfg=dict(TEXT, vocab_size=nvocab), r_text=R_TEXT, seeds=SEEDS, hyper=HYPER,
                trainable_modules=TRAINABLE_MODULES, trainable_text_modules=trainable_text_modules, use_text_lora=use_text_lora,
                prompt_ids=ids, latents=latents, noise=noise, timesteps=timesteps, pass_losses=[x.detach() for x in losses],
                groups=groups, census=census, text_grads=text_grads, grad_norm=total_norm.item(),
                unet_grad_norms={n: v.norm().item() for n, v in unet_grads.items()},
                after=after,
                source="reference utils/lora.py on transformers.CLIPTextModel and the reference's models/*.py over "
                       "oracle/diffusers_standin; handle_trainable_modules, the optimizer groups, the step of train.py:803-834 "
                       "and the clip + AdamW of :863-879 restated; fp32 CPU, eval mode")


def main():
    torch.set_num_threads(8)
    ref = ref_lora()
    golden = os.path.join(ROOT, "tests", "golden")
    for name, (modules, lora) in CASES.items():
        for frames in (4, 1):
            path = os.path.join(golden, f"text_train_{name}_f{frames}.pt")
            torch.save(case(ref, frames, modules, lora), path)
            print(path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
