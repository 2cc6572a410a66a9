"""Generates tests/golden/stable_lora_*.pt / .json from the REFERENCE's own stable-LoRA code: $T2V_REFERENCE_ROOT/stable_lora/lora.py
imported unmodified over tests/loralib_standin (a restatement of the loralib names it imports), the reference's models/*.py over
oracle/diffusers_standin, and the reference's utils/convert_diffusers_to_original_ms_text_to_video.py.  fp32, CPU, eval mode:
    T2V_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_golden_stable_lora.py
  stable_lora_modules.pt      one wrapped layer per case: state, x, y, dy, dx and the gradients of lora_A / lora_B
  stable_lora_unet_small_f4.pt  the small UNet under add_lora_to(["UNet3DConditionModel"]): injection census, prediction, loss,
                                every LoRA gradient norm and the 24 largest LoRA gradients of at
                                most 2,048 elements
  stable_lora_webui_keys.json   the webui key and shape of every lora_A / lora_B key of the ms-1.7b UNet"""
import contextlib
import importlib.util
import io
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
STANDIN = os.path.join(ROOT, "tests", "loralib_standin")

from helpers import seeded_state_dict  # noqa: E402
from oracle import leaves as L  # noqa: E402
from oracle.reference_import import REFERENCE_ROOT, import_reference_unet  # noqa: E402

SMALL = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)
SEARCH = [nn.Linear, nn.Conv2d, nn.Conv3d, nn.Embedding]


def _load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REFERENCE_ROOT, rel))
    mod = importlib.util.module_from_spec(spec)
    with contextlib.redirect_stdout(io.StringIO()):
        spec.loader.exec_module(mod)
    return mod


def ref_stable_lora():
    if STANDIN not in sys.path:
        sys.path.insert(0, STANDIN)
    return _load("_t2v_ref_stable_lora", os.path.join("stable_lora", "lora.py"))


def seed_lora_(module, seed):
    """Deterministic non-trivial LoRA weights (lora_B is zero-initialised by the reference)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in sorted(module.named_parameters()):
            if n.endswith("lora_B"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.05)
            elif n.endswith("lora_A"):
                p.copy_(torch.randn(p.shape, generator=g) / p.shape[1] ** 0.5)


class Target(nn.Module):
    def __init__(self, layer):
        super().__init__()
        self.layer = layer


MODULE_SPECS = {   # name: (layer, r, input shape); sizes kept small so the fixture stays a small file
    "linear": (lambda: nn.Linear(64, 96, bias=True), 16, (1, 24, 64)),
    "linear_nobias_r4": (lambda: nn.Linear(48, 40, bias=False), 4, (2, 10, 48)),
    "conv2d": (lambda: nn.Conv2d(16, 24, 3, padding=1), 16, (1, 16, 8, 8)),
    "conv2d_s2": (lambda: nn.Conv2d(16, 16, 3, stride=2, padding=1), 8, (1, 16, 8, 8)),
    "conv2d_1x1": (lambda: nn.Conv2d(24, 16, 1), 4, (1, 24, 6, 6)),
    "conv3d": (lambda: nn.Conv3d(16, 24, (3, 1, 1), padding=(1, 0, 0)), 12, (1, 16, 4, 4, 4)),
}


def module_cases(ref):
    g = torch.Generator().manual_seed(200)
    out = {}
    for name, (ctor, r, xshape) in MODULE_SPECS.items():
        torch.manual_seed(9)
        t = Target(ctor())
        with torch.no_grad():
            for n, p in t.named_parameters():
                p.copy_(torch.randn(p.shape, generator=g) / max(1, p[0].numel()) ** 0.5 if p.dim() > 1 else torch.randn(p.shape, generator=g) * 0.05)
        with contextlib.redirect_stdout(io.StringIO()):
            ref.add_lora_to(t, target_module=["Target"], search_class=SEARCH, r=r, dropout=0.1)()
        m = t.layer
        seed_lora_(m, 300 + len(out))
        m.eval()   # eval: the Linear input dropout is the identity (its mask is a torch RNG draw, not reproducible elsewhere)
        x = torch.randn(xshape, generator=g, requires_grad=True)
        y = m(x)
        dy = torch.randn(y.shape, generator=g)
        y.backward(dy)
        out[name] = dict(kind=type(m).__name__, r=r, scaling=float(m.scaling), stride=tuple(getattr(m, "stride", (1,))),
                         padding=tuple(getattr(m, "padding", (0,))), state={k: v.detach().clone() for k, v in m.state_dict().items()},
                         x=x.detach().clone(), y=y.detach().clone(), dy=dy, dx=x.grad.clone(),
                         grads={n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None})
    return out


def model_case(ref):
    Ref = import_reference_unet()
    m = Ref(**SMALL)
    sd = seeded_state_dict(m, 0)
    m.load_state_dict(sd)
    with contextlib.redirect_stdout(io.StringIO()):
        ref.add_lora_to(m, target_module=["UNet3DConditionModel"], search_class=SEARCH, r=8, dropout=0.1)()
    seed_lora_(m, 21)
    m.eval()
    wrapped = sorted((n, type(x).__name__) for n, x in m.named_modules() if hasattr(x, "lora_A"))
    shapes = {n: tuple(p.shape) for n, p in m.named_parameters() if "lora_" in n}
    trainable = sorted(n for n, p in m.named_parameters() if p.requires_grad)
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(1, 4, 4, 16, 16, generator=g)
    noise = torch.randn(1, 4, 4, 16, 16, generator=g)
    t = torch.tensor([437])
    ehs = torch.randn(1, 7, 64, generator=g)
    noisy = L.add_noise(lat, noise, t, L.ddpm_alphas_cumprod())
    pred = m(noisy, t, encoder_hidden_states=ehs).sample
    loss = torch.nn.functional.mse_loss(pred.float(), noise.float())
    loss.backward()
    grads = {n: p.grad for n, p in m.named_parameters() if "lora_" in n and p.grad is not None}
    # the 24 largest gradients among tensors of at most 2,048 elements (every gradient norm is kept as well)
    keep = sorted((n for n in grads if grads[n].numel() <= 2048), key=lambda n: -grads[n].norm().item())[:24]
    return dict(cfg=SMALL, r=8, lora_seed=21, base_seed=0, latents=lat, noise=noise, timesteps=t, text=ehs, pred=pred.detach(),
                loss=loss.detach(), wrapped=wrapped, shapes=shapes, trainable=trainable,
                grad_norms={n: v.norm().item() for n, v in grads.items()}, grads={n: grads[n].detach().clone() for n in keep},
                n_lora=len(grads), source="reference stable_lora/lora.py (add_lora_to) over tests/loralib_standin on the reference's "
                                          "models/*.py over oracle/diffusers_standin, fp32 CPU")


def webui_keys(ref):
    conv = _load("_t2v_ref_convert", os.path.join("utils", "convert_diffusers_to_original_ms_text_to_video.py"))
    Ref = import_reference_unet()
    with torch.device("meta"):
        m = Ref()
    with contextlib.redirect_stdout(io.StringIO()):
        ref.add_lora_to(m, target_module=["UNet3DConditionModel"], search_class=SEARCH, r=16, dropout=0.1)()
    sd = {k: v for k, v in m.state_dict().items() if "lora_" in k}
    with contextlib.redirect_stdout(io.StringIO()):
        new = conv.convert_unet_state_dict(dict(sd), strict_mapping=True)
    # the converter builds {new_key: tensor} by iterating {old_key: new_key} in the input's key order, so the two orders pair up
    by_new_shape = {k: tuple(v.shape) for k, v in new.items()}
    pairs = []
    mapping_new = list(new.keys())
    assert len(mapping_new) == len(sd), "converter merged keys"
    for old, new_key in zip(sd.keys(), mapping_new):   # dict order is preserved by the converter's comprehension
        pairs.append(dict(key=old, webui_key=new_key, shape=list(sd[old].shape), webui_shape=list(by_new_shape[new_key])))
    return dict(config="UNet3DConditionModel defaults (ms-1.7b)", r=16, keys=pairs,
                source="reference utils/convert_diffusers_to_original_ms_text_to_video.py convert_unet_state_dict(strict_mapping=True) "
                       "over the lora_A / lora_B keys of reference add_lora_to on the reference UNet")


def main():
    torch.set_num_threads(8)
    ref = ref_stable_lora()
    path = os.path.join(GOLD, "stable_lora_modules.pt")
    torch.save(module_cases(ref), path)
    print("stable_lora_modules", os.path.getsize(path) // 1024, "KiB")
    path = os.path.join(GOLD, "stable_lora_unet_small_f4.pt")
    torch.save(model_case(ref), path)
    print("stable_lora_unet_small_f4", os.path.getsize(path) // 1024, "KiB")
    path = os.path.join(GOLD, "stable_lora_webui_keys.json")
    with open(path, "w") as f:
        json.dump(webui_keys(ref), f, indent=0)
    print("stable_lora_webui_keys", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
