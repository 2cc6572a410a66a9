"""LoraHandler - the facade train.py uses to add / save LoRA adapters (reference utils/lora_handler.py:69-351).

Same constructor keywords, `add_lora_to_model(...) -> (params, negation)`, `save_lora_weights(model, save_path, step)`,
`deactivate_lora_train`, `LORA_VERSIONS`, and both file layouts: cloneofsimo (`<save_path>/lora/<step>_unet.pt`) and
stable_lora (`<save_path>/lora/full_weights/<step>_lora_text_to_video_unet.safetensors`, plus the webui file
`<save_path>/lora/webui_<step>_lora_text_to_video.safetensors`).  'stable_lora' (the reference's default) runs on
utils/stable_lora.py; its UNet targets are Linear / Conv2d / Conv3d (the UNet has no nn.Embedding).

Deviations from the reference, both so that a mistake fails instead of training something else:
  * stable_lora `lora_path`: a file that is found but does not match the injected modules' keys and shapes raises
    ValueError (the reference prints the error and trains fresh weights);
  * injecting stable_lora into a model that already carries cloneofsimo wrappers raises NotImplementedError (the reference
    would wrap the wrappers' own inner layers).
`lora_bias` other than 'none' behaves as 'none' with a warning: the LoRA optimizer group only takes parameters whose name
contains 'lora' (train.create_optimizer_params), so in the reference too a bias is only ever updated through
`trainable_modules`, which sets its requires_grad itself.
"""
import os
import warnings
from types import SimpleNamespace

import torch

from . import stable_lora
from .lora import (extract_lora_ups_down, inject_trainable_lora_extended, monkeypatch_or_replace_lora_extended,
                   save_lora_weight, train_patch_pipe)

FILE_BASENAMES = ["unet", "text_encoder"]
LORA_FILE_TYPES = [".pt", ".safetensors"]
CLONE_OF_SIMO_KEYS = ["model", "loras", "target_replace_module", "r"]
STABLE_LORA_KEYS = ["model", "target_module", "search_class", "r", "dropout", "lora_bias"]

lora_versions = dict(stable_lora="stable_lora", cloneofsimo="cloneofsimo")
lora_func_types = dict(loader="loader", injector="injector")
lora_args = dict(model=None, loras=None, target_replace_module=[], target_module=[], r=4, search_class=[torch.nn.Linear],
                 dropout=0, lora_bias="none")

LoraVersions = SimpleNamespace(**lora_versions)
LoraFuncTypes = SimpleNamespace(**lora_func_types)
LORA_VERSIONS = [LoraVersions.stable_lora, LoraVersions.cloneofsimo]
LORA_FUNC_TYPES = [LoraFuncTypes.loader, LoraFuncTypes.injector]


def filter_dict(_dict, keys=()):
    return {k: v for k, v in _dict.items() if k in keys}


class LoraHandler(object):
    def __init__(self, version=LoraVersions.cloneofsimo, use_unet_lora=False, use_text_lora=False, save_for_webui=False,
                 only_for_webui=False, lora_bias="none", unet_replace_modules=["UNet3DConditionModel"],
                 text_encoder_replace_modules=["CLIPEncoderLayer"]):
        self.version = version
        self.lora_loader = self.get_lora_func(func_type=LoraFuncTypes.loader)
        self.lora_injector = self.get_lora_func(func_type=LoraFuncTypes.injector)
        self.lora_bias = lora_bias
        self.use_unet_lora = use_unet_lora
        self.use_text_lora = use_text_lora
        self.save_for_webui = save_for_webui
        self.only_for_webui = only_for_webui
        self.unet_replace_modules = unet_replace_modules
        self.text_encoder_replace_modules = text_encoder_replace_modules
        self.use_lora = any([use_text_lora, use_unet_lora])
        if self.use_lora:
            print(f"Using LoRA Version: {self.version}")

    def is_cloneofsimo_lora(self):
        return self.version == LoraVersions.cloneofsimo

    def is_stable_lora(self):
        return self.version == LoraVersions.stable_lora

    def get_lora_func(self, func_type=LoraFuncTypes.loader):
        if self.is_cloneofsimo_lora():
            return monkeypatch_or_replace_lora_extended if func_type == LoraFuncTypes.loader else inject_trainable_lora_extended
        if self.is_stable_lora():
            return stable_lora.load_lora if func_type == LoraFuncTypes.loader else stable_lora.add_lora_to
        raise ValueError(f"LoRA version {self.version!r} does not exist (choose from {LORA_VERSIONS})")

    def check_lora_ext(self, lora_file: str):
        return lora_file.endswith(tuple(LORA_FILE_TYPES))

    def get_lora_file_path(self, lora_path: str, model):
        """First file in `lora_path` with a LoRA extension whose name contains 'unet' / 'text_encoder'."""
        if lora_path and os.path.exists(lora_path):
            base = FILE_BASENAMES[0] if model.__class__.__name__ == "UNet3DConditionModel" else FILE_BASENAMES[1]
            for fn in os.listdir(lora_path):
                if self.check_lora_ext(fn) and base in fn:
                    return os.path.join(lora_path, fn)
        return None

    def get_lora_func_args(self, lora_path, use_lora, model, replace_modules, r, dropout, lora_bias):
        # cloneofsimo: only model / loras / target_replace_module / r are forwarded - the YAML dropout is dropped
        # (reference :171-178, hazard H13); the wrappers keep their class-default dropout.
        if self.is_cloneofsimo_lora():
            return dict(model=model, loras=self.get_lora_file_path(lora_path, model), target_replace_module=replace_modules, r=r)
        return dict(model=model, lora_path=lora_path)

    def load_lora(self, model, lora_path=""):
        """stable_lora: load the first LoRA file in `lora_path` whose name contains 'unet' (ValueError if it does not fit)."""
        lora_file = self.get_lora_file_path(lora_path, model)
        if lora_file is None:
            if lora_path:
                print(f"Could not load LoRAs for {model.__class__.__name__}. Injecting new ones instead...")
            return
        self.lora_loader(model, lora_file)
        print(f"Successfully loaded LoRA from: {lora_file}")

    def do_lora_injection(self, model, replace_modules, bias="none", dropout=0, r=4, lora_loader_args=None):
        if self.is_stable_lora():
            search = [torch.nn.Linear, torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.Embedding]
            self.lora_injector(model, target_module=replace_modules, search_class=search, r=r, dropout=dropout,
                               lora_bias=self.lora_bias)()
            return None, None, False
        params, negation = self.lora_injector(**lora_loader_args)
        for up, down in extract_lora_ups_down(model, target_replace_module=replace_modules):
            if up is not None and down is not None:
                print(f"Lora successfully injected into {model.__class__.__name__}.")
            break
        return params, negation, True

    def add_lora_to_model(self, use_lora, model, replace_modules, dropout=0.0, lora_path="", r=16):
        params, negation = None, None
        args = self.get_lora_func_args(lora_path, use_lora, model, replace_modules, r, dropout, self.lora_bias)
        if use_lora:
            params, negation, hybrid = self.do_lora_injection(model, replace_modules, bias=self.lora_bias, lora_loader_args=args,
                                                              dropout=dropout, r=r)
            if not hybrid:
                self.load_lora(model, lora_path=lora_path)
        params = model if params is None else params
        return params, negation

    def deactivate_lora_train(self, models, deactivate=True):
        """stable_lora: set the train/eval mode of the LoRA modules and of each model (reference set_mode_group, used
        around previews); a no-op for cloneofsimo."""
        if self.is_stable_lora():
            stable_lora.set_mode_group(models, not deactivate)

    def save_cloneofsimo_lora(self, model, save_path, step):
        for name, cond, mods, sub in ((FILE_BASENAMES[0], self.use_unet_lora, self.unet_replace_modules, "unet"),
                                      (FILE_BASENAMES[1], self.use_text_lora, self.text_encoder_replace_modules, "text_encoder")):
            if cond and mods is not None:
                save_lora_weight(getattr(model, sub), f"{save_path}/{step}_{name}.pt", mods)
        train_patch_pipe(model, self.use_unet_lora, self.use_text_lora)

    def save_lora_weights(self, model=None, save_path: str = "", step: str = ""):
        save_path = f"{save_path}/lora"
        os.makedirs(save_path, exist_ok=True)
        if self.is_cloneofsimo_lora():
            if any([self.save_for_webui, self.only_for_webui]):
                warnings.warn("'save_for_webui' is only supported by the 'stable_lora' implementation")
            self.save_cloneofsimo_lora(model, save_path, step)
        if self.is_stable_lora():
            self.save_stable_lora(model.unet, save_path, step)

    def save_stable_lora(self, unet, save_path, step, suffix=""):
        """fp32 full weights and/or the fp16 webui file (see module docstring); returns the paths written."""
        if self.lora_bias != "none":
            warnings.warn(f"lora_bias={self.lora_bias!r} behaves as 'none' (only the lora_A / lora_B tensors are saved)")
        return stable_lora.save_lora(unet, save_path, step, save_for_webui=self.save_for_webui, only_webui=self.only_for_webui,
                                     suffix=suffix)
