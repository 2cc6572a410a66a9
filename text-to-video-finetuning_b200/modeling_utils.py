"""Minimal stand-ins for the diffusers ModelMixin / ConfigMixin surface that train.py and the pipelines touch:
`.config`, `from_pretrained(path, subfolder=...)`, `save_pretrained(dir)`, `.dtype`, `.device` (diffusers-format
`config.json` + `diffusion_pytorch_model.safetensors|bin`).  diffusers itself is not a dependency."""
import functools
import inspect
import json
import os

import torch


class FrozenConfig(dict):
    """dict with attribute access (diffusers FrozenDict behaviour used as `model.config.in_channels`)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def register_to_config(init):
    """Record the constructor arguments as `self.config` (same contract as diffusers' decorator)."""
    sig = inspect.signature(init)

    @functools.wraps(init)
    def wrapper(self, *args, **kwargs):
        bound = sig.bind(self, *args, **kwargs)
        bound.apply_defaults()
        cfg = {k: v for k, v in bound.arguments.items() if k != "self"}
        cfg["_class_name"] = type(self).__name__
        self._internal_config = FrozenConfig(cfg)
        init(self, *args, **kwargs)

    return wrapper


class ConfigMixin:
    config_name = "config.json"

    @property
    def config(self):
        return self._internal_config


class ModelMixin(torch.nn.Module):
    weights_name = "diffusion_pytorch_model"

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def enable_xformers_memory_efficient_attention(self, *a, **k):  # train.py:162 - attention here is always fused
        pass

    def enable_gradient_checkpointing(self):
        self._set_gradient_checkpointing(True)

    def disable_gradient_checkpointing(self):
        self._set_gradient_checkpointing(False)

    @classmethod
    def from_pretrained(cls, pretrained_model_path, subfolder=None, torch_dtype=None, **unused):
        root = os.path.join(pretrained_model_path, subfolder) if subfolder else pretrained_model_path
        with open(os.path.join(root, cls.config_name)) as f:
            cfg = json.load(f)
        params = inspect.signature(cls.__init__).parameters
        model = cls(**{k: v for k, v in cfg.items() if k in params})
        st = os.path.join(root, cls.weights_name + ".safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(root, cls.weights_name + ".bin"), map_location="cpu")
        model.load_state_dict(sd, strict=True)
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model.eval()

    def save_pretrained(self, save_directory, safe_serialization=True, state_dict=None, **unused):
        """state_dict: written instead of self.state_dict() (as in diffusers)."""
        os.makedirs(save_directory, exist_ok=True)
        cfg = {k: (list(v) if isinstance(v, tuple) else v) for k, v in self.config.items()}
        with open(os.path.join(save_directory, self.config_name), "w") as f:
            json.dump(cfg, f, indent=2)
        sd = {k: v.detach().cpu().contiguous() for k, v in (self.state_dict() if state_dict is None else state_dict).items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(save_directory, self.weights_name + ".safetensors"))
        else:
            torch.save(sd, os.path.join(save_directory, self.weights_name + ".bin"))
