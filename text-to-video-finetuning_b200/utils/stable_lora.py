"""Stable LoRA (the reference's `lora_version: stable_lora`, built on loralib) for the H100-native UNet.

The modules have loralib's attribute surface (`r`, `lora_alpha`, `scaling`, `lora_dropout`, `merge_weights`, `merged`,
`lora_A`, `lora_B`, `weight`, `bias`) and state-dict keys (`<name>.weight`, `<name>.bias`, `<name>.lora_A`, `<name>.lora_B`),
so checkpoints move between this build and the reference.  What differs is the forward pass:

    Linear   y = x W^T + b + scaling * (dropout(x) A^T) B^T     base GEMM, then down and up GEMMs on the same sm_90a kernel;
                                                                scaling and "+ base" ride in the up-projection's epilogue
    Conv2d   y = conv(x, W + scaling * view(B @ A))             ops.DeltaWeight: the delta is merged on the GPU
    Conv3d   y = conv3d(x, W + scaling * mean3(view(B @ A)))    (lora_delta.cu) and the conv stays ONE GEMM

`add_lora_to` wraps every exact nn.Linear / nn.Conv2d / nn.Conv3d below a module whose class name is a target, in place and
under the same attribute name; the wrapped module shares the original `weight` / `bias` Parameters.  lora_alpha = r, so
scaling = 1; merge_weights is False, so nothing is ever merged into the stored weights.
"""
import math
import os
import uuid
import warnings

import torch
import torch.nn as nn

from .. import ops

UNET_REPLACE = ["Transformer2DModel", "ResnetBlock2D"]
WEBUI_METADATA_KEY = "stable_lora_text_to_video"


class LoRALayer:
    """State shared by the three module kinds (loralib.LoRALayer)."""

    def _lora_init(self, r, lora_alpha, lora_dropout, merge_weights):
        self.r = r
        self.lora_alpha = lora_alpha
        self.lora_dropout = nn.Dropout(lora_dropout) if lora_dropout > 0 else nn.Identity()
        self.merged = False
        self.merge_weights = merge_weights
        self.scaling = self.lora_alpha / self.r

    def _reset_lora(self):
        nn.init.kaiming_uniform_(self.lora_A, a=math.sqrt(5))
        nn.init.zeros_(self.lora_B)

    def _dropout_p(self):
        d = self.lora_dropout
        return d.p if (self.training and isinstance(d, nn.Dropout)) else 0.0


class Linear(nn.Linear, LoRALayer):
    """A (r, in) kaiming-uniform, B (out, r) zeros; the dropout acts on the input of the low-rank branch only."""

    def __init__(self, in_features, out_features, r=0, lora_alpha=1, lora_dropout=0.0, merge_weights=False, bias=True, **kwargs):
        if r <= 0:
            raise ValueError("stable LoRA needs r > 0")
        nn.Linear.__init__(self, in_features, out_features, bias=bias, **kwargs)
        self._lora_init(r, lora_alpha, lora_dropout, merge_weights)
        self.lora_A = nn.Parameter(self.weight.new_zeros((r, in_features)))
        self.lora_B = nn.Parameter(self.weight.new_zeros((out_features, r)))
        self.weight.requires_grad = False
        self._reset_lora()

    def delta(self):
        return self.lora_B @ self.lora_A * self.scaling

    def forward(self, x):
        return stable_linear_forward(self, x)


def _cl(t):
    """Channels-last storage for conv weights: their memory then IS the [Cout, KH, KW, Cin] kernel layout."""
    return t.contiguous(memory_format=torch.channels_last if t.dim() == 4 else torch.channels_last_3d)


class Conv2d(nn.Conv2d, LoRALayer):
    """Square kernel k: A (r*k, in*k), B (out*k, r*k); W_eff = W + scaling * (B @ A).view(out, in, k, k).  No dropout."""

    def __init__(self, in_channels, out_channels, kernel_size, r=0, lora_alpha=1, lora_dropout=0.0, merge_weights=False, **kwargs):
        if r <= 0 or not isinstance(kernel_size, int):
            raise ValueError("stable LoRA Conv2d needs r > 0 and an int kernel size")
        nn.Conv2d.__init__(self, in_channels, out_channels, kernel_size, **kwargs)
        self._lora_init(r, lora_alpha, lora_dropout, merge_weights)
        k = kernel_size
        self.weight.data = _cl(self.weight.data)
        self.lora_A = nn.Parameter(self.weight.new_zeros((r * k, in_channels * k)))
        self.lora_B = nn.Parameter(self.weight.new_zeros((out_channels * k, r * k)))
        self.weight.requires_grad = False
        self._reset_lora()

    def delta(self):
        return (self.lora_B @ self.lora_A).view(self.weight.shape) * self.scaling

    def forward(self, x):
        return stable_conv_forward(self, x)


class Conv3d(nn.Conv3d, LoRALayer):
    """Kernel (k, 1, 1) with k = 3: A (3r, 3*in), B (3*out, 3r); the (out, in, 3, 3, 1) view of B @ A is averaged over its
    fourth axis into the (out, in, 3, 1, 1) delta.  No dropout."""

    def __init__(self, in_channels, out_channels, kernel_size, r=0, lora_alpha=1, lora_dropout=0.0, merge_weights=False, **kwargs):
        if r <= 0 or kernel_size != 3:
            raise ValueError("stable LoRA Conv3d needs r > 0 and a (3, 1, 1) kernel")
        nn.Conv3d.__init__(self, in_channels, out_channels, (kernel_size, 1, 1), **kwargs)
        self._lora_init(r, lora_alpha, lora_dropout, merge_weights)
        self.weight.data = _cl(self.weight.data)
        self.view_shape = (out_channels, in_channels, kernel_size, kernel_size, 1)
        self.force_disable_merge = True
        self.lora_A = nn.Parameter(self.weight.new_zeros((r * kernel_size, in_channels * kernel_size)))
        self.lora_B = nn.Parameter(self.weight.new_zeros((out_channels * kernel_size, r * kernel_size)))
        self.weight.requires_grad = False
        self._reset_lora()

    def delta(self):
        return torch.mean((self.lora_B @ self.lora_A).view(self.view_shape), dim=-2, keepdim=True) * self.scaling

    def forward(self, x):
        return stable_conv_forward(self, x, pads=(1, 1, 0, 0))


MODULES = (Linear, Conv2d, Conv3d)


# ------------------------------------------------------------------------------------------------ forward paths
def stable_linear_forward(m, x, residual=None, out_fp32=False, stats_rows=0):
    """x [rows, in] -> [rows, out]: base GEMM (+ residual), then x -> dropout -> A -> B with alpha = scaling and the base
    output as the up-projection's residual (GroupNorm statistics from that last epilogue)."""
    if out_fp32:  # only the per-clip time_emb_proj rows ask for fp32: widen the bf16 result (a [B, C] tensor)
        return stable_linear_forward(m, x, residual, False).float()
    x1, x2 = ops.fork(x)
    base = ops.linear(x1, m.weight, m.bias, residual)
    p = m._dropout_p()
    if p > 0:
        x2 = ops.dropout(x2, p)
    z = ops.linear(x2, m.lora_A)
    return ops.linear(z, m.lora_B, None, base, alpha=m.scaling, stats_rows=stats_rows)


def stable_conv_forward(m, x, rowbias=None, residual=None, stride=None, pads=None, rb_div=1, cin_pad=0, cout_pad=0, stats_rows=0):
    if stride is None:
        stride = m.stride[0]
    if pads is None:
        p = m.padding
        pads = (p[0], p[0], p[1], p[1]) if len(p) == 2 else (p[0], p[0], 0, 0)
    w = ops.DeltaWeight(m.weight, m.lora_A, m.lora_B, m.scaling, conv3d=isinstance(m, Conv3d))
    return ops.conv(x, w, m.bias, rowbias, residual, stride, pads, rb_div, False, cin_pad, cout_pad, stats_rows=stats_rows)


# ------------------------------------------------------------------------------------------------ injection
def _wrap(child, r, dropout):
    """The stable module for an exact nn.Linear / nn.Conv2d / nn.Conv3d, sharing its weight and bias (None otherwise)."""
    has_bias = child.bias is not None
    cls = type(child)
    if cls is nn.Linear:
        w = Linear(child.in_features, child.out_features, r=r, lora_alpha=r, lora_dropout=dropout, bias=has_bias,
                   device=child.weight.device)
    elif cls is nn.Conv2d:
        if child.kernel_size[0] != child.kernel_size[1] or child.groups != 1 or child.dilation != (1, 1):
            return None
        w = Conv2d(child.in_channels, child.out_channels, child.kernel_size[0], r=r, lora_alpha=r, lora_dropout=dropout,
                   stride=child.stride, padding=child.padding, bias=has_bias, device=child.weight.device)
    elif cls is nn.Conv3d:
        if tuple(child.kernel_size) != (3, 1, 1):
            return None
        w = Conv3d(child.in_channels, child.out_channels, 3, r=r, lora_alpha=r, lora_dropout=dropout, stride=child.stride,
                   padding=child.padding, bias=has_bias, device=child.weight.device)
    else:
        return None
    w.weight = child.weight
    if has_bias:
        w.bias = child.bias
    w.lora_A.data = w.lora_A.data.to(child.weight.dtype)
    w.lora_B.data = w.lora_B.data.to(child.weight.dtype)
    w.train(child.training)
    return w


def _targets(model, target_module, search_class):
    """(parent, name, child) for every `search_class` instance below a module whose class name is in target_module."""
    found, seen = [], set()
    for anc in model.modules():
        if anc.__class__.__name__ not in target_module:
            continue
        for fullname, mod in anc.named_modules():
            if not isinstance(mod, tuple(search_class)) or isinstance(mod, MODULES) or id(mod) in seen:
                continue
            *path, name = fullname.split(".")
            parent = anc.get_submodule(".".join(path)) if path else anc
            if isinstance(parent, MODULES):
                continue
            seen.add(id(mod))
            found.append((parent, name, mod))
    return found


def add_lora_to(model, target_module=UNET_REPLACE, search_class=(nn.Linear,), r=32, dropout=0, lora_bias="none"):
    """Wrap every nn.Linear / nn.Conv2d / nn.Conv3d below `target_module` in place; returns the unfreeze callable
    (`activate_lora_train`), as the reference does."""
    from .lora import _WRAPPERS
    if any(isinstance(mod, _WRAPPERS) for mod in model.modules()):
        raise NotImplementedError("this model already carries cloneofsimo LoRA wrappers; stable_lora cannot be injected on top "
                                  "of them (use one lora_version per model)")
    if any(c is nn.Embedding for c in search_class) and any(type(mod) is nn.Embedding for mod in model.modules()):
        raise NotImplementedError("stable LoRA on nn.Embedding (text-encoder targets) is not built")
    for parent, name, child in _targets(model, set(target_module), search_class):
        w = _wrap(child, r, dropout)
        if w is not None:
            parent._modules[name] = w
    return activate_lora_train(model, lora_bias)


def mark_only_lora_as_trainable(model, bias="none"):
    """requires_grad only for parameters whose name contains 'lora_'.  `bias` other than 'none' is accepted and behaves
    as 'none' (see lora_handler.LoraHandler)."""
    if bias != "none":
        warnings.warn(f"lora_bias={bias!r} behaves as 'none': the LoRA optimizer group only takes parameters named 'lora' "
                      "(use trainable_modules to train biases)")
    for n, p in model.named_parameters():
        p.requires_grad_("lora_" in n)


def activate_lora_train(model, bias):
    def unfreeze():
        print(model.__class__.__name__ + " LoRA set for training.")
        return mark_only_lora_as_trainable(model, bias=bias)
    return unfreeze


def set_mode(model, train=False):
    for m in model.modules():
        if hasattr(m, "merged"):
            m.train(train)


def set_mode_group(models, train):
    for model in models:
        set_mode(model, train)
        model.train(train)


# ------------------------------------------------------------------------------------------------ state dicts and files
def lora_state_dict(model, bias="none"):
    """fp32 CPU copies of every '<name>.lora_A' / '<name>.lora_B' tensor (loralib.lora_state_dict with bias='none')."""
    return {k: v.detach().to("cpu", torch.float32).contiguous() for k, v in model.state_dict().items() if "lora_" in k}


def merged_state_dict(model):
    """The plain state dict (no LoRA keys) with every wrapped weight replaced by W + delta, in fp32 on the CPU: what a plain
    UNet loads with strict=True."""
    sd = {k: v.detach().cpu().contiguous() for k, v in model.state_dict().items() if "lora_" not in k}
    with torch.no_grad():
        for name, m in model.named_modules():
            if isinstance(m, MODULES):
                w = m.weight.detach().float().cpu()
                d = m.delta().detach().float().cpu() if isinstance(m, Linear) else _delta_cpu(m)
                sd[f"{name}.weight" if name else "weight"] = (w + d.reshape(w.shape)).contiguous()
    return sd


def _delta_cpu(m):
    A, B = m.lora_A.detach().float().cpu(), m.lora_B.detach().float().cpu()
    ba = B @ A
    if isinstance(m, Conv3d):
        return torch.mean(ba.view(m.view_shape), dim=-2, keepdim=True) * m.scaling
    return ba.view(m.weight.shape) * m.scaling


# The reference's webui export renames the diffusers UNet keys to the ModelScope (CompVis) layout with
# convert_unet_state_dict(strict_mapping=True).  The LoRA keys only ever go through the block-prefix renames below; the
# stem renames of that converter match '.weight' / '.bias' keys only, so under strict mapping they leave LoRA keys alone.
_RESNET_RENAMES = [("norm1", "in_layers.0"), ("conv1", "in_layers.2"), ("norm2", "out_layers.0"), ("conv2", "out_layers.3"),
                   ("time_emb_proj", "emb_layers.1"), ("conv_shortcut", "skip_connection")]


def _block_renames():
    """(diffusers prefix, ModelScope prefix) pairs, in the order they are applied."""
    out = [("transformer_in", "input_blocks.0.1")]
    for i in range(4):
        for j in range(2):
            n = 3 * i + j + 1
            out.append((f"down_blocks.{i}.resnets.{j}.", f"input_blocks.{n}.0."))
            if i < 3:
                out.append((f"down_blocks.{i}.attentions.{j}.", f"input_blocks.{n}.1."))
            out.append((f"down_blocks.{i}.temp_convs.{j}.", f"input_blocks.{n}.0.temopral_conv."))
            if i < 3:
                out.append((f"down_blocks.{i}.temp_attentions.{j}.", f"input_blocks.{n}.2."))
        for j in range(3):
            n = 3 * i + j
            out.append((f"up_blocks.{i}.resnets.{j}.", f"output_blocks.{n}.0."))
            if i > 0:
                out.append((f"up_blocks.{i}.attentions.{j}.", f"output_blocks.{n}.1."))
            out.append((f"up_blocks.{i}.temp_convs.{j}.", f"output_blocks.{n}.0.temopral_conv."))
            if i > 0:
                out.append((f"up_blocks.{i}.temp_attentions.{j}.", f"output_blocks.{n}.2."))
        if i < 3:
            out.append((f"down_blocks.{i}.downsamplers.0.conv.", f"input_blocks.{3 * (i + 1)}.op."))
            out.append((f"up_blocks.{i}.upsamplers.0.", f"output_blocks.{3 * i + 2}.{1 if i == 0 else 3}."))
    out.append(("mid_block.attentions.0.", "middle_block.1."))
    for j in range(2):
        out.append((f"mid_block.resnets.{j}.", f"middle_block.{3 * j}."))
    out.append(("mid_block.temp_attentions.0.", "middle_block.2."))
    for j in range(2):
        out.append((f"mid_block.temp_convs.{j}.", f"middle_block.{3 * j}.temopral_conv."))
    return out


_BLOCK_RENAMES = _block_renames()


def webui_key(key):
    """(ModelScope key, unsqueeze) for one diffusers LoRA key: the webui name and whether the tensor gains a trailing unit
    axis (every non-bias key containing 'proj_', as the converter does)."""
    v = key
    if "resnets" in key:
        for hf, ms in _RESNET_RENAMES:
            v = v.replace(hf, ms)
    for hf, ms in _BLOCK_RENAMES:
        v = v.replace(hf, ms)
    return v, ("proj_" in key and "bias" not in key)


def webui_state_dict(lora_sd):
    out = {}
    for k, t in lora_sd.items():
        name, unsq = webui_key(k)
        out[name] = (t.unsqueeze(-1) if unsq else t).to(torch.float16).contiguous()
    return out


def save_lora(unet, output_dir, step, name="lora_text_to_video", save_for_webui=False, only_webui=False, suffix=""):
    """`<output_dir>/full_weights/<step>_<name>_unet<suffix>.safetensors` (fp32 LoRA state dict) unless only_webui, and with
    save_for_webui / only_webui `<output_dir>/webui_<step>_<name><suffix>.safetensors` (fp16, ModelScope keys).  Returns
    the paths written."""
    from safetensors.torch import save_file
    sd = lora_state_dict(unet)
    written = []
    if not only_webui:
        os.makedirs(os.path.join(output_dir, "full_weights"), exist_ok=True)
        path = os.path.join(output_dir, "full_weights", f"{step}_{name}_unet{suffix}.safetensors")
        save_file(sd, path)
        written.append(path)
    if save_for_webui or only_webui:
        meta = {WEBUI_METADATA_KEY: "v1", "lora_name": name + "_" + uuid.uuid4().hex.lower()[:5]}
        path = os.path.join(output_dir, f"webui_{step}_{name}{suffix}.safetensors")
        save_file(webui_state_dict(sd), path, metadata=meta)
        written.append(path)
    return written


def load_lora(model, lora_path):
    """Load a full-weights file into the injected modules.  Unlike the reference (which prints and continues), a file whose
    keys or shapes do not match the injected LoRA tensors raises ValueError instead of training fresh weights silently."""
    from safetensors.torch import load_file
    try:
        sd = load_file(lora_path)
    except Exception as e:   # not a safetensors file (e.g. a cloneofsimo .pt list)
        raise ValueError(f"{lora_path}: not a stable LoRA safetensors file ({e})") from e
    own = {k: v for k, v in model.state_dict().items() if "lora_" in k}
    if set(sd) != set(own):
        missing, extra = sorted(set(own) - set(sd)), sorted(set(sd) - set(own))
        raise ValueError(f"{lora_path} does not match the injected LoRA modules: {len(missing)} missing keys "
                         f"{missing[:3]}, {len(extra)} unexpected keys {extra[:3]}")
    bad = [k for k in sd if tuple(sd[k].shape) != tuple(own[k].shape)]
    if bad:
        raise ValueError(f"{lora_path}: shape mismatch for {bad[:3]} (file {tuple(sd[bad[0]].shape)}, model {tuple(own[bad[0]].shape)})")
    params = dict(model.named_parameters())
    with torch.no_grad():
        for k, v in sd.items():
            params[k].copy_(v.to(params[k].dtype))
