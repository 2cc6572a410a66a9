"""TEST ORACLE: an independent restatement of the loralib names the reference's stable_lora/lora.py imports (LoRALayer,
Linear, Conv2d, Embedding, mark_only_lora_as_trainable, lora_state_dict), so that the reference's unmodified stable_lora
code runs on a machine without loralib - as oracle/diffusers_standin does for diffusers.  Written from loralib's public
behaviour; parity with loralib itself is not pinned.  Never imported by the package."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


class LoRALayer:
    def __init__(self, r, lora_alpha, lora_dropout, merge_weights):
        self.r = r
        self.lora_alpha = lora_alpha
        self.lora_dropout = nn.Dropout(p=lora_dropout) if lora_dropout > 0.0 else (lambda x: x)
        self.merged = False
        self.merge_weights = merge_weights


class Linear(nn.Linear, LoRALayer):
    def __init__(self, in_features, out_features, r=0, lora_alpha=1, lora_dropout=0.0, fan_in_fan_out=False, merge_weights=True,
                 **kwargs):
        nn.Linear.__init__(self, in_features, out_features, **kwargs)
        LoRALayer.__init__(self, r=r, lora_alpha=lora_alpha, lora_dropout=lora_dropout, merge_weights=merge_weights)
        self.fan_in_fan_out = fan_in_fan_out
        if r > 0:
            self.lora_A = nn.Parameter(self.weight.new_zeros((r, in_features)))
            self.lora_B = nn.Parameter(self.weight.new_zeros((out_features, r)))
            self.scaling = self.lora_alpha / self.r
            self.weight.requires_grad = False
        self.reset_parameters()
        if fan_in_fan_out:
            self.weight.data = self.weight.data.transpose(0, 1)

    def reset_parameters(self):
        nn.Linear.reset_parameters(self)
        if hasattr(self, "lora_A"):
            nn.init.kaiming_uniform_(self.lora_A, a=math.sqrt(5))
            nn.init.zeros_(self.lora_B)

    def _w(self):
        return self.weight.transpose(0, 1) if self.fan_in_fan_out else self.weight

    def _delta(self):
        d = self.lora_B @ self.lora_A * self.scaling
        return d.transpose(0, 1) if self.fan_in_fan_out else d

    def train(self, mode=True):
        nn.Linear.train(self, mode)
        if self.merge_weights and self.r > 0:
            if mode and self.merged:
                self.weight.data -= self._delta()
                self.merged = False
            elif not mode and not self.merged:
                self.weight.data += self._delta()
                self.merged = True
        return self

    def forward(self, x):
        out = F.linear(x, self._w(), bias=self.bias)
        if self.r > 0 and not self.merged:
            out = out + (self.lora_dropout(x) @ self.lora_A.transpose(0, 1) @ self.lora_B.transpose(0, 1)) * self.scaling
        return out


class Conv2d(nn.Conv2d, LoRALayer):
    def __init__(self, in_channels, out_channels, kernel_size, r=0, lora_alpha=1, lora_dropout=0.0, merge_weights=True, **kwargs):
        nn.Conv2d.__init__(self, in_channels, out_channels, kernel_size, **kwargs)
        LoRALayer.__init__(self, r=r, lora_alpha=lora_alpha, lora_dropout=lora_dropout, merge_weights=merge_weights)
        if r > 0:
            self.lora_A = nn.Parameter(self.weight.new_zeros((r * kernel_size, in_channels * kernel_size)))
            self.lora_B = nn.Parameter(self.weight.new_zeros((out_channels * kernel_size, r * kernel_size)))
            self.scaling = self.lora_alpha / self.r
            self.weight.requires_grad = False
        self.reset_parameters()

    def reset_parameters(self):
        nn.Conv2d.reset_parameters(self)
        if hasattr(self, "lora_A"):
            nn.init.kaiming_uniform_(self.lora_A, a=math.sqrt(5))
            nn.init.zeros_(self.lora_B)

    def forward(self, x):
        if self.r > 0 and not self.merged:
            w = self.weight + (self.lora_B @ self.lora_A).view(self.weight.shape) * self.scaling
            return F.conv2d(x, w, self.bias, self.stride, self.padding, self.dilation, self.groups)
        return nn.Conv2d.forward(self, x)


class Embedding(nn.Embedding, LoRALayer):
    def __init__(self, num_embeddings, embedding_dim, r=0, lora_alpha=1, merge_weights=True, **kwargs):
        nn.Embedding.__init__(self, num_embeddings, embedding_dim, **kwargs)
        LoRALayer.__init__(self, r=r, lora_alpha=lora_alpha, lora_dropout=0, merge_weights=merge_weights)
        if r > 0:
            self.lora_A = nn.Parameter(self.weight.new_zeros((r, num_embeddings)))
            self.lora_B = nn.Parameter(self.weight.new_zeros((embedding_dim, r)))
            self.scaling = self.lora_alpha / self.r
            self.weight.requires_grad = False
        self.reset_parameters()

    def reset_parameters(self):
        nn.Embedding.reset_parameters(self)
        if hasattr(self, "lora_A"):
            nn.init.zeros_(self.lora_A)
            nn.init.normal_(self.lora_B)

    def forward(self, x):
        out = nn.Embedding.forward(self, x)
        if self.r > 0 and not self.merged:
            after_A = F.embedding(x, self.lora_A.transpose(0, 1), self.padding_idx, self.max_norm, self.norm_type,
                                  self.scale_grad_by_freq, self.sparse)
            out = out + (after_A @ self.lora_B.transpose(0, 1)) * self.scaling
        return out


def mark_only_lora_as_trainable(model, bias="none"):
    for n, p in model.named_parameters():
        if "lora_" not in n:
            p.requires_grad = False
    if bias == "none":
        return
    if bias == "all":
        for n, p in model.named_parameters():
            if "bias" in n:
                p.requires_grad = True
    elif bias == "lora_only":
        for m in model.modules():
            if isinstance(m, LoRALayer) and getattr(m, "bias", None) is not None:
                m.bias.requires_grad = True
    else:
        raise NotImplementedError(bias)


def lora_state_dict(model, bias="none"):
    sd = model.state_dict()
    if bias == "none":
        return {k: sd[k] for k in sd if "lora_" in k}
    if bias == "all":
        return {k: sd[k] for k in sd if "lora_" in k or "bias" in k}
    if bias == "lora_only":
        out = {}
        for k in sd:
            if "lora_" in k:
                out[k] = sd[k]
                b = k.split("lora_")[0] + "bias"
                if b in sd:
                    out[b] = sd[b]
        return out
    raise NotImplementedError(bias)
