"""CLIP text encoder on the H100-native kernels - SURVEY 8(f) row 2 (`text_encoder(token_ids)[0]`, train.py:784-790).

Drop-in for the `transformers.CLIPTextModel` the reference loads with `CLIPTextModel.from_pretrained(path,
subfolder="text_encoder")` (train.py:120): same parameter names and module class names (a Hugging Face checkpoint loads
unchanged, and LoRA injection finds `CLIPEncoderLayer` / `CLIPAttention` / `CLIPMLP` by class name as it does on the
transformers model), same call `model(input_ids)[0]` -> last_hidden_state (B, L, hidden).

Frozen encoder (no LoRA injected): a no-grad forward.  Per layer: LayerNorm -> fused Q|K|V GEMM (weights concatenated once)
-> causal attention (two batched wgmma GEMMs around the row-softmax kernel with the causal mask; L = 77 makes this
launch-bound, not worth a fused kernel) -> output projection with the residual in the GEMM epilogue -> LayerNorm -> fc1 ->
GELU -> fc2 (+ residual epilogue).  Embedding lookup (token + position) is one kernel; final LayerNorm as in
CLIPTextTransformer.

Encoder that trains (cloneofsimo LoRA wrappers, `use_text_lora`, train.py:571-572; and/or unfrozen parameters,
`train_text_encoder` with `trainable_text_modules`, train.py:579-595): `encode` runs the same layers as autograd ops (ops.py),
each projection through its wrapper (utils/lora.lora_linear_forward) or as a plain linear, so every trainable tensor - LoRA
factors, projection weights and biases, LayerNorm affines, token and position embeddings - gets its gradient, and the eval
forward (`forward`, then `encode` without a tape) reads the current weights.  A trainable projection weight is read through
its parameter-arena shadow (ops.weight_bf16), which the fused optimizer rewrites every step; a frozen one is cast to bf16
once (`_t2v_shadow`).  Embeddings: with LoRA only, no embedding gradient is formed (the tables are frozen)."""
import json
import os
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops, prims


class CLIPAttention(nn.Module):
    def __init__(self, C):
        super().__init__()
        # transformers' registration order: LoRA files list the wrapped projections in module order
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(C, C) for _ in range(4))


class CLIPMLP(nn.Module):
    def __init__(self, C, I):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(C, I), nn.Linear(I, C)


class CLIPEncoderLayer(nn.Module):
    def __init__(self, C, I, eps):
        super().__init__()
        self.self_attn = CLIPAttention(C)
        self.layer_norm1 = nn.LayerNorm(C, eps=eps)
        self.mlp = CLIPMLP(C, I)
        self.layer_norm2 = nn.LayerNorm(C, eps=eps)


class CLIPTextEmbeddings(nn.Module):
    def __init__(self, vocab, positions, C):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, C)
        self.position_embedding = nn.Embedding(positions, C)
        for e in (self.token_embedding, self.position_embedding):
            e.weight._t2v_lookup = True   # gathered in fp32 by embed_tokens: the parameter arena keeps no bf16 copy of it


class CLIPEncoder(nn.Module):
    def __init__(self, n, C, I, eps):
        super().__init__()
        self.layers = nn.ModuleList([CLIPEncoderLayer(C, I, eps) for _ in range(n)])


class CLIPTextTransformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.embeddings = CLIPTextEmbeddings(cfg.vocab_size, cfg.max_position_embeddings, cfg.hidden_size)
        self.encoder = CLIPEncoder(cfg.num_hidden_layers, cfg.hidden_size, cfg.intermediate_size, cfg.layer_norm_eps)
        self.final_layer_norm = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)


DEFAULTS = dict(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23, num_attention_heads=16,
                max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5)   # the OpenCLIP ViT-H text tower of ms-1.7b


class CLIPTextModel(nn.Module):
    def __init__(self, config=None, **kwargs):
        super().__init__()
        cfg = dict(DEFAULTS)
        cfg.update(config if isinstance(config, dict) else (vars(config) if config is not None else {}))
        cfg.update(kwargs)
        self.config = SimpleNamespace(**{k: cfg[k] for k in DEFAULTS})
        if self.config.hidden_act not in ("gelu", "quick_gelu"):
            raise NotImplementedError(f"hidden_act {self.config.hidden_act!r}")
        if self.config.hidden_size % self.config.num_attention_heads or self.config.hidden_size % 8:
            raise ValueError("hidden_size must be a multiple of the head count and of 8")
        self.text_model = CLIPTextTransformer(self.config)
        self.requires_grad_(False)
        self._packed = None

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **unused):
        root = os.path.join(path, subfolder) if subfolder else path
        with open(os.path.join(root, "config.json")) as f:
            raw = json.load(f)
        model = cls({k: raw[k] for k in DEFAULTS if k in raw})
        st = os.path.join(root, "model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(root, "pytorch_model.bin"), map_location="cpu")
        sd = {k: v for k, v in sd.items() if not k.endswith("position_ids")}
        model.load_state_dict(sd)
        return model

    def load_state_dict(self, state_dict, strict=True):
        self._packed = None
        for p in self.parameters():
            p.__dict__.pop("_t2v_shadow", None)
        return super().load_state_dict(state_dict, strict=strict)

    @property
    def dtype(self):
        return torch.float32

    def _pack(self, device):
        """bf16 kernel-layout copies of the frozen weights, with q|k|v concatenated (one GEMM per layer instead of three)."""
        if self._packed is not None and self._packed["device"] == device:
            return self._packed
        bf = lambda w: prims.cast_f32_bf16(w.detach().float().contiguous()).view(w.shape[0], 1, 1, w.shape[1])  # noqa: E731
        layers = []
        for lyr in self.text_model.encoder.layers:
            a = lyr.self_attn
            layers.append(dict(
                qkv_w=bf(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)),
                qkv_b=torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0).detach().float().contiguous(),
                out_w=bf(a.out_proj.weight), out_b=a.out_proj.bias.detach().float().contiguous(),
                fc1_w=bf(lyr.mlp.fc1.weight), fc1_b=lyr.mlp.fc1.bias.detach().float().contiguous(),
                fc2_w=bf(lyr.mlp.fc2.weight), fc2_b=lyr.mlp.fc2.bias.detach().float().contiguous()))
        self._packed = dict(device=device, layers=layers)
        return self._packed

    def lora_injected(self):
        from .utils.lora import _WRAPPERS
        return any(isinstance(m, _WRAPPERS) for m in self.modules())

    def trains(self):
        """True when LoRA is injected or any parameter trains: the weights may then change, and `forward` runs `encode`."""
        return self.lora_injected() or any(p.requires_grad for p in self.parameters())

    def base_trains(self):
        """True when a parameter of the encoder itself (not a LoRA factor) trains (`train_text_encoder`)."""
        return any(p.requires_grad for n, p in self.named_parameters() if "lora" not in n)

    def forward(self, input_ids, attention_mask=None, **unused):
        """input_ids (B, L) int64 -> (last_hidden_state (B, L, hidden) fp32,).  The causal mask is always applied and, like
        the reference's call (train.py:786), no padding mask is.  An encoder that trains runs `encode` (differentiable, and
        reading the current weights); a frozen one the no-grad forward over bf16 weights packed once."""
        if self.trains():
            B, L = input_ids.shape
            return (self.encode(input_ids).float().view(B, L, -1),)
        return self._forward_frozen(input_ids)

    def _frozen_shadows(self):
        """bf16 kernel-layout copies of the frozen projection weights, made once and read by ops.weight_bf16."""
        for m in self.text_model.encoder.modules():
            w = getattr(m, "weight", None)
            if type(m) is not nn.Linear or w.requires_grad:
                continue
            sh = getattr(w, "_t2v_shadow", None)
            if sh is None or sh.device != w.device:
                w._t2v_shadow = prims.cast_f32_bf16(w.detach().float().contiguous()).view(w.shape[0], 1, 1, w.shape[1])

    def encode(self, input_ids):
        """Autograd forward: input_ids (B, L) -> bf16 token matrix [B*L, hidden], the final-LayerNorm output.  Gradients reach
        every tensor with requires_grad (LoRA factors, and with train_text_encoder the unfrozen weights, norms and embeddings)."""
        from .layers import run_linear
        cfg = self.config
        ids = input_ids.to(torch.int64).contiguous()
        B, L = ids.shape
        C, H = cfg.hidden_size, cfg.num_attention_heads
        quick = cfg.hidden_act == "quick_gelu"
        emb = self.text_model.embeddings
        self._frozen_shadows()
        x = ops.embed_tokens(ids, emb.token_embedding.weight, emb.position_embedding.weight)          # [B*L, C] bf16
        for lyr in self.text_model.encoder.layers:
            a, ln1, ln2 = lyr.self_attn, lyr.layer_norm1, lyr.layer_norm2
            res, h = ops.fork(x)
            n1, n2, n3 = ops.fork(ops.layer_norm(h, ln1.weight, ln1.bias, ln1.eps), 3)
            q, k, v = (run_linear(m, t).view(B, L, C) for m, t in ((a.q_proj, n1), (a.k_proj, n2), (a.v_proj, n3)))
            x = run_linear(a.out_proj, ops.causal_attention(q, k, v, H).view(B * L, C), residual=res)
            res, h = ops.fork(x)
            h = ops.gelu(run_linear(lyr.mlp.fc1, ops.layer_norm(h, ln2.weight, ln2.bias, ln2.eps)), quick)
            x = run_linear(lyr.mlp.fc2, h, residual=res)
        fl = self.text_model.final_layer_norm
        return ops.layer_norm(x, fl.weight, fl.bias, fl.eps)

    def plain_state_dict(self):
        """fp32 CPU state dict under the plain Hugging Face keys, every cloneofsimo LoRA collapsed into its base weight
        (W + scale * up @ down): it loads with strict=True into transformers.CLIPTextModel and into this class."""
        from .utils.lora import _WRAPPERS
        wrappers = {n: m for n, m in self.named_modules() if isinstance(m, _WRAPPERS)}
        sd = {}
        for k, v in self.state_dict().items():
            head, _, leaf = k.rpartition(".")
            parent, _, child = head.rpartition(".")
            if parent in wrappers:
                if child == "linear":
                    sd[f"{parent}.{leaf}"] = v
                continue
            sd[k] = v
        for n, m in wrappers.items():
            up, down = m.lora_up.weight.detach().float(), m.lora_down.weight.detach().float()
            if not isinstance(m.selector, nn.Identity):
                down = m.selector.weight.detach().float() @ down
            sd[f"{n}.weight"] = m.linear.weight.detach().float() + m.scale * (up @ down)
        return {k: v.detach().float().cpu().contiguous() for k, v in sd.items()}

    @torch.no_grad()
    def _forward_frozen(self, input_ids):
        cfg = self.config
        ids = input_ids.to(torch.int64).contiguous()
        B, L = ids.shape
        C, H = cfg.hidden_size, cfg.num_attention_heads
        D = C // H
        emb = self.text_model.embeddings
        pk = self._pack(ids.device)
        x = prims.embed_tokens(ids, emb.token_embedding.weight.detach().float().contiguous(),
                               emb.position_embedding.weight.detach().float().contiguous())          # [B*L, C] bf16
        ld = (L + 7) // 8 * 8
        for lyr, w in zip(self.text_model.encoder.layers, pk["layers"]):
            n, _ = prims.layernorm_fwd(x, lyr.layer_norm1.weight.detach().float(), lyr.layer_norm1.bias.detach().float(), lyr.layer_norm1.eps)
            qkv = prims.conv_fwd(n.view(1, 1, B * L, C), w["qkv_w"], w["qkv_b"]).view(B, L, 3 * C)
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
            s = torch.empty((B, H, L, ld), device=x.device, dtype=torch.float32)
            prims.bgemm(q, (1, q.stride(1), q.stride(0), D), k, (1, k.stride(1), k.stride(0), D), s, (ld, H * L * ld, L * ld),
                        L, L, D, B, H, D ** -0.5, 1)
            p = prims.softmax_fwd(s, L, ld, causal_period=L)
            a = torch.empty((B, L, C), device=x.device, dtype=x.dtype)
            prims.bgemm(p, (1, ld, H * L * ld, L * ld), v, (0, v.stride(1), v.stride(0), D), a, (C, L * C, D), L, D, L, B, H, 1.0, 0)
            x = prims.conv_fwd(a.view(1, 1, B * L, C), w["out_w"], w["out_b"], None, x.view(1, 1, B * L, C)).view(B * L, C)
            n, _ = prims.layernorm_fwd(x, lyr.layer_norm2.weight.detach().float(), lyr.layer_norm2.bias.detach().float(), lyr.layer_norm2.eps)
            h = prims.conv_fwd(n.view(1, 1, B * L, C), w["fc1_w"], w["fc1_b"]).view(B * L, -1)
            h = prims.gelu_bf16(h, quick=cfg.hidden_act == "quick_gelu")
            x = prims.conv_fwd(h.view(1, 1, B * L, h.shape[-1]), w["fc2_w"], w["fc2_b"], None, x.view(1, 1, B * L, C)).view(B * L, C)
        fl = self.text_model.final_layer_norm
        out, _ = prims.layernorm_fwd(x, fl.weight.detach().float(), fl.bias.detach().float(), fl.eps)
        return (out.float().view(B, L, C),)
