"""UNet3DConditionModel - the text-to-video-ms-1.7b / zeroscope_v2_576w denoiser - on H100-native kernels.

Drop-in for the reference's models/unet_3d_condition.py: same class name, constructor keywords and defaults
(reference :86-107), same `forward` signature and `(B, C, F, H, W)` in/out contract (:325-337, :495-500), same module
tree and parameter names, `_set_gradient_checkpointing` (:318-323) and `set_attention_slice` (:253-316, a no-op here:
attention is always fused).  What differs is everything underneath: activations are bf16 channels-last frame batches,
the noisy latent is converted (and, in training, noised) by one kernel at the boundary, the time embedding is kept
per clip, and the whole pass runs on the hand-written sm_90a kernels (no ATen/cuDNN/cuBLAS on the path).
"""
from dataclasses import dataclass
from typing import Any, Dict, Optional, Tuple, Union

import torch
import torch.nn as nn

from .. import ops, prims
from ..layers import (TimestepEmbedding, Timesteps, Transformer2DModel, TransformerTemporalModel, _channels_last_, clip_stats_rows, run_conv,
                      run_group_norm)
from ..modeling_utils import ConfigMixin, ModelMixin, register_to_config
from .unet_3d_blocks import (CrossAttnDownBlock3D, CrossAttnUpBlock3D, DownBlock3D, StepContext, UNetMidBlock3DCrossAttn,
                             UpBlock3D, get_down_block, get_up_block, transformer_g_c)


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor


class _ToBf16(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return prims.cast_f32_bf16(x.contiguous())

    @staticmethod
    def backward(ctx, g):
        return g.float()


class UNet3DConditionModel(ModelMixin, ConfigMixin):
    _supports_gradient_checkpointing = True

    @register_to_config
    def __init__(
        self,
        sample_size: Optional[int] = None,
        in_channels: int = 4,
        out_channels: int = 4,
        down_block_types: Tuple[str] = ("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "DownBlock3D"),
        up_block_types: Tuple[str] = ("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D"),
        block_out_channels: Tuple[int] = (320, 640, 1280, 1280),
        layers_per_block: int = 2,
        downsample_padding: int = 1,
        mid_block_scale_factor: float = 1,
        act_fn: str = "silu",
        norm_num_groups: Optional[int] = 32,
        norm_eps: float = 1e-5,
        cross_attention_dim: int = 1024,
        attention_head_dim: Union[int, Tuple[int]] = 64,
    ):
        super().__init__()
        n_levels = len(block_out_channels)
        if len(down_block_types) != len(up_block_types) or n_levels != len(down_block_types):
            raise ValueError("down_block_types, up_block_types and block_out_channels must have the same length")
        if not isinstance(attention_head_dim, int) and len(attention_head_dim) != n_levels:
            raise ValueError("attention_head_dim must be an int or have one entry per block")
        if in_channels > 8 or out_channels > 8 or norm_num_groups is None:
            raise NotImplementedError("latent channels > 8 / norm-free variants are not implemented")
        head_dims = (attention_head_dim,) * n_levels if isinstance(attention_head_dim, int) else tuple(attention_head_dim)
        c0 = block_out_channels[0]
        temb_dim = c0 * 4
        self.sample_size = sample_size
        self.gradient_checkpointing = False

        self.conv_in = _channels_last_(nn.Conv2d(in_channels, c0, kernel_size=3, padding=1))
        self.time_proj = Timesteps(c0, True, 0)
        self.time_embedding = TimestepEmbedding(c0, temb_dim, act_fn=act_fn)
        self.transformer_in = TransformerTemporalModel(num_attention_heads=8, attention_head_dim=head_dims[0],
                                                       in_channels=c0, num_layers=1)

        common = dict(temb_channels=temb_dim, resnet_eps=norm_eps, resnet_act_fn=act_fn, resnet_groups=norm_num_groups,
                      cross_attention_dim=cross_attention_dim, dual_cross_attention=False)
        self.down_blocks = nn.ModuleList()
        ch = c0
        for i, kind in enumerate(down_block_types):
            self.down_blocks.append(get_down_block(kind, num_layers=layers_per_block, in_channels=ch,
                                                   out_channels=block_out_channels[i], add_downsample=i != n_levels - 1,
                                                   attn_num_head_channels=head_dims[i], downsample_padding=downsample_padding,
                                                   **common))
            ch = block_out_channels[i]

        self.mid_block = UNetMidBlock3DCrossAttn(in_channels=block_out_channels[-1], temb_channels=temb_dim, resnet_eps=norm_eps,
                                                 resnet_act_fn=act_fn, output_scale_factor=mid_block_scale_factor,
                                                 cross_attention_dim=cross_attention_dim, attn_num_head_channels=head_dims[-1],
                                                 resnet_groups=norm_num_groups, dual_cross_attention=False)

        self.up_blocks = nn.ModuleList()
        rev_ch, rev_hd = block_out_channels[::-1], head_dims[::-1]
        self.num_upsamplers = n_levels - 1
        prev = rev_ch[0]
        for i, kind in enumerate(up_block_types):
            self.up_blocks.append(get_up_block(kind, num_layers=layers_per_block + 1, in_channels=rev_ch[min(i + 1, n_levels - 1)],
                                               out_channels=rev_ch[i], prev_output_channel=prev, add_upsample=i != n_levels - 1,
                                               attn_num_head_channels=rev_hd[i], **common))
            prev = rev_ch[i]

        self.conv_norm_out = nn.GroupNorm(num_channels=c0, num_groups=norm_num_groups, eps=norm_eps)
        self.conv_act = nn.SiLU()
        self.conv_out = _channels_last_(nn.Conv2d(c0, out_channels, kernel_size=3, padding=1))

    # ------------------------------------------------------------------------------------------------ knobs
    def set_attention_slice(self, slice_size):
        """Accepted for API compatibility; the fused attention kernels never materialise per-head slices on the host."""

    def _set_gradient_checkpointing(self, value=False):
        self.gradient_checkpointing = value
        self.mid_block.gradient_checkpointing = value
        for module in list(self.down_blocks) + list(self.up_blocks):
            if isinstance(module, (CrossAttnDownBlock3D, DownBlock3D, CrossAttnUpBlock3D, UpBlock3D)):
                module.gradient_checkpointing = value

    # ------------------------------------------------------------------------------------------------ forward
    def _timesteps(self, timestep, batch, device):
        t = timestep
        if not torch.is_tensor(t):
            t = torch.tensor([t], dtype=torch.int64, device=device)
        elif t.dim() == 0:
            t = t[None]
        return t.to(device=device, dtype=torch.int64).expand(batch).contiguous()

    def forward_channels_last(self, x, timesteps, text, batch, num_frames):
        """Core pass on kernel-native tensors: x bf16 [B*F, H, W, 8] (latent channels zero-padded to 8),
        timesteps int64 [B], text bf16 [B*Lctx, ctx_dim]  ->  bf16 [B*F, H, W, 8]."""
        cfg = self.config
        H, W = x.shape[1], x.shape[2]
        forward_upsample_size = any(s % (2 ** self.num_upsamplers) != 0 for s in (H, W))

        emb = self.time_embedding(self.time_proj(timesteps))
        # trainable text states (text-encoder LoRA): their gradient is summed over every cross-attention in fp32
        texts = list(ops.fork_f32(text, self._n_cross_attention())) if text.requires_grad else None
        sc = StepContext(num_frames, ops.silu(emb), text, texts)

        h = run_conv(self.conv_in, x, cin_pad=8 - cfg.in_channels, stats_rows=clip_stats_rows(num_frames, H * W))   # -> transformer_in (per clip)
        if num_frames > 1:
            h = transformer_g_c(self.transformer_in, h, num_frames, self.gradient_checkpointing)

        # runtime.GradientBuckets: start a block's share of the gradient all-reduce as soon as its backward is through
        mark = getattr(self, "_t2v_grad_hook", None)
        h, keep = ops.fork(h)
        skips = [keep]
        for i, block in enumerate(self.down_blocks):
            h, res = block(ops.grad_mark(h, mark, f"down_blocks.{i}"), sc)
            skips.extend(res)

        h = self.mid_block(ops.grad_mark(h, mark, "mid_block"), sc)

        for i, block in enumerate(self.up_blocks):
            h = ops.grad_mark(h, mark, f"up_blocks.{i}")
            n = len(block.resnets)
            res, skips = skips[-n:], skips[:-n]
            size = None
            if i != len(self.up_blocks) - 1 and forward_upsample_size:
                size = tuple(skips[-1].shape[1:3])
            h = block(h, res, sc, upsample_size=size)

        h = run_group_norm(self.conv_norm_out, h, True, h.shape[0])
        return run_conv(self.conv_out, h, cout_pad=8 - cfg.out_channels)

    def _n_cross_attention(self):
        return sum(isinstance(m, Transformer2DModel) for m in self.modules())

    def forward(
        self,
        sample: torch.Tensor,
        timestep: Union[torch.Tensor, float, int],
        encoder_hidden_states: torch.Tensor,
        class_labels: Optional[torch.Tensor] = None,
        timestep_cond: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        cross_attention_kwargs: Optional[Dict[str, Any]] = None,
        down_block_additional_residuals: Optional[Tuple[torch.Tensor]] = None,
        mid_block_additional_residual: Optional[torch.Tensor] = None,
        return_dict: bool = True,
    ) -> Union[UNet3DConditionOutput, Tuple]:
        """sample (B, C, F, H, W), timestep scalar or (B,), encoder_hidden_states (B, L, ctx_dim) -> `.sample` (B, C, F, H, W).
        `attention_mask` is accepted and ignored exactly as in the reference (never reaches attention, H16)."""
        if down_block_additional_residuals is not None or mid_block_additional_residual is not None:
            raise NotImplementedError("ControlNet-style additional residuals are not on the finetune path")
        B, C, F, H, W = sample.shape
        x = prims.latents_to_nhwc8(sample.detach().float().contiguous())
        text = self.prepare_text(encoder_hidden_states)
        out = self.forward_channels_last(x, self._timesteps(timestep, B, sample.device), text, B, F)
        result = ops.from_nhwc8(out, B, self.config.out_channels, F)
        if sample.dtype != torch.float32:
            result = result.to(sample.dtype)
        return UNet3DConditionOutput(sample=result) if return_dict else (result,)

    @staticmethod
    def prepare_text(encoder_hidden_states):
        """(B, L, D) text states -> bf16 token matrix [B*L, D] (one sequence per clip; the reference repeats it F times)."""
        e = encoder_hidden_states
        if e.dtype == torch.bfloat16:
            t = e.contiguous()
        else:
            t = _ToBf16.apply(e.float())
        return t.reshape(-1, t.shape[-1])
