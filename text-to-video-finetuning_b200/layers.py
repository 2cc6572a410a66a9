"""Leaf modules of the text-to-video UNet, H100-native.

These classes carry the diffusers class names, constructor arguments and parameter names the reference relies on
(LoRA targets by class name: utils/lora.py:239-247 of the reference; state-dict keys: SURVEY.md appendix C), and own
exact `nn.Linear` / `nn.Conv2d` / `nn.Conv3d` / `nn.GroupNorm` / `nn.LayerNorm` children so module surgery keeps working.
Their forward passes, however, never call those children: they run the hand-written sm_90a kernels through ops.py.

Internal activation convention: bf16 channels-last frame batches `[N = B*F, H, W, C]`; token matrices `[rows, C]`
in the same frames-major order.  Nothing is permuted between spatial and temporal layers - temporal kernels take
strides instead (reference permutes at diffusers TransformerTemporalModel / TemporalConvLayer).
"""
from dataclasses import dataclass

import torch
import torch.nn as nn

from . import ops


@dataclass
class SampleOutput:
    sample: torch.Tensor


def _channels_last_(conv):
    """Store a conv weight physically as [Cout, K..., Cin] (torch channels_last) - the kernels' layout."""
    w = conv.weight
    fmt = torch.channels_last if w.dim() == 4 else torch.channels_last_3d
    conv.weight.data = w.data.contiguous(memory_format=fmt)
    return conv


# ------------------------------------------------------------------------------------------------ dispatch helpers
def _is_lora(m):
    return hasattr(m, "lora_down") and hasattr(m, "lora_up")


def _is_stable_lora(m):
    return hasattr(m, "lora_A") and hasattr(m, "lora_B")


def _lora_base(m):
    return m.linear if hasattr(m, "linear") else m.conv


def run_linear(m, x, residual=None, out_fp32=False, stats_rows=0):
    """Apply an nn.Linear (or a cloneofsimo / stable LoRA wrapper around one) to a token matrix.  stats_rows > 0: the output
    feeds a GroupNorm - let the GEMM epilogue produce its per-frame channel sums (stats_rows = tokens per frame)."""
    if _is_stable_lora(m):
        from .utils.stable_lora import stable_linear_forward
        return stable_linear_forward(m, x, residual, out_fp32, stats_rows)
    if _is_lora(m):
        from .utils.lora import lora_linear_forward
        return lora_linear_forward(m, x, residual, out_fp32, stats_rows)
    return ops.linear(x, m.weight, m.bias, residual, out_fp32, stats_rows=stats_rows)


def run_conv(m, x, rowbias=None, residual=None, stride=1, pads=(1, 1, 1, 1), rb_div=1, cin_pad=0, cout_pad=0, stats_rows=0):
    """Apply an nn.Conv2d / nn.Conv3d((3,1,1)) (or its LoRA wrapper) to a channels-last batch (stats_rows: see run_linear)."""
    if _is_stable_lora(m):
        from .utils.stable_lora import stable_conv_forward
        return stable_conv_forward(m, x, rowbias, residual, stride, pads, rb_div, cin_pad, cout_pad, stats_rows)
    if _is_lora(m):
        from .utils.lora import lora_conv_forward
        return lora_conv_forward(m, x, rowbias, residual, stride, pads, rb_div, cin_pad, cout_pad, stats_rows)
    return ops.conv(x, m.weight, m.bias, rowbias, residual, stride, pads, rb_div, False, cin_pad, cout_pad, stats_rows=stats_rows)


def clip_stats_rows(num_frames, hw):
    """Rows per statistics slot for a producer whose consumer normalises per CLIP.  One slot per clip would make every tile
    of a 16,384-row output red.add into the same C addresses (512-way same-address contention in L2, measured +7 us per
    GEMM); slots of about 4,096 rows (a whole number of frames, dividing the clip) keep the contention near that of the
    per-frame case, and the consumer adds the few slots of a clip while it finalises."""
    f = max(1, min(num_frames, 4096 // max(1, hw)))
    while num_frames % f:
        f -= 1
    return f * hw


def run_group_norm(m, x, silu, samples):
    return ops.group_norm(x, m.weight, m.bias, m.num_groups, m.eps, silu, samples)


def run_layer_norm(m, x):
    return ops.layer_norm(x, m.weight, m.bias, m.eps)


# ------------------------------------------------------------------------------------------------ embeddings
class Timesteps(nn.Module):
    """Sinusoidal timestep features [cos | sin] (flip_sin_to_cos=True, shift 0), unet_3d_condition.py:138."""

    def __init__(self, num_channels, flip_sin_to_cos=True, downscale_freq_shift=0):
        super().__init__()
        if not flip_sin_to_cos or downscale_freq_shift != 0:
            raise NotImplementedError("only the configuration used by UNet3DConditionModel is implemented")
        self.num_channels = num_channels

    def forward(self, timesteps):
        from . import prims
        return prims.timestep_embedding(timesteps.to(torch.int64).contiguous(), self.num_channels)


class TimestepEmbedding(nn.Module):
    """linear_2(SiLU(linear_1(t_emb)))  (unet_3d_condition.py:141-145)."""

    def __init__(self, in_channels, time_embed_dim, act_fn="silu"):
        super().__init__()
        if act_fn not in ("silu", "swish"):
            raise NotImplementedError(act_fn)
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, sample, condition=None):
        h = run_linear(self.linear_1, sample)
        return run_linear(self.linear_2, ops.silu(h))


# ------------------------------------------------------------------------------------------------ resnet family
class ResnetBlock2D(nn.Module):
    """GN-SiLU-conv3x3 (+ time embedding) - GN-SiLU-conv3x3 + (1x1) shortcut.  GroupNorm statistics are per frame.
    Fusions: SiLU into the GroupNorm apply pass; bias, time-embedding broadcast and the residual into conv epilogues."""

    def __init__(self, *, in_channels, out_channels=None, temb_channels=512, groups=32, eps=1e-6, dropout=0.0,
                 time_embedding_norm="default", non_linearity="swish", output_scale_factor=1.0, pre_norm=True, **unused):
        super().__init__()
        if time_embedding_norm != "default" or dropout != 0.0 or output_scale_factor != 1.0:
            raise NotImplementedError("ResnetBlock2D: only the configuration used by the 3-D UNet / SD-VAE is implemented")
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = _channels_last_(nn.Conv2d(in_channels, out_channels, 3, padding=1))
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels is not None else None
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = _channels_last_(nn.Conv2d(out_channels, out_channels, 3, padding=1))
        self.nonlinearity = nn.SiLU()
        self.conv_shortcut = _channels_last_(nn.Conv2d(in_channels, out_channels, 1)) if in_channels != out_channels else None

    def forward(self, x, temb_act=None, frames_per_clip=1):
        """x [N,H,W,Cin]; temb_act = SiLU(time embedding) as bf16 [B, temb_channels] (one row per clip)."""
        N, H, W, _ = x.shape
        x_skip, h = ops.fork(x)
        h = run_group_norm(self.norm1, h, True, N)
        rowbias = None
        if temb_act is not None and self.time_emb_proj is not None:
            rowbias = run_linear(self.time_emb_proj, temb_act, out_fp32=True)
        h = run_conv(self.conv1, h, rowbias=rowbias, rb_div=frames_per_clip, stats_rows=H * W)   # -> norm2
        h = run_group_norm(self.norm2, h, True, N)
        if self.conv_shortcut is not None:
            x_skip = run_conv(self.conv_shortcut, x_skip, pads=(0, 0, 0, 0))
        # -> the per-clip GroupNorm of the TemporalConvLayer that follows every resnet of the UNet (frames_per_clip = 1: per frame)
        return run_conv(self.conv2, h, residual=x_skip, stats_rows=clip_stats_rows(frames_per_clip, H * W))


class TemporalConvLayer(nn.Module):
    """Four [GroupNorm(32, per clip) - SiLU - Dropout - Conv3d (3,1,1)] stages plus identity; conv4 starts at zero.
    The clip is addressed as an image of W = H*W pixels and H = F rows, so the 3-tap temporal convolution is the same
    implicit-GEMM kernel with taps along the frame axis."""

    def __init__(self, in_dim, out_dim=None, dropout=0.0):
        super().__init__()
        out_dim = out_dim or in_dim
        self.in_dim, self.out_dim = in_dim, out_dim

        def stage(cin, cout, with_dropout):
            mods = [nn.GroupNorm(32, cin), nn.SiLU()]
            if with_dropout:
                mods.append(nn.Dropout(dropout))
            mods.append(_channels_last_(nn.Conv3d(cin, cout, (3, 1, 1), padding=(1, 0, 0))))
            return nn.Sequential(*mods)

        self.conv1 = stage(in_dim, out_dim, False)
        self.conv2 = stage(out_dim, in_dim, True)
        self.conv3 = stage(out_dim, in_dim, True)
        self.conv4 = stage(out_dim, in_dim, True)
        nn.init.zeros_(self.conv4[-1].weight)
        nn.init.zeros_(self.conv4[-1].bias)

    def forward(self, x, num_frames=1):
        N, H, W, C = x.shape
        B = N // num_frames
        identity, h = ops.fork(x)
        for i, seq in enumerate((self.conv1, self.conv2, self.conv3, self.conv4)):
            h = run_group_norm(seq[0], h, True, B)
            if i > 0 and self.training and seq[2].p > 0:  # nn.Dropout between SiLU and the conv (own RNG stream)
                h = ops.dropout(h, seq[2].p)
            h = h.view(B, num_frames, H * W, h.shape[-1])
            res = identity.view(B, num_frames, H * W, C) if i == 3 else None
            # the next stage normalises per clip; after conv4 (+ identity) a spatial layer follows, which normalises per frame
            h = run_conv(seq[-1], h, residual=res, pads=(1, 1, 0, 0), stats_rows=(H * W) if i == 3 else clip_stats_rows(num_frames, H * W))
            h = ops.view(h, N, H, W, -1)
        return h


class Downsample2D(nn.Module):
    def __init__(self, channels, use_conv=False, out_channels=None, padding=1, name="conv"):
        super().__init__()
        if not use_conv:
            raise NotImplementedError("Downsample2D without conv")
        self.padding = padding
        self.conv = _channels_last_(nn.Conv2d(channels, out_channels or channels, 3, stride=2, padding=padding))

    def forward(self, x):
        pads = (1, 1, 1, 1) if self.padding == 1 else (0, 1, 0, 1)  # the VAE pads (0,1,0,1) then convolves unpadded
        Ho, Wo = (x.shape[1] + pads[0] + pads[1] - 3) // 2 + 1, (x.shape[2] + pads[2] + pads[3] - 3) // 2 + 1
        return run_conv(self.conv, x, stride=2, pads=pads, stats_rows=Ho * Wo)


class Upsample2D(nn.Module):
    def __init__(self, channels, use_conv=False, use_conv_transpose=False, out_channels=None, name="conv"):
        super().__init__()
        if not use_conv or use_conv_transpose:
            raise NotImplementedError("Upsample2D variant")
        self.conv = _channels_last_(nn.Conv2d(channels, out_channels or channels, 3, padding=1))

    def forward(self, x, output_size=None):
        N, H, W, C = x.shape
        size = (2 * H, 2 * W) if output_size is None else tuple(output_size)
        return run_conv(self.conv, ops.upsample_nearest(x, size), stats_rows=size[0] * size[1])


# ------------------------------------------------------------------------------------------------ attention family
class Attention(nn.Module):
    """diffusers Attention: bias-free q/k/v projections, biased output projection, softmax(q k^T d^-0.5) v."""

    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64, dropout=0.0, bias=False, out_bias=True):
        super().__init__()
        inner = heads * dim_head
        ctx_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads, self.dim_head, self.inner_dim = heads, dim_head, inner
        self.is_cross = cross_attention_dim is not None
        self.to_q = nn.Linear(query_dim, inner, bias=bias)
        self.to_k = nn.Linear(ctx_dim, inner, bias=bias)
        self.to_v = nn.Linear(ctx_dim, inner, bias=bias)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim, bias=out_bias), nn.Dropout(dropout)])

    def set_processor(self, processor):  # train.py:138-150 sets AttnProcessor2_0; the kernels here are always fused
        pass

    def set_attention_slice(self, slice_size):
        pass

    @property
    def sliceable_head_dim(self):
        return self.heads

    def project_out(self, a, residual):
        return run_linear(self.to_out[0], a, residual=residual)


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        return ops.geglu(run_linear(self.proj, x))


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4, dropout=0.0, activation_fn="geglu"):
        super().__init__()
        if activation_fn != "geglu":
            raise NotImplementedError(activation_fn)
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(dropout), nn.Linear(dim * mult, dim)])

    def forward(self, x, residual=None):
        return run_linear(self.net[2], self.net[0](x), residual=residual)


class BasicTransformerBlock(nn.Module):
    """x += attn1(LN1 x); x += attn2(LN2 x, ctx); x += ff(LN3 x).  The three residual adds are GEMM epilogues.

    `attend(q, k, v, attn)` is supplied by the owning model: spatial layers run the batched wgmma attention,
    temporal layers the strided short-sequence kernel."""

    def __init__(self, dim, num_attention_heads, attention_head_dim, dropout=0.0, cross_attention_dim=None,
                 activation_fn="geglu", attention_bias=False, double_self_attention=False, **unused):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, num_attention_heads, attention_head_dim, dropout, attention_bias)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, None if double_self_attention else cross_attention_dim, num_attention_heads,
                               attention_head_dim, dropout, attention_bias)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim, dropout=dropout, activation_fn=activation_fn)

    @staticmethod
    def _fused(attn):
        """('qkv' | 'kv', FusedWeight) when the runtime arena laid this attention's projections out back to back and
        none of them is wrapped (LoRA) - then they run as one GEMM."""
        f = getattr(attn, "_t2v_fused", None)
        if f is None or not f[1].usable():
            return None
        if not all(type(m) is nn.Linear for m in (attn.to_q, attn.to_k, attn.to_v)):
            return None
        return f

    def forward(self, x, context, attend, attend_cross=None):
        for attn, norm in ((self.attn1, self.norm1), (self.attn2, self.norm2)):
            res, h = ops.fork(x)
            n = run_layer_norm(norm, h)
            fused = self._fused(attn)
            if fused is not None and fused[0] == "qkv" and not attn.is_cross:
                a = attend(ops.linear(n, fused[1]), None, None, attn)
            elif fused is not None and fused[0] == "kv" and attn.is_cross:
                q = run_linear(attn.to_q, n)
                a = attend_cross(q, ops.linear(context, fused[1]), None, attn)
            elif attn.is_cross:
                q = run_linear(attn.to_q, n)
                c1, c2 = ops.fork(context)
                k, v = run_linear(attn.to_k, c1), run_linear(attn.to_v, c2)
                a = attend_cross(q, k, v, attn)
            else:
                n1, n2, n3 = ops.fork(n, 3)
                q, k, v = run_linear(attn.to_q, n1), run_linear(attn.to_k, n2), run_linear(attn.to_v, n3)
                a = attend(q, k, v, attn)
            x = attn.project_out(a, res)
        res, h = ops.fork(x)
        return self.ff(run_layer_norm(self.norm3, h), residual=res)


class Transformer2DModel(nn.Module):
    """GroupNorm(eps 1e-6, per frame) - proj_in - BasicTransformerBlock(text cross-attention) - proj_out + residual,
    with linear projections (use_linear_projection=True as wired at unet_3d_blocks.py:319-330)."""

    def __init__(self, num_attention_heads=16, attention_head_dim=88, in_channels=None, num_layers=1, dropout=0.0,
                 norm_num_groups=32, cross_attention_dim=None, attention_bias=False, use_linear_projection=False,
                 only_cross_attention=False, upcast_attention=False, **unused):
        super().__init__()
        if not use_linear_projection or num_layers != 1 or only_cross_attention:
            raise NotImplementedError("Transformer2DModel: only the configuration used by the 3-D UNet is implemented")
        inner = num_attention_heads * attention_head_dim
        self.num_attention_heads, self.attention_head_dim, self.in_channels = num_attention_heads, attention_head_dim, in_channels
        self.norm = nn.GroupNorm(norm_num_groups, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(
            inner, num_attention_heads, attention_head_dim, dropout, cross_attention_dim, attention_bias=attention_bias)])
        self.proj_out = nn.Linear(inner, in_channels)

    def forward(self, x, encoder_hidden_states=None, num_frames=1, return_dict=True, **unused):
        """x [N,H,W,C]; encoder_hidden_states: bf16 token matrix [B*Lctx, ctx_dim] (one text sequence per clip)."""
        N, H, W, C = x.shape
        B = N // num_frames
        res, h = ops.fork(x)
        h = run_group_norm(self.norm, h, False, N).view(N * H * W, C)
        h = run_linear(self.proj_in, h)

        def attend(q, k, v, attn):  # per-frame spatial self-attention (k is None: q is the fused [rows, 3C] projection)
            L = H * W
            if k is None:
                return ops.attention_fused(q.view(N, L, -1), None, attn.heads).view(N * L, -1)
            return ops.attention(q.view(N, L, -1), k.view(N, L, -1), v.view(N, L, -1), attn.heads).view(N * L, -1)

        def attend_cross(q, k, v, attn):  # all frames of a clip attend to that clip's text tokens: K/V once per clip
            Lq = num_frames * H * W
            if v is None:                 # k is the fused [B*Lctx, 2C] projection of the text tokens
                return ops.attention_fused(q.view(B, Lq, -1), k.view(B, -1, k.shape[-1]), attn.heads).view(B * Lq, -1)
            return ops.attention(q.view(B, Lq, -1), k.view(B, -1, k.shape[-1]), v.view(B, -1, v.shape[-1]),
                                 attn.heads).view(B * Lq, -1)

        h = self.transformer_blocks[0](h, encoder_hidden_states, attend, attend_cross)
        # the TransformerTemporalModel that follows normalises per clip
        out = ops.view(run_linear(self.proj_out, h, residual=res.view(N * H * W, C), stats_rows=clip_stats_rows(num_frames, H * W)), N, H, W, C)
        return SampleOutput(sample=out) if return_dict else (out,)


class TransformerTemporalModel(nn.Module):
    """GroupNorm(eps 1e-6, per clip) - proj_in - BasicTransformerBlock(double self-attention over frames) - proj_out
    + residual.  Tokens stay frames-major; the attention kernel walks the frame axis with strides."""

    def __init__(self, num_attention_heads=16, attention_head_dim=88, in_channels=None, out_channels=None, num_layers=1,
                 dropout=0.0, norm_num_groups=32, cross_attention_dim=None, attention_bias=False, sample_size=None,
                 activation_fn="geglu", norm_elementwise_affine=True, double_self_attention=True):
        super().__init__()
        if num_layers != 1 or not double_self_attention:
            raise NotImplementedError("TransformerTemporalModel: only the configuration used by the 3-D UNet is implemented")
        inner = num_attention_heads * attention_head_dim
        self.num_attention_heads, self.attention_head_dim, self.in_channels = num_attention_heads, attention_head_dim, in_channels
        self.norm = nn.GroupNorm(norm_num_groups, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(
            inner, num_attention_heads, attention_head_dim, dropout, cross_attention_dim, activation_fn=activation_fn,
            attention_bias=attention_bias, double_self_attention=True)])
        self.proj_out = nn.Linear(inner, in_channels)

    def forward(self, x, num_frames=1, return_dict=True, **unused):
        N, H, W, C = x.shape
        B = N // num_frames
        res, h = ops.fork(x)
        h = run_group_norm(self.norm, h, False, B).view(N * H * W, C)
        h = run_linear(self.proj_in, h)

        def attend(q, k, v, attn):
            if k is None:
                return ops.temporal_attention_fused(q, attn.heads, B, num_frames, H * W)
            return ops.temporal_attention(q, k, v, attn.heads, B, num_frames, H * W)

        h = self.transformer_blocks[0](h, None, attend)
        out = ops.view(run_linear(self.proj_out, h, residual=res.view(N * H * W, C), stats_rows=H * W), N, H, W, C)
        return SampleOutput(sample=out) if return_dict else (out,)
