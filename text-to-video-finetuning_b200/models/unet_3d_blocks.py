"""Down / mid / up blocks of the 3-D UNet - same class names, constructor keywords, attribute names
(`resnets`, `temp_convs`, `attentions`, `temp_attentions`, `downsamplers`, `upsamplers`, `gradient_checkpointing`,
`has_cross_attention`) and therefore the same state-dict keys as the reference's models/unet_3d_blocks.py, rebuilt on
the H100-native leaves in layers.py.

Differences by design (H100-first, not a translation):
  * activations flow as bf16 channels-last frame batches [B*F, H, W, C]; no permutes between spatial and temporal layers
  * the time embedding is handed down once per clip (SiLU already applied) and broadcast inside the conv epilogue
  * text context is a per-clip token matrix; cross-attention K/V are computed once per clip, not once per frame
  * skip concatenation is a single channel-concat kernel on channels-last data

Reference semantics followed: layer order per block (unet_3d_blocks.py:368-419,517-569,632-652,746-798,856-875),
including the mid block applying temp_convs[0] unconditionally, and the per-sub-module activation checkpointing of
custom_checkpoint / cross_attn_g_c / up_down_g_c (unet_3d_blocks.py:30-153).
"""
import torch.nn as nn
from torch.utils.checkpoint import checkpoint

from .. import ops
from ..layers import (Downsample2D, ResnetBlock2D, TemporalConvLayer, Transformer2DModel, TransformerTemporalModel,
                      Upsample2D)


class StepContext:
    """Per-forward constants shared by all blocks."""

    __slots__ = ("num_frames", "temb_act", "text", "texts")

    def __init__(self, num_frames, temb_act, text, texts=None):
        self.num_frames = num_frames  # F
        self.temb_act = temb_act      # SiLU(time embedding), bf16 [B, 4*C0]
        self.text = text              # bf16 [B*Lctx, ctx_dim]
        self.texts = texts            # trainable text states: one ops.fork_f32 output per cross-attention, handed out in order

    def take_text(self):
        return self.texts.pop() if self.texts is not None else self.text


def _maybe_ckpt(enabled, fn, *args):
    """One activation-checkpoint unit (the reference's custom_checkpoint / cross_attn_g_c / up_down_g_c granularity).  The
    dropout seeds of the unit derive from a base seed drawn here, outside the recomputed function, so forward, recompute
    and backward agree on every mask; torch's own RNG-state bookkeeping is switched off (it cannot be graph-captured)."""
    base = ops.next_dropout_seed()   # drawn the same way with checkpointing on or off: both modes see the same masks

    def scoped(*a):
        with ops.dropout_seed_scope(base):
            return fn(*a)
    if enabled:
        return checkpoint(scoped, *args, use_reentrant=False, preserve_rng_state=False)
    return scoped(*args)


class _Block3D(nn.Module):
    """Shared machinery: one 'layer' = resnet -> temporal conv [-> spatial transformer -> temporal transformer]."""

    has_cross_attention = False

    def _new_resnet(self, cin, cout, temb_channels, eps, groups, dropout, act_fn, scale_shift, osf, pre_norm):
        return ResnetBlock2D(in_channels=cin, out_channels=cout, temb_channels=temb_channels, eps=eps, groups=groups,
                             dropout=dropout, time_embedding_norm=scale_shift, non_linearity=act_fn,
                             output_scale_factor=osf, pre_norm=pre_norm)

    def _new_attn_pair(self, channels, head_dim, cross_attention_dim, groups, use_linear_projection, only_cross_attention,
                       upcast_attention):
        heads = channels // head_dim
        spatial = Transformer2DModel(heads, head_dim, in_channels=channels, num_layers=1, cross_attention_dim=cross_attention_dim,
                                     norm_num_groups=groups, use_linear_projection=use_linear_projection,
                                     only_cross_attention=only_cross_attention, upcast_attention=upcast_attention)
        temporal = TransformerTemporalModel(heads, head_dim, in_channels=channels, num_layers=1,
                                            cross_attention_dim=cross_attention_dim, norm_num_groups=groups)
        return spatial, temporal

    # -- sub-module calls; each is its own checkpoint unit when gradient_checkpointing is on (reference g_c helpers)
    def _resnet(self, m, h, sc):
        f = lambda t, e: m(t, e, sc.num_frames)
        return _maybe_ckpt(self.gradient_checkpointing, f, h, sc.temb_act)

    def _temp_conv(self, m, h, sc, always=False):
        if sc.num_frames <= 1 and not always:
            return h
        f = lambda t: m(t, num_frames=sc.num_frames)
        return _maybe_ckpt(self.gradient_checkpointing, f, h)

    def _attn(self, m, h, sc):
        f = lambda t, c: m(t, c, num_frames=sc.num_frames).sample
        return _maybe_ckpt(self.gradient_checkpointing, f, h, sc.take_text())

    def _temp_attn(self, m, h, sc):
        if sc.num_frames <= 1:
            return h
        f = lambda t: m(t, num_frames=sc.num_frames).sample
        return _maybe_ckpt(self.gradient_checkpointing, f, h)


class UNetMidBlock3DCrossAttn(_Block3D):
    has_cross_attention = True

    def __init__(self, in_channels, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6, resnet_time_scale_shift="default",
                 resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True, attn_num_head_channels=1, output_scale_factor=1.0,
                 cross_attention_dim=1280, dual_cross_attention=False, use_linear_projection=True, upcast_attention=False):
        super().__init__()
        self.gradient_checkpointing = False
        self.attn_num_head_channels = attn_num_head_channels
        groups = resnet_groups if resnet_groups is not None else min(in_channels // 4, 32)
        mk = lambda: self._new_resnet(in_channels, in_channels, temb_channels, resnet_eps, groups, dropout, resnet_act_fn,
                                      resnet_time_scale_shift, output_scale_factor, resnet_pre_norm)
        resnets, temp_convs, attentions, temp_attentions = [mk()], [TemporalConvLayer(in_channels, in_channels, dropout=0.1)], [], []
        for _ in range(num_layers):
            s, t = self._new_attn_pair(in_channels, attn_num_head_channels, cross_attention_dim, groups, use_linear_projection,
                                       False, upcast_attention)
            attentions.append(s)
            temp_attentions.append(t)
            resnets.append(mk())
            temp_convs.append(TemporalConvLayer(in_channels, in_channels, dropout=0.1))
        self.resnets, self.temp_convs = nn.ModuleList(resnets), nn.ModuleList(temp_convs)
        self.attentions, self.temp_attentions = nn.ModuleList(attentions), nn.ModuleList(temp_attentions)

    def forward(self, hidden_states, sc):
        h = self._resnet(self.resnets[0], hidden_states, sc)
        h = self._temp_conv(self.temp_convs[0], h, sc, always=True)  # unconditional in the reference (:386-387)
        for attn, temp_attn, resnet, temp_conv in zip(self.attentions, self.temp_attentions, self.resnets[1:], self.temp_convs[1:]):
            h = self._attn(attn, h, sc)
            h = self._temp_attn(temp_attn, h, sc)
            h = self._resnet(resnet, h, sc)
            h = self._temp_conv(temp_conv, h, sc)
        return h


class _DownBase(_Block3D):
    def _build(self, with_attn, in_channels, out_channels, temb_channels, dropout, num_layers, resnet_eps, scale_shift, act_fn,
               groups, pre_norm, osf, add_downsample, downsample_padding, head_dim=None, cross_attention_dim=None,
               use_linear_projection=False, only_cross_attention=False, upcast_attention=False):
        self.gradient_checkpointing = False
        resnets, temp_convs, attentions, temp_attentions = [], [], [], []
        for i in range(num_layers):
            cin = in_channels if i == 0 else out_channels
            resnets.append(self._new_resnet(cin, out_channels, temb_channels, resnet_eps, groups, dropout, act_fn, scale_shift, osf, pre_norm))
            temp_convs.append(TemporalConvLayer(out_channels, out_channels, dropout=0.1))
            if with_attn:
                s, t = self._new_attn_pair(out_channels, head_dim, cross_attention_dim, groups, use_linear_projection,
                                           only_cross_attention, upcast_attention)
                attentions.append(s)
                temp_attentions.append(t)
        self.resnets, self.temp_convs = nn.ModuleList(resnets), nn.ModuleList(temp_convs)
        if with_attn:
            self.attentions, self.temp_attentions = nn.ModuleList(attentions), nn.ModuleList(temp_attentions)
        self.downsamplers = nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                        padding=downsample_padding, name="op")]) if add_downsample else None

    def forward(self, hidden_states, sc):
        h, skips = hidden_states, []
        attns = getattr(self, "attentions", None)
        for j, (resnet, temp_conv) in enumerate(zip(self.resnets, self.temp_convs)):
            h = self._resnet(resnet, h, sc)
            h = self._temp_conv(temp_conv, h, sc)
            if attns is not None:
                h = self._attn(attns[j], h, sc)
                h = self._temp_attn(self.temp_attentions[j], h, sc)
            h, keep = ops.fork(h)
            skips.append(keep)
        if self.downsamplers is not None:
            for d in self.downsamplers:
                h = d(h)
            h, keep = ops.fork(h)
            skips.append(keep)
        return h, tuple(skips)


class CrossAttnDownBlock3D(_DownBase):
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True,
                 attn_num_head_channels=1, cross_attention_dim=1280, output_scale_factor=1.0, downsample_padding=1,
                 add_downsample=True, dual_cross_attention=False, use_linear_projection=False, only_cross_attention=False,
                 upcast_attention=False):
        super().__init__()
        self.attn_num_head_channels = attn_num_head_channels
        self._build(True, in_channels, out_channels, temb_channels, dropout, num_layers, resnet_eps, resnet_time_scale_shift,
                    resnet_act_fn, resnet_groups, resnet_pre_norm, output_scale_factor, add_downsample, downsample_padding,
                    attn_num_head_channels, cross_attention_dim, use_linear_projection, only_cross_attention, upcast_attention)


class DownBlock3D(_DownBase):
    def __init__(self, in_channels, out_channels, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True,
                 output_scale_factor=1.0, add_downsample=True, downsample_padding=1):
        super().__init__()
        self._build(False, in_channels, out_channels, temb_channels, dropout, num_layers, resnet_eps, resnet_time_scale_shift,
                    resnet_act_fn, resnet_groups, resnet_pre_norm, output_scale_factor, add_downsample, downsample_padding)


class _UpBase(_Block3D):
    def _build(self, with_attn, in_channels, prev_output_channel, out_channels, temb_channels, dropout, num_layers, resnet_eps,
               scale_shift, act_fn, groups, pre_norm, osf, add_upsample, head_dim=None, cross_attention_dim=None,
               use_linear_projection=False, only_cross_attention=False, upcast_attention=False):
        self.gradient_checkpointing = False
        resnets, temp_convs, attentions, temp_attentions = [], [], [], []
        for i in range(num_layers):
            skip_c = in_channels if i == num_layers - 1 else out_channels
            cin = prev_output_channel if i == 0 else out_channels
            resnets.append(self._new_resnet(cin + skip_c, out_channels, temb_channels, resnet_eps, groups, dropout, act_fn,
                                            scale_shift, osf, pre_norm))
            temp_convs.append(TemporalConvLayer(out_channels, out_channels, dropout=0.1))
            if with_attn:
                s, t = self._new_attn_pair(out_channels, head_dim, cross_attention_dim, groups, use_linear_projection,
                                           only_cross_attention, upcast_attention)
                attentions.append(s)
                temp_attentions.append(t)
        self.resnets, self.temp_convs = nn.ModuleList(resnets), nn.ModuleList(temp_convs)
        if with_attn:
            self.attentions, self.temp_attentions = nn.ModuleList(attentions), nn.ModuleList(temp_attentions)
        self.upsamplers = nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)]) if add_upsample else None

    def forward(self, hidden_states, res_hidden_states_tuple, sc, upsample_size=None):
        h = hidden_states
        attns = getattr(self, "attentions", None)
        skips = list(res_hidden_states_tuple)
        for j, (resnet, temp_conv) in enumerate(zip(self.resnets, self.temp_convs)):
            h = ops.concat_channels(h, skips.pop())
            h = self._resnet(resnet, h, sc)
            h = self._temp_conv(temp_conv, h, sc)
            if attns is not None:
                h = self._attn(attns[j], h, sc)
                h = self._temp_attn(self.temp_attentions[j], h, sc)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                h = u(h, upsample_size)
        return h


class CrossAttnUpBlock3D(_UpBase):
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, prev_output_channel, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True,
                 attn_num_head_channels=1, cross_attention_dim=1280, output_scale_factor=1.0, add_upsample=True,
                 dual_cross_attention=False, use_linear_projection=False, only_cross_attention=False, upcast_attention=False):
        super().__init__()
        self.attn_num_head_channels = attn_num_head_channels
        self._build(True, in_channels, prev_output_channel, out_channels, temb_channels, dropout, num_layers, resnet_eps,
                    resnet_time_scale_shift, resnet_act_fn, resnet_groups, resnet_pre_norm, output_scale_factor, add_upsample,
                    attn_num_head_channels, cross_attention_dim, use_linear_projection, only_cross_attention, upcast_attention)


class UpBlock3D(_UpBase):
    def __init__(self, in_channels, prev_output_channel, out_channels, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True,
                 output_scale_factor=1.0, add_upsample=True):
        super().__init__()
        self._build(False, in_channels, prev_output_channel, out_channels, temb_channels, dropout, num_layers, resnet_eps,
                    resnet_time_scale_shift, resnet_act_fn, resnet_groups, resnet_pre_norm, output_scale_factor, add_upsample)


_DOWN = {"DownBlock3D": DownBlock3D, "CrossAttnDownBlock3D": CrossAttnDownBlock3D}
_UP = {"UpBlock3D": UpBlock3D, "CrossAttnUpBlock3D": CrossAttnUpBlock3D}


def get_down_block(down_block_type, num_layers, in_channels, out_channels, temb_channels, add_downsample, resnet_eps,
                   resnet_act_fn, attn_num_head_channels, resnet_groups=None, cross_attention_dim=None,
                   downsample_padding=None, dual_cross_attention=False, use_linear_projection=True,
                   only_cross_attention=False, upcast_attention=False, resnet_time_scale_shift="default"):
    if down_block_type not in _DOWN:
        raise ValueError(f"{down_block_type} does not exist.")
    kw = dict(num_layers=num_layers, in_channels=in_channels, out_channels=out_channels, temb_channels=temb_channels,
              add_downsample=add_downsample, resnet_eps=resnet_eps, resnet_act_fn=resnet_act_fn, resnet_groups=resnet_groups,
              downsample_padding=downsample_padding, resnet_time_scale_shift=resnet_time_scale_shift)
    if down_block_type == "CrossAttnDownBlock3D":
        if cross_attention_dim is None:
            raise ValueError("cross_attention_dim must be specified for CrossAttnDownBlock3D")
        kw.update(cross_attention_dim=cross_attention_dim, attn_num_head_channels=attn_num_head_channels,
                  dual_cross_attention=dual_cross_attention, use_linear_projection=use_linear_projection,
                  only_cross_attention=only_cross_attention, upcast_attention=upcast_attention)
    return _DOWN[down_block_type](**kw)


def get_up_block(up_block_type, num_layers, in_channels, out_channels, prev_output_channel, temb_channels, add_upsample,
                 resnet_eps, resnet_act_fn, attn_num_head_channels, resnet_groups=None, cross_attention_dim=None,
                 dual_cross_attention=False, use_linear_projection=True, only_cross_attention=False, upcast_attention=False,
                 resnet_time_scale_shift="default"):
    if up_block_type not in _UP:
        raise ValueError(f"{up_block_type} does not exist.")
    kw = dict(num_layers=num_layers, in_channels=in_channels, out_channels=out_channels, prev_output_channel=prev_output_channel,
              temb_channels=temb_channels, add_upsample=add_upsample, resnet_eps=resnet_eps, resnet_act_fn=resnet_act_fn,
              resnet_groups=resnet_groups, resnet_time_scale_shift=resnet_time_scale_shift)
    if up_block_type == "CrossAttnUpBlock3D":
        if cross_attention_dim is None:
            raise ValueError("cross_attention_dim must be specified for CrossAttnUpBlock3D")
        kw.update(cross_attention_dim=cross_attention_dim, attn_num_head_channels=attn_num_head_channels,
                  dual_cross_attention=dual_cross_attention, use_linear_projection=use_linear_projection,
                  only_cross_attention=only_cross_attention, upcast_attention=upcast_attention)
    return _UP[up_block_type](**kw)


def transformer_g_c(transformer, sample, num_frames, enabled=True):
    """(Checkpointed) call of a temporal transformer (reference helper of the same name, unet_3d_blocks.py:74-78)."""
    return _maybe_ckpt(enabled, lambda t: transformer(t, num_frames=num_frames).sample, sample)
