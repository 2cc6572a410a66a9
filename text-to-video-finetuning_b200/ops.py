"""Autograd layer of the hot path: every differentiable op is a torch.autograd.Function whose forward and backward
call the sm_90a kernels through prims.py.  PyTorch is used for tensor lifetime, streams and the autograd tape only.

Conventions
  * activations: bf16, channels-last; a frame batch is a 4-D tensor [N, H, W, C], a token matrix is [rows, C]
  * parameters stay fp32 `nn.Parameter`s with the diffusers names/shapes.  Conv weights are kept in torch
    channels_last memory format so that their storage *is* the [Cout, KH, KW, Cin] layout the kernels consume.
  * parameter gradients are accumulated by the kernels straight into `param.grad` (fp32, same physical layout);
    the Functions return None for them.  This is what lets the data-parallel step all-reduce one flat buffer.
  * fan-out of an activation is made explicit with `fork`, so gradient fan-in runs in our add kernel.
"""
import os

import torch
from torch.autograd import Function

from . import prims

# ---------------------------------------------------------------------------------------------------- parameters


def _phys(p):
    """The contiguous physical view of a weight: [Cout, KH, KW, Cin] for conv weights, [out, in] for linear."""
    if p.dim() == 4:
        v = p.permute(0, 2, 3, 1)
    elif p.dim() == 5:  # Conv3d (Cout, Cin, KT, 1, 1) -> [Cout, KT, 1, Cin]
        v = p.permute(0, 2, 3, 4, 1).reshape(p.shape[0], p.shape[2], p.shape[3] * p.shape[4], p.shape[1])
    elif p.dim() == 2:
        v = p.unsqueeze(1).unsqueeze(1)  # [out, 1, 1, in]
    else:
        raise ValueError(f"unsupported weight rank {p.dim()}")
    return v


class FusedWeight:
    """Several linear weights that sit back to back in the ParamArena (to_q|to_k|to_v of one Attention, or to_k|to_v for
    cross-attention) viewed as ONE [sum(out), 1, 1, in] matrix: one GEMM instead of three in forward, dgrad and wgrad."""

    def __init__(self, params, shadow, grad):
        self.params, self.shadow, self.grad = params, shadow, grad

    @property
    def requires_grad(self):
        return all(p.requires_grad for p in self.params)

    def usable(self):
        flags = {p.requires_grad for p in self.params}
        return len(flags) == 1   # all trainable or all frozen


class DeltaWeight:
    """A frozen conv weight plus a stable-LoRA delta, W_eff = base + scaling * view(B @ A) (utils/stable_lora.py): `_Conv`
    merges it into one bf16 weight (lora_delta.cu) and runs ONE GEMM with every epilogue of the plain conv; its backward
    projects the weight gradient onto A and B.  conv3d: the (3,1,1) view, which averages triples of B @ A."""

    def __init__(self, base, A, B, scaling, conv3d=False):
        self.base, self.A, self.B, self.scaling, self.conv3d = base, A, B, float(scaling), bool(conv3d)

    @property
    def requires_grad(self):
        return self.A.requires_grad or self.B.requires_grad

    def merged_bf16(self):
        return prims.lora_delta_merge(_cont(_phys(_f32(self.base))), _cont(_f32(self.A)), _cont(_f32(self.B)), self.scaling, self.conv3d)

    def grad_scratch(self):
        """Zeroed fp32 buffer in kernel layout for the gradient of W_eff (never the frozen base's own .grad)."""
        return torch.zeros(_phys(self.base).shape, device=self.base.device, dtype=torch.float32)

    def project_grad(self, dw, dA, dB):
        prims.lora_delta_grad(dw, _cont(_f32(self.A)), _cont(_f32(self.B)), self.scaling, self.conv3d, dA, dB)


def weight_bf16(p):
    """bf16 compute copy of a weight in kernel layout.  Uses the per-step flat shadow when the model has been
    prepared by runtime.ParamArena, otherwise casts on the fly (our cast kernel).  A DeltaWeight is merged here."""
    if isinstance(p, FusedWeight):
        return p.shadow
    if isinstance(p, DeltaWeight):
        return p.merged_bf16()
    sh = getattr(p, "_t2v_shadow", None)
    if sh is not None:
        return sh
    v = _phys(p.detach())
    if not v.is_contiguous():
        v = v.contiguous()
    if v.dtype == torch.bfloat16:
        return v
    return prims.cast_f32_bf16(v.float() if v.dtype != torch.float32 else v)


def grad_phys(p):
    """fp32 accumulation buffer for a weight, in kernel layout (allocates param.grad on first use)."""
    if isinstance(p, FusedWeight):
        return p.grad
    if p.grad is None:
        p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
    g = _phys(p.grad)
    if not g.is_contiguous() or g.dtype != torch.float32:
        raise RuntimeError("parameter gradients must be fp32 with the parameter's own memory format")
    return g


def grad_vec(p):
    if p.grad is None:
        p.grad = torch.zeros_like(p)
    if p.grad.dtype != torch.float32 or not p.grad.is_contiguous():
        raise RuntimeError("vector parameter gradients must be contiguous fp32")
    return p.grad


def _f32(p):
    if p is None:
        return None
    d = p.detach()
    return d if d.dtype == torch.float32 else d.float()


def _cont(t):
    return t if t.is_contiguous() else t.contiguous()


# ---------------------------------------------------------------------------------------------------- fork / add
class _Fork(Function):
    """y_1 = ... = y_n = x.  Backward sums the n incoming gradients with one kernel (instead of autograd's own)."""

    @staticmethod
    def forward(ctx, x, n):
        ctx.n = n
        return tuple(x.view_as(x) for _ in range(n))

    @staticmethod
    def backward(ctx, *gs):
        gs = [_cont(g) for g in gs if g is not None]
        if not gs:
            return None, None
        acc = gs[0]
        i = 1
        while i < len(gs):
            if i + 1 < len(gs):
                acc = prims.add_bf16(acc, gs[i], gs[i + 1])
                i += 2
            else:
                acc = prims.add_bf16(acc, gs[i])
                i += 1
        return acc, None


class _ForkF32(Function):
    """y_1 = ... = y_n = x with the n incoming gradients summed in fp32 (cast + add kernels) and rounded to bf16 once: the
    text states feed the cross-attention K|V projection of every UNet transformer, a fan-in too wide for a bf16 sum."""

    @staticmethod
    def forward(ctx, x, n):
        return tuple(x.view_as(x) for _ in range(n))

    @staticmethod
    def backward(ctx, *gs):
        gs = [_cont(g) for g in gs if g is not None]
        if not gs:
            return None, None
        acc = None
        for g in gs:
            g32 = torch.empty(g.shape, device=g.device, dtype=torch.float32)
            prims.cast_bf16_f32(g, g32)
            acc = g32 if acc is None else prims.add_f32(acc, g32)
        return prims.cast_f32_bf16(acc), None


def fork_f32(x, n):
    """fork(x, n) whose backward accumulates the gradient in fp32 (bf16 x only)."""
    if not x.requires_grad:
        return (x,) * n
    return _ForkF32.apply(x, n)


def carry(dst, src):
    """GroupNorm input statistics travel with the activation as a Python attribute (`_t2v_stats`: list of fp32 tensors
    [frames, Ck, 2] covering consecutive channel ranges, filled by the epilogue of the GEMM that produced the activation).
    Views and identity ops hand them on with this helper; anything that changes values simply does not."""
    st = getattr(src, "_t2v_stats", None)
    if st is not None:
        dst._t2v_stats = st
    return dst


def view(x, *shape):
    return carry(x.view(*shape), x)


def fork(x, n=2):
    if not x.requires_grad:
        return (x,) * n
    return tuple(carry(y, x) for y in _Fork.apply(x, n))


# ------------------------------------------------------------------------------------------- side stream for weight gradients
# Parameter gradients are leaves of the backward pass: nothing downstream in backward reads them.  Their kernels (wgrad
# GEMM + bias column sums, ~900 short launches per step) therefore run on a second stream, forked after the producer of dy
# and joined when the backward pass ends (and before a block's gradient range is all-reduced): on the GPU - and as a
# parallel branch of the captured CUDA graph - they fill the launch gaps and tails of the latency-bound main chain.
class _Side:
    enabled = not os.environ.get("T2V_NO_SIDE_WGRAD")
    streams = {}          # device index -> side stream
    pending = {}          # device index -> (main stream, tensors kept alive until the join)


def _side_join(dev_index):
    ent = _Side.pending.pop(dev_index, None)
    if ent is not None:
        main = ent[0]
        main.wait_stream(_Side.streams[dev_index])   # ent[1] (operand refs) dies here: memory is reused only after the join is enqueued


def join_side_streams():
    """Make the main stream(s) wait for every parameter-gradient kernel issued so far."""
    for d in list(_Side.pending):
        _side_join(d)


def _run_param_grads(fn, *keep):
    """Run fn() (kernels that only write parameter gradients) on the side stream of the current device."""
    t = keep[0]
    if not (_Side.enabled and t.is_cuda):
        fn()
        return
    d = t.device.index
    main = torch.cuda.current_stream(t.device)
    side = _Side.streams.get(d)
    if side is None:
        side = _Side.streams[d] = torch.cuda.Stream(device=t.device)
    task = torch._C._current_graph_task_id()   # one id per backward pass (-1 outside of one)
    ent = _Side.pending.get(d)
    if ent is None or ent[0] != main or ent[2] != task:
        if ent is not None:      # left over from another stream / an aborted backward pass
            _side_join(d)
        ent = _Side.pending[d] = (main, [], task)
        # join when this backward pass ends, whoever started it (also inside CUDA-graph capture and checkpoint recomputes)
        torch.autograd.Variable._execution_engine.queue_callback(lambda: _side_join(d))
    side.wait_stream(main)                 # fork: dy (and x) are complete on the main stream at this point
    with torch.cuda.stream(side):
        fn()
    ent[1].append(keep)                    # keep the operands alive: the caching allocator must not hand them out early


class _GradMark(Function):
    """Identity whose backward first calls `hook(key)`: placed on the main activation path at the input of a block, it
    fires once every gradient of that block (and of everything after it in forward order) has been launched - which is
    when runtime.GradientBuckets starts that block's share of the gradient all-reduce."""

    @staticmethod
    def forward(ctx, x, hook, key):
        ctx.hook, ctx.key = hook, key
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        join_side_streams()   # the block's parameter gradients must be complete before its range is all-reduced
        ctx.hook(ctx.key)
        return g, None, None


def grad_mark(x, hook, key):
    return carry(_GradMark.apply(x, hook, key), x) if hook is not None and x.requires_grad else x


# ---------------------------------------------------------------------------------------------------- conv / linear
class _Conv(Function):
    """y = conv(x, W) + bias + rowbias[n // rb_div] + residual on the wgmma implicit-GEMM kernel."""

    @staticmethod
    def forward(ctx, x, weight, bias, rowbias, residual, stride, pads, rb_div, out_fp32, cin_pad, cout_pad, alpha, anchor=None,
                stats_rows=0, stats_out=None):
        # `anchor`: a trainable tensor standing in for a FusedWeight (not a tensor) so that autograd still schedules
        # this node when x itself needs no gradient (cross-attention K|V projection of the text states)
        w = weight_bf16(weight)
        cin_pad = x.shape[-1] - w.shape[-1]        # boundary tensors arrive zero-padded to 8 channels
        cout_pad = (-w.shape[0]) % 8                # ... and leave padded to a multiple of 8
        if cin_pad or cout_pad:  # 3/4-channel boundary tensors are padded to 8 channels (TMA rows are >= 16 bytes)
            Co, KH, KW, Ci = w.shape
            wp = torch.zeros((Co + cout_pad, KH, KW, Ci + cin_pad), device=w.device, dtype=w.dtype)
            wp[:Co, :, :, :Ci] = w
            w = wp
        b = _f32(bias)
        if b is not None and cout_pad:
            b = torch.cat([b, b.new_zeros(cout_pad)])
        stats = None
        if stats_rows and stats_out is not None and not out_fp32 and not cout_pad:
            # GroupNorm statistics of y from the GEMM epilogue: one (sum, sum of squares) per frame and channel
            Ho, Wo = prims.out_hw(x.shape[1], x.shape[2], w.shape[1], w.shape[2], stride, pads)
            rows = x.shape[0] * Ho * Wo
            if rows % stats_rows == 0:
                stats = prims.stats_alloc(rows // stats_rows, w.shape[0], x.device)
                stats_out.append(stats)
        y = prims.conv_fwd(x, w, b, rowbias, residual, stride, pads, alpha, out_fp32, rb_div, stats=stats, stats_rows=stats_rows if stats is not None else 0)
        ctx.save_for_backward(x, w)
        ctx.weight, ctx.bias = weight, bias
        ctx.meta = (stride, pads, rb_div, cin_pad, cout_pad, rowbias.shape if rowbias is not None else None,
                    residual is not None, out_fp32, alpha)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        stride, pads, rb_div, cin_pad, cout_pad, rb_shape, has_res, out_fp32, alpha = ctx.meta
        weight, bias = ctx.weight, ctx.bias
        if out_fp32:
            dy = prims.silu_f32_to_bf16(_cont(dy), apply_silu=False)
        dy = _cont(dy)
        N, Ho, Wo, Co = dy.shape
        d_res = dy if (has_res and ctx.needs_input_grad[4]) else None
        if alpha != 1.0:
            assert rb_shape is None and bias is None, "alpha != 1 is only used by bias-free low-rank branches"
            dy = prims.scale_bf16(dy, alpha)
        d_rowbias = d_rowbias_full = None
        if rb_shape is not None and ctx.needs_input_grad[3]:
            d_rowbias_full = torch.zeros(rb_shape, device=dy.device, dtype=torch.float32)
            prims.colsum(dy, d_rowbias_full, rb_shape[0], (N // rb_shape[0]) * Ho * Wo, Co)
            d_rowbias = d_rowbias_full[:, :Co - cout_pad].contiguous() if cout_pad else d_rowbias_full
        # parameter gradients (bias column sums, weight gradient) are leaves: they run on the side stream
        gb = grad_vec(bias) if (bias is not None and bias.requires_grad) else None
        delta = isinstance(weight, DeltaWeight) and weight.requires_grad
        if delta:   # the wgrad lands in a scratch of W_eff's shape, then is projected onto the LoRA factors
            gw, gA, gB = weight.grad_scratch(), grad_vec(weight.A), grad_vec(weight.B)
        else:
            gw = grad_phys(weight) if weight.requires_grad else None

        def param_grads():
            # the plain bias gradient (column sums of dy) rides in the weight-gradient launch when both are wanted
            fuse_bias = gb is not None and gw is not None and not (cin_pad or cout_pad) and d_rowbias_full is None
            if gb is not None and not fuse_bias:
                if cout_pad:
                    tmp = torch.zeros(Co, device=dy.device, dtype=torch.float32)
                    prims.colsum(dy, tmp.view(1, Co), 1, N * Ho * Wo, Co)
                    gb.add_(tmp[:Co - cout_pad])
                elif d_rowbias_full is not None:
                    prims.colsum_f32(d_rowbias_full, gb)
                else:
                    prims.colsum(dy, gb.view(1, Co), 1, N * Ho * Wo, Co)
            if gw is not None:
                if cin_pad or cout_pad:
                    tmp = torch.zeros(w.shape, device=dy.device, dtype=torch.float32)
                    prims.conv_wgrad(x, dy, tmp, stride, pads)
                    gw.add_(tmp[:gw.shape[0], :, :, :gw.shape[3]])
                else:
                    prims.conv_wgrad(x, dy, gw, stride, pads, dbias=gb if fuse_bias else None)
                if delta:
                    weight.project_grad(gw, gA, gB)

        if gb is not None or gw is not None:
            _run_param_grads(param_grads, dy, x, d_rowbias_full, gw if delta else None)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = prims.conv_dgrad(dy, w, (x.shape[1], x.shape[2]), stride, pads)
        return dx, None, None, d_rowbias, d_res, None, None, None, None, None, None, None, None, None, None


def _with_stats(y, holder):
    if holder:
        y._t2v_stats = [holder[0]]
    return y


def conv(x, weight, bias=None, rowbias=None, residual=None, stride=1, pads=(1, 1, 1, 1), rb_div=1, out_fp32=False,
         cin_pad=0, cout_pad=0, alpha=1.0, stats_rows=0):
    """stats_rows > 0: also emit the per-(frame, channel) GroupNorm statistics of the output from the GEMM epilogue
    (stats_rows = output rows per frame); they ride on the returned tensor (see `carry`)."""
    holder = [] if stats_rows else None
    anchor = weight.A if isinstance(weight, DeltaWeight) and weight.requires_grad else None
    y = _Conv.apply(x, weight, bias, rowbias, residual, stride, tuple(pads), rb_div, out_fp32, cin_pad, cout_pad, float(alpha), anchor,
                    int(stats_rows), holder)
    return _with_stats(y, holder)


def linear(x, weight, bias=None, residual=None, out_fp32=False, alpha=1.0, stats_rows=0):
    """x [rows, in] -> [rows, out] through the same kernel (a 1x1 convolution over a rows x 1 image)."""
    rows, cin = x.shape
    res4 = residual.view(1, 1, rows, -1) if residual is not None else None
    anchor = weight.params[0] if isinstance(weight, FusedWeight) and weight.requires_grad else None
    holder = [] if stats_rows else None
    y = _Conv.apply(x.view(1, 1, rows, cin), weight, bias, None, res4, 1, (0, 0, 0, 0), 1, out_fp32, 0, 0, float(alpha), anchor,
                    int(stats_rows), holder)
    return _with_stats(y.view(rows, -1), holder)


# ---------------------------------------------------------------------------------------------------- norms
class _GroupNorm(Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, groups, eps, silu, samples, stats):
        shape = x.shape
        C = shape[-1]
        x3 = x.view(samples, -1, C)
        g32, b32 = _f32(gamma), _f32(beta)
        fps = 1
        if stats is not None:   # per-frame sums from the producer's epilogue; a sample spans fps frames (per-clip norms: F)
            frames = stats[0].shape[0]
            ok = (len(stats) <= 2 and frames % samples == 0 and sum(t.shape[1] for t in stats) == C
                  and all(t.shape[0] == frames and t.device == x.device for t in stats))
            fps = frames // samples if ok else 1
            stats = stats if ok else None
        y, stat, ab = prims.groupnorm_fwd(x3, g32, b32, groups, eps, silu, stats, fps)
        ctx.save_for_backward(x3, g32, stat, ab)
        ctx.gamma, ctx.beta = gamma, beta
        ctx.meta = (groups, silu, shape)
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        x3, g32, stat, ab = ctx.saved_tensors
        groups, silu, shape = ctx.meta
        dgamma = grad_vec(ctx.gamma) if ctx.gamma.requires_grad else None
        dbeta = grad_vec(ctx.beta) if ctx.beta.requires_grad else None
        dx = prims.groupnorm_bwd(_cont(dy).view(x3.shape), x3, g32, stat, ab, groups, silu, None, dgamma, dbeta)
        return dx.view(shape), None, None, None, None, None, None, None


_STATS_ENABLED = not os.environ.get("T2V_NO_EPILOGUE_STATS")   # A/B switch: GroupNorm computes its own sums


def group_norm(x, gamma, beta, groups, eps, silu, samples):
    """x [..., C] with `samples` independent normalisation samples (frames or clips) along the leading dims.  When the
    producer of x left its per-frame channel sums on the tensor (`carry`), the statistics pass is skipped."""
    stats = getattr(x, "_t2v_stats", None) if _STATS_ENABLED else None
    return _GroupNorm.apply(x, gamma, beta, groups, eps, silu, samples, stats)


class _LayerNorm(Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        g32, b32 = _f32(gamma), _f32(beta)
        y, stat = prims.layernorm_fwd(x, g32, b32, eps)
        ctx.save_for_backward(x, g32, stat)
        ctx.gamma, ctx.beta = gamma, beta
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g32, stat = ctx.saved_tensors
        dgamma = grad_vec(ctx.gamma) if ctx.gamma.requires_grad else None
        dbeta = grad_vec(ctx.beta) if ctx.beta.requires_grad else None
        return prims.layernorm_bwd(_cont(dy), x, g32, stat, None, dgamma, dbeta), None, None, None


def layer_norm(x, gamma, beta, eps=1e-5):
    return _LayerNorm.apply(x, gamma, beta, eps)


# ---------------------------------------------------------------------------------------------------- embeddings
class _EmbedTokens(Function):
    """x [B*L, C] bf16 = tok[ids] + pos[l] from the fp32 tables; the backward accumulates the tables' gradients (the trainable
    ones) with the deterministic embed_tokens_bwd kernel."""

    @staticmethod
    def forward(ctx, ids, tok, pos):
        ctx.save_for_backward(ids)
        ctx.tok, ctx.pos = tok, pos
        return prims.embed_tokens(ids, _cont(_f32(tok)), _cont(_f32(pos)))

    @staticmethod
    def backward(ctx, dy):
        ids, = ctx.saved_tensors
        tok, pos = ctx.tok, ctx.pos
        dtok = grad_vec(tok) if tok.requires_grad else None
        dpos = grad_vec(pos) if pos.requires_grad else None
        dy = _cont(dy)
        _run_param_grads(lambda: prims.embed_tokens_bwd(ids, dy, dtok, dpos, tok.shape[0]), dy, ids)
        return None, None, None


def embed_tokens(ids, tok, pos):
    """ids int64 [B, L] -> [B*L, C] bf16 (CLIPTextEmbeddings); differentiable in the token and position tables."""
    return _EmbedTokens.apply(ids, tok, pos)


# ---------------------------------------------------------------------------------------------------- activations
class _Geglu(Function):
    @staticmethod
    def forward(ctx, proj):
        ctx.save_for_backward(proj)
        return prims.geglu_fwd(proj)

    @staticmethod
    def backward(ctx, dout):
        (proj,) = ctx.saved_tensors
        return prims.geglu_bwd(proj, _cont(dout))


def geglu(proj):
    return _Geglu.apply(proj)


class _Silu(Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return prims.silu_bf16(x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return prims.silu_bf16_bwd(x, _cont(dy))


def silu(x):
    return _Silu.apply(x)


class _Gelu(Function):
    """The text encoder's MLP activation: exact erf GELU or CLIP's quick_gelu."""

    @staticmethod
    def forward(ctx, x, quick):
        ctx.save_for_backward(x)
        ctx.quick = quick
        return prims.gelu_bf16(x, quick=quick)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return prims.gelu_bwd(x, _cont(dy), quick=ctx.quick), None


def gelu(x, quick=False):
    return _Gelu.apply(x, bool(quick))


class _DropoutScaleAdd(Function):
    """base + scale * dropout_p(x) with a regenerated (not stored) mask."""

    @staticmethod
    def forward(ctx, x, base, p, scale, seed):
        ctx.meta = (p, scale, seed, base is not None)
        return prims.dropout_scale_add(x, base, p, scale, seed, dropout_epoch(x.device))

    @staticmethod
    def backward(ctx, dy):
        p, scale, seed, has_base = ctx.meta
        dy = _cont(dy)
        return prims.dropout_scale_add(dy, None, p, scale, seed, dropout_epoch(dy.device)), (dy if has_base else None), None, None, None


# Dropout masks are a pure function of (host seed, device epoch, element index).
#   * host seed: drawn from torch's default CPU generator at the call site.  Inside an activation-checkpointed sub-module the
#     seeds derive instead from ONE base seed drawn outside the checkpointed function and handed to it as an argument
#     (dropout_seed_scope), so the recomputed forward draws the SAME seeds and its activations match the masks the first
#     forward (and the backward) used - without touching torch's RNG-state save/restore (not capturable in a CUDA graph).
#   * device epoch: an int64 counter in device memory, bumped once per training step (step.DataParallelStep) and read by the
#     kernel when it RUNS - a replayed CUDA graph (whose host seeds are baked in at capture) gets fresh masks every step.
_epochs = {}


def dropout_epoch(device):
    device = torch.device(device)
    key = (device.type, device.index)
    t = _epochs.get(key)
    if t is None:
        t = _epochs[key] = torch.zeros(1, device=device, dtype=torch.int64)
    return t


def bump_dropout_epoch(device):
    prims.counter_add(dropout_epoch(device), 1)


import contextlib
import threading

_seed_scope = threading.local()


@contextlib.contextmanager
def dropout_seed_scope(base):
    """Inside the scope the n-th dropout call site gets seed splitmix(base, n) - a pure function of `base`."""
    prev = getattr(_seed_scope, "state", None)
    _seed_scope.state = [int(base), 0]
    try:
        yield
    finally:
        _seed_scope.state = prev


def next_dropout_seed():
    st = getattr(_seed_scope, "state", None)
    if st is None:
        return int(torch.randint(0, 1 << 62, (1,)).item())
    st[1] += 1
    z = (st[0] + st[1] * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return (z ^ (z >> 31)) >> 2


def dropout_scale_add(x, base, p, scale=1.0, seed=None):
    return _DropoutScaleAdd.apply(x, base, float(p), float(scale), next_dropout_seed() if seed is None else seed)


def dropout(x, p, seed=None):
    return _DropoutScaleAdd.apply(x, None, float(p), 1.0, next_dropout_seed() if seed is None else seed)


# ---------------------------------------------------------------------------------------------------- resampling / concat
class _Upsample(Function):
    @staticmethod
    def forward(ctx, x, out_hw):
        ctx.in_hw = (x.shape[1], x.shape[2])
        return prims.upsample_nearest_fwd(x, out_hw)

    @staticmethod
    def backward(ctx, dy):
        return prims.upsample_nearest_bwd(_cont(dy), ctx.in_hw), None


def upsample_nearest(x, out_hw):
    return _Upsample.apply(x, tuple(out_hw))


class _Concat(Function):
    @staticmethod
    def forward(ctx, a, b):
        ctx.ca = a.shape[-1]
        return prims.concat_channels(a, b)

    @staticmethod
    def backward(ctx, g):
        return prims.split_channels(_cont(g), ctx.ca)


def concat_channels(a, b):
    out = _Concat.apply(a, b)
    sa, sb = getattr(a, "_t2v_stats", None), getattr(b, "_t2v_stats", None)
    if sa is not None and sb is not None and len(sa) == 1 and len(sb) == 1:
        out._t2v_stats = [sa[0], sb[0]]   # channel ranges [0, Ca) and [Ca, Ca + Cb)
    return out


# ---------------------------------------------------------------------------------------------------- attention
def _rup8(n):
    return (n + 7) // 8 * 8


class _Flash:
    # Fused attention kernels (csrc/flash_attn.cu) are the default path for head_dim 64 (every attention of the UNet);
    # T2V_NO_FLASH_ATTN=1 selects the unfused bgemm / softmax / bgemm path (A/B switch, also what other head dims use).
    enabled = not os.environ.get("T2V_NO_FLASH_ATTN")


def _use_flash(q, heads):
    return _Flash.enabled and q.shape[-1] // heads == 64


def _attn_core_fwd(q, k, v, heads):
    """q [Nb, Lq, C], k/v [Nb, Lk, C]: row-contiguous views (arbitrary row pitch).  Returns (o contiguous, aux) where aux is
    the bf16 probability tensor P of the unfused path, or the fp32 log-sum-exp of the fused (flash) path."""
    if _use_flash(q, heads):
        return prims.flash_attn_fwd(q, k, v, heads)
    Nb, Lq, C = q.shape
    Lk = k.shape[1]
    D = C // heads
    ld = _rup8(Lk)
    scale = D ** -0.5
    s = torch.empty((Nb, heads, Lq, ld), device=q.device, dtype=torch.float32)
    prims.bgemm(q, (1, q.stride(1), q.stride(0), D), k, (1, k.stride(1), k.stride(0), D), s, (ld, heads * Lq * ld, Lq * ld),
                Lq, Lk, D, Nb, heads, scale, 1)
    p = prims.softmax_fwd(s, Lk, ld)
    del s
    o = torch.empty((Nb, Lq, C), device=q.device, dtype=q.dtype)
    prims.bgemm(p, (1, ld, heads * Lq * ld, Lq * ld), v, (0, v.stride(1), v.stride(0), D), o, (C, Lq * C, D), Lq, D, Lk, Nb, heads, 1.0, 0)
    return o, p


def _attn_core_bwd(q, k, v, p, do, dq, dk, dv, heads, o=None):
    """Gradients of _attn_core_fwd written into the (row-contiguous, possibly column-sliced) views dq / dk / dv.
    `p` is the aux tensor of the forward pass; an fp32 aux is the log-sum-exp of the fused path (which also needs `o`)."""
    if p.dtype == torch.float32 and p.dim() == 3:
        prims.flash_attn_bwd(q, k, v, o, do, p, heads, dq, dk, dv)
        return
    Nb, Lq, C = q.shape
    Lk = k.shape[1]
    D = C // heads
    ld = p.shape[-1]
    scale = D ** -0.5
    pd = (ld, heads * Lq * ld, Lq * ld)
    dod = (do.stride(1), do.stride(0), D)
    # dV = P^T dO and dK = dS^T Q contract over Lq.  For cross-attention (Lq = F*H*W >> Lk = 77) there are only
    # Nb*heads output tiles, so those two run split-K into an fp32 buffer (red.add) followed by one cast.
    split = Lq >= 2048 and Lk <= 256

    def over_lq(a_mat, b_mat, out):
        bd = (0, b_mat.stride(1), b_mat.stride(0), D)
        if not split:
            prims.bgemm(a_mat, (0,) + pd, b_mat, bd, out, (out.stride(1), out.stride(0), D), Lk, D, Lq, Nb, heads, 1.0, 0)
            return
        acc = torch.zeros((Nb, Lk, C), device=out.device, dtype=torch.float32)
        prims.bgemm(a_mat, (0,) + pd, b_mat, bd, acc, (C, Lk * C, D), Lk, D, Lq, Nb, heads, 1.0, 2)
        if out.is_contiguous():
            prims.cast_f32_bf16(acc, out)
        else:
            out.copy_(prims.cast_f32_bf16(acc))

    over_lq(p, do, dv)
    dp = torch.empty((Nb, heads, Lq, ld), device=q.device, dtype=torch.float32)  # dP = dO V^T
    prims.bgemm(do, (1,) + dod, v, (1, v.stride(1), v.stride(0), D), dp, pd, Lq, Lk, D, Nb, heads, 1.0, 1)
    ds = prims.softmax_bwd(p, dp, Lk, scale)
    del dp
    prims.bgemm(ds, (1,) + pd, k, (0, k.stride(1), k.stride(0), D), dq, (dq.stride(1), dq.stride(0), D), Lq, D, Lk, Nb, heads, 1.0, 0)  # dQ = dS K
    over_lq(ds, q, dk)                                                                                                                   # dK = dS^T Q


class _Attention(Function):
    """softmax(q k^T / sqrt(d)) v for token matrices q [Nb, Lq, H*D], k/v [Nb, Lk, H*D]; the four contractions run
    as batched GEMMs on the wgmma kernel, the row softmax in between as one HBM-bound pass."""

    @staticmethod
    def forward(ctx, q, k, v, heads):
        o, p = _attn_core_fwd(q, k, v, heads)
        ctx.save_for_backward(q, k, v, p, o)
        ctx.heads = heads
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, p, o = ctx.saved_tensors
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _attn_core_bwd(q, k, v, p, _cont(do), dq, dk, dv, ctx.heads, o)
        return dq, dk, dv, None


def attention(q, k, v, heads):
    return _Attention.apply(q, k, v, heads)


def causal_attention_fwd(q, k, v, heads):
    """CLIP text self-attention, q/k/v [B, L, C] row-contiguous views: two batched GEMMs around the row softmax with the
    causal mask (L = 77: launch-bound, no fused kernel).  Returns (o [B, L, C] bf16, P bf16 [B, heads, L, ld])."""
    B, L, C = q.shape
    D = C // heads
    ld = _rup8(L)
    s = torch.empty((B, heads, L, ld), device=q.device, dtype=torch.float32)
    prims.bgemm(q, (1, q.stride(1), q.stride(0), D), k, (1, k.stride(1), k.stride(0), D), s, (ld, heads * L * ld, L * ld),
                L, L, D, B, heads, D ** -0.5, 1)
    p = prims.softmax_fwd(s, L, ld, causal_period=L)
    del s
    o = torch.empty((B, L, C), device=q.device, dtype=q.dtype)
    prims.bgemm(p, (1, ld, heads * L * ld, L * ld), v, (0, v.stride(1), v.stride(0), D), o, (C, L * C, D), L, D, L, B, heads, 1.0, 0)
    return o, p


class _CausalAttention(Function):
    """Backward: the unfused path of _attn_core_bwd on the stored probabilities; the masked ones are zero, so softmax_bwd
    gives them a zero score gradient and the four GEMMs need no mask."""

    @staticmethod
    def forward(ctx, q, k, v, heads):
        o, p = causal_attention_fwd(q, k, v, heads)
        ctx.save_for_backward(q, k, v, p)
        ctx.heads = heads
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, p = ctx.saved_tensors
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _attn_core_bwd(q, k, v, p, _cont(do), dq, dk, dv, ctx.heads)
        return dq, dk, dv, None


def causal_attention(q, k, v, heads):
    return _CausalAttention.apply(q, k, v, heads)


class _AttentionFused(Function):
    """Same attention on fused projections: self-attention takes qkv [Nb, L, 3C] (kv None), cross-attention takes
    q [Nb, Lq, C] and kv [Nb, Lk, 2C].  q / k / v are column slices of those buffers (no copies), and the gradient is
    produced directly in the fused layout, so autograd never sees the slicing."""

    @staticmethod
    def forward(ctx, qkv, kv, heads):
        if kv is None:
            C = qkv.shape[-1] // 3
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        else:
            C = qkv.shape[-1]
            q, k, v = qkv, kv[..., :C], kv[..., C:]
        o, p = _attn_core_fwd(q, k, v, heads)
        ctx.save_for_backward(qkv, kv, p, o)
        ctx.heads = heads
        return o

    @staticmethod
    def backward(ctx, do):
        qkv, kv, p, o = ctx.saved_tensors
        dqkv = torch.empty_like(qkv)
        if kv is None:
            C = qkv.shape[-1] // 3
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
            dq, dk, dv = dqkv[..., :C], dqkv[..., C:2 * C], dqkv[..., 2 * C:]
            dkv = None
        else:
            C = qkv.shape[-1]
            dkv = torch.empty_like(kv)
            q, k, v = qkv, kv[..., :C], kv[..., C:]
            dq, dk, dv = dqkv, dkv[..., :C], dkv[..., C:]
        _attn_core_bwd(q, k, v, p, _cont(do), dq, dk, dv, ctx.heads, o)
        return dqkv, dkv, None


def attention_fused(qkv, kv, heads):
    return _AttentionFused.apply(qkv, kv, heads)


def _temporal_addr(B, F, HW, heads, D, ld_in, ld_out):
    # frames-major tokens: row of (b, f, hw) = (b*F + f)*HW + hw; a sequence runs over f with b, hw fixed
    return (B * HW, HW, F * HW, 1, HW, ld_in, ld_out, heads, F, D)


SMALL_TEMPORAL_MAX = 32   # clips of up to this many frames use attn_small (a warp per sequence); longer ones attn_long
MAX_FRAMES = 256          # attn_long keeps a whole sequence of q, k, v, dO in one CTA's shared memory


class _TemporalAttention(Function):
    """Self-attention along the frame axis on frames-major tokens [B*F*HW, H*D] (no permute; see attn_small.cu).
    `fused`: q is the [rows, 3C] QKV projection and k, v are None.  F <= 32 runs attn_small; 32 < F <= 256 runs attn_long,
    whose backward also needs the forward's o and row logsumexp."""

    @staticmethod
    def forward(ctx, q, k, v, heads, B, F, HW, fused):
        if fused:
            C = q.shape[-1] // 3
            qq, kk, vv = q[:, :C], q[:, C:2 * C], q[:, 2 * C:]
        else:
            C = q.shape[-1]
            qq, kk, vv = q, k, v
        addr = _temporal_addr(B, F, HW, heads, C // heads, q.shape[-1], C)
        o = torch.empty((q.shape[0], C), device=q.device, dtype=q.dtype)
        ctx.addr, ctx.fused, ctx.long = addr, fused, F > SMALL_TEMPORAL_MAX
        if ctx.long:
            lse = torch.empty((B * HW, heads, F), device=q.device, dtype=torch.float32)
            prims.attn_long_fwd(qq, kk, vv, o, lse, addr)
            ctx.save_for_backward(q, k, v, o, lse)
        else:
            prims.attn_small_fwd(qq, kk, vv, o, addr)
            ctx.save_for_backward(q, k, v)
        return o

    @staticmethod
    def backward(ctx, do):
        if ctx.long:
            q, k, v, o, lse = ctx.saved_tensors
            bwd = lambda q_, k_, v_, do_, dq_, dk_, dv_, addr: prims.attn_long_bwd(q_, k_, v_, o, do_, lse, dq_, dk_, dv_, addr)
        else:
            q, k, v = ctx.saved_tensors
            bwd = prims.attn_small_bwd
        do = _cont(do)
        if ctx.fused:
            C = q.shape[-1] // 3
            dqkv = torch.empty_like(q)
            bwd(q[:, :C], q[:, C:2 * C], q[:, 2 * C:], do, dqkv[:, :C], dqkv[:, C:2 * C], dqkv[:, 2 * C:], ctx.addr)
            return dqkv, None, None, None, None, None, None, None
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        bwd(q, k, v, do, dq, dk, dv, ctx.addr)
        return dq, dk, dv, None, None, None, None, None


def temporal_attention(q, k, v, heads, B, F, HW):
    return _TemporalAttention.apply(q, k, v, heads, B, F, HW, False)


def temporal_attention_fused(qkv, heads, B, F, HW):
    return _TemporalAttention.apply(qkv, None, None, heads, B, F, HW, True)


# ---------------------------------------------------------------------------------------------------- latent boundary
class _FromNhwc8(Function):
    """[B*F, H, W, 8] bf16 -> (B, C, F, H, W) fp32 (the `.sample` layout of UNet3DConditionModel.forward)."""

    @staticmethod
    def forward(ctx, x, B, C, F):
        ctx.meta = (B, C, F)
        return prims.nhwc8_to_latents(x, B, C, F)

    @staticmethod
    def backward(ctx, g):
        return prims.latents_to_nhwc8(_cont(g.float())), None, None, None


def from_nhwc8(x, B, C, F):
    return _FromNhwc8.apply(x, B, C, F)


class _MseLoss(Function):
    """mean((pred - target)^2) in fp32 straight from the channels-last prediction (train.py:827)."""

    @staticmethod
    def forward(ctx, pred, target):
        ctx.save_for_backward(pred, target)
        return prims.mse_loss_fwd(pred, target)

    @staticmethod
    def backward(ctx, g):
        pred, target = ctx.saved_tensors
        return prims.mse_loss_bwd(pred, target, _cont(g.float())), None


def mse_loss_nhwc8(pred, target):
    return _MseLoss.apply(pred, target)


class _VelocityMseLoss(Function):
    """mean((pred - v)^2) in fp32 for a v-prediction model (train.py:792-800): the velocity target
    sqrt(abar[t]) noise - sqrt(1 - abar[t]) x0 is formed inside the loss kernel, never stored."""

    @staticmethod
    def forward(ctx, pred, x0, noise, alphas_cumprod, timesteps):
        ctx.save_for_backward(pred, x0, noise, alphas_cumprod, timesteps)
        return prims.velocity_mse_loss_fwd(pred, x0, noise, alphas_cumprod, timesteps)

    @staticmethod
    def backward(ctx, g):
        pred, x0, noise, abar, t = ctx.saved_tensors
        return prims.velocity_mse_loss_bwd(pred, x0, noise, abar, t, _cont(g.float())), None, None, None, None


def velocity_mse_loss_nhwc8(pred, x0, noise, alphas_cumprod, timesteps):
    return _VelocityMseLoss.apply(pred, x0, noise, alphas_cumprod, timesteps)


class _DiffusionLoss(Function):
    """The Min-SNR-gamma weighted and / or pseudo-Huber objective of a step.LossObjective (snr_gamma, loss_type,
    huber_schedule, huber_c), forward and backward in one kernel each: the noise target, or the velocity when x0 is given."""

    @staticmethod
    def forward(ctx, pred, x0, noise, alphas_cumprod, timesteps, objective):
        ctx.objective = objective
        ctx.save_for_backward(pred, x0, noise, alphas_cumprod, timesteps)
        return prims.diffusion_loss_fwd(pred, x0, noise, alphas_cumprod, timesteps, objective)

    @staticmethod
    def backward(ctx, g):
        pred, x0, noise, abar, t = ctx.saved_tensors
        return prims.diffusion_loss_bwd(pred, x0, noise, abar, t, ctx.objective, _cont(g.float())), None, None, None, None, None


def diffusion_loss_nhwc8(pred, x0, noise, alphas_cumprod, timesteps, objective):
    """x0: the clean latents for a v-prediction model, None for epsilon."""
    return _DiffusionLoss.apply(pred, x0, noise, alphas_cumprod, timesteps, objective)
