"""Tensor-level wrappers over the C ABI (include/t2v_b200.h): each function takes/returns torch CUDA tensors, allocates
outputs with PyTorch's caching allocator and launches on torch's current stream.  No autograd here (see ops.py) and
no fallback: every function ends in a native call.

Layout contract: activations are bf16 channels-last `[N, H, W, C]` (or `[rows, C]` token matrices), convolution
weights are bf16 `[Cout, KH, KW, Cin]`, statistics / biases / parameter gradients are fp32.
"""
import ctypes

import torch

from . import native

_VP = ctypes.c_void_p


def _p(t):
    return _VP(0) if t is None else _VP(t.data_ptr())


def _stream():
    return _VP(torch.cuda.current_stream().cuda_stream)


def _chk_bf16(*ts):
    for t in ts:
        if t is not None:
            assert t.dtype == torch.bfloat16 and t.is_contiguous() and t.is_cuda, (t.dtype, t.shape, t.stride(), t.device)


def _chk_f32(*ts):
    for t in ts:
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda, (t.dtype, t.shape, t.stride())


def out_hw(H, W, KH, KW, stride, pads):
    return (H + pads[0] + pads[1] - KH) // stride + 1, (W + pads[2] + pads[3] - KW) // stride + 1


# ---------------------------------------------------------------------------------------------- tensor-core family
def _conv_scratch(dgrad, N, H, W, Ci, Co, KH, KW, stride, pads, device):
    """fp32 scratch the planner asks for when it wants to split the reduction of a few-tile problem over the SMs."""
    n = native.lib().t2v_conv_workspace_bytes(dgrad, N, H, W, Ci, Co, KH, KW, stride, *pads)
    if n <= 0:
        return None, 0
    return torch.empty(n // 4, device=device, dtype=torch.float32), n


def conv_fwd(x, w, bias=None, rowbias=None, residual=None, stride=1, pads=(0, 0, 0, 0), alpha=1.0, out_fp32=False, rowbias_div=1,
             stats=None, stats_rows=0):
    """x [N,H,W,Ci] bf16, w [Co,KH,KW,Ci] bf16 -> y [N,Ho,Wo,Co]; y = alpha*conv + bias[c] + rowbias[n,c] + residual.
    stats: zeroed fp32 [frames, Co, 2] to receive the per-(frame, channel) sum / sum of squares of y (GroupNorm input
    statistics from the GEMM epilogue), stats_rows = output rows per frame."""
    _chk_bf16(x, w, residual)
    _chk_f32(bias, rowbias)
    N, H, W, Ci = x.shape
    Co, KH, KW, Ci2 = w.shape
    assert Ci == Ci2, (x.shape, w.shape)
    Ho, Wo = out_hw(H, W, KH, KW, stride, pads)
    y = torch.empty((N, Ho, Wo, Co), device=x.device, dtype=torch.float32 if out_fp32 else torch.bfloat16)
    ws, ws_bytes = _conv_scratch(0, N, H, W, Ci, Co, KH, KW, stride, pads, x.device)
    epi = native.Epilogue(bias.data_ptr() if bias is not None else None, rowbias.data_ptr() if rowbias is not None else None,
                          residual.data_ptr() if residual is not None else None, float(alpha), int(out_fp32), int(rowbias_div),
                          ws.data_ptr() if ws is not None else None, ws_bytes,
                          stats.data_ptr() if stats is not None else None, Co, int(stats_rows), 0)
    if stats is not None:
        _chk_f32(stats)
        assert stats.shape[1:] == (Co, 2) and stats.shape[0] * stats_rows == N * Ho * Wo, (stats.shape, stats_rows, (N, Ho, Wo, Co))
    native.check(native.lib().t2v_conv_fwd(_p(x), _p(w), _p(y), N, H, W, Ci, Co, KH, KW, stride, *pads, ctypes.byref(epi), _stream()))
    return y


def conv_dgrad(dy, w, in_hw, stride=1, pads=(0, 0, 0, 0), residual=None):
    """dy [N,Ho,Wo,Co] -> dx [N,H,W,Ci] (+ residual, which may alias nothing)."""
    _chk_bf16(dy, w, residual)
    N = dy.shape[0]
    H, W = in_hw
    Co, KH, KW, Ci = w.shape
    dx = torch.empty((N, H, W, Ci), device=dy.device, dtype=torch.bfloat16)
    ws, ws_bytes = _conv_scratch(1, N, H, W, Ci, Co, KH, KW, stride, pads, dy.device)
    epi = native.Epilogue(None, None, residual.data_ptr() if residual is not None else None, 1.0, 0, 1,
                          ws.data_ptr() if ws is not None else None, ws_bytes)
    native.check(native.lib().t2v_conv_dgrad(_p(dy), _p(w), _p(dx), N, H, W, Ci, Co, KH, KW, stride, *pads, ctypes.byref(epi), _stream()))
    return dx


def conv_wgrad(x, dy, dw, stride=1, pads=(0, 0, 0, 0), dbias=None):
    """dw [Co,KH,KW,Ci] fp32 += dy^T * shifted(x);  dbias [Co] fp32 += column sums of dy (the layer's bias gradient, produced by
    the same launch whenever the tiling allows - include/t2v_b200.h)."""
    _chk_bf16(x, dy)
    _chk_f32(dw, dbias)
    N, H, W, Ci = x.shape
    Co, KH, KW, Ci2 = dw.shape
    assert Ci2 == Ci and dy.shape[-1] == Co
    if dbias is None:
        native.check(native.lib().t2v_conv_wgrad(_p(x), _p(dy), _p(dw), N, H, W, Ci, Co, KH, KW, stride, *pads, _stream()))
    else:
        assert dbias.numel() == Co and dbias.is_contiguous()
        native.check(native.lib().t2v_conv_wgrad_bias(_p(x), _p(dy), _p(dw), _p(dbias), N, H, W, Ci, Co, KH, KW, stride, *pads, _stream()))


def _mat(t, kmajor, ld, s1, s2):
    return native.Mat(t.data_ptr(), ld, s1, s2, int(kmajor))


def bgemm(a, a_desc, b, b_desc, c, c_desc, M, N, K, Z1, Z2, alpha=1.0, out_mode=0):
    """Raw strided-batched GEMM; *_desc = (kmajor, ld, stride_z1, stride_z2) / c_desc = (ld, stride_z1, stride_z2)."""
    mA, mB = _mat(a, *a_desc), _mat(b, *b_desc)
    native.check(native.lib().t2v_bgemm(ctypes.byref(mA), ctypes.byref(mB), _p(c), c_desc[0], c_desc[1], c_desc[2],
                                        M, N, K, Z1, Z2, float(alpha), out_mode, _stream()))


def flash_attn_fwd(q, k, v, heads):
    """Fused attention forward (head_dim 64).  q [Nb, Lq, C], k / v [Nb, Lk, C] bf16 row-contiguous views (column slices of
    fused projections allowed).  Returns o [Nb, Lq, C] bf16 and lse [Nb, heads, Lq] fp32."""
    for t in (q, k, v):
        assert t.dtype == torch.bfloat16 and t.is_cuda and t.dim() == 3 and t.stride(2) == 1, (t.dtype, t.shape, t.stride())
    Nb, Lq, C = q.shape
    Lk = k.shape[1]
    o = torch.empty((Nb, Lq, C), device=q.device, dtype=torch.bfloat16)
    lse = torch.empty((Nb, heads, Lq), device=q.device, dtype=torch.float32)
    native.check(native.lib().t2v_flash_attn_fwd(_p(q), _p(k), _p(v), _p(o), _p(lse), Nb, heads, Lq, Lk, C // heads, q.stride(1),
                                                 q.stride(0), k.stride(1), k.stride(0), v.stride(1), v.stride(0), o.stride(1),
                                                 o.stride(0), _stream()))
    return o, lse


def flash_attn_bwd(q, k, v, o, do, lse, heads, dq, dk, dv):
    """Gradients of flash_attn_fwd written into the (possibly column-sliced) views dq / dk / dv."""
    for t in (q, k, v, dq, dk, dv):
        assert t.dtype == torch.bfloat16 and t.is_cuda and t.dim() == 3 and t.stride(2) == 1, (t.dtype, t.shape, t.stride())
    _chk_bf16(o, do)
    _chk_f32(lse)
    Nb, Lq, C = q.shape
    Lk = k.shape[1]
    delta = torch.empty((Nb, heads, Lq), device=q.device, dtype=torch.float32)
    splits = native.lib().t2v_flash_attn_bwd_splits(Nb, heads, Lq, Lk)
    ws = torch.zeros((2, Nb, Lk, C), device=q.device, dtype=torch.float32) if splits > 1 else None
    native.check(native.lib().t2v_flash_attn_bwd(_p(q), _p(k), _p(v), _p(o), _p(do), _p(lse), _p(dq), _p(dk), _p(dv), _p(delta), _p(ws),
                                                 Nb, heads, Lq, Lk, C // heads, q.stride(1), q.stride(0), k.stride(1), k.stride(0),
                                                 v.stride(1), v.stride(0), o.stride(1), o.stride(0), dq.stride(1), dq.stride(0),
                                                 dk.stride(1), dk.stride(0), dv.stride(1), dv.stride(0), _stream()))
    if ws is not None:   # few keys, many queries: the kernel reduced fp32 partials; round once into the bf16 gradients
        for dst, src in ((dk, ws[0]), (dv, ws[1])):
            if dst.is_contiguous():
                cast_f32_bf16(src, dst)
            else:
                dst.copy_(cast_f32_bf16(src))


# ---------------------------------------------------------------------------------------------- norms
class _ZeroPool:
    """Zero-initialised fp32 scratch for red.add targets (GroupNorm statistics / gradient sums): slices of 4 MB chunks, one
    memset per chunk instead of one per call.  A slice is handed out once; a chunk dies with its last slice.  A chunk never
    crosses a CUDA-graph capture boundary (its memset belongs to exactly one graph, or to none)."""
    CHUNK = 1 << 20

    def __init__(self):
        self.state = {}   # device -> [chunk, pos, capture id]

    def take(self, n, device):
        n = (n + 63) // 64 * 64
        if n > self.CHUNK:
            return torch.zeros(n, device=device, dtype=torch.float32)
        cap = native.lib().t2v_stream_capture_id(_stream()) if device.type == "cuda" else 0
        st = self.state.get(device)
        if st is None or st[2] != cap or st[1] + n > self.CHUNK:
            st = self.state[device] = [torch.zeros(self.CHUNK, device=device, dtype=torch.float32), 0, cap]
        out = st[0][st[1]:st[1] + n]
        st[1] += n
        return out


_zero_pool = _ZeroPool()


def zeros_f32(shape, device):
    n = 1
    for d in shape:
        n *= d
    return _zero_pool.take(n, torch.device(device))[:n].view(shape)


def stats_alloc(frames, C, device):
    """Zeroed [frames, C, 2] buffer for epilogue statistics (conv_fwd(stats=...))."""
    return zeros_f32((frames, C, 2), device)


def channel_stats(x):
    """x [S,P,C] bf16 -> per-sample, per-channel (sum, sum of squares) [S,C,2] fp32: the statistics pass on its own."""
    _chk_bf16(x)
    S, P, C = x.shape
    st = stats_alloc(S, C, x.device)
    native.check(native.lib().t2v_channel_stats(_p(x), _p(st), S, P, C, C, _stream()))
    return st


def groupnorm_fwd(x, gamma, beta, G, eps, silu, stats=None, fps=1):
    """x [S,P,C] bf16 -> y, stat [S,G,2], ab [S,C,2].  stats: None (the kernel computes the sums itself) or a list of one or
    two fp32 tensors [S*fps, Ck, 2] with the per-frame sums of consecutive channel ranges (sum Ck == C) as produced by
    conv_fwd(stats=...); fps = frames per normalisation sample."""
    _chk_bf16(x)
    _chk_f32(gamma, beta)
    S, P, C = x.shape
    y = torch.empty_like(x)
    stat = torch.empty((S, G, 2), device=x.device, dtype=torch.float32)
    ab = torch.empty((S, C, 2), device=x.device, dtype=torch.float32)
    if stats:
        s0 = stats[0]
        s1 = stats[1] if len(stats) > 1 else None
        _chk_f32(s0, s1)
        C0 = s0.shape[1]
        assert s0.shape[0] == S * fps and C0 + (s1.shape[1] if s1 is not None else 0) == C, (s0.shape, S, fps, C)
        native.check(native.lib().t2v_groupnorm_fwd(_p(x), _p(gamma), _p(beta), _p(y), _p(stat), _p(ab), _p(s0), C0, C0, _p(s1),
                                                    s1.shape[1] if s1 is not None else 0, fps, _p(None), S, P, C, G, float(eps), int(silu),
                                                    _stream()))
    else:
        ws = zeros_f32((S, C, 2), x.device)
        native.check(native.lib().t2v_groupnorm_fwd(_p(x), _p(gamma), _p(beta), _p(y), _p(stat), _p(ab), _p(None), 0, 0, _p(None), 0, 1,
                                                    _p(ws), S, P, C, G, float(eps), int(silu), _stream()))
    return y, stat, ab


def groupnorm_bwd(dy, x, gamma, stat, ab, G, silu, add=None, dgamma=None, dbeta=None):
    _chk_bf16(dy, x, add)
    S, P, C = x.shape
    dx = torch.empty_like(x)
    ws = zeros_f32((S, C, 2), x.device)   # per-channel sums (red.add targets: zero on entry)
    native.check(native.lib().t2v_groupnorm_bwd(_p(dy), _p(x), _p(gamma), _p(stat), _p(ab), _p(add), _p(dx), _p(dgamma), _p(dbeta),
                                                _p(ws), S, P, C, G, int(silu), _stream()))
    return dx


def layernorm_fwd(x, gamma, beta, eps):
    _chk_bf16(x)
    rows, C = x.shape
    y = torch.empty_like(x)
    stat = torch.empty((rows, 2), device=x.device, dtype=torch.float32)
    native.check(native.lib().t2v_layernorm_fwd(_p(x), _p(gamma), _p(beta), _p(y), _p(stat), rows, C, float(eps), _stream()))
    return y, stat


def layernorm_bwd(dy, x, gamma, stat, add=None, dgamma=None, dbeta=None):
    _chk_bf16(dy, x, add)
    rows, C = x.shape
    dx = torch.empty_like(x)
    native.check(native.lib().t2v_layernorm_bwd(_p(dy), _p(x), _p(gamma), _p(stat), _p(add), _p(dx), _p(dgamma), _p(dbeta), rows, C, _stream()))
    return dx


# ---------------------------------------------------------------------------------------------- elementwise / glue
def geglu_fwd(proj):
    _chk_bf16(proj)
    M, I2 = proj.shape
    out = torch.empty((M, I2 // 2), device=proj.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_geglu_fwd(_p(proj), _p(out), M, I2 // 2, _stream()))
    return out


def geglu_bwd(proj, dout):
    _chk_bf16(proj, dout)
    M, I2 = proj.shape
    dproj = torch.empty_like(proj)
    native.check(native.lib().t2v_geglu_bwd(_p(proj), _p(dout), _p(dproj), M, I2 // 2, _stream()))
    return dproj


def silu_f32_to_bf16(x, apply_silu=True):
    _chk_f32(x)
    y = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_silu_f32_to_bf16(_p(x), _p(y), x.numel(), int(apply_silu), _stream()))
    return y


def silu_bwd_f32(x, dy):
    _chk_f32(x, dy)
    dx = torch.empty_like(x)
    native.check(native.lib().t2v_silu_bwd_f32(_p(x), _p(dy), _p(dx), x.numel(), 0, _stream()))
    return dx


def silu_bf16(x):
    _chk_bf16(x)
    y = torch.empty_like(x)
    native.check(native.lib().t2v_silu_bf16(_p(x), _p(y), x.numel(), _stream()))
    return y


def silu_bf16_bwd(x, dy):
    _chk_bf16(x, dy)
    dx = torch.empty_like(x)
    native.check(native.lib().t2v_silu_bf16_bwd(_p(x), _p(dy), _p(dx), x.numel(), _stream()))
    return dx


def add_bf16(a, b, c=None):
    _chk_bf16(a, b, c)
    out = torch.empty_like(a)
    native.check(native.lib().t2v_add_bf16(_p(a), _p(b), _p(c), _p(out), a.numel(), _stream()))
    return out


def scale_bf16(a, alpha):
    """alpha * a (bf16) - expressed as the add kernel's sibling via a 1x1 identity would be wasteful; uses add with itself
    is wrong for general alpha, so this has its own tiny kernel."""
    _chk_bf16(a)
    out = torch.empty_like(a)
    native.check(native.lib().t2v_scale_bf16(_p(a), _p(out), a.numel(), float(alpha), _stream()))
    return out


def dropout_scale_add(x, base, p, scale, seed, epoch=None):
    """base + scale * dropout_p(x); the mask is a pure function of (seed, *epoch, element index).  `epoch`: optional int64
    device counter read when the kernel runs (see counter_add) - it keeps the masks of a replayed CUDA graph fresh."""
    _chk_bf16(x, base)
    out = torch.empty_like(x)
    native.check(native.lib().t2v_dropout_scale_add(_p(x), _p(base), _p(out), x.numel(), float(p), float(scale), int(seed), _p(epoch), _stream()))
    return out


def counter_add(counter, value=1):
    """*counter += value on the device (int64 scalar tensor)."""
    assert counter.dtype == torch.int64 and counter.is_cuda
    native.check(native.lib().t2v_counter_add(_p(counter), int(value), _stream()))


def sqnorm_chunks(g, chunks, out, g_bf16=None):
    """out[0] (fp64) += sum of g^2 over the (offset, length) chunks of the flat fp32 buffer g (or of its bf16 twin g_bf16)."""
    _chk_f32(g)
    _chk_bf16(g_bf16)
    assert chunks.dtype == torch.int64 and out.dtype == torch.float64
    native.check(native.lib().t2v_sqnorm_chunks(_p(g), _p(g_bf16), _p(chunks), chunks.shape[0], _p(out), _stream()))


def adamw_prepare(hp_in, hp, state, sq, max_norm):
    """Device-side scalars of one optimizer step: step count, bias corrections, clip factor (see include/t2v_b200.h)."""
    _chk_f32(hp_in, hp)
    assert state.dtype == torch.int64 and sq.dtype == torch.float64 and hp.shape[0] == hp_in.shape[0]
    native.check(native.lib().t2v_adamw_prepare(_p(hp_in), _p(hp), hp_in.shape[0], _p(state), _p(sq), float(max_norm or 0.0), _stream()))


def adamw_chunks(p, g, m, v, shadow, n_shadow, chunks, hp_row, zero_grad=True, g_bf16=None):
    """Fused AdamW over the chunk table of one hyper-parameter set; hp_row: the set's 8 floats on the device.  g_bf16: read
    the gradient values from this bf16 twin of g (all-reduced gradients) - g itself is then only zeroed."""
    _chk_f32(p, g, m, v, hp_row)
    _chk_bf16(shadow, g_bf16)
    native.check(native.lib().t2v_adamw_chunks(_p(p), _p(g), _p(g_bf16), _p(m), _p(v), _p(shadow), int(n_shadow), _p(chunks), chunks.shape[0],
                                               _p(hp_row), int(bool(zero_grad)), _stream()))


def adamw8bit_chunks(p, g, shadow, n_shadow, chunks, hp_row, qmaps, m32, v32, code_m, code_v, absmax_m, absmax_v, zero_grad=True,
                     g_bf16=None):
    """Blockwise 8-bit AdamW over the (arena offset, length, state offset, bits) rows of one hyper-parameter set: fp32 m32 / v32
    for 32-bit rows, uint8 codes into qmaps (512 floats: signed map, unsigned map) times per-256-block absmax for 8-bit rows."""
    _chk_f32(p, g, hp_row, qmaps, m32, v32, absmax_m, absmax_v)
    _chk_bf16(shadow, g_bf16)
    assert chunks.dtype == torch.int64 and chunks.dim() == 2 and chunks.shape[1] == 4 and chunks.is_contiguous()
    assert code_m.dtype == code_v.dtype == torch.uint8 and code_m.is_cuda and code_v.is_cuda and qmaps.numel() == 512
    native.check(native.lib().t2v_adamw8bit_chunks(_p(p), _p(g), _p(g_bf16), _p(shadow), int(n_shadow), _p(chunks), chunks.shape[0],
                                                   _p(hp_row), _p(qmaps), _p(m32), _p(v32), _p(code_m), _p(code_v), _p(absmax_m),
                                                   _p(absmax_v), int(bool(zero_grad)), _stream()))


def _chk_ema(ema, step, chunks, cols):
    _chk_f32(ema)
    assert ema is not None and step.dtype == torch.int64 and step.is_cuda
    assert chunks.dtype == torch.int64 and chunks.dim() == 2 and chunks.shape[1] == cols and chunks.is_contiguous()


def adamw_ema_chunks(p, g, m, v, shadow, n_shadow, chunks, hp_row, ema, step, ema_decay, zero_grad=True, g_bf16=None):
    """adamw_chunks over (arena offset, length, EMA offset) rows, then the EMA of each updated element: with k = step[0]
    (device int64, read when the kernel runs), ema -= (1 - d_k) * (ema - p), d_1 = 0, d_k = min(ema_decay, k / (9 + k))."""
    _chk_f32(p, g, m, v, hp_row)
    _chk_bf16(shadow, g_bf16)
    _chk_ema(ema, step, chunks, 3)
    native.check(native.lib().t2v_adamw_ema_chunks(_p(p), _p(g), _p(g_bf16), _p(m), _p(v), _p(shadow), int(n_shadow), _p(chunks),
                                                   chunks.shape[0], _p(hp_row), int(bool(zero_grad)), _p(ema), _p(step), float(ema_decay),
                                                   _stream()))


def adamw8bit_ema_chunks(p, g, shadow, n_shadow, chunks, hp_row, qmaps, m32, v32, code_m, code_v, absmax_m, absmax_v, ema, step, ema_decay,
                         zero_grad=True, g_bf16=None):
    """adamw8bit_chunks over (arena offset, length, state offset, bits, EMA offset) rows plus the EMA of adamw_ema_chunks."""
    _chk_f32(p, g, hp_row, qmaps, m32, v32, absmax_m, absmax_v)
    _chk_bf16(shadow, g_bf16)
    _chk_ema(ema, step, chunks, 5)
    assert code_m.dtype == code_v.dtype == torch.uint8 and code_m.is_cuda and code_v.is_cuda and qmaps.numel() == 512
    native.check(native.lib().t2v_adamw8bit_ema_chunks(_p(p), _p(g), _p(g_bf16), _p(shadow), int(n_shadow), _p(chunks), chunks.shape[0],
                                                       _p(hp_row), _p(qmaps), _p(m32), _p(v32), _p(code_m), _p(code_v), _p(absmax_m),
                                                       _p(absmax_v), int(bool(zero_grad)), _p(ema), _p(step), float(ema_decay), _stream()))


def ema_swap_chunks(p, ema, shadow, n_shadow, rows):
    """Exchange p and ema over the (arena offset, length, EMA offset) rows and rewrite the bf16 shadow of the rows below
    n_shadow from the new p; a second call restores all three bit for bit."""
    _chk_f32(p, ema)
    _chk_bf16(shadow)
    assert rows.dtype == torch.int64 and rows.dim() == 2 and rows.shape[1] == 3 and rows.is_contiguous()
    native.check(native.lib().t2v_ema_swap_chunks(_p(p), _p(ema), _p(shadow), int(n_shadow), _p(rows), rows.shape[0], _stream()))


def _delta_geom(w, A, B, conv3d):
    """(Cout, Cin, k, r) of a stable-LoRA conv: w [Cout, KH, KW, Cin], A [r*k, Cin*k], B [Cout*k, r*k]."""
    Co, KH, KW, Ci = w.shape
    k = KH
    assert (KH, KW) == ((3, 1) if conv3d else (k, k)), (w.shape, conv3d)
    assert A.dim() == 2 and B.dim() == 2 and A.shape[1] == Ci * k and B.shape == (Co * k, A.shape[0]) and A.shape[0] % k == 0, \
        (w.shape, A.shape, B.shape)
    return Co, Ci, k, A.shape[0] // k


def lora_delta_merge(base, A, B, scaling, conv3d):
    """bf16 [Cout, KH, KW, Cin] = base + scaling * view(B @ A) for a stable-LoRA conv (include/t2v_b200.h); base is the fp32
    weight in the same physical layout, A and B the fp32 LoRA factors."""
    _chk_f32(base, A, B)
    Co, Ci, k, r = _delta_geom(base, A, B, conv3d)
    out = torch.empty(base.shape, device=base.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_lora_delta_merge(_p(base), _p(A), _p(B), float(scaling), k, int(bool(conv3d)), Co, Ci, r, _p(out),
                                                   _stream()))
    return out


def lora_delta_grad(dw, A, B, scaling, conv3d, dA, dB):
    """dA += B^T dBA, dB += dBA A^T with dBA = scaling * view^T(dw): the gradient of a merged stable-LoRA conv weight (fp32
    [Cout, KH, KW, Cin]) projected onto its factors."""
    _chk_f32(dw, A, B, dA, dB)
    assert dA.shape == A.shape and dB.shape == B.shape
    Co, Ci, k, r = _delta_geom(dw, A, B, conv3d)
    native.check(native.lib().t2v_lora_delta_grad(_p(dw), _p(A), _p(B), float(scaling), k, int(bool(conv3d)), Co, Ci, r, _p(dA), _p(dB),
                                                  _stream()))


def scale_cast_f32_bf16(src, dst, alpha):
    """dst (bf16) = alpha * src (fp32): gradient compression before the data-parallel all-reduce."""
    _chk_f32(src)
    _chk_bf16(dst)
    assert src.numel() == dst.numel()
    native.check(native.lib().t2v_scale_cast_f32_bf16(_p(src), _p(dst), src.numel(), float(alpha), _stream()))


def cast_bf16_f32(src, dst):
    _chk_bf16(src)
    _chk_f32(dst)
    assert src.numel() == dst.numel()
    native.check(native.lib().t2v_cast_bf16_f32(_p(src), _p(dst), src.numel(), _stream()))


def add_f32(a, b):
    _chk_f32(a, b)
    out = torch.empty_like(a)
    native.check(native.lib().t2v_add_f32(_p(a), _p(b), _p(out), a.numel(), _stream()))
    return out


def cast_f32_bf16(src, dst=None):
    assert src.dtype == torch.float32 and src.is_cuda
    if dst is None:
        dst = torch.empty(src.shape, device=src.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_cast_f32_bf16(_p(src), _p(dst), src.numel(), _stream()))
    return dst


def upsample_nearest_fwd(x, out_hw_):
    _chk_bf16(x)
    N, H, W, C = x.shape
    Ho, Wo = out_hw_
    y = torch.empty((N, Ho, Wo, C), device=x.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_upsample_nearest_fwd(_p(x), _p(y), N, H, W, Ho, Wo, C, _stream()))
    return y


def upsample_nearest_bwd(dy, in_hw):
    _chk_bf16(dy)
    N, Ho, Wo, C = dy.shape
    H, W = in_hw
    dx = torch.empty((N, H, W, C), device=dy.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_upsample_nearest_bwd(_p(dy), _p(dx), N, H, W, Ho, Wo, C, _stream()))
    return dx


def copy_cols(src, dst, M, C, src_ld, src_off, dst_ld, dst_off):
    native.check(native.lib().t2v_copy_cols(_p(src), _p(dst), M, C, src_ld, src_off, dst_ld, dst_off, _stream()))


def concat_channels(a, b):
    """[..., Ca] ++ [..., Cb] along the (contiguous) channel axis."""
    _chk_bf16(a, b)
    Ca, Cb = a.shape[-1], b.shape[-1]
    M = a.numel() // Ca
    out = torch.empty(a.shape[:-1] + (Ca + Cb,), device=a.device, dtype=torch.bfloat16)
    copy_cols(a, out, M, Ca, Ca, 0, Ca + Cb, 0)
    copy_cols(b, out, M, Cb, Cb, 0, Ca + Cb, Ca)
    return out


def split_channels(g, Ca):
    _chk_bf16(g)
    Ct = g.shape[-1]
    M = g.numel() // Ct
    a = torch.empty(g.shape[:-1] + (Ca,), device=g.device, dtype=torch.bfloat16)
    b = torch.empty(g.shape[:-1] + (Ct - Ca,), device=g.device, dtype=torch.bfloat16)
    copy_cols(g, a, M, Ca, Ct, 0, Ca, 0)
    copy_cols(g, b, M, Ct - Ca, Ct, Ca, Ct - Ca, 0)
    return a, b


def colsum(x, out, S, P, C):
    """out [S,C] fp32 += sum over P of x [S,P,C] bf16."""
    _chk_bf16(x)
    _chk_f32(out)
    native.check(native.lib().t2v_colsum(_p(x), _p(out), S, P, C, _stream()))


def colsum_f32(x, out):
    _chk_f32(x, out)
    native.check(native.lib().t2v_colsum_f32(_p(x), _p(out), x.shape[0], x.shape[1], _stream()))


def softmax_fwd(s, n_valid, ld_out, causal_period=0):
    """Row softmax of fp32 scores [..., ld_in] -> bf16 probabilities [..., ld_out]; causal_period > 0: row r of the
    flattened row index sees only columns <= r % causal_period (the CLIP text encoder's causal mask)."""
    _chk_f32(s)
    rows = s.numel() // s.shape[-1]
    p = torch.empty(s.shape[:-1] + (ld_out,), device=s.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_softmax_fwd(_p(s), _p(p), rows, n_valid, s.shape[-1], ld_out, int(causal_period), _stream()))
    return p


def gelu_bf16(x, quick=False):
    _chk_bf16(x)
    y = torch.empty_like(x)
    native.check(native.lib().t2v_gelu_bf16(_p(x), _p(y), x.numel(), int(bool(quick)), _stream()))
    return y


def gelu_bwd(x, dy, quick=False):
    """dx = dy * gelu'(x) (bf16), the backward of gelu_bf16."""
    _chk_bf16(x, dy)
    assert x.shape == dy.shape
    dx = torch.empty_like(x)
    native.check(native.lib().t2v_gelu_bwd_bf16(_p(x), _p(dy), _p(dx), x.numel(), int(bool(quick)), _stream()))
    return dx


def frames_u8_to_nhwc8(frames, out_hw):
    """uint8 RGB frames [F, H0, W0, 3] -> bilinear resize + (x / 127.5 - 1) -> bf16 [F, h, w, 8] (VAE input layout)."""
    assert frames.dtype == torch.uint8 and frames.is_cuda and frames.is_contiguous() and frames.shape[-1] == 3, (frames.dtype, frames.shape)
    F, H0, W0, _ = frames.shape
    h, w = out_hw
    out = torch.empty((F, h, w, 8), device=frames.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_frames_u8_to_nhwc8(_p(frames), _p(out), F, H0, W0, h, w, _stream()))
    return out


def frames_u8_to_nhwc8_ragged(packed, table, out_hw):
    """A ragged batch of clips in one launch: packed uint8 [nbytes] holds clip k's RGB frames [F_k, H0_k, W0_k, 3] at byte
    table[k, 0]; table int64 [n, 4] = (offset, F, H0, W0) per clip -> bf16 [sum F_k, h, w, 8], clip after clip, each slice
    bitwise equal to frames_u8_to_nhwc8 of that clip.  The table is checked against the buffer on the host (a device table
    is read back once), then copied to the device."""
    assert packed.dtype == torch.uint8 and packed.is_cuda and packed.is_contiguous() and packed.dim() == 1, (packed.dtype, packed.shape)
    assert table.dtype == torch.int64 and table.dim() == 2 and table.shape[1] == 4, (table.dtype, table.shape)
    rows = table.cpu()
    off, F, H0, W0 = rows.unbind(1)
    assert bool((F > 0).all() and (H0 > 0).all() and (W0 > 0).all() and (off >= 0).all()), rows
    assert int((off + F * H0 * W0 * 3).max()) <= packed.numel(), (rows, packed.numel())
    h, w = out_hw
    total = int(F.sum())
    out = torch.empty((total, h, w, 8), device=packed.device, dtype=torch.bfloat16)
    dev_table = table.to(packed.device, non_blocking=True).contiguous()
    native.check(native.lib().t2v_frames_u8_to_nhwc8_ragged(_p(packed), _p(dev_table), rows.shape[0], total, _p(out), h, w, _stream()))
    return out


def embed_tokens(ids, tok_emb, pos_emb):
    """ids int64 [B, L], tok_emb fp32 [vocab, C], pos_emb fp32 [>= L, C] -> bf16 [B*L, C] = tok_emb[ids] + pos_emb[l]."""
    assert ids.dtype == torch.int64 and ids.is_cuda and ids.is_contiguous()
    _chk_f32(tok_emb, pos_emb)
    B, L = ids.shape
    C = tok_emb.shape[1]
    out = torch.empty((B * L, C), device=ids.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_embed_tokens(_p(ids), _p(tok_emb), _p(pos_emb), _p(out), B * L, L, C, tok_emb.shape[0], _stream()))
    return out


def embed_tokens_bwd(ids, dy, dtok, dpos, vocab):
    """Backward of embed_tokens, accumulated: dtok fp32 [vocab, C][id] += sum of the rows of dy bf16 [B*L, C] with that (clamped)
    id, dpos fp32 [>= L, C][l] += sum over b of row (b, l).  Either gradient may be None (frozen table).  Deterministic."""
    assert ids.dtype == torch.int64 and ids.is_cuda and ids.is_contiguous()
    _chk_bf16(dy)
    _chk_f32(dtok, dpos)
    B, L = ids.shape
    C = dy.shape[1]
    assert dy.shape[0] == B * L, (dy.shape, ids.shape)
    assert dtok is None or dtok.shape == (vocab, C), (dtok.shape, vocab, C)
    assert dpos is None or (dpos.shape[0] >= L and dpos.shape[1] == C), (dpos.shape, L, C)
    native.check(native.lib().t2v_embed_tokens_bwd(_p(ids), _p(dy), _p(dtok), _p(dpos), B * L, L, C, int(vocab), _stream()))


def softmax_bwd(p, dp, n_valid, scale):
    _chk_bf16(p)
    _chk_f32(dp)
    rows = p.numel() // p.shape[-1]
    ds = torch.empty_like(p)
    native.check(native.lib().t2v_softmax_bwd(_p(p), _p(dp), _p(ds), rows, n_valid, p.shape[-1], dp.shape[-1], float(scale), _stream()))
    return ds


def _chk_rows_bf16(*ts):
    """bf16 CUDA matrices whose rows are contiguous (column slices of a wider matrix are fine)."""
    for t in ts:
        assert t.dtype == torch.bfloat16 and t.is_cuda and t.stride(-1) == 1, (t.dtype, t.shape, t.stride())


def attn_small_fwd(q, k, v, o, addr):
    """addr = (nseq, inner, outer_rows, inner_rows, seq_rows, ld_in, ld_out, heads, L, D); q/k/v may be column slices."""
    _chk_rows_bf16(q, k, v, o)
    native.check(native.lib().t2v_attn_small_fwd(_p(q), _p(k), _p(v), _p(o), *addr, _stream()))
    return o


def attn_small_bwd(q, k, v, do, dq, dk, dv, addr):
    _chk_rows_bf16(q, k, v, do, dq, dk, dv)
    native.check(native.lib().t2v_attn_small_bwd(_p(q), _p(k), _p(v), _p(do), _p(dq), _p(dk), _p(dv), *addr, _stream()))
    return dq, dk, dv


def attn_long_fwd(q, k, v, o, lse, addr):
    """attn_small_fwd for 1 <= L <= 256; also writes lse fp32 [nseq, heads, L] (natural-log row logsumexp of the scaled
    scores), which attn_long_bwd reads."""
    _chk_rows_bf16(q, k, v, o)
    _chk_f32(lse)
    native.check(native.lib().t2v_attn_long_fwd(_p(q), _p(k), _p(v), _p(o), _p(lse), *addr, _stream()))
    return o, lse


def attn_long_bwd(q, k, v, o, do, lse, dq, dk, dv, addr):
    """o / lse: the forward's outputs (delta = rowsum(dO o O) is formed from o)."""
    _chk_rows_bf16(q, k, v, o, do, dq, dk, dv)
    _chk_f32(lse)
    native.check(native.lib().t2v_attn_long_bwd(_p(q), _p(k), _p(v), _p(o), _p(do), _p(lse), _p(dq), _p(dk), _p(dv), *addr, _stream()))
    return dq, dk, dv


def timestep_embedding(t, dim):
    assert t.dtype == torch.int64 and t.is_cuda
    out = torch.empty((t.shape[0], dim), device=t.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_timestep_embedding(_p(t), _p(out), t.shape[0], dim, _stream()))
    return out


def latents_to_nhwc8(x0, noise=None, alphas_cumprod=None, timesteps=None):
    """(B,C,F,H,W) fp32 [-> add_noise] -> [B*F,H,W,8] bf16."""
    _chk_f32(x0, noise, alphas_cumprod)
    B, C, F, H, W = x0.shape
    out = torch.empty((B * F, H, W, 8), device=x0.device, dtype=torch.bfloat16)
    native.check(native.lib().t2v_latents_to_nhwc8(_p(x0), _p(noise), _p(alphas_cumprod), _p(timesteps), _p(out), B, C, F, H * W, _stream()))
    return out


def nhwc8_to_latents(x, B, C, F):
    _chk_bf16(x)
    _, H, W, _ = x.shape
    out = torch.empty((B, C, F, H, W), device=x.device, dtype=torch.float32)
    native.check(native.lib().t2v_nhwc8_to_latents(_p(x), _p(out), B, C, F, H * W, _stream()))
    return out


def vae_sample(moments, eps, B, F, scale):
    """moments [B*F,h,w,8] bf16, eps (B,4,F,h,w) fp32 -> latents (B,4,F,h,w) fp32."""
    _chk_bf16(moments)
    _chk_f32(eps)
    _, h, w, _ = moments.shape
    out = torch.empty((B, 4, F, h, w), device=moments.device, dtype=torch.float32)
    native.check(native.lib().t2v_vae_sample(_p(moments), _p(eps), _p(out), B, F, h * w, float(scale), _stream()))
    return out


def mse_loss_fwd(pred, target):
    _chk_bf16(pred)
    _chk_f32(target)
    B, C, F, H, W = target.shape
    loss = torch.empty((), device=pred.device, dtype=torch.float32)
    native.check(native.lib().t2v_mse_loss(_p(pred), _p(target), _p(loss), _p(None), _p(None), B, C, F, H * W, _stream()))
    return loss


def mse_loss_bwd(pred, target, gout):
    B, C, F, H, W = target.shape
    dpred = torch.empty_like(pred)
    native.check(native.lib().t2v_mse_loss(_p(pred), _p(target), _p(None), _p(gout), _p(dpred), B, C, F, H * W, _stream()))
    return dpred


def _chk_velocity(pred, x0, noise, alphas_cumprod, timesteps):
    _chk_bf16(pred)
    _chk_f32(x0, noise, alphas_cumprod)
    assert x0.shape == noise.shape and timesteps.dtype == torch.int64 and timesteps.is_cuda and timesteps.is_contiguous(), (
        x0.shape, noise.shape, timesteps.dtype)
    assert timesteps.shape == (x0.shape[0],), (timesteps.shape, x0.shape)


def velocity_mse_loss_fwd(pred, x0, noise, alphas_cumprod, timesteps):
    """mean((pred - v)^2), v = sqrt(abar[t]) noise - sqrt(1 - abar[t]) x0 formed in the kernel; pred [B*F,H,W,8] bf16."""
    _chk_velocity(pred, x0, noise, alphas_cumprod, timesteps)
    B, C, F, H, W = x0.shape
    loss = torch.empty((), device=pred.device, dtype=torch.float32)
    native.check(native.lib().t2v_velocity_mse_loss(_p(pred), _p(x0), _p(noise), _p(alphas_cumprod), _p(timesteps), _p(loss), _p(None),
                                                    _p(None), B, C, F, H * W, _stream()))
    return loss


def velocity_mse_loss_bwd(pred, x0, noise, alphas_cumprod, timesteps, gout):
    _chk_velocity(pred, x0, noise, alphas_cumprod, timesteps)
    B, C, F, H, W = x0.shape
    dpred = torch.empty_like(pred)
    native.check(native.lib().t2v_velocity_mse_loss(_p(pred), _p(x0), _p(noise), _p(alphas_cumprod), _p(timesteps), _p(None), _p(gout),
                                                    _p(dpred), B, C, F, H * W, _stream()))
    return dpred


_LOSS_FORMS = {"l2": 0, "huber": 1, "smooth_l1": 2}             # T2V_LOSS_*
_HUBER_SCHEDULES = {"constant": 0, "exponential": 1, "snr": 2}   # T2V_HUBER_*


def _loss_params(objective, x0, alphas_cumprod):
    """native.LossParams of a step.LossObjective; x0 given selects the velocity target (T2V_PRED_V)."""
    return native.LossParams(int(x0 is not None), _LOSS_FORMS[objective.loss_type], _HUBER_SCHEDULES[objective.huber_schedule],
                             alphas_cumprod.numel(), float(objective.huber_c) if objective.loss_type != "l2" else 0.0,
                             float(objective.snr_gamma or 0.0))


def _chk_diffusion(pred, x0, noise, alphas_cumprod, timesteps):
    _chk_bf16(pred)
    _chk_f32(noise, alphas_cumprod)
    if x0 is not None:
        _chk_f32(x0)
        assert x0.shape == noise.shape, (x0.shape, noise.shape)
    assert timesteps.dtype == torch.int64 and timesteps.is_cuda and timesteps.is_contiguous(), timesteps.dtype
    assert timesteps.shape == (noise.shape[0],), (timesteps.shape, noise.shape)


def diffusion_loss_fwd(pred, x0, noise, alphas_cumprod, timesteps, objective):
    """sum_e w_b psi(pred - y) / numel (t2v_diffusion_loss): `objective` a step.LossObjective (snr_gamma, loss_type,
    huber_schedule, huber_c); y the noise, or the velocity when x0 is given.  pred [B*F,H,W,8] bf16, the rest fp32."""
    _chk_diffusion(pred, x0, noise, alphas_cumprod, timesteps)
    B, C, F, H, W = noise.shape
    loss = torch.empty((), device=pred.device, dtype=torch.float32)
    params = _loss_params(objective, x0, alphas_cumprod)
    native.check(native.lib().t2v_diffusion_loss(_p(pred), _p(noise), _p(x0), _p(alphas_cumprod), _p(timesteps), ctypes.byref(params),
                                                 _p(loss), _p(None), _p(None), B, C, F, H * W, _stream()))
    return loss


def diffusion_loss_bwd(pred, x0, noise, alphas_cumprod, timesteps, objective, gout):
    """dpred = gout w_b psi'(pred - y) / numel, channels-last bf16 like pred."""
    _chk_diffusion(pred, x0, noise, alphas_cumprod, timesteps)
    B, C, F, H, W = noise.shape
    dpred = torch.empty_like(pred)
    params = _loss_params(objective, x0, alphas_cumprod)
    native.check(native.lib().t2v_diffusion_loss(_p(pred), _p(noise), _p(x0), _p(alphas_cumprod), _p(timesteps), ctypes.byref(params),
                                                 _p(None), _p(gout), _p(dpred), B, C, F, H * W, _stream()))
    return dpred
