"""GPU parity of the wgmma affine-TMA GEMM family (conv fwd / dgrad / wgrad, batched GEMM) through the C ABI.
Reference = plain PyTorch fp32 ops on the same bf16-rounded inputs (floating-point kernel => torch fp32 reference)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _lib():
    from t2v_b200 import native
    return native


def P(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def rel_err(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-6)).item()


def conv_ref(x, w, stride, pads):
    # x [N,H,W,C] bf16, w [Co,KH,KW,Ci] bf16 -> fp32 NHWC
    ph0, ph1, pw0, pw1 = pads
    xf = F.pad(x.float().permute(0, 3, 1, 2), (pw0, pw1, ph0, ph1))
    return F.conv2d(xf, w.float().permute(0, 3, 1, 2), stride=stride).permute(0, 2, 3, 1).contiguous()


CONV_CASES = [
    # N, H, W, Cin, Cout, KH, KW, stride, pads(h0,h1,w0,w1)
    (1, 1, 300, 320, 320, 1, 1, 1, (0, 0, 0, 0)),       # linear, ragged M
    (1, 1, 1024, 64, 2560, 1, 1, 1, (0, 0, 0, 0)),      # linear, wide N
    (4, 16, 16, 64, 96, 3, 3, 1, (1, 1, 1, 1)),
    (16, 32, 32, 320, 320, 3, 3, 1, (1, 1, 1, 1)),      # level-0 resnet conv at cfg 2
    (16, 4, 4, 128, 256, 3, 3, 1, (1, 1, 1, 1)),        # deep level: several frames per tile
    (2, 24, 40, 64, 64, 3, 3, 1, (1, 1, 1, 1)),         # non power-of-two spatial (cfg 3 style)
    (4, 16, 16, 8, 320, 3, 3, 1, (1, 1, 1, 1)),         # conv_in (4->8 padded channels)
    (4, 16, 16, 320, 8, 3, 3, 1, (1, 1, 1, 1)),         # conv_out
    (4, 16, 16, 64, 64, 3, 3, 2, (1, 1, 1, 1)),         # Downsample2D (UNet)
    (2, 16, 16, 128, 128, 3, 3, 2, (0, 1, 0, 1)),       # Downsample2D (VAE, asymmetric pad)
    (2, 6, 64, 64, 64, 3, 1, 1, (1, 1, 0, 0)),          # temporal conv: W=H*W, H=F, N=B
    (1, 3, 40, 192, 160, 1, 1, 1, (0, 0, 0, 0)),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fwd(case):
    nat = _lib()
    N, H, W, Ci, Co, KH, KW, s, pads = case
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(N, H, W, Ci, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Co, KH, KW, Ci, device="cuda", generator=g) / (KH * KW * Ci) ** 0.5).bfloat16()
    bias = torch.randn(Co, device="cuda", generator=g)
    ref = conv_ref(x, w, s, pads)
    Ho, Wo = ref.shape[1], ref.shape[2]
    rowbias = torch.randn(N, Co, device="cuda", generator=g)
    res = torch.randn(N, Ho, Wo, Co, device="cuda", generator=g).bfloat16()
    # plain
    y = torch.full((N, Ho, Wo, Co), float("nan"), device="cuda", dtype=torch.bfloat16)
    epi = nat.Epilogue(None, None, None, 1.0, 0, 1)
    nat.check(nat.lib().t2v_conv_fwd(P(x), P(w), P(y), N, H, W, Ci, Co, KH, KW, s, *pads, ctypes.byref(epi), stream()))
    torch.cuda.synchronize()
    e = rel_err(y, ref)
    assert e < 1e-2, f"plain conv rel err {e}"
    # fused epilogue, fp32 and bf16 output
    ref2 = 0.5 * ref + bias + rowbias[:, None, None, :] + res.float()
    for out_fp32, tol in ((1, 2e-3), (0, 1e-2)):
        y2 = torch.full((N, Ho, Wo, Co), float("nan"), device="cuda", dtype=torch.float32 if out_fp32 else torch.bfloat16)
        epi = nat.Epilogue(bias.data_ptr(), rowbias.data_ptr(), res.data_ptr(), 0.5, out_fp32, 1)
        nat.check(nat.lib().t2v_conv_fwd(P(x), P(w), P(y2), N, H, W, Ci, Co, KH, KW, s, *pads, ctypes.byref(epi), stream()))
        torch.cuda.synchronize()
        e = rel_err(y2, ref2)
        assert e < tol, f"epilogue conv rel err {e} (fp32 output: {out_fp32})"


DGRAD_CASES = [c for c in CONV_CASES if c[3] % 8 == 0 and c[4] % 8 == 0]


@pytest.mark.parametrize("case", DGRAD_CASES)
def test_conv_dgrad_wgrad(case):
    nat = _lib()
    N, H, W, Ci, Co, KH, KW, s, pads = case
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(N, H, W, Ci, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Co, KH, KW, Ci, device="cuda", generator=g) / (KH * KW * Ci) ** 0.5).bfloat16()
    xf = x.float().requires_grad_(True)
    wf = w.float().requires_grad_(True)
    ph0, ph1, pw0, pw1 = pads
    yf = F.conv2d(F.pad(xf.permute(0, 3, 1, 2), (pw0, pw1, ph0, ph1)), wf.permute(0, 3, 1, 2), stride=s).permute(0, 2, 3, 1)
    dy = torch.randn(yf.shape, device="cuda", generator=g).bfloat16()
    yf.backward(dy.float())
    # dgrad (+ residual add)
    other = torch.randn(N, H, W, Ci, device="cuda", generator=g).bfloat16()
    dx = torch.full((N, H, W, Ci), float("nan"), device="cuda", dtype=torch.bfloat16)
    epi = nat.Epilogue(None, None, other.data_ptr(), 1.0, 0, 1)
    nat.check(nat.lib().t2v_conv_dgrad(P(dy), P(w), P(dx), N, H, W, Ci, Co, KH, KW, s, *pads, ctypes.byref(epi), stream()))
    torch.cuda.synchronize()
    e = rel_err(dx, xf.grad + other.float())
    assert e < 1e-2, f"dgrad rel err {e}"
    # wgrad accumulates into fp32
    dw = torch.ones(Co, KH, KW, Ci, device="cuda", dtype=torch.float32)
    nat.check(nat.lib().t2v_conv_wgrad(P(x), P(dy), P(dw), N, H, W, Ci, Co, KH, KW, s, *pads, stream()))
    torch.cuda.synchronize()
    e = rel_err(dw, wf.grad + 1.0)
    assert e < 2e-3, f"wgrad rel err {e}"


WGRAD_BIAS_CASES = [
    # (conv case, forced wgmma N, column-sum pass instead of the fused row sums): row-sum MMAs next to every tile width class
    ((16, 32, 32, 320, 320, 3, 3, 1, (1, 1, 1, 1)), 0, 0),     # planner's own choice (split-K, Cout ragged against 128-row tiles)
    ((1, 1, 4096, 640, 640, 1, 1, 1, (0, 0, 0, 0)), 16, 0),    # narrowest tile
    ((1, 1, 4096, 640, 640, 1, 1, 1, (0, 0, 0, 0)), 48, 0),    # N not a multiple of 32: padded accumulator rows, ragged last chunk
    ((1, 1, 4096, 640, 640, 1, 1, 1, (0, 0, 0, 0)), 112, 0),
    ((1, 1, 2048, 1280, 320, 1, 1, 1, (0, 0, 0, 0)), 80, 0),
    ((1, 1, 2048, 1280, 320, 1, 1, 1, (0, 0, 0, 0)), 128, 1),  # widest tile, bias gradient through the column-sum kernel
    ((4, 16, 16, 64, 64, 3, 3, 2, (1, 1, 1, 1)), 0, 0),        # stride 2
    ((2, 6, 64, 64, 72, 3, 1, 1, (1, 1, 0, 0)), 0, 0),         # temporal conv, Cout = 72 (one ragged row tile)
    ((1, 3, 40, 192, 160, 1, 1, 1, (0, 0, 0, 0)), 0, 0),
]


@pytest.mark.parametrize("case,bn,colsum", WGRAD_BIAS_CASES)
def test_conv_wgrad_bias(case, bn, colsum, monkeypatch):
    """t2v_conv_wgrad_bias: the weight gradient is unchanged and dbias += column sums of dy (both accumulate)."""
    nat = _lib()
    N, H, W, Ci, Co, KH, KW, s, pads = case
    if bn:
        monkeypatch.setenv("T2V_FORCE_BN", str(bn))
    if colsum:
        monkeypatch.setenv("T2V_NO_ROWSUM_FUSE", "1")
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(N, H, W, Ci, device="cuda", generator=g).bfloat16()
    Ho = (H + pads[0] + pads[1] - KH) // s + 1
    Wo = (W + pads[2] + pads[3] - KW) // s + 1
    dy = (torch.randn(N, Ho, Wo, Co, device="cuda", generator=g) + 0.25).bfloat16()
    dw_ref = torch.ones(Co, KH, KW, Ci, device="cuda", dtype=torch.float32)
    nat.check(nat.lib().t2v_conv_wgrad(P(x), P(dy), P(dw_ref), N, H, W, Ci, Co, KH, KW, s, *pads, stream()))
    dw = torch.ones(Co, KH, KW, Ci, device="cuda", dtype=torch.float32)
    db = torch.full((Co,), 3.0, device="cuda", dtype=torch.float32)
    nat.check(nat.lib().t2v_conv_wgrad_bias(P(x), P(dy), P(dw), P(db), N, H, W, Ci, Co, KH, KW, s, *pads, stream()))
    torch.cuda.synchronize()
    want = 3.0 + dy.float().reshape(-1, Co).sum(0)
    e = rel_err(db, want)
    assert e < 1e-4, f"dbias rel err {e}"      # exact bf16 x 1.0 products, fp32 accumulation: only the summation order differs
    e = rel_err(dw, dw_ref)
    assert e < 1e-5, f"wgrad changed by the fused row sums: {e}"   # red.add order of split-K partials only


SPLITK_CASES = [
    (16, 4, 4, 640, 640, 3, 3, 1, (1, 1, 1, 1)),        # deepest resnet conv: 2 x 4 output tiles, 90 k-blocks
    (1, 16, 16, 1280, 1280, 3, 1, 1, (1, 1, 0, 0)),     # temporal conv at 4x4: W=H*W, H=F
    (4, 8, 8, 512, 256, 3, 3, 1, (1, 1, 1, 1)),
    (1, 1, 256, 5120, 1280, 1, 1, 1, (0, 0, 0, 0)),     # FeedForward out-projection on a small map
]


@pytest.mark.parametrize("case", SPLITK_CASES)
def test_conv_splitk_scratch(case):
    """Few-tile problems split their reduction over the SMs when the caller passes the scratch the planner asks for."""
    nat = _lib()
    N, H, W, Ci, Co, KH, KW, s, pads = case
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(N, H, W, Ci, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Co, KH, KW, Ci, device="cuda", generator=g) / (KH * KW * Ci) ** 0.5).bfloat16()
    bias = torch.randn(Co, device="cuda", generator=g)
    rowbias = torch.randn((N + 1) // 2, Co, device="cuda", generator=g)
    ref = conv_ref(x, w, s, pads)
    Ho, Wo = ref.shape[1], ref.shape[2]
    res = torch.randn(N, Ho, Wo, Co, device="cuda", generator=g).bfloat16()
    nbytes = nat.lib().t2v_conv_workspace_bytes(0, N, H, W, Ci, Co, KH, KW, s, *pads)
    assert nbytes == N * Ho * Wo * Co * 4, "planner should ask for split-K scratch on this shape"
    ws = torch.full((nbytes // 4,), float("nan"), device="cuda")
    rb_div = 2 if N > 1 else 1
    ref2 = 0.5 * ref + bias + rowbias[torch.arange(N, device="cuda") // rb_div][:, None, None, :] + res.float()
    for out_fp32, tol in ((0, 1e-2), (1, 2e-3)):
        y = torch.full((N, Ho, Wo, Co), float("nan"), device="cuda", dtype=torch.float32 if out_fp32 else torch.bfloat16)
        epi = nat.Epilogue(bias.data_ptr(), rowbias.data_ptr(), res.data_ptr(), 0.5, out_fp32, rb_div, ws.data_ptr(), nbytes)
        nat.check(nat.lib().t2v_conv_fwd(P(x), P(w), P(y), N, H, W, Ci, Co, KH, KW, s, *pads, ctypes.byref(epi), stream()))
        torch.cuda.synchronize()
        e = rel_err(y, ref2)
        assert e < tol, f"split-K conv fwd rel err {e}"
    # dgrad with residual
    dy = torch.randn(N, Ho, Wo, Co, device="cuda", generator=g).bfloat16()
    xf = x.float().requires_grad_(True)
    ph0, ph1, pw0, pw1 = pads
    F.conv2d(F.pad(xf.permute(0, 3, 1, 2), (pw0, pw1, ph0, ph1)), w.float().permute(0, 3, 1, 2), stride=s).permute(0, 2, 3, 1).backward(dy.float())
    other = torch.randn(N, H, W, Ci, device="cuda", generator=g).bfloat16()
    nb = nat.lib().t2v_conv_workspace_bytes(1, N, H, W, Ci, Co, KH, KW, s, *pads)
    assert nb in (0, N * H * W * Ci * 4)   # the data gradient of a wide projection has enough tiles without splitting
    ws = torch.full((max(nb, 4) // 4,), float("nan"), device="cuda")
    dx = torch.full((N, H, W, Ci), float("nan"), device="cuda", dtype=torch.bfloat16)
    epi = nat.Epilogue(None, None, other.data_ptr(), 1.0, 0, 1, ws.data_ptr() if nb else None, nb)
    nat.check(nat.lib().t2v_conv_dgrad(P(dy), P(w), P(dx), N, H, W, Ci, Co, KH, KW, s, *pads, ctypes.byref(epi), stream()))
    torch.cuda.synchronize()
    e = rel_err(dx, xf.grad + other.float())
    assert e < 1e-2, f"split-K dgrad rel err {e}"


BGEMM_CASES = [
    # M, N, K, Z1, Z2, a_kmajor, b_kmajor, out_mode, ldc
    (1024, 1024, 64, 2, 5, 1, 1, 1, 1024),   # S = Q K^T per (frame, head), fp32
    (1024, 64, 1024, 2, 5, 1, 0, 0, 64),     # O = P V
    (1024, 80, 64, 2, 5, 1, 1, 1, 80),       # cross-attention scores (Lk 77 -> 80)
    (200, 64, 136, 1, 3, 1, 0, 0, 64),       # ragged
    (320, 320, 2000, 1, 1, 0, 0, 2, 320),    # linear wgrad dW = dY^T X (split-K, accumulate)
    (1024, 64, 1024, 2, 5, 0, 0, 1, 64),     # dV = P^T dO
    (256, 512, 512, 3, 1, 1, 1, 0, 512),     # VAE-style d=512
    (1024, 77, 64, 2, 5, 1, 1, 1, 77),       # unpadded Lk 77: rows not 16-byte aligned, the epilogue's scalar path
]


@pytest.mark.parametrize("case", BGEMM_CASES)
def test_bgemm(case):
    nat = _lib()
    M, N, K, Z1, Z2, ak, bk, mode, ldc = case
    g = torch.Generator(device="cuda").manual_seed(3)
    A = torch.randn((Z1, Z2, M, K) if ak else (Z1, Z2, K, M), device="cuda", generator=g).bfloat16()
    B = torch.randn((Z1, Z2, N, K) if bk else (Z1, Z2, K, N), device="cuda", generator=g).bfloat16()
    Af = A.float() if ak else A.float().transpose(-1, -2)
    Bf = B.float() if bk else B.float().transpose(-1, -2)
    ref = 0.125 * Af @ Bf.transpose(-1, -2)
    dt = torch.bfloat16 if mode == 0 else torch.float32
    C = torch.zeros(Z1, Z2, M, ldc, device="cuda", dtype=dt)
    if mode == 2:
        C += 1.0
    mA = nat.Mat(A.data_ptr(), A.shape[-1], A.stride(0), A.stride(1), ak)
    mB = nat.Mat(B.data_ptr(), B.shape[-1], B.stride(0), B.stride(1), bk)
    nat.check(nat.lib().t2v_bgemm(ctypes.byref(mA), ctypes.byref(mB), P(C), ldc, C.stride(0), C.stride(1),
                                  M, N, K, Z1, Z2, 0.125, mode, stream()))
    torch.cuda.synchronize()
    out = C[..., :N].float() - (1.0 if mode == 2 else 0.0)
    e = rel_err(out, ref)
    assert e < (1e-2 if mode == 0 else 2e-3), f"bgemm rel err {e}"
