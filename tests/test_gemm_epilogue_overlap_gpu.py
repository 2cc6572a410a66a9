"""The GEMM's epilogue warpgroup takes each finished accumulator tile from the MMA warpgroups through shared memory (acc_full /
acc_empty mbarriers), so the next tile's main loop overlaps the previous tile's epilogue.  These cases stress that hand-off:
many tiles per CTA (the barrier phases wrap many times), epilogues longer than the main loop, one tile per CTA, every wgmma
N with ragged column chunks, mixed row-sum / plain tiles in one launch, statistics with ragged row tiles, split-K, and
bitwise determinism.  Reference: oracle/ops_ref.py on the same bf16 inputs, at the tolerances of tests/test_gemm_gpu.py."""
import pytest
import torch

from oracle import ops_ref as ref

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _prims():
    from t2v_b200 import prims
    return prims


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, device=DEV, generator=g) * scale).bfloat16()


def rel_err(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-6)).item()


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fwd_both(x, w, bias, res, stride, pads, out_fp32=False, stats_rows=0, rb=None, rb_div=1, alpha=1.0):
    """(native, oracle) forward outputs and, with stats_rows, their per-(frame, channel) statistics."""
    prims = _prims()
    N, H, W, _ = x.shape
    Co, KH, KW, _ = w.shape
    Ho, Wo = ref.out_hw(H, W, KH, KW, stride, pads)
    st = st_r = None
    if stats_rows:
        st = prims.stats_alloc(N * Ho * Wo // stats_rows, Co, x.device)
        st_r = ref.stats_alloc(N * Ho * Wo // stats_rows, Co, x.device)
    y = prims.conv_fwd(x, w, bias, rb, res, stride, pads, alpha, out_fp32, rb_div, stats=st, stats_rows=stats_rows if st is not None else 0)
    y_r = ref.conv_fwd(x, w, bias, rb, res, stride, pads, alpha, out_fp32, rb_div, stats=st_r, stats_rows=stats_rows if st_r is not None else 0)
    return y, y_r, st, st_r


def _check_fwd(y, y_r, st, st_r, out_fp32, what):
    e = rel_err(y, y_r)
    assert e < (2e-3 if out_fp32 else 1e-2), f"{what}: rel err {e}"
    if st is not None:
        # the epilogue sums the fp32 values before bf16 rounding, like the oracle
        for i, name in ((0, "sum"), (1, "sum of squares")):
            e = rel_err(st[..., i], st_r[..., i])
            assert e < 5e-3, f"{what}: statistics ({name}) rel err {e}"


def test_many_tiles_per_cta_fwd_dgrad():
    """16 x 64 x 64 x 320 -> 320 3x3 conv: >= 8 tiles per CTA, so acc_full / acc_empty change phase many times."""
    prims = _prims()
    N, H, W, C = 16, 64, 64, 320
    g = torch.Generator(device=DEV).manual_seed(21)
    x = _rnd(g, N, H, W, C)
    w = _rnd(g, C, 3, 3, C, scale=(9 * C) ** -0.5)
    bias = torch.randn(C, device=DEV, generator=g)
    res = _rnd(g, N, H, W, C)
    assert N * H * W // 128 * 3 >= 8 * _sm_count()
    y, y_r, st, st_r = _fwd_both(x, w, bias, res, 1, (1, 1, 1, 1), stats_rows=H * W)
    _check_fwd(y, y_r, st, st_r, False, "conv fwd")
    dy = _rnd(g, N, H, W, C)
    other = _rnd(g, N, H, W, C)
    dx = prims.conv_dgrad(dy, w, (H, W), 1, (1, 1, 1, 1), other)
    e = rel_err(dx, ref.conv_dgrad(dy, w, (H, W), 1, (1, 1, 1, 1), other))
    assert e < 1e-2, f"dgrad rel err {e}"


@pytest.mark.parametrize("out_fp32", [False, True])
def test_epilogue_longer_than_mainloop(out_fp32):
    """K = 64 (one k-block per tile) with bias, residual and statistics: the MMA warps wait on acc_empty on every tile."""
    rows, Ci, Co = 16384, 64, 320
    g = torch.Generator(device=DEV).manual_seed(22)
    x = _rnd(g, 1, 1, rows, Ci)
    w = _rnd(g, Co, 1, 1, Ci, scale=Ci ** -0.5)
    bias = torch.randn(Co, device=DEV, generator=g) * 0.5 + 1.0
    res = _rnd(g, 1, 1, rows, Co)
    y, y_r, st, st_r = _fwd_both(x, w, bias, res, 1, (0, 0, 0, 0), out_fp32=out_fp32, stats_rows=0 if out_fp32 else 1024)
    _check_fwd(y, y_r, st, st_r, out_fp32, f"K=64 linear (fp32 output: {out_fp32})")


@pytest.mark.parametrize("rows,Ci,Co", [(1024, 320, 320), (100, 64, 48)])
def test_one_tile_per_cta(rows, Ci, Co):
    """Fewer tiles than SMs (every CTA runs one tile), down to a single-tile launch."""
    g = torch.Generator(device=DEV).manual_seed(23)
    x = _rnd(g, 1, 1, rows, Ci)
    w = _rnd(g, Co, 1, 1, Ci, scale=Ci ** -0.5)
    bias = torch.randn(Co, device=DEV, generator=g)
    res = _rnd(g, 1, 1, rows, Co)
    y, y_r, _, _ = _fwd_both(x, w, bias, res, 1, (0, 0, 0, 0))
    _check_fwd(y, y_r, None, None, False, f"{rows} x {Ci} -> {Co}")


@pytest.mark.parametrize("bn", list(range(16, 129, 16)))
def test_every_block_n(bn, monkeypatch):
    """Every wgmma N, with Cout = 200 so the last column tile ends in a ragged chunk; bf16 and fp32 output, alpha and a
    per-frame row bias (the catch-all chunk body)."""
    monkeypatch.setenv("T2V_FORCE_BN", str(bn))
    g = torch.Generator(device=DEV).manual_seed(24)
    N, H, W, Ci, Co = 4, 16, 16, 96, 200
    x = _rnd(g, N, H, W, Ci)
    w = _rnd(g, Co, 3, 3, Ci, scale=(9 * Ci) ** -0.5)
    bias = torch.randn(Co, device=DEV, generator=g)
    res = _rnd(g, N, H, W, Co)
    rb = torch.randn(N, Co, device=DEV, generator=g)
    for out_fp32 in (False, True):
        y, y_r, _, _ = _fwd_both(x, w, bias, res, 1, (1, 1, 1, 1), out_fp32=out_fp32)
        _check_fwd(y, y_r, None, None, out_fp32, f"N={bn} (fp32 output: {out_fp32})")
        y, y_r, _, _ = _fwd_both(x, w, bias, res, 1, (1, 1, 1, 1), out_fp32=out_fp32, rb=rb, alpha=0.5)
        _check_fwd(y, y_r, None, None, out_fp32, f"N={bn}, alpha + row bias (fp32 output: {out_fp32})")


@pytest.mark.parametrize("case", [
    (16, 32, 32, 320, 320, 3, 3),    # split-K wgrad: only t[0] == t[2] == t[3] == 0 tiles carry row sums
    (1, 1, 4096, 640, 640, 1, 1),
    (2, 6, 64, 64, 72, 3, 1),        # ragged row tile
])
def test_wgrad_mixed_rowsum_tiles(case):
    """Weight gradient with the fused bias gradient: row-sum tiles and plain tiles in one launch; dW and dbias accumulate."""
    prims = _prims()
    N, H, W, Ci, Co, KH, KW = case
    pads = ((KH - 1) // 2, (KH - 1) // 2, (KW - 1) // 2, (KW - 1) // 2)
    g = torch.Generator(device=DEV).manual_seed(25)
    x = _rnd(g, N, H, W, Ci)
    dy = (torch.randn(N, H, W, Co, device=DEV, generator=g) + 0.25).bfloat16()
    dw = torch.ones(Co, KH, KW, Ci, device=DEV)
    db = torch.full((Co,), 3.0, device=DEV)
    dw_r, db_r = dw.clone(), db.clone()
    prims.conv_wgrad(x, dy, dw, 1, pads, db)
    ref.conv_wgrad(x, dy, dw_r, 1, pads, db_r)
    e = rel_err(dw, dw_r)
    assert e < 2e-3, f"dW rel err {e}"
    e = rel_err(db, db_r)
    assert e < 1e-4, f"dbias rel err {e}"


@pytest.mark.parametrize("N,H,W,seg", [
    (9, 4, 4, 16),     # 16-row frames, 144 rows: the last row tile is ragged
    (5, 4, 8, 32),     # 32-row frames, 160 rows
    (24, 4, 4, 16),
    (12, 4, 8, 32),
])
def test_statistics_segments(N, H, W, seg):
    """GroupNorm statistics over 16- and 32-row segments, including rows past the end in the last tile."""
    g = torch.Generator(device=DEV).manual_seed(26)
    Ci, Co = 128, 256
    x = _rnd(g, N, H, W, Ci)
    w = _rnd(g, Co, 3, 3, Ci, scale=(9 * Ci) ** -0.5)
    bias = torch.randn(Co, device=DEV, generator=g) * 0.5 + 1.0
    res = _rnd(g, N, H, W, Co)
    assert H * W == seg
    y, y_r, st, st_r = _fwd_both(x, w, bias, res, 1, (1, 1, 1, 1), stats_rows=seg)
    _check_fwd(y, y_r, st, st_r, False, f"statistics, {seg}-row frames")


def test_splitk_red_add():
    """A few-tile problem split over the SMs: the epilogue red.adds fp32 partials into the workspace."""
    prims = _prims()
    N, H, W, C = 16, 4, 4, 640
    assert prims.native.lib().t2v_conv_workspace_bytes(0, N, H, W, C, C, 3, 3, 1, 1, 1, 1, 1) > 0
    g = torch.Generator(device=DEV).manual_seed(27)
    x = _rnd(g, N, H, W, C)
    w = _rnd(g, C, 3, 3, C, scale=(9 * C) ** -0.5)
    bias = torch.randn(C, device=DEV, generator=g)
    res = _rnd(g, N, H, W, C)
    for out_fp32 in (False, True):
        y, y_r, _, _ = _fwd_both(x, w, bias, res, 1, (1, 1, 1, 1), out_fp32=out_fp32)
        _check_fwd(y, y_r, None, None, out_fp32, f"split-K (fp32 output: {out_fp32})")


def test_bf16_fwd_deterministic():
    """No atomics on the bf16 forward path: the same launch twice gives bitwise-equal outputs."""
    prims = _prims()
    g = torch.Generator(device=DEV).manual_seed(28)
    x = _rnd(g, 16, 32, 32, 320)
    w = _rnd(g, 320, 3, 3, 320, scale=(9 * 320) ** -0.5)
    bias = torch.randn(320, device=DEV, generator=g)
    res = _rnd(g, 16, 32, 32, 320)
    y0 = prims.conv_fwd(x, w, bias, None, res, 1, (1, 1, 1, 1))
    y1 = prims.conv_fwd(x, w, bias, None, res, 1, (1, 1, 1, 1))
    assert torch.equal(y0, y1)
