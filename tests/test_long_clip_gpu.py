"""Clips longer than 32 frames on the H100: t2v_attn_long_fwd / bwd against their fp32 restatement (tests/long_clip_ref.py)
with the tolerances of tests/test_kernels_gpu.py::test_temporal_attention, determinism, rejected shapes, the UNet at 48 and
64 frames against the oracle, a CUDA-graph step at 40 frames and train.main with a 48-frame validation preview."""
import pytest
import torch

import long_clip_ref as LC
from helpers import cosine, seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"


def close(a, b, tol, what="", floor=1e-6):
    a, b = a.float(), b.float()
    err = (a - b).abs().max().item() / max(b.abs().max().item(), floor)
    assert err < tol, f"{what}: rel-to-max error {err:.3e} >= {tol}"


def _case(B, F, HW, heads, D, fused, seed=7, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    C, rows = heads * D, B * F * HW
    rnd = lambda *s: (torch.randn(*s, device=DEV, generator=g) * scale).to(torch.bfloat16)
    if fused:
        qkv = rnd(rows, 3 * C)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    else:
        q, k, v = (rnd(rows, C) for _ in range(3))
    do = (torch.randn(rows, C, device=DEV, generator=g)).to(torch.bfloat16)
    addr = (B * HW, HW, F * HW, 1, HW, 3 * C if fused else C, C, heads, F, D)
    return q, k, v, do, addr


def _grads(q, fused, C):
    """gradient buffers in the layout of the inputs (the fused [rows, 3C] buffer when fused)"""
    rows = q.shape[0]
    buf = torch.zeros(rows, 3 * C, device=DEV, dtype=torch.bfloat16)
    if fused:
        return buf[:, :C], buf[:, C:2 * C], buf[:, 2 * C:]
    return tuple(buf.view(3, rows, C)[i] for i in range(3))


def _run(prims_or_ref, q, k, v, do, addr, o=None, lse=None):
    nseq, heads, L = addr[0], addr[7], addr[8]
    C = addr[6]
    o = torch.zeros_like(do) if o is None else o
    lse = torch.zeros(nseq, heads, L, device=DEV) if lse is None else lse
    prims_or_ref.attn_long_fwd(q, k, v, o, lse, addr)
    grads = _grads(q, addr[5] != C, C)
    prims_or_ref.attn_long_bwd(q, k, v, o, do, lse, *grads, addr)
    return o, lse, grads


CASES = [(1, 33, 16, 2, 64), (2, 48, 9, 5, 64), (1, 64, 64, 5, 64), (1, 100, 4, 1, 32), (1, 128, 16, 8, 64), (1, 256, 4, 2, 64),
         (2, 40, 1, 1, 64), (1, 1, 16, 2, 64), (2, 16, 9, 2, 64), (1, 32, 4, 8, 64)]


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("B,F,HW,heads,D", CASES)
def test_attn_long_matches_reference(B, F, HW, heads, D, fused):
    from t2v_b200 import prims
    q, k, v, do, addr = _case(B, F, HW, heads, D, fused)
    o, lse, grads = _run(prims, q, k, v, do, addr)
    # the reference backward runs on the kernel's own o and lse, so each gradient is checked on its own
    o_r, lse_r = torch.zeros_like(do), torch.zeros_like(lse)
    LC.attn_long_fwd(q, k, v, o_r, lse_r, addr)
    close(o, o_r, 1e-2, "attn_long fwd")
    assert (lse - lse_r).abs().max().item() < 1e-3 * max(1.0, lse_r.abs().max().item()), "attn_long lse"
    exp = _grads(q, fused, heads * D)
    LC.attn_long_bwd(q, k, v, o_r, do, lse_r, *exp, addr)
    # at L = 1, dq is exactly zero; delta from the bf16-rounded o leaves a residue at 2^-9 of dv's scale, not at 1e-6
    floor = 1e-3 * exp[2].abs().max().item()
    for name, a, b in zip("qkv", grads, exp):
        close(a, b, 1.5e-2, f"attn_long d{name}", floor)


@pytest.mark.parametrize("fused", [False, True])
def test_large_logits_stay_finite(fused):
    """|q.k| / sqrt(D) around 50: the online softmax must not overflow and the rows stay one-hot-like but finite."""
    from t2v_b200 import prims
    q, k, v, do, addr = _case(1, 96, 8, 2, 64, fused, seed=3, scale=4.0)
    o, lse, grads = _run(prims, q, k, v, do, addr)
    big = (q.float()[:, :64] * k.float()[:, :64]).sum(-1).abs().max().item() / 8
    assert big > 30, big
    for t in (o, lse, *grads):
        assert torch.isfinite(t.float()).all()
    o_r, lse_r = torch.zeros_like(do), torch.zeros_like(lse)
    LC.attn_long_fwd(q, k, v, o_r, lse_r, addr)
    close(o, o_r, 1e-2, "fwd")
    assert (lse - lse_r).abs().max().item() < 1e-3 * lse_r.abs().max().item()
    exp = _grads(q, fused, 128)
    LC.attn_long_bwd(q, k, v, o_r, do, lse_r, *exp, addr)
    for name, a, b in zip("qkv", grads, exp):
        close(a, b, 1.5e-2, f"d{name}")


def test_forward_and_backward_are_bitwise_deterministic():
    from t2v_b200 import prims
    q, k, v, do, addr = _case(2, 200, 16, 4, 64, True, seed=9)
    first = _run(prims, q, k, v, do, addr)
    for _ in range(2):
        again = _run(prims, q, k, v, do, addr)
        assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1])
        for a, b in zip(first[2], again[2]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("what", ["L=257", "D=48", "pitch"])
def test_rejected_shapes_raise_before_launching(what):
    from t2v_b200 import native, prims
    L, D, ld = {"L=257": (257, 64, 128), "D=48": (40, 48, 96), "pitch": (40, 64, 132)}[what]
    heads, HW = 2, 2
    rows = L * HW
    x = torch.zeros(rows, 3 * heads * D, device=DEV, dtype=torch.bfloat16)
    q = x[:, :heads * D]
    o = torch.zeros(rows, heads * D, device=DEV, dtype=torch.bfloat16)
    lse = torch.zeros(HW, heads, L, device=DEV)
    addr = (HW, HW, L * HW, 1, HW, ld, heads * D, heads, L, D)
    n0 = native.launch_count()
    with pytest.raises(RuntimeError, match="attn_long"):
        prims.attn_long_fwd(q, q, q, o, lse, addr)
    with pytest.raises(RuntimeError, match="attn_long"):
        prims.attn_long_bwd(q, q, q, o, o, lse, q, q, q, addr)
    assert native.launch_count() == n0


SMALL = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)


def test_small_unet_48_frames_matches_oracle():
    from test_unet_gpu import _case as unet_case
    from test_unet_gpu import _check
    _check(*unet_case(SMALL, 1, 48, (16, 16)))


def test_small_unet_64_frames_with_gradient_checkpointing_matches_oracle():
    """The backward runs on recomputed activations: the recompute must reproduce o and lse of the first forward."""
    from test_unet_gpu import _case as unet_case
    from test_unet_gpu import _check
    _check(*unet_case(SMALL, 1, 64, (8, 8), ckpt=True))


def test_graph_step_at_40_frames_matches_eager():
    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from oracle import leaves as L
    steppers = []
    for graph in (False, True):
        m = UNet3DConditionModel(**SMALL)
        m.load_state_dict(seeded_state_dict(m, 2))
        m = m.cuda().eval().requires_grad_(True)
        steppers.append(S.DataParallelStep(m, L.ddpm_alphas_cumprod().cuda(), passes=1, use_graph=graph))
    g = torch.Generator().manual_seed(5)
    lat = (torch.randn(1, 4, 40, 8, 8, generator=g) * 0.9).cuda()
    noise = torch.randn(1, 4, 40, 8, 8, generator=g).cuda()
    ehs = torch.randn(1, 7, 64, generator=g).cuda()
    for ts in ([999], [250], [3]):
        t = torch.tensor(ts, device="cuda")
        eager = steppers[0](lat, noise, t, ehs).item()
        replay = steppers[1](lat, noise, t, ehs).item()
        assert abs(eager - replay) <= 2e-3 * eager, (ts, eager, replay)
        ga, gb = steppers[1].arena.grad, steppers[0].arena.grad
        assert cosine(ga, gb) > 0.999 and abs(ga.norm().item() - gb.norm().item()) <= 2e-2 * gb.norm().item(), ts
    assert len(steppers[1]._graphs) == 1


def test_train_main_40_frames_with_48_frame_preview_gpu(tmp_path):
    from test_v_prediction_cpu import _pipeline_folder
    from t2v_b200 import prims, sampling, train
    from test_v_prediction_cpu import ZEROSCOPE
    root = _pipeline_folder(str(tmp_path / "pipe"), ZEROSCOPE)
    decoded, calls = [], {"long": 0}
    dec, fwd = sampling.decode_latents, prims.attn_long_fwd

    def d(vae, lat):
        decoded.append(lat.float().cpu())
        return dec(vae, lat)

    def f(*a):
        calls["long"] += 1
        return fwd(*a)
    sampling.decode_latents, prims.attn_long_fwd = d, f
    try:
        r = train.main(pretrained_model_path=root, output_dir=str(tmp_path / "out"), dataset_types=["synthetic"],
                       train_data=dict(n=2, n_sample_frames=40, height=64, width=64), max_train_steps=2, learning_rate=1e-4,
                       checkpointing_steps=10, seed=0, shuffle=False, device="cuda:0", eval_train=True, trainable_modules=["attn1"],
                       load_side_models=True, validation_steps=2,
                       validation_data=dict(prompt="a dog", sample_preview=True, num_frames=48, width=32, height=32,
                                            num_inference_steps=2, guidance_scale=2.0))
    finally:
        sampling.decode_latents, prims.attn_long_fwd = dec, fwd
    assert r["steps"] == 2
    assert r["stepper"].use_graph and len(r["stepper"]._graphs) == 1
    assert calls["long"] > 0
    assert len(decoded) == 1 and 48 in decoded[0].shape and torch.isfinite(decoded[0]).all()
    assert len(list((tmp_path / "out" / "samples").iterdir())) == 1
