"""v-prediction on the H100: the fused velocity loss kernel (t2v_velocity_mse_loss) against its fp32 restatement
(tests/v_prediction_ref.py), the small UNet end to end against the oracle, CUDA-graph replays with changing timesteps, and
train.main on a v-prediction, zero-terminal-SNR pipeline folder with a validation preview."""
import pytest
import torch

import v_prediction_ref as V
from helpers import cosine, rel_l2, seeded_state_dict
from oracle import ops_ref

pytestmark = pytest.mark.gpu

SMALL = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)


def _kernel_inputs(B=2, C=4, F=3, H=5, W=7, seed=0):
    from t2v_b200 import step as S
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, C, F, H, W, generator=g) * 2.0
    noise = torch.randn(B, C, F, H, W, generator=g)
    pred = ops_ref.latents_to_nhwc8(torch.randn(B, C, F, H, W, generator=g))     # bf16 [B*F, H, W, 8], channels C..7 zero
    t = torch.tensor([0, 999] + [417] * (B - 2))[:B]
    abar = S.ddpm_alphas_cumprod()
    return [x.cuda() for x in (pred, x0, noise, abar, t)]


@pytest.mark.parametrize("shape", [dict(B=2, C=4, F=3, H=5, W=7), dict(B=2, C=4, F=16, H=32, W=32), dict(B=3, C=8, F=2, H=9, W=4)])
def test_velocity_loss_kernel_matches_reference(shape):
    from t2v_b200 import prims
    pred, x0, noise, abar, t = _kernel_inputs(**shape)
    if shape["B"] == 3:
        t = torch.tensor([999, 0, 531], device="cuda")
    loss = prims.velocity_mse_loss_fwd(pred, x0, noise, abar, t)
    loss_r = V.velocity_mse_loss_fwd(pred.cpu(), x0.cpu(), noise.cpu(), abar.cpu(), t.cpu())
    assert abs(loss.item() - loss_r.item()) <= 1e-5 * loss_r.item(), (loss.item(), loss_r.item())
    gout = torch.tensor(0.37, device="cuda")     # 1 / accumulation-style scale, not 1
    d = prims.velocity_mse_loss_bwd(pred, x0, noise, abar, t, gout)
    d_r = V.velocity_mse_loss_bwd(pred.cpu(), x0.cpu(), noise.cpu(), abar.cpu(), t.cpu(), gout.cpu())
    C = shape["C"]
    assert d.dtype == torch.bfloat16 and d.shape == pred.shape
    assert rel_l2(d.float().cpu()[..., :C], d_r.float()[..., :C]) < 5e-3
    assert not d[..., C:].float().any(), "padded channels must get a zero gradient"
    # the noise-target kernel on the same operands is a different loss: the operands really select the objective
    assert abs(prims.mse_loss_fwd(pred, noise).item() - loss.item()) > 0.1 * loss.item()


def test_velocity_loss_of_the_rounded_target_is_at_bf16_level():
    from t2v_b200 import prims
    _, x0, noise, abar, t = _kernel_inputs(B=2, C=4, F=4, H=16, W=16)
    v = V.get_velocity(x0, noise, t, abar)
    pred = ops_ref.latents_to_nhwc8(v.cpu()).cuda()            # bf16 of the velocity
    loss = prims.velocity_mse_loss_fwd(pred, x0, noise, abar, t).item()
    # bf16 keeps 8 significant bits: |rounding error| <= 2^-9 |v|
    assert 0 < loss <= 2.0 ** -18 * v.pow(2).mean().item(), (loss, v.pow(2).mean().item())


def test_small_unet_v_prediction_matches_oracle():
    from oracle import leaves as L
    from oracle import unet3d_ref as R
    from test_unet_gpu import _check
    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    sd = seeded_state_dict(m, 0)
    m.load_state_dict(sd)
    m = m.cuda().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(2, 4, 4, 16, 16, generator=g) * 0.18215 * 5
    noise = torch.randn(2, 4, 4, 16, 16, generator=g)
    t = torch.tensor([999, 250])
    ehs = torch.randn(2, 7, 64, generator=g)
    abar = L.ddpm_alphas_cumprod()
    loss, pred = S.finetune_loss(m, lat.cuda(), noise.cuda(), t.cuda(), ehs.cuda(), abar.cuda(), return_pred=True,
                                 prediction_type="v_prediction")
    loss.backward()
    torch.cuda.synchronize()
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    loss_r, pred_r = V.finetune_loss(p, R.full_config(**SMALL), lat, noise, t, ehs, abar, prediction_type="v_prediction")
    loss_r.backward()
    grads = {n: (q.grad.detach().cpu() if q.grad is not None else None, p[n].grad) for n, q in m.named_parameters()}
    _check(loss.item(), loss_r.item(), pred.detach().float().cpu(), pred_r.detach(), grads)


def test_graph_replay_with_changing_timesteps_matches_eager():
    """The velocity coefficients are read on the device: every replay of the captured step uses that step's timesteps."""
    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    steppers = []
    for graph in (False, True):
        m = UNet3DConditionModel(**SMALL)
        m.load_state_dict(seeded_state_dict(m, 2))
        m = m.cuda().eval().requires_grad_(True)
        steppers.append(S.DataParallelStep(m, S.schedule_from_config({"rescale_betas_zero_snr": True})[0].cuda(), passes=1,
                                           use_graph=graph, prediction_type="v_prediction"))
    g = torch.Generator().manual_seed(5)
    lat = (torch.randn(2, 4, 2, 16, 16, generator=g) * 2).cuda()
    noise = torch.randn(2, 4, 2, 16, 16, generator=g).cuda()
    ehs = torch.randn(2, 7, 64, generator=g).cuda()
    eager, graph = [], []
    schedule = ([0, 999], [999, 0], [500, 3], [0, 999])
    for ts in schedule:
        t = torch.tensor(ts, device="cuda")
        eager.append(steppers[0](lat, noise, t, ehs).item())
        graph.append(steppers[1](lat, noise, t, ehs).item())
        # two models, two runs: split-K reduction order moves the small-model loss at the 1e-4 level (DESIGN §5: 2e-3)
        assert abs(eager[-1] - graph[-1]) <= 2e-3 * eager[-1], (ts, eager[-1], graph[-1])
        ga, gb = steppers[1].arena.grad, steppers[0].arena.grad       # bf16 level, as in tests/test_unet_gpu.py
        assert cosine(ga, gb) > 0.999 and abs(ga.norm().item() - gb.norm().item()) <= 2e-2 * gb.norm().item(), ts
    assert len(steppers[1]._graphs) == 1
    # every replay matches the eager step of ITS timesteps more closely than the eager step of any other timesteps
    for k, ts in enumerate(schedule):
        others = [abs(graph[k] - eager[j]) for j in range(len(schedule)) if schedule[j] != ts]
        assert abs(graph[k] - eager[k]) < min(others), (k, graph, eager)


def test_train_main_v_prediction_gpu(tmp_path):
    from test_v_prediction_cpu import V_ZERO_SNR, run_v_training
    from t2v_b200 import step as S
    r, calls = run_v_training(tmp_path, "cuda:0", validate=True)
    assert r["steps"] == 2 and r["stepper"].prediction_type == "v_prediction"
    assert r["stepper"].use_graph and len(r["stepper"]._graphs) == 1
    assert calls["v"] > 0 and calls["eps"] == 0, calls          # captured once, replayed: the noise-target loss never ran
    assert torch.equal(r["stepper"].abar.cpu(), S.schedule_from_config(V_ZERO_SNR)[0])
    assert len(calls["decoded"]) == 1 and torch.isfinite(calls["decoded"][0]).all()
    assert len(list((tmp_path / "out" / "samples").iterdir())) == 1
