"""v-prediction checkpoints on the CPU: the noise schedule and prediction type read from scheduler/scheduler_config.json
(step.schedule_from_config against the DDPMScheduler formulas), the velocity target's identities, the v-prediction step
over the emulated primitives against its fp32 restatement (tests/v_prediction_ref.py), train.main on a v-prediction
pipeline folder, and the DPM-Solver++ sampler for a v-model."""
import json
import math
import os

import numpy as np
import pytest
import torch

import v_prediction_ref as V
from helpers import rel_l2, seeded_state_dict

SMALL = dict(block_out_channels=(32, 64, 64, 64), attention_head_dim=32, cross_attention_dim=32)
TINY = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)
ZEROSCOPE = {"_class_name": "DDPMScheduler", "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear",
             "num_train_timesteps": 1000, "prediction_type": "epsilon", "clip_sample": False, "steps_offset": 1}


def _cumprod32(betas):
    return torch.cumprod(1.0 - torch.as_tensor(betas, dtype=torch.float32), dim=0)


# ------------------------------------------------------------------------------------------------ schedule from config
def test_scaled_linear_defaults_equal_ddpm_alphas_cumprod_bitwise():
    from t2v_b200 import step as S
    want = S.ddpm_alphas_cumprod()
    for cfg in ({}, ZEROSCOPE, {"beta_schedule": "scaled_linear"}):
        abar, ptype = S.schedule_from_config(cfg)
        assert abar.dtype == torch.float32 and torch.equal(abar, want), cfg
        assert ptype == "epsilon"


def test_linear_schedule():
    from t2v_b200 import step as S
    abar, _ = S.schedule_from_config({"beta_schedule": "linear", "beta_start": 0.0001, "beta_end": 0.02, "num_train_timesteps": 500})
    assert abar.shape == (500,)
    assert torch.allclose(abar, _cumprod32(np.linspace(0.0001, 0.02, 500)), rtol=0, atol=1e-6)


def test_scaled_linear_schedule_other_constants():
    from t2v_b200 import step as S
    abar, _ = S.schedule_from_config({"beta_schedule": "scaled_linear", "beta_start": 0.0001, "beta_end": 0.03, "num_train_timesteps": 700})
    betas = np.linspace(math.sqrt(0.0001), math.sqrt(0.03), 700) ** 2
    assert abar.shape == (700,) and torch.allclose(abar, _cumprod32(betas), rtol=0, atol=1e-6)


def test_squaredcos_cap_v2_schedule():
    from t2v_b200 import step as S
    T = 1000
    abar, _ = S.schedule_from_config({"beta_schedule": "squaredcos_cap_v2", "num_train_timesteps": T})
    f = [math.cos((i / T + 0.008) / 1.008 * math.pi / 2) ** 2 for i in range(T + 1)]
    betas = [min(1 - f[i + 1] / f[i], 0.999) for i in range(T)]
    assert betas[-1] == 0.999                                    # the cap is active at the end of the schedule
    assert torch.equal(abar, _cumprod32(np.array(betas, dtype=np.float32)))
    # the cosine schedule's closed form abar(t) = f(t) / f(0) holds until the cap
    closed = torch.tensor([f[i + 1] / f[0] for i in range(T)], dtype=torch.float64)
    assert torch.allclose(abar[:900].double(), closed[:900], rtol=1e-4, atol=1e-6)


def test_trained_betas_replace_the_formula():
    from t2v_b200 import step as S
    betas = np.linspace(0.001, 0.05, 64).tolist()
    abar, _ = S.schedule_from_config({"beta_schedule": "linear", "trained_betas": betas, "num_train_timesteps": 1000})
    assert abar.shape == (64,) and torch.equal(abar, _cumprod32(np.array(betas, dtype=np.float32)))
    # a null trained_betas (what diffusers writes) keeps the formula
    abar2, _ = S.schedule_from_config({"beta_schedule": "scaled_linear", "trained_betas": None})
    assert torch.equal(abar2, S.ddpm_alphas_cumprod())


@pytest.mark.parametrize("schedule", ["linear", "scaled_linear", "squaredcos_cap_v2"])
def test_rescale_betas_zero_snr(schedule):
    from t2v_b200 import step as S
    base, _ = S.schedule_from_config({"beta_schedule": schedule})
    abar, _ = S.schedule_from_config({"beta_schedule": schedule, "rescale_betas_zero_snr": True})
    assert abar.dtype == torch.float32 and abar.shape == base.shape
    assert abar[-1].item() == 0.0
    assert abs(abar[0].item() - base[0].item()) <= 1e-7
    snr = abar.double() / (1 - abar.double())
    assert bool((snr[1:] < snr[:-1]).all())
    # Algorithm 1 in fp64: sqrt(abar) shifted and scaled linearly, so the rescaled sqrt(abar) is an affine map of the old one
    s = base.double().sqrt()
    want = ((s - s[-1]) * s[0] / (s[0] - s[-1])) ** 2
    assert torch.allclose(abar.double(), want, rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("cfg,word", [({"prediction_type": "sample"}, "sample"), ({"prediction_type": "x0"}, "x0"),
                                      ({"beta_schedule": "sigmoid"}, "sigmoid"), ({"beta_schedule": "cosine"}, "cosine")])
def test_unknown_values_raise(cfg, word):
    from t2v_b200 import step as S
    with pytest.raises(ValueError, match=word):
        S.schedule_from_config(cfg)


def test_loader_defaults_without_a_scheduler_folder(tmp_path):
    from t2v_b200 import step as S
    abar, ptype = S.load_noise_schedule(str(tmp_path))
    assert torch.equal(abar, S.ddpm_alphas_cumprod()) and ptype == "epsilon"
    os.makedirs(tmp_path / "scheduler")
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(dict(ZEROSCOPE, prediction_type="v_prediction")))
    abar, ptype = S.load_noise_schedule(str(tmp_path))
    assert torch.equal(abar, S.ddpm_alphas_cumprod()) and ptype == "v_prediction"


def test_train_main_rejects_an_unsupported_config_before_loading_the_unet(tmp_path):
    """The pretrained folder has no unet/ at all: the ValueError must come first, not a missing-file error."""
    from t2v_b200 import train
    os.makedirs(tmp_path / "scheduler")
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(dict(ZEROSCOPE, prediction_type="sample")))
    with pytest.raises(ValueError, match="sample"):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "out"), dataset_types=["synthetic"], device="cpu")


def test_step_rejects_an_unknown_prediction_type():
    from t2v_b200 import step as S
    with pytest.raises(ValueError, match="sample"):
        S.DataParallelStep(torch.nn.Linear(2, 2), S.ddpm_alphas_cumprod(), adopt=False, prediction_type="sample")


# ------------------------------------------------------------------------------------------------ velocity target
def test_get_velocity_identities_fp64():
    """x_t = sqrt(a) x0 + sqrt(1-a) eps and v = sqrt(a) eps - sqrt(1-a) x0 are a rotation: sqrt(a) x_t - sqrt(1-a) v = x0 and
    sqrt(1-a) x_t + sqrt(a) v = eps, for every timestep including both ends of a zero-terminal-SNR schedule."""
    from oracle import leaves as L
    from t2v_b200 import step as S
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(4, 4, 3, 5, 6, generator=g, dtype=torch.float64)
    eps = torch.randn(4, 4, 3, 5, 6, generator=g, dtype=torch.float64)
    for abar in (S.ddpm_alphas_cumprod(), S.schedule_from_config({"rescale_betas_zero_snr": True})[0]):
        abar = abar.double()
        t = torch.tensor([0, 17, 600, 999])
        xt = L.add_noise(x0, eps, t, abar)
        v = V.get_velocity(x0, eps, t, abar)
        a = abar[t].view(-1, 1, 1, 1, 1)
        assert torch.allclose(a.sqrt() * xt - (1 - a).sqrt() * v, x0, rtol=0, atol=1e-12)
        assert torch.allclose((1 - a).sqrt() * xt + a.sqrt() * v, eps, rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------ step over emulated primitives
def _small_case():
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    sd = seeded_state_dict(m, 5)
    m.load_state_dict(sd)
    m.eval().requires_grad_(True)
    g = torch.Generator().manual_seed(11)
    # latents of std 3: at t = 999 the velocity is ~ -x0, so its loss is far from the noise target's (std 1)
    lat = torch.randn(2, 4, 2, 16, 16, generator=g) * 3.0
    noise = torch.randn(2, 4, 2, 16, 16, generator=g)
    t = torch.tensor([0, 999])
    ehs = torch.randn(2, 5, 32, generator=g)
    return m, sd, lat, noise, t, ehs


def test_v_prediction_step_matches_oracle_on_emulated_prims():
    """fp32 activations between the emulated primitives and bf16 weight shadows, as in tests/test_data_parallel_cpu.py."""
    from oracle import ops_ref
    from oracle import unet3d_ref as R
    from t2v_b200 import step as S
    m, sd, lat, noise, t, ehs = _small_case()
    abar = S.ddpm_alphas_cumprod()
    calls = {"v": 0}
    old = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        with V.emulated_prims():
            from t2v_b200 import prims
            fwd = prims.velocity_mse_loss_fwd

            def counted(*a):
                calls["v"] += 1
                return fwd(*a)
            prims.velocity_mse_loss_fwd = counted
            loss = S.finetune_loss(m, lat, noise, t, ehs, abar, prediction_type="v_prediction")
            loss.backward()
            with torch.no_grad():
                loss_eps = S.finetune_loss(m, lat, noise, t, ehs, abar)
    finally:
        ops_ref.BF = old
    assert calls["v"] == 1
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    loss_r, _ = V.finetune_loss(p, R.full_config(**SMALL), lat, noise, t, ehs, abar, prediction_type="v_prediction")
    loss_r.backward()
    assert abs(loss.item() - loss_r.item()) <= 2e-2 * loss_r.item(), (loss.item(), loss_r.item())
    # the epsilon target on the same inputs is far away: the test sees which target ran
    assert abs(loss_eps.item() - loss_r.item()) > 0.1 * loss_r.item(), (loss_eps.item(), loss_r.item())
    top = max(v.grad.norm().item() for v in p.values() if v.grad is not None)
    errs = sorted(rel_l2(q.grad, p[n].grad) for n, q in m.named_parameters()
                  if p[n].grad is not None and p[n].grad.norm().item() >= 1e-5 * top)
    # bf16 storage between the emulated primitives: the bound of tests/test_data_parallel_cpu.py
    assert len(errs) > 500 and errs[len(errs) // 2] < 4e-2 and errs[-1] < 0.15, (len(errs), errs[len(errs) // 2], errs[-5:])


def test_velocity_loss_primitives_against_autograd():
    """The hand-written backward of the restated primitive equals autograd of its forward (fp32, no rounding)."""
    from oracle import ops_ref
    from t2v_b200 import step as S
    g = torch.Generator().manual_seed(2)
    x0, noise = torch.randn(2, 3, 2, 4, 4, generator=g), torch.randn(2, 3, 2, 4, 4, generator=g)
    pred32 = torch.randn(2 * 2, 4, 4, 8, generator=g)
    pred32[..., 3:] = 0
    t, abar = torch.tensor([5, 990]), S.ddpm_alphas_cumprod()
    old = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        p = pred32.clone().requires_grad_(True)
        V.velocity_mse_loss_fwd(p, x0, noise, abar, t).backward()
        got = V.velocity_mse_loss_bwd(pred32, x0, noise, abar, t, torch.tensor(1.0))
    finally:
        ops_ref.BF = old
    assert torch.allclose(got[..., :3], p.grad[..., :3], rtol=1e-6, atol=1e-9) and not got[..., 3:].any()


# ------------------------------------------------------------------------------------------------ train.main
def _pipeline_folder(root, scheduler):
    """unet / vae (with decoder) / text_encoder / tokenizer / scheduler, all tiny; the scheduler config is the argument."""
    from transformers import CLIPTextConfig
    from transformers import CLIPTextModel as HF
    from test_pipeline_train import _tiny_tokenizer
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.vae import AutoencoderKL
    unet = UNet3DConditionModel(**TINY)
    unet.load_state_dict(seeded_state_dict(unet, 0))
    unet.save_pretrained(os.path.join(root, "unet"))
    torch.manual_seed(1)
    AutoencoderKL(block_out_channels=(32, 32, 64, 64), layers_per_block=1, build_decoder=True).save_pretrained(os.path.join(root, "vae"))
    nvocab = _tiny_tokenizer(os.path.join(root, "tokenizer"))
    HF(CLIPTextConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=1, vocab_size=nvocab,
                      max_position_embeddings=77, hidden_act="gelu")).save_pretrained(os.path.join(root, "text_encoder"))
    os.makedirs(os.path.join(root, "scheduler"), exist_ok=True)
    with open(os.path.join(root, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump(scheduler, f)
    return root


V_ZERO_SNR = dict(ZEROSCOPE, prediction_type="v_prediction", rescale_betas_zero_snr=True)


def run_v_training(tmp_path, device, validate):
    """Two optimizer steps of train.main on a v-prediction, zero-terminal-SNR pipeline folder; returns main's result, the
    number of velocity-loss and noise-loss forwards, and the latents the validation preview decoded."""
    from t2v_b200 import prims, sampling, train
    root = _pipeline_folder(str(tmp_path / "pipe"), V_ZERO_SNR)
    calls = {"v": 0, "eps": 0, "decoded": []}
    fv, fe, dec = prims.velocity_mse_loss_fwd, prims.mse_loss_fwd, sampling.decode_latents

    def v(*a):
        calls["v"] += 1
        return fv(*a)

    def e(*a):
        calls["eps"] += 1
        return fe(*a)

    def d(vae, lat):
        calls["decoded"].append(lat.float().cpu())
        return dec(vae, lat)
    prims.velocity_mse_loss_fwd, prims.mse_loss_fwd, sampling.decode_latents = v, e, d
    try:
        r = train.main(pretrained_model_path=root, output_dir=str(tmp_path / "out"), dataset_types=["synthetic"],
                       train_data=dict(n=2, n_sample_frames=2, height=64, width=64), max_train_steps=2, learning_rate=1e-4,
                       checkpointing_steps=10, seed=0, shuffle=False, device=device, eval_train=True, trainable_modules=["attn1"],
                       load_side_models=validate, validation_steps=2 if validate else 0,
                       validation_data=dict(prompt="a dog", sample_preview=True, num_frames=2, width=32, height=32,
                                            num_inference_steps=2, guidance_scale=2.0) if validate else None)
    finally:
        prims.velocity_mse_loss_fwd, prims.mse_loss_fwd, sampling.decode_latents = fv, fe, dec
    return r, calls


def test_train_main_takes_the_v_path_cpu(tmp_path):
    from t2v_b200 import step as S
    with V.emulated_prims():
        r, calls = run_v_training(tmp_path, "cpu", validate=True)
    assert r["steps"] == 2 and r["stepper"].prediction_type == "v_prediction"
    # two passes per video step (train.py:814-834), two steps; the noise-target loss never ran
    assert calls["v"] == 4 and calls["eps"] == 0, calls
    abar = r["stepper"].abar
    assert torch.equal(abar.cpu(), S.schedule_from_config(V_ZERO_SNR)[0]) and abar[-1].item() == 0.0
    assert len(calls["decoded"]) == 1 and torch.isfinite(calls["decoded"][0]).all()
    assert len(os.listdir(tmp_path / "out" / "samples")) == 1


# ------------------------------------------------------------------------------------------------ sampler
def _eps_fn(x, t):
    return 0.7 * torch.sin(x + 0.001 * t) + 0.2 * x


def test_v_sampler_trajectory_matches_eps_sampler():
    """A v-model that is the exact image of a fixed eps-model (v = alpha eps - sigma x0_hat) must walk the same trajectory."""
    from t2v_b200 import step as S
    from t2v_b200.sampling import DPMSolverMultistep
    for abar, steps in ((S.ddpm_alphas_cumprod(), 25), (S.schedule_from_config({"beta_schedule": "linear"})[0], 10)):
        se = DPMSolverMultistep(abar, steps)
        sv = DPMSolverMultistep(abar, steps, prediction_type="v_prediction")
        x0 = torch.randn(3, 7, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
        xe, xv = x0.clone(), x0.clone()
        for t in se.timesteps.tolist():
            xe = se.step(_eps_fn(xe, t), xe)
            a, s = sv.alpha[t], sv.sigma[t]
            eps = _eps_fn(xv, t)
            xv = sv.step(a * eps - s * (xv - s * eps) / a, xv)
            assert (xe - xv).abs().max().item() < 1e-6, t
        assert torch.isfinite(xe).all()


class _StubVModel(torch.nn.Module):
    """sample_latents' UNet interface: model(x, t, text).sample -> a bounded velocity."""

    def forward(self, x, t, text):
        class Out:
            pass
        o = Out()
        o.sample = torch.tanh(x) * 0.5 + 0.01 * text.mean()
        return o


def test_zero_terminal_snr_sampling_is_finite():
    from t2v_b200 import step as S
    from t2v_b200.sampling import DPMSolverMultistep, sample_latents
    abar, ptype = S.schedule_from_config(V_ZERO_SNR)
    assert abar[-1].item() == 0.0 and ptype == "v_prediction"
    s = DPMSolverMultistep(abar, 5, prediction_type=ptype)
    assert int(s.timesteps[0]) == 999 and s.alpha[999].item() == 2.0 ** -12     # abar[T-1] raised to 2^-24
    assert abar[-1].item() == 0.0                                                 # the caller's schedule is not modified
    assert torch.isfinite(s.lam).all()
    cond, uncond = torch.ones(1, 3, 4), torch.zeros(1, 3, 4)
    lat = sample_latents(_StubVModel(), abar, cond, uncond, (1, 4, 2, 4, 4), num_inference_steps=5, guidance_scale=3.0,
                         generator=torch.Generator().manual_seed(0), device="cpu", prediction_type=ptype)
    assert lat.shape == (1, 4, 2, 4, 4) and torch.isfinite(lat).all()
