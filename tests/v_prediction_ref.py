"""fp32 restatement of the v-prediction training target (tests only), next to oracle/ops_ref.py and oracle/unet3d_ref.py
which restate the epsilon path.

Reference train.py:792-800 picks the loss target from the scheduler's prediction_type:
    epsilon       target = noise
    v_prediction  target = noise_scheduler.get_velocity(latents, noise, timesteps)
and DDPMScheduler.get_velocity is  sqrt(abar_t) * noise - sqrt(1 - abar_t) * latents  (Salimans & Ho 2022, section 4).
PARITY UNPINNED: diffusers is not installed, so this restatement is checked only against the identities it must satisfy
(tests/test_v_prediction_cpu.py), like the rest of the oracle."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import leaves as L
from oracle import ops_ref
from oracle import unet3d_ref as R


def get_velocity(latents, noise, timesteps, alphas_cumprod):
    """DDPMScheduler.get_velocity: abar gathered per sample, broadcast over (C, F, H, W), in the latents' dtype."""
    a = alphas_cumprod.to(latents.dtype)[timesteps].view(-1, *([1] * (latents.dim() - 1)))
    return a.sqrt() * noise - (1 - a).sqrt() * latents


def finetune_loss(p, cfg, latents, noise, timesteps, encoder_hidden_states, alphas_cumprod=None, prediction_type="epsilon"):
    """train.py:751-834, one UNet pass: add_noise -> UNet -> F.mse_loss(pred.float(), target.float()) with the target of
    train.py:792-800."""
    if alphas_cumprod is None:
        alphas_cumprod = L.ddpm_alphas_cumprod()
    if prediction_type == "epsilon":
        return R.finetune_loss(p, cfg, latents, noise, timesteps, encoder_hidden_states, alphas_cumprod)
    if prediction_type != "v_prediction":
        raise ValueError(f"Unknown prediction type {prediction_type}")
    noisy = L.add_noise(latents, noise, timesteps, alphas_cumprod)
    pred = R.unet3d_forward(p, cfg, noisy, timesteps, encoder_hidden_states)
    target = get_velocity(latents, noise, timesteps, alphas_cumprod)
    return F.mse_loss(pred.float(), target.float(), reduction="mean"), pred


# ---------------------------------------------------------------------------------- primitives (prims.* signatures)
def velocity_mse_loss_fwd(pred, x0, noise, alphas_cumprod, timesteps):
    B, C, Fr, H, W = x0.shape
    p = ops_ref.nhwc8_to_latents(pred, B, C, Fr)
    return ((p - get_velocity(x0, noise, timesteps, alphas_cumprod)) ** 2).mean()


def velocity_mse_loss_bwd(pred, x0, noise, alphas_cumprod, timesteps, gout):
    B, C, Fr, H, W = x0.shape
    p = ops_ref.nhwc8_to_latents(pred, B, C, Fr)
    g = 2.0 * (p - get_velocity(x0, noise, timesteps, alphas_cumprod)) / p.numel() * gout
    return ops_ref.latents_to_nhwc8(g)


PRIMS = ("velocity_mse_loss_fwd", "velocity_mse_loss_bwd")


@contextlib.contextmanager
def emulated_prims():
    """helpers.emulated_prims() plus the velocity loss above: the whole v-prediction step on the CPU."""
    from helpers import emulated_prims as base
    from t2v_b200 import prims
    saved = {n: getattr(prims, n) for n in PRIMS}
    with base():
        for n in PRIMS:
            setattr(prims, n, globals()[n])
        try:
            yield
        finally:
            for n, fn in saved.items():
                setattr(prims, n, fn)
