"""Validation preview - SURVEY 8(f) row 4 (reference train.py:908-958: every `validation_steps` the trained UNet, in eval mode,
samples a short clip with `DPMSolverMultistepScheduler` through `TextToVideoSDPipeline` and writes it with `export_to_video`).

Here: the same sampler written out (DPM-Solver++ (2M), lower-order final step - the diffusers defaults the reference uses -
on the training run's noise schedule and prediction type, epsilon or v), classifier-free guidance with the frozen CLIP text encoder, the H100-native UNet
and VAE decoder, and OpenCV for the .mp4.  Nothing here is on the training hot path; it runs a handful of UNet forwards."""
import math
import os

import torch


class DPMSolverMultistep:
    """DPM-Solver++ multistep, order 2 (midpoint), for an epsilon- or v-prediction model.

    With alpha_t = sqrt(abar_t), sigma_t = sqrt(1 - abar_t), lambda_t = log(alpha_t / sigma_t), the data prediction is
    x0 = (x - sigma_t eps) / alpha_t ('epsilon') or x0 = alpha_t x - sigma_t v ('v_prediction'), and one step s -> t
    (h = lambda_t - lambda_s) is
        first order   x_t = (sigma_t / sigma_s) x_s - alpha_t (e^{-h} - 1) D0
        second order  x_t = (sigma_t / sigma_s) x_s - alpha_t (e^{-h} - 1) (D0 + D1 / 2),  D1 = (D0 - D0_prev) / r,  r = h_prev / h
    The first step and (for fewer than 15 steps) the last step are first order.  A zero-terminal-SNR schedule (abar[T-1] = 0)
    has its last abar raised to 2^-24, as diffusers' DPMSolverMultistepScheduler does, so sigma / alpha stays finite."""

    def __init__(self, alphas_cumprod, num_inference_steps, lower_order_final=True, prediction_type="epsilon"):
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"prediction_type {prediction_type!r} is not supported; expected 'epsilon' or 'v_prediction'")
        self.prediction_type = prediction_type
        ac = alphas_cumprod.double().cpu().clone()
        if ac[-1] == 0:
            ac[-1] = 2.0 ** -24
        T = ac.shape[0]
        ts = torch.linspace(0, T - 1, num_inference_steps + 1).round().long().flip(0)[:-1]   # 'linspace' spacing, descending
        self.timesteps = ts
        self.alpha = ac.sqrt()
        self.sigma = (1 - ac).sqrt()
        self.lam = torch.log(self.alpha) - torch.log(self.sigma)
        self.n = num_inference_steps
        self.lower_order_final = lower_order_final and num_inference_steps < 15
        self.prev_x0, self.prev_t, self.i = None, None, 0

    def _coef(self, t):
        if t < 0:      # the step after the last training timestep lands on clean data
            return 1.0, 0.0, float("inf")
        return float(self.alpha[t]), float(self.sigma[t]), float(self.lam[t])

    def step(self, eps, x):
        """eps: the model output at the current timestep (a velocity for 'v_prediction')."""
        s = int(self.timesteps[self.i])
        t = int(self.timesteps[self.i + 1]) if self.i + 1 < self.n else -1
        a_s, sg_s, lam_s = self._coef(s)
        if self.prediction_type == "v_prediction":
            x0 = a_s * x - sg_s * eps
        else:
            x0 = (x - sg_s * eps) / a_s
        if t < 0:
            # final step to t = 0: e^{-h} -> 0, sigma_t -> 0: x_0 = x0-prediction (plus the second-order correction's limit)
            a_t, sg_t, lam_t = float(self.alpha[0]), float(self.sigma[0]), float(self.lam[0])
        else:
            a_t, sg_t, lam_t = self._coef(t)
        h = lam_t - lam_s
        first = self.prev_x0 is None or (self.lower_order_final and self.i == self.n - 1)
        if first:
            out = (sg_t / sg_s) * x - a_t * math.expm1(-h) * x0
        else:
            h0 = lam_s - float(self.lam[self.prev_t])
            r0 = h0 / h
            d1 = (x0 - self.prev_x0) / r0
            out = (sg_t / sg_s) * x - a_t * math.expm1(-h) * x0 - 0.5 * a_t * math.expm1(-h) * d1
        self.prev_x0, self.prev_t = x0, s
        self.i += 1
        return out


@torch.no_grad()
def sample_latents(unet, alphas_cumprod, cond, uncond, shape, num_inference_steps=25, guidance_scale=9.0, generator=None, device="cuda",
                   prediction_type="epsilon"):
    """Classifier-free-guided sampling of a latent clip (B, 4, F, h, w) with the UNet in eval mode; guidance mixes the model
    outputs, whichever quantity they predict (as the diffusers pipeline does)."""
    was_training = unet.training
    unet.eval()
    try:
        x = torch.randn(shape, generator=generator, device="cpu").to(device)
        sched = DPMSolverMultistep(alphas_cumprod, num_inference_steps, prediction_type=prediction_type)
        for t in sched.timesteps.tolist():
            tt = torch.full((shape[0],), t, device=device, dtype=torch.int64)
            e_c = unet(x, tt, cond).sample.float()
            if guidance_scale != 1.0 and uncond is not None:
                e_u = unet(x, tt, uncond).sample.float()
                e_c = e_u + guidance_scale * (e_c - e_u)
            x = sched.step(e_c, x)
        return x
    finally:
        unet.train(was_training)


@torch.no_grad()
def decode_latents(vae, latents):
    """(B, 4, F, h, w) scaled latents -> uint8 video (B, F, H, W, 3): the pipeline's decode_latents + tensor2vid."""
    B, C, F, h, w = latents.shape
    z = (latents / 0.18215).permute(0, 2, 1, 3, 4).reshape(B * F, C, h, w)
    img = vae.decode(z).sample
    img = ((img.float() / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8)
    return img.view(B, F, 3, img.shape[-2], img.shape[-1]).permute(0, 1, 3, 4, 2).contiguous().cpu()


def export_to_video(frames_u8, path, fps=8):
    """uint8 (F, H, W, 3) RGB -> .mp4 (OpenCV; the reference uses diffusers.utils.export_to_video, also OpenCV)."""
    import cv2
    F, H, W, _ = frames_u8.shape
    w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (W, H))
    for f in frames_u8.numpy():
        w.write(cv2.cvtColor(f, cv2.COLOR_RGB2BGR))
    w.release()
    return path


@torch.no_grad()
def validation_sample(unet, vae, text_encoder, tokenizer, validation_data, out_dir, step, fallback_prompt, device,
                      alphas_cumprod=None, prediction_type="epsilon"):
    """reference train.py:908-958 with the `validation_data:` YAML section (prompt, sample_preview, num_frames, width, height,
    num_inference_steps, guidance_scale).  The solver uses the training schedule and prediction type (the reference builds
    its solver from the pipeline's scheduler config, train.py:925); without one, the ms-1.7b / zeroscope defaults."""
    vd = dict(validation_data or {})
    if not vd.get("sample_preview", True):
        return None
    from .step import ddpm_alphas_cumprod
    from .utils.dataset import get_prompt_ids
    prompt = vd.get("prompt") or fallback_prompt or ""
    os.makedirs(out_dir, exist_ok=True)
    cond = text_encoder(get_prompt_ids(prompt, tokenizer).to(device))[0]
    uncond = text_encoder(get_prompt_ids("", tokenizer).to(device))[0]
    shape = (1, 4, int(vd.get("num_frames", 16)), int(vd.get("height", 256)) // 8, int(vd.get("width", 256)) // 8)
    abar = ddpm_alphas_cumprod() if alphas_cumprod is None else alphas_cumprod
    lat = sample_latents(unet, abar, cond, uncond, shape, int(vd.get("num_inference_steps", 25)),
                         float(vd.get("guidance_scale", 9.0)), device=device, prediction_type=prediction_type)
    video = decode_latents(vae, lat)[0]
    name = "".join(c if c.isalnum() else "_" for c in prompt)[:40] or "sample"
    path = os.path.join(out_dir, f"{step}_{name}.mp4")
    export_to_video(video, path, fps=int(vd.get("fps", 8)))
    return path
