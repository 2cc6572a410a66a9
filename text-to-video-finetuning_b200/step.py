"""Training-step glue of the hot path: the H100-native equivalents of the reference's
`tensor_to_vae_latent` (train.py:339-347), `sample_noise` (:349-358), `noise_scheduler.add_noise` (:760) and the
epsilon / v-prediction MSE of `finetune_unet` (:720-836), the noise schedule of the checkpoint's scheduler config (:119), plus
the data-parallel step object used by train.py and bench.py."""
import json
import math
import os
from typing import NamedTuple, Optional

import torch
import torch.distributed as dist

from . import ops, prims
from .runtime import GradientBuckets, GraphedStep, ParamArena, allreduce_gradients

PREDICTION_TYPES = ("epsilon", "v_prediction")
BETA_SCHEDULES = ("linear", "scaled_linear", "squaredcos_cap_v2")
LOSS_TYPES = ("l2", "huber", "smooth_l1")
HUBER_SCHEDULES = ("constant", "exponential", "snr")


class LossObjective(NamedTuple):
    """The per-pass training objective (diffusers' --snr_gamma, --loss_type, --huber_schedule, --huber_c), for B samples
    with a_b = alphas_cumprod[t_b], d = pred - target:
        loss = mean_b(w_b * mean_{c,f,h,w} psi(d))
        psi  'l2': d^2   'huber': 2 c_b (sqrt(d^2 + c_b^2) - c_b)   'smooth_l1': 2 (sqrt(d^2 + c_b^2) - c_b)
        c_b  'constant': huber_c   'exponential': huber_c ** (t_b / T)
             'snr': (1 - huber_c) / (1 + sigma_b)^2 + huber_c, sigma_b = sqrt((1 - a_b) / a_b)   (huber_c at a_b = 0)
        w_b  snr_gamma None: 1; else, with snr_b = a_b / (1 - a_b), min(snr_b, gamma) / snr_b for 'epsilon' (1 at a_b = 0)
             and min(snr_b, gamma) / (snr_b + 1) for 'v_prediction' (0 at a_b = 0)   (Hang et al. 2023, Min-SNR-gamma)
    Build it with loss_objective(), which validates the values."""
    snr_gamma: Optional[float] = None
    loss_type: str = "l2"
    huber_schedule: str = "snr"
    huber_c: float = 0.1

    @property
    def plain(self):
        """The unweighted MSE: the step then runs mse_loss / velocity_mse_loss, the kernels of the default objective."""
        return self.loss_type == "l2" and self.snr_gamma is None


def loss_objective(snr_gamma=None, loss_type="l2", huber_schedule="snr", huber_c=0.1):
    """A validated LossObjective.  An unknown loss_type or huber_schedule, snr_gamma <= 0, or (for 'huber' / 'smooth_l1')
    huber_c <= 0 or, with 'exponential', huber_c > 1 raises ValueError.  Under 'l2' huber_c is not used."""
    if loss_type not in LOSS_TYPES:
        raise ValueError(f"loss_type {loss_type!r} is not supported; expected one of {LOSS_TYPES}")
    if huber_schedule not in HUBER_SCHEDULES:
        raise ValueError(f"huber_schedule {huber_schedule!r} is not supported; expected one of {HUBER_SCHEDULES}")
    if snr_gamma is not None:
        if isinstance(snr_gamma, bool) or not isinstance(snr_gamma, (int, float)) or not snr_gamma > 0:
            raise ValueError(f"snr_gamma = {snr_gamma!r}: expected None or a number > 0")
        snr_gamma = float(snr_gamma)
    if loss_type != "l2":
        if isinstance(huber_c, bool) or not isinstance(huber_c, (int, float)) or not (huber_c > 0 and math.isfinite(huber_c)):
            raise ValueError(f"huber_c = {huber_c!r}: expected a finite number > 0")
        if huber_schedule == "exponential" and huber_c > 1:
            raise ValueError(f"huber_c = {huber_c!r}: the 'exponential' huber_schedule needs huber_c <= 1")
        huber_c = float(huber_c)
    return LossObjective(snr_gamma, loss_type, huber_schedule, huber_c)


def ddpm_alphas_cumprod(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, device=None):
    """'scaled_linear' DDPM schedule of the ms-1.7b / zeroscope scheduler config (DDPMScheduler.alphas_cumprod)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    a = torch.cumprod(1.0 - betas, dim=0)
    return a.to(device) if device is not None else a


def _rescale_zero_terminal_snr(betas):
    """Lin et al. 2023, 'Common Diffusion Noise Schedules and Sample Steps are Flawed', Algorithm 1: shift sqrt(abar) so its
    last value is 0, scale it so its first value is unchanged, and rebuild the betas from ratios of consecutive abar."""
    abar_sqrt = torch.cumprod(1.0 - betas, dim=0).sqrt()
    first, last = abar_sqrt[0].clone(), abar_sqrt[-1].clone()
    abar_sqrt = (abar_sqrt - last) * (first / (first - last))
    abar = abar_sqrt ** 2
    alphas = torch.cat([abar[0:1], abar[1:] / abar[:-1]])
    return 1.0 - alphas


def schedule_from_config(config):
    """A diffusers scheduler config (the dict of scheduler/scheduler_config.json) -> (alphas_cumprod fp32 [T], prediction_type),
    computed as DDPMScheduler.__init__ does (reference train.py:119 builds its DDPMScheduler from this file).  Missing keys
    take the ms-1.7b / zeroscope values, so `{}` gives `ddpm_alphas_cumprod()`.  Keys it does not act on (clip_sample,
    steps_offset, ...) only concern sampling; an unknown beta_schedule or prediction_type raises ValueError."""
    cfg = dict(config or {})
    prediction_type = cfg.get("prediction_type") or "epsilon"
    if prediction_type not in PREDICTION_TYPES:
        # 'sample' too: the reference's loss target (train.py:792-800) knows only these two
        raise ValueError(f"prediction_type {prediction_type!r} is not supported; expected one of {PREDICTION_TYPES}")
    T = int(cfg.get("num_train_timesteps", 1000))
    beta_start, beta_end = float(cfg.get("beta_start", 0.00085)), float(cfg.get("beta_end", 0.012))
    schedule = cfg.get("beta_schedule", "scaled_linear")
    if cfg.get("trained_betas") is not None:
        betas = torch.tensor(cfg["trained_betas"], dtype=torch.float32)
    elif schedule == "linear":
        betas = torch.linspace(beta_start, beta_end, T, dtype=torch.float32)
    elif schedule == "scaled_linear":
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, T, dtype=torch.float32) ** 2
    elif schedule == "squaredcos_cap_v2":
        def abar(s):
            return math.cos((s + 0.008) / 1.008 * math.pi / 2) ** 2
        betas = torch.tensor([min(1 - abar((i + 1) / T) / abar(i / T), 0.999) for i in range(T)], dtype=torch.float32)
    else:
        raise ValueError(f"beta_schedule {schedule!r} is not supported; expected one of {BETA_SCHEDULES}")
    if cfg.get("rescale_betas_zero_snr", False):
        betas = _rescale_zero_terminal_snr(betas)
    return torch.cumprod(1.0 - betas, dim=0), prediction_type


def load_noise_schedule(pretrained_model_path):
    """(alphas_cumprod, prediction_type) of `<pretrained_model_path>/scheduler/scheduler_config.json`; a folder without that
    file (a UNet-only checkpoint) gets the ms-1.7b / zeroscope defaults, `ddpm_alphas_cumprod()` and 'epsilon'."""
    path = os.path.join(pretrained_model_path, "scheduler", "scheduler_config.json")
    if not os.path.isfile(path):
        return ddpm_alphas_cumprod(), "epsilon"
    with open(path) as f:
        return schedule_from_config(json.load(f))


def sample_noise(latents, noise_strength=0.0, use_offset_noise=False, generator=None):
    """train.py:349-358: Gaussian noise, optionally plus `strength * randn(B, C, F, 1, 1)` offset noise."""
    noise = torch.randn(latents.shape, device=latents.device, dtype=latents.dtype, generator=generator)
    if use_offset_noise:
        b, c, f = latents.shape[:3]
        noise = noise + noise_strength * torch.randn(b, c, f, 1, 1, device=latents.device, dtype=latents.dtype, generator=generator)
    return noise


def finetune_loss(unet, latents, noise, timesteps, encoder_hidden_states, alphas_cumprod, return_pred=False, prediction_type="epsilon",
                  snr_gamma=None, loss_type="l2", huber_schedule="snr", huber_c=0.1):
    """One UNet pass of finetune_unet:
       noisy = add_noise(latents, noise, t)  ->  pred = unet(noisy, t, text)  ->  mse(pred.float(), target.float())
    with target = noise for prediction_type 'epsilon' and get_velocity(latents, noise, t) for 'v_prediction' (train.py:792-800).
    add_noise is fused into the layout-conversion kernel at the input, the loss reads the channels-last prediction
    directly (and forms the velocity per element), so no (B,C,F,H,W) activation is ever materialised.
    snr_gamma / loss_type / huber_schedule / huber_c replace the MSE by the objective of LossObjective; with their defaults
    the loss is the MSE above."""
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"prediction_type {prediction_type!r} is not supported; expected one of {PREDICTION_TYPES}")
    objective = loss_objective(snr_gamma, loss_type, huber_schedule, huber_c)
    B, C, F, H, W = latents.shape
    x = prims.latents_to_nhwc8(latents.float().contiguous(), noise.float().contiguous(), alphas_cumprod, timesteps.to(torch.int64).contiguous())
    text = unet.prepare_text(encoder_hidden_states)
    pred = unet.forward_channels_last(x, timesteps.to(torch.int64).contiguous(), text, B, F)
    if not objective.plain:
        x0 = latents.float().contiguous() if prediction_type == "v_prediction" else None
        loss = ops.diffusion_loss_nhwc8(pred, x0, noise.float().contiguous(), alphas_cumprod, timesteps.to(torch.int64).contiguous(),
                                        objective)
    elif prediction_type == "v_prediction":
        loss = ops.velocity_mse_loss_nhwc8(pred, latents.float().contiguous(), noise.float().contiguous(), alphas_cumprod,
                                           timesteps.to(torch.int64).contiguous())
    else:
        loss = ops.mse_loss_nhwc8(pred, noise.float().contiguous())
    if return_pred:
        return loss, prims.nhwc8_to_latents(pred.detach(), B, C, F)
    return loss


class DataParallelStep:
    """One optimisation micro-step per call: fwd + bwd of `passes` UNet passes over one clip batch per rank; on the boundary
    of a gradient-accumulation window ONE gradient all-reduce and, when an optimizer is attached, the fused AdamW step -
    the whole thing captured in a CUDA graph and replayed (`use_graph`).

    `passes=2` reproduces the reference's two-pass video step (train.py:814-834, H3: loss = loss_0 + loss_1);
    throughput is reported per pass with passes=1.

    Gradient bookkeeping (reference: accelerator.accumulate / backward / optimizer.step / zero_grad, train.py:739-879):
      * gradients accumulate in the flat fp32 buffer across the micro-steps of a window; every loss is scaled by
        1 / accumulation (what accelerator.backward does);
      * the all-reduce runs only on the window's last micro-step;
      * with an attached optim.FusedAdamW the update kernel consumes and zeroes the gradients and rewrites the bf16 shadow,
        so neither a memset nor a cast pass remains in the step.  Without one (a torch optimizer, or fwd+bwd only) the
        buffer is zeroed at the start of each window and the shadow is re-cast from the masters every call.

    `prediction_type` picks the loss target of every pass: the noise ('epsilon') or the velocity ('v_prediction').
    `snr_gamma`, `loss_type`, `huber_schedule` and `huber_c` pick the objective (LossObjective, validated by loss_objective);
    each pass takes it, and the two passes' losses are summed and scaled by 1 / accumulation as the MSE's are.

    `text_encoder` (a text_encoder.CLIPTextModel that trains: cloneofsimo LoRA injected, `use_text_lora`, and/or parameters
    unfrozen by `train_text_encoder`): the call then takes the prompt token ids (B, L) in place of the text states, and the
    step follows train.py:803-834: the encoder runs once, in the step (and the graph); with passes=2 and F > 1, pass 0 is the
    full clip on the detached states and pass 1 only frame 1 of the clip on the trainable states - the one pass whose
    gradient reaches the text encoder; with F = 1 one pass on the trainable states.  The arena adopts the trainable text
    tensors next to the UNet's parameters, so clipping, the optimizers and the EMA cover them.  With LoRA only, those are the
    LoRA factors (the frozen encoder weights stay outside); when base weights train, every text parameter is adopted, as the
    UNet's are, so the text optimizer group (which lists the frozen ones too, train.py:579-595) lives in the arena and the
    trainable projection weights are read through the arena's bf16 shadow."""

    def __init__(self, unet, alphas_cumprod, passes=1, use_graph=False, adopt=True, optimizer=None, accumulation=1,
                 prediction_type="epsilon", text_encoder=None, snr_gamma=None, loss_type="l2", huber_schedule="snr", huber_c=0.1):
        if prediction_type not in PREDICTION_TYPES:
            raise ValueError(f"prediction_type {prediction_type!r} is not supported; expected one of {PREDICTION_TYPES}")
        self.objective = loss_objective(snr_gamma, loss_type, huber_schedule, huber_c)
        self.unet = unet
        self.abar = alphas_cumprod
        self.prediction_type = prediction_type
        self.passes = passes
        self.text_encoder = text_encoder
        text_params = ()
        if text_encoder is not None:
            every = text_encoder.base_trains()
            text_params = [p for p in text_encoder.parameters() if p.requires_grad or every]
        self.arena = ParamArena(unet, extra=text_params) if adopt else None
        self.use_graph = use_graph
        self.sync_gradients = True   # set False to run fwd+bwd only (profiling on a single rank)
        self.optimizer = optimizer
        self.accumulation = max(1, int(accumulation))
        self._micro = 0
        self._graphs = {}
        # A capture draws the dropout host seeds from torch's CPU generator (twice in warm-up, once in the capture) and the
        # graph keeps the last ones.  capture_rng: graph key (without the optimizer generation) -> the CPU generator state at
        # the start of its capture.  replay_rng: states a resumed run captures those keys from, so its graphs hold the seeds
        # of the run it continues (train.py, save_training_state).
        self.capture_rng, self.replay_rng = {}, {}
        self._gscale = None
        # world > 1: per-block gradient all-reduces are issued from inside the backward pass (overlap), see GradientBuckets
        self.buckets = None
        if (self.arena is not None and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
                and not os.environ.get("T2V_NO_OVERLAP")):
            self.buckets = GradientBuckets(self.arena, unet)
            self.buckets.install()

    def attach_optimizer(self, optimizer):
        self.optimizer = optimizer
        self._graphs = {}
        self.capture_rng = {}

    def _fwd_bwd(self, latents, noise, timesteps, text, first, last):
        """first / last: position of this micro-step inside its accumulation window."""
        fused = self.optimizer is not None and hasattr(self.optimizer, "launch")
        if self.arena is not None and not fused:
            if first:
                self.arena.zero_grads()
            self.arena.refresh_shadow()
        elif fused and first and not self.optimizer.covers_all_trainable():
            self.arena.zero_grads()   # trainable parameters outside the optimizer would otherwise accumulate forever
        ops.bump_dropout_epoch(latents.device)
        if self._gscale is None or self._gscale.device != latents.device:
            self._gscale = torch.empty((), device=latents.device, dtype=torch.float32)
            self._gscale.fill_(1.0 / self.accumulation)
        total = None
        reduce_now = last and self.sync_gradients
        overlap = self.buckets is not None and reduce_now
        if self.text_encoder is None:
            runs = [(latents, noise, text)] * self.passes
        else:
            B, L = text.shape                              # text = prompt token ids
            states = self.text_encoder.encode(text).view(B, L, -1)
            if self.passes > 1 and latents.shape[2] > 1:
                runs = [(latents, noise, states.detach()), (latents[:, :, 1:2], noise[:, :, 1:2], states)]
            else:
                runs = [(latents, noise, states)]
        for i, (lat, nz, st) in enumerate(runs):
            loss = finetune_loss(self.unet, lat, nz, timesteps, st, self.abar, prediction_type=self.prediction_type,
                                 **self.objective._asdict())
            if overlap:
                self.buckets.armed = i == len(runs) - 1   # gradients are final only in the last pass
            loss.backward(self._gscale if self.accumulation > 1 else None)
            total = loss.detach() if total is None else total + loss.detach()
        comm = None
        if overlap:
            self.buckets.finish()
            if fused:
                comm = self.buckets.comm          # bf16 all-reduced gradients: the update reads them directly
            else:
                self.buckets.widen()              # a torch optimizer / a test wants them in param.grad (fp32)
        elif reduce_now and self.arena is not None:
            allreduce_gradients(self.arena)
        if fused and last:
            self.optimizer.launch(zero_grad=True, grad_bf16=comm)
        return total

    def __call__(self, latents, noise, timesteps, encoder_hidden_states):
        """encoder_hidden_states: the text states (B, L, D), or with a text encoder attached its token ids (B, L)."""
        if self.arena is not None:
            self.arena.check_layout()
            self.arena.reattach_grads()
        first = self._micro % self.accumulation == 0
        last = (self._micro + 1) % self.accumulation == 0
        self._micro += 1
        fused = self.optimizer is not None and hasattr(self.optimizer, "launch")
        if fused and last:
            self.optimizer.push_hyperparams()   # learning rate of this step -> device (outside the graph)
        args = (latents, noise, timesteps, encoder_hidden_states)
        if self.use_graph:
            key = (first, last, self.passes, self.sync_gradients, getattr(self.optimizer, "generation", 0),
                   tuple(tuple(a.shape) for a in args))
            g = self._graphs.get(key)
            if g is None:
                seeds_key = key[:4] + key[5:]
                recorded = self.replay_rng.pop(seeds_key, None)
                live = None
                if recorded is not None:   # draw the seeds the interrupted run drew, then give the live stream back
                    live = torch.get_rng_state()
                    torch.set_rng_state(recorded)
                self.capture_rng[seeds_key] = torch.get_rng_state()
                # the capture runs the step for real (warm-up + capture replays nothing): keep the optimizer state and the
                # weights of those dry runs out of the training trajectory
                g = self._graphs[key] = GraphedStep(lambda *a: self._fwd_bwd(*a, first, last), args, snapshot=self._snapshot())
                if live is not None:
                    torch.set_rng_state(live)
            return g(*args)
        return self._fwd_bwd(*args, first, last)

    def _snapshot(self):
        """Tensors the dry runs of a graph capture must not change for good: weights, gradients and optimizer state."""
        keep = []
        if self.arena is not None:
            keep += [self.arena.master, self.arena.grad, self.arena.shadow]
        opt = self.optimizer
        if opt is not None and hasattr(opt, "launch"):
            keep += opt.state_tensors()
        keep.append(ops.dropout_epoch(self.abar.device))
        return keep

    @property
    def _graph(self):   # bench.py / tests poke at this to drop captured graphs before tearing NCCL down
        return self._graphs

    @_graph.setter
    def _graph(self, value):
        self._graphs = {} if value is None else value
