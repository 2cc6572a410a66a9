"""float64 restatement of the training objectives of step.LossObjective (tests only): Min-SNR-gamma weighting (Hang et al.,
'Efficient Diffusion Training via Min-SNR Weighting Strategy', ICCV 2023) and the scheduled pseudo-Huber / smooth-L1 loss
(Khrapov & Popov, 'Improving Diffusion Models's Data-Corruption Resistance using Scheduled Pseudo-Huber Loss', 2024), written
from their formulas, not from csrc/elementwise.cu (which rewrites them to avoid cancellation and division by zero):

    a_b = abar[t_b], snr_b = a_b / (1 - a_b), sigma_b = sqrt((1 - a_b) / a_b), d = pred - y (y: noise, or the velocity)
    psi   l2: d^2   huber: 2 c_b (sqrt(d^2 + c_b^2) - c_b)   smooth_l1: 2 (sqrt(d^2 + c_b^2) - c_b)
    c_b   constant: huber_c   exponential: exp(-t_b (-ln huber_c) / T)   snr: (1 - huber_c) / (1 + sigma_b)^2 + huber_c
    w_b   None: 1   epsilon: min(snr_b, gamma) / snr_b   v_prediction: min(snr_b, gamma) / (snr_b + 1)
    loss = mean_b(w_b mean_{c,f,h,w} psi)
with the limits at a_b = 0 taken explicitly: epsilon weight 1, v weight 0, snr-scheduled c_b = huber_c.
PARITY UNPINNED: diffusers is not installed, so these are checked against the identities they must satisfy
(tests/test_loss_objective_cpu.py).  The prims restatements below are patched into t2v_b200.prims by `emulated()`, as
tests/text_train_ref.py patches its own."""
import contextlib

import torch


def _col(x, ndim):
    return x.view(-1, *([1] * (ndim - 1)))


def target(x0, noise, timesteps, alphas_cumprod, prediction_type, dtype=torch.float64):
    """y: the noise ('epsilon') or DDPMScheduler.get_velocity: sqrt(a) noise - sqrt(1 - a) x0 ('v_prediction')."""
    if prediction_type == "epsilon":
        return noise.to(dtype)
    a = _col(alphas_cumprod.detach().cpu().to(dtype)[timesteps.cpu()].to(noise.device), noise.dim())
    return a.sqrt() * noise.to(dtype) - (1 - a).sqrt() * x0.to(dtype)


def snr_weight(a, snr_gamma, prediction_type):
    """w_b of abar[t_b] (any float dtype); 1 when snr_gamma is None."""
    if snr_gamma is None:
        return torch.ones_like(a)
    snr = a / (1 - a)                      # 0 at a = 0, inf at a = 1
    m = torch.clamp(snr, max=snr_gamma)    # min(snr, gamma)
    if prediction_type == "epsilon":
        return torch.where(a > 0, m / snr, torch.ones_like(a))
    return torch.where(a > 0, m / (snr + 1), torch.zeros_like(a))


def huber_scale(a, timesteps, huber_c, huber_schedule, T):
    """c_b of abar[t_b] and t_b."""
    if huber_schedule == "constant":
        return torch.full_like(a, huber_c)
    if huber_schedule == "exponential":
        return torch.exp(-timesteps.to(a.dtype) * (-torch.log(torch.tensor(huber_c, dtype=a.dtype))) / T)
    assert huber_schedule == "snr", huber_schedule
    sigma = ((1 - a) / a).sqrt()
    return torch.where(a > 0, (1 - huber_c) / (1 + sigma) ** 2 + huber_c, torch.full_like(a, huber_c))


def psi(d, c, loss_type):
    if loss_type == "l2":
        return d * d
    s = (d * d + c * c).sqrt() - c
    return 2 * c * s if loss_type == "huber" else 2 * s


def dpsi(d, c, loss_type):
    if loss_type == "l2":
        return 2 * d
    r = d / (d * d + c * c).sqrt()
    return 2 * c * r if loss_type == "huber" else 2 * r


def terms(objective, alphas_cumprod, timesteps, prediction_type, dtype=torch.float64):
    """(w_b, c_b) as [B] tensors of `dtype`; c_b is None under 'l2'."""
    a = alphas_cumprod.detach().cpu().to(dtype)[timesteps.cpu()]
    w = snr_weight(a, objective.snr_gamma, prediction_type)
    c = None
    if objective.loss_type != "l2":
        c = huber_scale(a, timesteps.cpu(), objective.huber_c, objective.huber_schedule, alphas_cumprod.numel())
    return w, c


def objective_loss(pred, x0, noise, timesteps, alphas_cumprod, objective, prediction_type, dtype=torch.float64):
    """The pass loss of (B, C, F, H, W) pred, differentiable (autograd) in `dtype`."""
    w, c = terms(objective, alphas_cumprod, timesteps, prediction_type, dtype)
    d = pred.to(dtype) - target(x0, noise, timesteps, alphas_cumprod, prediction_type, dtype)
    cc = None if c is None else _col(c.to(d.device), d.dim())
    per_sample = psi(d, cc, objective.loss_type).flatten(1).mean(1)
    return (w.to(d.device) * per_sample).mean()


def objective_dpred(pred, x0, noise, timesteps, alphas_cumprod, objective, prediction_type, gout, dtype=torch.float64):
    """d loss / d pred written out: gout w_b psi'(d) / numel."""
    w, c = terms(objective, alphas_cumprod, timesteps, prediction_type, dtype)
    d = pred.to(dtype) - target(x0, noise, timesteps, alphas_cumprod, prediction_type, dtype)
    cc = None if c is None else _col(c.to(d.device), d.dim())
    return float(gout) * _col(w.to(d.device), d.dim()) * dpsi(d, cc, objective.loss_type) / d.numel()


# ---------------------------------------------------------------------------------- primitives (prims.* signatures)
def diffusion_loss_fwd(pred, x0, noise, alphas_cumprod, timesteps, objective):
    from oracle import ops_ref
    B, C, Fr, H, W = noise.shape
    ptype = "epsilon" if x0 is None else "v_prediction"
    p = ops_ref.nhwc8_to_latents(pred, B, C, Fr)
    return objective_loss(p, x0, noise, timesteps, alphas_cumprod, objective, ptype).float()


def diffusion_loss_bwd(pred, x0, noise, alphas_cumprod, timesteps, objective, gout):
    from oracle import ops_ref
    B, C, Fr, H, W = noise.shape
    ptype = "epsilon" if x0 is None else "v_prediction"
    p = ops_ref.nhwc8_to_latents(pred, B, C, Fr)
    return ops_ref.latents_to_nhwc8(objective_dpred(p, x0, noise, timesteps, alphas_cumprod, objective, ptype, gout).float())


PRIMS = ("diffusion_loss_fwd", "diffusion_loss_bwd")


@contextlib.contextmanager
def emulated():
    """helpers.emulated_prims() plus the two loss primitives above: a step with any objective on the CPU."""
    from helpers import emulated_prims
    from t2v_b200 import prims
    saved = {n: getattr(prims, n) for n in PRIMS}
    with emulated_prims():
        for n in PRIMS:
            setattr(prims, n, globals()[n])
        try:
            yield
        finally:
            for n, fn in saved.items():
                setattr(prims, n, fn)
