"""Min-SNR-gamma weighting and scheduled pseudo-Huber losses on the CPU: the float64 restatement's identities
(tests/loss_objective_ref.py), the validation of the four options, the step over the emulated primitives against autograd
through the restatement (one pass, two passes, B = 2 with different timesteps, accumulation 2, both prediction types),
train.main end to end with a resume that changes the options, and the default objective staying on the MSE kernels."""
import contextlib
import itertools
import math
import shutil

import pytest
import torch

import loss_objective_ref as LO
from helpers import rel_l2, seeded_state_dict

SMALL = dict(block_out_channels=(32, 64, 64, 64), attention_head_dim=32, cross_attention_dim=32)
LOSSES = ("l2", "huber", "smooth_l1")
SCHEDULES = ("constant", "exponential", "snr")


def _zero_snr():
    from t2v_b200 import step as S
    abar = S.schedule_from_config({"rescale_betas_zero_snr": True})[0]
    assert abar[-1].item() == 0.0
    return abar


def _obj(**kw):
    from t2v_b200 import step as S
    return S.loss_objective(**kw)


# ------------------------------------------------------------------------------------------------ identities (float64)
def test_snr_gamma_above_every_snr_is_plain_mse_under_epsilon():
    from t2v_b200 import step as S
    g = torch.Generator().manual_seed(0)
    x0, noise, pred = (torch.randn(4, 4, 2, 3, 5, generator=g, dtype=torch.float64) for _ in range(3))
    t = torch.tensor([0, 1, 500, 999])
    for abar in (S.ddpm_alphas_cumprod(), _zero_snr()):
        a = abar.double()
        gamma = float((a / (1 - a)).max()) * (1 + 1e-12)
        got = LO.objective_loss(pred, x0, noise, t, abar, _obj(snr_gamma=gamma), "epsilon")
        want = ((pred - noise) ** 2).mean()
        assert abs(got.item() - want.item()) <= 1e-14 * want.item(), (got.item(), want.item())
        # and a gamma below some snr changes it: the weight is live
        low = LO.objective_loss(pred, x0, noise, t, abar, _obj(snr_gamma=1.0), "epsilon")
        assert low.item() < want.item() * (1 - 1e-3)


def test_huber_tends_to_the_square_for_small_errors():
    d = torch.tensor([1e-3, -2e-4, 5e-5], dtype=torch.float64)
    for c in (0.1, 0.5, 2.0):
        ratio = LO.psi(d, torch.tensor(c, dtype=torch.float64), "huber") / d ** 2
        assert torch.allclose(ratio, torch.ones_like(ratio), rtol=1e-4 / c ** 2, atol=0), (c, ratio)
    # and to 2 c |d| (linear) for large ones
    big = torch.tensor([1e4, -3e4], dtype=torch.float64)
    r = LO.psi(big, torch.tensor(0.1, dtype=torch.float64), "huber") / (2 * 0.1 * big.abs())
    assert torch.allclose(r, torch.ones_like(r), rtol=1e-4)


def test_smooth_l1_tends_to_twice_the_absolute_error():
    d = torch.tensor([0.3, -1.7, 4.0, -0.01], dtype=torch.float64)
    prev = math.inf
    for c in (1e-2, 1e-4, 1e-6, 1e-9):
        err = float((LO.psi(d, torch.tensor(c, dtype=torch.float64), "smooth_l1") / (2 * d.abs()) - 1).abs().max())
        assert err <= prev
        prev = err
    assert prev < 1e-6


@pytest.mark.parametrize("ptype", ["epsilon", "v_prediction"])
def test_limits_at_zero_abar_are_finite(ptype):
    abar = _zero_snr()
    t = torch.tensor([len(abar) - 1, 0, 500])
    a = abar.double()[t]
    w = LO.snr_weight(a, 5.0, ptype)
    assert torch.isfinite(w).all() and w[0].item() == (1.0 if ptype == "epsilon" else 0.0)
    c = LO.huber_scale(a, t, 0.1, "snr", len(abar))
    assert torch.isfinite(c).all() and c[0].item() == 0.1
    # a = 1 (snr = inf) is finite too: both weights tend to 0
    assert LO.snr_weight(torch.tensor([1.0], dtype=torch.float64), 5.0, ptype).item() == 0.0
    g = torch.Generator().manual_seed(1)
    x0, noise = torch.randn(3, 4, 2, 3, 3, generator=g, dtype=torch.float64), torch.randn(3, 4, 2, 3, 3, generator=g, dtype=torch.float64)
    pred = torch.randn(3, 4, 2, 3, 3, generator=g, dtype=torch.float64)
    for loss_type, sched in itertools.product(LOSSES, SCHEDULES):
        o = _obj(snr_gamma=5.0, loss_type=loss_type, huber_schedule=sched)
        assert math.isfinite(LO.objective_loss(pred, x0, noise, t, abar, o, ptype).item()), o
        assert torch.isfinite(LO.objective_dpred(pred, x0, noise, t, abar, o, ptype, 1.0)).all(), o


def test_closed_forms_of_the_weights_and_scales():
    a = torch.tensor([0.9, 0.5, 0.01], dtype=torch.float64)
    snr = a / (1 - a)                                  # 9, 1, 1/99
    assert torch.allclose(LO.snr_weight(a, 5.0, "epsilon"), torch.tensor([5 / 9, 1.0, 1.0], dtype=torch.float64))
    assert torch.allclose(LO.snr_weight(a, 5.0, "v_prediction"), torch.minimum(snr, torch.tensor(5.0)) / (snr + 1))
    t = torch.tensor([0, 500, 1000])
    assert torch.allclose(LO.huber_scale(a, t, 0.1, "exponential", 1000), torch.tensor([1.0, 0.1 ** 0.5, 0.1], dtype=torch.float64))
    assert torch.allclose(LO.huber_scale(a, t, 0.1, "snr", 1000), 0.9 / (1 + ((1 - a) / a).sqrt()) ** 2 + 0.1)


@pytest.mark.parametrize("ptype", ["epsilon", "v_prediction"])
def test_written_out_derivative_equals_autograd(ptype):
    abar = _zero_snr()
    g = torch.Generator().manual_seed(2)
    x0, noise = torch.randn(3, 4, 2, 3, 5, generator=g, dtype=torch.float64), torch.randn(3, 4, 2, 3, 5, generator=g, dtype=torch.float64)
    t = torch.tensor([len(abar) - 1, 0, 321])
    for loss_type, sched, gamma in itertools.product(LOSSES, SCHEDULES, (None, 5.0)):
        o = _obj(snr_gamma=gamma, loss_type=loss_type, huber_schedule=sched)
        p = torch.randn(3, 4, 2, 3, 5, generator=g, dtype=torch.float64).requires_grad_(True)
        LO.objective_loss(p, x0, noise, t, abar, o, ptype).mul(0.37).backward()
        got = LO.objective_dpred(p.detach(), x0, noise, t, abar, o, ptype, 0.37)
        assert torch.allclose(got, p.grad, rtol=1e-12, atol=1e-18), o


# ------------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("kw,word", [(dict(loss_type="l1"), "loss_type"), (dict(loss_type="huber", huber_schedule="cosine"), "huber_schedule"),
                                     (dict(huber_schedule="linear"), "huber_schedule"),
                                     (dict(snr_gamma=0), "snr_gamma"), (dict(snr_gamma=-5.0), "snr_gamma"), (dict(snr_gamma="5"), "snr_gamma"),
                                     (dict(loss_type="huber", huber_c=0.0), "huber_c"), (dict(loss_type="smooth_l1", huber_c=-0.1), "huber_c"),
                                     (dict(loss_type="huber", huber_schedule="exponential", huber_c=1.5), "exponential")])
def test_invalid_options_raise(kw, word):
    from t2v_b200 import step as S
    with pytest.raises(ValueError, match=word):
        S.loss_objective(**kw)
    with pytest.raises(ValueError, match=word):
        S.DataParallelStep(torch.nn.Linear(2, 2), S.ddpm_alphas_cumprod(), adopt=False, **kw)


def test_valid_options_and_l2_ignores_the_huber_keys():
    from t2v_b200 import step as S
    assert S.loss_objective() == S.LossObjective(None, "l2", "snr", 0.1) and S.loss_objective().plain
    assert S.loss_objective(huber_c=5.0, huber_schedule="exponential").plain        # l2: huber_c is not used
    assert not S.loss_objective(snr_gamma=5).plain and S.loss_objective(snr_gamma=5).snr_gamma == 5.0
    assert S.loss_objective(loss_type="huber", huber_schedule="constant", huber_c=3.0).huber_c == 3.0   # > 1 fine unless exponential


def test_train_main_rejects_bad_options_before_loading_the_unet(tmp_path):
    """The pretrained folder has no unet/ at all: the ValueError must come first, not a missing-file error."""
    from t2v_b200 import train
    for kw, word in ((dict(loss_type="mae"), "mae"), (dict(snr_gamma=-1), "snr_gamma"),
                     (dict(loss_type="huber", huber_schedule="exponential", huber_c=2.0), "exponential")):
        with pytest.raises(ValueError, match=word):
            train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "out"), dataset_types=["synthetic"], device="cpu",
                       **kw)


# ------------------------------------------------------------------------------------------------ step over emulated primitives
def _model():
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    m.load_state_dict(seeded_state_dict(m, 5))
    return m.eval().requires_grad_(True)


def _inputs(B, F, abar):
    g = torch.Generator().manual_seed(11)
    lat = torch.randn(B, 4, F, 8, 8, generator=g) * 2.0
    noise = torch.randn(B, 4, F, 8, 8, generator=g)
    t = torch.tensor([len(abar) - 1, 0, 100, 640][:B])
    return lat, noise, t, torch.randn(B, 3, 32, generator=g)


def _run_step(case, reference):
    """Loss per micro-step, the dpred of every loss backward, and the arena gradient of one optimisation window."""
    from oracle import ops_ref
    from t2v_b200 import ops, prims
    from t2v_b200 import step as S
    abar = _zero_snr()
    B, F, passes, accumulation, ptype, opts = case
    want = S.loss_objective(**opts)
    lat, noise, t, ehs = _inputs(B, F, abar)
    dpreds, losses = [], []
    old_bf = ops_ref.BF
    ops_ref.BF = torch.float32
    saved = ops.diffusion_loss_nhwc8, prims.diffusion_loss_bwd
    try:
        with LO.emulated():
            if reference:
                def op(pred, x0, nz, a, ts, objective):
                    assert objective == want and (x0 is not None) == (ptype == "v_prediction")
                    pred.register_hook(lambda g: dpreds.append(g.detach().clone()))
                    p = ops_ref.nhwc8_to_latents(pred, nz.shape[0], nz.shape[1], nz.shape[2])
                    return LO.objective_loss(p, x0, nz, ts, abar, want, ptype).float()
                ops.diffusion_loss_nhwc8 = op
            else:
                bwd = prims.diffusion_loss_bwd

                def rec(*a):
                    d = bwd(*a)
                    dpreds.append(d.clone())
                    return d
                prims.diffusion_loss_bwd = rec
            st = S.DataParallelStep(_model(), abar, passes=passes, accumulation=accumulation, prediction_type=ptype, **opts)
            k = B // accumulation
            for j in range(accumulation):
                s = slice(j * k, (j + 1) * k)
                losses.append(float(st(lat[s], noise[s], t[s], ehs[s])))
            grad = st.arena.grad.clone()
    finally:
        ops.diffusion_loss_nhwc8, prims.diffusion_loss_bwd = saved
        ops_ref.BF = old_bf
    return losses, dpreds, grad


STEP_CASES = {
    # (B, F, passes, accumulation, prediction type, options)
    "eps_gamma_b2": (2, 2, 1, 1, "epsilon", dict(snr_gamma=5.0)),
    "v_gamma_huber_snr_two_pass": (2, 2, 2, 1, "v_prediction", dict(snr_gamma=5.0, loss_type="huber")),
    "eps_smooth_l1_exponential_accumulation": (2, 1, 1, 2, "epsilon", dict(loss_type="smooth_l1", huber_schedule="exponential")),
    "v_huber_constant_b2": (2, 2, 1, 1, "v_prediction", dict(loss_type="huber", huber_schedule="constant", huber_c=0.3)),
    "eps_gamma_smooth_l1_snr_two_pass_accumulation": (4, 2, 2, 2, "epsilon", dict(snr_gamma=2.0, loss_type="smooth_l1")),
}


@pytest.mark.parametrize("case", list(STEP_CASES))
def test_step_matches_autograd_through_the_restatement(case):
    losses, dpreds, grad = _run_step(STEP_CASES[case], reference=False)
    losses_r, dpreds_r, grad_r = _run_step(STEP_CASES[case], reference=True)
    B, F, passes, accumulation, _, _ = STEP_CASES[case]
    assert len(dpreds) == len(dpreds_r) == passes * accumulation
    for a, b in zip(losses, losses_r):
        assert math.isfinite(a) and abs(a - b) <= 1e-5 * abs(b), (losses, losses_r)
    for a, b in zip(dpreds, dpreds_r):
        assert (a - b).abs().max() <= 1e-5 * b.abs().max(), (a - b).abs().max()
    assert grad_r.norm() > 0 and rel_l2(grad, grad_r) <= 1e-5, rel_l2(grad, grad_r)


def test_options_change_the_step():
    """The same inputs under the default objective give another loss and gradient: the options reach the kernel."""
    base = _run_step((2, 2, 1, 1, "epsilon", {}), reference=False)
    weighted = _run_step(STEP_CASES["eps_gamma_b2"], reference=False)
    assert abs(base[0][0] - weighted[0][0]) > 1e-3 * base[0][0]
    assert rel_l2(weighted[2], base[2]) > 1e-2


# ------------------------------------------------------------------------------------------------ default objective
@pytest.mark.parametrize("ptype", ["epsilon", "v_prediction"])
def test_default_objective_runs_the_mse_kernels(ptype):
    from oracle import ops_ref
    from t2v_b200 import prims
    from t2v_b200 import step as S
    import v_prediction_ref as V
    abar = _zero_snr()
    lat, noise, t, ehs = _inputs(2, 2, abar)
    names = ("mse_loss_fwd", "mse_loss_bwd", "velocity_mse_loss_fwd", "velocity_mse_loss_bwd", "diffusion_loss_fwd", "diffusion_loss_bwd")
    calls = dict.fromkeys(names, 0)
    old_bf = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        with V.emulated_prims(), LO.emulated():
            saved = {n: getattr(prims, n) for n in names}

            def counted(n):
                def run(*a):
                    calls[n] += 1
                    return saved[n](*a)
                return run
            for n in names:
                setattr(prims, n, counted(n))
            try:
                st = S.DataParallelStep(_model(), abar, passes=2, prediction_type=ptype, loss_type="l2", huber_schedule="constant",
                                        huber_c=7.0)
                st(lat, noise, t, ehs)
            finally:
                for n, fn in saved.items():
                    setattr(prims, n, fn)
    finally:
        ops_ref.BF = old_bf
    pre = "velocity_mse_loss" if ptype == "v_prediction" else "mse_loss"
    assert calls[pre + "_fwd"] == 2 and calls[pre + "_bwd"] == 2, calls
    assert sum(calls.values()) == 4, calls


# ------------------------------------------------------------------------------------------------ train.main
@contextlib.contextmanager
def _emulated_with_optimizer():
    """tests/ema_ref.py's emulation (the fused optimizer kernels) plus the loss primitives."""
    from ema_ref import emulated as ema_emulated
    from t2v_b200 import prims
    saved = {n: getattr(prims, n) for n in LO.PRIMS}
    with ema_emulated():
        for n in LO.PRIMS:
            setattr(prims, n, getattr(LO, n))
        try:
            yield
        finally:
            for n, fn in saved.items():
                setattr(prims, n, fn)


def test_train_main_with_options_and_a_resume_that_changes_them(tmp_path, monkeypatch):
    from test_resume_cpu import _main, _record_losses, _synthetic, _unet_folder
    root = _unet_folder(str(tmp_path / "model"))
    calls = {"new": 0}
    fwd = LO.diffusion_loss_fwd

    def counted(*a):
        calls["new"] += 1
        return fwd(*a)
    monkeypatch.setattr(LO, "diffusion_loss_fwd", counted)
    losses = _record_losses(monkeypatch)
    opts_a = dict(snr_gamma=5.0, loss_type="huber", huber_schedule="snr", huber_c=0.1)
    opts_b = dict(snr_gamma=1.0, loss_type="smooth_l1", huber_schedule="exponential", huber_c=0.05)
    part = str(tmp_path / "part")
    with _emulated_with_optimizer():
        r = _main(**_synthetic(root, **opts_a), output_dir=part, max_train_steps=1, save_training_state=True)
        assert r["steps"] == 1 and r["stepper"].objective == tuple(opts_a.values()) and calls["new"] == 2   # two passes
        first = list(losses)
        resumed = {}
        for name, opts in (("same", opts_a), ("changed", opts_b)):
            del losses[:]
            calls["new"] = 0
            out = str(tmp_path / name)
            shutil.copytree(part, out)
            res = _main(**_synthetic(root, **opts), output_dir=out, max_train_steps=3, resume_from_checkpoint=out)
            assert res["steps"] == 3 and calls["new"] == 4 and res["stepper"].objective == tuple(opts.values()), (name, calls)
            resumed[name] = list(losses)
    assert all(math.isfinite(v) for v in first + resumed["same"] + resumed["changed"])
    # the resumed run takes the options of its own call: same data and weights, another objective, another loss
    assert all(abs(a - b) > 1e-3 * abs(a) for a, b in zip(resumed["same"], resumed["changed"])), resumed
    # and the same options continue the saved run bit for bit
    del losses[:]
    with _emulated_with_optimizer():
        _main(**_synthetic(root, **opts_a), output_dir=str(tmp_path / "full"), max_train_steps=3)
    assert first + resumed["same"] == losses, (first, resumed["same"], losses)
