#!/usr/bin/env python
"""Cost of the training objectives (snr_gamma, loss_type) on an H100.

Kernels: every variant of the loss kernel - today's MSE (mse_loss / velocity_mse_loss) and t2v_diffusion_loss with each loss
form (l2, huber, smooth_l1, 'snr' Huber schedule) with and without Min-SNR-gamma weighting, for both prediction types - at the
latent shapes of bench.py's workloads (cfg 2: 1x4x16x32x32; lora: 1x4x16x40x72; zeroscope: 1x4x24x40x72).  Forward and
backward are timed separately with CUDA events over --kernel-launches launches after a warm-up, and reported next to the
algorithmic bytes: forward reads pred (bf16, 8 channels) and the fp32 noise (and x0 for the velocity); backward reads the same
and writes dpred (bf16, 8 channels).  GB/s = bytes / time.  The launches are captured in a CUDA graph and replayed, so the
time is the device's (the forward's includes its 4-byte memset of the loss), not the host call's.

Step: the cfg-2 step of bench.py (one fwd+bwd pass + FusedAdamW, CUDA-graph replay) with the default objective,
snr_gamma 5, and loss_type 'huber' (snr schedule), alternated --reps times in one process, each leg re-captured and timed over
--steps replays after --warmup.  The card's name and power limit are read in the same run.
Usage: python tools/loss_objective_bench.py [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from t2v_b200 import prims  # noqa: E402
from t2v_b200 import step as S  # noqa: E402
from t2v_b200.optim import FusedAdamW  # noqa: E402

SHAPES = {"cfg2": (1, 4, 16, 32, 32), "lora": (1, 4, 16, 40, 72), "zeroscope": (1, 4, 24, 40, 72)}
STEP_LEGS = {"default": {}, "snr_gamma_5": dict(snr_gamma=5.0), "huber": dict(loss_type="huber")}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def variants():
    """(name, prediction type, fwd(pred, x0, noise, abar, t), bwd(..., gout)) for every kernel variant."""
    out = [("mse", "epsilon", lambda p, x, n, a, t: prims.mse_loss_fwd(p, n), lambda p, x, n, a, t, g: prims.mse_loss_bwd(p, n, g)),
           ("velocity_mse", "v_prediction", prims.velocity_mse_loss_fwd, prims.velocity_mse_loss_bwd)]
    for ptype in ("epsilon", "v_prediction"):
        for form in ("l2", "huber", "smooth_l1"):
            for gamma in (None, 5.0):
                if form == "l2" and gamma is None:
                    continue               # the default objective: the two kernels above
                o = S.loss_objective(gamma, form, "snr", 0.1)
                v = ptype == "v_prediction"
                out.append((f"{form}{'+gamma5' if gamma else ''}/{'v' if v else 'eps'}", ptype,
                            lambda p, x, n, a, t, o=o, v=v: prims.diffusion_loss_fwd(p, x if v else None, n, a, t, o),
                            lambda p, x, n, a, t, g, o=o, v=v: prims.diffusion_loss_bwd(p, x if v else None, n, a, t, o, g)))
    return out


def graphed_ms(fn, n, per_graph=50):
    """ms per launch of fn: `per_graph` launches captured in one CUDA graph, replayed until n launches have run, timed with
    CUDA events, so the host-side call (ctypes, allocation) does not enter the kernel time."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(per_graph):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    reps = max(1, n // per_graph)
    return bench.time_events(g.replay, reps) / per_graph


def kernel_table(abar, n):
    rows = []
    for shape_name, (B, C, F, H, W) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        x0 = torch.randn(B, C, F, H, W, device="cuda", generator=g)
        noise = torch.randn(B, C, F, H, W, device="cuda", generator=g)
        pred = torch.randn(B * F, H, W, 8, device="cuda", generator=g).to(torch.bfloat16)
        t = torch.randint(0, abar.numel(), (B,), device="cuda", generator=g)
        gout = torch.ones((), device="cuda")
        px = B * F * H * W
        for name, ptype, fwd, bwd in variants():
            reads = px * 16 + B * C * F * H * W * 4 * (2 if ptype == "v_prediction" else 1)
            f_args, b_args = (pred, x0, noise, abar, t), (pred, x0, noise, abar, t, gout)
            f_ms = graphed_ms(lambda: fwd(*f_args), n)
            b_ms = graphed_ms(lambda: bwd(*b_args), n)
            rows.append(dict(shape=shape_name, variant=name, fwd_us=round(1000 * f_ms, 2), bwd_us=round(1000 * b_ms, 2),
                             fwd_bytes=reads, bwd_bytes=reads + px * 16, fwd_GBps=round(reads / f_ms / 1e6, 1),
                             bwd_GBps=round((reads + px * 16) / b_ms / 1e6, 1)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-launches", type=int, default=2000)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    report = {"gpu": gpu_info(), "timing": "CUDA events; step legs alternated in one process; each number one timed batch"}
    abar = S.ddpm_alphas_cumprod(device=dev)
    report["kernels"] = kernel_table(abar, args.kernel_launches)
    if not args.skip_step:
        unet = bench.build_unet(dev)
        step = S.DataParallelStep(unet, abar, passes=1, use_graph=True)
        opt = FusedAdamW(step.arena, [dict(params=[p for p in unet.parameters() if p.requires_grad])], lr=5e-6, betas=(0.9, 0.999),
                         eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
        step.attach_optimizer(opt)
        devin = [x.to(dev) for x in bench.synthetic_inputs(1, bench.CFG2, 1234)]
        step_ms = {k: [] for k in STEP_LEGS}
        for _ in range(args.reps):
            for k, opts in STEP_LEGS.items():
                step.objective = S.loss_objective(**opts)
                step._graph = None          # the captured graph holds one loss kernel: capture again for this objective
                for _ in range(args.warmup):
                    step(*devin)
                torch.cuda.synchronize()
                step_ms[k].append(round(bench.time_events(lambda: step(*devin), args.steps), 3))
        report["cfg2_step_ms"] = step_ms
        report["cfg2_step"] = (f"cfg-2 step (one fwd+bwd pass + FusedAdamW, CUDA-graph replay), {args.steps} steps after "
                               f"{args.warmup} warm-up, {args.reps} alternations")
    line = json.dumps(report)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
