#!/usr/bin/env python
"""Step time of v-prediction next to epsilon prediction on an H100.

cfg 2 (the ms-1.7b UNet as bench.py builds it, latents 1x4x16x32x32, one fwd+bwd pass + fused AdamW, CUDA-graph replay):
the same step object runs with prediction_type 'epsilon' and 'v_prediction', alternated --reps times in one process, each
leg re-captured and timed over --steps replays after --warmup.  The velocity loss reads one more fp32 latent tensor (x0,
256 KB at cfg 2) than the noise loss; the loss kernels alone (forward + backward launch pair) are timed the same way.
The card's name and power limit are read in the same run.  Usage: python tools/prediction_type_bench.py [--out FILE]"""
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

TYPES = ("epsilon", "v_prediction")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def loss_kernels(devin, abar, n):
    """ms per forward + backward pair of each loss kernel at the cfg-2 latent shape."""
    lat, noise, t, _ = devin
    B, C, F, H, W = lat.shape
    pred = torch.randn(B * F, H, W, 8, device=lat.device).to(torch.bfloat16)
    gout = torch.ones((), device=lat.device)
    legs = {"epsilon": lambda: (prims.mse_loss_fwd(pred, noise), prims.mse_loss_bwd(pred, noise, gout)),
            "v_prediction": lambda: (prims.velocity_mse_loss_fwd(pred, lat, noise, abar, t),
                                     prims.velocity_mse_loss_bwd(pred, lat, noise, abar, t, gout))}
    out = {k: [] for k in TYPES}
    for _ in range(3):
        for k in TYPES:
            for _ in range(10):
                legs[k]()
            out[k].append(bench.time_events(legs[k], n))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    report = {"gpu": gpu_info(), "timing": "CUDA events; prediction types alternated in one process; each number one timed batch"}

    abar = S.ddpm_alphas_cumprod(device=dev)
    unet = bench.build_unet(dev)
    step = S.DataParallelStep(unet, abar, passes=1, use_graph=True)
    opt = FusedAdamW(step.arena, [dict(params=[p for p in unet.parameters() if p.requires_grad])], lr=5e-6, betas=(0.9, 0.999),
                     eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
    step.attach_optimizer(opt)
    devin = [x.to(dev) for x in bench.synthetic_inputs(1, bench.CFG2, 1234)]
    step_ms = {k: [] for k in TYPES}
    loss = {k: [] for k in TYPES}
    for _ in range(args.reps):
        for k in TYPES:
            step.prediction_type = k
            step._graph = None          # the captured graph holds one loss kernel: capture again for this objective
            for _ in range(args.warmup):
                step(*devin)
            torch.cuda.synchronize()
            step_ms[k].append(bench.time_events(lambda: step(*devin), args.steps))
            loss[k].append(float(step(*devin).item()))
    report["cfg2_step_ms"] = step_ms
    report["cfg2_last_loss"] = loss
    report["cfg2_step"] = (f"cfg-2 step (one fwd+bwd pass + FusedAdamW, CUDA-graph replay), {args.steps} steps after "
                           f"{args.warmup} warm-up, {args.reps} alternations")
    report["loss_kernels_fwd_bwd_us"] = {k: [round(1000 * v, 2) for v in vs]
                                         for k, vs in loss_kernels(devin, abar, args.kernel_launches).items()}
    line = json.dumps(report)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
