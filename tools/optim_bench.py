#!/usr/bin/env python
"""Optimizer cost of blockwise 8-bit AdamW (optim.AdamW8bit) next to fp32 AdamW (optim.FusedAdamW), each with and without the
weight EMA (`ema_decay`, `use_ema`), on an H100.

cfg 2 (the ms-1.7b UNet as bench.py builds it, all 1.41 B parameters trainable, random gradient):
  * launch() time of each optimizer (global-norm clip + update), CUDA events, the two alternated and each timed twice;
  * algorithmic bytes per trainable parameter and the achieved TB/s against the 3.35 TB/s data-sheet HBM3 bandwidth;
  * optimizer-state bytes, from torch.cuda.memory_allocated before and after constructing the optimizer, and the EMA's share;
  * the cfg-2 step (CUDA-graph replay, --steps timed after --warmup) with each optimizer attached, alternated, each twice.
LoRA workload (bench.py --workload lora): the state and launch() lines, and how much of the state saving comes from covering
only the trainable tensors (a compact fp32 state, computed) and how much from 8 bits.
The card's name and power limit are read in the same run.  Usage: python tools/optim_bench.py [--out FILE]"""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from t2v_b200 import step as S  # noqa: E402
from t2v_b200.optim import AdamW8bit, FusedAdamW  # noqa: E402
from t2v_b200.runtime import ParamArena, _align  # noqa: E402

HBM_TBS = 3.35   # H100 SXM data sheet
EMA_DECAY = 0.9999
OPTIMIZERS = (("fused_adamw", FusedAdamW, None), ("fused_adamw_ema", FusedAdamW, EMA_DECAY), ("adamw8bit", AdamW8bit, None),
              ("adamw8bit_ema", AdamW8bit, EMA_DECAY))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def make(cls, arena, params, ema_decay):
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    opt = cls(arena, [dict(params=params)], lr=5e-6, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0, ema_decay=ema_decay)
    torch.cuda.synchronize()
    return opt, torch.cuda.memory_allocated() - before


def algorithmic_bytes(opt):
    """Bytes one launch() moves: 4 (gradient read of the norm) + 34 per fp32-state element; 4 + 22 per 8-bit element plus
    16 per 256-element block (absmax of m and v, read and written); 8 more per element with an EMA (its read and write)."""
    total = 0
    for s in opt._sets:
        for row in s["chunks"].tolist():
            n = row[1]
            total += 26 * n + 16 * ((n + 255) // 256) if len(row) == 4 and row[3] == 8 else 38 * n
    return total + (8 * opt.ema.numel() if opt.ema is not None else 0)


def time_launch(opt, arena, n):
    """launch() as the step runs it (it zeroes the gradient it consumed), after a random gradient and two warm-up launches."""
    arena.grad.normal_()
    opt.push_hyperparams()
    for _ in range(2):
        opt.launch()
    torch.cuda.synchronize()
    return bench.time_events(opt.launch, n)


def optimizer_leg(arena, params, reps, n):
    opts, out = {}, {}
    for name, cls, ema_decay in OPTIMIZERS:
        opts[name], mem = make(cls, arena, params, ema_decay)
        out[name] = {"state_bytes_allocated": mem, "trainable_elements": opts[name].trainable_elements,
                     "algorithmic_bytes": algorithmic_bytes(opts[name]), "launch_ms": [],
                     "ema_bytes": 4 * opts[name].ema.numel() if ema_decay is not None else 0}
        out[name]["bytes_per_param"] = out[name]["algorithmic_bytes"] / out[name]["trainable_elements"]
    for _ in range(reps):
        for name, _, _ in OPTIMIZERS:
            out[name]["launch_ms"].append(time_launch(opts[name], arena, n))
    for name, _, _ in OPTIMIZERS:
        best = min(out[name]["launch_ms"])
        out[name]["achieved_tbs"] = out[name]["algorithmic_bytes"] / (best / 1e3) / 1e12
        out[name]["frac_of_hbm_peak"] = out[name]["achieved_tbs"] / HBM_TBS
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=10, help="launch() calls per timed batch")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    report = {"gpu": gpu_info(), "hbm_peak_tbs": HBM_TBS, "timing": "CUDA events; optimizers alternated; each number one timed batch"}

    # ---- cfg 2: every parameter trainable
    unet = bench.build_unet(dev)
    step = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device=dev), passes=1, use_graph=True)
    trainable = [p for p in unet.parameters() if p.requires_grad]
    report["cfg2"] = optimizer_leg(step.arena, trainable, args.reps, args.launches)
    gc.collect()
    torch.cuda.empty_cache()
    devin = [x.to(dev) for x in bench.synthetic_inputs(1, bench.CFG2, 1234)]
    step_ms = {name: [] for name, _, _ in OPTIMIZERS}
    for _ in range(args.reps):
        for name, cls, ema_decay in OPTIMIZERS:
            opt, _ = make(cls, step.arena, trainable, ema_decay)
            step.attach_optimizer(opt)
            for _ in range(args.warmup):
                step(*devin)
            torch.cuda.synchronize()
            step_ms[name].append(bench.time_events(lambda: step(*devin), args.steps))
            step.attach_optimizer(None)
            del opt
            gc.collect()
            torch.cuda.empty_cache()
    for name, _, _ in OPTIMIZERS:
        report["cfg2"][name]["step_ms"] = step_ms[name]
    report["cfg2"]["step"] = f"cfg-2 step (one fwd+bwd pass + optimizer, CUDA-graph replay), {args.steps} steps after {args.warmup} warm-up"
    del step, unet, trainable, devin
    gc.collect()
    torch.cuda.empty_cache()

    # ---- LoRA: the base weights frozen, 29 M LoRA parameters trainable
    from t2v_b200.utils.lora_handler import LoraHandler
    unet = bench.build_unet(dev)
    unet.requires_grad_(False)
    handler = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    torch.manual_seed(4321)
    handler.add_lora_to_model(True, unet, handler.unet_replace_modules, 0.1, "", r=bench.WORKLOADS["lora"]["lora_rank"])
    unet = unet.to(dev)
    arena = ParamArena(unet)
    trainable = [p for p in unet.parameters() if p.requires_grad]
    lora = optimizer_leg(arena, trainable, args.reps, args.launches)
    fused, q8 = lora["fused_adamw"]["state_bytes_allocated"], lora["adamw8bit"]["state_bytes_allocated"]
    compact32 = 8 * sum(_align(p.numel()) for p in trainable)
    lora["saving"] = {"fused_minus_8bit_bytes": fused - q8, "compact_fp32_state_bytes (computed)": compact32,
                      "share_from_compact_state": (fused - compact32) / (fused - q8),
                      "share_from_8_bits": (compact32 - q8) / (fused - q8)}
    report["lora"] = lora

    text = json.dumps(report, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
