#!/usr/bin/env python
"""Temporal attention past 32 frames on an H100: kernel table and training step.

Kernel table: the temporal-attention geometries of an ms-1.7b step at 256^2 (latents 32x32; the four UNet levels with their
width C = 64 * heads, and transformer_in: 8 heads of 64 over 320 channels at 32x32), fused QKV input [rows, 3C], for
L in {16, 24, 32, 48, 64, 128, 256}.  Forward and backward are each timed with CUDA events over --launches back-to-back
launches after warm-up.  Bytes are algorithmic, computed from the shapes (each operand read once, each result written once):
  attn_long  fwd q, k, v -> o, lse          bwd q, k, v, o, dO, lse -> dq, dk, dv
  attn_small fwd q, k, v -> o               bwd q, k, v, dO -> dq, dk, dv
At L <= 32 both kernels are timed on the same operands.

Step: the cfg-2 model (ms-1.7b UNet, latents 1x4xFx32x32) with gradient checkpointing, one fwd+bwd pass + FusedAdamW as a
CUDA-graph replay, at F in {32, 48, 64}: full finetune, or LoRA r16 when the full finetune runs out of memory (reported).
The card's name and power limit are read in the same run.  Usage: python tools/long_clip_bench.py [--out FILE]"""
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
from t2v_b200 import prims  # noqa: E402
from t2v_b200 import step as S  # noqa: E402
from t2v_b200.optim import FusedAdamW  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
GEOMS = {"level0 HW=1024 C=320": (1024, 5), "level1 HW=256 C=640": (256, 10), "level2 HW=64 C=1280": (64, 20),
         "level3 HW=16 C=1280": (16, 20), "transformer_in HW=1024 C=512": (1024, 8)}
LENGTHS = (16, 24, 32, 48, 64, 128, 256)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def kernel_row(HW, heads, L, launches, D=64):
    C, rows, nseq = heads * D, L * HW, HW
    g = torch.Generator(device="cuda").manual_seed(L)
    qkv = torch.randn(rows, 3 * C, device="cuda", generator=g).to(torch.bfloat16)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    do = torch.randn(rows, C, device="cuda", generator=g).to(torch.bfloat16)
    o = torch.empty_like(do)
    lse = torch.empty(nseq, heads, L, device="cuda")
    dqkv = torch.empty_like(qkv)
    dq, dk, dv = dqkv[:, :C], dqkv[:, C:2 * C], dqkv[:, 2 * C:]
    addr = (nseq, HW, L * HW, 1, HW, 3 * C, C, heads, L, D)
    t = rows * C * 2
    lse_b = nseq * heads * L * 4
    legs = {"long_fwd": (lambda: prims.attn_long_fwd(q, k, v, o, lse, addr), 4 * t + lse_b),
            "long_bwd": (lambda: prims.attn_long_bwd(q, k, v, o, do, lse, dq, dk, dv, addr), 8 * t + lse_b)}
    if L <= 32:
        legs["small_fwd"] = (lambda: prims.attn_small_fwd(q, k, v, o, addr), 4 * t)
        legs["small_bwd"] = (lambda: prims.attn_small_bwd(q, k, v, do, dq, dk, dv, addr), 7 * t)
    prims.attn_long_fwd(q, k, v, o, lse, addr)
    row = {"L": L}
    for name, (fn, nbytes) in legs.items():
        for _ in range(20):
            fn()
        ms = bench.time_events(fn, launches)
        gbs = nbytes / (ms * 1e-3) / 1e9
        row[name] = {"us": round(1000 * ms, 2), "MB": round(nbytes / 1e6, 2), "GB/s": round(gbs, 1),
                     "of_3.35TB/s": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)}
    return row


def step_row(F, steps, warmup, dev):
    """ms/step, frames/s and peak memory of one configuration; full finetune first, LoRA r16 if that runs out of memory."""
    for mode in ("full", "lora_r16"):
        unet = step = opt = None
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        try:
            unet = bench.build_unet(dev)
            if mode == "lora_r16":
                from t2v_b200.utils.lora_handler import LoraHandler
                unet.requires_grad_(False)
                handler = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
                torch.manual_seed(4321)
                handler.add_lora_to_model(True, unet, handler.unet_replace_modules, 0.1, "", r=16)
                unet = unet.to(dev).train()
            unet._set_gradient_checkpointing(True)
            step = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device=dev), passes=1, use_graph=True)
            opt = FusedAdamW(step.arena, [dict(params=[p for p in unet.parameters() if p.requires_grad])], lr=5e-6,
                             betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
            step.attach_optimizer(opt)
            cfg = dict(bench.CFG2, frames=F)
            devin = [x.to(dev) for x in bench.synthetic_inputs(1, cfg, 1234)]
            for _ in range(warmup):
                step(*devin)
            torch.cuda.synchronize()
            ms = bench.time_events(lambda: step(*devin), steps)
            loss = float(step(*devin).item())
            return {"F": F, "mode": mode, "ms_per_step": round(ms, 2), "frames_per_s": round(F / (ms / 1e3), 1),
                    "peak_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2), "loss": loss}
        except torch.cuda.OutOfMemoryError as e:
            oom = str(e).splitlines()[0]
        finally:
            del unet, step, opt
            gc.collect()
            torch.cuda.empty_cache()
        print(json.dumps({"F": F, "mode": mode, "out_of_memory": oom}), flush=True)
    return {"F": F, "out_of_memory": "full and lora_r16"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", default="32,48,64")
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    report = {"gpu": gpu_info(), "timing": "CUDA events, one timed batch per entry after 20 warm-up launches / --warmup steps"}
    table = {}
    for name, (HW, heads) in GEOMS.items():
        table[name] = [kernel_row(HW, heads, L, args.launches) for L in LENGTHS]
        print(json.dumps({name: table[name]}), flush=True)
    report["kernels"] = table
    if not args.no_step:
        report["step_cfg2_256_ckpt"] = [step_row(int(f), args.steps, args.warmup, dev) for f in args.frames.split(",")]
    line = json.dumps(report)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
