#!/usr/bin/env python
"""Text-encoder LoRA (`use_text_lora`) on an H100.
Step: the cfg-3 LoRA workload of bench.py (ms-1.7b UNet, r 16 on UNet3DConditionModel, 16 frames 320x576, gradient
checkpointing, seeded weights) in the reference's two-pass video step with FusedAdamW, replayed as a CUDA graph: UNet LoRA only
(two full-clip passes) against UNet + text LoRA (r 16 on CLIPEncoderLayer of the seeded ViT-H text tower; the text encoder runs
in the step, pass 1 is frame 1 only).  ms/step and peak memory, alternated in one process.
Text tower: one eager forward + backward of the injected encoder on one prompt (CUDA events, after warm-up) and its native
launch count.
gelu_bwd: t2v_gelu_bwd_bf16 launches captured in a CUDA graph (so no host work is timed), the replay timed with CUDA events;
bytes = x + dy read, dx written (6 B/element).
The card's name and power limit are read in the same run.  Usage: python tools/text_lora_bench.py [--out FILE]"""
import argparse
import contextlib
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from t2v_b200 import native, prims  # noqa: E402
from t2v_b200 import step as S  # noqa: E402
from t2v_b200.optim import FusedAdamW  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def text_encoder(dev, r):
    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils.lora import inject_trainable_lora_extended
    torch.manual_seed(2024)
    te = CLIPTextModel()   # the ViT-H text tower of ms-1.7b, seeded weights
    with contextlib.redirect_stdout(sys.stderr):
        inject_trainable_lora_extended(te, {"CLIPEncoderLayer"}, r=r)
    te = te.to(dev).train()
    with torch.no_grad():
        for n, p in te.named_parameters():
            if "lora_up" in n:
                p.normal_(0.0, 0.01)
    return te


def step_row(with_text, steps, warmup, dev):
    wl = bench.WORKLOADS["lora"]
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    from t2v_b200.utils.lora_handler import LoraHandler
    unet = bench.build_unet(dev)
    unet.requires_grad_(False)
    handler = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    torch.manual_seed(4321)
    with contextlib.redirect_stdout(sys.stderr):
        handler.add_lora_to_model(True, unet, handler.unet_replace_modules, 0.1, "", r=wl["lora_rank"])
    unet = unet.to(dev).train()
    with torch.no_grad():
        for n, p in unet.named_parameters():
            if "lora_up" in n:
                p.normal_(0.0, 0.01)
    unet._set_gradient_checkpointing(True)
    te = text_encoder(dev, wl["lora_rank"]) if with_text else None
    abar = S.ddpm_alphas_cumprod(device=dev)
    step = S.DataParallelStep(unet, abar, passes=2, use_graph=True, text_encoder=te)
    trainable = [p for p in step.arena.params if p.requires_grad]
    opt = FusedAdamW(step.arena, [dict(params=trainable)], lr=5e-6, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
    step.attach_optimizer(opt)
    lat, noise, t, text = [x.to(dev) for x in bench.synthetic_inputs(1, wl, 1234)]
    if with_text:
        text = torch.randint(0, 49408, (1, 77), device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    devin = (lat, noise, t, text)
    for _ in range(warmup):
        step(*devin)
    torch.cuda.synchronize()
    ms = bench.time_events(lambda: step(*devin), steps)
    row = {"text_lora": with_text, "ms_per_step": round(ms, 2), "peak_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2),
           "trainable": sum(p.numel() for p in trainable), "loss": float(step(*devin).item())}
    del step, opt, unet, te
    return row


def text_row(dev, r, reps):
    te = text_encoder(dev, r)
    ids = torch.randint(0, 49408, (1, 77), device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    g = torch.randn(77, 1024, device=dev).to(torch.bfloat16)

    def fwd_bwd():
        te.encode(ids).backward(g)
    for _ in range(3):
        fwd_bwd()
    torch.cuda.synchronize()
    n0 = native.launch_count()
    fwd_bwd()
    torch.cuda.synchronize()
    launches = native.launch_count() - n0
    ms = bench.time_events(fwd_bwd, reps)
    base_bytes = sum(2 * p.numel() for n, p in te.named_parameters() if p.dim() == 2 and "lora" not in n and "embedding" not in n)
    return {"text_fwd_bwd_ms": round(ms, 3), "native_launches": launches, "bf16_projection_weights_GB": round(base_bytes / 1e9, 3)}


def gelu_rows(dev):
    rows = []
    for n, launches in ((77 * 4096, 200), (1 << 26, 20)):
        x = torch.randn(n, device=dev).to(torch.bfloat16)
        dy = torch.randn(n, device=dev).to(torch.bfloat16)
        for quick in (False, True):
            prims.gelu_bwd(x, dy, quick)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(launches):
                    prims.gelu_bwd(x, dy, quick)
            graph.replay()
            ms = bench.time_events(graph.replay, 10) / launches
            rows.append({"n": n, "quick": quick, "us": round(1000 * ms, 2), "GB/s": round(6 * n / (ms * 1e-3) / 1e9, 1)})
            del graph
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "gelu_bwd": gelu_rows(dev), "text_tower": text_row(dev, 16, 20), "step": []}
    for _ in range(a.rounds):
        for with_text in (False, True):
            res["step"].append(step_row(with_text, a.steps, a.warmup, dev))
            print(json.dumps(res["step"][-1]), file=sys.stderr, flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
