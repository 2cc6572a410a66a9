#!/usr/bin/env python
"""Text-encoder training (`train_text_encoder`, `trainable_text_modules: ['all']`) on an H100.
Step: the cfg-3 LoRA workload (ms-1.7b UNet, r 16 on UNet3DConditionModel, 16 frames 320x576, gradient checkpointing) and the
cfg-2 full finetune (every UNet parameter, 16 frames 256x256) of bench.py, in the reference's two-pass video step with
FusedAdamW, replayed as a CUDA graph: the text states given (text encoder off) against the seeded ViT-H text tower trained in
the step (pass 1 is frame 1 only), every text parameter in the arena and the optimizer.  ms/step and peak memory, alternated in
one process; a configuration that does not fit the card is reported as such.
embed_tokens_bwd: t2v_embed_tokens_bwd launches at B x 77 rows x 1024 channels, vocab 49,408, on tokenizer-like prompts (a
start id, a few words, the pad id repeated to 77), captured in a CUDA graph and timed with CUDA events.
The card's name and power limit are read in the same run.  Usage: python tools/text_train_bench.py [--out FILE]"""
import argparse
import contextlib
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402
from t2v_b200 import prims  # noqa: E402
from t2v_b200 import step as S  # noqa: E402
from t2v_b200.optim import FusedAdamW  # noqa: E402
from text_lora_bench import gpu_info  # noqa: E402

VOCAB = 49408


def prompts(B, dev, seed=7):
    """B padded prompts: start id, 4 to 12 word ids, end id, then the pad id to 77 (CLIP's tokenizer pads with the end id)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((B, 77), VOCAB - 1, dtype=torch.int64)
    for b in range(B):
        n = int(torch.randint(4, 13, (1,), generator=g))
        ids[b, 0] = VOCAB - 2
        ids[b, 1:1 + n] = torch.randint(0, VOCAB - 2, (n,), generator=g)
    return ids.to(dev)


def step_row(workload, with_text, steps, warmup, dev):
    wl = bench.WORKLOADS[workload]
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    row = {"workload": workload, "train_text_encoder": with_text}
    unet = te = step = opt = None
    try:
        unet = bench.build_unet(dev)
        if wl["lora_rank"]:
            from t2v_b200.utils.lora_handler import LoraHandler
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
        unet._set_gradient_checkpointing(bool(wl["grad_ckpt"]))
        if with_text:
            from t2v_b200.text_encoder import CLIPTextModel
            torch.manual_seed(2024)
            te = CLIPTextModel().requires_grad_(True).to(dev).train()   # the ViT-H text tower, seeded weights, all trainable
        abar = S.ddpm_alphas_cumprod(device=dev)
        step = S.DataParallelStep(unet, abar, passes=2, use_graph=True, text_encoder=te)
        trainable = [p for p in step.arena.params if p.requires_grad]
        opt = FusedAdamW(step.arena, [dict(params=trainable)], lr=5e-6, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
                         max_grad_norm=1.0)
        step.attach_optimizer(opt)
        lat, noise, t, text = [x.to(dev) for x in bench.synthetic_inputs(1, wl, 1234)]
        if with_text:
            text = prompts(1, dev)
        devin = (lat, noise, t, text)
        for _ in range(warmup):
            step(*devin)
        torch.cuda.synchronize()
        ms = bench.time_events(lambda: step(*devin), steps)
        row.update(ms_per_step=round(ms, 2), trainable=sum(p.numel() for p in trainable),
                   text_trainable=sum(p.numel() for p in te.parameters()) if te is not None else 0,
                   loss=float(step(*devin).item()))
    except torch.cuda.OutOfMemoryError as e:
        row.update(ms_per_step=None, out_of_memory=str(e).splitlines()[0])
    row["peak_GB"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    del unet, te, step, opt
    gc.collect()
    torch.cuda.empty_cache()
    return row


def embed_rows(dev):
    rows = []
    for B in (1, 8, 32):
        ids = prompts(B, dev, seed=B)
        dy = torch.randn(B * 77, 1024, device=dev).to(torch.bfloat16)
        dtok = torch.zeros(VOCAB, 1024, device=dev)
        dpos = torch.zeros(77, 1024, device=dev)
        launches = 100
        prims.embed_tokens_bwd(ids, dy, dtok, dpos, VOCAB)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(launches):
                prims.embed_tokens_bwd(ids, dy, dtok, dpos, VOCAB)
        graph.replay()
        us = 1000 * bench.time_events(graph.replay, 10) / launches
        distinct = int(torch.unique(ids).numel())
        nbytes = dy.numel() * 2 + 2 * 4 * 1024 * (distinct + 77)   # dy read once, each written row read and written
        rows.append({"rows": B * 77, "C": 1024, "distinct_ids": distinct, "us": round(us, 2), "GB/s": round(nbytes / (us * 1e-6) / 1e9, 1)})
        del graph
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workloads", default="lora,cfg2")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "embed_tokens_bwd": embed_rows(dev), "step": []}
    print(json.dumps(res["embed_tokens_bwd"]), file=sys.stderr, flush=True)
    for _ in range(a.rounds):
        for workload in a.workloads.split(","):
            for with_text in (False, True):
                res["step"].append(step_row(workload, with_text, a.steps, a.warmup, dev))
                print(json.dumps(res["step"][-1]), file=sys.stderr, flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
