#!/usr/bin/env python
"""Cost of `save_training_state` on an H100: bytes written and wall time to save and to load the resumable training state
(training_state.save / training_state.load, each ending in a device synchronise) for

  * cfg 2: the ms-1.7b UNet as bench.py builds it, all 1.41 B parameters trainable, fused AdamW with the EMA
    (fp32 master 5.6 GB, AdamW moments 11.3 GB, EMA 5.6 GB);
  * LoRA (bench.py --workload lora): the same UNet frozen, 29 M cloneofsimo rank-16 LoRA parameters, fused AdamW with the EMA.

Two CUDA-graph steps run first, so the state holds real moments and a recorded capture.  The state goes to a temporary
folder (--dir to choose where), which is removed afterwards.  The card's name and power limit are read in the same run.
Usage: python tools/resume_bench.py [--dir DIR] [--out FILE]"""
import argparse
import gc
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from t2v_b200 import step as S  # noqa: E402
from t2v_b200 import training_state as TS  # noqa: E402
from t2v_b200.optim import FusedAdamW  # noqa: E402
from t2v_b200.utils.dataset import EpochOrder  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def folder_bytes(path):
    return {n: os.path.getsize(os.path.join(path, n)) for n in sorted(os.listdir(path))}


def leg(unet, wl, dev, where):
    step = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device=dev), passes=1, use_graph=True)
    trainable = [p for p in unet.parameters() if p.requires_grad]
    opt = FusedAdamW(step.arena, [dict(params=trainable)], lr=5e-6, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
                     max_grad_norm=1.0, ema_decay=0.9999)
    step.attach_optimizer(opt)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 1.0)
    order = EpochOrder(torch.utils.data.RandomSampler(range(16)))
    devin = [x.to(dev) for x in bench.synthetic_inputs(1, wl, 1234)]
    for _ in range(2):
        step(*devin)
        opt._opt_called = True
        sched.step()
    torch.cuda.synchronize()
    n = sum(p.numel() for p in trainable)
    man = TS.manifest(1, "cloneofsimo", opt, True, step, 2, 1)
    path = tempfile.mkdtemp(prefix="resume_bench_", dir=where)
    try:
        t = time.perf_counter()
        TS.save(path, rank=0, world=1, man=man, stepper=step, optimizer=opt, sched=sched, order=order, loader=None)
        torch.cuda.synchronize()
        save_s = time.perf_counter() - t
        files = folder_bytes(os.path.join(path, TS.STATE_DIR))
        before = opt.ema.clone()
        opt.ema.zero_()
        t = time.perf_counter()
        TS.load(os.path.join(path, TS.STATE_DIR), rank=0, stepper=step, optimizer=opt, sched=sched, order=order, loader=None)
        torch.cuda.synchronize()
        load_s = time.perf_counter() - t
        assert torch.equal(before, opt.ema), "the EMA did not round-trip"
    finally:
        shutil.rmtree(path, ignore_errors=True)
    out = {"trainable_parameters": n, "bytes_written": sum(files.values()), "files": files, "save_s": save_s, "load_s": load_s,
           "computed_bytes": {"fp32_master": 4 * n, "adamw_moments": 8 * n, "ema": 4 * opt.ema.numel()}}
    step.attach_optimizer(None)
    del step, opt, sched, devin
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None, help="where the temporary state folder goes (default: the system temp dir)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    report = {"gpu": gpu_info(), "timing": "host wall clock around training_state.save / load, each ending in a device synchronise",
              "target": os.path.abspath(args.dir or tempfile.gettempdir())}
    report["cfg2"] = leg(bench.build_unet(dev), bench.CFG2, dev, args.dir)
    gc.collect()
    torch.cuda.empty_cache()
    from t2v_b200.utils.lora_handler import LoraHandler
    wl = bench.WORKLOADS["lora"]
    unet = bench.build_unet(dev)
    unet.requires_grad_(False)
    handler = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    torch.manual_seed(4321)
    handler.add_lora_to_model(True, unet, handler.unet_replace_modules, 0.1, "", r=wl["lora_rank"])
    unet = unet.to(dev).train()
    unet._set_gradient_checkpointing(True)
    report["lora"] = leg(unet, wl, dev, args.dir)
    line = json.dumps(report)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
