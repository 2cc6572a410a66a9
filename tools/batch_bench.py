#!/usr/bin/env python
"""train_batch_size > 1 on an H100: the ragged resize kernel and the LoRA step at B = 1, 2, 4.

Ragged kernel: batches of 2, 4, 6 and 8 clips of 16 frames, 480p (480x854) and 1080p (1080x1920) sources alternating, resized
to 256x256 and to 320x576 by ONE `frames_u8_to_nhwc8_ragged` launch, timed with CUDA events over --launches launches after
warm-up; next to it, the same batch as one `frames_u8_to_nhwc8` launch per clip.  Algorithmic bytes, from the shapes: the
bf16 [sum F, h, w, 8] output written once (16 B per pixel) plus every source pixel a bilinear tap touches read once (3 B;
rows in the union of y0 / y1 times columns in the union of x0 / x1, per frame) - a downscale touches a fraction of the source.

Step: the ms-1.7b UNet with cloneofsimo LoRA r16 on UNet3DConditionModel, latents Bx4x16x32x32 (16 frames at 256x256), text
Bx77x1024, the two-pass video step of train.main (passes=2) + FusedAdamW as one CUDA-graph replay, at B in {1, 2, 4}:
ms/step, frames/s (B * 16 frames per step) and peak allocated memory, for the --configs list (batch size, and a `c` suffix
for gradient checkpointing).  The card's name, power limit and SM clocks are read in the same run.
Usage: python tools/batch_bench.py [--out FILE]"""
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
SOURCES = {"480p": (480, 854), "1080p": (1080, 1920)}
TARGETS = ((256, 256), (320, 576))
FRAMES = 16


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def taps(n_in, n_out):
    """Source indices the half-pixel bilinear resize reads along one axis (same arithmetic as the kernel, in fp32)."""
    s = torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32)
    f = ((torch.arange(n_out, dtype=torch.float32) + 0.5) * s - 0.5).clamp_min(0.0)
    i0 = f.to(torch.int64).clamp_max(n_in - 1)
    return len(set(i0.tolist()) | set((i0 + 1).clamp_max(n_in - 1).tolist()))


def kernel_row(n_clips, hw, launches):
    names = [("480p", "1080p")[k % 2] for k in range(n_clips)]
    g = torch.Generator(device="cuda").manual_seed(n_clips)
    clips = [torch.randint(0, 256, (FRAMES,) + SOURCES[n] + (3,), device="cuda", generator=g, dtype=torch.uint8) for n in names]
    packed = torch.cat([c.reshape(-1) for c in clips])
    offs, off = [], 0
    for c in clips:
        offs.append(off)
        off += c.numel()
    table = torch.tensor([[o, FRAMES, c.shape[1], c.shape[2]] for o, c in zip(offs, clips)], dtype=torch.int64)
    out_bytes = n_clips * FRAMES * hw[0] * hw[1] * 16
    in_bytes = sum(FRAMES * taps(SOURCES[n][0], hw[0]) * taps(SOURCES[n][1], hw[1]) * 3 for n in names)
    dev_table = table.cuda()
    # the kernel alone: the wrapper's host-side table check and H2D are outside the timed launches
    out = torch.empty((n_clips * FRAMES, hw[0], hw[1], 8), device="cuda", dtype=torch.bfloat16)
    lib, stream = prims.native.lib(), prims._stream()

    def ragged():
        prims.native.check(lib.t2v_frames_u8_to_nhwc8_ragged(prims._p(packed), prims._p(dev_table), n_clips, n_clips * FRAMES,
                                                             prims._p(out), hw[0], hw[1], stream))

    def per_clip():
        for c in clips:
            prims.frames_u8_to_nhwc8(c, hw)
    assert torch.equal(prims.frames_u8_to_nhwc8_ragged(packed, table, hw), torch.cat([prims.frames_u8_to_nhwc8(c, hw) for c in clips]))
    row = {"clips": "+".join(names), "out_hw": list(hw)}
    for name, fn in (("ragged_one_launch", ragged), ("one_launch_per_clip", per_clip)):
        for _ in range(10):
            fn()
        ms = bench.time_events(fn, launches)
        gbs = (in_bytes + out_bytes) / (ms * 1e-3) / 1e9
        row[name] = {"us": round(1000 * ms, 1), "GB/s": round(gbs, 1), "of_3.35TB/s": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)}
    row["MB_read"], row["MB_written"] = round(in_bytes / 1e6, 2), round(out_bytes / 1e6, 2)
    return row


def step_row(B, ckpt, steps, warmup, dev):
    from t2v_b200.utils.lora_handler import LoraHandler
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    unet = bench.build_unet(dev)
    unet.requires_grad_(False)
    handler = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    torch.manual_seed(4321)
    handler.add_lora_to_model(True, unet, handler.unet_replace_modules, 0.1, "", r=16)
    unet = unet.to(dev).train()
    unet._set_gradient_checkpointing(ckpt)
    step = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device=dev), passes=2, use_graph=True)
    opt = FusedAdamW(step.arena, [dict(params=[p for p in unet.parameters() if p.requires_grad])], lr=5e-6,
                     betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
    step.attach_optimizer(opt)
    devin = [x.to(dev) for x in bench.synthetic_inputs(B, bench.CFG2, 1234)]
    for _ in range(warmup):
        step(*devin)
    torch.cuda.synchronize()
    with bench.ClockSampler(0) as clocks:
        ms = bench.time_events(lambda: step(*devin), steps)
    loss = float(step(*devin).item())
    row = {"B": B, "grad_ckpt": ckpt, "ms_per_step": round(ms, 2), "frames_per_s": round(B * FRAMES / (ms / 1e3), 1),
           "peak_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2), "loss": loss, "clocks": clocks.summary()}
    del unet, step, opt, devin
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    # B=4 without checkpointing does not fit 80 GB next to the graph's memory pool
    ap.add_argument("--configs", default="1,2,1c,2c,4c", help="batch sizes; suffix c = gradient checkpointing")
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    report = {"gpu": gpu_info(), "timing": "CUDA events over --launches launches / --steps steps after warm-up"}
    rows = []
    for hw in TARGETS:
        for n in (2, 4, 6, 8):
            rows.append(kernel_row(n, hw, args.launches))
            print(json.dumps(rows[-1]), flush=True)
    report["ragged_resize"] = rows
    if not args.no_step:
        report["lora_r16_step_16f_256"] = []
        for c in args.configs.split(","):
            report["lora_r16_step_16f_256"].append(step_row(int(c.rstrip("c")), c.endswith("c"), args.steps, args.warmup, dev))
            print(json.dumps(report["lora_r16_step_16f_256"][-1]), flush=True)
    line = json.dumps(report)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
