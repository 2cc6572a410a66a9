#!/usr/bin/env python
"""Stable LoRA on an H100: kernel table and training step against cloneofsimo.

Kernel table: every distinct conv of the ms-1.7b UNet (Conv2d 3x3 / 1x1, Conv3d (3,1,1)) at rank 16, with how often it occurs.
t2v_lora_delta_merge and t2v_lora_delta_grad are timed with CUDA events over --launches back-to-back launches after warm-up.
Bytes and FLOPs are algorithmic, computed from the shapes:
  merge  reads the fp32 base, A and B, writes the bf16 W_eff;   FLOP = 2 * (Cout k) * (Cin k) * (r k)  (every element of B @ A)
  grad   reads the fp32 dW, A and B, read-modify-writes dA, dB; FLOP = 2 x the merge's (dB = dBA A^T and dA = B^T dBA)
`per_unet_pass_ms` sums count x time over the table: one merge of every wrapped conv, or one projection.

Step: the cfg-3 LoRA workload of bench.py (ms-1.7b UNet, r 16 on UNet3DConditionModel, 16 frames 320x576, gradient checkpointing,
one pass + FusedAdamW replayed as a CUDA graph), cloneofsimo and stable_lora alternated in one process: ms/step and peak
memory.  One extra eager step of each stable_lora round times, with CUDA events around the calls, the merges, the gradient
projections and the full-size conv weight-gradient GEMMs that only stable LoRA needs; their share is given against that eager
step's own time.  The card's name and power limit are read in the same run.  Usage: python tools/stable_lora_bench.py [--out FILE]"""
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
import torch.nn as nn  # noqa: E402

import bench  # noqa: E402
from t2v_b200 import ops, prims  # noqa: E402
from t2v_b200 import step as S  # noqa: E402
from t2v_b200.optim import FusedAdamW  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi name, power.limit, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}


def conv_shapes():
    """{(conv3d, k, Cin, Cout): count} over the ms-1.7b UNet (built on the meta device)."""
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    with torch.device("meta"):
        m = UNet3DConditionModel()
    out = {}
    for mod in m.modules():
        if type(mod) in (nn.Conv2d, nn.Conv3d):
            key = (type(mod) is nn.Conv3d, mod.kernel_size[0], mod.in_channels, mod.out_channels)
            out[key] = out.get(key, 0) + 1
    return out


def kernel_row(conv3d, k, cin, cout, count, r, launches):
    g = torch.Generator(device="cuda").manual_seed(cin * 7 + cout)
    kh, kw = (3, 1) if conv3d else (k, k)
    base = torch.randn(cout, kh, kw, cin, device="cuda", generator=g)
    A = torch.randn(r * k, cin * k, device="cuda", generator=g)
    B = torch.randn(cout * k, r * k, device="cuda", generator=g)
    dw = torch.randn_like(base)
    dA, dB = torch.zeros_like(A), torch.zeros_like(B)
    flop = 2.0 * (cout * k) * (cin * k) * (r * k)
    ab = 4 * (A.numel() + B.numel())
    legs = {"merge": (lambda: prims.lora_delta_merge(base, A, B, 1.0, conv3d), 6 * base.numel() + ab, flop),
            "grad": (lambda: prims.lora_delta_grad(dw, A, B, 1.0, conv3d, dA, dB), 4 * base.numel() + 3 * ab, 2 * flop)}
    row = {"conv": ("Conv3d(3,1,1)" if conv3d else f"Conv2d {k}x{k}") + f" {cin}->{cout}", "count": count, "r": r}
    for name, (fn, nbytes, fl) in legs.items():
        for _ in range(20):
            fn()
        ms = bench.time_events(fn, launches)
        row[name] = {"us": round(1000 * ms, 2), "GB/s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                     "TFLOP/s": round(fl / (ms * 1e-3) / 1e12, 2)}
    return row


class _Timed:
    """CUDA events around the stable-LoRA-only work of one eager step (merges, projections, wgrads into W_eff scratch)."""

    def __init__(self):
        self.events = {"merge": [], "grad_projection": [], "extra_wgrad": []}
        self.saved = {}

    def _wrap(self, name, fn, pick):
        def run(*a, **k):
            if not pick(*a, **k):
                return fn(*a, **k)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn(*a, **k)
            e.record()
            self.events[name].append((s, e))
            return out
        return run

    def __enter__(self):
        for n in ("lora_delta_merge", "lora_delta_grad", "conv_wgrad"):
            self.saved[n] = getattr(prims, n)
        prims.lora_delta_merge = self._wrap("merge", self.saved["lora_delta_merge"], lambda *a, **k: True)
        prims.lora_delta_grad = self._wrap("grad_projection", self.saved["lora_delta_grad"], lambda *a, **k: True)
        prims.conv_wgrad = self._wrap("extra_wgrad", self.saved["conv_wgrad"], lambda x, dy, dw, *a, **k: getattr(dw, "_delta_scratch", False))
        self.saved_scratch = ops.DeltaWeight.grad_scratch

        def scratch(w):
            t = self.saved_scratch(w)
            t._delta_scratch = True
            return t
        ops.DeltaWeight.grad_scratch = scratch
        return self

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(prims, n, f)
        ops.DeltaWeight.grad_scratch = self.saved_scratch

    def totals_ms(self):
        torch.cuda.synchronize()
        return {k: round(sum(s.elapsed_time(e) for s, e in v), 2) for k, v in self.events.items()} | \
            {k + "_calls": len(v) for k, v in self.events.items()}


def step_row(version, steps, warmup, dev):
    wl = bench.WORKLOADS["lora"]
    unet = step = opt = None
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    try:
        from t2v_b200.utils.lora_handler import LoraHandler
        unet = bench.build_unet(dev)
        unet.requires_grad_(False)
        handler = LoraHandler(version=version, use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
        torch.manual_seed(4321)
        with contextlib.redirect_stdout(sys.stderr):
            handler.add_lora_to_model(True, unet, handler.unet_replace_modules, 0.1, "", r=wl["lora_rank"])
        unet = unet.to(dev).train()
        with torch.no_grad():   # both up / B factors start at zero: give the branch signal
            for n, p in unet.named_parameters():
                if "lora_up" in n or "lora_B" in n:
                    p.normal_(0.0, 0.01)
        unet._set_gradient_checkpointing(True)
        abar = S.ddpm_alphas_cumprod(device=dev)
        step = S.DataParallelStep(unet, abar, passes=1, use_graph=True)
        trainable = [p for p in unet.parameters() if p.requires_grad]
        opt = FusedAdamW(step.arena, [dict(params=trainable)], lr=5e-6, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=1.0)
        step.attach_optimizer(opt)
        devin = [x.to(dev) for x in bench.synthetic_inputs(1, wl, 1234)]
        for _ in range(warmup):
            step(*devin)
        torch.cuda.synchronize()
        ms = bench.time_events(lambda: step(*devin), steps)
        row = {"version": version, "ms_per_step": round(ms, 2), "peak_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2),
               "trainable": sum(p.numel() for p in trainable), "loss": float(step(*devin).item())}
        if version == "stable_lora":
            eager = S.DataParallelStep(unet, abar, passes=1, use_graph=False, adopt=False)
            eager.arena = step.arena
            eager.sync_gradients = False
            eager(*devin)
            torch.cuda.synchronize()
            eager_ms = bench.time_events(lambda: eager(*devin), 1)
            with _Timed() as t:
                eager(*devin)
                parts = t.totals_ms()
            row["eager_step_ms"] = round(eager_ms, 2)
            row["stable_only_ms"] = parts
            row["share_of_eager_step"] = {k: round(parts[k] / eager_ms, 4) for k in ("merge", "grad_projection", "extra_wgrad")}
            step.arena.zero_grads()
        return row
    except torch.cuda.OutOfMemoryError as e:
        return {"version": version, "out_of_memory": str(e).splitlines()[0]}
    finally:
        del unet, step, opt
        gc.collect()
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rank", type=int, default=16)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    report = {"gpu": gpu_info(), "timing": "CUDA events after 20 warm-up launches / --warmup steps"}
    rows = [kernel_row(*key, count, args.rank, args.launches) for key, count in sorted(conv_shapes().items())]
    for r in rows:
        print(json.dumps(r), flush=True)
    report["kernels"] = rows
    report["per_unet_pass_ms"] = {leg: round(sum(r["count"] * r[leg]["us"] for r in rows) / 1000, 3) for leg in ("merge", "grad")}
    if not args.no_step:
        report["step_cfg3"] = []
        for _ in range(args.rounds):
            for version in ("cloneofsimo", "stable_lora"):
                row = step_row(version, args.steps, args.warmup, dev)
                print(json.dumps(row), flush=True)
                report["step_cfg3"].append(row)
    line = json.dumps(report)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
