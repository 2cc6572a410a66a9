#!/usr/bin/env python
"""A/B timing of the GroupNorm+SiLU kernels (csrc/norms.cu) with their current sigmoid against the hardware-tanh sigmoid they
used before, 0.5 tanh.approx(z / 2) + 0.5, at the largest GroupNorm+SiLU launches of a cfg-2 training step
(tests/golden/norm_launches.json).  The old variant is the in-tree csrc with only sigmoidf_ replaced, built into a temporary
directory; both libraries are loaded into one process and timed alternately with CUDA events.  The forward gets the producer
sums the step passes; every backward call gets a fresh zeroed workspace (zeroed outside the timed window).
  python tools/gn_sigmoid_bench.py [--reps 200] [--rounds 7]"""
import argparse
import ctypes
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from t2v_b200 import native, prims  # noqa: E402

OLD_SIGMOID = r'''__device__ __forceinline__ float sigmoidf_(float z) {
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * z));
    return fmaf(0.5f, t, 0.5f);
}'''


def build_old(tmp):
    """The library with the tanh sigmoid in norms.cu, compiled file by file in parallel into `tmp`."""
    src = os.path.join(tmp, "pkg", "csrc")   # common.h includes ../../include/t2v_b200.h
    shutil.copytree(native.CSRC, src)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    path = os.path.join(src, "norms.cu")
    with open(path) as f:
        text = f.read()
    text, n = re.subn(r"__device__ __forceinline__ float sigmoidf_\(float z\) \{\n.*?\n\}\n", lambda _: OLD_SIGMOID + "\n", text, flags=re.S)
    assert n == 1, "sigmoidf_ not found in norms.cu"
    with open(path, "w") as f:
        f.write(text)
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    flags = [fl for fl in native.NVCC_FLAGS if fl != "-shared"]
    cus = sorted(os.path.join(src, f) for f in os.listdir(src) if f.endswith(".cu"))

    def compile_one(cu):
        obj = cu[:-3] + ".o"
        res = subprocess.run([nvcc] + flags + ["-c", cu, "-o", obj], capture_output=True, text=True)
        if res.returncode:
            raise RuntimeError(res.stdout + res.stderr)
        return obj

    with ThreadPoolExecutor(len(cus)) as ex:
        objs = list(ex.map(compile_one, cus))
    lib = os.path.join(tmp, "libt2v_b200_tanh_sigmoid.so")
    res = subprocess.run([nvcc] + native.NVCC_FLAGS + ["-o", lib] + objs, capture_output=True, text=True)
    if res.returncode:
        raise RuntimeError(res.stdout + res.stderr)
    return native._declare(ctypes.CDLL(lib))


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def cases():
    with open(os.path.join(ROOT, "tests", "golden", "norm_launches.json")) as f:
        recs = [r for r in json.load(f) if r["kind"].startswith("groupnorm") and r["silu"]]
    out = []
    for kind in ("groupnorm_fwd", "groupnorm_bwd"):
        out += sorted((r for r in recs if r["kind"] == kind), key=lambda r: -r["S"] * r["P"] * r["C"])[:3]
    return out


def runner(lib, r, reps):
    """A closure that launches `r` once on `lib` (inputs shared by both libraries) and the bytes one launch moves."""
    S, P, C, G = r["S"], r["P"], r["C"], r["G"]
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(S, P, C, device="cuda", generator=g) * 2 + 0.5).bfloat16()
    gamma = 1 + 0.5 * torch.randn(C, device="cuda", generator=g)
    beta = 1.5 * torch.randn(C, device="cuda", generator=g)
    y = torch.empty_like(x)
    stat = torch.empty(S, G, 2, device="cuda")
    ab = torch.empty(S, C, 2, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if r["kind"] == "groupnorm_fwd":
        xf = x.view(r["frames"], -1, C)
        if r["stats"] == 2:
            st = [prims.channel_stats(xf[..., :r["C0"]].contiguous()), prims.channel_stats(xf[..., r["C0"]:].contiguous())]
        else:
            st = [prims.channel_stats(xf)]
        s1 = st[1] if len(st) > 1 else None
        args = (_p(x), _p(gamma), _p(beta), _p(y), _p(stat), _p(ab), _p(st[0]), r["C0"], r["C0"], _p(s1),
                C - r["C0"], r["fps"], _p(None), S, P, C, G, float(r["eps"]), 1, stream)
        return (lambda i: native.check(lib.t2v_groupnorm_fwd(*args))), None, 2 * x.numel() * 2
    _, stat, ab = prims.groupnorm_fwd(x, gamma, beta, G, 1e-5, 1)
    dy = torch.randn(S, P, C, device="cuda", generator=g).bfloat16()
    dx = torch.empty_like(x)
    dgamma, dbeta = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    ws = torch.zeros(reps, S * C * 2, device="cuda")

    def run(i):
        native.check(lib.t2v_groupnorm_bwd(_p(dy), _p(x), _p(gamma), _p(stat), _p(ab), _p(None), _p(dx), _p(dgamma), _p(dbeta),
                                           _p(ws[i]), S, P, C, G, 1, stream))
    # sums pass reads x, dy; apply pass reads x, dy and writes dx
    return run, ws, 5 * x.numel() * 2


def time_one(run, ws, reps):
    if ws is not None:
        ws.zero_()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(reps):
        run(i)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name(0)} ({smi})")
    native.build()
    new = native.lib()
    with tempfile.TemporaryDirectory() as tmp:
        old = build_old(tmp)
        for r in cases():
            runs = {name: runner(lib, r, args.reps) for name, lib in (("tanh", old), ("new", new))}
            for name, (run, ws, _) in runs.items():   # warm-up
                time_one(run, ws, min(20, args.reps))
            times = {name: [] for name in runs}
            for _ in range(args.rounds):
                for name, (run, ws, _) in runs.items():
                    times[name].append(time_one(run, ws, args.reps))
            nbytes = runs["new"][2]
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            spread = {k: (min(v), max(v)) for k, v in times.items()}
            tag = f'{r["kind"]} S={r["S"]} P={r["P"]} C={r["C"]}'
            print(f"{tag}: tanh {med['tanh']:.2f} us [{spread['tanh'][0]:.2f}, {spread['tanh'][1]:.2f}], "
                  f"new {med['new']:.2f} us [{spread['new'][0]:.2f}, {spread['new'][1]:.2f}], "
                  f"new/old {med['new'] / med['tanh']:.3f}, {nbytes / med['new'] / 1e3:.0f} GB/s (new)")


if __name__ == "__main__":
    main()
