#!/usr/bin/env python
"""Device time of the normalisation and activation family of one cfg-2 finetune step: GroupNorm, LayerNorm, GEGLU and SiLU.

One eager cfg-2 step records every call of these primitives with its multiplicity (profiling.record_calls).  Each distinct
call is then replayed as a CUDA graph of back-to-back launches between CUDA events (profiling.replay_us), twice:
  warm  the same operands every launch: they sit in L2, as in the step, where the producer has just written them;
  cold  rotating operand copies whose footprint exceeds L2.
Algorithmic bytes come from the shapes (algo_bytes below); `frac` is bytes / time over 3.35 TB/s (H100 SXM HBM3, data
sheet).  A call is one primitive call: groupnorm_bwd is its sums and apply kernels together, and a groupnorm_fwd without
producer statistics is its sums and apply kernels together.

Prints a table on stderr and one JSON line on stdout.  Usage: python tools/norm_bench.py [--small] [--reps N]"""
import argparse
import collections
import inspect
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
from t2v_b200.profiling import record_calls, replay_us  # noqa: E402

HBM_BPS = 3.35e12
KINDS = ("groupnorm_fwd", "groupnorm_bwd", "layernorm_fwd", "layernorm_bwd", "geglu_fwd", "geglu_bwd",
         "silu_bf16", "silu_bf16_bwd", "silu_f32_to_bf16", "silu_bwd_f32")
SIGS = {n: inspect.signature(getattr(prims, n)) for n in KINDS}


def _nb(t):
    if t is None:
        return 0
    if isinstance(t, (list, tuple)):
        return sum(_nb(v) for v in t)
    return t.numel() * t.element_size()


def algo_bytes(name, a, k):
    """(signature, bytes the call must move at least) from the call's arguments."""
    b = SIGS[name].bind(*a, **k)
    b.apply_defaults()
    v = b.arguments
    if name == "groupnorm_fwd":
        x = v["x"]
        Sn, P, C = x.shape
        small = _nb(v["gamma"]) + _nb(v["beta"]) + Sn * v["G"] * 8 + Sn * C * 8   # gamma, beta; stat and ab written
        own = not v["stats"]                                                       # no producer sums: x is read twice
        sig = f"{Sn}x{P}x{C} g{v['G']} silu{int(bool(v['silu']))} " + ("own-sums" if own else f"stats{len(v['stats'])} fps{v['fps']}")
        return sig, (3 if own else 2) * _nb(x) + small + _nb(v["stats"])
    if name == "groupnorm_bwd":
        x = v["x"]
        Sn, P, C = x.shape
        small = _nb(v["gamma"]) + _nb(v["stat"]) + _nb(v["ab"]) + _nb(v["dgamma"]) + _nb(v["dbeta"])
        sig = f"{Sn}x{P}x{C} g{v['G']} silu{int(bool(v['silu']))}" + (" add" if v["add"] is not None else "")
        return sig, 2 * _nb(x) + 3 * _nb(x) + _nb(v["add"]) + small            # sums: x, dy; apply: x, dy, dx (+ add)
    if name == "layernorm_fwd":
        x = v["x"]
        return f"{x.shape[0]}x{x.shape[1]}", 2 * _nb(x) + x.shape[0] * 8 + _nb(v["gamma"]) + _nb(v["beta"])
    if name == "layernorm_bwd":
        x = v["x"]
        sig = f"{x.shape[0]}x{x.shape[1]}" + (" add" if v["add"] is not None else "")
        return sig, 3 * _nb(x) + _nb(v["add"]) + _nb(v["stat"]) + _nb(v["gamma"]) + _nb(v["dgamma"]) + _nb(v["dbeta"])
    if name == "geglu_fwd":
        p = v["proj"]
        return f"{p.shape[0]}x{p.shape[1] // 2}", _nb(p) + _nb(p) // 2
    if name == "geglu_bwd":
        p = v["proj"]
        return f"{p.shape[0]}x{p.shape[1] // 2}", 2 * _nb(p) + _nb(v["dout"])
    x = v["x"]
    out = x.numel() * (4 if name == "silu_bwd_f32" else 2)
    return "x".join(map(str, x.shape)), _nb(x) + _nb(v.get("dy")) + out


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power, mhz = (s.strip() for s in r.stdout.strip().split(","))
        return {"name": name, "power_limit": power, "sm_max_clock": mhz}
    except Exception:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "sm_max_clock": "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="debug-size UNet (not the cfg-2 step)")
    ap.add_argument("--reps", type=int, default=20, help="launches per replayed graph (warm; cold uses at least 4 operand sets)")
    ap.add_argument("--tag", default="", help="label copied into the JSON line")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    unet = bench.build_unet(dev, args.small)
    step = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device=dev), passes=1, use_graph=False)
    inputs = [x.to(dev) for x in bench.synthetic_inputs(1, bench.CFG2, 1234)]
    step(*inputs)
    torch.cuda.synchronize()
    calls = record_calls(lambda: step(*inputs), KINDS, algo_bytes)
    del step, unet
    torch.cuda.empty_cache()

    rows = []
    with bench.ClockSampler(0) as clocks:
        for key, (cnt, (sig, nbytes)) in calls.items():
            warm = replay_us(key, dev, reps=args.reps, batches=3)
            cold = replay_us(key, dev, reps=8, cold=True, batches=3)
            rows.append(dict(kind=key[0], sig=sig, n=cnt, bytes=nbytes, warm_us=warm, cold_us=cold))
    kinds = collections.OrderedDict((k, dict(n=0, bytes=0, warm_ms=0.0, cold_ms=0.0)) for k in KINDS)
    for r in rows:
        s = kinds[r["kind"]]
        s["n"] += r["n"]
        s["bytes"] += r["n"] * r["bytes"]
        s["warm_ms"] += r["n"] * r["warm_us"] / 1e3
        s["cold_ms"] += r["n"] * r["cold_us"] / 1e3
    kinds = {k: s for k, s in kinds.items() if s["n"]}
    total = dict(n=sum(s["n"] for s in kinds.values()), bytes=sum(s["bytes"] for s in kinds.values()),
                 warm_ms=sum(s["warm_ms"] for s in kinds.values()), cold_ms=sum(s["cold_ms"] for s in kinds.values()))
    for s in list(kinds.values()) + [total]:
        s["bound_ms"] = s["bytes"] / HBM_BPS * 1e3
        s["warm_frac"] = s["bound_ms"] / s["warm_ms"]
        s["cold_frac"] = s["bound_ms"] / s["cold_ms"]
    info = card()

    err = sys.stderr
    print(f"{info['name']}, power limit {info['power_limit']}, max SM clock {info['sm_max_clock']}; clocks during replay {clocks.summary()}", file=err)
    print(f"{'kind':18s} {'calls':>5s} {'GB':>7s} {'bound ms':>8s} {'warm ms':>8s} {'frac':>5s} {'cold ms':>8s} {'frac':>5s}", file=err)
    for k, s in list(kinds.items()) + [("family", total)]:
        print(f"{k:18s} {s['n']:5d} {s['bytes'] / 1e9:7.3f} {s['bound_ms']:8.3f} {s['warm_ms']:8.3f} {s['warm_frac']:5.2f} "
              f"{s['cold_ms']:8.3f} {s['cold_frac']:5.2f}", file=err)
    print(file=err)
    for r in sorted(rows, key=lambda r: -r["n"] * r["cold_us"]):
        print(f"  {r['kind']:16s} {r['sig']:34s} n={r['n']:3d} {r['bytes'] / 1e6:8.2f} MB  warm {r['warm_us']:7.2f} us "
              f"({r['bytes'] / (r['warm_us'] * 1e-6) / HBM_BPS:4.2f})  cold {r['cold_us']:7.2f} us "
              f"({r['bytes'] / (r['cold_us'] * 1e-6) / HBM_BPS:4.2f})", file=err)
    print(json.dumps(dict(tag=args.tag, card=info, clocks=clocks.summary(), small=args.small, family=total, kinds=kinds,
                          launches=rows)), flush=True)


if __name__ == "__main__":
    main()
