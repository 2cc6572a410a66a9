#!/usr/bin/env python
"""Regenerates tests/golden/norm_launches.json: every distinct launch of the normalisation and activation kernels in one cfg-2
training step (bench.py's default workload), forward and backward:
  groupnorm_fwd / groupnorm_bwd   S, P, C, G, eps, silu; forward: the producer statistics the step passes (none, or one or two
                                  sources with their frame count and the channel split C0) and fps; backward: whether dgamma /
                                  dbeta are accumulated and whether a residual gradient is added
  layernorm_fwd / layernorm_bwd   rows, C, eps; backward: dgamma / dbeta, residual gradient
  geglu_fwd / geglu_bwd           M, I (proj is [M][2I])
  silu_bf16 / silu_bf16_bwd / silu_f32_to_bf16 / silu_bwd_f32   the tensor shape (silu_f32_to_bf16: also apply_silu)
They are recorded on the CPU by running the full-size UNet forward and backward over oracle/ops_ref.py with the four GEMM
primitives replaced by allocators (as make_gemm_plans.step_problems() does) and the recorded primitives wrapped by recorders.
tests/test_norm_step_gpu.py runs every launch; tests/test_norm_step_cpu.py checks that this script reproduces the table.
  python tests/golden/make_norm_launches.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "norm_launches.json")

KINDS = ("groupnorm_fwd", "groupnorm_bwd", "layernorm_fwd", "layernorm_bwd", "geglu_fwd", "geglu_bwd", "silu_bf16", "silu_bf16_bwd",
         "silu_f32_to_bf16", "silu_bwd_f32")


def _records(name, args, kw):
    """The launch record of prims.<name>(*args, **kw)."""
    def arg(i, key, default=None):
        return args[i] if len(args) > i else kw.get(key, default)

    if name == "groupnorm_fwd":
        x, G, eps, silu, stats, fps = args[0], arg(3, "G"), arg(4, "eps"), arg(5, "silu"), arg(6, "stats"), arg(7, "fps", 1)
        S, P, C = x.shape
        rec = {"S": S, "P": P, "C": C, "G": G, "eps": float(eps), "silu": int(bool(silu)), "stats": 0, "frames": 0, "C0": C, "fps": 1}
        if stats:
            rec.update(stats=len(stats), frames=stats[0].shape[0], C0=stats[0].shape[1], fps=int(fps))
        return rec
    if name == "groupnorm_bwd":
        x, G, silu = args[1], arg(5, "G"), arg(6, "silu")
        S, P, C = x.shape
        return {"S": S, "P": P, "C": C, "G": G, "silu": int(bool(silu)), "add": int(arg(7, "add") is not None),
                "dgamma": int(arg(8, "dgamma") is not None), "dbeta": int(arg(9, "dbeta") is not None)}
    if name == "layernorm_fwd":
        rows, C = args[0].shape
        return {"rows": rows, "C": C, "eps": float(arg(3, "eps"))}
    if name == "layernorm_bwd":
        rows, C = args[1].shape
        return {"rows": rows, "C": C, "add": int(arg(4, "add") is not None), "dgamma": int(arg(5, "dgamma") is not None),
                "dbeta": int(arg(6, "dbeta") is not None)}
    if name in ("geglu_fwd", "geglu_bwd"):
        M, I2 = args[0].shape
        return {"M": M, "I": I2 // 2}
    rec = {"shape": list(args[0].shape)}
    if name == "silu_f32_to_bf16":
        rec["apply"] = int(bool(arg(1, "apply_silu", True)))
    return rec


def step_launches():
    """The distinct norm / activation launches of one cfg-2 step (batch 1, 16 frames, 32x32 latents, 77 text tokens), in first
    call order, as {"kind": ..., **fields}."""
    import torch

    import bench
    from helpers import emulated_prims
    from t2v_b200 import prims
    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from oracle import leaves as L

    seen, keys = [], set()

    def recorder(name, fn):
        def run(*args, **kw):
            rec = {"kind": name, **_records(name, args, kw)}
            key = json.dumps(rec, sort_keys=True)
            if key not in keys:
                keys.add(key)
                seen.append(rec)
            return fn(*args, **kw)
        return run

    def conv_fwd(x, w, bias=None, rowbias=None, residual=None, stride=1, pads=(0, 0, 0, 0), alpha=1.0, out_fp32=False,
                 rowbias_div=1, stats=None, stats_rows=0):
        Ho, Wo = prims.out_hw(x.shape[1], x.shape[2], w.shape[1], w.shape[2], stride, pads)
        return torch.zeros((x.shape[0], Ho, Wo, w.shape[0]), dtype=torch.float32 if out_fp32 else torch.bfloat16)

    def conv_dgrad(dy, w, in_hw, stride=1, pads=(0, 0, 0, 0), residual=None):
        return torch.zeros((dy.shape[0], in_hw[0], in_hw[1], w.shape[3]), dtype=torch.bfloat16)

    def nothing(*args, **kw):
        return None

    wl = bench.WORKLOADS["cfg2"]
    F, (H, W) = wl["frames"], wl["latent_hw"]
    torch.manual_seed(0)
    m = UNet3DConditionModel().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    lat, noise = torch.randn(1, 4, F, H, W), torch.randn(1, 4, F, H, W)
    ehs = torch.randn(1, wl["text_len"], wl["text_dim"])
    with emulated_prims():   # restores the native functions on exit
        for name in KINDS:
            setattr(prims, name, recorder(name, getattr(prims, name)))
        for name, fn in {"conv_fwd": conv_fwd, "conv_dgrad": conv_dgrad, "conv_wgrad": nothing, "bgemm": nothing}.items():
            setattr(prims, name, fn)
        loss = S.finetune_loss(m, lat, noise, torch.tensor([417]), ehs, L.ddpm_alphas_cumprod())
        loss.backward()
    return seen


def write(launches, path=OUT):
    with open(path, "w") as f:
        f.write("[\n" + ",\n".join(json.dumps(r, separators=(",", ":")) for r in launches) + "\n]\n")


def main():
    launches = step_launches()
    write(launches)
    counts = {k: sum(r["kind"] == k for r in launches) for k in KINDS}
    print(f"{OUT}: {len(launches)} launches {counts}")


if __name__ == "__main__":
    main()
