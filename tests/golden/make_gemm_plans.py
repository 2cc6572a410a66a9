#!/usr/bin/env python
"""Regenerates tests/golden/gemm_plans.json: the launches the GEMM planner (csrc/gemm_plan.cu) picks, queried through
t2v_gemm_plan, for
  * every distinct GEMM problem of one cfg-2 training step (bench.py's default workload): fwd, dgrad and wgrad of every
    convolution and linear layer and every batched attention GEMM, with the workspace, statistics and bias-gradient options
    the step passes.  They are recorded on the CPU by running the full-size UNet forward and backward over oracle/ops_ref.py
    with the four GEMM primitives replaced by recorders that only allocate their outputs;
  * every case of tests/test_gemm_gpu.py, with the planner overrides it sets;
each at 132 SMs (H100 SXM) and 114 SMs (H100 PCIe).  tests/test_gemm_plan.py requires the planner to reproduce the table
exactly, so a change that moves plans on purpose regenerates it, and the diff of this file shows which launches moved.
  python tests/golden/make_gemm_plans.py [--lib other_build.so]
--lib queries another library that exports t2v_gemm_plan (e.g. an older planner built for comparison)."""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "gemm_plans.json")

SM_COUNTS = (132, 114)
# every environment variable the planner reads (T2V_FORCE_*: sweep / test overrides, T2V_NO_*: A/B switches)
PLANNER_ENV = ("T2V_FORCE_BN", "T2V_FORCE_SPLITS", "T2V_FORCE_FWD_SPLITS", "T2V_FORCE_STAGES", "T2V_NO_SPLIT", "T2V_NO_ROWSUM_FUSE")
KINDS = ("fwd", "dgrad", "wgrad", "bgemm")
CONV_FIELDS = ("N", "H", "W", "Cin", "Cout", "KH", "KW", "stride", "pads", "workspace", "stats_rows", "dbias")
BGEMM_FIELDS = ("M", "N", "K", "Z1", "Z2", "b_kmajor", "out_mode")


def conv_problem(kind, N, H, W, Cin, Cout, KH, KW, stride, pads, workspace=0, stats_rows=0, dbias=0):
    return {"kind": kind, "N": N, "H": H, "W": W, "Cin": Cin, "Cout": Cout, "KH": KH, "KW": KW, "stride": stride,
            "pads": list(pads), "workspace": int(workspace), "stats_rows": int(stats_rows), "dbias": int(dbias)}


def bgemm_problem(M, N, K, Z1, Z2, b_kmajor, out_mode):
    return {"kind": "bgemm", "M": M, "N": N, "K": K, "Z1": Z1, "Z2": Z2, "b_kmajor": int(b_kmajor), "out_mode": out_mode}


def step_problems():
    """The GEMM problems of one cfg-2 step (batch 1, 16 frames, 32x32 latents, 77 text tokens), in call order."""
    import torch

    import bench
    from helpers import emulated_prims
    from t2v_b200 import prims
    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from oracle import leaves as L

    seen = []

    def conv_fwd(x, w, bias=None, rowbias=None, residual=None, stride=1, pads=(0, 0, 0, 0), alpha=1.0, out_fp32=False,
                 rowbias_div=1, stats=None, stats_rows=0):
        N, H, W, Ci = x.shape
        Co, KH, KW, _ = w.shape
        # prims.conv_fwd always offers the split-K scratch the planner asks for
        seen.append(conv_problem("fwd", N, H, W, Ci, Co, KH, KW, stride, pads, 1, stats_rows if stats is not None else 0))
        Ho, Wo = prims.out_hw(H, W, KH, KW, stride, pads)
        return torch.zeros((N, Ho, Wo, Co), dtype=torch.float32 if out_fp32 else torch.bfloat16)

    def conv_dgrad(dy, w, in_hw, stride=1, pads=(0, 0, 0, 0), residual=None):
        Co, KH, KW, Ci = w.shape
        seen.append(conv_problem("dgrad", dy.shape[0], in_hw[0], in_hw[1], Ci, Co, KH, KW, stride, pads, 1))
        return torch.zeros((dy.shape[0], in_hw[0], in_hw[1], Ci), dtype=torch.bfloat16)

    def conv_wgrad(x, dy, dw, stride=1, pads=(0, 0, 0, 0), dbias=None):
        N, H, W, Ci = x.shape
        Co, KH, KW, _ = dw.shape
        seen.append(conv_problem("wgrad", N, H, W, Ci, Co, KH, KW, stride, pads, dbias=dbias is not None))

    def bgemm(a, a_desc, b, b_desc, c, c_desc, M, N, K, Z1, Z2, alpha=1.0, out_mode=0):
        seen.append(bgemm_problem(M, N, K, Z1, Z2, b_desc[0], out_mode))

    wl = bench.WORKLOADS["cfg2"]
    F, (H, W) = wl["frames"], wl["latent_hw"]
    torch.manual_seed(0)
    m = UNet3DConditionModel().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    lat, noise = torch.randn(1, 4, F, H, W), torch.randn(1, 4, F, H, W)
    ehs = torch.randn(1, wl["text_len"], wl["text_dim"])
    with emulated_prims():
        hooks = {"conv_fwd": conv_fwd, "conv_dgrad": conv_dgrad, "conv_wgrad": conv_wgrad, "bgemm": bgemm}
        for name, fn in hooks.items():   # emulated_prims() restores the native functions on exit
            setattr(prims, name, fn)
        loss = S.finetune_loss(m, lat, noise, torch.tensor([417]), ehs, L.ddpm_alphas_cumprod())
        loss.backward()
    return seen


def test_problems():
    """The problems tests/test_gemm_gpu.py runs, each with the environment it runs under."""
    import test_gemm_gpu as T
    out = []
    for c in T.CONV_CASES:
        out.append((conv_problem("fwd", *c), {}))
    for c in T.DGRAD_CASES:
        out += [(conv_problem("dgrad", *c), {}), (conv_problem("wgrad", *c), {})]
    for c, bn, colsum in T.WGRAD_BIAS_CASES:
        env = {}
        if bn:
            env["T2V_FORCE_BN"] = str(bn)
        if colsum:
            env["T2V_NO_ROWSUM_FUSE"] = "1"
        out += [(conv_problem("wgrad", *c), env), (conv_problem("wgrad", *c, dbias=1), env)]
    for c in T.SPLITK_CASES:
        out += [(conv_problem("fwd", *c, workspace=1), {}), (conv_problem("dgrad", *c, workspace=1), {})]
    for M, N, K, Z1, Z2, _, bk, mode, _ in T.BGEMM_CASES:
        out.append((bgemm_problem(M, N, K, Z1, Z2, bk, mode), {}))
    return out


def to_struct(prob):
    from t2v_b200 import native
    s = native.GemmProblem()
    s.kind = KINDS.index(prob["kind"])
    if prob["kind"] == "bgemm":
        s.gemm_m, s.gemm_n, s.gemm_k, s.z1, s.z2 = prob["M"], prob["N"], prob["K"], prob["Z1"], prob["Z2"]
        s.b_kmajor, s.out_mode = prob["b_kmajor"], prob["out_mode"]
    else:
        for f in CONV_FIELDS:
            if f != "pads":
                setattr(s, f, prob[f])
        s.pad_h0, s.pad_h1, s.pad_w0, s.pad_w1 = prob["pads"]
    return s


def query(lib, prob, env, sm_count, max_out=8):
    """The launches `lib`'s planner makes for `prob` under `env` (the planner overrides) on `sm_count` SMs, as dicts."""
    from t2v_b200 import native
    saved = {k: os.environ.pop(k, None) for k in PLANNER_ENV}
    os.environ.update(env)
    try:
        out = (native.GemmPlan * max_out)()
        n = lib.t2v_gemm_plan(ctypes.byref(to_struct(prob)), sm_count, out, max_out)
    finally:
        for k in PLANNER_ENV:
            os.environ.pop(k, None)
            if saved[k] is not None:
                os.environ[k] = saved[k]
    if n < 0 or n > max_out:
        raise RuntimeError(f"t2v_gemm_plan({prob}, {env}, {sm_count}) returned {n}")
    return [{f: (list(getattr(p, f)) if isinstance(getattr(p, f), ctypes.Array) else getattr(p, f)) for f, _ in p._fields_}
            for p in out[:n]]


def load(path=""):
    """The in-tree library (built if stale), or the library at `path`."""
    from t2v_b200 import native
    if not path:
        native.build()
        return native.lib()
    lib = ctypes.CDLL(os.path.abspath(path))
    lib.t2v_gemm_plan.argtypes = [ctypes.POINTER(native.GemmProblem), ctypes.c_int32, ctypes.POINTER(native.GemmPlan), ctypes.c_int32]
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default="", help="library to query (default: the in-tree build)")
    ap.add_argument("--out", default=OUT)
    args = ap.parse_args()
    lib = load(args.lib)
    cases, keys = [], set()
    for prob, env in [(p, {}) for p in step_problems()] + test_problems():
        key = json.dumps([prob, env], sort_keys=True)
        if key not in keys:
            keys.add(key)
            cases.append((prob, env))
    with open(args.out, "w") as f:
        f.write("[\n")
        for i, (prob, env) in enumerate(cases):
            rec = {"problem": prob, "env": env, "plans": {str(s): query(lib, prob, env, s) for s in SM_COUNTS}}
            f.write(json.dumps(rec, separators=(",", ":")) + (",\n" if i + 1 < len(cases) else "\n"))
        f.write("]\n")
    print(f"{args.out}: {len(cases)} problems x {len(SM_COUNTS)} SM counts")


if __name__ == "__main__":
    main()
