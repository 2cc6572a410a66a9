#!/usr/bin/env python
"""Regenerates tests/golden/optim_launches.json: every distinct launch of the optimizer kernels (csrc/optim.cu: sqnorm_chunks,
adamw_prepare, adamw_chunks, adamw8bit_chunks, adamw_ema_chunks, adamw8bit_ema_chunks, ema_swap_chunks), of the stable-LoRA
delta kernels (csrc/lora_delta.cu: lora_delta_merge, lora_delta_grad) and of the gradient compression before the data-parallel
all-reduce (scale_cast_f32_bf16) in the training steps.

The chunk tables are built by the real code paths on the meta device: the parameter groups by train.create_optimizer_params /
param_optim (as train.main builds them), the tables by the FusedAdamW / AdamW8bit constructors over the step's ParamArena, the
compression ranges by runtime.GradientBuckets (its collective replaced by a no-op).  A table is not written out; a record holds
  update kinds      workload, variant, cols (2 / 3: + EMA offset; 8-bit 4 / 5: + state offset, bits), g16 (the gradient read from
                    the bf16 twin), hp (lr, beta1, beta2, eps, weight_decay of the set), ema_decay (EMA kinds), n_rows, hist
                    (rows per power-of-two length bucket: key b counts the rows of length in (2^(b-1), 2^b]), total (arena
                    elements), n_shadow, n_state (fp32 moment elements; 8-bit kinds also n_state8), n_ema, rows8 / rows32 (8-bit
                    kinds), above_shadow (some row starts at or above n_shadow), over_grid (more rows than the 1,056-block grid
                    of a 132-SM H100), sha256 of the int64 table
  sqnorm_chunks     workload, variant, g16, n_rows, hist, total, sha256 of the (offset, length) table
  ema_swap_chunks   workload, variant, n_rows, hist, total, n_shadow, n_ema, sha256 of the (offset, length, EMA offset) table
  adamw_prepare     n_sets, max_norm
  lora_delta_*      Cout, Cin, k, r, conv3d, scaling
  scale_cast_f32_bf16   workload, n (one piece), world (the kernel scales by 1 / world)
Records are deduplicated by everything but their labels (workload, variant), in first-call order: identical tables share a
record.  tables() rebuilds every table on the CPU from the same workloads, keyed by its digest.
Workloads:
  full         cfg2 / zeroscope (one table): the whole ms-1.7b UNet trainable, one group per parameter (lr 5e-6, wd 1e-2,
               max_grad_norm 1.0); FusedAdamW and AdamW8bit, each without and with EMA (decay 0.9999), each reading the fp32
               gradient and its bf16 twin
  train_config the reference's train_config.yaml: UNet 'all', cloneofsimo UNet LoRA rank 16 and text-encoder LoRA rank 16 (extra
               arena parameters), lr 5e-6, adam_weight_decay 0
  lora         bench.WORKLOADS["lora"]: UNet frozen, cloneofsimo LoRA rank 16 on every UNet linear (29,246,112 trainable
               elements between frozen base weights), one group, lr 5e-6, wd 1e-2
  stable_lora  stable_lora_config.yaml at rank 16 (the UNet adapters; its use_text_lora is not built for stable_lora): the
               lora_delta launches of one 8-frame 48 x 48 training pass, and FusedAdamW plus AdamW8bit with EMA over the LoRA group
  text_train   train_config.yaml with train_text_encoder and trainable_text_modules 'all', extra_unet_params {lr: 1e-5,
               weight_decay: 1e-4}
  buckets      GradientBuckets pieces (at most 2^26 elements) of the full and the lora step at world sizes 2, 6 and 8
plus synthetic launches (marked "synthetic": 1, with their table in "rows") of live paths no workload reaches (synthetic()).
tests/test_optim_step_gpu.py runs every launch; tests/test_optim_step_cpu.py checks that this script reproduces the file.
  python tests/golden/make_optim_launches.py"""
import contextlib
import hashlib
import inspect
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
OUT = os.path.join(ROOT, "tests", "golden", "optim_launches.json")

UPDATE_KINDS = ("adamw_chunks", "adamw8bit_chunks", "adamw_ema_chunks", "adamw8bit_ema_chunks")
KINDS = ("sqnorm_chunks", "adamw_prepare") + UPDATE_KINDS + ("ema_swap_chunks", "lora_delta_merge", "lora_delta_grad",
                                                             "scale_cast_f32_bf16")
LABELS = ("workload", "variant")
GRID = 8 * 132        # chunk_grid() blocks on a 132-SM H100 SXM
WORLDS = (2, 6, 8)
MAX_NORM = 1.0
EMA_DECAY = 0.9999


def digest(table):
    import torch
    t = table.to(torch.int64).contiguous()
    return hashlib.sha256(t.numpy().tobytes()).hexdigest()


def hist(lengths):
    out = {}
    for n in lengths:
        b = max(0, (int(n) - 1).bit_length())
        out[str(b)] = out.get(str(b), 0) + 1
    return dict(sorted(out.items(), key=lambda kv: int(kv[0])))


# ---------------------------------------------------------------------------------------------- workloads (meta device)
def _setup(trainable_modules=None, use_unet_lora=False, use_text_lora=False, train_text_encoder=False, trainable_text_modules=None,
           lora_version="cloneofsimo", extra_unet_params=None, lr=5e-6):
    """train.main's model, LoRA and group construction (train.py) on the meta device; returns (unet, text_encoder, groups,
    arena) with the arena laid out as DataParallelStep lays it out."""
    import torch

    from t2v_b200 import train as T
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.runtime import ParamArena
    from t2v_b200.utils.lora_handler import LoraHandler
    dev = torch.device("meta")
    with dev:
        unet = UNet3DConditionModel()
    unet.requires_grad_(False)
    lm = LoraHandler(version=lora_version, use_unet_lora=use_unet_lora, use_text_lora=use_text_lora,
                     unet_replace_modules=["UNet3DConditionModel"], text_encoder_replace_modules=["CLIPEncoderLayer"])
    with dev:
        unet_lora, unet_neg = lm.add_lora_to_model(use_unet_lora, unet, lm.unet_replace_modules, 0.1, "", r=16)
    te = text_lora = text_neg = None
    if use_text_lora or train_text_encoder:
        from t2v_b200.text_encoder import CLIPTextModel
        with dev:
            te = CLIPTextModel()
            text_lora, text_neg = lm.add_lora_to_model(use_text_lora, te, lm.text_encoder_replace_modules, 0.1, "", r=16)
        if train_text_encoder:
            T.handle_trainable_modules(te, trainable_text_modules, is_enabled=True, negation=text_neg)
    T.handle_trainable_modules(unet, trainable_modules, is_enabled=True, negation=unet_neg)
    extra = extra_unet_params or {}
    groups = T.create_optimizer_params([
        T.param_optim(unet, trainable_modules is not None, extra_params=extra, negation=unet_neg),
        T.param_optim(te, train_text_encoder, extra_params=extra, negation=text_neg),
        T.param_optim(text_lora, use_text_lora, is_lora=True, extra_params={**{"lr": lr}, **extra}),
        T.param_optim(unet_lora, use_unet_lora, is_lora=True, extra_params={**{"lr": lr}, **extra}),
    ], lr)
    text_params = ()
    if te is not None:
        every = te.base_trains()
        text_params = [p for p in te.parameters() if p.requires_grad or every]
    arena = ParamArena(unet, device=dev, extra=text_params)
    return unet, te, groups, arena


def _bench_lora():
    """bench.py's lora workload: the frozen UNet with cloneofsimo rank-16 LoRA on UNet3DConditionModel, one group."""
    import torch

    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.runtime import ParamArena
    from t2v_b200.utils.lora_handler import LoraHandler
    dev = torch.device("meta")
    with dev:
        unet = UNet3DConditionModel()
    unet.requires_grad_(False)
    h = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    with dev:
        h.add_lora_to_model(True, unet, h.unet_replace_modules, 0.1, "", r=16)
    arena = ParamArena(unet, device=dev)
    return unet, [dict(params=[p for p in unet.parameters() if p.requires_grad])], arena


def _stable_pass(unet):
    """One training pass (forward and backward) of the stable-LoRA UNet at the config's 8 frames of 384 x 384 (48 x 48 latents)."""
    import torch

    from oracle import leaves as L
    from t2v_b200 import step as S
    dev = torch.device("meta")
    unet.train()
    for mod in unet.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    B, F, hw = 1, 8, (48, 48)
    lat, noise = torch.zeros(B, 4, F, *hw, device=dev), torch.zeros(B, 4, F, *hw, device=dev)
    loss = S.finetune_loss(unet, lat, noise, torch.full((B,), 417, device=dev), torch.zeros(B, 77, 1024, device=dev),
                           L.ddpm_alphas_cumprod().to(dev))
    loss.backward()


class _Tables:
    """id(device table) -> host table of an optimizer's sets (the device copies on meta hold no values)."""

    def __init__(self):
        self.host = {}

    def add(self, opt):
        for s in opt._sets:
            self.host[id(s["chunks"])] = s["chunks_host"]
            self.host[id(s["norm_chunks"])] = s["chunks_host"][:, :2].contiguous()
            if "ema_chunks" in s:
                self.host[id(s["ema_chunks"])] = s["ema_chunks_host"]
        if opt.ema is not None:
            self.host[id(opt._ema_swap)] = __import__("torch").cat([s["ema_chunks_host"][:, [0, 1, -1]] for s in opt._sets]).contiguous()

    def __call__(self, t):
        return self.host[id(t)]


def _record(name, A, ctx):
    """The launch record of a prims.<name> call with bound arguments A (with "kind") and, for the table kinds, the host table."""
    opt, ar = ctx.get("opt"), ctx.get("arena")
    lab = {"workload": ctx.get("workload"), "variant": ctx.get("variant")}
    if name == "sqnorm_chunks":
        t = ctx["tables"](A["chunks"])
        return {"kind": name, **lab, "g16": int(A.get("g_bf16") is not None), "n_rows": t.shape[0], "hist": hist(t[:, 1].tolist()),
                "total": ar.total, "sha256": digest(t)}, t
    if name == "adamw_prepare":
        return {"kind": name, "n_sets": A["hp_in"].shape[0], "max_norm": float(A["max_norm"] or 0.0)}, None
    if name in UPDATE_KINDS:
        eight, ema = "8bit" in name, "ema" in name
        t = ctx["tables"](A["chunks"])
        (s,) = [s for s in opt._sets if A["chunks"] is s["chunks"] or A["chunks"] is s.get("ema_chunks")]
        rec = {"kind": name, **lab, "cols": t.shape[1], "g16": int(A.get("g_bf16") is not None), "hp": [float(v) for v in s["key"]]}
        if ema:
            rec["ema_decay"] = float(A["ema_decay"])
        rec.update(n_rows=t.shape[0], hist=hist(t[:, 1].tolist()), total=ar.total, n_shadow=int(A["n_shadow"]))
        if eight:
            rec.update(n_state=A["m32"].numel(), n_state8=A["code_m"].numel(), rows8=int((t[:, 3] == 8).sum()),
                       rows32=int((t[:, 3] == 32).sum()))
        else:
            rec["n_state"] = A["m"].numel()
        rec["n_ema"] = A["ema"].numel() if ema else 0
        rec.update(above_shadow=int(bool((t[:, 0] >= int(A["n_shadow"])).any())), over_grid=int(t.shape[0] > GRID), sha256=digest(t))
        return rec, t
    if name == "ema_swap_chunks":
        t = ctx["tables"](A["rows"])
        return {"kind": name, **lab, "n_rows": t.shape[0], "hist": hist(t[:, 1].tolist()), "total": ar.total,
                "n_shadow": int(A["n_shadow"]), "n_ema": A["ema"].numel(), "sha256": digest(t)}, t
    if name == "lora_delta_merge" or name == "lora_delta_grad":
        w = A["base"] if name == "lora_delta_merge" else A["dw"]
        Co, KH, KW, Ci = w.shape
        return {"kind": name, "Cout": Co, "Cin": Ci, "k": KH, "r": A["A"].shape[0] // KH, "conv3d": int(bool(A["conv3d"])),
                "scaling": float(A["scaling"])}, None
    if name == "scale_cast_f32_bf16":
        return {"kind": name, "workload": ctx.get("workload"), "n": A["src"].numel(), "world": ctx["world"]}, None
    raise KeyError(name)


def _key(rec):
    return json.dumps({k: v for k, v in rec.items() if k not in LABELS}, sort_keys=True)


def _optimizers(ctx, workload, groups, arena, variants, lr=5e-6, weight_decay=1e-2):
    """Builds each (class, ema, g16) variant over `groups` with train.main's constructor defaults (`lr`, `weight_decay`: the
    run's learning_rate and adam_weight_decay) and runs one launch() (and, with EMA, ema_weights()) under the recorders."""
    import torch

    from t2v_b200 import optim as O
    for cls, ema, g16 in variants:
        opt = getattr(O, cls)(arena, groups, lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=weight_decay, max_grad_norm=MAX_NORM,
                              ema_decay=EMA_DECAY if ema else None)
        ctx["tables"].add(opt)
        ctx.update(workload=workload, variant=f"{cls}{'+ema' if ema else ''}{'+g16' if g16 else ''}", opt=opt, arena=arena)
        comm = torch.zeros(arena.total, device=arena.master.device, dtype=torch.bfloat16) if g16 else None
        opt.launch(zero_grad=True, grad_bf16=comm)
        if ema:
            with opt.ema_weights():
                pass


def _buckets(ctx, workload, unet, arena):
    """GradientBuckets' compression pieces of one step at each world size: every block range as the backward marks it, then
    finish()."""
    import torch.distributed as dist

    from t2v_b200.runtime import GradientBuckets

    class _Done:
        def wait(self):
            return None

    saved = dist.all_reduce
    dist.all_reduce = lambda *a, **k: _Done()
    try:
        for world in WORLDS:
            b = GradientBuckets(arena, unet, compress=True)
            b.world = world
            ctx.update(workload=workload, variant=None, world=world)
            b.armed = True
            for key in sorted(b.ranges, key=lambda k: -b.ranges[k][0]):   # the backward reaches the last block first
                b.on_block_done(key)
            b.finish()
    finally:
        dist.all_reduce = saved


def _full_variants():
    return [(cls, ema, g16) for cls in ("FusedAdamW", "AdamW8bit") for ema in (False, True) for g16 in (False, True)]


def run_workloads(observe=None):
    """Runs every workload with the census kinds recorded; returns ([distinct records in first-call order], {sha256: host
    table}).  `observe(name, fn) -> fn`: when given, every public prims function (after the recorders) is wrapped by it."""
    import torch

    import make_attn_launches as MA
    import make_glue_launches as MG
    from helpers import emulated_prims
    from t2v_b200 import ops, prims

    seen, keys, tables = [], set(), {}
    ctx = {"tables": _Tables()}
    signatures = {n: inspect.signature(getattr(prims, n)) for n in KINDS}   # the native entry points' argument names

    def recorder(name, fn):
        sig = signatures[name]

        def run(*args, **kw):
            bound = sig.bind(*args, **kw)
            bound.apply_defaults()
            rec, t = _record(name, bound.arguments, ctx)
            k = _key(rec)
            if k not in keys:
                keys.add(k)
                seen.append(rec)
            if t is not None:
                tables.setdefault(rec["sha256"], t)
            if name in ("lora_delta_merge", "lora_delta_grad"):
                return fn(*args, **kw)
            return None
        return run

    def merge_alloc(base, A, B, scaling, conv3d):
        return torch.zeros(base.shape, dtype=torch.bfloat16, device=base.device)

    def nothing(*args, **kw):
        return None

    public = [n for n, v in vars(prims).items() if callable(v) and not n.startswith("_") and getattr(v, "__module__", None) == prims.__name__]
    saved = [(prims, n, getattr(prims, n)) for n in dict.fromkeys(MG.PATCHED_PRIMS + KINDS + tuple(public))]
    saved += [(ops, n, getattr(ops, n)) for n in MA.PATCHED_OPS]
    saved_flash, saved_epochs = ops._Flash.enabled, dict(ops._epochs)
    try:
        with emulated_prims(), torch.random.fork_rng(devices=[]), contextlib.redirect_stdout(io.StringIO()):
            for name, fn in MA._gemm_allocators(prims).items():
                setattr(prims, name, fn)
            for name, fn in MG.stand_ins().items():
                setattr(prims, name, fn)
            prims.lora_delta_merge, prims.lora_delta_grad = merge_alloc, nothing
            MA.Recorder().install(prims, ops)
            for name in KINDS:
                setattr(prims, name, recorder(name, getattr(prims, name)))
            if observe is not None:
                for name in public:
                    setattr(prims, name, observe(name, getattr(prims, name)))
            ops._Flash.enabled = True

            unet, _, groups, arena = _setup(trainable_modules=["all"])
            _optimizers(ctx, "full", groups, arena, _full_variants())
            _buckets(ctx, "full", unet, arena)
            del unet, groups, arena

            _, _, groups, arena = _setup(trainable_modules=["all"], use_unet_lora=True, use_text_lora=True)
            _optimizers(ctx, "train_config", groups, arena, [("FusedAdamW", False, False)], weight_decay=0.0)
            del groups, arena

            unet, groups, arena = _bench_lora()
            _optimizers(ctx, "lora", groups, arena, [("FusedAdamW", False, False)])
            _buckets(ctx, "lora", unet, arena)
            del unet, groups, arena

            unet, _, groups, arena = _setup(use_unet_lora=True, lora_version="stable_lora", lr=2e-5)
            ctx.update(workload="stable_lora", variant=None)
            _stable_pass(unet)
            _optimizers(ctx, "stable_lora", groups, arena, [("FusedAdamW", False, False), ("AdamW8bit", True, False)], lr=2e-5,
                        weight_decay=0.0)
            del unet, groups, arena

            _, _, groups, arena = _setup(trainable_modules=["all"], use_unet_lora=True, use_text_lora=True, train_text_encoder=True,
                                         trainable_text_modules=["all"], extra_unet_params={"lr": 1e-5, "weight_decay": 1e-4})
            _optimizers(ctx, "text_train", groups, arena, [("FusedAdamW", False, False)], weight_decay=0.0)
            del groups, arena
    finally:
        for mod, n, fn in saved:
            setattr(mod, n, fn)
        ops._Flash.enabled = saved_flash
        ops._epochs.clear()
        ops._epochs.update(saved_epochs)
    return seen, tables


# ---------------------------------------------------------------------------------------------- synthetic launches
SYNTH_8BIT = ((4160, 8), (65856, 8), (1024, 32), (4224, 8), (4288, 8))   # (elements, bits) of five tensors, arena order
SYNTH_SHADOW_AT = 3                                                    # tensors 3 and 4 lie past n_shadow

# (conv3d, k, Cin, Cout, r): conv_in / conv_out (4 channels), the ms-1.7b levels up to 2560 -> 1280, ranks 4..64, ragged sizes
MERGE_SHAPES = [
    (False, 3, 4, 320, 16), (False, 3, 320, 4, 16), (False, 1, 640, 320, 4), (False, 1, 2560, 1280, 16),
    (False, 3, 1280, 1280, 16), (False, 3, 2560, 1280, 64), (False, 3, 37, 100, 5), (False, 1, 33, 7, 3),
    (True, 3, 320, 320, 16), (True, 3, 1280, 1280, 64), (True, 3, 41, 19, 4),
]


def synth_8bit_rows(ema):
    """AdamW8bit's rows over SYNTH_8BIT: 8-bit tensors whose last 256-block holds 64, 64 (a second 65,536-element row then a
    320-element one), 128 and 192 elements, one fp32 tensor; with ema the EMA offset (the compact EMA in arena order)."""
    rows, off, s8, s32, e = [], 0, 0, 0, 0
    for n, bits in SYNTH_8BIT:
        for lo in range(0, n, 1 << 16):
            r = [off + lo, min(1 << 16, n - lo), (s8 if bits == 8 else s32) + lo, bits]
            rows.append(r + ([e + lo] if ema else []))
        off += n
        e += n
        if bits == 8:
            s8 += -(-n // 256) * 256
        else:
            s32 += n
    return rows, off, s8, s32


def synthetic():
    """Live kernel paths no recorded workload reaches:
      the ragged 8-bit blocks (every 8-bit row of the full UNet covers whole 256-element blocks): SYNTH_8BIT, two sets' worth of
        tensors in one launch (8-bit and fp32 rows, rows past n_shadow), without EMA reading fp32 gradients and with EMA reading
        the bf16 twin;
      lora_delta_merge / lora_delta_grad at the MERGE_SHAPES the stable-LoRA step does not produce (scaling 0.75 / 1.5);
      adamw_prepare over two hyper-parameter sets (every workload above makes one: train.main gives the text-encoder and LoRA
        groups the UNet's extra_unet_params, so their hyper-parameters coincide)."""
    out = [{"kind": "adamw_prepare", "n_sets": 2, "max_norm": MAX_NORM, "synthetic": 1}]
    for kind, ema in (("adamw8bit_chunks", False), ("adamw8bit_ema_chunks", True)):
        rows, total, s8, s32 = synth_8bit_rows(ema)
        n_shadow = sum(n for n, _ in SYNTH_8BIT[:SYNTH_SHADOW_AT])
        rec = {"kind": kind, "workload": "synthetic", "variant": None, "cols": 5 if ema else 4, "g16": int(ema),
               "hp": [1e-3, 0.9, 0.999, 1e-8, 1e-2]}
        if ema:
            rec["ema_decay"] = 0.7
        rec.update(n_rows=len(rows), total=total, n_shadow=n_shadow, n_state=s32, n_state8=s8, n_ema=total if ema else 0,
                   rows=rows, synthetic=1)
        out.append(rec)
    for conv3d, k, ci, co, r in MERGE_SHAPES:
        geo = {"Cout": co, "Cin": ci, "k": k, "r": r, "conv3d": int(conv3d)}
        out.append({"kind": "lora_delta_merge", **geo, "scaling": 0.75, "synthetic": 1})
        out.append({"kind": "lora_delta_grad", **geo, "scaling": 1.5, "synthetic": 1})
    return out


def step_launches():
    """The distinct launches of the workloads plus the synthetic ones."""
    seen, _ = run_workloads()
    keys = {_key(r) for r in seen}
    for r in synthetic():
        plain = {k: v for k, v in r.items() if k != "synthetic"}
        assert _key(plain) not in keys, f"a workload already reaches the synthetic launch {plain}"
        seen.append(r)
    return seen


_TABLES = {}


def tables():
    """{sha256: int64 host table} of every recorded table (built once per process)."""
    if not _TABLES:
        _TABLES.update(run_workloads()[1])
    return _TABLES


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
