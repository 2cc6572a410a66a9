#!/usr/bin/env python
"""Regenerates tests/golden/attn_launches.json: every distinct launch of the attention kernels in the training steps and
encoders the product runs, forward and backward:
  flash_attn_fwd / flash_attn_bwd   Nb, Lq, Lk, heads, D; row pitches of q / k / v / o (and dO / dq / dk / dv); `fused`: q, k, v
                                    are column slices of one [.., 3C] QKV projection ("qkv"), k, v of one [.., 2C] K|V projection
                                    ("kv"), or separate matrices ("none"); backward: the dK/dV query-split count on 132 SMs
                                    (H100 SXM) and on 114 SMs (H100 PCIe), from splits() below
  attn_small_* / attn_long_*        the SeqAddr tuple `addr` = (nseq, inner, outer_rows, inner_rows, seq_rows, ld_in, ld_out,
                                    heads, L, D), the token rows of the buffers and `fused`
  composite                         the unfused bgemm / softmax / bgemm path (ops._attn_core_fwd / _bwd, causal_attention_fwd):
                                    the flash fields, `causal` (the causal_period of softmax_fwd, 0 for none) and `bwd` (whether
                                    a backward of it runs; then also the gradient pitches)
Workloads, all recorded through the real model code with the step's parameter arena (so the attention projections are fused
where the step fuses them):
  cfg2        bench.WORKLOADS["cfg2"]: 1 x 16 frames x 32 x 32 latents, full finetune
  lora        bench.WORKLOADS["lora"]: 1 x 16 x 40 x 72 with the bench's cloneofsimo LoRA (unfused q / k / v projections)
  zeroscope   bench.WORKLOADS["zeroscope"]: 1 x 24 x 40 x 72, full finetune
  image       4 single-frame 512^2 images (1 frame, 64 x 64 latents): its cross-attention at Lq = 4096, Lk = 77, Nb = 4 splits
              the dK/dV query range on both SM counts
  long48/64   1 x 48 and 1 x 64 frames at 32 x 32 (attn_long)
  batch2      2 x 16 frames x 32 x 32 (train_batch_size 2): temporal sequences of the second clip start outer_rows = F HW
              token rows in, the one SeqAddr term a single clip never uses
  text        the use_text_lora encoder forward and backward (text_encoder.DEFAULTS widths, 1 x 77 tokens)
  vae         AutoencoderKL encode of one 16-frame 256^2 batch, forward only (mid-block attention: 1 head, d = 512)
plus one synthetic attn_long launch at the kernel's limit L = 256 with the transformer_in geometry of DESIGN.md 3.2 (HW = 1024,
C = 512, 8 heads, fused QKV): a 256-frame step does not fit a card.
Everything runs on the meta device over oracle/ops_ref.py: the GEMMs and the attention prims are replaced by allocators, so
no value is computed and the census takes seconds.  step_launches() leaves the process as it found it: every prims / ops
function it replaces (PATCHED_PRIMS, PATCHED_OPS) is put back, and the CPU random state and the dropout epochs are restored,
so later tests in the same process run the real kernels on unchanged state.  Records are deduplicated by their whole content, in first-call order.
Counts: 55 flash_attn_fwd, 55 flash_attn_bwd (23 of them split the dK/dV query range on both 132 and 114 SMs), 20
attn_small_fwd, 20 attn_small_bwd, 11 attn_long_fwd, 11 attn_long_bwd, 2 composite (174 launches).
tests/test_attn_step_gpu.py runs every launch; tests/test_attn_step_cpu.py checks that this script reproduces the table.
  python tests/golden/make_attn_launches.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "attn_launches.json")

KINDS = ("flash_attn_fwd", "flash_attn_bwd", "attn_small_fwd", "attn_small_bwd", "attn_long_fwd", "attn_long_bwd", "composite")
SM_COUNTS = (132, 114)   # H100 SXM5, H100 PCIe
BM = BN = 64             # flash_attn.cu query / key block


def splits(Nb, heads, Lq, Lk, sms):
    """t2v_flash_attn_bwd_splits restated: the dK/dV kernel splits the query range when the key blocks alone leave SMs idle
    and there are at least 8 query blocks."""
    ctas = -(-Lk // BN) * heads * Nb
    nqb = -(-Lq // BM)
    if ctas >= sms or nqb < 8:
        return 1
    return min(-(-2 * sms // ctas), nqb // 4)


def _fused(q, k, C):
    if q.stride(-2) == 3 * C:
        return "qkv"
    if k.stride(-2) == 2 * C:
        return "kv"
    return "none"


def _rows3(t):
    """Row pitch of a [Nb, L, C] view whose batch stride is L rows (every attention operand of the product)."""
    assert t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1), (tuple(t.shape), t.stride())
    return t.stride(1)


def _core(q, k, v, heads):
    Nb, Lq, C = q.shape
    return {"Nb": Nb, "Lq": Lq, "Lk": k.shape[1], "heads": heads, "D": C // heads, "q_ld": _rows3(q), "k_ld": _rows3(k),
            "v_ld": _rows3(v), "fused": _fused(q, k, C)}


def _grads(do, dq, dk, dv):
    return {"do_ld": _rows3(do), "dq_ld": _rows3(dq), "dk_ld": _rows3(dk), "dv_ld": _rows3(dv)}


def _temporal(q, o, addr):
    C = addr[7] * addr[9]
    return {"addr": list(addr), "rows": q.shape[0], "fused": "qkv" if addr[5] == 3 * C else "none"}


class Recorder:
    def __init__(self):
        self.seen, self.keys, self.composite = [], set(), {}

    def add(self, rec):
        key = json.dumps(rec, sort_keys=True)
        if key not in self.keys:
            self.keys.add(key)
            self.seen.append(rec)

    def install(self, prims, ops):
        import torch

        def flash_fwd(q, k, v, heads):
            self.add({"kind": "flash_attn_fwd", **_core(q, k, v, heads), "o_ld": q.shape[2]})
            Nb, Lq, C = q.shape
            return torch.zeros((Nb, Lq, C), dtype=q.dtype, device=q.device), torch.zeros((Nb, heads, Lq), device=q.device)

        def flash_bwd(q, k, v, o, do, lse, heads, dq, dk, dv):
            rec = {"kind": "flash_attn_bwd", **_core(q, k, v, heads), "o_ld": _rows3(o), **_grads(do, dq, dk, dv)}
            rec.update({f"splits_{n}": splits(rec["Nb"], heads, rec["Lq"], rec["Lk"], n) for n in SM_COUNTS})
            self.add(rec)

        def small_fwd(q, k, v, o, addr):
            self.add({"kind": "attn_small_fwd", **_temporal(q, o, addr)})
            return o

        def small_bwd(q, k, v, do, dq, dk, dv, addr):
            self.add({"kind": "attn_small_bwd", **_temporal(q, do, addr)})
            return dq, dk, dv

        def long_fwd(q, k, v, o, lse, addr):
            self.add({"kind": "attn_long_fwd", **_temporal(q, o, addr)})
            return o, lse

        def long_bwd(q, k, v, o, do, lse, dq, dk, dv, addr):
            self.add({"kind": "attn_long_bwd", **_temporal(q, do, addr)})
            return dq, dk, dv

        def composite_fwd(q, k, v, heads, causal):
            rec = {"kind": "composite", **_core(q, k, v, heads), "causal": causal, "bwd": 0}
            key = json.dumps(_core(q, k, v, heads), sort_keys=True)
            if key not in self.composite:
                self.composite[key] = rec
                self.seen.append(rec)
            Nb, Lq, C = q.shape
            ld = (k.shape[1] + 7) // 8 * 8
            return (torch.zeros((Nb, Lq, C), dtype=q.dtype, device=q.device),
                    torch.zeros((Nb, heads, Lq, ld), dtype=torch.bfloat16, device=q.device))

        real_core_fwd, real_core_bwd = ops._attn_core_fwd, ops._attn_core_bwd

        def core_fwd(q, k, v, heads):
            if ops._use_flash(q, heads):
                return real_core_fwd(q, k, v, heads)
            return composite_fwd(q, k, v, heads, 0)

        def core_bwd(q, k, v, p, do, dq, dk, dv, heads, o=None):
            if p.dtype == torch.float32 and p.dim() == 3:
                return real_core_bwd(q, k, v, p, do, dq, dk, dv, heads, o)
            rec = self.composite[json.dumps(_core(q, k, v, heads), sort_keys=True)]   # the forward of this backward
            rec.update(bwd=1, **_grads(do, dq, dk, dv))

        prims.flash_attn_fwd, prims.flash_attn_bwd = flash_fwd, flash_bwd
        prims.attn_small_fwd, prims.attn_small_bwd = small_fwd, small_bwd
        prims.attn_long_fwd, prims.attn_long_bwd = long_fwd, long_bwd
        ops._attn_core_fwd, ops._attn_core_bwd = core_fwd, core_bwd
        ops.causal_attention_fwd = lambda q, k, v, heads: composite_fwd(q, k, v, heads, q.shape[1])


def _gemm_allocators(prims):
    import torch

    def conv_fwd(x, w, bias=None, rowbias=None, residual=None, stride=1, pads=(0, 0, 0, 0), alpha=1.0, out_fp32=False,
                 rowbias_div=1, stats=None, stats_rows=0):
        Ho, Wo = prims.out_hw(x.shape[1], x.shape[2], w.shape[1], w.shape[2], stride, pads)
        return torch.zeros((x.shape[0], Ho, Wo, w.shape[0]), dtype=torch.float32 if out_fp32 else torch.bfloat16, device=x.device)

    def conv_dgrad(dy, w, in_hw, stride=1, pads=(0, 0, 0, 0), residual=None):
        return torch.zeros((dy.shape[0], in_hw[0], in_hw[1], w.shape[3]), dtype=torch.bfloat16, device=dy.device)

    def nothing(*args, **kw):
        return None

    def dropout_scale_add(x, base, p, scale, seed, epoch=None):   # the oracle reads the dropout epoch back (no meta value)
        return x if base is None else base + x

    def gelu_bwd(x, dy, quick=False):   # not in the oracle (tests/text_lora_ref.py restates it)
        return torch.zeros_like(dy)

    return {"conv_fwd": conv_fwd, "conv_dgrad": conv_dgrad, "conv_wgrad": nothing, "bgemm": nothing,
            "dropout_scale_add": dropout_scale_add, "gelu_bwd": gelu_bwd}


def _unet_step(B, F, hw, lora=False, prediction_type="epsilon", text=None):
    """One training pass of the full-size UNet over the step's parameter arena (fused projections), as DataParallelStep
    runs it; `lora`: the bench's cloneofsimo rank-16 LoRA on every UNet linear (q / k / v then stay separate GEMMs);
    `prediction_type`: the loss target (the velocity loss of a v-prediction step); `text`: the text states (B, 77, 1024), by
    default frozen zeros (a trained text encoder hands states that need a gradient)."""
    import torch

    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.runtime import ParamArena
    from oracle import leaves as L
    dev = torch.device("meta")
    with dev:
        m = UNet3DConditionModel()
    if lora:
        from t2v_b200.utils.lora_handler import LoraHandler
        m.requires_grad_(False)
        h = LoraHandler(version="cloneofsimo", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
        with dev:
            h.add_lora_to_model(True, m, h.unet_replace_modules, 0.0, "", r=16)
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    ParamArena(m, device=dev)
    lat, noise = torch.zeros(B, 4, F, *hw, device=dev), torch.zeros(B, 4, F, *hw, device=dev)
    ehs = torch.zeros(B, 77, 1024, device=dev) if text is None else text
    loss = S.finetune_loss(m, lat, noise, torch.full((B,), 417, device=dev), ehs, L.ddpm_alphas_cumprod().to(dev),
                           prediction_type=prediction_type)
    loss.backward()


def _text_step():
    """The use_text_lora encoder: forward and backward into its LoRA factors (train.py's injection)."""
    import torch

    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils.lora import inject_trainable_lora_extended
    dev = torch.device("meta")
    with dev:
        te = CLIPTextModel()
        inject_trainable_lora_extended(te, {"CLIPEncoderLayer"}, r=16)
    out = te.encode(torch.zeros(1, 77, dtype=torch.int64, device=dev))
    out.float().sum().backward()


def _vae_encode():
    import torch

    from t2v_b200.vae import AutoencoderKL
    dev = torch.device("meta")
    with dev:
        vae = AutoencoderKL()
    with torch.no_grad():
        vae.encode_moments(torch.zeros(16, 3, 256, 256, device=dev))


def synthetic_long():
    """attn_long at L = 256: transformer_in of one 256-frame clip at 32 x 32 latents (HW 1024, C 512, fused QKV)."""
    from t2v_b200 import ops
    B, F, HW, heads, D = 1, 256, 1024, 8, 64
    addr = ops._temporal_addr(B, F, HW, heads, D, 3 * heads * D, heads * D)
    rec = {"addr": list(addr), "rows": B * F * HW, "fused": "qkv"}
    return [{"kind": "attn_long_fwd", **rec}, {"kind": "attn_long_bwd", **rec}]


# every prims / ops attribute the census replaces; all of them are restored when it returns
PATCHED_PRIMS = ("flash_attn_fwd", "flash_attn_bwd", "attn_small_fwd", "attn_small_bwd", "attn_long_fwd", "attn_long_bwd",
                 "conv_fwd", "conv_dgrad", "conv_wgrad", "bgemm", "dropout_scale_add", "gelu_bwd")
PATCHED_OPS = ("_attn_core_fwd", "_attn_core_bwd", "causal_attention_fwd")


def step_launches():
    """The distinct attention launches of the workloads above, in first call order, as {"kind": ..., **fields}."""
    import torch

    import bench
    from helpers import emulated_prims
    from t2v_b200 import ops, prims

    rec = Recorder()
    saved = [(prims, n, getattr(prims, n)) for n in PATCHED_PRIMS] + [(ops, n, getattr(ops, n)) for n in PATCHED_OPS]
    saved_flash, saved_epochs = ops._Flash.enabled, dict(ops._epochs)
    try:
        with emulated_prims(), torch.random.fork_rng(devices=[]):   # the model code draws dropout seeds and LoRA weights
            for name, fn in _gemm_allocators(prims).items():
                setattr(prims, name, fn)
            rec.install(prims, ops)
            ops._Flash.enabled = True
            for wl in ("cfg2", "lora", "zeroscope"):
                w = bench.WORKLOADS[wl]
                _unet_step(1, w["frames"], w["latent_hw"], lora=bool(w["lora_rank"]))
            _unet_step(4, 1, (64, 64))
            for F in (48, 64):
                _unet_step(1, F, (32, 32))
            _unet_step(2, 16, (32, 32))
            _text_step()
            _vae_encode()
    finally:
        for mod, n, fn in saved:
            setattr(mod, n, fn)
        ops._Flash.enabled = saved_flash
        ops._epochs.clear()   # drops the meta device's dropout epoch
        ops._epochs.update(saved_epochs)
    for r in synthetic_long():
        rec.add(r)
    return rec.seen


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
