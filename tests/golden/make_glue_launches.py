#!/usr/bin/env python
"""Regenerates tests/golden/glue_launches.json: every distinct launch of the glue kernels of csrc/elementwise.cu (layout,
loss, noise, embedding, bias-gradient, fan-in, resampling and cast kernels) in the training steps, the text-encoder steps,
the VAE encode and the data-side resize.  Fields (those that select a code path or a shape):
  latents_to_nhwc8        B, C, F, H, W; noise: add_noise fused (then B timesteps are read)
  nhwc8_to_latents        B, C, F, H, W
  mse_loss_* / velocity_mse_loss_*   B, C, F, H, W of the target
  timestep_embedding      B (one timestep per sample), dim
  colsum                  S (row-bias segments; 1 for a plain bias), P rows per segment, C, blocks = ceil(C / 4096): the
                          column blocks of t2v_colsum (every block after the first starts at col0 > 0)
  colsum_f32              S, C
  upsample_nearest_*      N, H, W, Ho, Wo, C
  concat_channels         M rows, Ca, Cb;  split_channels  M, Ct, Ca
  add_bf16                n, inputs (2 or 3);  add_f32  n;  scale_bf16  n, alpha
  cast_f32_bf16           n, into (1: into a given buffer);  cast_bf16_f32  n
  dropout_scale_add       n, p, scale, base (1: forward with a base, 0: the backward)
  embed_tokens            B, L, C, vocab, pos_rows;  embed_tokens_bwd  the same plus dtok / dpos (which tables accumulate)
  gelu_bf16 / gelu_bwd    n, quick (CLIP's quick_gelu, else the erf form)
  vae_sample              B, F, h, w, scale
  frames_u8_to_nhwc8      F, H0, W0, h, w;  frames_u8_to_nhwc8_ragged  clips [[F, H0, W0], ..], h, w
Every output that accumulates (colsum, colsum_f32, embed_tokens_bwd) always does: the census records no flag for it.
Workloads, all through the real model code:
  cfg2, lora, zeroscope, image (4 x 1 frame at 64 x 64 latents), batch2 (2 x 16 frames), as tests/golden/make_attn_launches.py
  vpred       the cfg2 step with prediction_type v_prediction, and the image batch with it (the velocity loss at B = 4)
  text_lora   the use_text_lora encoder forward and backward (1 x 77 tokens)
  text_train  train_text_encoder with every module trainable: embed_tokens_bwd into both tables, and the cfg2 step on its
              states (the fp32 fan-in of their gradient)
  vae         AutoencoderKL encode of one 16-frame 256^2 batch
  resize      utils.dataset.frames_to_latents of 4-frame clips: 1280x720 -> 576x320 and 480x640 -> 256x256 (one clip each),
              and one ragged batch of both sizes -> 256x256 (the ragged kernel), each followed by the VAE encode and vae_sample
plus synthetic launches (marked "synthetic": 1) of live paths no workload reaches (synthetic()): colsum at C = 10240 (the GEGLU
projection width, whose bias gradient is a plain colsum when the weight is frozen and the bias trains; no recorded step reaches
C > 4096): three column blocks, the last one 2048 wide; nhwc8_to_latents of a returned prediction; scale_bf16 of a LoRA branch
with scale != 1; quick_gelu; embed_tokens_bwd with the token table frozen.
Everything runs on the meta device over oracle/ops_ref.py (the data-side batches: uint8 frames on meta, the ragged table on the
CPU), the GEMM and attention prims replaced by allocators as in make_attn_launches.py, and the prims the oracle lacks
(gelu_bwd, embed_tokens_bwd, velocity_mse_loss_*, frames_u8_to_nhwc8_ragged) by local stand-ins that only allocate.
step_launches() leaves every prims / ops function, the dropout epochs and the CPU random state as it found them.
Records are deduplicated by their whole content, in first-call order.
Counts (235 launches, 6 of them synthetic): 6 latents_to_nhwc8 (5 with add_noise), 1 nhwc8_to_latents, 5 + 5 mse_loss_fwd /
_bwd, 2 + 2 velocity_mse_loss_fwd / _bwd, 3 timestep_embedding, 25 colsum (8 with S > 1 row-bias segments, 1 past the first
column block), 9 colsum_f32, 15 + 15 upsample_nearest_fwd / _bwd, 32 concat_channels, 32 split_channels, 43 add_bf16 (6 of them
3-input), 1 add_f32, 1 scale_bf16, 20 cast_f32_bf16, 1 cast_bf16_f32, 4 dropout_scale_add, 1 embed_tokens, 2 embed_tokens_bwd,
2 gelu_bf16, 2 gelu_bwd, 3 vae_sample, 2 frames_u8_to_nhwc8, 1 frames_u8_to_nhwc8_ragged.
tests/test_glue_step_gpu.py runs every launch; tests/test_glue_step_cpu.py checks that this script reproduces the table.
  python tests/golden/make_glue_launches.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
OUT = os.path.join(ROOT, "tests", "golden", "glue_launches.json")

KINDS = ("latents_to_nhwc8", "nhwc8_to_latents", "mse_loss_fwd", "mse_loss_bwd", "velocity_mse_loss_fwd", "velocity_mse_loss_bwd",
         "timestep_embedding", "colsum", "colsum_f32", "upsample_nearest_fwd", "upsample_nearest_bwd", "concat_channels",
         "split_channels", "add_bf16", "add_f32", "scale_bf16", "cast_f32_bf16", "cast_bf16_f32", "dropout_scale_add",
         "embed_tokens", "embed_tokens_bwd", "gelu_bf16", "gelu_bwd", "vae_sample", "frames_u8_to_nhwc8",
         "frames_u8_to_nhwc8_ragged")
COLSUM_BLOCK = 4096   # t2v_colsum's column block
RESIZE_FRAMES = 4


def _arg(args, kw, i, key, default=None):
    return args[i] if len(args) > i else kw.get(key, default)


def _lat(shape):
    B, C, F, H, W = shape
    return {"B": B, "C": C, "F": F, "H": H, "W": W}


def record(name, args, kw):
    """The launch record of prims.<name>(*args, **kw) (without "kind")."""
    a = lambda i, key, default=None: _arg(args, kw, i, key, default)   # noqa: E731
    if name == "latents_to_nhwc8":
        return {**_lat(args[0].shape), "noise": int(a(1, "noise") is not None)}
    if name == "nhwc8_to_latents":
        x, B, C, F = args[0], a(1, "B"), a(2, "C"), a(3, "F")
        return {"B": B, "C": C, "F": F, "H": x.shape[1], "W": x.shape[2]}
    if name in ("mse_loss_fwd", "mse_loss_bwd", "velocity_mse_loss_fwd", "velocity_mse_loss_bwd"):
        return _lat(args[1].shape)
    if name == "timestep_embedding":
        return {"B": args[0].shape[0], "dim": a(1, "dim")}
    if name == "colsum":
        S, P, C = a(2, "S"), a(3, "P"), a(4, "C")
        return {"S": S, "P": P, "C": C, "blocks": -(-C // COLSUM_BLOCK)}
    if name == "colsum_f32":
        return {"S": args[0].shape[0], "C": args[0].shape[1]}
    if name == "upsample_nearest_fwd":
        N, H, W, C = args[0].shape
        Ho, Wo = a(1, "out_hw_")
        return {"N": N, "H": H, "W": W, "Ho": Ho, "Wo": Wo, "C": C}
    if name == "upsample_nearest_bwd":
        N, Ho, Wo, C = args[0].shape
        H, W = a(1, "in_hw")
        return {"N": N, "H": H, "W": W, "Ho": Ho, "Wo": Wo, "C": C}
    if name == "concat_channels":
        x, y = args[0], args[1]
        return {"M": x.numel() // x.shape[-1], "Ca": x.shape[-1], "Cb": y.shape[-1]}
    if name == "split_channels":
        g = args[0]
        return {"M": g.numel() // g.shape[-1], "Ct": g.shape[-1], "Ca": a(1, "Ca")}
    if name == "add_bf16":
        return {"n": args[0].numel(), "inputs": 3 if a(2, "c") is not None else 2}
    if name in ("add_f32", "cast_bf16_f32"):
        return {"n": args[0].numel()}
    if name == "scale_bf16":
        return {"n": args[0].numel(), "alpha": float(a(1, "alpha"))}
    if name == "cast_f32_bf16":
        return {"n": args[0].numel(), "into": int(a(1, "dst") is not None)}
    if name == "dropout_scale_add":
        return {"n": args[0].numel(), "p": float(a(2, "p")), "scale": float(a(3, "scale")), "base": int(a(1, "base") is not None)}
    if name == "embed_tokens":
        ids, tok, pos = args[0], args[1], args[2]
        return {"B": ids.shape[0], "L": ids.shape[1], "C": tok.shape[1], "vocab": tok.shape[0], "pos_rows": pos.shape[0]}
    if name == "embed_tokens_bwd":
        ids, dy, dtok, dpos, vocab = args[0], args[1], a(2, "dtok"), a(3, "dpos"), a(4, "vocab")
        return {"B": ids.shape[0], "L": ids.shape[1], "C": dy.shape[1], "vocab": int(vocab),
                "pos_rows": dpos.shape[0] if dpos is not None else 0, "dtok": int(dtok is not None), "dpos": int(dpos is not None)}
    if name in ("gelu_bf16", "gelu_bwd"):
        return {"n": args[0].numel(), "quick": int(bool(a(1 if name == "gelu_bf16" else 2, "quick", False)))}
    if name == "vae_sample":
        m = args[0]
        return {"B": a(2, "B"), "F": a(3, "F"), "h": m.shape[1], "w": m.shape[2], "scale": float(a(4, "scale"))}
    if name == "frames_u8_to_nhwc8":
        F, H0, W0, _ = args[0].shape
        h, w = a(1, "out_hw")
        return {"F": F, "H0": H0, "W0": W0, "h": h, "w": w}
    if name == "frames_u8_to_nhwc8_ragged":
        h, w = a(2, "out_hw")
        return {"clips": [[int(v) for v in row[1:]] for row in args[1].tolist()], "h": h, "w": w}
    raise KeyError(name)


def stand_ins():
    """Allocating stand-ins for the glue prims oracle/ops_ref.py does not state, and for dropout_scale_add (the oracle reads the
    dropout epoch back, which the meta device cannot)."""
    import torch

    def gelu_bwd(x, dy, quick=False):
        return torch.zeros_like(dy)

    def embed_tokens_bwd(ids, dy, dtok, dpos, vocab):
        return None

    def velocity_mse_loss_fwd(pred, x0, noise, alphas_cumprod, timesteps):
        return torch.zeros((), device=pred.device)

    def velocity_mse_loss_bwd(pred, x0, noise, alphas_cumprod, timesteps, gout):
        return torch.zeros_like(pred)

    def frames_u8_to_nhwc8_ragged(packed, table, out_hw):
        return torch.zeros((int(table[:, 1].sum()), out_hw[0], out_hw[1], 8), dtype=torch.bfloat16, device=packed.device)

    def dropout_scale_add(x, base, p, scale, seed, epoch=None):
        return x if base is None else base + x

    return {"gelu_bwd": gelu_bwd, "embed_tokens_bwd": embed_tokens_bwd, "velocity_mse_loss_fwd": velocity_mse_loss_fwd,
            "velocity_mse_loss_bwd": velocity_mse_loss_bwd, "frames_u8_to_nhwc8_ragged": frames_u8_to_nhwc8_ragged,
            "dropout_scale_add": dropout_scale_add}


def _text_train():
    """train_text_encoder with trainable_text_modules 'all': every encoder parameter trains, the embeddings included, and its
    states feed the cfg-2 UNet step (their gradient fans in from every cross-attention in fp32: cast_bf16_f32, add_f32)."""
    import torch

    import bench
    import make_attn_launches as MA
    from t2v_b200.text_encoder import CLIPTextModel
    dev = torch.device("meta")
    with dev:
        te = CLIPTextModel()
    te.requires_grad_(True)
    text = te.encode(torch.zeros(1, 77, dtype=torch.int64, device=dev)).float().view(1, 77, -1)
    w = bench.WORKLOADS["cfg2"]
    MA._unet_step(1, w["frames"], w["latent_hw"], text=text)


def _resize():
    """The data side: frames_to_latents (resize kernel, VAE encode, vae_sample) of one clip per fixed source size and of one
    ragged batch of both."""
    import torch

    from t2v_b200.utils import dataset as D
    from t2v_b200.vae import AutoencoderKL
    dev = torch.device("meta")
    with dev:
        vae = AutoencoderKL()
    F = RESIZE_FRAMES
    for (H0, W0), (h, w) in (((720, 1280), (320, 576)), ((640, 480), (256, 256))):
        batch = {"frames_u8": torch.zeros(1, F, H0, W0, 3, dtype=torch.uint8, device=dev), "pixel_hw": torch.tensor([[h, w]])}
        D.frames_to_latents(batch, vae, dev)
    sizes = ((720, 1280), (640, 480))
    offs = [0, F * 720 * 1280 * 3]
    table = torch.tensor([[o, F, H0, W0] for o, (H0, W0) in zip(offs, sizes)], dtype=torch.int64)
    nbytes = sum(F * H0 * W0 * 3 for H0, W0 in sizes)
    batch = {D.PACKED_KEY: torch.zeros(nbytes, dtype=torch.uint8, device=dev), D.TABLE_KEY: table,
             "pixel_hw": torch.tensor([[256, 256], [256, 256]])}
    D.frames_to_latents(batch, vae, dev)


def synthetic():
    """Live kernel paths no recorded workload reaches:
      colsum at the GEGLU projection width (C = 10240: column blocks 0, 4096, 8192), 1024 rows: the bias gradient of a frozen
        proj weight at the 1280-channel level of a 16-frame 32 x 32 step (8 x 8 tokens x 16 frames);
      nhwc8_to_latents of the cfg-2 prediction (finetune_loss(return_pred=True): validation and sampling);
      scale_bf16 of a cloneofsimo LoRA up-projection gradient with lora scale 0.5 and no dropout (the first-level 320-channel
        linear of a cfg-2 step);
      gelu_bf16 / gelu_bwd in CLIP's quick_gelu form (a quick_gelu encoder, CLIP ViT-L/14: 77 tokens x 3072);
      embed_tokens_bwd into the position table alone (trainable_text_modules that leave the token table frozen)."""
    return [{"kind": "colsum", "S": 1, "P": 1024, "C": 10240, "blocks": 3, "synthetic": 1},
            {"kind": "nhwc8_to_latents", "B": 1, "C": 4, "F": 16, "H": 32, "W": 32, "synthetic": 1},
            {"kind": "scale_bf16", "n": 16 * 32 * 32 * 320, "alpha": 0.5, "synthetic": 1},
            {"kind": "gelu_bf16", "n": 77 * 3072, "quick": 1, "synthetic": 1},
            {"kind": "gelu_bwd", "n": 77 * 3072, "quick": 1, "synthetic": 1},
            {"kind": "embed_tokens_bwd", "B": 1, "L": 77, "C": 1024, "vocab": 49408, "pos_rows": 77, "dtok": 0, "dpos": 1, "synthetic": 1}]


PATCHED_PRIMS = tuple(dict.fromkeys(KINDS + ("flash_attn_fwd", "flash_attn_bwd", "attn_small_fwd", "attn_small_bwd", "attn_long_fwd",
                                             "attn_long_bwd", "conv_fwd", "conv_dgrad", "conv_wgrad", "bgemm")))


def run_workloads(observe=None):
    """Runs every census workload with the glue prims recorded; returns the distinct records in first-call order.
    `observe(name, fn) -> fn`: when given, every public prims function (after the census's own replacements) is wrapped by it,
    so a caller sees every prims call the workloads make."""
    import torch

    import bench
    import make_attn_launches as MA
    from helpers import emulated_prims
    from t2v_b200 import ops, prims

    seen, keys = [], set()

    def add(rec):
        key = json.dumps(rec, sort_keys=True)
        if key not in keys:
            keys.add(key)
            seen.append(rec)

    def recorder(name, fn):
        def run(*args, **kw):
            add({"kind": name, **record(name, args, kw)})
            return fn(*args, **kw)
        return run

    public = [n for n, v in vars(prims).items() if callable(v) and not n.startswith("_") and getattr(v, "__module__", None) == prims.__name__]
    saved = [(prims, n, getattr(prims, n)) for n in dict.fromkeys(PATCHED_PRIMS + tuple(public))]
    saved += [(ops, n, getattr(ops, n)) for n in MA.PATCHED_OPS]
    saved_flash, saved_epochs = ops._Flash.enabled, dict(ops._epochs)
    try:
        with emulated_prims(), torch.random.fork_rng(devices=[]):
            for name, fn in MA._gemm_allocators(prims).items():
                setattr(prims, name, fn)
            for name, fn in stand_ins().items():
                setattr(prims, name, fn)
            MA.Recorder().install(prims, ops)
            for name in KINDS:
                setattr(prims, name, recorder(name, getattr(prims, name)))
            if observe is not None:
                for name in public:
                    setattr(prims, name, observe(name, getattr(prims, name)))
            ops._Flash.enabled = True
            for wl in ("cfg2", "lora", "zeroscope"):
                w = bench.WORKLOADS[wl]
                MA._unet_step(1, w["frames"], w["latent_hw"], lora=bool(w["lora_rank"]))
            MA._unet_step(4, 1, (64, 64))
            MA._unet_step(2, 16, (32, 32))
            w = bench.WORKLOADS["cfg2"]
            MA._unet_step(1, w["frames"], w["latent_hw"], prediction_type="v_prediction")
            MA._unet_step(4, 1, (64, 64), prediction_type="v_prediction")
            MA._text_step()
            _text_train()
            MA._vae_encode()
            _resize()
    finally:
        for mod, n, fn in saved:
            setattr(mod, n, fn)
        ops._Flash.enabled = saved_flash
        ops._epochs.clear()   # drops the meta device's dropout epoch
        ops._epochs.update(saved_epochs)
    return seen


def step_launches():
    """The distinct glue launches of the workloads above plus the synthetic ones, as {"kind": ..., **fields}."""
    seen = run_workloads()
    keys = {json.dumps(r, sort_keys=True) for r in seen}
    for r in synthetic():
        plain = {k: v for k, v in r.items() if k != "synthetic"}
        assert json.dumps(plain, sort_keys=True) not in keys, f"a workload already reaches the synthetic launch {plain}"
        seen.append(r)
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
