"""`python train.py --config cfg.yaml` - the reference's training entry point on the H100-native hot path.

`main(**yaml)` accepts the same keyword surface as the reference's `train.py:457-514`, so the v2 YAML configs load
unchanged (keys this build does not act on - trackers, text-encoder options it refuses - are accepted and ignored).
What this file owns is the *step*: parameter selection (`handle_trainable_modules`, :316-337), LoRA injection through
`LoraHandler` (:557-572), optimizer parameter groups (`create_optimizer_params`, :205-236), and per optimisation step:
noise + timestep sampling (:751-757), the fused add_noise -> UNet fwd+bwd -> MSE step (`step.DataParallelStep`, two
passes per video step like :814-834), ONE gradient all-reduce across ranks, clipping, AdamW, LR schedule, LoRA / UNet
checkpoints.  One process per GPU (`torchrun --nproc-per-node N train.py --config ...`); no accelerate.

Data (SURVEY 8(f) rows 2-3): `dataset_types` in ('json', 'single_video', 'image', 'folder') build the reference's dataset
classes (utils/dataset.py: OpenCV decode -> ONE resize + normalise kernel on the GPU -> batched AutoencoderKL.encode);
`cache_latents: True` writes / `cached_latent_dir` reads the reference's latent cache (`cached_{i}.pt`, train.py:266-314);
`dataset_types: ['synthetic']` needs no files.  `train_batch_size` > 1 batches items of one (frames, height, width) group
(utils.dataset.ShapeGroupedBatches; batch size 1 keeps the plain DataLoader); with data parallelism every rank must then see
a single group.  Prompts go through the frozen CLIP text encoder (text_encoder.py) with a
per-prompt embedding cache; a batch that already carries `text_embeds` skips it.  `use_text_lora` (cloneofsimo only) injects
LoRA into the text encoder (train.py:571-572), `train_text_encoder` with `trainable_text_modules` unfreezes its parameters by
name (train.py:579-595, 763-773); either way the encoder runs inside the step on every batch's `prompt_ids` (step.py).
Checkpoints (8(f) row 4): LoRA in the cloneofsimo list format or the stable_lora safetensors files (full weights and the webui
file), the UNet in diffusers layout, and - when the pretrained folder
is a full pipeline - the complete pipeline directory (`save_pipe`, train.py:395-449), plus a validation sample every
`validation_steps` (sampling.py: DPM-Solver++ preview with the trained UNet in eval mode, train.py:908-958).
"""
import argparse
import contextlib
import itertools
import math
import os
import time
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist

from .models.unet_3d_condition import UNet3DConditionModel
from .ops import MAX_FRAMES
from .step import DataParallelStep, load_noise_schedule, loss_objective, sample_noise
from .utils.lora_handler import LORA_VERSIONS, LoraHandler

already_printed_trainables = False


def handle_trainable_modules(model, trainable_modules=None, is_enabled=True, negation=None):
    """requires_grad by name-substring match; 'all' unlocks everything; LoRA params are never touched here."""
    global already_printed_trainables
    if trainable_modules is None:
        return
    count = 0
    if any(name == "all" for name in trainable_modules):
        model.requires_grad_(True)
        count = len(list(model.parameters()))
    else:
        model.requires_grad_(False)
        for name, param in model.named_parameters():
            if "lora" not in name and any(tm in name for tm in trainable_modules):
                param.requires_grad_(is_enabled)
                count += 1
    if count > 0 and not already_printed_trainables:
        already_printed_trainables = True
        print(f"{count} params have been processed.")


def param_optim(model, condition, extra_params=None, is_lora=False, negation=None):
    extra_params = extra_params if extra_params and len(extra_params.keys()) > 0 else None
    return {"model": model, "condition": condition, "extra_params": extra_params, "is_lora": is_lora, "negation": negation}


def _group(name=None, param=None, lr=None, extra=None, params=None):
    g = {"params": params} if params is not None else {"name": name, "params": param, "lr": lr}
    if extra:
        g.update(extra)
    return g


def create_optimizer_params(model_list, lr):
    groups = []
    for spec in model_list:
        model, condition, extra, is_lora, _ = spec.values()
        if not condition:
            continue
        if is_lora and isinstance(model, list):  # list of parameter iterators from the injector
            groups.append(_group(params=itertools.chain(*model), extra=extra))
        elif is_lora:
            groups += [_group(n, p, lr, extra) for n, p in model.named_parameters() if "lora" in n]
        else:
            groups += [_group(n, p, lr, extra) for n, p in model.named_parameters() if "lora" not in n]
    return groups


def _lr_lambda(kind, warmup, total):
    """diffusers.optimization.get_scheduler semantics (train.py:626-631): plain 'constant' has no warm-up."""
    def f(step):
        if kind == "constant":
            return 1.0
        if step < warmup:
            return float(step) / max(1, warmup)
        if kind == "constant_with_warmup":
            return 1.0
        prog = (step - warmup) / max(1, total - warmup)
        if kind == "linear":
            return max(0.0, 1.0 - prog)
        if kind == "cosine":
            return 0.5 * (1.0 + math.cos(math.pi * min(1.0, prog)))
        raise ValueError(f"unknown lr_scheduler {kind!r}")
    return f


class CachedLatents(torch.utils.data.Dataset):
    """The reference's latent cache: cached_{i}.pt = {pixel_values: latents (4,F,h,w), prompt_ids, text_prompt, ...}
    (train.py:266-314, utils/dataset.py:589-603) plus an optional precomputed 'text_embeds' (77, 1024) entry."""

    def __init__(self, cache_dir):
        self.files = sorted(os.path.join(cache_dir, f) for f in os.listdir(cache_dir) if f.endswith(".pt"))
        if not self.files:
            raise FileNotFoundError(f"no cached_*.pt latents under {cache_dir}")

    def __len__(self):
        return len(self.files)

    def __getitem__(self, i):
        return torch.load(self.files[i], map_location="cpu")


class SyntheticLatents(torch.utils.data.Dataset):
    def __init__(self, n=64, frames=16, hw=(32, 32), text_len=77, text_dim=1024, seed=0):
        self.n, self.shape, self.tshape, self.seed = n, (4, frames, hw[0], hw[1]), (text_len, text_dim), seed

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 100003 + i)
        return {"pixel_values": torch.randn(self.shape, generator=g) * 0.18215, "text_embeds": torch.randn(self.tshape, generator=g)}


def needs_vae(batch, latent_source):
    """True when the batch holds pictures that still go through the VAE: raw frames (`frames_u8`, or a ragged batch packed by
    utils.dataset.collate_raw), or `pixel_values` from a dataset of pictures.  `pixel_values` of a latent source (the cache,
    the synthetic set) are latents.  Decided by keys and source, never by shape: a 4-frame pixel clip [B, 4, 3, h, w] and a
    latent clip [B, 4, 3, h, w] look alike."""
    from .utils.dataset import PACKED_KEY
    return "frames_u8" in batch or PACKED_KEY in batch or not latent_source


def handle_cache_latents(should_cache, output_dir, train_dataloader, vae, device, cached_latent_dir=None):
    """reference train.py:266-314: encode every item once and store it as cached_{i}.pt = {pixel_values: latents (4, F, h, w)
    fp16, prompt_ids, text_prompt, dataset} (the reference's `batch[k] = v[0]` item format).  Returns the cache directory
    (None when caching is off); an existing `cached_latent_dir` is used as is."""
    if not should_cache:
        return None
    if cached_latent_dir is not None:
        return os.path.abspath(cached_latent_dir)
    from .utils.dataset import frames_to_latents
    cache_save_dir = os.path.join(output_dir, "cached_latents")
    os.makedirs(cache_save_dir, exist_ok=True)
    for i, batch in enumerate(train_dataloader):
        latents = frames_to_latents(batch, vae, device)
        item = {"pixel_values": latents[0].to(torch.float16).cpu()}
        for k, v in batch.items():
            if k in ("frames_u8", "pixel_values", "pixel_hw"):
                continue
            v0 = v[0]
            item[k] = v0.reshape(-1) if (torch.is_tensor(v0) and k == "prompt_ids") else v0
        torch.save(item, os.path.join(cache_save_dir, f"cached_{i}.pt"))
    return cache_save_dir


class TextEmbedder:
    """prompt ids -> encoder_hidden_states through the frozen text encoder (train.py:784-790), cached per distinct prompt:
    a finetune run repeats a handful of prompts thousands of times."""

    def __init__(self, text_encoder, device, max_entries=4096):
        self.enc, self.device, self.cache, self.max = text_encoder, device, {}, max_entries

    def __call__(self, prompt_ids):
        ids = prompt_ids.reshape(-1, prompt_ids.shape[-1]).to(torch.int64).cpu()
        out = []
        for row in ids:
            key = row.numpy().tobytes()
            e = self.cache.get(key)
            if e is None:
                e = self.enc(row[None].to(self.device))[0][0]
                if len(self.cache) < self.max:
                    self.cache[key] = e
            out.append(e)
        return torch.stack(out)


def _load_optional(cls, root, subfolder):
    return cls.from_pretrained(root, subfolder=subfolder) if os.path.isfile(os.path.join(root, subfolder, "config.json")) else None


def main(
    pretrained_model_path: str,
    output_dir: str,
    train_data: Dict = None,
    validation_data: Dict = None,
    extra_train_data: list = [],
    dataset_types: Tuple[str] = ("json",),
    shuffle: bool = True,
    validation_steps: int = 100,
    trainable_modules: Tuple[str] = None,
    trainable_text_modules: Tuple[str] = None,
    extra_unet_params=None,
    extra_text_encoder_params=None,
    train_batch_size: int = 1,
    max_train_steps: int = 500,
    learning_rate: float = 5e-5,
    scale_lr: bool = False,
    lr_scheduler: str = "constant",
    lr_warmup_steps: int = 0,
    adam_beta1: float = 0.9,
    adam_beta2: float = 0.999,
    adam_weight_decay: float = 1e-2,
    adam_epsilon: float = 1e-08,
    max_grad_norm: float = 1.0,
    gradient_accumulation_steps: int = 1,
    gradient_checkpointing: bool = False,
    text_encoder_gradient_checkpointing: bool = False,
    checkpointing_steps: int = 500,
    resume_from_checkpoint: Optional[str] = None,
    resume_step: Optional[int] = None,
    mixed_precision: Optional[str] = "fp16",
    use_8bit_adam: bool = False,
    use_ema: bool = False,
    ema_decay: float = 0.9999,
    enable_xformers_memory_efficient_attention: bool = True,
    enable_torch_2_attn: bool = False,
    seed: Optional[int] = None,
    train_text_encoder: bool = False,
    use_offset_noise: bool = False,
    rescale_schedule: bool = False,
    offset_noise_strength: float = 0.1,
    extend_dataset: bool = False,
    cache_latents: bool = False,
    cached_latent_dir=None,
    lora_version: str = LORA_VERSIONS[0],
    save_lora_for_webui: bool = False,
    only_lora_for_webui: bool = False,
    lora_bias: str = "none",
    use_unet_lora: bool = False,
    use_text_lora: bool = False,
    unet_lora_modules: Tuple[str] = ("ResnetBlock2D",),
    text_encoder_lora_modules: Tuple[str] = ("CLIPEncoderLayer",),
    save_pretrained_model: bool = True,
    lora_rank: int = 16,
    lora_path: str = "",
    lora_unet_dropout: float = 0.1,
    lora_text_dropout: float = 0.1,
    logger_type: str = "tensorboard",
    save_training_state: bool = False,
    snr_gamma: Optional[float] = None,
    loss_type: str = "l2",
    huber_schedule: str = "snr",
    huber_c: float = 0.1,
    **kwargs,
):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device(kwargs.get("device") or f"cuda:{local}")   # "device" is a test hook (CPU runs use emulated primitives)
    if dev.type == "cuda":
        torch.cuda.set_device(dev)
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    if train_text_encoder and trainable_text_modules is None:
        # the reference trains no text parameter then (the encoder stays frozen, train.py:543, 579): refuse, do not train nothing
        raise NotImplementedError("train_text_encoder needs trainable_text_modules (e.g. ['all']) to name the text-encoder "
                                  "parameters to train; use_text_lora with lora_version 'cloneofsimo' trains a LoRA of it")
    if use_text_lora and lora_version == "stable_lora":
        raise NotImplementedError("use_text_lora is implemented for lora_version 'cloneofsimo' only")
    # text_encoder_gradient_checkpointing is accepted and has no effect: the text activations are 77 tokens per prompt
    fused_adamw = bool(kwargs.get("fused_adamw", True))   # optim.FusedAdamW on the flat arena (SURVEY 8(f) row 1); False: torch AdamW
    if use_8bit_adam and not fused_adamw:
        raise ValueError("use_8bit_adam runs optim.AdamW8bit on the flat arena; it cannot be combined with fused_adamw=False")
    if use_ema:   # the EMA is updated inside the fused optimizer step (optim.FusedAdamW ema_decay)
        if not fused_adamw:
            raise ValueError("use_ema keeps the EMA inside the fused optimizer step; it cannot be combined with fused_adamw=False")
        from .optim import check_ema_decay
        check_ema_decay(ema_decay)
    # noise schedule and loss target of the checkpoint (train.py:119, 792-800); an unsupported config fails here, before any
    # weights move.  `rescale_schedule` stays a no-op: in the reference it never reaches add_noise (SURVEY H5).
    abar, prediction_type = load_noise_schedule(pretrained_model_path)
    # the objective (Min-SNR-gamma weighting, pseudo-Huber / smooth-L1 loss) is configuration, not training state: a resumed
    # run takes it from this call, like the learning rate
    objective = loss_objective(snr_gamma, loss_type, huber_schedule, huber_c)
    # temporal attention runs on clips of 1..256 frames (attn_small.cu); a longer clip fails here, not in the first step
    for section, key, data in (("train_data", "n_sample_frames", train_data), ("validation_data", "num_frames", validation_data)):
        frames = int((data or {}).get(key, 16))
        if frames > MAX_FRAMES:
            raise ValueError(f"{section}.{key} = {frames}: temporal attention supports at most {MAX_FRAMES} frames")
    if seed is not None:
        # model construction and LoRA initialisation (lora_down ~ N(0, 1/r)) must be identical on every rank: the reference
        # gets that from accelerate/DDP broadcasting rank 0's parameters at wrap time (train.py:661).  The per-rank stream
        # (noise, timesteps, dropout) is seeded after the model is built.
        torch.manual_seed(seed)
    if rank == 0:
        os.makedirs(output_dir, exist_ok=True)

    unet = UNet3DConditionModel.from_pretrained(pretrained_model_path, subfolder="unet")
    unet.requires_grad_(False)
    if scale_lr:
        learning_rate = learning_rate * gradient_accumulation_steps * train_batch_size * world

    lora_manager = LoraHandler(version=lora_version, use_unet_lora=use_unet_lora, use_text_lora=use_text_lora,
                               save_for_webui=save_lora_for_webui, only_for_webui=only_lora_for_webui,
                               unet_replace_modules=list(unet_lora_modules),
                               text_encoder_replace_modules=list(text_encoder_lora_modules), lora_bias=lora_bias)
    unet_lora_params, unet_negation = lora_manager.add_lora_to_model(use_unet_lora, unet, lora_manager.unet_replace_modules,
                                                                     lora_unet_dropout, lora_path, r=lora_rank)
    text_encoder = text_lora_params = text_negation = None
    text_trains = use_text_lora or train_text_encoder
    if text_trains:   # the text encoder, its LoRA and its trainable set must exist before the parameter arena is built
        from .text_encoder import CLIPTextModel
        switch = "use_text_lora" if use_text_lora else "train_text_encoder"
        text_encoder = _load_optional(CLIPTextModel, pretrained_model_path, "text_encoder")
        if text_encoder is None:
            raise FileNotFoundError(f"{switch} needs the text encoder of the pipeline: {pretrained_model_path}/text_encoder is missing")
        text_lora_params, text_negation = lora_manager.add_lora_to_model(use_text_lora, text_encoder,
                                                                         lora_manager.text_encoder_replace_modules,
                                                                         lora_text_dropout, lora_path, r=lora_rank)
        if train_text_encoder:   # train.py:768-773 (the reference applies it on the first step, before any update)
            handle_trainable_modules(text_encoder, trainable_text_modules, is_enabled=True, negation=text_negation)
            if not text_encoder.base_trains():
                raise ValueError(f"trainable_text_modules={list(trainable_text_modules)!r} matches no text-encoder parameter")
        text_encoder = text_encoder.to(dev).train()
    unet = unet.to(dev)
    unet.train()
    if kwargs.get("eval_train", False):  # train.py:779-781
        unet.eval()
        if text_encoder is not None:
            text_encoder.eval()
    handle_trainable_modules(unet, trainable_modules, is_enabled=True, negation=unet_negation)
    unet._set_gradient_checkpointing(gradient_checkpointing)

    extra_unet_params = extra_unet_params or {}
    # train.py:581-595: UNet, text encoder (train_text_encoder), text LoRA, UNet LoRA; the text-encoder and text LoRA groups
    # take extra_unet_params, as in the reference (SURVEY H4)
    groups = create_optimizer_params([
        param_optim(unet, trainable_modules is not None, extra_params=extra_unet_params, negation=unet_negation),
        param_optim(text_encoder, train_text_encoder, extra_params=extra_unet_params, negation=text_negation),
        param_optim(text_lora_params, use_text_lora, is_lora=True, extra_params={**{"lr": learning_rate}, **extra_unet_params}),
        param_optim(unet_lora_params, use_unet_lora, is_lora=True, extra_params={**{"lr": learning_rate}, **extra_unet_params}),
    ], learning_rate)

    abar = abar.to(dev)
    use_graph = bool(kwargs.get("use_cuda_graph", dev.type == "cuda"))   # replay the whole step as one CUDA graph (static shapes)
    stepper = DataParallelStep(unet, abar, passes=2, use_graph=use_graph, accumulation=gradient_accumulation_steps,
                               prediction_type=prediction_type, text_encoder=text_encoder, **objective._asdict())
    # parameters now live in the flat arena.  Every rank must start from rank 0's weights (DDP does this at wrap time).
    if world > 1:
        dist.broadcast(stepper.arena.master, src=0)
        stepper.arena.refresh_shadow()
    if seed is not None:
        torch.manual_seed(seed + rank)
    if fused_adamw:
        from .optim import AdamW8bit, FusedAdamW
        cls = AdamW8bit if use_8bit_adam else FusedAdamW
        optimizer = cls(stepper.arena, groups, lr=learning_rate, betas=(adam_beta1, adam_beta2), weight_decay=adam_weight_decay,
                        eps=adam_epsilon, max_grad_norm=max_grad_norm, ema_decay=ema_decay if use_ema else None)
        stepper.attach_optimizer(optimizer)   # the update (clip + AdamW + shadow refresh + grad zeroing) is part of the step graph
    else:
        optimizer = torch.optim.AdamW(groups, lr=learning_rate, betas=(adam_beta1, adam_beta2), weight_decay=adam_weight_decay,
                                      eps=adam_epsilon)
    # stepped once per OPTIMIZER step, so warm-up and total are counted in optimizer steps (the reference scales both by the
    # accumulation factor, train.py:626-631, because accelerate steps its scheduler on every micro-step)
    sched = torch.optim.lr_scheduler.LambdaLR(optimizer, _lr_lambda(lr_scheduler, lr_warmup_steps, max_train_steps))

    kinds = [dataset_types] if isinstance(dataset_types, str) else list(dataset_types)
    # frozen side models, loaded only when the pretrained folder has them (a UNet-only folder trains from latents + embeddings)
    vae = tokenizer = None
    if dev.type == "cuda" or kwargs.get("load_side_models"):
        from .text_encoder import CLIPTextModel
        from .vae import AutoencoderKL
        vae = _load_optional(AutoencoderKL, pretrained_model_path, "vae")
        if vae is not None:
            vae = vae.to(dev).eval()
        if text_encoder is None:
            text_encoder = _load_optional(CLIPTextModel, pretrained_model_path, "text_encoder")
            if text_encoder is not None:
                text_encoder = text_encoder.to(dev).eval()
        if os.path.isdir(os.path.join(pretrained_model_path, "tokenizer")):
            from transformers import CLIPTokenizer
            tokenizer = CLIPTokenizer.from_pretrained(pretrained_model_path, subfolder="tokenizer")
    # a text encoder that trains is run by the step on every batch: no embedding cache
    embed_text = TextEmbedder(text_encoder, dev) if text_encoder is not None and not text_trains else None
    if cached_latent_dir:
        dataset = CachedLatents(cached_latent_dir)
    elif "synthetic" in kinds:
        td = train_data or {}
        dataset = SyntheticLatents(n=td.get("n", 64), frames=td.get("n_sample_frames", 16),
                                   hw=(td.get("height", 256) // 8, td.get("width", 256) // 8),
                                   text_dim=unet.config.cross_attention_dim)
    else:
        from .utils.dataset import extend_datasets, get_train_dataset
        if vae is None:
            raise FileNotFoundError(f"dataset_types={kinds} need the VAE of the pipeline: {pretrained_model_path}/vae is missing")
        if tokenizer is None or text_encoder is None:
            raise FileNotFoundError(f"dataset_types={kinds} need {pretrained_model_path}/tokenizer and /text_encoder for the prompts")
        parts = get_train_dataset(kinds, train_data, tokenizer)
        for extra in extra_train_data or []:
            parts += get_train_dataset(kinds, extra, tokenizer)
        extend_datasets(parts, ["train_data", "frames", "image_dir", "video_files"], extend=extend_dataset)
        parts = [d for d in parts if len(d) > 0]
        if not parts:
            raise FileNotFoundError(f"dataset_types={kinds}: no training items found under {train_data}")
        dataset = torch.utils.data.ConcatDataset(parts)
        if cache_latents:   # encode once, then train from the cache (reference handle_cache_latents)
            if rank == 0:
                handle_cache_latents(True, output_dir, torch.utils.data.DataLoader(dataset, batch_size=1, shuffle=False), vae, dev)
            if world > 1:
                dist.barrier()
            dataset = CachedLatents(os.path.join(output_dir, "cached_latents"))
    # the cache and the synthetic set hold latents; every other source holds pictures (raw frames, or pixel_values in [-1, 1]
    # from a dataset built with device_preprocess=False) that still go through the VAE
    latent_source = isinstance(dataset, (CachedLatents, SyntheticLatents))
    sampler = torch.utils.data.distributed.DistributedSampler(dataset, world, rank, shuffle=shuffle) if world > 1 else None
    # the epoch's item order and position, recorded for a resume; the order is the plain sampler's
    from .utils.dataset import EpochOrder
    order = EpochOrder(sampler if sampler is not None else (
        torch.utils.data.RandomSampler(dataset) if shuffle else torch.utils.data.SequentialSampler(dataset)))
    if train_batch_size > 1:
        # items differ in shape (native sizes, buckets, images next to videos): batches of one shape group each
        from .utils.dataset import ShapeGroupedBatches
        loader = ShapeGroupedBatches(dataset, train_batch_size, order, single_key=world > 1,
                                     sync_device=dev if world > 1 and dist.get_backend() == "nccl" else None)
    else:
        loader = torch.utils.data.DataLoader(dataset, batch_size=train_batch_size, sampler=order)

    global_step, micro, epoch = 0, 0, 0
    from . import training_state as TS

    def state_manifest():
        return TS.manifest(world, lora_version, optimizer, use_ema, stepper, global_step, epoch)

    def save_state(path):
        TS.save(path, rank=rank, world=world, man=state_manifest(), stepper=stepper, optimizer=optimizer, sched=sched,
                order=order, loader=loader)

    resume_rng, skip_batches = None, 0
    target = _resume_target(resume_from_checkpoint, output_dir)
    if target is not None:
        state_dir = os.path.join(target, TS.STATE_DIR)
        if TS.is_complete(state_dir):
            saved = TS.read_manifest(state_dir)
            TS.check(saved, state_manifest())
            resume_rng = TS.load(state_dir, rank=rank, stepper=stepper, optimizer=optimizer, sched=sched, order=order, loader=loader)
            global_step = int(saved["global_step"])
            epoch = int(saved["epoch"]) - 1   # the loop below re-enters the saved epoch
            micro = stepper._micro = global_step * gradient_accumulation_steps
            if rank == 0:
                print(f"resumed from {state_dir} at step {global_step}")
        elif resume_step is not None:
            # the reference's resume (train.py:842-846): skip the first resume_step batches of the first epoch, load nothing
            skip_batches = int(resume_step)
        else:
            raise ValueError(f"resume_from_checkpoint={resume_from_checkpoint!r}: {state_dir} holds no complete training state; "
                             "train with save_training_state: True to write one next to every checkpoint (or give resume_step "
                             "to only skip batches, as the reference does)")
    t0 = time.time()
    step_times, t_iter = [], time.perf_counter()
    while global_step < max_train_steps:
        if sampler is not None:
            sampler.set_epoch(epoch)   # a new shuffle every epoch
        epoch += 1
        batches = iter(loader)
        if resume_rng is not None:   # after the iterator's own draw, which the uninterrupted run made before the checkpoint
            TS.restore_rng(resume_rng, dev)
            resume_rng = None
        for batch in batches:
            if skip_batches:
                skip_batches -= 1
                continue
            if needs_vae(batch, latent_source):
                from .utils.dataset import frames_to_latents
                latents = frames_to_latents(batch, vae, dev)        # raw clip -> resize/normalise kernel -> batched VAE encode
            else:
                latents = batch["pixel_values"].to(dev, torch.float32)
            if text_trains:   # the step encodes the token ids itself
                if "prompt_ids" not in batch:
                    raise ValueError(f"{switch} trains the text encoder, so every batch needs 'prompt_ids'; this one has "
                                     f"{sorted(batch)} (the synthetic dataset and a latent cache of text_embeds only have none)")
                text = batch["prompt_ids"].reshape(latents.shape[0], -1).to(dev, torch.int64)
            elif "text_embeds" in batch:
                text = batch["text_embeds"].to(dev, torch.float32)
            elif embed_text is not None and "prompt_ids" in batch:
                text = embed_text(batch["prompt_ids"])                # frozen CLIP text encoder, cached per prompt
            else:
                raise FileNotFoundError("batch has neither 'text_embeds' nor a text encoder to turn 'prompt_ids' into them "
                                        f"({pretrained_model_path}/text_encoder is missing)")
            noise = sample_noise(latents, offset_noise_strength, use_offset_noise and not rescale_schedule)
            timesteps = torch.randint(0, abar.shape[0], (latents.shape[0],), device=dev, dtype=torch.int64)
            # single-frame data breaks out after the first pass (train.py:832), video runs both, batch by batch
            stepper.passes = 1 if latents.shape[2] <= 1 else 2
            loss = stepper(latents, noise, timesteps, text)   # fused: on a window boundary this includes clip + AdamW
            micro += 1
            if micro % gradient_accumulation_steps:
                continue  # gradients keep accumulating in the flat buffer (loss scaled by 1 / accumulation)
            if fused_adamw:
                optimizer._opt_called = True   # the update ran inside the step (graph); keeps LambdaLR's order check quiet
            else:
                if max_grad_norm is not None:
                    torch.nn.utils.clip_grad_norm_([p for g in optimizer.param_groups for p in g["params"] if p.grad is not None], max_grad_norm)
                optimizer.step()
            sched.step()
            global_step += 1
            if kwargs.get("_time_steps"):   # test hook: synchronous wall time of the WHOLE iteration (data, noise, step, optimizer)
                torch.cuda.synchronize()
                now = time.perf_counter()
                step_times.append(now - t_iter)
                t_iter = now
            if rank == 0 and (global_step % 10 == 0 or global_step == 1):
                print(f"step {global_step}/{max_train_steps} loss {loss.item():.5f} ({(time.time() - t0) / global_step:.3f} s/step)")
            if rank == 0 and global_step % checkpointing_steps == 0:
                save_checkpoint(unet, lora_manager, output_dir, global_step, use_unet_lora, save_pretrained_model,
                                pretrained_model_path=pretrained_model_path, ema=optimizer if use_ema else None,
                                text_encoder=text_encoder if text_trains else None)
            if rank == 0 and validation_data and validation_steps and global_step % validation_steps == 0 and vae is not None \
                    and text_encoder is not None and tokenizer is not None and getattr(vae, "decoder", None) is not None:
                from .sampling import validation_sample
                with optimizer.ema_weights() if use_ema else contextlib.nullcontext(), \
                        _text_preview(text_encoder) if text_trains else contextlib.nullcontext():   # preview what a user would export
                    validation_sample(unet, vae, text_encoder, tokenizer, validation_data, os.path.join(output_dir, "samples"), global_step,
                                      batch.get("text_prompt", [""])[0] if isinstance(batch.get("text_prompt"), (list, tuple)) else "",
                                      dev, alphas_cumprod=abar, prediction_type=prediction_type)
            if save_training_state and global_step % checkpointing_steps == 0:
                save_state(os.path.join(output_dir, f"checkpoint-{global_step}"))
            if global_step >= max_train_steps:
                break
        skip_batches = 0   # the reference skips in the first epoch only
    if resume_rng is not None:   # resumed at or past max_train_steps: no epoch ran
        TS.restore_rng(resume_rng, dev)
    if world > 1:
        dist.barrier()
    if rank == 0:
        save_checkpoint(unet, lora_manager, output_dir, global_step, use_unet_lora, save_pretrained_model, final=True,
                        pretrained_model_path=pretrained_model_path, ema=optimizer if use_ema else None,
                        text_encoder=text_encoder if text_trains else None)
    if save_training_state:
        save_state(output_dir)
    return {"steps": global_step, "step_times": step_times, "stepper": stepper, "optimizer": optimizer}


def _resume_target(resume_from_checkpoint, output_dir):
    """The checkpoint folder to resume from: a `checkpoint-N/` folder or a final `output_dir`; "latest" / True: the one under
    output_dir with the complete training state of the highest step (None, a fresh start, when there is none yet)."""
    if resume_from_checkpoint is None or resume_from_checkpoint is False or resume_from_checkpoint == "":
        return None
    if resume_from_checkpoint is True or resume_from_checkpoint == "latest":
        from .training_state import latest
        found = latest(output_dir)
        if found is None:
            print(f"resume_from_checkpoint={resume_from_checkpoint!r}: no complete training state under {output_dir}; starting from step 0")
        return found
    return str(resume_from_checkpoint)


@contextlib.contextmanager
def _text_preview(text_encoder):
    """The validation preview encodes through the trained text encoder in eval mode (LoRA dropout off) and without a tape."""
    was = text_encoder.training
    text_encoder.eval()
    try:
        with torch.no_grad():
            yield
    finally:
        text_encoder.train(was)


PIPELINE_PARTS = ("vae", "text_encoder", "tokenizer", "scheduler")


def save_pipe(pretrained_model_path, unet, path, unet_state_dict=None):
    """reference save_pipe (train.py:395-449): a complete TextToVideoSDPipeline directory - the trained UNet in diffusers
    layout plus the frozen parts and model_index.json of the pretrained pipeline, so `from_pretrained(path)` of a diffusers
    pipeline (or train.main again) can load it.  A UNet-only pretrained folder yields a UNet-only checkpoint.
    unet_state_dict: written instead of unet.state_dict() (stable LoRA: the merged weights)."""
    import shutil
    os.makedirs(path, exist_ok=True)
    unet.save_pretrained(os.path.join(path, "unet"), state_dict=unet_state_dict)
    copied = []
    for part in PIPELINE_PARTS:
        src = os.path.join(pretrained_model_path, part)
        if os.path.isdir(src):
            shutil.copytree(src, os.path.join(path, part), dirs_exist_ok=True)
            copied.append(part)
    index = os.path.join(pretrained_model_path, "model_index.json")
    if os.path.isfile(index):
        shutil.copyfile(index, os.path.join(path, "model_index.json"))
    elif copied:
        import json
        with open(os.path.join(path, "model_index.json"), "w") as f:
            json.dump({"_class_name": "TextToVideoSDPipeline", "unet": ["diffusers", "UNet3DConditionModel"],
                       "vae": ["diffusers", "AutoencoderKL"], "text_encoder": ["transformers", "CLIPTextModel"],
                       "tokenizer": ["transformers", "CLIPTokenizer"], "scheduler": ["diffusers", "DDIMScheduler"]}, f, indent=2)
    return copied


def save_checkpoint(unet, lora_manager, output_dir, step, use_unet_lora, save_pretrained_model, final=False, pretrained_model_path=None,
                    ema=None, text_encoder=None):
    """LoRA files and, with save_pretrained_model, the pipeline directory.
      cloneofsimo: `lora/<step>_unet.pt` (list format).
      stable_lora: `lora/full_weights/<step>_lora_text_to_video_unet.safetensors` (fp32) unless only_lora_for_webui, and with
        save_lora_for_webui / only_lora_for_webui `lora/webui_<step>_lora_text_to_video.safetensors` (fp16, ModelScope keys).
        `unet/` holds the delta merged into the base weights under the plain keys, so it loads into a plain UNet with
        strict=True (the reference writes the lora_A / lora_B keys into unet/ as well, which a plain UNet load rejects).
    ema (`use_ema`): the optimizer holding the EMA of the weights; the EMA weights are then written as well: the LoRA files
    with an `_ema` suffix and (save_pretrained_model) `unet_ema/` in the diffusers UNet layout.
    text_encoder (`use_text_lora` / `train_text_encoder`): with LoRA injected, `lora/<step>_text_encoder.pt` (and `_ema`) in
    the same list format; with save_pretrained_model `text_encoder/model.safetensors` holding the trained encoder under the
    plain Hugging Face keys, any LoRA collapsed into its base weight (the reference writes the wrapper keys, which
    transformers.CLIPTextModel does not load as the trained encoder).  When the encoder's own weights train and ema is given,
    `text_encoder_ema/` holds the EMA weights in the same layout."""
    path = output_dir if final else os.path.join(output_dir, f"checkpoint-{step}")
    os.makedirs(path, exist_ok=True)
    stable = use_unet_lora and lora_manager.is_stable_lora()
    lora_dir = os.path.join(path, "lora")

    def save_lora(suffix=""):
        if text_encoder is not None and text_encoder.lora_injected():
            from .utils.lora import save_lora_weight
            os.makedirs(lora_dir, exist_ok=True)
            save_lora_weight(text_encoder, os.path.join(lora_dir, f"{step}_text_encoder{suffix}.pt"), lora_manager.text_encoder_replace_modules)
        if not use_unet_lora:
            return
        os.makedirs(lora_dir, exist_ok=True)
        if stable:
            lora_manager.save_stable_lora(unet, lora_dir, step, suffix=suffix)
        else:   # the reference saves the LoRA files and (save_pretrained_model) the pipeline: train.py:908-958
            from .utils.lora import save_lora_weight
            save_lora_weight(unet, os.path.join(lora_dir, f"{step}_unet{suffix}.pt"), lora_manager.unet_replace_modules)

    def unet_sd():
        if not stable:
            return None
        from .utils.stable_lora import merged_state_dict
        return merged_state_dict(unet)

    save_lora()
    if save_pretrained_model:
        if pretrained_model_path is not None:
            save_pipe(pretrained_model_path, unet, path, unet_state_dict=unet_sd())
        else:
            unet.save_pretrained(os.path.join(path, "unet"), state_dict=unet_sd())
        if text_encoder is not None and os.path.isdir(os.path.join(path, "text_encoder")):
            save_text_encoder(text_encoder, os.path.join(path, "text_encoder"))
    if ema is not None:
        with ema.ema_weights():
            save_lora("_ema")
            if save_pretrained_model:
                unet.save_pretrained(os.path.join(path, "unet_ema"), state_dict=unet_sd())
                if text_encoder is not None and text_encoder.base_trains() and os.path.isdir(os.path.join(path, "text_encoder")):
                    import shutil
                    ema_dir = os.path.join(path, "text_encoder_ema")
                    os.makedirs(ema_dir, exist_ok=True)
                    shutil.copyfile(os.path.join(path, "text_encoder", "config.json"), os.path.join(ema_dir, "config.json"))
                    save_text_encoder(text_encoder, ema_dir)


def save_text_encoder(text_encoder, te_dir):
    """The encoder's current weights as `te_dir/model.safetensors` under the plain Hugging Face keys (next to the config.json
    save_pipe copied); a pretrained `pytorch_model.bin` there is removed, so the folder holds one set of weights."""
    from safetensors.torch import save_file
    if os.path.isfile(os.path.join(te_dir, "pytorch_model.bin")):
        os.remove(os.path.join(te_dir, "pytorch_model.bin"))
    save_file(text_encoder.plain_state_dict(), os.path.join(te_dir, "model.safetensors"), metadata={"format": "pt"})


def load_config(path):
    import yaml
    with open(path) as f:
        return yaml.safe_load(f)


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--config", type=str, default="./configs/v2/train_config.yaml")
    main(**load_config(parser.parse_args().config))
