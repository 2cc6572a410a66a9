"""Resumable training state (`save_training_state`, `resume_from_checkpoint`): everything a stopped `train.main` run needs
to continue bit for bit, written next to a checkpoint as `<checkpoint>/training_state/`:

  manifest.json   rank 0: world size, lora_version, optimizer kind, use_ema, the trainable (name, shape) list in arena order,
                  global_step and epoch - what a resume checks before it loads anything
  shared.pt       rank 0: the trainable fp32 master weights by name (the exact arena bits, not the fp16 / merged export
                  files), the optimizer state (moments or 8-bit codes and absmax, fp32 small-tensor moments, the EMA, the
                  device step count; torch AdamW's state_dict with fused_adamw False), the LR scheduler's step count
  rank{r}.pt      every rank: the CPU / CUDA / `random` / numpy RNG states, the dropout epoch, the data position (the
                  epoch's shuffle seed and items consumed, items waiting in ShapeGroupedBatches' buffers) and the CPU
                  generator state at the start of each CUDA-graph capture

The folder is written as `training_state.tmp/` by all ranks (a barrier between the writes and the rename) and renamed into
place by rank 0, so a run killed while saving leaves no folder that looks complete.  Every rank must see the same file
system.  Checkpoints are written at optimizer-step boundaries only: the accumulation window is closed and the fused
optimizer has zeroed the gradients."""
import json
import os
import random
import shutil

import numpy as np
import torch
import torch.distributed as dist

from . import ops

STATE_DIR = "training_state"
MANIFEST = "manifest.json"


def _barrier(world):
    if world > 1:
        dist.barrier()


def _cpu(obj):
    if torch.is_tensor(obj):
        return obj.detach().cpu()
    if isinstance(obj, dict):
        return {k: _cpu(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_cpu(v) for v in obj)
    return obj


def trainable_names(stepper):
    """(name, param) of every trainable arena parameter in arena order; text-encoder LoRA factors are prefixed."""
    names = {id(p): "unet." + n for n, p in stepper.unet.named_parameters()}
    if stepper.text_encoder is not None:
        names.update((id(p), "text_encoder." + n) for n, p in stepper.text_encoder.named_parameters() if id(p) not in names)
    return [(names[id(p)], p) for p in stepper.arena.params if p.requires_grad]


def optimizer_kind(optimizer):
    from .optim import AdamW8bit, FusedAdamW
    if isinstance(optimizer, AdamW8bit):
        return "adamw8bit"
    return "fused_adamw" if isinstance(optimizer, FusedAdamW) else "torch_adamw"


def _spans(arena):
    return [(lo, hi) for lo, hi in arena.trainable_spans if hi > lo]


def _optimizer_state(optimizer, arena):
    """FusedAdamW's fp32 moments cover the whole arena, frozen ranges included (zero forever): keep the trainable spans."""
    if optimizer_kind(optimizer) == "torch_adamw":
        return {"torch": _cpu(optimizer.state_dict())}
    fused = optimizer.state_dict()["fused"]
    out = {"step": int(fused["step"])}
    for name, t in fused.items():
        if name == "step":
            continue
        out[name] = [t[lo:hi].cpu() for lo, hi in _spans(arena)] if t.numel() == arena.total else t.cpu()
    return out


def _load_optimizer_state(optimizer, arena, state):
    if "torch" in state:
        saved = state["torch"]
        # the moments come from the state; the hyper-parameters (lr, betas, weight decay, ...) from the new config
        groups = [dict(g_saved, **{k: v for k, v in g.items() if k != "params"})
                  for g_saved, g in zip(saved["param_groups"], optimizer.param_groups)]
        optimizer.load_state_dict({"state": saved["state"], "param_groups": groups})
        return
    mine = optimizer.state_dict()["fused"]
    with torch.no_grad():
        for name, t in mine.items():
            if name == "step":
                continue
            if isinstance(state[name], list):
                for (lo, hi), part in zip(_spans(arena), state[name]):
                    t[lo:hi].copy_(part)
            else:
                t.copy_(state[name])
    optimizer.state_dev.fill_(state["step"])


def _rng_state(device):
    np_state = np.random.get_state()
    d = {"torch": torch.get_rng_state(), "random": random.getstate(),
         "numpy": (np_state[0], torch.from_numpy(np_state[1].copy()), *np_state[2:])}
    if device.type == "cuda":
        d["cuda"] = torch.cuda.get_rng_state(device)
    return d


def restore_rng(state, device):
    torch.set_rng_state(state["torch"])
    random.setstate(state["random"])
    name, keys, *rest = state["numpy"]
    np.random.set_state((name, keys.numpy(), *rest))
    if "cuda" in state and device.type == "cuda":
        torch.cuda.set_rng_state(state["cuda"], device)


def manifest(world, lora_version, optimizer, use_ema, stepper, global_step, epoch):
    return {"world_size": world, "lora_version": lora_version, "optimizer": optimizer_kind(optimizer), "use_ema": bool(use_ema),
            "trainables": [[n, list(p.shape)] for n, p in trainable_names(stepper)], "global_step": global_step, "epoch": epoch}


def save(path, *, rank, world, man, stepper, optimizer, sched, order, loader):
    """Write `<path>/training_state/` (collective: every rank calls it at the same step)."""
    if stepper._micro % stepper.accumulation:
        raise RuntimeError("training state saved inside an accumulation window")
    arena = stepper.arena
    if optimizer_kind(optimizer) != "torch_adamw" and optimizer.covers_all_trainable():
        # the update kernel consumed and zeroed every trainable gradient: nothing of the window is lost
        assert all(int(torch.count_nonzero(arena.grad[lo:hi])) == 0 for lo, hi in _spans(arena)), "gradients are not zero"
    tmp, final = os.path.join(path, STATE_DIR + ".tmp"), os.path.join(path, STATE_DIR)
    if rank == 0:
        shutil.rmtree(tmp, ignore_errors=True)
        os.makedirs(tmp)
    _barrier(world)
    dev = arena.master.device
    data = {"order": order.state_dict()}
    if hasattr(loader, "state_dict"):
        data["grouper"] = loader.state_dict()
    torch.save({"rng": _rng_state(dev), "dropout_epoch": int(ops.dropout_epoch(dev).item()), "data": data,
                "capture_rng": list({**stepper.replay_rng, **stepper.capture_rng}.items())}, os.path.join(tmp, f"rank{rank}.pt"))
    if rank == 0:
        torch.save({"weights": {n: p.detach().cpu() for n, p in trainable_names(stepper)},
                    "optimizer": _optimizer_state(optimizer, arena), "scheduler": sched.state_dict()},
                   os.path.join(tmp, "shared.pt"))
        with open(os.path.join(tmp, MANIFEST), "w") as f:
            json.dump(man, f, indent=1)
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)
    _barrier(world)
    if rank == 0:
        old = final + ".old"
        if os.path.isdir(final):
            shutil.rmtree(old, ignore_errors=True)
            os.rename(final, old)
        os.rename(tmp, final)
        shutil.rmtree(old, ignore_errors=True)
    _barrier(world)
    return final


def is_complete(state_dir):
    """True when `state_dir` holds a manifest and the shared and per-rank files it implies."""
    try:
        with open(os.path.join(state_dir, MANIFEST)) as f:
            world = int(json.load(f)["world_size"])
    except (OSError, ValueError, KeyError):
        return False
    return all(os.path.isfile(os.path.join(state_dir, n)) for n in ["shared.pt"] + [f"rank{r}.pt" for r in range(world)])


def latest(output_dir):
    """The checkpoint folder (a `checkpoint-N/` or `output_dir` itself) with the complete state of the highest step, or None."""
    if not os.path.isdir(output_dir):
        return None
    found = []
    for d in [output_dir] + [os.path.join(output_dir, n) for n in os.listdir(output_dir) if n.startswith("checkpoint-")]:
        s = os.path.join(d, STATE_DIR)
        if is_complete(s):
            with open(os.path.join(s, MANIFEST)) as f:
                found.append((int(json.load(f)["global_step"]), d == output_dir, d))
    return max(found)[2] if found else None


def check(man, want):
    """ValueError unless the saved run and this one agree on what the state's layout depends on."""
    for key, what in (("world_size", "world size"), ("optimizer", "optimizer"), ("use_ema", "use_ema")):
        if man[key] != want[key]:
            raise ValueError(f"cannot resume: the saved state has {what} {man[key]!r}, this run {want[key]!r}")
    if man["trainables"] != want["trainables"]:
        saved, mine = {n: s for n, s in man["trainables"]}, {n: s for n, s in want["trainables"]}
        diff = sorted(set(saved) ^ set(mine))[:3] or [n for n in mine if saved.get(n) != mine[n]][:3] or ["(order)"]
        raise ValueError(f"cannot resume: the trainable parameters differ from the saved state's ({len(saved)} saved, "
                         f"{len(mine)} here; e.g. {diff})")


def read_manifest(state_dir):
    with open(os.path.join(state_dir, MANIFEST)) as f:
        return json.load(f)


def load(state_dir, *, rank, stepper, optimizer, sched, order, loader):
    """Load a checked state into this run (weights, optimizer, scheduler, dropout epoch, data position, capture states).
    Returns this rank's RNG states: the caller restores them once the first epoch's data iterator exists (a DataLoader
    draws its base seed from the CPU generator when the iterator is made)."""
    shared = torch.load(os.path.join(state_dir, "shared.pt"), map_location="cpu", weights_only=True)
    mine = torch.load(os.path.join(state_dir, f"rank{rank}.pt"), map_location="cpu", weights_only=True)
    arena = stepper.arena
    with torch.no_grad():
        for n, p in trainable_names(stepper):
            p.copy_(shared["weights"][n])
    arena.refresh_shadow()   # the bf16 compute copy (and the stable-LoRA merges made from it) see the restored weights
    _load_optimizer_state(optimizer, arena, shared["optimizer"])
    # the step count only: the schedule itself (warm-up, total, kind, base LR) is the new config's
    sched.last_epoch = int(shared["scheduler"]["last_epoch"])
    lrs = [base * f(sched.last_epoch) for base, f in zip(sched.base_lrs, sched.lr_lambdas)]
    for g, lr in zip(optimizer.param_groups, lrs):
        g["lr"] = lr
    sched._last_lr = lrs
    ops.dropout_epoch(arena.master.device).fill_(int(mine["dropout_epoch"]))
    order.resume(mine["data"]["order"])
    if "grouper" in mine["data"]:
        loader.load_state_dict(mine["data"]["grouper"])
    stepper.replay_rng = {tuple(k): v for k, v in mine["capture_rng"]}
    return mine["rng"]
