"""`save_training_state` / `resume_from_checkpoint` on the emulated primitives (deterministic on the CPU): N steps in one
go against K steps, a new `train.main` resumed from the saved state, and N - K more.  Weights, optimizer state, EMA and
every micro-step's loss must be bitwise those of the uninterrupted run."""
import json
import math
import os
import random
import shutil
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from ema_ref import emulated as ema_emulated   # emulated primitives, 8-bit AdamW and the EMA kernels included
from helpers import emulated_prims, seeded_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = dict(block_out_channels=(32, 64, 64, 64), attention_head_dim=32, cross_attention_dim=32)


def _unet_folder(root):
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    m.load_state_dict(seeded_state_dict(m, 0))
    m.save_pretrained(os.path.join(root, "unet"))
    return root


def _record_losses(monkeypatch):
    from t2v_b200 import step as S
    seen, orig = [], S.DataParallelStep.__call__

    def call(self, *args):
        loss = orig(self, *args)
        seen.append(float(loss))
        return loss
    monkeypatch.setattr(S.DataParallelStep, "__call__", call)
    return seen


def _main(**kw):
    """One train.main run from a fresh process-wide state: the dropout epoch counter and the `random` / numpy streams
    (train.main seeds torch only) start where a new process would have them."""
    from t2v_b200 import ops, train
    for t in ops._epochs.values():
        t.zero_()
    random.seed(0)
    np.random.seed(0)
    return train.main(**kw)


def _bits(r):
    """Everything that must continue bit for bit: the arena master (trainable and frozen) and the optimizer state."""
    opt = r["optimizer"]
    d = {"master": r["stepper"].arena.master.detach().cpu().clone()}
    if hasattr(opt, "state_dev"):
        for k, v in opt.state_dict()["fused"].items():
            d[k] = v.detach().cpu().clone() if torch.is_tensor(v) else v
    else:
        for i, s in opt.state_dict()["state"].items():
            d.update({f"{i}.{k}": v.detach().cpu().clone() for k, v in s.items()})
    return d


def _assert_same(a, b):
    assert a.keys() == b.keys(), (sorted(a), sorted(b))
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def _synthetic(root, **extra):
    kw = dict(pretrained_model_path=root, dataset_types=["synthetic"], train_data=dict(n=3, n_sample_frames=2, height=64, width=64),
              learning_rate=1e-3, checkpointing_steps=1, seed=0, shuffle=False, device="cpu", max_grad_norm=1.0,
              use_unet_lora=True, lora_version="cloneofsimo", lora_rank=4, unet_lora_modules=["UNet3DConditionModel"],
              lora_unet_dropout=0.1, save_pretrained_model=False)
    kw.update(extra)
    return kw


def _resume_matches(tmp_path, monkeypatch, ctx, kw, n, k, target="final"):
    """Runs N, then K + resume to N; asserts the two trajectories are bitwise equal and returns the K run's output dir."""
    losses = _record_losses(monkeypatch)
    part = str(tmp_path / "part")
    with ctx():
        full = _main(**kw, output_dir=str(tmp_path / "full"), max_train_steps=n)
        want = list(losses)
        del losses[:]
        _main(**kw, output_dir=part, max_train_steps=k, save_training_state=True)
        first = list(losses)
        del losses[:]
        src = {"final": part, "checkpoint": os.path.join(part, f"checkpoint-{k}")}.get(target, target)
        resumed = _main(**kw, output_dir=part, max_train_steps=n, resume_from_checkpoint=src)
    assert len(want) >= n and all(math.isfinite(v) for v in want)
    assert first + losses == want, (first, losses, want)
    assert resumed["steps"] == n
    _assert_same(_bits(full), _bits(resumed))
    return part


# ------------------------------------------------------------------------------------------------ bitwise continuation
@pytest.mark.parametrize("case", ["fp32_ema_shuffle_epoch", "adamw8bit_ema", "accumulation", "torch_adamw"])
def test_resume_is_bitwise(tmp_path, monkeypatch, case):
    root = _unet_folder(str(tmp_path / "model"))
    extra = {
        # 2 items: the epoch boundary falls between K = 1 and N = 3; warm-up runs across the resume
        "fp32_ema_shuffle_epoch": dict(use_ema=True, ema_decay=0.9, shuffle=True, lr_scheduler="constant_with_warmup", lr_warmup_steps=2,
                                       train_data=dict(n=2, n_sample_frames=2, height=64, width=64)),
        # full finetune: the 32 x 32 attention matrices keep fp32 moments, the larger feed-forward ones get 8-bit codes
        "adamw8bit_ema": dict(use_8bit_adam=True, use_ema=True, use_unet_lora=False, trainable_modules=["attn1", "attn2", "ff.net"]),
        "accumulation": dict(gradient_accumulation_steps=2),
        "torch_adamw": dict(fused_adamw=False, shuffle=True),
    }[case]
    n, k = 3, 1
    part = _resume_matches(tmp_path, monkeypatch, ema_emulated, _synthetic(root, **extra), n, k,
                           target="checkpoint" if case == "accumulation" else "final")
    man = json.load(open(os.path.join(part, "training_state", "manifest.json")))
    assert man["global_step"] == k and man["world_size"] == 1 and man["use_ema"] == bool(extra.get("use_ema"))
    if case == "adamw8bit_ema":
        assert man["optimizer"] == "adamw8bit"
        saved = torch.load(os.path.join(part, "training_state", "shared.pt"), weights_only=True)["optimizer"]
        assert saved["code_m"].numel() > 0 and saved["exp_avg32"].numel() > 0 and "ema" in saved


def test_resume_stable_lora(tmp_path, monkeypatch):
    import contextlib

    from stable_lora_ref import patched_prims

    @contextlib.contextmanager
    def ctx():
        with ema_emulated(), patched_prims():
            yield
    root = _unet_folder(str(tmp_path / "model"))
    _resume_matches(tmp_path, monkeypatch, ctx, _synthetic(root, lora_version="stable_lora", use_ema=True), 3, 1)


def test_resume_text_lora_raw_video(tmp_path, monkeypatch):
    """cloneofsimo UNet + text-encoder LoRA on raw videos: frame windows drawn with `random`, prompts through the step."""
    from test_dataset import _write_video
    from test_pipeline_train import _pipeline_folder
    from text_lora_ref import emulated
    root = _pipeline_folder(str(tmp_path / "pipe"))
    vids = tmp_path / "vids"
    vids.mkdir()
    for i in range(2):
        _write_video(str(vids / f"v{i}.mp4"), n=10, hw=(64, 64))
    kw = _synthetic(root, dataset_types=["folder"], use_text_lora=True, lora_text_dropout=0.1, load_side_models=True,
                    shuffle=True, unet_lora_modules=["UNet3DConditionModel"], text_encoder_lora_modules=["CLIPEncoderLayer"],
                    train_data=dict(width=64, height=64, n_sample_frames=2, fps=8, path=str(vids), fallback_prompt="a video"))
    threads = torch.get_num_threads()
    torch.set_num_threads(1)   # on several threads two identical runs of this case can differ in the last bits
    try:
        _resume_matches(tmp_path, monkeypatch, emulated, kw, 3, 1)
    finally:
        torch.set_num_threads(threads)


def test_resume_batch_two_keeps_buffered_items(tmp_path, monkeypatch):
    """Batch 2 over 3 videos and 2 images in order: at step 2 the third video waits in the grouper's buffer; the state
    holds it, and the resumed run pairs it with the next epoch's first video."""
    import contextlib

    from oracle import ops_ref
    from ragged_ref import emulated_ragged
    from test_batch_cpu import _media, _pipe

    @contextlib.contextmanager
    def ctx():
        old = ops_ref.BF
        ops_ref.BF = torch.float32
        try:
            with emulated_prims(), emulated_ragged():
                yield
        finally:
            ops_ref.BF = old
    root = _pipe(str(tmp_path / "pipe"))
    vids, imgs = _media(str(tmp_path), [(48, 64), (40, 24), (48, 64)], n_images=2)
    kw = _synthetic(root, dataset_types=["folder", "image"], train_batch_size=2, load_side_models=True,
                    train_data=dict(width=32, height=32, n_sample_frames=2, fps=8, path=vids, image_dir=imgs, fallback_prompt="a clip"))
    part = _resume_matches(tmp_path, monkeypatch, ctx, kw, 3, 2, target="checkpoint")
    rank0 = torch.load(os.path.join(part, "checkpoint-2", "training_state", "rank0.pt"), weights_only=True)
    buffers = rank0["data"]["grouper"]["buffers"]
    assert [len(items) for _, items in buffers] == [1] and "frames_u8" in buffers[0][1][0]
    assert rank0["data"]["order"]["consumed"] == 5


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _rank_worker(rank, world, port, tmp, root, result):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank),
                      T2V_GRAD_COMPRESS="0")
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ema_ref import emulated as emu
    from t2v_b200 import step as S
    losses, orig = [], S.DataParallelStep.__call__

    def call(self, *args):
        loss = orig(self, *args)
        losses.append(float(loss))
        return loss
    S.DataParallelStep.__call__ = call
    kw = _synthetic(root, shuffle=True, use_ema=True, train_data=dict(n=4, n_sample_frames=2, height=64, width=64))
    out = {}
    with emu():
        full = _main(**kw, output_dir=os.path.join(tmp, "full"), max_train_steps=3)
        out["want"], losses[:] = list(losses), []
        _main(**kw, output_dir=os.path.join(tmp, "part"), max_train_steps=1, save_training_state=True)
        out["first"], losses[:] = list(losses), []
        resumed = _main(**kw, output_dir=os.path.join(tmp, "part"), max_train_steps=3, resume_from_checkpoint="latest")
        out["rest"] = list(losses)
    out["full"], out["resumed"] = _bits(full), _bits(resumed)
    torch.save(out, f"{result}.{rank}")
    dist.destroy_process_group()


def test_resume_two_gloo_ranks(tmp_path):
    root = _unet_folder(str(tmp_path / "model"))
    res = str(tmp_path / "res")
    port = 29500 + (os.getpid() * 11) % 2000
    mp.spawn(_rank_worker, args=(2, port, str(tmp_path), root, res), nprocs=2, join=True)
    got = [torch.load(f"{res}.{r}", weights_only=True) for r in range(2)]
    for g in got:
        assert len(g["want"]) == 3 and g["first"] + g["rest"] == g["want"]
        _assert_same(g["full"], g["resumed"])
    assert got[0]["want"] != got[1]["want"]   # each rank trains on its own items
    files = sorted(os.listdir(os.path.join(str(tmp_path), "part", "training_state")))
    assert files == ["manifest.json", "rank0.pt", "rank1.pt", "shared.pt"]


# ------------------------------------------------------------------------------------------------ latest, refusals, fallback
def test_latest_skips_an_incomplete_state(tmp_path, monkeypatch):
    from t2v_b200 import training_state as TS
    root = _unet_folder(str(tmp_path / "model"))
    kw = _synthetic(root)
    losses = _record_losses(monkeypatch)
    part = str(tmp_path / "part")
    with emulated_prims():
        _main(**kw, output_dir=part, max_train_steps=2, save_training_state=True)
        # a run killed while saving step 5, and one killed before the rename of step 6
        shutil.copytree(os.path.join(part, "checkpoint-2", "training_state"), os.path.join(part, "checkpoint-5", "training_state"))
        with open(os.path.join(part, "checkpoint-5", "training_state", "manifest.json"), "w") as f:
            json.dump(dict(json.load(open(os.path.join(part, "training_state", "manifest.json"))), global_step=5), f)
        os.remove(os.path.join(part, "checkpoint-5", "training_state", "shared.pt"))
        shutil.copytree(os.path.join(part, "checkpoint-2", "training_state"), os.path.join(part, "checkpoint-6", "training_state.tmp"))
        assert TS.latest(part) in (part, os.path.join(part, "checkpoint-2"))
        del losses[:]
        r = _main(**kw, output_dir=part, max_train_steps=3, resume_from_checkpoint="latest")
    assert r["steps"] == 3 and len(losses) == 1
    assert TS.latest(str(tmp_path / "nothing")) is None


def _refuse(tmp_path, monkeypatch, state_from, **kw):
    from t2v_b200 import step as S

    def no_step(*a, **k):
        raise AssertionError("a step ran before the refusal")
    monkeypatch.setattr(S.DataParallelStep, "__call__", no_step)
    with emulated_prims(), pytest.raises(ValueError) as e:
        _main(**{**kw, "output_dir": str(tmp_path / "again"), "max_train_steps": 3, "resume_from_checkpoint": state_from})
    return str(e.value)


def test_refusals(tmp_path, monkeypatch):
    root = _unet_folder(str(tmp_path / "model"))
    kw = _synthetic(root)
    part = str(tmp_path / "part")
    with emulated_prims():
        _main(**kw, output_dir=part, max_train_steps=1, save_training_state=True)
        _main(**kw, output_dir=str(tmp_path / "plain"), max_train_steps=1)
    assert "trainable parameters differ" in _refuse(tmp_path, monkeypatch, part, **{**kw, "lora_rank": 8})
    assert "optimizer" in _refuse(tmp_path, monkeypatch, part, **{**kw, "fused_adamw": False})
    assert "use_ema" in _refuse(tmp_path, monkeypatch, part, **{**kw, "use_ema": True})
    # a state written by two ranks
    state = os.path.join(part, "training_state")
    man = json.load(open(os.path.join(state, "manifest.json")))
    with open(os.path.join(state, "manifest.json"), "w") as f:
        json.dump(dict(man, world_size=2), f)
    shutil.copy(os.path.join(state, "rank0.pt"), os.path.join(state, "rank1.pt"))
    assert "world size" in _refuse(tmp_path, monkeypatch, part, **kw)
    # no state at all, and no resume_step
    msg = _refuse(tmp_path, monkeypatch, str(tmp_path / "plain"), **kw)
    assert os.path.join(str(tmp_path / "plain"), "training_state") in msg and "save_training_state" in msg


def test_resume_step_without_state_skips_batches(tmp_path, monkeypatch):
    """The reference's resume: no state to load, the first resume_step batches of the first epoch are skipped."""
    from t2v_b200 import step as S
    root = _unet_folder(str(tmp_path / "model"))
    kw = _synthetic(root, train_data=dict(n=4, n_sample_frames=2, height=64, width=64))
    seen, orig = [], S.DataParallelStep.__call__

    def call(self, latents, *a):
        seen.append(latents.detach().cpu().clone())
        return orig(self, latents, *a)
    monkeypatch.setattr(S.DataParallelStep, "__call__", call)
    with emulated_prims():
        _main(**kw, output_dir=str(tmp_path / "plain"), max_train_steps=1)
        r = _main(**kw, output_dir=str(tmp_path / "again"), max_train_steps=3, resume_from_checkpoint=str(tmp_path / "plain"),
                  resume_step=2)
    from t2v_b200.train import SyntheticLatents
    items = SyntheticLatents(n=4, frames=2, hw=(8, 8), text_dim=32)
    assert r["steps"] == 3 and r["optimizer"].steps == 3
    # items 2, 3 of epoch 1, then item 0 of epoch 2 (the skip is for the first epoch only)
    for got, i in zip(seen[1:], [2, 3, 0]):
        assert torch.equal(got[0], items[i]["pixel_values"])
