"""train_batch_size > 1 on raw data, host side: `collate_raw` packing, the shape-grouping iterator, the raw-or-latent decision,
and `train.main` at batch 2 over the emulated primitives (one rank, and two gloo ranks)."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from helpers import emulated_prims, seeded_state_dict
from ragged_ref import emulated_ragged

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = dict(block_out_channels=(32, 64, 64, 64), attention_head_dim=32, cross_attention_dim=32)


def _item(F, H0, W0, hw, seed, prompt="p"):
    g = torch.Generator().manual_seed(seed)
    return {"frames_u8": torch.randint(0, 256, (F, H0, W0, 3), generator=g, dtype=torch.uint8), "pixel_hw": torch.tensor(hw),
            "prompt_ids": torch.full((1, 77), seed, dtype=torch.int64), "text_prompt": prompt, "dataset": "folder"}


def test_collate_raw_packs_clips_of_different_native_sizes():
    from t2v_b200.utils import dataset as D
    items = [_item(3, 17, 23, (16, 16), 0, "a"), _item(3, 40, 30, (16, 16), 1, "b"), _item(3, 9, 64, (16, 16), 2, "c")]
    b = D.collate_raw(items)
    packed, table = b[D.PACKED_KEY], b[D.TABLE_KEY]
    assert packed.dtype == torch.uint8 and packed.dim() == 1 and packed.is_contiguous()
    assert packed.is_pinned() == torch.cuda.is_available()
    assert table.tolist() == [[0, 3, 17, 23], [3 * 17 * 23 * 3, 3, 40, 30], [3 * 17 * 23 * 3 + 3 * 40 * 30 * 3, 3, 9, 64]]
    assert packed.numel() == sum(it["frames_u8"].numel() for it in items)
    for (off, F, H0, W0), it in zip(table.tolist(), items):
        assert torch.equal(packed[off:off + F * H0 * W0 * 3].view(F, H0, W0, 3), it["frames_u8"])
    assert b["prompt_ids"].shape == (3, 1, 77) and b["prompt_ids"][:, 0, 0].tolist() == [0, 1, 2]
    assert b["text_prompt"] == ["a", "b", "c"] and b["dataset"] == ["folder"] * 3
    assert b["pixel_hw"].tolist() == [[16, 16]] * 3
    with pytest.raises(AssertionError):
        D.collate_raw([_item(3, 8, 8, (16, 16), 0), _item(2, 8, 8, (16, 16), 1)])     # F differs
    with pytest.raises(AssertionError):
        D.collate_raw([_item(3, 8, 8, (16, 16), 0), _item(3, 8, 8, (16, 24), 1)])     # target size differs


class _Keyed(torch.utils.data.Dataset):
    """Item i: a tiny raw clip whose (F, h, w) group is keys[i]; carries its index."""

    def __init__(self, keys):
        self.keys = keys

    def __len__(self):
        return len(self.keys)

    def __getitem__(self, i):
        F, h, w = self.keys[i]
        it = _item(F, 4 + i % 3, 5 + i % 2, (h, w), i)
        it["index"] = i
        return it


def _indices(batch):
    return batch["prompt_ids"][:, 0, 0].tolist()


def _grouper(ds, bs, seed=None):
    from t2v_b200.utils.dataset import ShapeGroupedBatches
    sampler = (torch.utils.data.SequentialSampler(ds) if seed is None
               else torch.utils.data.RandomSampler(ds, generator=torch.Generator().manual_seed(seed)))
    return ShapeGroupedBatches(ds, bs, sampler)


KEYS = [(2, 16, 16)] * 7 + [(1, 16, 16)] * 5 + [(2, 16, 24)] * 4 + [(3, 8, 8)]


@pytest.mark.parametrize("bs", [2, 3, 4])
def test_grouper_homogeneous_complete_and_reproducible(bs):
    from t2v_b200.utils.dataset import group_key
    ds = _Keyed(KEYS)
    epochs = 5

    def run(seed):
        gr = _grouper(ds, bs, seed)
        seen = []
        for _ in range(epochs):
            for b in gr:
                idx = _indices(b)
                assert len(idx) == bs                                   # never short
                assert len({group_key(ds[i]) for i in idx}) == 1        # homogeneous
                seen += idx
        pending = [it["index"] for v in gr.buffers.values() for it in v]
        return seen, pending

    seen, pending = run(seed=11)
    counts = np.bincount(seen + pending, minlength=len(ds))
    assert (counts == epochs).all(), counts                              # every item once per epoch, counting carry-over
    assert run(seed=11) == (seen, pending)                               # reproducible from the seed
    assert run(seed=12)[0] != seen


def test_grouper_carries_partial_groups_into_the_next_epoch():
    ds = _Keyed([(2, 16, 16), (1, 16, 16), (2, 16, 16), (3, 8, 8)])
    gr = _grouper(ds, 2)
    assert [_indices(b) for b in gr] == [[0, 2]]
    assert gr.pending() == 2
    assert [_indices(b) for b in gr] == [[1, 1], [0, 2], [3, 3]]        # a carried item pairs with its next-epoch twin
    assert gr.pending() == 0


def test_grouper_at_batch_one_keeps_the_loader_order():
    ds = _Keyed(KEYS)
    g1, g2 = torch.Generator().manual_seed(5), torch.Generator().manual_seed(5)
    loader = torch.utils.data.DataLoader(ds, batch_size=1, sampler=torch.utils.data.RandomSampler(ds, generator=g1))
    from t2v_b200.utils.dataset import ShapeGroupedBatches
    gr = ShapeGroupedBatches(ds, 1, torch.utils.data.RandomSampler(ds, generator=g2))
    for _ in range(2):
        assert [int(b["index"][0]) for b in loader] == [_indices(b)[0] for b in gr]


def test_cached_latents_are_grouped_by_shape():
    from t2v_b200.utils.dataset import ShapeGroupedBatches

    class Lat(torch.utils.data.Dataset):
        shapes = [(4, 2, 4, 4), (4, 2, 4, 6), (4, 2, 4, 4), (4, 2, 4, 6), (4, 1, 4, 4), (4, 1, 4, 4)]

        def __len__(self):
            return len(self.shapes)

        def __getitem__(self, i):
            return {"pixel_values": torch.zeros(self.shapes[i]), "prompt_ids": torch.full((77,), i)}

    batches = list(ShapeGroupedBatches(Lat(), 2, range(6)))
    assert [b["prompt_ids"][:, 0].tolist() for b in batches] == [[0, 2], [1, 3], [4, 5]]
    assert [tuple(b["pixel_values"].shape) for b in batches] == [(2, 4, 2, 4, 4), (2, 4, 2, 4, 6), (2, 4, 1, 4, 4)]


def test_a_four_frame_pixel_clip_is_pixels():
    """[B, F=4, 3, h, w] pixel_values look like [B, C=4, F=3, h, w] latents: the decision is made from keys and source."""
    from t2v_b200.train import needs_vae
    from t2v_b200.utils.dataset import PACKED_KEY
    pix = {"pixel_values": torch.zeros(1, 4, 3, 16, 16), "prompt_ids": torch.zeros(1, 1, 77, dtype=torch.int64)}
    assert needs_vae(pix, latent_source=False)
    assert not needs_vae(pix, latent_source=True)
    assert needs_vae({"frames_u8": torch.zeros(1, 4, 8, 8, 3, dtype=torch.uint8)}, latent_source=False)
    assert needs_vae({PACKED_KEY: torch.zeros(8, dtype=torch.uint8)}, latent_source=False)


def test_frames_to_latents_packed_matches_per_clip_cpu():
    from oracle import ops_ref
    from t2v_b200.utils import dataset as D
    from t2v_b200.vae import AutoencoderKL
    items = [_item(2, 24, 40, (16, 16), 0), _item(2, 9, 13, (16, 16), 1)]
    eps = torch.randn(2, 4, 2, 2, 2, generator=torch.Generator().manual_seed(3))
    old = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        with emulated_prims(), emulated_ragged():
            torch.manual_seed(1)
            vae = AutoencoderKL(block_out_channels=(32, 32, 64, 64), layers_per_block=1).eval()
            got = D.frames_to_latents(D.collate_raw(items), vae, torch.device("cpu"), eps=eps)
            want = torch.cat([D.frames_to_latents({"frames_u8": it["frames_u8"][None], "pixel_hw": it["pixel_hw"][None]}, vae,
                                                  torch.device("cpu"), eps=eps[b:b + 1]) for b, it in enumerate(items)])
    finally:
        ops_ref.BF = old
    assert got.shape == (2, 4, 2, 2, 2)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ train.main at batch 2
def _pipe(root):
    """unet / vae / text_encoder / tokenizer / scheduler folder on the SMALL UNet."""
    import json

    from transformers import CLIPTextConfig
    from transformers import CLIPTextModel as HF
    from test_pipeline_train import _tiny_tokenizer
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.vae import AutoencoderKL
    unet = UNet3DConditionModel(**SMALL)
    unet.load_state_dict(seeded_state_dict(unet, 0))
    unet.save_pretrained(os.path.join(root, "unet"))
    torch.manual_seed(1)
    AutoencoderKL(block_out_channels=(32, 32, 64, 64), layers_per_block=1).save_pretrained(os.path.join(root, "vae"))
    nvocab = _tiny_tokenizer(os.path.join(root, "tokenizer"))
    HF(CLIPTextConfig(hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=1, vocab_size=nvocab,
                      max_position_embeddings=77, hidden_act="gelu")).save_pretrained(os.path.join(root, "text_encoder"))
    os.makedirs(os.path.join(root, "scheduler"), exist_ok=True)
    with open(os.path.join(root, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump({"_class_name": "DDIMScheduler", "beta_schedule": "scaled_linear", "prediction_type": "epsilon"}, f)
    return root


def _media(tmp, video_sizes, n_images=0):
    import cv2
    from test_dataset import _write_video
    vids, imgs = os.path.join(tmp, "vids"), os.path.join(tmp, "imgs")
    os.makedirs(vids, exist_ok=True)
    os.makedirs(imgs, exist_ok=True)
    for i, hw in enumerate(video_sizes):
        _write_video(os.path.join(vids, f"v{i}.mp4"), n=6, hw=hw)
    for i in range(n_images):
        cv2.imwrite(os.path.join(imgs, f"i{i}.png"), np.full((40, 50, 3), 60 * i + 20, np.uint8))
    return vids, imgs


def _record_steps(monkeypatch):
    from t2v_b200 import step as S
    seen, orig = [], S.DataParallelStep.__call__

    def call(self, latents, noise, timesteps, text):
        seen.append((tuple(latents.shape), self.passes))
        return orig(self, latents, noise, timesteps, text)
    monkeypatch.setattr(S.DataParallelStep, "__call__", call)
    return seen


def _main_kwargs(tmp, root, vids, imgs, kinds, steps):
    return dict(pretrained_model_path=root, output_dir=os.path.join(tmp, "out"), dataset_types=kinds,
                train_data=dict(width=32, height=32, n_sample_frames=2, fps=8, path=vids, image_dir=imgs, fallback_prompt="a clip"),
                train_batch_size=2, max_train_steps=steps, learning_rate=1e-3, checkpointing_steps=100, seed=0, shuffle=False,
                device="cpu", eval_train=True, use_unet_lora=True, lora_version="cloneofsimo", lora_rank=4,
                unet_lora_modules=["UNet3DConditionModel"], load_side_models=True, save_pretrained_model=False)


def test_train_main_batch_two_cpu(tmp_path, capsys, monkeypatch):
    """Videos at two native sizes + an image folder, batch 2: homogeneous batches, and the video batch after the image batch
    runs two passes."""
    from oracle import ops_ref
    from t2v_b200 import train
    root = _pipe(str(tmp_path / "pipe"))
    vids, imgs = _media(str(tmp_path), [(48, 64), (40, 24), (48, 64), (40, 24)], n_images=2)
    seen = _record_steps(monkeypatch)
    old = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        with emulated_prims(), emulated_ragged():
            r = train.main(**_main_kwargs(str(tmp_path), root, vids, imgs, ["folder", "image"], 4))
    finally:
        ops_ref.BF = old
    log = capsys.readouterr().out
    losses = [float(ln.split("loss")[1].split()[0]) for ln in log.splitlines() if ln.startswith("step ")]
    assert r["steps"] == 4 and losses and all(math.isfinite(v) for v in losses), log
    # sequential order: 4 videos -> 2 video batches, 2 images -> 1 image batch, then the next epoch's first video batch
    assert seen == [((2, 4, 2, 4, 4), 2), ((2, 4, 2, 4, 4), 2), ((2, 4, 1, 4, 4), 1), ((2, 4, 2, 4, 4), 2)], seen


def _dp_worker(rank, world, port, tmp, root, vids, kinds, result):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from helpers import emulated_prims
    from oracle import ops_ref
    from ragged_ref import emulated_ragged
    from t2v_b200 import train
    ops_ref.BF = torch.float32
    out = {}
    try:
        with emulated_prims(), emulated_ragged():
            r = train.main(**_main_kwargs(tmp, root, vids, os.path.join(tmp, "imgs"), kinds, 2))
        out["steps"] = r["steps"]
    except ValueError as e:
        out["error"] = str(e)
    torch.save(out, f"{result}.{rank}")
    dist.destroy_process_group()


def _run_two_ranks(tmp_path, video_sizes, kinds=("folder",), n_images=0):
    root = _pipe(str(tmp_path / "pipe"))
    vids, _ = _media(str(tmp_path), video_sizes, n_images=n_images)
    res = str(tmp_path / "res")
    port = 29500 + (os.getpid() * 7) % 2000
    mp.spawn(_dp_worker, args=(2, port, str(tmp_path), root, vids, list(kinds), res), nprocs=2, join=True)
    return [torch.load(f"{res}.{r}", weights_only=False) for r in range(2)]


def test_two_ranks_one_group_key_trains(tmp_path):
    """Clips of two native sizes resized to one target: one group key, so data-parallel training at batch 2 runs."""
    got = _run_two_ranks(tmp_path, [(48, 64), (40, 24), (48, 64), (40, 24)] * 2)
    assert [g.get("steps") for g in got] == [2, 2], got


def test_two_ranks_second_group_key_raises_on_every_rank(tmp_path):
    """Rank 1 meets an image (1 frame) next to its videos (2 frames): both ranks raise the ValueError, neither hangs."""
    got = _run_two_ranks(tmp_path, [(48, 64)] * 3, kinds=("folder", "image"), n_images=1)
    for g in got:
        assert "error" in g and "train_batch_size > 1 with data-parallel" in g["error"], got
