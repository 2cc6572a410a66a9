"""Datasets of the finetune step - SURVEY 8(f) row 3 (reference utils/dataset.py, train.py:266-314).

Same class names, constructor keywords, `__getname__()` tags and item keys (`pixel_values`, `prompt_ids`, `text_prompt`,
`dataset`) as the reference's VideoJsonDataset / SingleVideoDataset / ImageDataset / VideoFolderDataset / CachedDataset, so
the `train_data:` section of the v2 YAML configs maps onto them unchanged.  What differs (H100-first):

  * decoding uses OpenCV (`cv2.VideoCapture`; decord is not available) and stops at RAW frames: an item carries
    `frames_u8` uint8 [F, H0, W0, 3] (RGB) and `pixel_hw`, the target size;
  * resize + normalisation run on the GPU in ONE kernel (`prims.frames_u8_to_nhwc8`: bilinear, x / 127.5 - 1, bf16
    channels-last - the layout AutoencoderKL.encode consumes), see `frames_to_latents`; all frames of a clip are encoded as one
    batch (the reference encodes frame by frame with vae slicing);
  * `pixel_values` (float [F, 3, h, w] in [-1, 1], the reference's item format) is still produced - on the CPU, with the same
    arithmetic - when a dataset is built with `device_preprocess=False` (tests, foreign consumers);
  * train_batch_size > 1: `ShapeGroupedBatches` batches items of one (F, h, w) group, `collate_raw` packs clips of different
    native sizes into one buffer, and `frames_to_latents` resizes them with ONE ragged kernel launch
    (`prims.frames_u8_to_nhwc8_ragged`); the reference resizes on the CPU before collation instead.
"""
import json
import os
import random
from glob import glob

import numpy as np
import torch
from torch.utils.data import Dataset

VID_TYPES = (".mp4", ".avi", ".mov", ".webm", ".flv", ".mjpeg")
IMG_TYPES = (".png", ".jpg", ".jpeg", ".bmp")


# ------------------------------------------------------------------------------------------------ helpers (reference :22-108)
def normalize_input(item, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5), use_simple_norm=False):
    """uint8 / float frames [F, C, H, W] in 0..255 -> [-1, 1] (reference normalize_input: both of its branches reduce to
    x / 127.5 - 1 for the default mean = std = 0.5)."""
    item = item.float()
    if use_simple_norm or (tuple(mean) == (0.5, 0.5, 0.5) and tuple(std) == (0.5, 0.5, 0.5)):
        return item / 127.5 - 1.0
    m = torch.tensor(mean).view(1, -1, 1, 1)
    s = torch.tensor(std).view(1, -1, 1, 1)
    return (item / 255.0 - m) / s


def get_prompt_ids(prompt, tokenizer):
    return tokenizer(prompt, truncation=True, padding="max_length", max_length=tokenizer.model_max_length, return_tensors="pt").input_ids


def read_caption_file(caption_file):
    with open(caption_file, "r", encoding="utf8") as t:
        return t.read()


def get_text_prompt(text_prompt="", fallback_prompt="", file_path="", ext_types=(".mp4",), use_caption=False):
    """One caption file per media file (same stem, .txt) when use_caption is set; otherwise the given prompt."""
    try:
        if not use_caption:
            return text_prompt
        if len(text_prompt) > 1:
            return text_prompt
        for ext in ext_types:
            if file_path.endswith(ext):
                cand = file_path[:-len(ext)] + ".txt"
                if os.path.exists(cand):
                    return read_caption_file(cand)
        return fallback_prompt
    except OSError:
        print(f"Couldn't read prompt caption for {file_path}. Using fallback.")
        return fallback_prompt


def get_video_frames(n_total, start_idx, sample_rate=1, max_frames=24):
    frame_number = sorted((0, start_idx, n_total))[1]
    return list(range(frame_number, n_total, sample_rate))[:max_frames]


def sensible_buckets(m_width, m_height, w, h, min_size=192):
    """Aspect-ratio bucketing of the reference (utils/bucketing.py): keep one side, snap the other to a nearby bucket."""
    def closest(m_size, size):
        cands = [max(min_size, abs(int(m_size - m))) for m in (64, 128, 192)]
        return cands[min(range(len(cands)), key=lambda i: abs(cands[i] - size))]
    if h > w:
        return closest(m_width, m_width / (h / w)), m_height
    if h < w:
        return m_width, closest(m_height, m_height / (w / h))
    return m_width, m_height


class VideoReader:
    """Minimal decord.VideoReader stand-in on cv2.VideoCapture: len(), get_avg_fps(), get_batch(indices) -> uint8 [n, H, W, 3] RGB."""

    def __init__(self, path):
        import cv2
        self._cv2 = cv2
        self.path = path
        cap = cv2.VideoCapture(path)
        if not cap.isOpened():
            raise FileNotFoundError(f"cannot open video {path!r}")
        self._n = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
        self._fps = float(cap.get(cv2.CAP_PROP_FPS)) or 8.0
        cap.release()

    def __len__(self):
        return self._n

    def get_avg_fps(self):
        return self._fps

    def get_batch(self, indices):
        cv2 = self._cv2
        want = [int(i) for i in indices]
        cap = cv2.VideoCapture(self.path)
        frames, pos = {}, -1
        for idx in sorted(set(want)):
            if idx != pos + 1:
                cap.set(cv2.CAP_PROP_POS_FRAMES, idx)
            ok, f = cap.read()
            pos = idx
            if not ok:
                break
            frames[idx] = cv2.cvtColor(f, cv2.COLOR_BGR2RGB)
        cap.release()
        if not frames:
            raise RuntimeError(f"no frames decoded from {self.path!r}")
        last = frames[max(frames)]
        return torch.from_numpy(np.stack([frames.get(i, last) for i in want]))


def _read_image(path):
    import cv2
    img = cv2.imread(path, cv2.IMREAD_COLOR)
    if img is None:
        raise FileNotFoundError(path)
    return torch.from_numpy(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))


def _cpu_pixel_values(frames_u8, hw):
    """The reference's item format: float [F, 3, h, w] in [-1, 1] (bilinear resize like the device kernel)."""
    x = frames_u8.permute(0, 3, 1, 2).float()
    if tuple(x.shape[-2:]) != tuple(hw):
        x = torch.nn.functional.interpolate(x, size=tuple(hw), mode="bilinear", align_corners=False)
    return normalize_input(x)


class _Base(Dataset):
    device_preprocess = True

    def _example(self, frames_u8, hw, prompt, prompt_ids):
        ex = {"prompt_ids": prompt_ids, "text_prompt": prompt, "dataset": self.__getname__(), "pixel_hw": torch.tensor(hw)}
        if self.device_preprocess:
            ex["frames_u8"] = frames_u8.contiguous()
        else:
            ex["pixel_values"] = _cpu_pixel_values(frames_u8, hw)
        return ex

    def _target_hw(self, frames_u8):
        if getattr(self, "use_bucketing", False):
            h0, w0 = frames_u8.shape[1:3]
            w, h = sensible_buckets(self.width, self.height, w0, h0)
            return int(h), int(w)
        return int(self.height), int(self.width)

    def _prompt_ids(self, prompt):
        return get_prompt_ids(prompt, self.tokenizer) if self.tokenizer is not None else torch.zeros((1, 77), dtype=torch.int64)


# ------------------------------------------------------------------------------------------------ datasets
class VideoJsonDataset(_Base):
    """JSON produced by the Video-BLIP2 preprocessor: {"data": [{"video_path": ..., "data": [{"frame_index", "prompt"}, ...]}]}
    (or per-clip entries with "clip_path" + "prompt")."""

    def __init__(self, tokenizer=None, width=256, height=256, n_sample_frames=4, sample_start_idx=1, frame_step=1, json_path="",
                 json_data=None, vid_data_key="video_path", preprocessed=False, use_bucketing=False, device_preprocess=True, **kwargs):
        self.tokenizer, self.use_bucketing, self.preprocessed, self.vid_data_key = tokenizer, use_bucketing, preprocessed, vid_data_key
        self.width, self.height, self.n_sample_frames = width, height, n_sample_frames
        self.sample_start_idx, self.frame_step, self.device_preprocess = sample_start_idx, frame_step, device_preprocess
        self.train_data = self.load_from_json(json_path, json_data)

    def load_from_json(self, path, json_data):
        try:
            if json_data is None:
                with open(path) as f:
                    json_data = json.load(f)
            out = []
            for data in json_data["data"]:
                for nested in data["data"]:
                    entry = {self.vid_data_key: data[self.vid_data_key], "frame_index": nested.get("frame_index", 0), "prompt": nested["prompt"]}
                    if nested.get("clip_path") is not None:
                        entry["clip_path"] = nested["clip_path"]
                    out.append(entry)
            return out
        except (OSError, KeyError, TypeError, ValueError):
            print("Non-existant JSON path. Skipping.")
            return None

    @staticmethod
    def __getname__():
        return "json"

    def __len__(self):
        return len(self.train_data) if self.train_data is not None else 0

    def __getitem__(self, index):
        d = self.train_data[index]
        path = d.get("clip_path") or d[self.vid_data_key]
        vr = VideoReader(path)
        start = 0 if d.get("clip_path") else d["frame_index"]
        idxs = get_video_frames(len(vr), start, self.frame_step, self.n_sample_frames)
        frames = vr.get_batch(idxs)
        prompt = d["prompt"]
        return self._example(frames, self._target_hw(frames), prompt, self._prompt_ids(prompt))


class SingleVideoDataset(_Base):
    """One video cut into consecutive chunks of n_sample_frames (every frame_step-th frame), one prompt for all."""

    def __init__(self, tokenizer=None, width=256, height=256, n_sample_frames=4, frame_step=1, single_video_path="", single_video_prompt="",
                 use_caption=False, use_bucketing=False, device_preprocess=True, **kwargs):
        self.tokenizer, self.use_bucketing, self.device_preprocess = tokenizer, use_bucketing, device_preprocess
        self.width, self.height, self.n_sample_frames, self.frame_step = width, height, n_sample_frames, frame_step
        self.single_video_path, self.single_video_prompt = single_video_path, single_video_prompt
        self.frames = []
        if os.path.exists(single_video_path):
            self.create_video_chunks()

    def create_video_chunks(self):
        n = len(VideoReader(self.single_video_path))
        idx = list(range(1, n, self.frame_step))
        chunks = [idx[i:i + self.n_sample_frames] for i in range(0, len(idx), self.n_sample_frames)]
        self.frames = [c for c in chunks if len(c) == self.n_sample_frames] or chunks[:1]
        return self.frames

    @staticmethod
    def __getname__():
        return "single_video"

    def __len__(self):
        return len(self.frames)

    def __getitem__(self, index):
        frames = VideoReader(self.single_video_path).get_batch(self.frames[index])
        prompt = self.single_video_prompt
        return self._example(frames, self._target_hw(frames), prompt, self._prompt_ids(prompt))


class ImageDataset(_Base):
    """A folder of images trained as single-frame clips; captions from `<image>.txt` or single_img_prompt."""

    def __init__(self, tokenizer=None, width=256, height=256, base_width=256, base_height=256, use_caption=False, image_dir="",
                 single_img_prompt="", use_bucketing=False, fallback_prompt="", device_preprocess=True, **kwargs):
        self.tokenizer, self.use_bucketing, self.device_preprocess = tokenizer, use_bucketing, device_preprocess
        self.width, self.height = width, height
        self.use_caption, self.single_img_prompt, self.fallback_prompt = use_caption, single_img_prompt, fallback_prompt
        self.image_dir = self.get_images_list(image_dir)

    def get_images_list(self, image_dir):
        if os.path.isdir(image_dir):
            return sorted(os.path.join(image_dir, x) for x in os.listdir(image_dir) if x.lower().endswith(IMG_TYPES))
        return []

    @staticmethod
    def __getname__():
        return "image"

    def __len__(self):
        return len(self.image_dir)

    def __getitem__(self, index):
        path = self.image_dir[index]
        frames = _read_image(path)[None]
        prompt = get_text_prompt(file_path=path, text_prompt=self.single_img_prompt, fallback_prompt=self.fallback_prompt,
                                 ext_types=IMG_TYPES, use_caption=True)
        return self._example(frames, self._target_hw(frames), prompt, self._prompt_ids(prompt))


class VideoFolderDataset(_Base):
    """A folder of .mp4 files with optional same-stem .txt captions; a random window of n_sample_frames at ~fps."""

    def __init__(self, tokenizer=None, width=256, height=256, n_sample_frames=16, fps=8, path="./data", fallback_prompt="",
                 use_bucketing=False, device_preprocess=True, **kwargs):
        self.tokenizer, self.use_bucketing, self.device_preprocess = tokenizer, use_bucketing, device_preprocess
        self.fallback_prompt = fallback_prompt
        self.video_files = sorted(glob(f"{path}/*.mp4"))
        self.width, self.height, self.n_sample_frames, self.fps = width, height, n_sample_frames, fps

    @staticmethod
    def __getname__():
        return "folder"

    def __len__(self):
        return len(self.video_files)

    def __getitem__(self, index):
        path = self.video_files[index]
        vr = VideoReader(path)
        n = self.n_sample_frames
        every = min(len(vr), max(1, round(vr.get_avg_fps() / self.fps)))
        eff = len(vr) // every
        n = min(n, eff)
        start = random.randint(0, eff - n)
        frames = vr.get_batch(every * np.arange(start, start + n))
        cap = path[:-4] + ".txt"
        prompt = read_caption_file(cap) if os.path.exists(cap) else self.fallback_prompt
        return self._example(frames, self._target_hw(frames), prompt, self._prompt_ids(prompt))


class CachedDataset(Dataset):
    """The latent cache written by handle_cache_latents (reference :589-603): cached_{i}.pt dicts with `pixel_values` = latents
    (4, F, h, w), `prompt_ids` (77,), `text_prompt`, `dataset`; an optional `text_embeds` (77, D) entry skips the text encoder."""

    def __init__(self, cache_dir=""):
        self.cache_dir = cache_dir
        self.cached_data_list = self.get_files_list()

    def get_files_list(self):
        return sorted(os.path.join(self.cache_dir, x) for x in os.listdir(self.cache_dir) if x.endswith(".pt"))

    def __len__(self):
        return len(self.cached_data_list)

    def __getitem__(self, index):
        return torch.load(self.cached_data_list[index], map_location="cpu", weights_only=False)


# ------------------------------------------------------------------------------------------------ batches of B > 1
PACKED_KEY, TABLE_KEY = "frames_packed", "frames_table"


def collate_raw(items):
    """Items of one shape group (same F, same target `pixel_hw`; native sizes may differ) -> one batch: every clip's
    `frames_u8` back to back in ONE contiguous uint8 buffer (pinned when CUDA is present, so it crosses to the device in one
    asynchronous copy) under `frames_packed`, and `frames_table` int64 [B, 4] = (byte offset, F, H0, W0) per clip, the
    operands of prims.frames_u8_to_nhwc8_ragged.  `prompt_ids` and `pixel_hw` are stacked, `text_prompt` / `dataset` kept as
    lists."""
    hw = items[0]["pixel_hw"]
    F = items[0]["frames_u8"].shape[0]
    assert all(torch.equal(it["pixel_hw"], hw) for it in items), [tuple(it["pixel_hw"].tolist()) for it in items]
    assert all(it["frames_u8"].shape[0] == F for it in items), [it["frames_u8"].shape[0] for it in items]
    sizes = [it["frames_u8"].numel() for it in items]
    packed = torch.empty(sum(sizes), dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    table = torch.empty((len(items), 4), dtype=torch.int64)
    off = 0
    for k, (it, n) in enumerate(zip(items, sizes)):
        fr = it["frames_u8"]
        packed[off:off + n].copy_(fr.reshape(-1))
        table[k] = torch.tensor([off, fr.shape[0], fr.shape[1], fr.shape[2]])
        off += n
    batch = {PACKED_KEY: packed, TABLE_KEY: table, "pixel_hw": torch.stack([it["pixel_hw"] for it in items])}
    for k in items[0]:
        if k in ("frames_u8", "pixel_hw"):
            continue
        v = [it[k] for it in items]
        batch[k] = torch.stack(v) if torch.is_tensor(v[0]) else v
    return batch


def group_key(item):
    """What must agree across the items of one batch: (F, h, w) of the clip the step trains on.  A raw item's target size is
    its `pixel_hw` (its native size may differ); a `pixel_values` item (pixels [F, 3, h, w] or cached latents [4, F, h, w])
    is keyed by its exact shape, which default_collate needs equal."""
    if "frames_u8" in item:
        h, w = (int(v) for v in item["pixel_hw"].view(-1)[:2])
        return ("frames", int(item["frames_u8"].shape[0]), h, w)
    return ("pixel_values",) + tuple(item["pixel_values"].shape)


class ShapeGroupedBatches:
    """Batches of `batch_size` items that share one `group_key`, for train_batch_size > 1 (batch size 1 keeps the plain
    DataLoader).  Each pass (`for batch in grouper`) is one epoch: it walks the sampler's item order, buffers every item
    under its key and yields a batch as soon as a buffer holds `batch_size` items.  Buffers that are not full at the end of
    an epoch carry over into the next, so no item is dropped and no batch is short (a short batch would be one more shape,
    one more CUDA-graph capture).  The order is a pure function of the sampler's order, so a seeded sampler gives a
    reproducible grouping.

    single_key: data-parallel training (world > 1) steps every rank with the same shape, so only data with one group key
    is supported there.  Before yielding each batch, and once at the end of each epoch, every rank joins one small
    all-reduce of (error flag, key): a rank that meets a second key, or whose key differs from another rank's, makes EVERY
    rank raise the same ValueError at the same point instead of leaving the others waiting in the step's collectives."""

    def __init__(self, dataset, batch_size, sampler, collate=None, single_key=False, sync_device=None):
        self.dataset, self.batch_size, self.sampler = dataset, int(batch_size), sampler
        self.collate = collate or _collate_group
        self.single_key, self.sync_device = single_key, sync_device
        self.buffers = {}   # key -> items waiting for a full batch (kept across epochs)
        self._key = None

    def pending(self):
        return sum(len(v) for v in self.buffers.values())

    def __iter__(self):
        for i in self.sampler:
            item = self.dataset[i]
            key = group_key(item)
            if self.single_key:
                if self._key is None:
                    self._key = key
                elif key != self._key:
                    self._agree(f"item {i} has group key {key}, this rank's earlier items {self._key}")
            buf = self.buffers.setdefault(key, [])
            buf.append(item)
            if len(buf) == self.batch_size:
                del self.buffers[key]
                if self.single_key:
                    self._agree(None)
                yield self.collate(buf)
        if self.single_key:
            self._agree(None)

    def state_dict(self):
        """The items waiting in the buffers (the items themselves: reading them again would draw new random frame windows)
        and the single_key group key."""
        return {"buffers": [(k, list(v)) for k, v in self.buffers.items()], "key": self._key}

    def load_state_dict(self, state):
        self.buffers = {tuple(k): list(v) for k, v in state["buffers"]}
        self._key = None if state["key"] is None else tuple(state["key"])

    def _agree(self, error):
        """One all-reduce (MAX) of [error, key, -key], the key as 5 integers: the ranks' keys agree iff max == -max(-key)."""
        import torch.distributed as dist
        key = [0] * 5
        if self._key is not None:
            key = [1 + (self._key[0] == "frames")] + list(self._key[1:]) + [0] * (5 - len(self._key))
        v = torch.tensor([1 if error else 0] + key + [-k for k in key], dtype=torch.int64, device=self.sync_device)
        dist.all_reduce(v, op=dist.ReduceOp.MAX)
        v = v.tolist()
        if v[0] or v[1:6] != [-k for k in v[6:]]:
            raise ValueError("train_batch_size > 1 with data-parallel training needs every item of every rank to share one "
                             "(frames, height, width) group: grouping different shapes across ranks is not supported. "
                             + (error or "another rank met a different group key") + ". Use one target size and one "
                             "n_sample_frames (no use_bucketing, no mix of images and videos), or train_batch_size 1.")


class EpochOrder(torch.utils.data.Sampler):
    """The item order of one epoch of `base` (a RandomSampler, SequentialSampler or DistributedSampler) and how many of its
    items have been handed out, so a resumed run continues at the same item of the same shuffle.

    A RandomSampler without a generator seeds itself with one int64 drawn from torch's default CPU generator when its pass
    starts; that same draw is made here, recorded in `seed` and handed to the sampler as its generator, so the order and the
    generator's stream are exactly those of the plain sampler.  A DistributedSampler's order is its (seed, epoch) and a
    SequentialSampler's is fixed.  `resume(state)` makes the next pass replay the recorded shuffle (no draw) and skip the
    items already consumed."""

    def __init__(self, base):
        self.base = base
        self.draws = isinstance(base, torch.utils.data.RandomSampler) and base.generator is None
        self.seed, self.consumed, self._resume = None, 0, None

    def __len__(self):
        return len(self.base)

    def __iter__(self):
        resume, self._resume = self._resume, None
        if self.draws:
            self.seed = resume["seed"] if resume else int(torch.empty((), dtype=torch.int64).random_().item())
            self.base.generator = torch.Generator()
            self.base.generator.manual_seed(self.seed)
        self.consumed = 0
        it = iter(self.base)
        for _ in range(resume["consumed"] if resume else 0):
            next(it)
            self.consumed += 1
        for i in it:
            self.consumed += 1
            yield i

    def state_dict(self):
        d = {"seed": self.seed, "consumed": self.consumed}
        if isinstance(self.base, torch.utils.data.distributed.DistributedSampler):
            d["sampler_seed"], d["sampler_epoch"] = self.base.seed, self.base.epoch
        return d

    def resume(self, state):
        if "sampler_epoch" in state:
            self.base.set_epoch(state["sampler_epoch"])
        self._resume = dict(state)


def _collate_group(items):
    return collate_raw(items) if "frames_u8" in items[0] else torch.utils.data.default_collate(items)


# ------------------------------------------------------------------------------------------------ device side
@torch.no_grad()
def frames_to_latents(batch, vae, device, generator=None, eps=None):
    """A collated batch of raw clips -> latents (B, 4, F, h/8, w/8) * 0.18215 on `device`: H2D of the uint8 frames, one
    resize + normalise kernel, ONE batched VAE encode of all B*F frames, fused sample / rearrange / scale kernel
    (reference: normalize_input on the CPU, then tensor_to_vae_latent with per-frame slicing, train.py:339-347).
    A `collate_raw` batch (clips of different native sizes) goes through the ragged kernel in one launch.
    eps: the sampling noise (B, 4, F, h/8, w/8); drawn from `generator` when None."""
    from .. import prims
    if PACKED_KEY in batch:
        table = batch[TABLE_KEY]
        B, F = table.shape[0], int(table[0, 1])
        hw = tuple(int(v) for v in batch["pixel_hw"].view(-1, 2)[0])
        nhwc8 = prims.frames_u8_to_nhwc8_ragged(batch[PACKED_KEY].to(device, non_blocking=True), table, hw)
    elif "frames_u8" in batch:
        fr = batch["frames_u8"]                       # [B, F, H0, W0, 3] uint8
        B, F = fr.shape[:2]
        hw = tuple(int(v) for v in batch["pixel_hw"].view(-1, 2)[0])
        x = fr.reshape((B * F,) + tuple(fr.shape[2:])).to(device, non_blocking=True).contiguous()
        nhwc8 = prims.frames_u8_to_nhwc8(x, hw)
    else:
        pv = batch["pixel_values"].to(device, torch.float32)   # [B, F, 3, h, w] in [-1, 1]
        B, F = pv.shape[:2]
        nhwc8 = prims.latents_to_nhwc8(pv.reshape(B * F, 3, 1, pv.shape[-2], pv.shape[-1]).contiguous())
    mom = vae.encode_moments_nhwc8(nhwc8)
    _, h, w, _ = mom.shape
    if eps is None:
        eps = torch.randn((B, 4, F, h, w), device=mom.device, dtype=torch.float32, generator=generator)
    return prims.vae_sample(mom, eps.to(mom.device, torch.float32).contiguous(), B, F, 0.18215)


DATASETS = {cls.__getname__(): cls for cls in (VideoJsonDataset, SingleVideoDataset, ImageDataset, VideoFolderDataset)}


def get_train_dataset(dataset_types, train_data, tokenizer):
    """reference train.py `get_train_dataset`: one dataset per entry of dataset_types, built from the `train_data:` section."""
    out = []
    for kind in dataset_types:
        if kind not in DATASETS:
            raise ValueError(f"Dataset type not found: {kind} not in {sorted(DATASETS)}")
        out.append(DATASETS[kind](**dict(train_data or {}), tokenizer=tokenizer))
    if not out:
        raise ValueError("Dataset type not found: no dataset_types given")
    return out


def extend_datasets(datasets, dataset_items, extend=False):
    """reference train.py `extend_datasets`: repeat the shorter datasets' file lists up to the longest one."""
    biggest = max((len(d) for d in datasets), default=0)
    for d in datasets:
        for item in dataset_items:
            v = getattr(d, item, None)
            if v is None or not extend or len(v) == 0 or len(v) >= biggest:
                continue
            reps = biggest // len(v)
            setattr(d, item, (v * reps + v[:biggest - len(v) * reps]))
            print(f"New {d.__getname__()} dataset length: {len(d)}")
