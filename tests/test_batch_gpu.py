"""train_batch_size > 1 on raw data, on the GPU: the ragged resize kernel against the single-clip kernel (bitwise) and the CPU
restatement, `frames_to_latents` of a packed batch against per-clip encodes, and `train.main` at batch 2 with graph replay
over videos of two native sizes plus images, with bucketing."""
import math
import os

import numpy as np
import pytest
import torch

from helpers import rel_l2
from ragged_ref import frames_u8_to_nhwc8_ragged as ragged_ref

pytestmark = pytest.mark.gpu


def _pack(clips):
    packed = torch.cat([c.reshape(-1) for c in clips])
    offs = np.cumsum([0] + [c.numel() for c in clips[:-1]]).tolist()
    table = torch.tensor([[o, c.shape[0], c.shape[1], c.shape[2]] for o, c in zip(offs, clips)], dtype=torch.int64)
    return packed, table


@pytest.mark.parametrize("out_hw", [(64, 64), (32, 48), (257, 131)])
def test_ragged_resize_is_bitwise_the_single_clip_kernel(out_hw):
    """Mixed F (1 included), odd native sizes, down- and up-scaling in one batch."""
    from oracle import ops_ref
    from t2v_b200 import prims
    g = torch.Generator().manual_seed(0)
    shapes = [(3, 90, 120), (1, 17, 23), (5, 481, 853), (2, 64, 64), (1, 7, 301), (4, 33, 31)]
    clips = [torch.randint(0, 256, s + (3,), generator=g, dtype=torch.uint8) for s in shapes]
    packed, table = _pack(clips)
    got = prims.frames_u8_to_nhwc8_ragged(packed.cuda(), table, out_hw)
    torch.cuda.synchronize()
    assert got.shape == (sum(s[0] for s in shapes), out_hw[0], out_hw[1], 8) and got.dtype == torch.bfloat16
    assert (got[..., 3:] == 0).all()
    f0 = 0
    for c in clips:
        one = prims.frames_u8_to_nhwc8(c.cuda(), out_hw)
        assert torch.equal(got[f0:f0 + c.shape[0]].view(torch.int16), one.view(torch.int16))
        f0 += c.shape[0]
    want = ragged_ref(packed, table, out_hw).float()
    assert (got.float().cpu() - want).abs().max().item() < 2e-2     # bf16 rounding of values in [-1, 1]
    # a device-resident table gives the same result
    assert torch.equal(prims.frames_u8_to_nhwc8_ragged(packed.cuda(), table.cuda(), out_hw), got)


def test_ragged_resize_rejects_a_table_that_overruns_the_buffer():
    from t2v_b200 import prims
    packed = torch.zeros(2 * 8 * 8 * 3, dtype=torch.uint8, device="cuda")
    table = torch.tensor([[0, 2, 8, 8], [8 * 8 * 3, 2, 8, 8]], dtype=torch.int64)
    with pytest.raises(AssertionError):
        prims.frames_u8_to_nhwc8_ragged(packed, table, (16, 16))


def test_frames_to_latents_packed_matches_per_clip():
    from t2v_b200.utils import dataset as D
    from t2v_b200.vae import AutoencoderKL
    g = torch.Generator().manual_seed(1)
    items = [{"frames_u8": torch.randint(0, 256, (3,) + hw + (3,), generator=g, dtype=torch.uint8), "pixel_hw": torch.tensor((64, 96)),
              "prompt_ids": torch.zeros(1, 77, dtype=torch.int64), "text_prompt": "x"} for hw in ((90, 120), (41, 203))]
    torch.manual_seed(3)
    vae = AutoencoderKL(block_out_channels=(32, 32, 64, 64), layers_per_block=1).cuda().eval()
    inputs = []
    orig = vae.encode_moments_nhwc8

    def capture(x):
        inputs.append(x.clone())
        return orig(x)
    vae.encode_moments_nhwc8 = capture
    eps = torch.randn(2, 4, 3, 8, 12, generator=g).cuda()
    dev = torch.device("cuda")
    got = D.frames_to_latents(D.collate_raw(items), vae, dev, eps=eps)
    want = torch.cat([D.frames_to_latents({"frames_u8": it["frames_u8"][None], "pixel_hw": it["pixel_hw"][None]}, vae, dev,
                                          eps=eps[b:b + 1]) for b, it in enumerate(items)])
    assert got.shape == (2, 4, 3, 8, 12)
    assert torch.equal(inputs[0], torch.cat(inputs[1:]))                # the VAE input: exactly the per-clip inputs
    assert rel_l2(got, want) < 4e-2, rel_l2(got, want)                   # a batched encode may plan its GEMMs differently


def test_train_main_batch_two_graph_replay_with_bucketing(tmp_path, capsys, monkeypatch):
    """Videos at two native sizes (one bucket) + images (another frame count), batch 2, CUDA-graph replay: every step is
    homogeneous, one capture per (F, h, w, passes), and video batches after an image batch run two passes."""
    from test_batch_cpu import _media, _record_steps
    from test_pipeline_train import _pipeline_folder
    from t2v_b200 import train
    root = _pipeline_folder(str(tmp_path / "pipe"))
    vids, imgs = _media(str(tmp_path), [(48, 64), (96, 128), (48, 64), (96, 128)], n_images=2)
    seen = _record_steps(monkeypatch)
    r = train.main(pretrained_model_path=root, output_dir=str(tmp_path / "out"), dataset_types=["folder", "image"],
                   train_data=dict(width=256, height=256, n_sample_frames=2, fps=8, path=vids, image_dir=imgs, use_bucketing=True,
                                   fallback_prompt="a clip"),
                   train_batch_size=2, max_train_steps=5, learning_rate=1e-4, checkpointing_steps=100, seed=0, shuffle=False,
                   device="cuda:0", trainable_modules=["attn1", "attn2"], save_pretrained_model=False)
    log = capsys.readouterr().out
    losses = [float(ln.split("loss")[1].split()[0]) for ln in log.splitlines() if ln.startswith("step ")]
    assert r["steps"] == 5 and losses and all(math.isfinite(v) for v in losses), log
    video, image = ((2, 4, 2, 24, 32), 2), ((2, 4, 1, 24, 32), 1)       # landscape bucket of 256: 192 x 256
    assert seen == [video, video, image, video, video], seen
    st = r["stepper"]
    assert st.use_graph and len(st._graphs) == len(set(seen)) == 2
