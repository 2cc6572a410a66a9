"""cloneofsimo text-encoder LoRA (`use_text_lora`) on emulated primitives: injection census, the autograd encoder against
transformers + an fp32 LoRA restatement, the step's pass structure (train.py:803-834), optimizer groups, refusals, checkpoint
files, the collapsed `text_encoder/` folder and `train.main` with the reference's train_config.yaml settings."""
import os

import pytest
import torch
import torch.nn as nn

from helpers import seeded_state_dict
from text_lora_ref import emulated

SMALL = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, vocab_size=100,
             max_position_embeddings=77)
# the reference's train_config.yaml, minus paths and data (tests/golden/reference_configs_v2/train_config.yaml)
TRAIN_CONFIG = dict(lora_version="cloneofsimo", use_unet_lora=True, use_text_lora=True, lora_unet_dropout=0.1, lora_text_dropout=0.1,
                    save_lora_for_webui=True, only_lora_for_webui=False, save_pretrained_model=True,
                    unet_lora_modules=["UNet3DConditionModel"], text_encoder_lora_modules=["CLIPEncoderLayer"], lora_rank=16,
                    learning_rate=5e-6, adam_weight_decay=0, extra_unet_params=None, extra_text_encoder_params=None,
                    trainable_modules=["all"], trainable_text_modules=["all"], gradient_checkpointing=True,
                    text_encoder_gradient_checkpointing=False, train_text_encoder=False, use_offset_noise=False)


class _TorchLora(nn.Module):
    """fp32 restatement of a cloneofsimo LoraInjectedLinear in eval mode: base(x) + scale * up(down(x))."""

    def __init__(self, lin, wrapper):
        super().__init__()
        self.lin, self.scale = lin, wrapper.scale
        self.up = nn.Parameter(wrapper.lora_up.weight.detach().cpu().clone())
        self.down = nn.Parameter(wrapper.lora_down.weight.detach().cpu().clone())

    def forward(self, x):
        return self.lin(x) + self.scale * ((x @ self.down.T) @ self.up.T)


def _pair(hidden_act="gelu", seed=0):
    """(transformers.CLIPTextModel, our injected CLIPTextModel with the same weights and non-zero lora_up)."""
    from transformers import CLIPTextConfig
    from transformers import CLIPTextModel as HF
    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils.lora import inject_trainable_lora_extended
    torch.manual_seed(seed)
    hf = HF(CLIPTextConfig(hidden_act=hidden_act, **SMALL)).eval()
    m = CLIPTextModel(dict(hidden_act=hidden_act, **SMALL))
    m.load_state_dict({k: v for k, v in hf.state_dict().items() if not k.endswith("position_ids")})
    inject_trainable_lora_extended(m, {"CLIPEncoderLayer"}, r=4)
    for mod in m.modules():
        if hasattr(mod, "lora_up"):
            nn.init.normal_(mod.lora_up.weight, std=0.05)
    return hf, m.eval()


def _restate(hf, m):
    """Wrap hf's projections with _TorchLora copies of m's factors; returns {module name: wrapper}."""
    ref = {}
    for n, w in m.named_modules():
        if hasattr(w, "lora_up"):
            parent_name, leaf = n.rsplit(".", 1)
            parent = hf.get_submodule(parent_name)
            ref[n] = _TorchLora(getattr(parent, leaf), w)
            setattr(parent, leaf, ref[n])
    hf.requires_grad_(False)
    for t in ref.values():
        t.up.requires_grad_(True)
        t.down.requires_grad_(True)
    return ref


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def test_injection_census_matches_transformers():
    """The YAML's text_encoder_lora_modules resolve by class name as on transformers.CLIPTextModel: 6 wrappers per layer,
    138 on the 23-layer ViT-H tower, same names and shapes."""
    from transformers import CLIPTextConfig
    from transformers import CLIPTextModel as HF
    from t2v_b200.text_encoder import DEFAULTS, CLIPTextModel
    from t2v_b200.utils.lora import inject_trainable_lora_extended
    census = []
    with torch.device("meta"):
        for model in (HF(CLIPTextConfig(**DEFAULTS)), CLIPTextModel()):
            inject_trainable_lora_extended(model, {"CLIPEncoderLayer"}, r=16)
            census.append([(n, tuple(m.lora_down.weight.shape), tuple(m.lora_up.weight.shape))
                           for n, m in model.named_modules() if hasattr(m, "lora_up")])
    assert census[0] == census[1]
    assert len(census[1]) == 138
    assert {n.rsplit(".", 1)[1] for n, _, _ in census[1]} == {"q_proj", "k_proj", "v_proj", "out_proj", "fc1", "fc2"}
    shapes = dict((n.split("layers.0.")[1], (d, u)) for n, d, u in census[1] if ".layers.0." in n)
    assert shapes["mlp.fc1"] == ((16, 1024), (4096, 16)) and shapes["mlp.fc2"] == ((16, 4096), (1024, 16))
    with torch.device("meta"):
        attn_only = CLIPTextModel()
        inject_trainable_lora_extended(attn_only, {"CLIPAttention"}, r=16)
    assert sum(hasattr(m, "lora_up") for m in attn_only.modules()) == 4 * 23


@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
def test_encoder_forward_backward_matches_transformers(act):
    hf, m = _pair(act)
    ids = torch.randint(0, SMALL["vocab_size"], (2, 77), generator=torch.Generator().manual_seed(1))
    with emulated():
        out = m.encode(ids)
        g = torch.randn(out.shape, generator=torch.Generator().manual_seed(2))
        out.backward(g.to(out.dtype))
    ref = _restate(hf, m)
    o = hf(ids)[0]
    o.backward(g.to(torch.bfloat16).float().view(o.shape))
    assert _rel(out.float().view(o.shape), o) < 2e-2
    for n, w in m.named_modules():
        if hasattr(w, "lora_up"):
            assert _rel(w.lora_up.weight.grad, ref[n].up.grad) < 4e-2, n
            assert _rel(w.lora_down.weight.grad, ref[n].down.grad) < 4e-2, n
    # base weights, norms and embeddings stay frozen: no gradient is formed for them
    assert all(p.grad is None for n, p in m.named_parameters() if "lora" not in n)
    with emulated(), torch.no_grad():
        ev = m(ids)[0]
    assert _rel(ev, o.detach()) < 2e-2


def _tiny_models():
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils.lora import inject_trainable_lora_extended
    unet = UNet3DConditionModel(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)
    unet.load_state_dict(seeded_state_dict(unet, 0))
    unet.requires_grad_(False)
    unet.train()
    for mod in unet.modules():
        if isinstance(mod, nn.Dropout):
            mod.p = 0.0
    for n, p in unet.named_parameters():
        if "attn2.to_out" in n:
            p.requires_grad_(True)
    te = CLIPTextModel(dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=1, vocab_size=50))
    te.load_state_dict(seeded_state_dict(te, 3))
    torch.manual_seed(4)
    inject_trainable_lora_extended(te, {"CLIPEncoderLayer"}, r=4)
    for mod in te.modules():
        if hasattr(mod, "lora_up"):
            nn.init.normal_(mod.lora_up.weight, std=0.05)
    return unet, te.eval()


@pytest.mark.parametrize("frames,accumulation", [(3, 1), (1, 1), (3, 2)])
def test_step_pass_structure(frames, accumulation):
    """Pass 0: full clip on detached states; pass 1: frame 1 on the trainable states (the only gradient into the text
    LoRA); F = 1: one pass on the trainable states.  Both scaled by 1 / accumulation."""
    from oracle import leaves as L
    from t2v_b200 import step as S
    unet, te = _tiny_models()
    abar = L.ddpm_alphas_cumprod()
    g = torch.Generator().manual_seed(5)
    lat, noise = torch.randn(1, 4, frames, 8, 8, generator=g), torch.randn(1, 4, frames, 8, 8, generator=g)
    t = torch.tensor([300])
    ids = torch.randint(0, 50, (1, 77), generator=g)
    text_params = [p for p in te.parameters() if p.requires_grad]
    with emulated():
        stepper = S.DataParallelStep(unet, abar, passes=2, adopt=True, accumulation=accumulation, text_encoder=te)
        assert all(p.grad is not None and p.grad.data_ptr() >= stepper.arena.grad.data_ptr() for p in text_params)
        loss = stepper(lat, noise, t, ids)
        got_text = [p.grad.clone() for p in text_params]
        got_unet = [p.grad.clone() for p in unet.parameters() if p.requires_grad]
        # manual restatement with the same primitives
        stepper.arena.zero_grads()
        states = te.encode(ids).view(1, 77, -1)
        want = 0.0
        runs = [(lat, noise, states.detach()), (lat[:, :, 1:2], noise[:, :, 1:2], states)] if frames > 1 else [(lat, noise, states)]
        for la, nz, st in runs:
            li = S.finetune_loss(unet, la, nz, t, st, abar)
            (li / accumulation).backward()
            want += li.item()
    assert loss.item() == pytest.approx(want, rel=1e-5)
    for a, p in zip(got_text, text_params):
        assert _rel(a, p.grad) < 1e-5 and p.grad.norm() > 0
    for a, p in zip(got_unet, [p for p in unet.parameters() if p.requires_grad]):   # temporal ones stay zero at F = 1
        assert torch.allclose(a, p.grad, rtol=1e-5, atol=1e-8)


def test_text_states_fan_in_is_fp32():
    """The states' gradient over every cross-attention is summed in fp32 and rounded once."""
    from t2v_b200 import ops
    x = torch.randn(6, 8).to(torch.bfloat16).requires_grad_(True)
    outs = ops.fork_f32(x, 5)
    gs = [torch.full((6, 8), v, dtype=torch.bfloat16) for v in (1.0, 2 ** -8, 2 ** -8, 2 ** -8, 2 ** -8)]
    with emulated():
        torch.autograd.backward(list(outs), gs)
    # a bf16 running sum would drop every 2^-8 term against 1.0; fp32 keeps them: 1 + 2^-6 is a bf16 value
    assert torch.all(x.grad.float() == 1.0 + 2 ** -6)


def _run_tiny(tmp_path, **extra):
    from test_pipeline_train import _run
    with emulated():
        return _run(tmp_path, "cpu", **{**TRAIN_CONFIG, **extra})


def test_refusals(tmp_path):
    from t2v_b200 import train
    with pytest.raises(NotImplementedError):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "o"), train_text_encoder=True, device="cpu")
    with pytest.raises(NotImplementedError):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "o"), use_text_lora=True,
                   lora_version="stable_lora", device="cpu")
    with pytest.raises(ValueError, match="prompt_ids"):
        _run_tiny(tmp_path, dataset_types=["synthetic"], train_data=dict(n=2, n_sample_frames=2, height=64, width=64))


def test_train_config_yaml_settings(tmp_path):
    """train.main with the reference's train_config.yaml settings: groups (H4), files, reload, collapsed text_encoder/."""
    from safetensors.torch import load_file
    from transformers import CLIPTextModel as HF
    from t2v_b200.text_encoder import CLIPTextModel
    r, out, root = _run_tiny(tmp_path, cache_latents=True, checkpointing_steps=1, extra_unet_params={"weight_decay": 0.25})
    assert r["steps"] == 2
    opt = r["optimizer"]
    te = r["stepper"].text_encoder
    groups = opt.param_groups
    # order: UNet (trainable_modules, one group per tensor), text LoRA (one group), UNet LoRA (one group)
    text_ids = {id(p) for p in te.parameters() if p.requires_grad}
    lora_groups = [g for g in groups if "name" not in g]
    assert len(lora_groups) == 2
    assert {id(p) for p in lora_groups[0]["params"]} == text_ids
    assert lora_groups[0]["lr"] == 5e-6 and lora_groups[0]["weight_decay"] == 0.25   # H4: built from extra_unet_params
    assert groups.index(lora_groups[0]) == len(groups) - 2
    # files
    lora_dir = os.path.join(out, "checkpoint-1", "lora")
    assert sorted(os.listdir(lora_dir)) == ["1_text_encoder.pt", "1_unet.pt"]
    saved = torch.load(os.path.join(out, "lora", "2_text_encoder.pt"))
    wrappers = [m for m in te.modules() if hasattr(m, "lora_up")]
    assert len(saved) == 2 * len(wrappers) == 12
    for i, w in enumerate(wrappers):
        assert torch.equal(saved[2 * i], w.lora_up.weight.detach().cpu())
        assert torch.equal(saved[2 * i + 1], w.lora_down.weight.detach().cpu())
    # text_encoder/ holds W + up @ down under the plain keys: strict load into transformers and into ours
    sd = load_file(os.path.join(out, "text_encoder", "model.safetensors"))
    hf = HF.from_pretrained(os.path.join(out, "text_encoder")).eval()
    hf.load_state_dict(sd, strict=True)
    ours = CLIPTextModel.from_pretrained(out, subfolder="text_encoder")
    ids = torch.randint(0, 100, (1, 77), generator=torch.Generator().manual_seed(0))
    te.eval()
    with emulated(), torch.no_grad():
        want = te(ids)[0]
        plain = ours(ids)[0]
    got = hf(ids)[0].detach()
    assert _rel(got, want) < 2e-2 and _rel(plain, want) < 2e-2
    # lora_path reloads the text encoder's LoRA file (the first file whose name contains text_encoder)
    reload_dir = tmp_path / "reload"
    reload_dir.mkdir()
    torch.save(saved, reload_dir / "2_text_encoder.pt")
    r2, _, _ = _run_tiny(tmp_path / "second", max_train_steps=0, lora_path=str(reload_dir), save_pretrained_model=False)
    w2 = [m for m in r2["stepper"].text_encoder.modules() if hasattr(m, "lora_up")]
    for i, w in enumerate(w2):
        assert torch.equal(w.lora_up.weight.detach().cpu(), saved[2 * i])


def test_clip_norm_covers_optimizer_params_only(tmp_path):
    """No embedding gradient exists, and every trainable tensor of the run is in an optimizer group (so the clip norm is
    the norm over the optimizer's parameters)."""
    r, _, _ = _run_tiny(tmp_path, max_train_steps=1, save_pretrained_model=False)
    te, opt = r["stepper"].text_encoder, r["optimizer"]
    assert te.text_model.embeddings.token_embedding.weight.grad is None
    assert all(p.grad is None for n, p in te.named_parameters() if "lora" not in n)
    in_groups = {id(p) for g in opt.param_groups for p in g["params"]}
    assert {id(p) for p in r["stepper"].arena.params if p.requires_grad} == in_groups


def _two_rank_worker(rank, world, port, root):
    """One rank of `train.main` with text LoRA over gloo: its own copy of the tiny pipeline and a LoRA initialisation that
    differs from the other rank's until rank 0's weights are broadcast."""
    import sys
    import torch.distributed as dist
    tests = os.path.dirname(os.path.abspath(__file__))
    sys.path[:0] = [os.path.dirname(tests), tests]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank),
                      T2V_GRAD_COMPRESS="0")
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import pathlib
    import test_pipeline_train
    from test_pipeline_train import _run
    from text_lora_ref import emulated
    make_folder = test_pipeline_train._pipeline_folder

    def folder_then_rank_seed(root_):
        out = make_folder(root_)        # seeds its own weights: the same pipeline on both ranks
        torch.manual_seed(100 + rank)   # seed=None below: each rank then draws its own lora_down, until the broadcast
        return out
    test_pipeline_train._pipeline_folder = folder_then_rank_seed
    with emulated():
        r, _, _ = _run(pathlib.Path(root) / f"rank{rank}", "cpu",
                       **{**TRAIN_CONFIG, **dict(seed=None, max_train_steps=2, learning_rate=1e-3, save_pretrained_model=False)})
    st = r["stepper"]
    torch.save({"text": {n: p.detach().clone() for n, p in st.text_encoder.named_parameters() if "lora" in n},
                "unet": {n: p.detach().clone() for n, p in st.unet.named_parameters() if "lora" in n},
                "overlapped": st.buckets.last_overlapped}, os.path.join(root, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_ranks_end_identical(tmp_path):
    """world size 2: rank 0's weights are broadcast over the text-LoRA factors too, every step all-reduces their gradients
    (after the text encoder's backward), so both ranks end with bit-identical text-LoRA and UNet-LoRA weights, and those moved."""
    import torch.multiprocessing as mp
    from t2v_b200.utils.lora import inject_trainable_lora_extended  # noqa: F401  (import check before spawning)
    port = 29500 + (os.getpid() + 977) % 2000
    mp.spawn(_two_rank_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{i}.pt", weights_only=False) for i in range(2))
    assert r0["text"].keys() == r1["text"].keys() and len(r0["text"]) == 12
    for part in ("text", "unet"):
        for n in r0[part]:
            assert torch.equal(r0[part][n], r1[part][n]), n
    assert all(r0["text"][n].abs().max() > 0 for n in r0["text"] if "lora_up" in n)   # lora_up starts at zero: it trained
    assert r0["overlapped"] > 0
