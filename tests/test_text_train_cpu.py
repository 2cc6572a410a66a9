"""`train_text_encoder` with `trainable_text_modules` on emulated primitives: the step, the gradients of every trainable text
tensor (embeddings included) and one AdamW step against the REFERENCE's own code (tests/golden/make_golden_text_train.py), the
optimizer groups and the requires_grad census, the refusals, and `train.main` end to end (what moves, the saved
`text_encoder/`, no stale frozen forward, resume, two gloo ranks)."""
import contextlib
import io
import os
import sys

import pytest
import torch

from helpers import seeded_state_dict
from oracle import ops_ref
from text_train_ref import emulated

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLDEN)
CASES = ["all", "substring", "all_lora"]


def golden(name, frames):
    return torch.load(os.path.join(GOLDEN, f"text_train_{name}_f{frames}.pt"), weights_only=False)


def build(c, device):
    """This repo's models from the fixture's seeds, set up as train.main sets them up: LoRA injected, the UNet's and the text
    encoder's trainable sets, and the optimizer groups in the reference's order.  Returns (unet, te, groups)."""
    from make_golden_lora import seed_lora_
    from t2v_b200 import train
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils import lora as mylora
    unet = UNet3DConditionModel(**c["unet_cfg"])
    unet.load_state_dict(seeded_state_dict(unet, c["seeds"]["unet_base"]))
    unet.requires_grad_(False)
    te = CLIPTextModel(c["text_cfg"])
    te.load_state_dict(seeded_state_dict(te, c["seeds"]["text_base"]))
    text_lora = None
    if c["use_text_lora"]:
        with contextlib.redirect_stdout(io.StringIO()):
            text_lora, _ = mylora.inject_trainable_lora_extended(te, {"CLIPEncoderLayer"}, r=c["r_text"])
        seed_lora_(te, c["seeds"]["text_lora"])
    train.handle_trainable_modules(unet, c["trainable_modules"])
    train.handle_trainable_modules(te, c["trainable_text_modules"])
    h = c["hyper"]
    extra = h["extra_unet_params"]
    groups = train.create_optimizer_params([
        train.param_optim(unet, True, extra_params=extra),
        train.param_optim(te, True, extra_params=extra),
        train.param_optim(text_lora, c["use_text_lora"], is_lora=True, extra_params={"lr": h["lr"], **extra}),
    ], h["lr"])
    return unet.to(device).eval(), te.to(device).eval(), groups


@contextlib.contextmanager
def fp32_emulation():
    old = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        with emulated():
            yield
    finally:
        ops_ref.BF = old


def run_step(c, device, monkeypatch, fused=False):
    """One optimizer step: DataParallelStep (two passes, the encoder inside) and AdamW with the clip over UNet + text."""
    from t2v_b200 import step as S
    unet, te, groups = build(c, device)
    losses = []
    finetune_loss = S.finetune_loss

    def record_loss(*a, **k):
        loss = finetune_loss(*a, **k)
        losses.append(loss.detach())
        return loss
    monkeypatch.setattr(S, "finetune_loss", record_loss)
    h = c["hyper"]
    # the parameter arena keeps bf16 copies of the weights for the kernels, so the fp32 CPU check runs without it
    stepper = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device=device), passes=2, text_encoder=te, adopt=fused)
    if fused:
        from t2v_b200.optim import FusedAdamW
        opt = FusedAdamW(stepper.arena, groups, lr=h["lr"], betas=h["betas"], eps=h["eps"], weight_decay=h["weight_decay"],
                         max_grad_norm=h["max_grad_norm"])
    else:
        opt = torch.optim.AdamW(groups, lr=h["lr"], betas=h["betas"], eps=h["eps"], weight_decay=h["weight_decay"])
    stepper(c["latents"].to(device), c["noise"].to(device), c["timesteps"].to(device), c["prompt_ids"].to(device))
    grads = {n: p.grad.detach().float().cpu().clone() for n, p in te.named_parameters() if p.grad is not None}
    unet_norms = {n: p.grad.norm().item() for n, p in unet.named_parameters() if p.grad is not None and p.grad.any()}
    if fused:
        opt.step()
        norm = opt.last_grad_norm()
    else:
        norm = torch.nn.utils.clip_grad_norm_(list(unet.parameters()) + list(te.parameters()), h["max_grad_norm"]).item()
        opt.step()
    return unet, te, opt, losses, grads, unet_norms, norm


@pytest.mark.parametrize("frames", [4, 1])
@pytest.mark.parametrize("name", CASES)
def test_step_matches_reference(name, frames, monkeypatch):
    c = golden(name, frames)
    with fp32_emulation():
        unet, te, opt, losses, grads, unet_norms, norm = run_step(c, "cpu", monkeypatch)
    want = c["pass_losses"]
    assert len(losses) == len(want) == (2 if frames > 1 else 1)
    for got, ref in zip(losses, want):
        assert abs(got.item() - ref.item()) <= 1e-4 * abs(ref.item()), (got.item(), ref.item())
    # every trainable text tensor has its gradient, and only those
    assert sorted(grads) == sorted(c["text_grads"])
    # floor: a key-projection bias has a zero gradient in exact arithmetic (the softmax ignores a per-row constant), so both
    # sides hold rounding noise there
    top = max(g.norm() for g in c["text_grads"].values())
    for n, ref in c["text_grads"].items():
        assert (grads[n] - ref).norm() <= 1e-4 * max(ref.norm(), 1e-4 * top), n
    tok = "text_model.embeddings.token_embedding.weight"
    if tok in grads:   # rows of ids no prompt uses stay exactly zero
        unused = torch.ones(grads[tok].shape[0], dtype=torch.bool)
        unused[c["prompt_ids"].flatten()] = False
        assert unused.any() and not grads[tok][unused].any() and not c["text_grads"][tok][unused].any()
        assert (c["prompt_ids"] == c["prompt_ids"][0, -1]).sum() > 10   # the pad id repeats
    top = max(c["unet_grad_norms"].values())
    assert sorted(unet_norms) == sorted(c["unet_grad_norms"])
    for n, gn in c["unet_grad_norms"].items():
        assert abs(unet_norms[n] - gn) <= 1e-4 * max(gn, 1e-3 * top), n
    assert abs(norm - c["grad_norm"]) <= 1e-4 * c["grad_norm"]
    # the AdamW update g / (|g| + eps) of an element whose gradient is near eps amplifies the gradient's rounding, so the
    # update is compared as a whole and each element within a tenth of the learning rate
    unet0, te0, _ = build(c, "cpu")
    params, start = dict(te.named_parameters()), dict(te0.named_parameters())
    params.update({"unet." + n: p for n, p in unet.named_parameters()})
    start.update({"unet." + n: p for n, p in unet0.named_parameters()})
    lr = c["hyper"]["lr"]
    for n, ref in c["after"].items():
        got, step = params[n].detach().cpu(), ref - start[n].detach()
        if n.split("unet.")[-1] in c["census"] or n.startswith("unet."):
            assert step.norm() > 0 and (got - ref).norm() <= 1e-3 * step.norm() and (got - ref).abs().max() <= 0.1 * lr, n
        else:   # frozen
            assert torch.equal(got, ref), n


@pytest.mark.parametrize("name", CASES)
def test_groups_and_census_match_reference(name):
    """The optimizer groups (order, names, sizes, lr, weight decay - the text groups built from extra_unet_params, SURVEY H4)
    and which text tensors require a gradient, against the reference restatement."""
    c = golden(name, 1)
    _, te, groups = build(c, "cpu")
    got = [(g.get("name"), len(list(g["params"])) if not isinstance(g["params"], torch.Tensor) else 1, g["lr"], g.get("weight_decay"))
           for g in torch.optim.AdamW(groups).param_groups]
    want = [tuple(x) for x in c["groups"]]
    # the reference names its LoRA group "param" (create_optim_params' default); ours has no name
    want = [(None if w[0] == "param" else w[0],) + w[1:] for w in want]
    # the UNet groups come first; this UNet registers mid_block before up_blocks, the reference's after, so they are compared
    # as a set - the text groups that follow keep the reference's order exactly
    n_unet = sum(1 for w in want if w[0] is not None and not w[0].startswith("text_model."))
    assert sorted(got[:n_unet]) == sorted(want[:n_unet]) and got[n_unet:] == want[n_unet:]
    assert len(got) == len(want) and all(w[0] is None or w[0].startswith("text_model.") for w in want[n_unet:])
    assert sorted(n for n, p in te.named_parameters() if p.requires_grad) == c["census"]


def test_embed_tokens_backward_restatement():
    """The emulated embed_tokens_bwd against an fp64 index_add: accumulates, clamps out-of-range ids, skips a null table."""
    from text_train_ref import embed_tokens_bwd
    g = torch.Generator().manual_seed(0)
    ids = torch.tensor([[0, 3, 3, 49, 60, -2], [3, 3, 3, 7, 49, 0]])
    dy = torch.randn(12, 16, generator=g).to(torch.bfloat16)
    dtok, dpos = torch.randn(50, 16, generator=g), torch.randn(8, 16, generator=g)
    want_tok, want_pos = dtok.double().clone(), dpos.double().clone()
    for r, i in enumerate(ids.flatten().clamp(0, 49).tolist()):
        want_tok[i] += dy[r].double()
        want_pos[r % 6] += dy[r].double()
    embed_tokens_bwd(ids, dy, dtok, dpos, 50)
    assert torch.allclose(dtok.double(), want_tok, atol=1e-5) and torch.allclose(dpos.double(), want_pos, atol=1e-5)
    before = dtok.clone()
    embed_tokens_bwd(ids, dy, None, dpos, 50)
    assert torch.equal(before, dtok)


def test_refusals(tmp_path):
    from t2v_b200 import train
    with pytest.raises(NotImplementedError, match="trainable_text_modules"):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "o"), train_text_encoder=True, device="cpu")
    with pytest.raises(ValueError, match="matches no text-encoder parameter"):
        _run(tmp_path, trainable_text_modules=["no_such_module"])
    with pytest.raises(ValueError, match="prompt_ids"):
        _run(tmp_path / "s", dataset_types=["synthetic"], train_data=dict(n=2, n_sample_frames=2, height=64, width=64))


def _run(tmp_path, **extra):
    from test_pipeline_train import _run as run
    kw = dict(train_text_encoder=True, trainable_text_modules=["all"], save_pretrained_model=False, learning_rate=1e-3,
              adam_weight_decay=0.0)
    kw.update(extra)
    with emulated():
        return run(tmp_path, "cpu", **kw)


def _text_state(te):
    return {n: p.detach().clone() for n, p in te.named_parameters()}


def test_train_main_end_to_end(tmp_path):
    """Trained text tensors move and frozen ones do not; `text_encoder/` and `text_encoder_ema/` load strictly into
    transformers.CLIPTextModel with the trained (EMA) values; after the steps the frozen-forward entry point
    `text_encoder(ids)[0]` is the eval `encode` of the trained weights (no stale bf16 pack)."""
    from safetensors.torch import load_file
    from transformers import CLIPTextModel as HF
    from t2v_b200.text_encoder import CLIPTextModel
    root = str(tmp_path / "pipe0")
    from test_pipeline_train import _pipeline_folder
    te0 = CLIPTextModel.from_pretrained(_pipeline_folder(root), subfolder="text_encoder")
    before = _text_state(te0)
    r, out, _ = _run(tmp_path, trainable_text_modules=["layers.0.mlp", "final_layer_norm", "token_embedding"], use_ema=True,
                     ema_decay=0.5, save_pretrained_model=True)
    te = r["stepper"].text_encoder
    after = _text_state(te)
    trained = {n for n, p in te.named_parameters() if p.requires_grad}
    assert trained == {n for n in before if "layers.0.mlp" in n or "final_layer_norm" in n or "token_embedding" in n}
    for n in before:
        moved = not torch.equal(before[n], after[n].cpu())
        assert moved == (n in trained), n
    # the saved folders
    hf = HF.from_pretrained(os.path.join(out, "text_encoder")).eval()
    sd = load_file(os.path.join(out, "text_encoder", "model.safetensors"))
    hf.load_state_dict(sd, strict=True)
    for n, v in after.items():
        assert torch.equal(sd[n], v.cpu()), n
    opt = r["optimizer"]
    with emulated(), opt.ema_weights():
        ema = _text_state(te)
    sd_ema = load_file(os.path.join(out, "text_encoder_ema", "model.safetensors"))
    HF.from_pretrained(os.path.join(out, "text_encoder_ema")).load_state_dict(sd_ema, strict=True)
    for n in before:
        assert torch.equal(sd_ema[n], ema[n].cpu()), n
        assert torch.equal(ema[n], after[n]) == (n not in trained), n
    assert not os.path.exists(os.path.join(out, "lora"))   # no LoRA injected: no LoRA list files
    # the public forward reads the trained weights
    ids = torch.randint(0, 50, (2, 77), generator=torch.Generator().manual_seed(3))
    te.eval()
    with emulated(), torch.no_grad():
        got = te(ids)[0]
        want = te.encode(ids).float().view(got.shape)
        stale = CLIPTextModel.from_pretrained(root, subfolder="text_encoder")(ids)[0]
    assert torch.equal(got, want)
    assert not torch.allclose(got, stale)


def test_all_with_text_lora_trains_base_and_factors(tmp_path):
    """`trainable_text_modules: ['all']` with cloneofsimo text LoRA (the reference's train_config.yaml with train_text_encoder):
    the wrapped base weights train too, the LoRA factors stay in their own group, and both move."""
    from test_text_lora_cpu import TRAIN_CONFIG
    r, out, _ = _run(tmp_path, **{**TRAIN_CONFIG, "train_text_encoder": True, "save_pretrained_model": True})
    te, opt = r["stepper"].text_encoder, r["optimizer"]
    names = {id(p): n for n, p in te.named_parameters()}
    lora_groups = [g for g in opt.param_groups if "name" not in g]
    assert {names.get(id(p)) for p in lora_groups[0]["params"]} == {n for n in names.values() if "lora" in n}
    text_groups = [g["name"] for g in opt.param_groups if g.get("name") in set(names.values())]
    assert text_groups == [n for n in names.values() if "lora" not in n]
    assert all(p.requires_grad for p in te.parameters())
    assert os.path.isfile(os.path.join(out, "lora", "2_text_encoder.pt"))
    from safetensors.torch import load_file
    from transformers import CLIPTextModel as HF
    HF.from_pretrained(os.path.join(out, "text_encoder")).load_state_dict(load_file(os.path.join(out, "text_encoder", "model.safetensors")),
                                                                          strict=True)


def test_resume_round_trip(tmp_path, monkeypatch):
    """Three steps in one go against one step, a saved training state and a resumed run: bitwise the same weights (text
    parameters included) and optimizer state."""
    import test_resume_cpu as R
    from test_pipeline_train import _pipeline_folder
    from test_dataset import _write_video
    root = _pipeline_folder(str(tmp_path / "pipe"))
    vids = tmp_path / "vids"
    vids.mkdir()
    for i in range(2):
        _write_video(str(vids / f"v{i}.mp4"), n=10, hw=(64, 64))
    kw = R._synthetic(root, dataset_types=["folder"], use_unet_lora=False, trainable_modules=["attn2"], train_text_encoder=True,
                      trainable_text_modules=["all"], load_side_models=True, use_ema=True, ema_decay=0.9,
                      train_data=dict(width=64, height=64, n_sample_frames=2, fps=8, path=str(vids), fallback_prompt="a video"))
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        part = R._resume_matches(tmp_path, monkeypatch, emulated, kw, 3, 1)
    finally:
        torch.set_num_threads(threads)
    import json
    man = json.load(open(os.path.join(part, "training_state", "manifest.json")))
    assert "text_encoder.text_model.embeddings.token_embedding.weight" in json.dumps(man)


def _two_rank_worker(rank, world, port, root):
    import pathlib

    import torch.distributed as dist
    tests = os.path.dirname(os.path.abspath(__file__))
    sys.path[:0] = [os.path.dirname(tests), tests]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank),
                      T2V_GRAD_COMPRESS="0")
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from test_pipeline_train import _run as run
    from text_train_ref import emulated
    with emulated():
        r, _, _ = run(pathlib.Path(root) / f"rank{rank}", "cpu", train_text_encoder=True, trainable_text_modules=["all"],
                      save_pretrained_model=False, max_train_steps=2, learning_rate=1e-3, seed=None)
    st = r["stepper"]
    torch.save({n: p.detach().clone() for n, p in st.text_encoder.named_parameters()}, os.path.join(root, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_text_weights_identical(tmp_path):
    """world size 2, each rank on its own clip: every text parameter's gradient is all-reduced after the encoder's backward,
    so both ranks end with bit-identical text weights, and they moved."""
    import torch.multiprocessing as mp
    from test_pipeline_train import _pipeline_folder
    from t2v_b200.text_encoder import CLIPTextModel
    port = 29500 + (os.getpid() + 1391) % 2000
    mp.spawn(_two_rank_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{i}.pt", weights_only=False) for i in range(2))
    start = dict(CLIPTextModel.from_pretrained(_pipeline_folder(str(tmp_path / "p")), subfolder="text_encoder").named_parameters())
    assert r0.keys() == r1.keys()
    for n in r0:
        assert torch.equal(r0[n], r1[n]), n
    assert sum(not torch.equal(r0[n], start[n].detach()) for n in r0) == len(r0)


def test_embedding_tables_have_no_bf16_shadow():
    """The token and position tables are gathered from their fp32 masters: the arena stores them with the vectors, outside the
    bf16 shadow that the fused optimizer rewrites every step; the projections keep theirs."""
    from t2v_b200.runtime import ParamArena
    from t2v_b200.text_encoder import CLIPTextModel
    te = CLIPTextModel(dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2, vocab_size=50))
    te.load_state_dict(seeded_state_dict(te, 1))
    te.requires_grad_(True)
    emb = te.text_model.embeddings
    want = emb.token_embedding.weight.detach().clone()
    with emulated():
        arena = ParamArena(te)
    mats = sum(p.numel() for p in te.parameters() if p.dim() == 2) - emb.token_embedding.weight.numel() - emb.position_embedding.weight.numel()
    assert arena.n_mat < mats + 64 * 8 and arena.n_mat >= mats
    for t in (emb.token_embedding.weight, emb.position_embedding.weight):
        assert getattr(t, "_t2v_shadow", None) is None and t.grad is not None
        assert t.data_ptr() >= arena.master.data_ptr() + 4 * arena.n_mat
    assert torch.equal(emb.token_embedding.weight.detach(), want)
    assert te.text_model.encoder.layers[0].mlp.fc1.weight._t2v_shadow is not None
