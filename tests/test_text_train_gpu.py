"""`train_text_encoder` on the H100: the t2v_embed_tokens_bwd kernel against an fp64 index_add, the step against the
reference's fixtures (tests/golden/make_golden_text_train.py) at the cloneofsimo tolerances of DESIGN §5, the text-parameter
gradients of a ViT-H-width encoder against fp32 torch autograd, graph replay against eager, and `train.main` with FusedAdamW,
8-bit AdamW and the EMA covering the text parameters."""
import os

import pytest
import torch

from helpers import cosine, seeded_state_dict

pytestmark = pytest.mark.gpu
VOCAB = 49408


def _ref(ids, dy, dtok0, dpos0):
    from text_train_ref import embed_tokens_bwd
    dtok, dpos = dtok0.double().clone(), dpos0.double().clone()
    embed_tokens_bwd(ids, dy, dtok, dpos, VOCAB, dtype=torch.float64)
    return dtok, dpos


def _ids(kind, B, g):
    if kind == "padded":   # start id, a few words, the pad id repeated (CLIP's tokenizer layout)
        ids = torch.full((B, 77), VOCAB - 1, dtype=torch.int64)
        ids[:, 0] = VOCAB - 2
        ids[:, 1:9] = torch.randint(0, VOCAB - 2, (B, 8), generator=g)
        return ids
    if kind == "all_equal":
        return torch.full((B, 77), 1234, dtype=torch.int64)
    if kind == "ends":
        return torch.randint(0, 2, (B, 77), generator=g) * (VOCAB - 1)
    if kind == "out_of_range":   # clamped as the forward clamps: below 0 -> 0, at or above vocab -> vocab - 1
        ids = torch.randint(1, VOCAB - 1, (B, 77), generator=g)   # in range, never 0 or vocab - 1 themselves
        bad = torch.tensor(OUT_OF_RANGE)
        pos = torch.randperm(B * 77, generator=g)[:len(OUT_OF_RANGE)]
        ids.view(-1)[pos] = bad
        return ids
    return torch.randint(0, VOCAB, (B, 77), generator=g)


OUT_OF_RANGE = [-1, -7, -1, VOCAB, VOCAB + 100, VOCAB, -(2 ** 40), 2 ** 40]   # repeats included


@pytest.mark.parametrize("C", [128, 1024])
@pytest.mark.parametrize("B", [1, 2, 8])
@pytest.mark.parametrize("kind", ["padded", "all_equal", "ends", "out_of_range", "random"])
def test_embed_tokens_bwd_matches_fp64(kind, B, C):
    from t2v_b200 import prims
    g = torch.Generator().manual_seed(B * 1000 + C)
    ids = _ids(kind, B, g)
    dy = torch.randn(B * 77, C, generator=g).to(torch.bfloat16)
    # accumulation into a non-zero gradient (the previous micro-step's)
    dtok0 = torch.zeros(VOCAB, C)
    rows = torch.randint(0, VOCAB, (64,), generator=g)
    dtok0[rows] = torch.randn(64, C, generator=g)
    dtok0[ids.clamp(0, VOCAB - 1).flatten()[:5]] = torch.randn(5, C, generator=g)
    dpos0 = torch.randn(77, C, generator=g)
    want_tok, want_pos = _ref(ids, dy, dtok0, dpos0)
    dev = "cuda"
    outs = []
    for _ in range(2):
        dtok, dpos = dtok0.to(dev), dpos0.to(dev)
        prims.embed_tokens_bwd(ids.to(dev), dy.to(dev), dtok, dpos, VOCAB)
        outs.append((dtok.cpu(), dpos.cpu()))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])   # bitwise reproducible
    dtok, dpos = outs[0]
    # fp32 sums of at most B*77 bf16 terms: each element within 2^-20 of the sum of |terms| (plus what it started at)
    mag_tok = _ref(ids, dy.abs(), dtok0.abs(), torch.zeros_like(dpos0))[0]
    mag_pos = _ref(ids, dy.abs(), torch.zeros_like(dtok0), dpos0.abs())[1]
    assert ((dtok.double() - want_tok).abs() <= 2 ** -20 * (mag_tok + 1e-30)).all()
    assert ((dpos.double() - want_pos).abs() <= 2 ** -20 * (mag_pos + 1e-30)).all()
    untouched = torch.ones(VOCAB, dtype=torch.bool)
    untouched[ids.clamp(0, VOCAB - 1).flatten()] = False
    assert torch.equal(dtok[untouched], dtok0[untouched])
    if kind == "out_of_range":
        # every out-of-range id was placed, and rows 0 and vocab - 1 receive exactly their rows' sums (no in-range id is 0 or
        # vocab - 1 here), the rows the forward kernel read for them
        flat = ids.flatten()
        assert int((flat < 0).sum()) == 4 and int((flat >= VOCAB).sum()) == 4
        for row, sel in ((0, flat < 0), (VOCAB - 1, flat >= VOCAB)):
            want = dtok0[row].double() + dy[sel].double().sum(0)
            assert (dtok[row].double() - want).abs().max() <= 2 ** -20 * (dtok0[row].abs().double() + dy[sel].abs().double().sum(0)).max()
            assert not torch.equal(dtok[row], dtok0[row])
        tok = torch.randn(VOCAB, C, generator=g)
        fwd = prims.embed_tokens(ids.to(dev), tok.to(dev), torch.zeros(77, C, device=dev))
        assert torch.equal(fwd.cpu(), tok[flat.clamp(0, VOCAB - 1)].to(torch.bfloat16))   # the forward read the same rows
    # a frozen table: null pointer, nothing written
    dtok = dtok0.to(dev)
    prims.embed_tokens_bwd(ids.to(dev), dy.to(dev), None, dpos0.to(dev), VOCAB)
    assert torch.equal(dtok.cpu(), dtok0)


@pytest.mark.parametrize("frames", [4, 1])
@pytest.mark.parametrize("name", ["all", "substring", "all_lora"])
def test_step_matches_reference_gpu(name, frames, monkeypatch):
    """The fixtures on the CUDA kernels with the parameter arena and FusedAdamW: losses within 3e-3, >= 97 % of the text
    gradient tensors with cosine > 0.98 (DESIGN §5), the clip norm within 2 %, each trained tensor's update along the
    reference's (cosine > 0.95) and the frozen ones untouched."""
    from test_text_train_cpu import golden, run_step
    c = golden(name, frames)
    unet, te, opt, losses, grads, unet_norms, norm = run_step(c, "cuda", monkeypatch, fused=True)
    for got, ref in zip(losses, c["pass_losses"]):
        assert abs(got.item() - ref.item()) <= 3e-3 * abs(ref.item()), (got.item(), ref.item())
    assert sorted(grads) == sorted(c["text_grads"])
    top = max(g.norm() for g in c["text_grads"].values())
    big = [n for n, ref in c["text_grads"].items() if ref.norm() > 1e-3 * top]   # skips the zero-in-exact-arithmetic k_proj.bias
    cos = [cosine(grads[n], c["text_grads"][n]) for n in big]
    assert sum(x > 0.98 for x in cos) >= 0.97 * len(cos), sorted(zip(cos, big))[:5]
    assert abs(norm - c["grad_norm"]) <= 2e-2 * c["grad_norm"]
    tok = "text_model.embeddings.token_embedding.weight"
    if tok in grads:
        unused = torch.ones(grads[tok].shape[0], dtype=torch.bool)
        unused[c["prompt_ids"].flatten()] = False
        assert not grads[tok][unused].any()
    # the update itself, against the reference's: AdamW's first step is about lr * sign(g) per element, so an element-wise
    # bound of a few lr would let wrong-signed updates through; the update's direction does not (bf16 emulation: >= 0.968)
    from test_text_train_cpu import build
    params, start = dict(te.named_parameters()), dict(build(c, "cpu")[1].named_parameters())
    for n, ref in c["after"].items():
        if n not in params:
            continue
        got, s0 = params[n].detach().cpu(), start[n].detach()
        if n in c["census"]:
            assert cosine(got - s0, ref - s0) > 0.95, (n, cosine(got - s0, ref - s0))
        else:   # frozen: untouched
            assert torch.equal(got, ref) and torch.equal(got, s0), n


def test_vith_width_gradients_match_fp32_autograd():
    """ViT-H widths (1024 hidden, 16 heads, 4096 MLP, vocab 49,408; two layers), every parameter trainable: the gradients of
    `encode` fed a states gradient against fp32 transformers autograd fed the same one."""
    from transformers import CLIPTextConfig
    from transformers import CLIPTextModel as HF
    from t2v_b200.runtime import ParamArena
    from t2v_b200.text_encoder import DEFAULTS, CLIPTextModel
    cfg = dict(DEFAULTS, num_hidden_layers=2)
    hf = HF(CLIPTextConfig(**cfg))
    sd = {k: v for k, v in seeded_state_dict(hf, 9).items() if not k.endswith("position_ids")}
    hf.load_state_dict(sd, strict=False)
    ours = CLIPTextModel(cfg)
    ours.load_state_dict(sd)
    ours.requires_grad_(True)
    hf, ours = hf.cuda(), ours.cuda().train()
    arena = ParamArena(ours)   # the step's layout: bf16 shadows of the trainable projections
    g = torch.Generator().manual_seed(3)
    ids = torch.full((2, 77), VOCAB - 1, dtype=torch.int64)
    ids[:, :10] = torch.randint(0, VOCAB, (2, 10), generator=g)
    ids = ids.cuda()
    dstates = torch.randn(2, 77, 1024, generator=g).cuda().to(torch.bfloat16)
    out = ours.encode(ids)
    out.backward(dstates.view(out.shape))
    torch.cuda.synchronize()
    o = hf(ids)[0]
    o.backward(dstates.float())
    want = dict(hf.named_parameters())
    cos = {n: cosine(p.grad.float().cpu(), want[n].grad.float().cpu()) for n, p in ours.named_parameters()
           if want[n].grad.norm() > 1e-3 * max(q.grad.norm() for q in want.values() if q.grad is not None)}
    assert len(cos) >= 0.9 * len(want)
    assert sum(x > 0.98 for x in cos.values()) >= 0.97 * len(cos), sorted((v, k) for k, v in cos.items())[:5]
    assert arena.grad.abs().sum() > 0


def _tiny(seed=0):
    import torch.nn as nn
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.text_encoder import CLIPTextModel
    unet = UNet3DConditionModel(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)
    unet.load_state_dict(seeded_state_dict(unet, seed))
    unet.requires_grad_(False)
    for n, p in unet.named_parameters():
        if "attn2" in n:
            p.requires_grad_(True)
    for m in unet.modules():
        if isinstance(m, nn.Dropout):
            m.p = 0.0
    te = CLIPTextModel(dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, vocab_size=300))
    te.load_state_dict(seeded_state_dict(te, seed + 1))
    te.requires_grad_(True)
    return unet.cuda().train(), te.cuda().train()


def _collect():
    """Free captured graphs now: a CUDA graph that the cyclic garbage collector destroys while a later test is capturing
    would invalidate that capture."""
    import gc
    gc.collect()
    torch.cuda.synchronize()


def test_graph_replay_matches_eager():
    """The same seeded two-pass step, replayed as a CUDA graph and run eagerly, with FusedAdamW attached: same losses and
    the same text weights after three steps, within the run-to-run spread of the GEMMs' reduction order."""
    from t2v_b200 import step as S
    from t2v_b200.optim import FusedAdamW
    g = torch.Generator().manual_seed(11)
    lat, noise = torch.randn(1, 4, 4, 16, 16, generator=g).cuda(), torch.randn(1, 4, 4, 16, 16, generator=g).cuda()
    t = torch.tensor([500]).cuda()
    ids = torch.full((1, 77), 299, dtype=torch.int64)
    ids[0, :6] = torch.tensor([298, 5, 17, 40, 40, 77])
    ids = ids.cuda()
    res = {}
    for graph in (False, True):
        unet, te = _tiny()
        st = S.DataParallelStep(unet, S.ddpm_alphas_cumprod(device="cuda"), passes=2, use_graph=graph, text_encoder=te)
        opt = FusedAdamW(st.arena, [dict(params=[p for p in st.arena.params if p.requires_grad])], lr=1e-3, max_grad_norm=1.0)
        st.attach_optimizer(opt)
        losses = [st(lat, noise, t, ids).item() for _ in range(3)]
        res[graph] = losses, {n: p.detach().float().cpu().clone() for n, p in te.named_parameters()}
        del st, opt
        _collect()
    (l0, w0), (l1, w1) = res[False], res[True]
    assert all(abs(a - b) <= 1e-3 * abs(a) for a, b in zip(l0, l1)), (l0, l1)
    start = dict(_tiny()[1].named_parameters())
    for n in w0:
        if n.endswith("k_proj.bias"):   # zero gradient in exact arithmetic: AdamW turns its rounding noise into a full step
            continue
        d0 = w0[n] - start[n].detach().cpu()
        assert d0.norm() > 0, n
        # AdamW's g / (sqrt(v) + eps) turns the reduction-order rounding of a small gradient element into up to a full
        # +-lr step, so the trajectories may part by a few such steps
        assert (w1[n] - w0[n]).norm() <= 0.15 * d0.norm() + 1e-7 and (w1[n] - w0[n]).abs().max() <= 6e-3, n


@pytest.mark.parametrize("opt", ["fused_ema", "adamw8bit_ema"])
def test_train_main_optimizers_cover_text(tmp_path, opt):
    """train.main with CUDA graphs: FusedAdamW or 8-bit AdamW, both with the EMA, move every text parameter; the EMA lies
    between the start and the trained weights, and the saved `text_encoder_ema/` holds it."""
    from safetensors.torch import load_file
    from test_pipeline_train import _pipeline_folder, _run
    from t2v_b200.text_encoder import CLIPTextModel
    _collect()
    extra = dict(use_ema=True, ema_decay=0.5, use_8bit_adam=opt == "adamw8bit_ema")
    r, out, root = _run(tmp_path, "cuda:0", train_text_encoder=True, trainable_text_modules=["all"], save_pretrained_model=True,
                        max_train_steps=3, **extra)
    te, o = r["stepper"].text_encoder, r["optimizer"]
    start = dict(CLIPTextModel.from_pretrained(_pipeline_folder(str(tmp_path / "p")), subfolder="text_encoder").named_parameters())
    trained = {n: p.detach().cpu().clone() for n, p in te.named_parameters()}
    with o.ema_weights():
        ema = {n: p.detach().cpu().clone() for n, p in te.named_parameters()}
    moved = [n for n in trained if not torch.equal(trained[n], start[n].detach())]
    assert len(moved) == len(trained)
    assert sum(not torch.equal(ema[n], trained[n]) for n in trained) == len(trained)
    sd = load_file(os.path.join(out, "text_encoder_ema", "model.safetensors"))
    for n in ema:
        assert torch.equal(sd[n], ema[n]), n
    assert all(torch.isfinite(v).all() for v in trained.values())
    del r, te, o
    _collect()
