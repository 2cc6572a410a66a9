"""cloneofsimo text-encoder LoRA on the H100: the gelu backward kernel, the injected encoder against transformers + an fp32
LoRA restatement (including one ViT-H-width layer), graph replay against eager, `train.main` with the reference's
train_config.yaml settings, and a profiler pass showing that the text forward + backward runs on the project's kernels."""
import os

import pytest
import torch
import torch.nn as nn

from test_text_lora_cpu import TRAIN_CONFIG, _rel, _restate, _tiny_models
from text_lora_ref import gelu_grad_f32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("quick", [False, True])
@pytest.mark.parametrize("n", [8, 77 * 4096, 3 * 1000 * 1000 + 8])
def test_gelu_bwd_matches_fp32_autograd(n, quick):
    from t2v_b200 import prims
    g = torch.Generator(device=DEV).manual_seed(n)
    x = (3 * torch.randn(n, device=DEV, generator=g)).to(torch.bfloat16)
    dy = torch.randn(n, device=DEV, generator=g).to(torch.bfloat16)
    xf = x.float().requires_grad_(True)
    y = xf * torch.sigmoid(1.702 * xf) if quick else torch.nn.functional.gelu(xf)
    (want,) = torch.autograd.grad(y, xf, dy.float())
    got = prims.gelu_bwd(x, dy, quick).float()
    # one bf16 rounding of the fp32 product (erff / __expf against torch's: at most one bf16 ulp apart)
    assert torch.all((got - want).abs() <= 2 ** -7 * want.abs() + 1e-30)
    assert torch.allclose(want, dy.float() * gelu_grad_f32(x, quick), rtol=1e-5, atol=1e-6)


def _pair(cfg, seed=0):
    from transformers import CLIPTextConfig
    from transformers import CLIPTextModel as HF
    from t2v_b200.text_encoder import CLIPTextModel
    from t2v_b200.utils.lora import inject_trainable_lora_extended
    torch.manual_seed(seed)
    hf = HF(CLIPTextConfig(**cfg)).eval()
    m = CLIPTextModel(cfg)
    m.load_state_dict({k: v for k, v in hf.state_dict().items() if not k.endswith("position_ids")})
    inject_trainable_lora_extended(m, {"CLIPEncoderLayer"}, r=16)
    for mod in m.modules():
        if hasattr(mod, "lora_up"):
            nn.init.normal_(mod.lora_up.weight, std=0.02)
    return hf, m.to(DEV).eval()


@pytest.mark.parametrize("cfg", [
    dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, vocab_size=100, hidden_act="gelu"),
    dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, vocab_size=100, hidden_act="quick_gelu"),
    dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=1, num_attention_heads=16, vocab_size=1000, hidden_act="gelu"),
], ids=["small-gelu", "small-quick", "vith-width-layer"])
def test_encoder_matches_transformers_fp32(cfg):
    cfg = dict(cfg, max_position_embeddings=77)
    hf, m = _pair(cfg)
    ids = torch.randint(0, cfg["vocab_size"], (2, 77), generator=torch.Generator().manual_seed(1))
    out = m.encode(ids.to(DEV))
    gcpu = torch.randn(out.shape, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16)
    out.backward(gcpu.to(DEV))
    torch.cuda.synchronize()
    ref = _restate(hf, m)
    o = hf(ids)[0]
    o.backward(gcpu.float().view(o.shape))
    assert _rel(out.float().cpu().view(o.shape), o) < 2e-2
    cos = []
    for n, w in m.named_modules():
        if hasattr(w, "lora_up"):
            for got, want in ((w.lora_up.weight.grad, ref[n].up.grad), (w.lora_down.weight.grad, ref[n].down.grad)):
                assert _rel(got.cpu(), want) < 5e-2, n
                cos.append(torch.nn.functional.cosine_similarity(got.cpu().double().flatten(), want.double().flatten(), dim=0).item())
    assert min(cos) > 0.998
    assert all(p.grad is None for n, p in m.named_parameters() if "lora" not in n)
    with torch.no_grad():
        ev = m(ids.to(DEV))[0].cpu()
    assert _rel(ev, o.detach()) < 2e-2


def test_graph_replay_matches_eager():
    from oracle import leaves as L
    from t2v_b200 import step as S
    unet, te = _tiny_models()
    unet, te = unet.to(DEV), te.to(DEV)
    abar = L.ddpm_alphas_cumprod().to(DEV)
    g = torch.Generator().manual_seed(5)
    args = (torch.randn(1, 4, 3, 8, 8, generator=g).to(DEV), torch.randn(1, 4, 3, 8, 8, generator=g).to(DEV),
            torch.tensor([300], device=DEV), torch.randint(0, 50, (1, 77), generator=g).to(DEV))
    stepper = S.DataParallelStep(unet, abar, passes=2, use_graph=False, text_encoder=te)
    text_params = [p for p in te.parameters() if p.requires_grad]

    def run():
        stepper.arena.zero_grads()
        loss = stepper(*args).item()
        return loss, torch.cat([p.grad.flatten() for p in text_params]).clone()
    loss_e, eager = run()
    _, eager2 = run()
    stepper.use_graph = True
    run()
    loss_g, graph = run()
    torch.cuda.synchronize()
    assert loss_g == pytest.approx(loss_e, rel=1e-3)
    assert all(p.grad.norm() > 0 for p in text_params)
    # the weight-gradient reductions add with red.add, so two eager steps differ too: the replay must stay within that spread
    spread, err = _rel(eager2, eager), _rel(graph, eager)
    assert err <= 3 * spread + 1e-3, (err, spread)
    assert torch.nn.functional.cosine_similarity(graph.double(), eager.double(), dim=0) > 0.999


@pytest.mark.parametrize("variant", ["adamw", "ema", "8bit"])
def test_train_main_train_config(tmp_path, variant, monkeypatch):
    """train.main with the train_config.yaml settings on the tiny pipeline (with a VAE decoder for the preview): cache_latents,
    CUDA graph, checkpoints, a preview through the LoRA encoder in eval mode, the LoRA files, the collapsed text_encoder/ and
    a reload through lora_path."""
    import test_pipeline_train
    import test_v_prediction_cpu as vp
    from test_pipeline_train import _run
    from t2v_b200 import sampling
    monkeypatch.setattr(test_pipeline_train, "_pipeline_folder", lambda root: vp._pipeline_folder(root, vp.ZEROSCOPE))
    previews, preview = [], sampling.validation_sample

    def spy(unet, vae, text_encoder, *a, **k):
        previews.append((text_encoder.lora_injected(), text_encoder.training, torch.is_grad_enabled()))
        return preview(unet, vae, text_encoder, *a, **k)
    monkeypatch.setattr(sampling, "validation_sample", spy)
    extra = {"ema": dict(use_ema=True), "8bit": dict(use_8bit_adam=True), "adamw": {}}[variant]
    vd = dict(prompt="a red ball", num_frames=2, width=64, height=64, num_inference_steps=2, guidance_scale=9, sample_preview=True)
    kw = {**TRAIN_CONFIG, **extra, **dict(cache_latents=True, checkpointing_steps=1, validation_steps=2, validation_data=vd,
                                          max_train_steps=2, learning_rate=1e-3)}
    r, out, root = _run(tmp_path, DEV, **kw)
    assert r["steps"] == 2
    te = r["stepper"].text_encoder
    moved = [m.lora_up.weight.detach().abs().max().item() for m in te.modules() if hasattr(m, "lora_up")]
    assert all(v > 0 for v in moved)   # the text LoRA trained (lora_up starts at zero)
    want = ["1_text_encoder.pt", "1_unet.pt"] + (["1_text_encoder_ema.pt", "1_unet_ema.pt"] if variant == "ema" else [])
    assert sorted(os.listdir(os.path.join(out, "checkpoint-1", "lora"))) == sorted(want)
    assert os.path.isfile(os.path.join(out, "text_encoder", "model.safetensors"))
    assert previews == [(True, False, False)]
    assert any(f.endswith(".mp4") for f in os.listdir(os.path.join(out, "samples")))
    saved = torch.load(os.path.join(out, "lora", "2_text_encoder.pt"))
    reload_dir = tmp_path / "reload"
    reload_dir.mkdir()
    torch.save(saved, reload_dir / "2_text_encoder.pt")
    r2, _, _ = _run(tmp_path / "second", DEV, **{**TRAIN_CONFIG, **dict(max_train_steps=0, lora_path=str(reload_dir),
                                                                      save_pretrained_model=False)})
    w2 = [m for m in r2["stepper"].text_encoder.modules() if hasattr(m, "lora_up")]
    assert all(torch.equal(w.lora_up.weight.detach().cpu(), saved[2 * i]) for i, w in enumerate(w2))


def _project_kernels():
    """Names of every __global__ function defined in the project's CUDA sources."""
    import glob
    import re
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "text-to-video-finetuning_b200", "csrc")
    names = set()
    for fn in glob.glob(os.path.join(src, "*.cu")) + glob.glob(os.path.join(src, "*.cuh")):
        text = open(fn).read()
        names |= set(re.findall(r"__global__\s+(?:void\s+)?(?:__launch_bounds__\([^)]*\)\s+)?(?:void\s+)?(\w+)\s*\(", text))
    return names


def test_text_forward_backward_runs_native_kernels():
    import re
    from torch.profiler import ProfilerActivity, profile
    ours = _project_kernels()
    assert {"gelu_bwd_kernel", "gelu_kernel"} <= ours
    _, m = _pair(dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=1, num_attention_heads=16, vocab_size=1000,
                      hidden_act="gelu", max_position_embeddings=77))
    m.train()
    ids = torch.randint(0, 1000, (1, 77), device=DEV)
    g = torch.randn(77, 1024, device=DEV).to(torch.bfloat16)
    m.encode(ids).backward(g)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.encode(ids).backward(g)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    foreign = sorted(n for n in names if not ours & set(re.findall(r"\w+", n)) and "memset" not in n.lower()
                     and "memcpy" not in n.lower())
    assert not foreign, foreign
    assert names
