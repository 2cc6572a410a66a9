"""Stable LoRA on the H100: the lora_delta.cu kernels' refusal of unsupported views (their element-wise check at every launch of
the stable-LoRA step is tests/test_optim_step_gpu.py), the module and small-UNet fixtures made from the reference's stable_lora/lora.py, and train.main with the CUDA-graph step."""
import contextlib
import io
import math
import os

import pytest
import torch

from helpers import cosine, rel_l2, seeded_state_dict
from test_stable_lora_cpu import (MODULE_CASES, SMALL, _load_small_case, _small_stable, check_module)

pytestmark = pytest.mark.gpu

DEV = "cuda:0"

def _factors(conv3d, k, cin, cout, r, seed=0):
    g = torch.Generator().manual_seed(seed)
    kh, kw = (3, 1) if conv3d else (k, k)
    base = torch.randn(cout, kh, kw, cin, generator=g) * 0.05
    A = torch.randn(r * k, cin * k, generator=g) / (cin * k) ** 0.5
    B = torch.randn(cout * k, r * k, generator=g) * 0.05
    return base.to(DEV), A.to(DEV), B.to(DEV)


def test_kernels_reject_unsupported_views():
    from t2v_b200 import native, prims
    base, A, B = _factors(False, 3, 16, 16, 4)
    lib = native.lib()
    rc = lib.t2v_lora_delta_merge(prims._p(base), prims._p(A), prims._p(B), 1.0, 5, 0, 16, 16, 4, prims._p(base), prims._stream())
    assert rc < 0 and b"kernel size" in lib.t2v_last_error()
    rc = lib.t2v_lora_delta_grad(prims._p(base), prims._p(A), prims._p(B), 1.0, 1, 1, 16, 16, 4, prims._p(A), prims._p(B), prims._stream())
    assert rc < 0


@pytest.mark.parametrize("name", MODULE_CASES)
def test_module_matches_reference_fixture_gpu(name):
    """The cloneofsimo module fixtures' bf16 tolerance (tests/test_lora_reference_golden.py, DESIGN §5)."""
    check_module(name, DEV, torch.bfloat16, 1.5e-2)


def test_small_unet_matches_reference_fixture_gpu():
    """Same bars as the cloneofsimo whole-model fixture (tests/test_lora_reference_golden.py)."""
    from t2v_b200 import step as S
    c = _load_small_case()
    m = _small_stable(c, DEV)
    m.requires_grad_(False)
    for n, p in m.named_parameters():
        p.requires_grad_("lora_" in n)
    loss, pred = S.finetune_loss(m, c["latents"].to(DEV), c["noise"].to(DEV), c["timesteps"].to(DEV), c["text"].to(DEV),
                                 S.ddpm_alphas_cumprod(device=DEV), return_pred=True)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - c["loss"].item()) <= 3e-3 * abs(c["loss"].item()), (loss.item(), c["loss"].item())
    assert rel_l2(pred.float().cpu(), c["pred"]) < 4e-2 and cosine(pred.float().cpu(), c["pred"]) > 0.999
    params = dict(m.named_parameters())
    assert sum(1 for n, p in params.items() if "lora_" in n and p.grad is not None) == c["n_lora"]
    top = max(c["grad_norms"].values())
    rel = sorted(abs(params[n].grad.float().norm().item() - gn) / gn for n, gn in c["grad_norms"].items() if gn > 1e-3 * top)
    assert len(rel) > 100 and rel[len(rel) // 2] < 2e-2 and rel[int(0.95 * len(rel))] < 0.1, (len(rel), rel[len(rel) // 2], rel[-5:])
    for n, g_ref in c["grads"].items():
        assert cosine(params[n].grad.float().cpu(), g_ref) > 0.98, n


def _train(tmp_path, tag, use_graph, **extra):
    from t2v_b200 import train
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    m.load_state_dict(seeded_state_dict(m, 0))
    root = str(tmp_path / "model")
    if not os.path.isdir(root):
        m.save_pretrained(os.path.join(root, "unet"))
    out = str(tmp_path / tag)
    kw = dict(pretrained_model_path=root, output_dir=out, dataset_types=["synthetic"], train_data=dict(n=4, n_sample_frames=4, height=64, width=64),
              max_train_steps=3, learning_rate=1e-3, checkpointing_steps=2, seed=0, shuffle=False, device=DEV, max_grad_norm=1.0,
              use_unet_lora=True, lora_rank=8, unet_lora_modules=["UNet3DConditionModel"], lora_unet_dropout=0.0,
              use_cuda_graph=use_graph, save_lora_for_webui=True, eval_train=True)   # eval_train: the UNet's own dropout off
    kw.update(extra)
    log = io.StringIO()
    with contextlib.redirect_stdout(log):
        r = train.main(**kw)
    r["log"] = log.getvalue()
    return r, out, {k: v.clone() for k, v in m.state_dict().items()}


def _step1_loss(log):
    return [float(ln.split("loss")[1].split()[0]) for ln in log.splitlines() if ln.startswith("step 1/")][0]


def _train_init(tmp_path):
    """The LoRA weights train.main starts from (seed 0: the model is built and injected right after manual_seed)."""
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.utils import stable_lora as S
    torch.manual_seed(0)
    m = UNet3DConditionModel.from_pretrained(str(tmp_path / "model"), subfolder="unet")
    with contextlib.redirect_stdout(io.StringIO()):
        S.add_lora_to(m, ["UNet3DConditionModel"], [torch.nn.Linear, torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.Embedding], r=8)()
    return {k: v.detach().cpu() for k, v in m.state_dict().items() if "lora_" in k}


def test_train_main_graph_matches_eager_and_checkpoints_reload(tmp_path):
    from safetensors.torch import load_file
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.utils.lora_handler import LoraHandler
    rg, out_g, before = _train(tmp_path, "graph", True)
    re_, out_e, _ = _train(tmp_path, "eager", False)
    assert rg["stepper"].use_graph and len(rg["stepper"]._graphs) == 1 and not re_["stepper"].use_graph
    sd_g = {k: v.detach().cpu() for k, v in rg["stepper"].unet.state_dict().items()}
    sd_e = {k: v.detach().cpu() for k, v in re_["stepper"].unet.state_dict().items()}
    # only lora_A / lora_B move; the frozen base is bit-identical
    for k, v in sd_g.items():
        if "lora_" not in k:
            assert torch.equal(v, before[k]), k
    lora_keys = [k for k in sd_g if "lora_" in k]
    assert any(sd_g[k].abs().max() > 0 for k in lora_keys if k.endswith("lora_B"))
    # graph and eager agree.  The first step's loss is the same computation; after it, AdamW turns every gradient element into a
    # step of about lr whatever its size, so elements whose gradient is near zero move by +-lr on the sign of run-to-run noise
    # (split-K red.add order): the updates are compared by direction, not bit for bit.
    l_g, l_e = _step1_loss(rg["log"]), _step1_loss(re_["log"])
    assert abs(l_g - l_e) <= 2e-3 * abs(l_e), (l_g, l_e)
    cat = lambda sd: torch.cat([sd[k].flatten() for k in lora_keys])  # noqa: E731
    init = cat(_train_init(tmp_path))
    assert cosine(cat(sd_g) - init, cat(sd_e) - init) > 0.9
    # checkpoints: the final full-weights file reloads into a fresh model bit for bit, unet/ loads strictly
    f = load_file(os.path.join(out_g, "lora", "full_weights", "3_lora_text_to_video_unet.safetensors"))
    for k in lora_keys:
        assert torch.equal(f[k], sd_g[k]), k
    assert os.path.isfile(os.path.join(out_g, "checkpoint-2", "lora", "webui_2_lora_text_to_video.safetensors"))
    UNet3DConditionModel.from_pretrained(out_g, subfolder="unet")
    m2 = UNet3DConditionModel(**SMALL)
    h = LoraHandler(version="stable_lora", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    with contextlib.redirect_stdout(io.StringIO()):
        h.add_lora_to_model(True, m2, h.unet_replace_modules, lora_path=os.path.join(out_g, "lora", "full_weights"), r=8)
    for k, v in m2.state_dict().items():
        if "lora_" in k:
            assert torch.equal(v, sd_g[k]), k


def test_train_main_stable_with_checkpointing_8bit_and_ema(tmp_path):
    """Gradient checkpointing (the merge runs again in the recompute), 8-bit AdamW and the EMA files."""
    r, out, _ = _train(tmp_path, "ckpt", True, gradient_checkpointing=True, use_8bit_adam=True, use_ema=True, ema_decay=0.9)
    sd = r["stepper"].unet.state_dict()
    assert all(math.isfinite(v.abs().max().item()) for k, v in sd.items() if "lora_" in k)
    files = os.listdir(os.path.join(out, "lora", "full_weights"))
    assert "3_lora_text_to_video_unet.safetensors" in files and "3_lora_text_to_video_unet_ema.safetensors" in files
    assert os.path.isfile(os.path.join(out, "lora", "webui_3_lora_text_to_video_ema.safetensors"))
    assert os.path.isdir(os.path.join(out, "unet_ema"))
