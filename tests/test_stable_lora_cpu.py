"""Stable LoRA (`lora_version: stable_lora`, utils/stable_lora.py) on CPU: the fixtures made from the reference's own
stable_lora/lora.py (tests/golden/make_golden_stable_lora.py) against this repo's modules over the emulated primitives
(oracle/ops_ref.py plus tests/stable_lora_ref.py), injection census, webui key map, checkpoint files and train.main."""
import contextlib
import io
import json
import os

import pytest
import torch

from helpers import rel_l2, seeded_state_dict
from oracle import ops_ref
from stable_lora_ref import patched_prims

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SMALL = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)
MODULE_CASES = ["linear", "linear_nobias_r4", "conv2d", "conv2d_s2", "conv2d_1x1", "conv3d"]


@contextlib.contextmanager
def fp32_prims():
    old = ops_ref.BF
    ops_ref.BF = torch.float32
    try:
        with patched_prims():
            yield
    finally:
        ops_ref.BF = old


def _quiet():
    return contextlib.redirect_stdout(io.StringIO())


def _modules():
    return torch.load(os.path.join(GOLD, "stable_lora_modules.pt"), weights_only=False)


def _small_model(seed=0):
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    m = UNet3DConditionModel(**SMALL)
    m.load_state_dict(seeded_state_dict(m, seed))
    return m


def build_module(c):
    """This repo's stable module for one fixture case, with the fixture's weights."""
    from t2v_b200.utils import stable_lora as S
    st, r = c["state"], c["r"]
    w = st["weight"]
    if c["kind"] == "Linear":
        m = S.Linear(w.shape[1], w.shape[0], r=r, lora_alpha=r, bias="bias" in st)
    elif c["kind"] == "Conv2d":
        m = S.Conv2d(w.shape[1], w.shape[0], w.shape[2], r=r, lora_alpha=r, stride=c["stride"], padding=c["padding"])
    else:
        m = S.Conv3d(w.shape[1], w.shape[0], 3, r=r, lora_alpha=r, stride=c["stride"], padding=c["padding"])
    m.load_state_dict(st)
    return m.eval()


def run_module(m, c, device, act):
    """Feed a fixture case through the module the way layers.run_linear / run_conv do; returns (y, dx) in the fixture layout."""
    x = c["x"].to(device)
    if c["kind"] == "Linear":
        xin = x.reshape(-1, x.shape[-1]).to(act).contiguous().requires_grad_(True)
        y = m(xin)
        y.backward(c["dy"].reshape(y.shape).to(device).to(act))
        return y.reshape(c["y"].shape), xin.grad.reshape(x.shape)
    if c["kind"] == "Conv2d":
        xin = x.permute(0, 2, 3, 1).to(act).contiguous().requires_grad_(True)
        y = m(xin)
        y.backward(c["dy"].permute(0, 2, 3, 1).to(device).to(act).contiguous())
        return y.permute(0, 3, 1, 2), xin.grad.permute(0, 3, 1, 2)
    B, C, F, H, W = x.shape   # (B, C, F, H, W) <-> [B, F, H*W, C]
    to_cl = lambda t: t.permute(0, 2, 3, 4, 1).reshape(B, F, H * W, t.shape[1])  # noqa: E731
    from_cl = lambda t: t.reshape(B, F, H, W, t.shape[-1]).permute(0, 4, 1, 2, 3)  # noqa: E731
    xin = to_cl(x).to(act).contiguous().requires_grad_(True)
    y = m(xin)
    y.backward(to_cl(c["dy"]).to(device).to(act).contiguous())
    return from_cl(y), from_cl(xin.grad)


def close(a, b, tol, what):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs().max().item() / max(b.abs().max().item(), 1e-6)
    assert err < tol, f"{what}: rel-to-max error {err:.3e} >= {tol}"


def check_module(name, device, act, tol):
    c = _modules()[name]
    m = build_module(c).to(device)
    y, dx = run_module(m, c, device, act)
    close(y, c["y"], tol, f"{name}: y")
    close(dx, c["dx"], 1.4 * tol, f"{name}: dx")
    for n in ("lora_A", "lora_B"):
        close(getattr(m, n).grad, c["grads"][n], 1.4 * tol, f"{name}: d{n}")
    assert m.weight.grad is None   # the frozen base never receives a gradient


# ------------------------------------------------------------------------------------------------ fixtures and oracle
def test_reference_over_loralib_standin_reproduces_fixtures():
    from oracle.reference_import import reference_available
    if not reference_available():
        pytest.skip("T2V_REFERENCE_ROOT does not point at a checkout of the reference")
    from golden import make_golden_stable_lora as G
    fresh = G.module_cases(G.ref_stable_lora())
    for name, c in _modules().items():
        for key in ("y", "dx"):
            assert torch.allclose(fresh[name][key], c[key], rtol=1e-5, atol=1e-6), (name, key)
        for n in ("lora_A", "lora_B"):
            assert torch.allclose(fresh[name]["grads"][n], c["grads"][n], rtol=1e-5, atol=1e-6), (name, n)


@pytest.mark.parametrize("name", MODULE_CASES)
def test_module_wiring_matches_reference_fixture(name):
    """y, dx, dA, dB of each wrapped layer over the fp32 emulated primitives against the reference class's autograd."""
    with fp32_prims():
        check_module(name, "cpu", torch.float32, 1e-4)


def test_injection_matches_reference_injector():
    from t2v_b200.utils import stable_lora as S
    c = torch.load(os.path.join(GOLD, "stable_lora_unet_small_f4.pt"), weights_only=False)
    m = _small_model()
    with _quiet():
        S.add_lora_to(m, ["UNet3DConditionModel"], [torch.nn.Linear, torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.Embedding], r=8,
                      dropout=0.1)()
    assert sorted((n, type(x).__name__) for n, x in m.named_modules() if hasattr(x, "lora_A")) == c["wrapped"]
    assert {n: tuple(p.shape) for n, p in m.named_parameters() if "lora_" in n} == c["shapes"]
    assert sorted(n for n, p in m.named_parameters() if p.requires_grad) == c["trainable"]
    # base keys unchanged: the wrapped modules share the original weight / bias Parameters under the same names
    plain = _small_model()
    assert sorted(k for k in m.state_dict() if "lora_" not in k) == sorted(plain.state_dict())
    conv = m.down_blocks[0].resnets[0].conv1
    assert conv.scaling == 1.0 and conv.lora_B.abs().max() == 0 and conv.weight.is_contiguous(memory_format=torch.channels_last)
    assert m.down_blocks[0].attentions[0].transformer_blocks[0].attn1.to_q.lora_dropout.p == 0.1


def test_small_unet_matches_reference_fixture():
    """Whole-model stable LoRA on the emulated primitives (fp32): loss, prediction and LoRA gradients."""
    from t2v_b200 import step as St
    c = _load_small_case()
    with fp32_prims():
        m = _small_stable(c, "cpu")
        loss, pred = St.finetune_loss(m, c["latents"], c["noise"], c["timesteps"], c["text"], St.ddpm_alphas_cumprod(), return_pred=True)
        loss.backward()
    assert abs(loss.item() - c["loss"].item()) <= 1e-5 * abs(c["loss"].item())
    assert rel_l2(pred.float(), c["pred"]) < 1e-4
    params = dict(m.named_parameters())
    for n, g_ref in c["grads"].items():
        assert rel_l2(params[n].grad, g_ref) < 1e-3, n


def _load_small_case():
    return torch.load(os.path.join(GOLD, "stable_lora_unet_small_f4.pt"), weights_only=False)


def _small_stable(c, device):
    """This repo's small UNet with the fixture's base and LoRA weights (same seeding as the generator)."""
    from golden.make_golden_stable_lora import seed_lora_
    from t2v_b200.utils import stable_lora as S
    m = _small_model(c["base_seed"])
    with _quiet():
        S.add_lora_to(m, ["UNet3DConditionModel"], [torch.nn.Linear, torch.nn.Conv2d, torch.nn.Conv3d, torch.nn.Embedding],
                      r=c["r"], dropout=0.1)()
    seed_lora_(m, c["lora_seed"])
    return m.to(device).eval()


# ------------------------------------------------------------------------------------------------ files
def test_webui_key_map_matches_reference_converter():
    """Every lora key of the ms-1.7b UNet maps to the webui key and shape the reference's converter produces."""
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.utils import stable_lora as S
    ref = json.load(open(os.path.join(GOLD, "stable_lora_webui_keys.json")))
    with torch.device("meta"):
        m = UNet3DConditionModel()
    with _quiet():
        S.add_lora_to(m, ["UNet3DConditionModel"], [torch.nn.Linear, torch.nn.Conv2d, torch.nn.Conv3d], r=ref["r"])()
    shapes = {k: list(v.shape) for k, v in m.state_dict().items() if "lora_" in k}
    assert shapes == {e["key"]: e["shape"] for e in ref["keys"]}
    for e in ref["keys"]:
        name, unsq = S.webui_key(e["key"])
        assert name == e["webui_key"], e
        assert (e["shape"] + [1] if unsq else e["shape"]) == e["webui_shape"], e


def _inject(m, r=4, **kw):
    from t2v_b200.utils.lora_handler import LoraHandler
    h = LoraHandler(version="stable_lora", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"], **kw)
    with _quiet():
        h.add_lora_to_model(True, m, h.unet_replace_modules, dropout=0.1, r=r)
    return h


def _randomise_lora(m, seed=4):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "lora_" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)


def test_save_files_webui_format_and_round_trip(tmp_path):
    from safetensors import safe_open
    from safetensors.torch import load_file
    from t2v_b200.utils.lora_handler import LoraHandler
    m = _small_model()
    h = _inject(m, save_for_webui=True)
    _randomise_lora(m)
    with _quiet():
        h.save_stable_lora(m, str(tmp_path / "lora"), 7)
    full = tmp_path / "lora" / "full_weights" / "7_lora_text_to_video_unet.safetensors"
    webui = tmp_path / "lora" / "webui_7_lora_text_to_video.safetensors"
    sd = load_file(str(full))
    own = {k: v for k, v in m.state_dict().items() if "lora_" in k}
    assert set(sd) == set(own) and all(v.dtype == torch.float32 for v in sd.values())
    with safe_open(str(webui), "pt") as f:
        meta = f.metadata()
        keys = list(f.keys())
        assert all(f.get_tensor(k).dtype == torch.float16 for k in keys)
    assert meta["stable_lora_text_to_video"] == "v1" and len(meta["lora_name"]) == len("lora_text_to_video_") + 5
    assert meta["lora_name"].startswith("lora_text_to_video_") and len(keys) == len(sd)
    # lora_path: a fresh model loads the full-weights file bit for bit
    m2 = _small_model()
    h2 = LoraHandler(version="stable_lora", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    with _quiet():
        h2.add_lora_to_model(True, m2, h2.unet_replace_modules, dropout=0.1, lora_path=str(full.parent), r=4)
    for k, v in m2.state_dict().items():
        if "lora_" in k:
            assert torch.equal(v, own[k]), k


def test_only_webui_skips_full_weights(tmp_path):
    m = _small_model()
    h = _inject(m, only_for_webui=True)
    with _quiet():
        written = h.save_stable_lora(m, str(tmp_path), 3)
    assert [os.path.basename(p) for p in written] == ["webui_3_lora_text_to_video.safetensors"]
    assert not os.path.exists(tmp_path / "full_weights")


def test_mismatched_file_raises(tmp_path):
    from t2v_b200.utils.lora_handler import LoraHandler
    m = _small_model()
    h = _inject(m, r=4)
    with _quiet():
        h.save_stable_lora(m, str(tmp_path), 1)
    m2 = _small_model()
    h2 = LoraHandler(version="stable_lora", use_unet_lora=True, unet_replace_modules=["UNet3DConditionModel"])
    with pytest.raises(ValueError, match="shape mismatch"), _quiet():   # rank 8 model, rank 4 file
        h2.add_lora_to_model(True, m2, h2.unet_replace_modules, lora_path=str(tmp_path / "full_weights"), r=8)
    bad = tmp_path / "bad"
    bad.mkdir()
    torch.save([torch.zeros(2)], bad / "1_unet.pt")   # a cloneofsimo file
    m3 = _small_model()
    with pytest.raises(ValueError), _quiet():
        h2.add_lora_to_model(True, m3, h2.unet_replace_modules, lora_path=str(bad), r=4)


def test_mixed_versions_and_text_lora_refused(tmp_path):
    from t2v_b200 import train
    from t2v_b200.utils import lora as mylora
    from t2v_b200.utils.lora_handler import LoraHandler
    m = _small_model()
    with _quiet():
        mylora.inject_trainable_lora_extended(m, {"UNet3DConditionModel"}, r=4)
    with pytest.raises(NotImplementedError):
        LoraHandler(version="stable_lora", use_unet_lora=True).add_lora_to_model(True, m, ["UNet3DConditionModel"])
    with pytest.raises(NotImplementedError):
        train.main(pretrained_model_path=str(tmp_path), output_dir=str(tmp_path / "o"), use_text_lora=True, device="cpu")


def test_lora_bias_behaves_as_none():
    from t2v_b200.utils import stable_lora as S
    m = _small_model()
    with pytest.warns(UserWarning, match="behaves as 'none'"), _quiet():
        S.add_lora_to(m, ["UNet3DConditionModel"], [torch.nn.Linear, torch.nn.Conv2d, torch.nn.Conv3d], r=4, lora_bias="all")()
    assert all("lora_" in n for n, p in m.named_parameters() if p.requires_grad)


def test_deactivate_lora_train_sets_modes():
    from t2v_b200.utils import stable_lora as S
    m = _small_model().train()
    h = _inject(m)
    h.deactivate_lora_train([m], True)
    assert not m.training and all(not x.training for x in m.modules() if isinstance(x, S.MODULES))
    h.deactivate_lora_train([m], False)
    assert m.training and all(x.training for x in m.modules() if isinstance(x, S.MODULES))


def test_merged_state_dict_reproduces_the_stable_model():
    """save_pretrained_model writes W + delta under the plain keys: a plain UNet loading it (strict) computes what the stable
    model computes."""
    from t2v_b200.utils import stable_lora as S
    m = _small_model()
    _inject(m)
    _randomise_lora(m)
    m.eval()
    plain = _small_model().eval()
    plain.load_state_dict(S.merged_state_dict(m), strict=True)
    x, t, ehs = torch.randn(1, 4, 2, 8, 8), torch.tensor([500]), torch.randn(1, 7, 64)
    with fp32_prims(), torch.no_grad():
        y = m(x, t, ehs).sample
        assert rel_l2(plain(x, t, ehs).sample, y) < 1e-5
        assert rel_l2(_small_model().eval()(x, t, ehs).sample, y) > 1e-3


# ------------------------------------------------------------------------------------------------ train.main
def test_train_main_default_version_cpu(tmp_path, capsys):
    """No lora_version key: stable_lora (the reference's default) trains 2 steps and writes its checkpoint files; the base
    weights stay bit-identical, and unet/ holds the merged weights under the plain keys."""
    from safetensors.torch import load_file
    from t2v_b200 import train
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.utils import stable_lora as S
    m = _small_model()
    root = str(tmp_path / "model")
    m.save_pretrained(os.path.join(root, "unet"))
    before = {k: v.clone() for k, v in m.state_dict().items()}
    out = str(tmp_path / "out")
    with patched_prims():
        r = train.main(pretrained_model_path=root, output_dir=out, dataset_types=["synthetic"],
                       train_data=dict(n=4, n_sample_frames=2, height=64, width=64), max_train_steps=2, learning_rate=1e-3,
                       checkpointing_steps=1, seed=0, shuffle=False, device="cpu", max_grad_norm=1.0, use_unet_lora=True,
                       lora_rank=4, unet_lora_modules=["UNet3DConditionModel"], save_lora_for_webui=True)
    assert r["steps"] == 2
    unet = r["stepper"].unet
    for step, where in ((1, os.path.join(out, "checkpoint-1")), (2, out)):
        lora = load_file(os.path.join(where, "lora", "full_weights", f"{step}_lora_text_to_video_unet.safetensors"))
        assert any(k.endswith("lora_B") and v.abs().max() > 0 for k, v in lora.items())
        assert os.path.isfile(os.path.join(where, "lora", f"webui_{step}_lora_text_to_video.safetensors"))
    final = load_file(os.path.join(out, "lora", "full_weights", "2_lora_text_to_video_unet.safetensors"))
    merged = UNet3DConditionModel.from_pretrained(out, subfolder="unet")   # strict load of the plain keys
    fresh = _small_model()
    _inject(fresh)
    fresh.load_state_dict({**before, **final}, strict=False)
    ref = S.merged_state_dict(fresh)
    for k, v in merged.state_dict().items():
        assert torch.allclose(v, ref[k], rtol=0, atol=1e-6), k
    for k, v in unet.state_dict().items():
        if "lora_" not in k:
            assert torch.equal(v.cpu(), before[k]), k
