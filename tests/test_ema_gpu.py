"""EMA of the trained weights on the GPU: both fused update kernels against the EMAModel restatement (tests/ema_ref.py) and
bit-identical to the kernels without EMA on everything else, the swap kernel's round trip, CUDA-graph replays of a small-UNet
step, and `train.main` with `use_ema`, LoRA and a validation preview."""
import contextlib
import os

import pytest
import torch

import ema_ref as ref

pytestmark = pytest.mark.gpu


def _rows_with_ema(rows, lens, offs, ema_base):
    """Append the EMA offset of each row's first element (rows lie inside one tensor)."""
    out = []
    for r in rows:
        i = max(j for j in range(len(offs)) if offs[j] <= r[0])
        out.append(tuple(r) + (ema_base[i] + r[0] - offs[i],))
    return torch.tensor(out, dtype=torch.int64)


def _ema_layout(lens):
    """EMA of the tensors in reverse order, so that a kernel that ignored the EMA column would be caught."""
    base, n = [0] * len(lens), 0
    for i in reversed(range(len(lens))):
        base[i] = n
        n += lens[i]
    return base, n


def _check_ema(ema_out, ema_in, p_out, rows, k, decay):
    """The kernel's EMA equals EMAModel.step on the kernel's own new weights, bit for bit."""
    want = ema_in.clone()
    omd = ref.one_minus_decay(k, decay)
    for off, n, e in rows:
        ref.ema_step(want[e:e + n], p_out[off:off + n], omd)
    assert torch.equal(ema_out, want), (k, decay, float((ema_out - want).abs().max()))


@pytest.mark.parametrize("bf16_grad", [False, True])
@pytest.mark.parametrize("k,decay", [(1, 0.9999), (2, 0.9999), (123456, 0.9999), (50, 0.5)])
def test_adamw_ema_kernel(bf16_grad, k, decay):
    from t2v_b200 import prims
    lens = [4160, 65856, 1024, 320]                 # ragged last rows: 65,856 = 65,536 + 320
    offs = [0, 4160, 70016, 71040]
    n_shadow = offs[3]                              # the last tensor has no bf16 shadow
    rows = [(o + lo, min(65536, n - lo)) for o, n in zip(offs, lens) for lo in range(0, n, 65536)]
    base, n_ema = _ema_layout(lens)
    ema_rows = _rows_with_ema(rows, lens, offs, base)
    total = offs[3] + lens[3]
    g = torch.Generator().manual_seed(k)
    st = {"p": torch.randn(total, generator=g), "g": torch.randn(total, generator=g) * 0.1, "m": torch.randn(total, generator=g) * 1e-2,
          "v": torch.rand(total, generator=g) * 1e-4, "shadow": torch.randn(total, generator=g).bfloat16()}
    g16 = (torch.randn(total, generator=g) * 0.1).bfloat16().cuda() if bf16_grad else None
    ema_in = torch.randn(n_ema, generator=g)
    hp = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 1e-2, 1 - 0.9 ** k, (1 - 0.999 ** k) ** 0.5, 0.7], dtype=torch.float32).cuda()
    a = {n: t.cuda() for n, t in st.items()}
    b = {n: t.cuda() for n, t in st.items()}
    ema, step = ema_in.cuda(), torch.tensor([k], dtype=torch.int64).cuda()
    prims.adamw_chunks(a["p"], a["g"], a["m"], a["v"], a["shadow"], n_shadow, torch.tensor(rows, dtype=torch.int64).cuda(), hp, True, g16)
    prims.adamw_ema_chunks(b["p"], b["g"], b["m"], b["v"], b["shadow"], n_shadow, ema_rows.cuda(), hp, ema, step, decay, True, g16)
    torch.cuda.synchronize()
    for n in st:
        assert torch.equal(a[n], b[n]), n
    assert int(step) == k
    _check_ema(ema.cpu(), ema_in, b["p"].cpu(), ema_rows[:, [0, 1, 2]].tolist(), k, decay)


@pytest.mark.parametrize("bf16_grad", [False, True])
@pytest.mark.parametrize("k,decay", [(1, 0.9999), (2, 0.9999), (123456, 0.9999), (50, 0.5)])
def test_adamw8bit_ema_kernel(bf16_grad, k, decay):
    from test_adamw8bit import _hp, _kernel_case
    from t2v_b200 import prims
    from t2v_b200.optim import dynamic_map
    st, tables, n_shadow, _, gen = _kernel_case(5)   # 8-bit rows with ragged blocks and rows, a 32-bit row, two sets
    lens, offs = [4160, 65856, 1024, 4224], [0, 4160, 70016, 71040]
    base, n_ema = _ema_layout(lens)
    ema_tables = [_rows_with_ema(t.tolist(), lens, offs, base) for t in tables]
    qmaps = torch.cat([dynamic_map(True), dynamic_map(False)]).cuda()
    st["g"] = torch.randn(st["p"].numel(), generator=gen) * 0.1
    g16 = (torch.randn(st["p"].numel(), generator=gen) * 0.1).bfloat16().cuda() if bf16_grad else None
    ema_in = torch.randn(n_ema, generator=gen)
    a = {n: t.cuda() for n, t in st.items()}
    b = {n: t.cuda() for n, t in st.items()}
    ema, step = ema_in.cuda(), torch.tensor([k], dtype=torch.int64).cuda()
    for table, et, hp in zip(tables, ema_tables, _hp(k)):
        hp = hp.cuda()
        prims.adamw8bit_chunks(a["p"], a["g"], a["shadow"], n_shadow, table.cuda(), hp, qmaps, a["m32"], a["v32"], a["code_m"], a["code_v"],
                               a["absmax_m"], a["absmax_v"], True, g16)
        prims.adamw8bit_ema_chunks(b["p"], b["g"], b["shadow"], n_shadow, et.cuda(), hp, qmaps, b["m32"], b["v32"], b["code_m"], b["code_v"],
                                   b["absmax_m"], b["absmax_v"], ema, step, decay, True, g16)
    torch.cuda.synchronize()
    for n in st:
        assert torch.equal(a[n], b[n]), n
    rows = torch.cat(ema_tables)[:, [0, 1, 4]].tolist()
    assert sum(r[1] for r in rows) == n_ema
    _check_ema(ema.cpu(), ema_in, b["p"].cpu(), rows, k, decay)


def test_swap_kernel_round_trip():
    from t2v_b200 import prims
    lens, offs = [4160, 65856, 1024, 320], [0, 4160, 70016, 71040]
    n_shadow = offs[3]
    total = offs[3] + lens[3] + 256                 # a tail no row covers
    rows = [(o + lo, min(65536, n - lo)) for o, n in zip(offs, lens) for lo in range(0, n, 65536)]
    base, n_ema = _ema_layout(lens)
    ema_rows = _rows_with_ema(rows, lens, offs, base).cuda()
    g = torch.Generator().manual_seed(9)
    p = torch.randn(total, generator=g).cuda()
    ema = torch.randn(n_ema, generator=g).cuda()
    shadow = p.bfloat16()
    p0, e0, s0 = p.clone(), ema.clone(), shadow.clone()
    prims.ema_swap_chunks(p, ema, shadow, n_shadow, ema_rows)
    torch.cuda.synchronize()
    for off, n, e in ema_rows.tolist():
        assert torch.equal(p[off:off + n], e0[e:e + n]) and torch.equal(ema[e:e + n], p0[off:off + n])
    assert torch.equal(p[-256:], p0[-256:])
    assert torch.equal(shadow[:n_shadow], p[:n_shadow].bfloat16()) and torch.equal(shadow[n_shadow:], s0[n_shadow:])
    prims.ema_swap_chunks(p, ema, shadow, n_shadow, ema_rows)
    torch.cuda.synchronize()
    assert torch.equal(p, p0) and torch.equal(ema, e0) and torch.equal(shadow, s0)


def test_graph_replays_use_each_steps_decay():
    """A small-UNet step with FusedAdamW(ema_decay) replayed as a CUDA graph, and the same step eager: after every step the
    EMA equals the restatement applied to that run's own weights (1e-6 relative), so the capture's dry runs left no trace
    and each replay read its own step count."""
    from helpers import seeded_state_dict
    from t2v_b200 import step as S
    from t2v_b200.models.unet_3d_condition import UNet3DConditionModel
    from t2v_b200.optim import FusedAdamW
    from oracle import leaves as L
    small = dict(block_out_channels=(64, 128, 128, 128), attention_head_dim=64, cross_attention_dim=64)
    g = torch.Generator().manual_seed(5)
    lat = (torch.randn(1, 4, 2, 8, 8, generator=g) * 0.9).cuda()
    noise = torch.randn(1, 4, 2, 8, 8, generator=g).cuda()
    ehs = torch.randn(1, 7, 64, generator=g).cuda()
    for graph in (False, True):
        m = UNet3DConditionModel(**small)
        m.load_state_dict(seeded_state_dict(m, 2))
        m = m.cuda().eval().requires_grad_(False)
        trainable = [p for n, p in m.named_parameters() if "attn" in n]
        for p in trainable:
            p.requires_grad_(True)
        st = S.DataParallelStep(m, L.ddpm_alphas_cumprod().cuda(), passes=1, use_graph=graph)
        opt = FusedAdamW(st.arena, trainable, lr=1e-3, max_grad_norm=1.0, ema_decay=0.7)
        st.attach_optimizer(opt)
        track = [p.detach().clone() for p in trainable]
        for k in range(1, 6):
            st(lat, noise, torch.tensor([100 * k], device="cuda"), ehs)
            omd = ref.one_minus_decay(k, 0.7)
            for p, t in zip(trainable, track):
                ref.ema_step(t, p.detach(), omd)
            with opt.ema_weights():
                ema = torch.cat([p.detach().reshape(-1) for p in trainable])
            want = torch.cat([t.reshape(-1) for t in track])
            assert float((ema - want).norm() / want.norm()) <= 1e-6 and float((ema - want).abs().max()) <= 1e-6 * float(want.abs().max()), (graph, k)
        assert opt.steps == 5
        assert not graph or len(st._graphs) == 1


def test_train_main_ema_lora_preview_gpu(tmp_path, monkeypatch):
    from test_v_prediction_cpu import ZEROSCOPE, _pipeline_folder
    from t2v_b200 import sampling, train
    from t2v_b200.optim import FusedAdamW
    root = _pipeline_folder(str(tmp_path / "pipe"), ZEROSCOPE)
    decoded, swaps = [], []
    dec, swap = sampling.decode_latents, FusedAdamW.ema_weights

    def d(vae, lat):
        decoded.append(lat.float().cpu())
        return dec(vae, lat)

    @contextlib.contextmanager
    def spy(self):
        before = [t.clone() for t in (self.arena.master, self.arena.shadow, self.ema)]
        with swap(self):
            yield
        swaps.append(all(torch.equal(a, b) for a, b in zip(before, (self.arena.master, self.arena.shadow, self.ema))))

    monkeypatch.setattr(sampling, "decode_latents", d)
    monkeypatch.setattr(FusedAdamW, "ema_weights", spy)
    out = str(tmp_path / "out")
    r = train.main(pretrained_model_path=root, output_dir=out, dataset_types=["synthetic"],
                   train_data=dict(n=2, n_sample_frames=4, height=64, width=64), max_train_steps=2, learning_rate=1e-4,
                   checkpointing_steps=1, seed=0, shuffle=False, device="cuda:0", eval_train=True, use_unet_lora=True,
                   lora_version="cloneofsimo", lora_rank=4, unet_lora_modules=["UNet3DConditionModel"], trainable_modules=None,
                   load_side_models=True, validation_steps=2, use_ema=True, ema_decay=0.9,
                   validation_data=dict(prompt="a dog", sample_preview=True, num_frames=4, width=32, height=32, num_inference_steps=2,
                                        guidance_scale=2.0))
    assert r["steps"] == 2 and r["optimizer"].steps == 2 and r["optimizer"].ema is not None
    assert r["stepper"].use_graph and len(r["stepper"]._graphs) == 1
    assert len(decoded) == 1 and torch.isfinite(decoded[0]).all()
    assert len(swaps) == 4 and all(swaps)    # checkpoint 1, preview, checkpoint 2, final save
    for d_, step in ((out, 2), (os.path.join(out, "checkpoint-1"), 1), (os.path.join(out, "checkpoint-2"), 2)):
        assert os.path.isfile(os.path.join(d_, "lora", f"{step}_unet_ema.pt")), d_
        assert os.path.isfile(os.path.join(d_, "unet_ema", "diffusion_pytorch_model.safetensors")), d_
