"""`save_training_state` / `resume_from_checkpoint` on the H100 with the step replayed as a CUDA graph.  The GEMM weight
gradients accumulate with `red.add`, so two uninterrupted runs already differ in the last bits: a resumed run passes when
its relative distance to an uninterrupted run is within 3x the distance between two uninterrupted runs, plus 1e-3.  The
graphs the resumed run captures must hold the dropout seeds of the run it continues."""
import gc
import os

import pytest
import torch

from helpers import rel_l2
from test_resume_cpu import _main
from test_train_loop import _pretrained


def _record_capture_seeds(monkeypatch):
    """The dropout host seeds drawn while each CUDA graph is built (warm-up and capture), one list per graph."""
    from t2v_b200 import ops, runtime
    graphs, orig = [], runtime.GraphedStep.__init__

    def init(self, *a, **k):
        seeds, real = [], ops.next_dropout_seed

        def rec():
            s = real()
            seeds.append(s)
            return s
        ops.next_dropout_seed = rec
        try:
            orig(self, *a, **k)
        finally:
            ops.next_dropout_seed = real
        graphs.append(seeds)
    monkeypatch.setattr(runtime.GraphedStep, "__init__", init)
    return graphs


def _kw(root, **extra):
    kw = dict(pretrained_model_path=root, dataset_types=["synthetic"], train_data=dict(n=3, n_sample_frames=4, height=64, width=64),
              learning_rate=1e-3, checkpointing_steps=2, seed=0, shuffle=True, device="cuda:0", max_grad_norm=1.0, use_ema=True,
              use_unet_lora=True, lora_version="cloneofsimo", lora_rank=4, unet_lora_modules=["UNet3DConditionModel"],
              lora_unet_dropout=0.1, save_pretrained_model=False)
    kw.update(extra)
    return kw


def _run(**kw):
    """One train.main run -> its trainable weights (arena order), EMA, step counts and recorded capture keys.  The run's
    CUDA graphs are released here, before the next run captures its own."""
    r = _main(**kw)
    st, opt = r["stepper"], r["optimizer"]
    out = dict(w=torch.cat([p.detach().reshape(-1) for p in st.arena.params if p.requires_grad]).float().cpu(),
               ema=opt.ema.detach().float().cpu(), steps=r["steps"], opt_steps=opt.steps, graphs=len(st._graphs),
               use_graph=st.use_graph, keys=set(st.capture_rng))
    torch.cuda.synchronize()
    st._graphs = {}
    del r, st, opt
    gc.collect()
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["lora_fp32_ema", "full_8bit_ema"])
def test_resume_gpu_matches_uninterrupted(tmp_path, monkeypatch, variant):
    root, _ = _pretrained(tmp_path)
    extra = {} if variant == "lora_fp32_ema" else dict(use_unet_lora=False, use_8bit_adam=True, trainable_modules=["attn1", "attn2"])
    kw = _kw(root, **extra)
    graphs = _record_capture_seeds(monkeypatch)
    n, k = 5, 2
    a = _run(**kw, output_dir=str(tmp_path / "a"), max_train_steps=n)
    b = _run(**kw, output_dir=str(tmp_path / "b"), max_train_steps=n)
    assert a["use_graph"] and a["graphs"] == 1
    seeds_a = graphs[0]
    del graphs[:]
    part = _run(**kw, output_dir=str(tmp_path / "c"), max_train_steps=k, save_training_state=True)
    del graphs[:]
    c = _run(**kw, output_dir=str(tmp_path / "c"), max_train_steps=n, resume_from_checkpoint=str(tmp_path / "c" / f"checkpoint-{k}"))
    assert c["steps"] == n and c["opt_steps"] == n
    # the resumed run recaptured its graph from the recorded generator state: the seeds the uninterrupted run's graph holds
    assert len(graphs) == 1 and seeds_a and graphs[0] == seeds_a
    assert c["keys"] == a["keys"]
    for name in ("w", "ema"):
        noise, got = rel_l2(b[name], a[name]), rel_l2(c[name], a[name])
        assert got <= 3 * noise + 1e-3, (name, got, noise)
    assert not torch.equal(a["w"], part["w"])   # the resumed run trained on


@pytest.mark.gpu
def test_resume_gpu_checkpoint_contents_unchanged_when_off(tmp_path):
    """Without save_training_state a checkpoint holds exactly what it held before the option existed."""
    root, _ = _pretrained(tmp_path)
    out = str(tmp_path / "o")
    _run(**_kw(root), output_dir=out, max_train_steps=2)
    assert sorted(os.listdir(out)) == ["checkpoint-2", "lora"]
    assert sorted(os.listdir(os.path.join(out, "checkpoint-2"))) == ["lora"]
