"""fp32/fp64 torch restatement of the text-encoder-training primitive prims.embed_tokens_bwd (csrc/elementwise.cu
embed_tokens_bwd_kernel), written from its contract: dtok[clamp(id)] += sum of the rows of dy with that id, dpos[l] += sum over b
of row (b, l), the ids clamped to [0, vocab) as the forward kernel clamps them, either gradient None when its table is frozen.
Used by the CPU tests (patched into prims next to oracle/ops_ref.py and tests/text_lora_ref.py) and as the reference of the GPU
kernel test."""
import contextlib

import torch


def embed_tokens_bwd(ids, dy, dtok, dpos, vocab, dtype=torch.float32):
    B, L = ids.shape
    g = dy.to(dtype).reshape(B * L, -1)
    if dtok is not None:
        acc = torch.zeros(dtok.shape, dtype=dtype, device=dtok.device)
        acc.index_add_(0, ids.reshape(-1).clamp(0, vocab - 1).to(dtok.device), g.to(dtok.device))
        dtok += acc.to(dtok.dtype)
    if dpos is not None:
        dpos[:L] += g.view(B, L, -1).sum(0).to(dpos.device, dpos.dtype)


@contextlib.contextmanager
def emulated():
    """The emulation of tests/ema_ref.py (oracle/ops_ref.py, 8-bit AdamW and the EMA) and tests/text_lora_ref.py (gelu_bwd),
    plus embed_tokens_bwd (tests only)."""
    import ema_ref
    import text_lora_ref
    from t2v_b200 import prims
    saved = prims.embed_tokens_bwd
    with ema_ref.emulated(), text_lora_ref.emulated():
        prims.embed_tokens_bwd = embed_tokens_bwd
        try:
            yield
        finally:
            prims.embed_tokens_bwd = saved
