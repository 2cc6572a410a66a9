"""CPU restatement of prims.frames_u8_to_nhwc8_ragged in terms of the single-clip one in oracle/ops_ref.py, and a switch that
puts it in place of the native call for CPU runs (tests only)."""
import contextlib

import torch


def frames_u8_to_nhwc8_ragged(packed, table, out_hw):
    """packed uint8 [nbytes], table int64 [n, 4] = (byte offset, F, H0, W0) -> each clip resized alone, concatenated."""
    from oracle import ops_ref
    outs = []
    for off, F, H0, W0 in table.tolist():
        clip = packed[off:off + F * H0 * W0 * 3].view(F, H0, W0, 3)
        outs.append(ops_ref.frames_u8_to_nhwc8(clip, out_hw))
    return torch.cat(outs)


@contextlib.contextmanager
def emulated_ragged():
    """Use inside helpers.emulated_prims(): its swap covers the primitives oracle/ops_ref.py restates."""
    from t2v_b200 import prims
    saved = prims.frames_u8_to_nhwc8_ragged
    prims.frames_u8_to_nhwc8_ragged = frames_u8_to_nhwc8_ragged
    try:
        yield
    finally:
        prims.frames_u8_to_nhwc8_ragged = saved
