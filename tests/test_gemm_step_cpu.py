"""The checks of tests/gemm_check.py have teeth, shown without a GPU.  The fp32 oracle (oracle/ops_ref.py: fp32 accumulation,
one rounding to bf16) stands in for the kernel on step problems small enough for the CPU; the checks must accept its output with
the eps constants the GPU test uses, and must reject outputs broken the way a tiling, epilogue or reduction defect would break
them.  The old max|y - r| / max|r| < 1e-2 metric accepts a residual added after rounding the accumulator."""
import pytest
import torch

import gemm_check as C
from oracle import ops_ref as O

# (kind, N, H, W, Cin, Cout, KH, KW, stride, stats_rows, dbias): step problems the CPU can run in seconds
PROBLEMS = {
    "conv3x3_4x4_stats": ("fwd", 16, 4, 4, 1280, 1280, 3, 3, 1, 16, 0),       # deepest resnet conv, split-K, per-frame statistics
    "temporal_conv_16x16": ("fwd", 1, 16, 16, 1280, 1280, 3, 1, 1, 16, 0),    # h-line statistics (h = frame), K = 3840
    "wgrad_text_tokens": ("wgrad", 1, 1, 77, 1024, 320, 1, 1, 1, 0, 0),       # cross-attention K/V: ragged k-block of 13 rows
    "dgrad_stride2": ("dgrad", 16, 8, 8, 1280, 1280, 3, 3, 2, 0, 0),          # Downsample2D: one launch per parity class
    "wgrad_time_emb_proj": ("wgrad", 1, 1, 1, 1280, 320, 1, 1, 1, 0, 1),      # W = 1: one real pixel in a 64-pixel k-block
}


def _record(name):
    kind, N, H, W, Ci, Co, KH, KW, s, rows, db = PROBLEMS[name]
    pads = [KH // 2, KH // 2, KW // 2, KW // 2]
    for rec in C.step_records():
        p = rec["problem"]
        if (p["kind"], p["N"], p["H"], p["W"], p["Cin"], p["Cout"], p["KH"], p["KW"], p["stride"], p["pads"], p["stats_rows"],
                p["dbias"]) == (kind, N, H, W, Ci, Co, KH, KW, s, pads, rows, db):
            return rec
    raise AssertionError(f"{name} is not a step problem of tests/golden/gemm_plans.json")


_CACHE = {}


def _case(name):
    """(problem, inputs, reference, oracle outputs) of a named problem, computed once."""
    if name not in _CACHE:
        rec = _record(name)
        p = rec["problem"]
        inp = C.make_inputs(p, "cpu")
        pads = tuple(p["pads"])
        if p["kind"] == "fwd":
            y = O.conv_fwd(inp["x"], inp["w"], inp["bias"], inp["rowbias"], inp["residual"], p["stride"], pads,
                           rowbias_div=C.rowbias_div(p))
            outs = {"y": y, "stats": O.channel_stats(y.reshape(-1, p["stats_rows"], p["Cout"])) if p["stats_rows"] else None}
        elif p["kind"] == "dgrad":
            outs = {"dx": O.conv_dgrad(inp["dy"], inp["w"], (p["H"], p["W"]), p["stride"], pads, inp["residual"])}
        else:
            dw = torch.ones((p["Cout"], p["KH"], p["KW"], p["Cin"]))
            db = torch.full((p["Cout"],), 3.0) if p["dbias"] else None
            O.conv_wgrad(inp["x"], inp["dy"], dw, p["stride"], pads, db)
            outs = {"dw": dw, "dbias": db}
        _CACHE[name] = (rec, inp, C.reference(p, inp), outs)
    return _CACHE[name]


def _check(name, outs):
    """Every check the GPU test applies to the step's launch of `name`, on `outs`."""
    rec, _, ref, _ = _case(name)
    p = rec["problem"]
    C.check_outputs(ref, outs, name, rec["plans"]["132"])
    if p["kind"] == "fwd" and p["stats_rows"]:
        C.check_stats(outs["stats"], outs["y"], p["stats_rows"], f"{name} stats", rec["plans"]["132"])


def test_selection_matches_gpu_parametrization():
    recs = C.step_records()
    kinds = [r["problem"]["kind"] for r in recs]
    assert (len(recs), kinds.count("fwd"), kinds.count("dgrad"), kinds.count("wgrad")) == (192, 74, 52, 66)
    assert len({C.problem_id(r["problem"]) for r in recs}) == len(recs)
    import test_gemm_step_gpu as G
    (mark,) = [m for m in G.test_step_gemm.pytestmark if m.name == "parametrize"]
    assert mark.args[1] == recs


@pytest.mark.parametrize("name", list(PROBLEMS))
def test_oracle_output_passes(name):
    rec, inp, ref, outs = _case(name)
    _check(name, outs)
    if rec["problem"]["kind"] == "fwd":   # the plain fp32-output launch
        p = rec["problem"]
        y32 = O.conv_fwd(inp["x"], inp["w"], stride=p["stride"], pads=tuple(p["pads"]), out_fp32=True)
        C.check_outputs(C.reference(p, inp, epilogue=False), {"y": y32}, f"{name} plain fp32")


def _frame_outputs(name, rowbias_times):
    """The oracle's fwd output with frame 5's time-embedding row added `rowbias_times` times."""
    rec, inp, _, outs = _case(name)
    p = rec["problem"]
    rb = inp["rowbias"].clone()
    rb[5 // C.rowbias_div(p)] *= rowbias_times
    y5 = O.conv_fwd(inp["x"][5:6], inp["w"], inp["bias"], rb[5 // C.rowbias_div(p)][None], inp["residual"][5:6], p["stride"],
                    tuple(p["pads"]))
    y = outs["y"].clone()
    y[5] = y5[0]
    return {"y": y, "stats": O.channel_stats(y.reshape(-1, p["stats_rows"], p["Cout"]))}


def _dropped_kblock():
    """One k-block (input channels 64..127 of the centre tap) left out of the second 128-row tile (frames 8..15)."""
    rec, inp, _, outs = _case("conv3x3_4x4_stats")
    p = rec["problem"]
    w = inp["w"].clone()
    w[:, 1, 1, 64:128] = 0
    y2 = O.conv_fwd(inp["x"], w, inp["bias"], inp["rowbias"], inp["residual"], p["stride"], tuple(p["pads"]),
                    rowbias_div=C.rowbias_div(p))
    y = outs["y"].clone()
    y.view(-1, p["Cout"])[128:256] = y2.view(-1, p["Cout"])[128:256]
    return {"y": y, "stats": O.channel_stats(y.reshape(-1, p["stats_rows"], p["Cout"]))}


def _stats_mutation(how):
    rec, _, _, outs = _case("conv3x3_4x4_stats")
    st = outs["stats"].clone()
    if how == "missing":
        st[6] = 0
    else:   # frame 6's sums added to frame 7
        st[7] += st[6]
        st[6] = 0
    return {"y": outs["y"], "stats": st}


def _ragged_tile(how):
    """dw of the 77-token projection: rows 256..319 (Cout 320 = two full 128-row tiles and a ragged one) not written, or
    holding the previous tile's values."""
    _, _, _, outs = _case("wgrad_text_tokens")
    dw = outs["dw"].clone()
    dw[256:320] = float("nan") if how == "nan" else dw[128:192]
    return {"dw": dw, "dbias": None}


def _dbias_without_ragged_kblock():
    """The bias gradient of time_emb_proj without the rows of its only (ragged) k-block: nothing added to dbias = 3."""
    _, _, _, outs = _case("wgrad_time_emb_proj")
    return {"dw": outs["dw"], "dbias": torch.full_like(outs["dbias"], 3.0)}


MUTATIONS = {
    "kblock_dropped_from_one_tile": ("conv3x3_4x4_stats", _dropped_kblock),
    "ragged_row_tile_unwritten": ("wgrad_text_tokens", lambda: _ragged_tile("nan")),
    "ragged_row_tile_previous_values": ("wgrad_text_tokens", lambda: _ragged_tile("previous")),
    "frame_stats_missing": ("conv3x3_4x4_stats", lambda: _stats_mutation("missing")),
    "frame_stats_to_neighbour": ("conv3x3_4x4_stats", lambda: _stats_mutation("neighbour")),
    "rowbias_twice_in_one_frame": ("conv3x3_4x4_stats", lambda: _frame_outputs("conv3x3_4x4_stats", 2.0)),
    "rowbias_missing_in_one_frame": ("conv3x3_4x4_stats", lambda: _frame_outputs("conv3x3_4x4_stats", 0.0)),
    "dbias_without_ragged_kblock": ("wgrad_time_emb_proj", _dbias_without_ragged_kblock),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_rejected(mutation):
    name, make = MUTATIONS[mutation]
    with pytest.raises(AssertionError, match="out of bound"):
        _check(name, make())


def test_double_rounding_rejected_and_missed_by_old_metric():
    """The residual added after the accumulator (with bias and row bias) was rounded to bf16: y = bf16(bf16(acc) + residual).
    Where the residual cancels the accumulator the error is up to 2^-9 |acc|, far above 2^-8 |y| but below 1e-2 max|y|."""
    name = "temporal_conv_16x16"
    rec, inp, ref, _ = _case(name)
    p = rec["problem"]
    acc = O.conv_fwd(inp["x"], inp["w"], inp["bias"], inp["rowbias"], None, p["stride"], tuple(p["pads"]), out_fp32=True,
                     rowbias_div=C.rowbias_div(p))
    y = (acc.bfloat16().float() + inp["residual"].float()).bfloat16()
    assert C.old_metric(y, ref["y"][0]) < 1e-2
    with pytest.raises(AssertionError, match="out of bound"):
        _check(name, {"y": y, "stats": O.channel_stats(y.reshape(-1, p["stats_rows"], p["Cout"]))})
