"""Every GEMM problem of a cfg-2 training step (the step records of tests/golden/gemm_plans.json), run through the prims entry
points the step calls (so split-K scratch, follow-up passes and epilogue variants are chosen as in training) and checked element
by element against a float64 reference (tests/gemm_check.py).

  fwd:   the step's epilogue (bias, per-clip row bias, residual, bf16 output, GroupNorm statistics when the problem has them)
         and a plain fp32-output run;
  dgrad: with the residual (gradient fan-in), bf16 output; the same plan with fp32 output measures the accumulation error;
  wgrad: accumulated into dw = 1 and, with the fused bias gradient, dbias = 3.
On 132 or 114 SMs the plans are pinned to the table first, so the numbers checked are those of the pinned plans.  fwd and dgrad
launches without a split write their output without atomics, so a second call must reproduce it bit for bit (CUDA-graph
replays rely on that).  Each check prints one GEMMCHECK line: max |y - r| / m and the relative L2 error."""
import ctypes

import pytest
import torch

import gemm_check as C

pytestmark = pytest.mark.gpu

RECORDS = C.step_records()


def _plans(rec):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got = C.plans_on(rec, sms)
    want = rec["plans"].get(str(sms))
    if want is not None:
        assert got == want, f"{C.problem_id(rec['problem'])}: the planner moved on {sms} SMs:\n  table {want}\n  now   {got}"
    return got


def _report(pid, res):
    for name, (ratio, l2) in res.items():
        print(f"GEMMCHECK {pid} {name} ratio={ratio:.3e} l2={l2:.3e}")


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _fwd(p, inp, plan, pid):
    from t2v_b200 import prims
    Ho, Wo = C.out_hw(p)
    rows = p["stats_rows"]

    def run():
        st = prims.stats_alloc(p["N"] * Ho * Wo // rows, p["Cout"], inp["x"].device) if rows else None
        y = prims.conv_fwd(inp["x"], inp["w"], inp["bias"], inp["rowbias"], inp["residual"], p["stride"], tuple(p["pads"]),
                           rowbias_div=C.rowbias_div(p), stats=st, stats_rows=rows)
        return y, st

    y, st = run()
    res = C.check_outputs(C.reference(p, inp), {"y": y}, pid, plan)
    if rows:
        C.check_stats(st, y, rows, f"{pid} stats", plan)
    if all(q["splits"] == 1 for q in plan):
        y2, _ = run()
        assert torch.equal(_bits(y), _bits(y2)), f"{pid}: a second call changed the output"
    y32 = prims.conv_fwd(inp["x"], inp["w"], stride=p["stride"], pads=tuple(p["pads"]), out_fp32=True)
    res["y_fp32"] = C.check_outputs(C.reference(p, inp, epilogue=False), {"y": y32}, f"{pid} plain fp32", plan)["y"]
    return res


def _dgrad(p, inp, plan, pid):
    from t2v_b200 import native, prims

    def run():
        return prims.conv_dgrad(inp["dy"], inp["w"], (p["H"], p["W"]), p["stride"], tuple(p["pads"]), inp["residual"])

    dx = run()
    ref = C.reference(p, inp)
    res = C.check_outputs(ref, {"dx": dx}, pid, plan)
    if all(q["splits"] == 1 for q in plan):
        assert torch.equal(_bits(dx), _bits(run())), f"{pid}: a second call changed the output"
    # the same plan with fp32 output: the accumulation error without the final rounding
    N, H, W, Ci, Co, KH, KW, s = (p[k] for k in ("N", "H", "W", "Cin", "Cout", "KH", "KW", "stride"))
    dx32 = torch.empty((N, H, W, Ci), device="cuda", dtype=torch.float32)
    nb = native.lib().t2v_conv_workspace_bytes(1, N, H, W, Ci, Co, KH, KW, s, *p["pads"])
    ws = torch.empty(max(nb, 4) // 4, device="cuda", dtype=torch.float32)
    epi = native.Epilogue(None, None, inp["residual"].data_ptr(), 1.0, 1, 1, ws.data_ptr() if nb > 0 else None, nb)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    native.check(native.lib().t2v_conv_dgrad(ctypes.c_void_p(inp["dy"].data_ptr()), ctypes.c_void_p(inp["w"].data_ptr()),
                                             ctypes.c_void_p(dx32.data_ptr()), N, H, W, Ci, Co, KH, KW, s, *p["pads"],
                                             ctypes.byref(epi), stream))
    r, m, _, kind, names = ref["dx"]
    res["dx_fp32"] = C.check(dx32, r, m, C.EPS[kind], False, f"{pid} dx fp32", names, plan)
    return res


def _wgrad(p, inp, plan, pid):
    from t2v_b200 import prims
    dw = torch.ones((p["Cout"], p["KH"], p["KW"], p["Cin"]), device="cuda", dtype=torch.float32)
    db = torch.full((p["Cout"],), 3.0, device="cuda", dtype=torch.float32) if p["dbias"] else None
    prims.conv_wgrad(inp["x"], inp["dy"], dw, p["stride"], tuple(p["pads"]), db)
    return C.check_outputs(C.reference(p, inp), {"dw": dw, "dbias": db}, pid, plan)


@pytest.mark.parametrize("rec", RECORDS, ids=[C.problem_id(r["problem"]) for r in RECORDS])
def test_step_gemm(rec):
    p = rec["problem"]
    pid = C.problem_id(p)
    plan = _plans(rec)
    inp = C.make_inputs(p, "cuda")
    res = {"fwd": _fwd, "dgrad": _dgrad, "wgrad": _wgrad}[p["kind"]](p, inp, plan, pid)
    _report(pid, res)
