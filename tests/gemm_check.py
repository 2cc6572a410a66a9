"""Element-wise checks of the convolution GEMM entry points (prims.conv_fwd / conv_dgrad / conv_wgrad) against a float64
reference.  Shared by tests/test_gemm_step_gpu.py (the kernels, at every GEMM problem of a cfg-2 training step) and
tests/test_gemm_step_cpu.py (the same checks against the fp32 oracle and against deliberately broken outputs, without a GPU).

Reference r: the float64 result of the same operation on the same bf16 inputs.  Magnitude m: the same operation on absolute
values (|x| * |w| + |bias| + |rowbias| + |residual|, |x|^T |dy| (+ |dw|) for the weight gradient, sum |dy| (+ |dbias|) for the
bias gradient); it bounds every partial sum an fp32 accumulation can form.  Every element must satisfy
    bf16 output:                              |y - r| <= 2^-8 |r| + eps m    (one round-to-nearest of the fp32 result, fp32 accumulation)
    fp32 output, weight and bias gradients:   |y - r| <= eps m
and the relative L2 error must be at most 2^-8 (bf16 output) or 16 eps (fp32).  A tolerance relative to the tensor's largest
element (max|y - r| / max|r| < 1e-2, the metric of the per-kernel tests) lets small elements be wrong by many bf16 ulps; this
bound does not.

GroupNorm statistics from the conv_fwd epilogue are sums over the bf16 values the launch stores, the values the consumer reads
(include/t2v_b200.h; the split-K finishing pass and the standalone statistics pass sum the same values).  They are checked
against float64 sums of that output, which the element check ties to r:  per (frame, channel) over the n rows of the frame,
|S - sum y| <= n 2^-24 sum |y|  and  |Q - sum y^2| <= n 2^-24 sum y^2  (fp32 summation of n terms in any order; the squares of
bf16 values are exact in fp32).  The sums of the unrounded fp32 values (oracle/ops_ref.conv_fwd) differ from these by up to
2^-9 |y| per element, more than fp32 summation allows.

eps, per kind: the next power of two at or above 4x the largest |y - r| / m measured over the step's problems with fp32 output
(the data gradient through an fp32-output launch of the same plan), on one NVIDIA H100 80GB HBM3 at a 400 W power limit:
    fwd    1.55e-6 (2^-19.3, 16x8x8 2560 -> 1280 3x3, K = 23040, unsplit)      eps = 2^-17
    dgrad  1.17e-6 (2^-19.7, 16x16x16 1280 -> 1280 3x3)                         eps = 2^-17
    wgrad  1.90e-6 (2^-19.0, the bias gradient over 16384 rows; dw: 1.25e-6)     eps = 2^-17
The error grows with the length of an unsplit reduction; split-K problems stay near 1e-7.  tests/test_gemm_step_cpu.py holds eps
below the ceiling at which a residual added after rounding the accumulator is still rejected (about 2^-11)."""
import json
import math
import os
import sys
import zlib

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_gemm_plans as M  # noqa: E402

U_BF16 = 2.0 ** -8    # unit roundoff of round-to-nearest to bf16 (8 significand bits)
U_F32 = 2.0 ** -24
EPS = {"fwd": 2.0 ** -17, "dgrad": 2.0 ** -17, "wgrad": 2.0 ** -17}

DIMS = {"act": ("n", "h", "w", "c"), "weight": ("co", "kh", "kw", "ci"), "bias": ("co",), "stats": ("frame", "c")}


# ---------------------------------------------------------------------------------------------- problems
def _key(prob, env):
    return json.dumps([prob, env], sort_keys=True)


def step_records():
    """The records of tests/golden/gemm_plans.json that belong to the cfg-2 training step: every record that is not a case of
    tests/test_gemm_gpu.py (make_gemm_plans.test_problems())."""
    with open(M.OUT) as f:
        records = json.load(f)
    tests = {_key(p, e) for p, e in M.test_problems()}
    return [r for r in records if _key(r["problem"], r["env"]) not in tests]


def problem_id(p):
    s = f'{p["kind"]}-{p["N"]}x{p["H"]}x{p["W"]}-{p["Cin"]}to{p["Cout"]}-k{p["KH"]}x{p["KW"]}s{p["stride"]}'
    if p["pads"] != [0, 0, 0, 0]:
        s += "p" + "".join(map(str, p["pads"]))
    if p["stats_rows"]:
        s += f'-st{p["stats_rows"]}'
    if p["dbias"]:
        s += "-db"
    return s


def plans_on(rec, sm_count):
    """The launches the in-tree planner makes for `rec` on `sm_count` SMs (t2v_gemm_plan)."""
    from t2v_b200 import native
    return M.query(native.lib(), rec["problem"], rec["env"], sm_count)


def out_hw(p):
    return ((p["H"] + p["pads"][0] + p["pads"][1] - p["KH"]) // p["stride"] + 1,
            (p["W"] + p["pads"][2] + p["pads"][3] - p["KW"]) // p["stride"] + 1)


def rowbias_div(p):
    """Frames per clip of the per-clip time-embedding row: 16 when the batch is a multiple of 16 frames."""
    return 16 if p["N"] % 16 == 0 else 1


# ---------------------------------------------------------------------------------------------- inputs and references
def make_inputs(p, device):
    """Seeded inputs (seed = crc32 of the problem id): activations N(0, 1) bf16, weights N(0, 1/fan_in) bf16, a bias with mean
    0.5 (statistics carry a common mode), output gradients N(0.25, 1) (the bias gradient is not ~0)."""
    g = torch.Generator(device=device).manual_seed(zlib.crc32(problem_id(p).encode()))
    N, H, W, Ci, Co, KH, KW = (p[k] for k in ("N", "H", "W", "Cin", "Cout", "KH", "KW"))
    Ho, Wo = out_hw(p)

    def randn(*shape):
        return torch.randn(shape, device=device, generator=g)

    def weight():
        return (randn(Co, KH, KW, Ci) / math.sqrt(KH * KW * Ci)).bfloat16()

    if p["kind"] == "fwd":
        return {"x": randn(N, H, W, Ci).bfloat16(), "w": weight(), "bias": randn(Co) + 0.5,
                "rowbias": randn(N // rowbias_div(p), Co), "residual": randn(N, Ho, Wo, Co).bfloat16()}
    if p["kind"] == "dgrad":
        return {"dy": (randn(N, Ho, Wo, Co) + 0.25).bfloat16(), "w": weight(), "residual": randn(N, H, W, Ci).bfloat16()}
    return {"x": randn(N, H, W, Ci).bfloat16(), "dy": (randn(N, Ho, Wo, Co) + 0.25).bfloat16()}


def _conv(x, w, p):
    """NHWC convolution of float64 tensors (w [Co][KH][KW][Ci])."""
    pads = p["pads"]
    xp = F.pad(x.permute(0, 3, 1, 2), (pads[2], pads[3], pads[0], pads[1]))
    return F.conv2d(xp, w.permute(0, 3, 1, 2), stride=p["stride"]).permute(0, 2, 3, 1)


@torch.enable_grad()
def _dgrad(dy, w, p):
    x = torch.zeros((p["N"], p["H"], p["W"], p["Cin"]), dtype=dy.dtype, device=dy.device, requires_grad=True)
    return torch.autograd.grad(_conv(x, w, p), x, dy)[0]


@torch.enable_grad()
def _wgrad(x, dy, p):
    w = torch.zeros((p["Cout"], p["KH"], p["KW"], p["Cin"]), dtype=dy.dtype, device=dy.device, requires_grad=True)
    return torch.autograd.grad(_conv(x, w, p), w, dy)[0]


def reference(p, inp, epilogue=True):
    """{output name: (r, m, rounded, kind of eps, dims)} of the launch prims makes for problem `p` with inputs `inp`.
    fwd: `epilogue` adds bias, row bias and residual with bf16 output (the step's launch); otherwise a plain fp32 output.
    wgrad: accumulates into dw = 1 and, when the problem has it, dbias = 3."""
    d = {k: v.double() for k, v in inp.items()}
    a = {k: v.abs() for k, v in d.items()}
    kind = p["kind"]
    if kind == "fwd":
        r, m = _conv(d["x"], d["w"], p), _conv(a["x"], a["w"], p)
        if epilogue:
            rows = torch.arange(p["N"], device=r.device) // rowbias_div(p)
            for t in ("bias", "rowbias", "residual"):
                r = r + (d[t][rows][:, None, None, :] if t == "rowbias" else d[t])
                m = m + (a[t][rows][:, None, None, :] if t == "rowbias" else a[t])
        return {"y": (r, m, epilogue, "fwd", DIMS["act"])}
    if kind == "dgrad":
        r = _dgrad(d["dy"], d["w"], p) + d["residual"]
        m = _dgrad(a["dy"], a["w"], p) + a["residual"]
        return {"dx": (r, m, True, "dgrad", DIMS["act"])}
    out = {"dw": (1.0 + _wgrad(d["x"], d["dy"], p), 1.0 + _wgrad(a["x"], a["dy"], p), False, "wgrad", DIMS["weight"])}
    if p["dbias"]:
        out["dbias"] = (3.0 + d["dy"].reshape(-1, p["Cout"]).sum(0), 3.0 + a["dy"].reshape(-1, p["Cout"]).sum(0), False, "wgrad",
                        DIMS["bias"])
    return out


# ---------------------------------------------------------------------------------------------- checks
def _coords(flat, shape, names):
    out = []
    for n in reversed(shape):
        out.append(flat % n)
        flat //= n
    return ", ".join(f"{k}={v}" for k, v in zip(names, reversed(out)))


def _plan_text(plan):
    if not plan:
        return ""
    keys = ("block_n", "num_stages", "splits", "kb_per_split", "num_tiles", "box", "tdim", "kdim", "flags", "st", "follow")
    return "\n  plan: " + "; ".join(str({k: q[k] for k in keys}) for q in plan)


def _fail(what, ok, err, bound, y, r, m, shape, names, extra, plan):
    score = torch.where(ok, torch.full_like(err, -1.0), (err - bound) / bound.clamp_min(1e-300)).nan_to_num(nan=math.inf)
    i = int(score.flatten().argmax())
    yv, rv, mv, bv = (float(t.flatten()[i]) for t in (y, r, m, bound))
    raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of bound; worst at ({_coords(i, shape, names)}): "
                         f"y={yv!r} r={rv!r} m={mv!r} |y-r|={abs(yv - rv)!r} > bound {bv!r}{extra}{_plan_text(plan)}")


def check(y, r, m, eps, rounded, what, names, plan=None):
    """Asserts the per-element bound and the L2 bound of `y` against the float64 reference `r` with magnitude `m`.  Returns
    (max |y - r| / m, relative L2 error).  `names` label the dimensions in the report of the worst element."""
    assert y.shape == r.shape, (what, tuple(y.shape), tuple(r.shape))
    yd = y.double()
    err = (yd - r).abs()
    bound = eps * m + (U_BF16 * r.abs() if rounded else 0.0)
    ok = err <= bound                          # NaN compares false
    l2 = float((yd - r).norm() / r.norm().clamp_min(1e-300))
    l2_max = U_BF16 if rounded else 16 * eps
    ratio = float(torch.where(m > 0, err / m.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0)).nan_to_num(nan=math.inf).max())
    if not bool(ok.all()):
        _fail(what, ok, err, bound, yd, r, m, tuple(y.shape), names, f"; rel L2 {l2:.3e}", plan)
    assert l2 <= l2_max, f"{what}: relative L2 error {l2:.3e} > {l2_max:.3e}{_plan_text(plan)}"
    return ratio, l2


def check_stats(st, y, stats_rows, what, plan=None):
    """Asserts that the [frames][C][2] epilogue statistics `st` are the per-(frame, channel) sum and sum of squares of the bf16
    output `y` (rows flattened in [N][Ho][Wo] order, `stats_rows` rows per frame) up to fp32 summation."""
    C = y.shape[-1]
    yd = y.double().reshape(-1, stats_rows, C)
    assert tuple(st.shape) == (yd.shape[0], C, 2), (what, tuple(st.shape), tuple(yd.shape))
    sd = st.double()
    for j, (name, t, mag) in enumerate((("sum", yd, yd.abs()), ("sum of squares", yd * yd, yd * yd))):
        want, bound = t.sum(1), stats_rows * U_F32 * mag.sum(1)
        err = (sd[..., j] - want).abs()
        ok = err <= bound
        if not bool(ok.all()):
            _fail(f"{what} ({name})", ok, err, bound, sd[..., j], want, mag.sum(1), tuple(want.shape), DIMS["stats"], "", plan)


def check_outputs(ref, outs, what, plan=None):
    """check() of every output named in `ref` (reference()); returns {name: (ratio, l2)}."""
    return {name: check(outs[name], r, m, EPS[kind], rounded, f"{what} {name}", names, plan)
            for name, (r, m, rounded, kind, names) in ref.items()}


def old_metric(y, r):
    """max|y - r| / max|r|: the per-kernel tests' tolerance metric (they accept < 1e-2 for bf16 output)."""
    return float((y.double() - r).abs().max() / r.abs().max())
