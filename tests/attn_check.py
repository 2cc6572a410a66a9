"""Element-wise checks of the attention entry points (prims.flash_attn_fwd / flash_attn_bwd, attn_small_fwd / _bwd,
attn_long_fwd / _bwd, and the unfused bgemm / softmax / bgemm composite of ops._attn_core_fwd / _bwd and
ops.causal_attention_fwd) against a float64 reference.  Shared by tests/test_attn_step_gpu.py (the kernels, at every launch of
tests/golden/attn_launches.json) and tests/test_attn_step_cpu.py (the same checks against an fp32 restatement of the kernels
and against deliberately broken outputs, without a GPU).

Every launch is a set of Z = (batch or sequence) x heads independent problems Q [Lq, D], K, V [Lk, D], dO [Lq, D] (the
"canonical" form: gather() reads them out of the step's layout, scatter() writes them into it).  Reference, per problem, in
float64 from the bf16 inputs (causal: key j visible to query i only for j <= i):
    s = scale Q K^T,  P = softmax(s),  o = P V,  lse = logsumexp(s)
    dP = dO V^T,  delta = rowsum(dO o),  dS = P (dP - delta) scale,  dq = dS K,  dk = dS^T Q,  dv = P^T dO
Magnitudes, the same sums over absolute values:
    m_o = P |V|,  m_dv = P^T |dO|,  a = P (|dO| |V|^T + rowsum(|dO| m_o)) scale,  m_dq = a |K|,  m_dk = a^T |Q|
(delta's term uses m_o, not |o|: the kernels form delta from the stored bf16 O, whose own error is bounded in units of m_o, or as
rowsum(P dP), whose terms are bounded by |dO| P|V|.)  Every element must satisfy
    bf16 output:  |y - r| <= 2^-8 |r| + eps m
    lse (fp32):   |lse - r| <= eps_lse (1 + |r| + scale max_j sum_d |q_d k_jd|)
and the relative L2 error must be at most 2^-8 (bf16) or 16 eps_lse (lse).  P and dS are rounded to bf16 before their MMA by
design (8 significand bits), so eps is 2^-6 to 2^-9, not 2^-17 as for the GEMM: a rounding of every term of a sum costs up
to 2^-9 m.  The measured ratios follow: o and dv (a sum over bf16 P) reach 2^-8.2, dq and dk (over bf16 dS) 2^-10; lse
(fp32 throughout) 2^-22.4.  The old tolerance max|y - r| / max|r| < 1e-2 lets small rows be wrong by many ulps; this bound does not.

Inputs (make_inputs; seed = crc32 of the launch id, drawn on the CPU): q, k ~ 1.2 N(0, 1), v, dO ~ N(0, 1), dO with a per-row
mean of +-(0.5 .. 1.5) so that delta matters.  Key channel 0 is 2 for every key (a common-offset channel), key channel 1 is 2
on the keys of a ragged last 64-key tile (a tail channel).  Query rows i with i % 8 = t (every step-th of them, at most about
32 per problem and type) are shaped, and each property is asserted:
    t = 1  near-uniform: q = 0.02 N(0, 1); the row's max score within 1 of its mean
    t = 2  common offset: q_0 = 40 / (2 scale); every score of the row >= 30 above zero, lse about 40
    t = 3  peaked: q = beta k_j* on channels >= 2; key j* at least 20 above every other key of the row
    t = 4  (Lk > 64) q = beta k_j* with j* in the last key tile, 3 above the rest: the row max moves to the last tile, so the
           online-softmax rescale alpha of every earlier tile matters
    t = 5  (Lk % 64 != 0) the tail channel lifts the ragged last tile to >= 10 % of the row's P mass
The checks print the worst element's (problem, head, row, d), that row's max score and P mass in the ragged tile, and the
launch record when they fail.

eps, per kernel family and output: the next power of two at or above 4x the largest ratio (check()) measured in two full runs of
tests/test_attn_step_gpu.py, on one NVIDIA H100 80GB HBM3 at a 700 W power limit (1980 MHz max SM clock); values in EPS.
The two runs printed identical ratios for all 355 outputs, the dk / dv of the 20 split flash backwards (reduced with
red.add.f32) included.  The composite's eps come from its one launch with a backward (CLIP) and the VAE forward (o: 1.25e-03)."""
import json
import math
import os
import zlib

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LAUNCHES = os.path.join(HERE, "golden", "attn_launches.json")

U_BF16 = 2.0 ** -8
TILE = 64            # key tile of flash_attn.cu and attn_long; the ragged tile is the last one when Lk % 64 != 0
EPS = {                          # measured max ratio (launch)
    "flash.o": 2.0 ** -6,        # 2.56e-03  flash_attn_fwd 48x20h 16x16, qkv
    "flash.lse": 2.0 ** -20,     # 1.78e-07  flash_attn_fwd 16x5h 2880x2880
    "flash.dq": 2.0 ** -8,       # 8.10e-04  flash_attn_bwd 16x20h 180x180
    "flash.dk": 2.0 ** -8,       # 5.62e-04  flash_attn_bwd 48x20h 16x16, qkv
    "flash.dv": 2.0 ** -6,       # 2.86e-03  flash_attn_bwd 64x20h 16x16, qkv
    "small.o": 2.0 ** -6,        # 3.30e-03  attn_small_fwd 2880 seqs x 5h, L 16
    "small.dq": 2.0 ** -8,       # 5.69e-04  attn_small_bwd 2880 seqs x 8h, L 16
    "small.dk": 2.0 ** -8,       # 7.70e-04  attn_small_bwd 2880 seqs x 5h, L 16
    "small.dv": 2.0 ** -6,       # 3.06e-03  attn_small_bwd 2880 seqs x 5h, L 16
    "long.o": 2.0 ** -6,         # 2.28e-03  attn_long_fwd 1024 seqs x 5h, L 48
    "long.lse": 2.0 ** -20,      # 1.70e-07  attn_long_fwd 1024 seqs x 8h, L 256
    "long.dq": 2.0 ** -8,        # 6.07e-04  attn_long_bwd 1024 seqs x 8h, L 256
    "long.dk": 2.0 ** -8,        # 5.80e-04  attn_long_bwd 1024 seqs x 5h, L 48
    "long.dv": 2.0 ** -6,        # 2.80e-03  attn_long_bwd 1024 seqs x 8h, L 256
    "composite.o": 2.0 ** -6,    # 2.77e-03  composite 1x16h 77x77 causal (CLIP)
    "composite.dq": 2.0 ** -9,   # 4.35e-04  composite 1x16h 77x77 causal
    "composite.dk": 2.0 ** -7,   # 9.83e-04  composite 1x16h 77x77 causal
    "composite.dv": 2.0 ** -6,   # 2.29e-03  composite 1x16h 77x77 causal
}
PEAK_GAP, OFFSET, TAIL_MASS, UNIFORM_SPREAD = 20.0, 30.0, 0.10, 1.0
REF_CHUNK = 1 << 25   # score elements per float64 reference chunk (256 MB per matrix)
OUT_CHUNK = 1 << 24   # output elements per chunk (128 MB per float64 tensor)


def launches():
    with open(LAUNCHES) as f:
        return json.load(f)


def family(r):
    k = r["kind"]
    return "composite" if k == "composite" else k.split("_")[1] if k.startswith("attn_") else "flash"


def is_temporal(r):
    return "addr" in r


def launch_id(r):
    k = r["kind"]
    if is_temporal(r):
        nseq, inner, outer, inner_rows, seq_rows, ld_in, ld_out, heads, L, D = r["addr"]
        return f'{k}-n{nseq}x{heads}h-L{L}-d{D}-seq{seq_rows}-ld{ld_in}' + ("-qkv" if r["fused"] == "qkv" else "")
    s = f'{k}-{r["Nb"]}x{r["heads"]}h-{r["Lq"]}x{r["Lk"]}-d{r["D"]}-' + r["fused"]
    if k == "composite":
        s += (f'-causal{r["causal"]}' if r["causal"] else "") + ("-bwd" if r["bwd"] else "-fwd")
    elif k == "flash_attn_bwd":
        s += f'-s{r["splits_132"]}'
    return s


def geometry(r):
    """(Z, Lq, Lk, D, heads, causal) of the launch's canonical problems."""
    if is_temporal(r):
        nseq, heads, L, D = r["addr"][0], r["addr"][7], r["addr"][8], r["addr"][9]
        return nseq * heads, L, L, D, heads, False
    return r["Nb"] * r["heads"], r["Lq"], r["Lk"], r["D"], r["heads"], bool(r.get("causal", 0))


def has_bwd(r):
    return r["kind"].endswith("bwd") or (r["kind"] == "composite" and r["bwd"])


# ---------------------------------------------------------------------------------------------- layout
def seq_rows_index(addr, device):
    """[nseq, L] token row of (sequence z, frame l): (z / inner) outer_rows + (z % inner) inner_rows + l seq_rows."""
    nseq, inner, outer_rows, inner_rows, seq_rows = addr[:5]
    L = addr[8]
    z = torch.arange(nseq, device=device)
    return ((z // inner) * outer_rows + (z % inner) * inner_rows)[:, None] + torch.arange(L, device=device)[None] * seq_rows


def gather(r, t, heads, D, addr=None):
    """Canonical [Z, L, D] copy of a layout view: [Nb, L, heads*D] (flash / composite) or token rows [rows, heads*D] walked with
    the launch's SeqAddr (temporal; `addr` overrides it)."""
    if is_temporal(r):
        t = t[seq_rows_index(addr or r["addr"], t.device)]           # [nseq, L, C]
    n, L = t.shape[0], t.shape[1]
    return t.reshape(n, L, heads, D).permute(0, 2, 1, 3).reshape(n * heads, L, D)


def scatter(r, canon, t, heads, D, addr=None):
    """Writes canonical [Z, L, D] values into the layout view t (the inverse of gather)."""
    Z, L, _ = canon.shape
    v = canon.reshape(Z // heads, heads, L, D).permute(0, 2, 1, 3).reshape(Z // heads, L, heads * D).to(t.dtype)
    if is_temporal(r):
        t[seq_rows_index(addr or r["addr"], t.device)] = v
    else:
        t.copy_(v)


def layout(r, device, fill=None):
    """The step's buffers of launch r: {"q", "k", "v", "do"} views (column slices of one [.., 3C] or [.., 2C] projection where
    the step fuses them) and the underlying buffers under "buffers"; `fill`: their initial value."""
    Z, Lq, Lk, D, heads, _ = geometry(r)
    C = heads * D

    def new(*shape):
        return torch.full(shape, math.nan if fill is None else fill, dtype=torch.bfloat16, device=device)

    if is_temporal(r):
        rows = r["rows"]
        if r["fused"] == "qkv":
            qkv = new(rows, 3 * C)
            out = {"q": qkv[:, :C], "k": qkv[:, C:2 * C], "v": qkv[:, 2 * C:], "buffers": [qkv]}
        else:
            out = {n: new(rows, C) for n in "qkv"}
            out["buffers"] = [out["q"], out["k"], out["v"]]
        out["do"] = new(rows, r["addr"][6])
        return out
    Nb = r["Nb"]
    if r["fused"] == "qkv":
        qkv = new(Nb, Lq, 3 * C)
        out = {"q": qkv[..., :C], "k": qkv[..., C:2 * C], "v": qkv[..., 2 * C:], "buffers": [qkv]}
    elif r["fused"] == "kv":
        q, kv = new(Nb, Lq, C), new(Nb, Lk, 2 * C)
        out = {"q": q, "k": kv[..., :C], "v": kv[..., C:], "buffers": [q, kv]}
    else:
        out = {"q": new(Nb, Lq, C), "k": new(Nb, Lk, C), "v": new(Nb, Lk, C)}
        out["buffers"] = [out["q"], out["k"], out["v"]]
    out["do"] = new(Nb, Lq, C)
    return out


# ---------------------------------------------------------------------------------------------- inputs
def _gen(r):
    return torch.Generator().manual_seed(zlib.crc32(launch_id(r).encode()))


def _special_rows(Lq, t, lo=0):
    step = max(1, Lq // 256)
    i = torch.arange(t, Lq, 8)
    i = i[(i // 8) % step == 0]
    return i[i >= lo]


def _scores(Q, K, rows, causal, scale):
    """float64 [Z, n, Lk] scaled scores of query rows `rows`, masked keys -inf."""
    s = scale * (Q[:, rows].double() @ K.double().transpose(1, 2))
    if causal:
        s = s.masked_fill(torch.arange(K.shape[1])[None, None, :] > rows[None, :, None], -math.inf)
    return s


def _peak(Q, K, rows, targets, gap, causal, scale):
    """Q[:, rows, 2:] = beta K[:, target, 2:] with beta per row so that key `target` is `gap` above every other key."""
    kt = K[:, targets, 2:]                                                  # [Z, n, D-2]
    dots = kt @ K[:, :, 2:].transpose(1, 2)                                 # [Z, n, Lk]
    own = dots.gather(2, targets[None, :, None].expand(dots.shape[0], -1, 1)).squeeze(2)
    others = dots.scatter(2, targets[None, :, None].expand(dots.shape[0], -1, 1), -math.inf)
    if causal:
        others = others.masked_fill(torch.arange(K.shape[1])[None, None, :] > rows[None, :, None], -math.inf)
    beta = (gap * 1.25) / (scale * (own - others.max(2).values).clamp_min(1e-3))
    Q[:, rows] = 0
    Q[:, rows, 2:] = beta[..., None] * kt


def make_inputs(r, device="cpu"):
    """Canonical bf16 {"Q", "K", "V", "dO"} [Z, L, D] of launch r with the shaped rows of the module docstring (each property
    asserted), on `device`."""
    Z, Lq, Lk, D, heads, causal = geometry(r)
    scale = D ** -0.5
    g = _gen(r)
    Q = 1.2 * torch.randn(Z, Lq, D, generator=g)
    K = 1.2 * torch.randn(Z, Lk, D, generator=g)
    V = torch.randn(Z, Lk, D, generator=g)
    mu = (0.5 + torch.rand(Z, Lq, 1, generator=g)) * (torch.randint(0, 2, (Z, Lq, 1), generator=g) * 2 - 1)
    dO = torch.randn(Z, Lq, D, generator=g) + mu
    ragged = Lk % TILE != 0
    tail0 = (Lk - 1) // TILE * TILE                       # first key of the last tile
    K[..., 0] = 2.0
    K[..., 1] = 0.0
    if ragged:
        K[:, tail0:, 1] = 2.0
    Q[..., 1] = 0.0
    K = K.bfloat16().float()
    lo = TILE if causal else 0                            # causal rows before the last tile see one tile only

    rows_u = _special_rows(Lq, 1)
    Q[:, rows_u] = 0.02 * torch.randn(Z, len(rows_u), D, generator=g)
    rows_o = _special_rows(Lq, 2)
    Q[:, rows_o, 0] = OFFSET * 4 / 3 / (2 * scale)
    rows_p = _special_rows(Lq, 3, 1 if causal else 0) if Lk > 1 else rows_u[:0]
    if len(rows_p):
        lim = (rows_p + 1) if causal else torch.full_like(rows_p, Lk)
        _peak(Q, K, rows_p, (rows_p * 7919 + 13) % lim, PEAK_GAP, causal, scale)
    rows_l = _special_rows(Lq, 4, lo) if Lk > TILE else rows_u[:0]
    if len(rows_l):
        hi = (rows_l + 1).clamp_max(Lk) if causal else torch.full_like(rows_l, Lk)
        _peak(Q, K, rows_l, tail0 + (rows_l * 7919) % (hi - tail0), 3.0, causal, scale)
    rows_t = _special_rows(Lq, 5, lo) if ragged and Lk > TILE else rows_u[:0]
    if len(rows_t):
        Q[:, rows_t] *= 0.3
        Q[:, rows_t, 1] = 0
        s = _scores(Q.bfloat16().float(), K, rows_t, causal, scale)
        w = torch.softmax(s, -1)
        tail = w[..., tail0:].sum(-1).clamp(1e-30, 1 - 1e-12)
        boost = (math.log(0.25 / 0.75) - torch.log(tail / (1 - tail))).clamp_min(0)   # lifts the tail's share to 25 %
        Q[:, rows_t, 1] = (boost / (2 * scale)).float()
    out = {"Q": Q.bfloat16(), "K": K.bfloat16(), "V": V.bfloat16(), "dO": dO.bfloat16()}
    _assert_teeth(out, r, rows_u, rows_o, rows_p, rows_l, rows_t, tail0)
    return {n: t.to(device) for n, t in out.items()}


def _assert_teeth(inp, r, rows_u, rows_o, rows_p, rows_l, rows_t, tail0):
    Z, Lq, Lk, D, heads, causal = geometry(r)
    scale = D ** -0.5
    Q, K = inp["Q"].float(), inp["K"].float()
    what = launch_id(r)
    if Lk > 1:
        s = _scores(Q, K, rows_u, causal, scale)
        fin = torch.isfinite(s)
        mean = torch.where(fin, s, 0).sum(-1) / fin.sum(-1)
        assert float((s.max(-1).values - mean).max()) <= UNIFORM_SPREAD, f"{what}: near-uniform rows are not uniform"
    s = _scores(Q, K, rows_o, causal, scale)
    assert float(torch.where(torch.isfinite(s), s, math.inf).min()) >= OFFSET, f"{what}: offset rows below {OFFSET}"
    if len(rows_p):
        s = _scores(Q, K, rows_p, causal, scale)
        top = s.topk(2, -1).values
        assert float((top[..., 0] - top[..., 1]).min()) >= PEAK_GAP, f"{what}: peaked rows not {PEAK_GAP} above the rest"
    if Lk > TILE:
        s = _scores(Q, K, rows_l, causal, scale)
        assert bool((s.argmax(-1) >= tail0).all()), f"{what}: rows whose max is in the last key tile do not have it there"
    if len(rows_t):
        p = torch.softmax(_scores(Q, K, rows_t, causal, scale), -1)
        assert float(p[..., tail0:].sum(-1).min()) >= TAIL_MASS, f"{what}: ragged tile holds < {TAIL_MASS:.0%} of the P mass"
    rm = inp["dO"].double().mean(-1).abs()
    assert float(rm.mean()) >= 0.5, f"{what}: dO per-row mean too small for delta to matter"


# ---------------------------------------------------------------------------------------------- reference
def _mask(Lq, Lk, device):
    return torch.arange(Lk, device=device)[None, :] > torch.arange(Lq, device=device)[:, None]


def _chunk_reference(q, k, v, do, causal):
    """{output: (r, m)} in float64 of the problems q, k, v [z, L, D] (bf16): o and lse, and with dO `do` also dq, dk, dv (for
    lse, m is the bracket of its bound)."""
    Lq, D = q.shape[1:]
    Lk = k.shape[1]
    scale = D ** -0.5
    q, k, v = q.double(), k.double(), v.double()
    s = scale * (q @ k.transpose(1, 2))
    sa = scale * (q.abs() @ k.abs().transpose(1, 2))
    if causal:
        mask = _mask(Lq, Lk, q.device)
        s = s.masked_fill(mask, -math.inf)
        sa = sa.masked_fill(mask, 0)
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse[..., None])
    del s
    o, mo = P @ v, P @ v.abs()
    out = {"o": (o, mo), "lse": (lse, 1 + lse.abs() + sa.max(-1).values)}
    del sa
    if do is None:
        return out
    do = do.double()
    dS = P * (do @ v.transpose(1, 2) - (do * o).sum(-1, keepdim=True)) * scale
    a = P * (do.abs() @ v.abs().transpose(1, 2) + (do.abs() * mo).sum(-1, keepdim=True)) * scale
    out["dq"] = dS @ k, a @ k.abs()
    out["dk"] = dS.transpose(1, 2) @ q, a.transpose(1, 2) @ q.abs()
    out["dv"] = P.transpose(1, 2) @ do, P.transpose(1, 2) @ do.abs()
    return out


def _chunks(inp):
    """Slices of the problem axis such that one slice's float64 score matrices hold at most REF_CHUNK elements and its
    outputs at most OUT_CHUNK: the reference of the largest launch stays within a few GB."""
    Z, Lq, D = inp["Q"].shape
    Lk = inp["K"].shape[1]
    step = max(1, min(REF_CHUNK // (Lq * Lk), OUT_CHUNK // (max(Lq, Lk) * D)))
    return [slice(z0, min(Z, z0 + step)) for z0 in range(0, Z, step)]


def reference(inp, causal, bwd):
    """{output: (r, m)} in float64 of the whole launch (o and lse, and with `bwd` dq, dk, dv), computed chunk by chunk."""
    parts = [_chunk_reference(inp["Q"][sl], inp["K"][sl], inp["V"][sl], inp["dO"][sl] if bwd else None, causal) for sl in _chunks(inp)]
    return {n: tuple(torch.cat([p[n][i] for p in parts]) for i in (0, 1)) for n in parts[0]}


# ---------------------------------------------------------------------------------------------- checks
def _row_context(inp, z, row, key_side, causal, heads, label):
    """The worst element's problem / head / row and, for its query row, the max score and the P mass in the ragged tile."""
    Q, K = inp["Q"][z].double(), inp["K"][z].double()
    Lk, D = K.shape
    where = f"{label}={z // heads}, head={z % heads}, {'key' if key_side else 'row'}={row}"
    if key_side:
        s = D ** -0.5 * (Q @ K[row])
        if causal:
            s = s.masked_fill(torch.arange(Q.shape[0], device=s.device) < row, -math.inf)
        return f"({where}); scores of this key over the queries: max {float(s.max()):.4g}"
    s = D ** -0.5 * (K @ Q[row])
    if causal:
        s = s.masked_fill(torch.arange(Lk, device=s.device) > row, -math.inf)
    p = torch.softmax(s, 0)
    tail0 = (Lk - 1) // TILE * TILE
    return (f"({where}); row max score {float(s.max()):.4g} (mean {float(s[torch.isfinite(s)].mean()):.4g}), "
            f"P mass in the last key tile [{tail0}, {Lk}): {float(p[tail0:].sum()):.4g}")


def _elements(y, ref, m, eps, rounded, what, context):
    """The per-element bound of `y` (any chunk of an output): raises on the worst violation; returns (ratio, sum (y - r)^2,
    sum r^2)."""
    assert tuple(y.shape) == tuple(ref.shape), (what, tuple(y.shape), tuple(ref.shape))
    yd = y.double()
    err = (yd - ref).abs()
    bound = eps * m + (U_BF16 * ref.abs() if rounded else 0.0)
    ok = err <= bound                          # NaN compares false
    excess = (err - U_BF16 * ref.abs()).clamp_min(0) if rounded else err
    ratio = float(torch.where(m > 0, excess / m.clamp_min(1e-300), torch.where(excess > 0, math.inf, 0.0)).nan_to_num(nan=math.inf).max())
    if not bool(ok.all()):
        score = torch.where(ok, torch.full_like(err, -1.0), (err - bound) / bound.clamp_min(1e-300)).nan_to_num(nan=math.inf)
        i = int(score.flatten().argmax())
        yv, rv, mv, bv = (float(t.flatten()[i]) for t in (yd, ref, m, bound))
        ctx = context(i) if context else str(i)
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of bound; worst at {ctx}: y={yv!r} r={rv!r} "
                             f"m={mv!r} |y-r|={abs(yv - rv)!r} > bound {bv!r}")
    return ratio, float(((yd - ref) ** 2).sum()), float((ref ** 2).sum())


def _l2(what, e2, r2, rounded, eps):
    l2 = math.sqrt(e2) / max(math.sqrt(r2), 1e-300)
    l2_max = U_BF16 if rounded else 16 * eps
    assert l2 <= l2_max, f"{what}: relative L2 error {l2:.3e} > {l2_max:.3e}"
    return l2


def check(y, ref, m, key, rounded, what, context=None):
    """Asserts the per-element and L2 bounds of `y` against float64 `ref` with magnitude `m` (eps EPS[key]).  Returns
    (ratio, relative L2 error), ratio = max (|y - r| - 2^-8 |r|) / m for bf16 output, max |y - r| / m otherwise.  `context(flat
    index)` describes the worst element."""
    ratio, e2, r2 = _elements(y, ref, m, EPS[key], rounded, what, context)
    return ratio, _l2(what, e2, r2, rounded, EPS[key])


def check_outputs(r, inp, outs, what, ref=None):
    """check() of every canonical output in `outs` ({"o": [Z, Lq, D], "lse": [Z, Lq], "dq", "dk", "dv"}) of launch r with
    inputs `inp`; returns {name: (ratio, l2)}.  The reference is computed and compared one chunk of problems at a time unless
    a whole-launch `ref` (reference()) is given."""
    Z, Lq, Lk, D, heads, causal = geometry(r)
    bwd = any(n in outs for n in ("dq", "dk", "dv"))
    fam = family(r)
    label = "seq" if is_temporal(r) else "b"
    tally = {n: [0.0, 0.0, 0.0] for n in outs}
    for sl in ([slice(0, Z)] if ref is not None else _chunks(inp)):
        chunk = ref if ref is not None else _chunk_reference(inp["Q"][sl], inp["K"][sl], inp["V"][sl], inp["dO"][sl] if bwd else None,
                                                             causal)
        for name, y in outs.items():
            rv, m = chunk[name]
            shape = tuple(rv.shape)

            def context(i, shape=shape, name=name, z0=sl.start):
                z, rest = divmod(i, math.prod(shape[1:]))
                row = rest // shape[2] if len(shape) == 3 else rest
                d = f", d={rest % shape[2]}" if len(shape) == 3 else ""
                return _row_context(inp, z0 + z, row, name in ("dk", "dv"), causal, heads, label).replace(")", d + ")", 1) + \
                    f"\n  launch: {json.dumps(r)}"

            ratio, e2, r2 = _elements(y[sl], rv, m, EPS[f"{fam}.{name}"], name != "lse", f"{what} {name}", context)
            t = tally[name]
            t[0], t[1], t[2] = max(t[0], ratio), t[1] + e2, t[2] + r2
        del chunk
    return {n: (t[0], _l2(f"{what} {n}", t[1], t[2], n != "lse", EPS[f"{fam}.{n}"])) for n, t in tally.items()}


def old_metric(y, ref):
    """max|y - r| / max|r|: the per-kernel tests' tolerance metric (they accept < 1e-2, 1.5e-2 for gradients)."""
    return float((y.double() - ref).abs().max() / ref.abs().max())
