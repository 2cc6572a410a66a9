"""Element-wise checks of the optimizer kernels (csrc/optim.cu), the stable-LoRA delta kernels (csrc/lora_delta.cu) and the
gradient compression (scale_cast_f32_bf16) against a float64 reference written from each operation's definition, not from
oracle/ops_ref.py, tests/adamw8bit_ref.py or tests/ema_ref.py.  Shared by tests/test_optim_step_gpu.py (the kernels, at every
launch of tests/golden/optim_launches.json, on the real chunk tables) and tests/test_optim_step_cpu.py (the same checks against
fp32 restatements and deliberately broken outputs, without a GPU).

Definitions (hp: the set's fp32 row lr, beta1, beta2, eps, weight_decay, bc1, sqrt(bc2), clip, read as float64):
    AdamW (torch.optim.AdamW, decoupled decay first)   g' = clip g;  p' = p (1 - lr wd);  m' = b1 m + (1 - b1) g';
                                                       v' = b2 v + (1 - b2) g'^2;  p'' = p' - (lr / bc1) m' / (sqrt(v') / sqrt(bc2) + eps)
    clip (clip_grad_norm_)                             min(1, max_norm / (norm + 1e-6))
    8-bit (optim.AdamW8bit)                            m = map_m[code] absmax_m (v alike), the update above, absmax' = max |m'| of
                                                       the 256-block, code' = the smallest i with m' / absmax' <= (map[i] + map[i+1]) / 2
                                                       (the code of 0.0 when absmax' = 0)
    EMA (diffusers EMAModel)                           d_1 = 0, d_k = min(decay, k / (9 + k));  e' = e - (1 - d) (e - p'')
    stable-LoRA delta (loralib)                        W = base + s view(B A) (Conv3d: the mean of the three columns of each triple);
                                                       dA += B^T dBA, dB += dBA A^T with dBA = s view^T(dW) (Conv3d: dW / 3 on each)
    compression                                        x / world
Magnitude m: the same expression on absolute values.  Every element must satisfy
    fp32 outputs (p, m, v, EMA, absmax, sum of squares with m = r, dA, dB)   |y - r| <= eps m + 2^-149
    bf16 outputs (the merged weight, the compression at world 6)              |y - r| <= 2^-8 |r| + eps m
    8-bit codes   the code of the float64 value, or a neighbour when the value lies within eps (m' / absmax' + |x| max_block m /
                  absmax') of the midpoint between them.  A float64 value exactly on a midpoint accepts both codes: bf16 gradients
                  at k = 1 put m' / absmax' exactly on a midpoint in float64 while the kernel's fp32 quotient of two rounded
                  values lands on either side (426 of 33.5 M codes of the full AdamW8bit table on the H100)
    adamw_prepare bias terms and clip factor within 1 fp32 ulp of float32(1 - b1^k), float32(sqrt(1 - b2^k)) and the clip factor;
                  the step count + 1 exactly; sq[1] = sqrt(sq[0]) and sq[0] back to 0
and bit for bit: the bf16 shadow (RNE of the new p, rows below n_shadow only), the zeroed gradients, the EMA against fp32
EMAModel.step on the kernel's own new p, the ema_swap round trip, and the compression at world 2 and 8 (fp32(1 / world) x is
exact there) against RNE of the exact product.  Every element no row covers (frozen gaps, the shadow past n_shadow, the 8-bit
block padding, the guard elements around every buffer) holds SENTINEL and must come back unchanged.

Inputs repeat one seeded odd-length PATTERN per buffer (element i of a buffer holds pattern[i % PATTERN]), with exact zeros in g
and v, tiny v where eps dominates, and magnitudes over many decades.  Two states per update launch: k = 1 from the zero state
a run starts from (m = v = 0, codes of 0.0, absmax 0) with no clipping, and k = 1000 from random moments with clip 0.3712.

eps: the next power of two at or above 4x the largest ratio measured over the census and both states on one NVIDIA H100 80GB
HBM3 at a 700 W power limit (EPS), 2^-22 where nothing beyond one rounding shows up.  No kernel exceeded its bound; the check
found no kernel defect in this family."""
import json
import math
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LAUNCHES = os.path.join(HERE, "golden", "optim_launches.json")

U_BF16 = 2.0 ** -8
EPS = {                       # measured max ratio (launch, state)
    "p": 2.0 ** -19,          # 3.80e-07  adamw8bit_ema_chunks stable_lora AdamW8bit+ema, k 1000
    "m": 2.0 ** -21,          # 1.16e-07  adamw8bit_ema_chunks full AdamW8bit+ema, k 1000
    "v": 2.0 ** -20,          # 2.26e-07  adamw8bit_ema_chunks full AdamW8bit+ema, k 1000
    "ema": 2.0 ** -19,        # 3.97e-07  adamw8bit_ema_chunks full AdamW8bit+ema+g16, k 1000
    "absmax": 2.0 ** -20,     # 2.24e-07  adamw8bit_ema_chunks full AdamW8bit+ema, k 1000
    "code": 2.0 ** -22,       # band of the 8-bit codes: no code outside it
    "sq": 2.0 ** -23,         # 2.33e-08  sqnorm_chunks full FusedAdamW
    "merge": 2.0 ** -21,      # 9.26e-08  lora_delta_merge
    "dA": 2.0 ** -20,         # 1.52e-07  lora_delta_grad
    "dB": 2.0 ** -20,         # 1.76e-07  lora_delta_grad Cout 320, Cin 4, k 3
    "cast": 2.0 ** -22,       # 0         scale_cast_f32_bf16 world 6
}
SUBNORMAL = 2.0 ** -149         # fp32 outputs: plus one subnormal spacing (a subnormal result has no relative precision)
PATTERN = (1 << 20) + 7
SLAB = 1 << 25                  # elements per reference slab
CLIP = 0.3712                   # the clip factor of the k = 1000 state
STATES = ((1, False), (1000, True))   # (k, from random moments with clipping)
SENT32 = 0x7FBADA55             # a signalling-NaN payload no kernel writes
SENT16 = 0x7FA5
SENT8 = 0xA5
QBLOCK = 256


def launches():
    with open(LAUNCHES) as f:
        return json.load(f)


def launch_id(r):
    skip = ("hist", "rows", "hp")
    fields = "-".join(f"{k}{v[:12] if k == 'sha256' else v}" for k, v in r.items() if k not in skip and k != "kind")
    return f'{r["kind"]}-{fields}'


def table(r):
    """The launch's int64 host table: its "rows" (synthetic) or the generator's table with the recorded digest."""
    if "rows" in r:
        return torch.tensor(r["rows"], dtype=torch.int64)
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_optim_launches as MO
    t = MO.tables()[r["sha256"]]
    assert MO.digest(t) == r["sha256"]
    return t


def qmaps():
    from t2v_b200.optim import dynamic_map
    return torch.cat([dynamic_map(True), dynamic_map(False)])


# ---------------------------------------------------------------------------------------------- patterns
def patterns(seed, device):
    """{buffer: fp32 pattern of PATTERN elements} (codes: uint8, g16: bf16 values)."""
    g = torch.Generator().manual_seed(seed)
    n = PATTERN

    def decades(lo, hi):
        return torch.randn(n, generator=g, dtype=torch.float64) * 10.0 ** (lo + (hi - lo) * torch.rand(n, generator=g, dtype=torch.float64))

    def zeros(x, frac):
        return torch.where(torch.rand(n, generator=g) < frac, torch.zeros_like(x), x)

    p = zeros(decades(-6, 1), 0.01)
    p[::997] = 1e-30
    gr = zeros(decades(-9, 0), 0.02)
    m = zeros(decades(-9, -1), 0.01)
    v = zeros(decades(-18, -2) ** 2, 0.02).abs()
    v[::101] = 1e-24                         # sqrt(v) / sqrt(bc2) far below eps
    e = p * (1 + 0.01 * torch.randn(n, generator=g, dtype=torch.float64))
    out = {"p": p, "g": gr, "m": m, "v": v, "ema": e}
    out = {k: t.float().to(device) for k, t in out.items()}
    out["g16"] = decades(-9, 0).bfloat16().to(device)
    out["qm"] = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8).to(device)
    out["qv"] = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8).to(device)
    am = 10.0 ** (-6 + 5 * torch.rand(n, generator=g, dtype=torch.float64))
    am[::13] = 0.0
    out["am"] = am.float().to(device)
    out["av"] = (am * am).float().to(device)
    return out


def pat(P, idx):
    return P[idx % PATTERN]


# ---------------------------------------------------------------------------------------------- guarded buffers
GUARD = 4096


class Buf:
    """A SENTINEL-filled buffer of n elements with GUARD sentinel elements on each side; `covered` marks written elements."""

    def __init__(self, n, dtype, device):
        self.n, self.dtype = n, dtype
        self.flat = torch.empty(n + 2 * GUARD, dtype=dtype, device=device)
        self.bits().fill_(sentinel(dtype))
        self.t = self.flat[GUARD:GUARD + n]
        self.covered = torch.zeros(n, dtype=torch.bool, device=device)

    def bits(self, t=None):
        t = self.flat if t is None else t
        return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.uint8: torch.uint8}[self.dtype])

    def assert_untouched(self, what):
        s = sentinel(self.dtype)
        b = self.bits()
        assert bool((b[:GUARD] == s).all() and (b[-GUARD:] == s).all()), f"{what}: a guard element was written"
        inner = self.bits(self.t)
        for a in range(0, self.n, SLAB):
            e = min(self.n, a + SLAB)
            bad = (inner[a:e] != s) & ~self.covered[a:e]
            if bool(bad.any()):
                i = a + int(bad.nonzero()[0])
                raise AssertionError(f"{what}: element {i} outside every row was written ({int(bad.sum())} in [{a}, {e}))")


def sentinel(dtype):
    return {torch.float32: SENT32, torch.bfloat16: SENT16, torch.uint8: SENT8}[dtype]


# ---------------------------------------------------------------------------------------------- row batches
def batches(tab, limit=SLAB):
    """Consecutive groups of whole rows of at most `limit` elements (one row if it is longer)."""
    out, lo, acc = [], 0, 0
    lens = tab[:, 1].tolist()
    for i, n in enumerate(lens):
        if acc and acc + n > limit:
            out.append((lo, i))
            lo, acc = i, 0
        acc += n
    out.append((lo, len(lens)))
    return out


def expand(starts, lens, device):
    """The element indices of rows (start, len): cat(arange(s, s + n))."""
    starts, lens = starts.to(device), lens.to(device)
    tot = int(lens.sum())
    first = torch.cumsum(lens, 0) - lens
    return torch.repeat_interleave(starts - first, lens, output_size=tot) + torch.arange(tot, device=device)


# ---------------------------------------------------------------------------------------------- float64 definitions
def hp_row(hp5, k, clip):
    """The set's 8-float row as adamw_prepare writes it (fp32 of the exact values)."""
    lr, b1, b2, eps, wd = (float(torch.tensor(x, dtype=torch.float32)) for x in hp5)
    return torch.tensor([lr, b1, b2, eps, wd, 1 - b1 ** k, math.sqrt(1 - b2 ** k), clip], dtype=torch.float32)


def adamw_ref(p, g, m, v, hp):
    """float64 AdamW of one element vector; returns {name: (r, m)} for p, m, v and the update magnitude."""
    lr, b1, b2, eps, wd, bc1, sbc2, clip = (float(x) for x in hp)
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    gc = clip * g
    pd = p * (1 - lr * wd)
    m1 = b1 * m + (1 - b1) * gc
    mm1 = (b1 * m).abs() + ((1 - b1) * gc).abs()
    v1 = b2 * v + (1 - b2) * gc * gc
    mv1 = (b2 * v).abs() + (1 - b2) * gc * gc
    den = v1.sqrt() / sbc2 + eps
    upd = (lr / bc1) * m1 / den
    mupd = (lr / bc1) * mm1 / den
    return {"p": (pd - upd, pd.abs() + mupd), "m": (m1, mm1), "v": (v1, mv1)}


def ema_d(k, decay):
    return 0.0 if k <= 1 else min(float(torch.tensor(decay, dtype=torch.float32)), k / (9.0 + k))


def ema_ref(e, p1, mp1, k, decay):
    d = ema_d(k, decay)
    e = e.double()
    return e - (1 - d) * (e - p1), e.abs() + (1 - d) * (e.abs() + mp1)


def ema_fp32(e, p_new, k, decay):
    """EMAModel.step in fp32 on the kernel's own new p: s -= (1 - d) * (s - p), each operation rounded."""
    omd = torch.tensor(1.0 - ema_d(k, decay), dtype=torch.float64).float()
    return e - omd * (e - p_new)


def mids(qmap):
    q = qmap.double()
    return 0.5 * (q[:-1] + q[1:])


def code_ref(x, band, qmap, zero_code, absmax_zero):
    """(reference code, lower acceptable, upper acceptable) of normalised values x (float64) with tolerance band."""
    md = mids(qmap).to(x.device)
    c = torch.searchsorted(md, x.contiguous(), side="left").clamp(max=255)
    lo_ok = (c > 0) & ((x - md[(c - 1).clamp(min=0)]).abs() <= band)
    hi_ok = (c < 255) & ((md[c.clamp(max=254)] - x).abs() <= band)
    zc = torch.full_like(c, zero_code)
    c = torch.where(absmax_zero, zc, c)
    return c, torch.where(absmax_zero, zc, c - lo_ok.long()), torch.where(absmax_zero, zc, c + hi_ok.long())


# ---------------------------------------------------------------------------------------------- element checks
def _ratio(err, m):
    pos = m > 0
    r = torch.where(pos, err / m.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.nan_to_num(nan=math.inf).max()) if err.numel() else 0.0


def check(y, r, m, key, what, rounded=False):
    """|y - r| <= eps m (+ 2^-8 |r| for a bf16 output); returns (ratio, relative L2)."""
    yd = y.double()
    err = (yd - r).abs()
    eps = EPS[key]
    bound = eps * m + (U_BF16 * r.abs() if rounded else SUBNORMAL)
    ok = err <= bound
    l2 = float((yd - r).norm() / r.norm().clamp_min(1e-300)) if y.numel() else 0.0
    excess = (err - (U_BF16 * r.abs() if rounded else SUBNORMAL)).clamp_min(0)
    if not bool(ok.all()):
        score = torch.where(ok, torch.full_like(err, -1.0), (err - bound) / bound.clamp_min(1e-300)).nan_to_num(nan=math.inf)
        i = int(score.argmax())
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of bound; worst at {i}: y={float(yd[i])!r} "
                             f"r={float(r[i])!r} m={float(m[i])!r} > bound {float(bound[i])!r}; rel L2 {l2:.3e}")
    return _ratio(excess, m), l2


def check_exact(y, ref, what):
    yb = y.contiguous().view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.uint8: torch.uint8}[y.dtype])
    rb = ref.contiguous().view(yb.dtype)
    bad = yb != rb
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ in bits; first at {i}: y={float(y[i])!r} "
                             f"r={float(ref[i])!r}")


class Worst(dict):
    def add(self, name, res):
        old = self.get(name, (0.0, 0.0))
        self[name] = (max(old[0], res[0]), max(old[1], res[1]))


# ---------------------------------------------------------------------------------------------- one update launch
def alloc_update(r, tab, k, moments, device, seed=0):
    """The buffers of update launch `r` at step k (moments: random state; else the zero state), filled on the rows."""
    kind = r["kind"]
    eight, ema = "8bit" in kind, "ema" in kind
    P = patterns(seed, device)
    qm_map = qmaps()
    zero_m = int((qm_map[:256] == 0).nonzero()[0, 0])
    b = {"p": Buf(r["total"], torch.float32, device), "g": Buf(r["total"], torch.float32, device),
         "shadow": Buf(max(r["n_shadow"], 8), torch.bfloat16, device)}
    if r["g16"]:
        b["g16"] = Buf(r["total"], torch.bfloat16, device)
    if eight:
        b["m32"], b["v32"] = Buf(r["n_state"], torch.float32, device), Buf(r["n_state"], torch.float32, device)
        b["qm"], b["qv"] = Buf(r["n_state8"], torch.uint8, device), Buf(r["n_state8"], torch.uint8, device)
        b["am"], b["av"] = Buf(r["n_state8"] // QBLOCK, torch.float32, device), Buf(r["n_state8"] // QBLOCK, torch.float32, device)
    else:
        b["m"], b["v"] = Buf(r["n_state"], torch.float32, device), Buf(r["n_state"], torch.float32, device)
    if ema:
        b["ema"] = Buf(r["n_ema"], torch.float32, device)
    for lo, hi in batches(tab):
        rows = tab[lo:hi]
        ia = expand(rows[:, 0], rows[:, 1], device)
        b["p"].t[ia] = pat(P["p"], ia)
        b["g"].t[ia] = pat(P["g"], ia)
        if r["g16"]:
            b["g16"].t[ia] = pat(P["g16"], ia)
        sh = rows[:, 0] < r["n_shadow"]
        if bool(sh.any()):
            ish = expand(rows[sh, 0], rows[sh, 1], device)
            b["shadow"].t[ish] = pat(P["p"], ish).bfloat16()
        if ema:
            ie = expand(rows[:, -1], rows[:, 1], device)
            b["ema"].t[ie] = pat(P["ema"], ie)
        if eight:
            for bits, names in ((32, ("m32", "v32")), (8, ("qm", "qv"))):
                sel = rows[:, 3] == bits
                if not bool(sel.any()):
                    continue
                ist = expand(rows[sel, 2], rows[sel, 1], device)
                if bits == 32:
                    b["m32"].t[ist] = pat(P["m"], ist) if moments else 0.0
                    b["v32"].t[ist] = pat(P["v"], ist) if moments else 0.0
                else:
                    b["qm"].t[ist] = pat(P["qm"], ist) if moments else zero_m
                    b["qv"].t[ist] = pat(P["qv"], ist) if moments else 0
                    blk = torch.unique(ist // QBLOCK)
                    b["am"].t[blk] = pat(P["am"], blk) if moments else 0.0
                    b["av"].t[blk] = pat(P["av"], blk) if moments else 0.0
        else:
            b["m"].t[ia] = pat(P["m"], ia) if moments else 0.0
            b["v"].t[ia] = pat(P["v"], ia) if moments else 0.0
    return b, P


def check_update(r, tab, k, moments, b, P, what, device):
    """Checks every output of update launch `r` run at step k; returns {output: (ratio, l2)}."""
    kind = r["kind"]
    eight, ema = "8bit" in kind, "ema" in kind
    hp = hp_row(r["hp"], k, CLIP if moments else 1.0)
    qmap = qmaps().to(device)
    zero_m = int((qmap[:256] == 0).nonzero()[0, 0])
    decay = r.get("ema_decay", 0.0)
    res = Worst()
    for lo, hi in batches(tab):
        rows = tab[lo:hi]
        ia = expand(rows[:, 0], rows[:, 1], device)
        for n in ("p", "g"):
            b[n].covered[ia] = True
        if "g16" in b:
            b["g16"].covered[ia] = True
        g_in = pat(P["g16"], ia).float() if r["g16"] else pat(P["g"], ia)
        p_in = pat(P["p"], ia)
        p_out = b["p"].t[ia]
        nbits = rows[:, 3] if eight else torch.full((rows.shape[0],), 32, dtype=torch.int64)
        per_el_bits = torch.repeat_interleave(nbits.to(device), rows[:, 1].to(device))
        if eight:
            ist = expand(rows[:, 2], rows[:, 1], device)
        else:
            ist = ia
        m_in = torch.zeros_like(p_in, dtype=torch.float64)
        v_in = torch.zeros_like(p_in, dtype=torch.float64)
        is32 = per_el_bits == 32
        if moments:
            m_in[is32] = pat(P["m"], ist[is32]).double()
            v_in[is32] = pat(P["v"], ist[is32]).double()
            if eight:
                is8 = ~is32
                blk = ist[is8] // QBLOCK
                m_in[is8] = qmap[:256][pat(P["qm"], ist[is8]).long()].double() * pat(P["am"], blk).double()
                v_in[is8] = qmap[256:][pat(P["qv"], ist[is8]).long()].double() * pat(P["av"], blk).double()
        ref = adamw_ref(p_in, g_in, m_in, v_in, hp)
        res.add("p", check(p_out, *ref["p"], "p", f"{what} p"))
        # moments: fp32 rows
        if bool(is32.any()):
            mb, vb = ("m32", "v32") if eight else ("m", "v")
            i32 = ist[is32]
            b[mb].covered[i32] = True
            b[vb].covered[i32] = True
            res.add("m", check(b[mb].t[i32], ref["m"][0][is32], ref["m"][1][is32], "m", f"{what} m"))
            res.add("v", check(b[vb].t[i32], ref["v"][0][is32], ref["v"][1][is32], "v", f"{what} v"))
        if eight and bool((~is32).any()):
            is8 = ~is32
            i8 = ist[is8]
            blk = i8 // QBLOCK
            ub, inv = torch.unique(blk, return_inverse=True)
            for mom, qb, ab, qmp, zc in (("m", "qm", "am", qmap[:256], zero_m), ("v", "qv", "av", qmap[256:], 0)):
                b[qb].covered[i8] = True
                b[ab].covered[ub] = True
                x, mx = ref[mom][0][is8], ref[mom][1][is8]
                amax = torch.zeros(ub.numel(), dtype=torch.float64, device=device).scatter_reduce(0, inv, x.abs(), "amax")
                mmax = torch.zeros(ub.numel(), dtype=torch.float64, device=device).scatter_reduce(0, inv, mx, "amax")
                res.add("absmax", check(b[ab].t[ub], amax, mmax, "absmax", f"{what} absmax_{mom}"))
                a_el, mm_el = amax[inv], mmax[inv]
                xn = x / a_el.clamp_min(1e-300)
                band = EPS["code"] * (mx + xn.abs() * mm_el) / a_el.clamp_min(1e-300)
                c, c_lo, c_hi = code_ref(xn, band, qmp, zc, a_el == 0)
                got = b[qb].t[i8].long()
                bad = (got < c_lo) | (got > c_hi)
                if bool(bad.any()):
                    i = int(bad.nonzero()[0])
                    raise AssertionError(f"{what} code_{mom}: {int(bad.sum())} of {bad.numel()} codes off; first at {i}: got {int(got[i])} "
                                         f"want {int(c[i])} (accepted {int(c_lo[i])}..{int(c_hi[i])}), x={float(xn[i])!r}")
                res.add("code", (0.0, float((got != c).double().mean())))
        # shadow: RNE of the new p below n_shadow
        sh = ia < r["n_shadow"]
        if bool(sh.any()):
            b["shadow"].covered[ia[sh]] = True
            check_exact(b["shadow"].t[ia[sh]], p_out[sh].bfloat16(), f"{what} shadow")
        check_exact(b["g"].t[ia], torch.zeros_like(p_out), f"{what} zeroed g")
        if "g16" in b:
            check_exact(b["g16"].t[ia], pat(P["g16"], ia), f"{what} g16 (read only)")
        if ema:
            ie = expand(rows[:, -1], rows[:, 1], device)
            b["ema"].covered[ie] = True
            e_in = pat(P["ema"], ie)
            check_exact(b["ema"].t[ie], ema_fp32(e_in, p_out, k, decay), f"{what} ema vs EMAModel.step on the new p")
            res.add("ema", check(b["ema"].t[ie], *ema_ref(e_in, ref["p"][0], ref["p"][1], k, decay), "ema", f"{what} ema"))
    for n, buf in b.items():
        buf.assert_untouched(f"{what} {n}")
    return dict(res)


# ---------------------------------------------------------------------------------------------- sqnorm, ema_swap, prepare
SQ_PRESET = 12.375


def alloc_sqnorm(r, tab, device, seed=0):
    P = patterns(seed, device)
    name = "g16" if r["g16"] else "g"
    buf = Buf(r["total"], torch.bfloat16 if r["g16"] else torch.float32, device)
    for lo, hi in batches(tab):
        ia = expand(tab[lo:hi, 0], tab[lo:hi, 1], device)
        buf.t[ia] = pat(P[name], ia)
    out = torch.tensor([SQ_PRESET, -1.0], dtype=torch.float64, device=device)
    return buf, out, P


def check_sqnorm(r, tab, buf, out, P, what, device):
    name = "g16" if r["g16"] else "g"
    s = torch.zeros((), dtype=torch.float64, device=device)
    for lo, hi in batches(tab):
        ia = expand(tab[lo:hi, 0], tab[lo:hi, 1], device)
        buf.covered[ia] = True
        s += (pat(P[name], ia).double() ** 2).sum()
    buf.assert_untouched(f"{what} g")
    ref = s + SQ_PRESET
    assert float(out[1]) == -1.0, f"{what}: sq[1] written"
    return {"sq": check(out[:1], ref.view(1), ref.view(1), "sq", f"{what} sum of squares")}


def alloc_swap(r, tab, device, seed=0):
    P = patterns(seed, device)
    b = {"p": Buf(r["total"], torch.float32, device), "ema": Buf(r["n_ema"], torch.float32, device),
         "shadow": Buf(max(r["n_shadow"], 8), torch.bfloat16, device)}
    for lo, hi in batches(tab):
        rows = tab[lo:hi]
        ia, ie = expand(rows[:, 0], rows[:, 1], device), expand(rows[:, 2], rows[:, 1], device)
        b["p"].t[ia], b["ema"].t[ie] = pat(P["p"], ia), pat(P["ema"], ie)
        sh = ia < r["n_shadow"]
        b["shadow"].t[ia[sh]] = pat(P["p"], ia[sh]).bfloat16()
    return b, P


def check_swap(r, tab, b, P, what, device, swapped):
    """After one swap (swapped) p holds the EMA, the EMA p and the shadow RNE of the EMA; after two, everything as it was."""
    for lo, hi in batches(tab):
        rows = tab[lo:hi]
        ia, ie = expand(rows[:, 0], rows[:, 1], device), expand(rows[:, 2], rows[:, 1], device)
        p0, e0 = pat(P["p"], ia), pat(P["ema"], ie)
        b["p"].covered[ia] = True
        b["ema"].covered[ie] = True
        check_exact(b["p"].t[ia], e0 if swapped else p0, f"{what} p")
        check_exact(b["ema"].t[ie], p0 if swapped else e0, f"{what} ema")
        sh = ia < r["n_shadow"]
        b["shadow"].covered[ia[sh]] = True
        check_exact(b["shadow"].t[ia[sh]], (e0 if swapped else p0)[sh].bfloat16(), f"{what} shadow")
    for n, buf in b.items():
        buf.assert_untouched(f"{what} {n}")


def ulp32(x):
    x = abs(float(x))
    if x == 0:
        return 2.0 ** -149
    return 2.0 ** (math.frexp(x)[1] - 24)


def check_prepare(hp_in, hp_out, step_before, step_after, sq_before, sq_after, max_norm, what):
    """adamw_prepare's device scalars against their definitions (host tensors)."""
    k = int(step_before) + 1
    assert int(step_after) == k, f"{what}: step {int(step_after)} != {k}"
    norm = math.sqrt(float(sq_before))
    assert float(sq_after[0]) == 0.0, f"{what}: sq[0] not reset"
    assert float(sq_after[1]) == norm, f"{what}: sq[1] {float(sq_after[1])!r} != sqrt(sq[0]) {norm!r}"
    clip = 1.0 if max_norm <= 0 else min(1.0, float(torch.tensor(max_norm, dtype=torch.float32)) / (norm + 1e-6))
    for s in range(hp_in.shape[0]):
        b1, b2 = float(hp_in[s, 1]), float(hp_in[s, 2])
        assert torch.equal(hp_out[s, :5], hp_in[s]), f"{what}: set {s} hyper-parameters not copied"
        for j, want in ((5, 1 - b1 ** k), (6, math.sqrt(1 - b2 ** k)), (7, clip)):
            w32 = float(torch.tensor(want, dtype=torch.float64).float())
            got = float(hp_out[s, j])
            assert abs(got - w32) <= ulp32(w32), f"{what}: set {s} hp[{j}] = {got!r}, want {w32!r} (exact {want!r}) within 1 ulp"


# ---------------------------------------------------------------------------------------------- stable-LoRA delta
def delta_inputs(r, device, seed=0):
    g = torch.Generator().manual_seed(seed + r["Cout"] * 7919 + r["Cin"] * 31 + r["k"] + 101 * r["r"] + 5 * r["conv3d"])
    co, ci, k, rk = r["Cout"], r["Cin"], r["k"], r["r"] * r["k"]
    kh, kw = (3, 1) if r["conv3d"] else (k, k)
    out = {"base": torch.randn(co, kh, kw, ci, generator=g) * 0.05, "A": torch.randn(rk, ci * k, generator=g) / (ci * k) ** 0.5,
           "B": torch.randn(co * k, rk, generator=g) * 0.05, "dw": torch.randn(co, kh, kw, ci, generator=g),
           "dA": 1 + torch.randn(rk, ci * k, generator=g), "dB": 1 + torch.randn(co * k, rk, generator=g)}
    return {n: t.to(device) for n, t in out.items()}


def _logical(phys, conv3d):
    """[Cout, KH, KW, Cin] -> (Cout, Cin, KH, KW) (Conv3d: (Cout, Cin, 3, 1))."""
    return phys.permute(0, 3, 1, 2)


def delta_ref(r, inp):
    """{output: (r, m, mode)} of lora_delta_merge or lora_delta_grad in float64."""
    co, ci, k, conv3d = r["Cout"], r["Cin"], r["k"], r["conv3d"]
    s = float(torch.tensor(r["scaling"], dtype=torch.float32))
    A, B = inp["A"].double(), inp["B"].double()
    if r["kind"] == "lora_delta_merge":
        ba, mba = B @ A, B.abs() @ A.abs()
        if conv3d:
            d = ba.view(co, ci, 3, 3, 1).mean(-2)
            md = mba.view(co, ci, 3, 3, 1).mean(-2)
        else:
            d, md = ba.view(co, ci, k, k), mba.view(co, ci, k, k)
        base = inp["base"].double()
        dphys, mdphys = d.permute(0, 2, 3, 1), md.permute(0, 2, 3, 1)
        return {"merged": (base + s * dphys, base.abs() + abs(s) * mdphys, "bf16")}
    dw = _logical(inp["dw"].double(), conv3d)
    if conv3d:
        dba = (s * dw / 3).unsqueeze(-2).expand(co, ci, 3, 3, 1).reshape(co * 3, ci * 3)
    else:
        dba = (s * dw).reshape(co * k, ci * k)
    pa, pb = inp["dA"].double(), inp["dB"].double()
    return {"dA": (pa + B.t() @ dba, pa.abs() + B.abs().t() @ dba.abs(), "f32"),
            "dB": (pb + dba @ A.t(), pb.abs() + dba.abs() @ A.abs().t(), "f32")}


def check_delta(r, inp, out, what):
    ref = delta_ref(r, inp)
    res = {}
    for name, (rv, m, mode) in ref.items():
        y = out[name].reshape(-1)
        res[name] = check(y, rv.reshape(-1).to(y.device), m.reshape(-1).to(y.device), "merge" if name == "merged" else name,
                          f"{what} {name}", rounded=mode == "bf16")
    return res


# ---------------------------------------------------------------------------------------------- compression
def cast_inputs(n, device, seed=0):
    g = torch.Generator().manual_seed(seed + 17)
    x = torch.randn(min(n, PATTERN), generator=g, dtype=torch.float64) * 10.0 ** (-8 + 9 * torch.rand(min(n, PATTERN), generator=g, dtype=torch.float64))
    return x.float().to(device)


def check_cast(r, x_pat, y, what):
    """y (bf16, n elements) against x / world; x_pat repeats with period PATTERN."""
    world = r["world"]
    alpha = torch.tensor(1.0 / world, dtype=torch.float32)
    exact = world & (world - 1) == 0
    worst = (0.0, 0.0)
    for a in range(0, y.numel(), PATTERN):
        part = y[a:a + PATTERN]
        x = x_pat[:part.numel()]
        if exact:
            check_exact(part, (x * alpha.to(x.device)).bfloat16(), f"{what} y")
        else:
            rv = x.double() / world
            worst = max(worst, check(part, rv, rv.abs(), "cast", f"{what} y", rounded=True))
    return {"y": worst}
