"""Element-wise checks of the glue kernels of csrc/elementwise.cu (layout, loss, noise, timestep embedding, bias gradients, fan-in,
resampling, casts, dropout, token embedding, GELU, VAE sampling, frame resize) against a float64 reference written from the
operation's definition (diffusers / torch semantics), not from oracle/ops_ref.py.  Shared by tests/test_glue_step_gpu.py (the
kernels, at every launch of tests/golden/glue_launches.json) and tests/test_glue_step_cpu.py (the same checks against fp32
restatements and deliberately broken outputs, without a GPU).

Reference r: the float64 result of the operation on the same bf16 / fp32 / uint8 inputs.  Magnitude m: the same expression on
absolute values of every term, so that it bounds what fp32 rounding of each intermediate can contribute:
    add_noise / velocity   |sqrt(abar) x0| + |sqrt(1 - abar) eps|
    mse loss               mean((|pred| + |target|)^2), target's m as above for the velocity; dpred 2 (|pred| + |target|) |g| / N
    timestep embedding     1 + |t f|: the argument t f is rounded in fp32, as the upstream fp32 formula rounds it
    colsum / colsum_f32    |preset| + sum |x|;   embed_tokens_bwd  |preset| + sum |dy| over the rows summed
    add (2 or 3 inputs)    |a| + |b| (+ |c|);   scale  |alpha a|;   embed_tokens  |tok| + |pos|;   upsample backward  sum |dy|
    dropout                |base| + |k x| over kept elements, k = scale / (1 - p)
    GELU (erf)             |gelu(x)| + |x| (the fp32 cancellation in 1 + erff(x / sqrt 2) for very negative x is conditioning)
    quick_gelu             |y| + |x| s (1 - s) (1 + 1.702 |x|) (the fp32 argument and exponential of the sigmoid)
    their derivatives      |dy| times the m of the derivative, the same way
    vae_sample             scale (|mean| + exp(lv / 2) |eps| (1 + |lv| / 2))
    resize                 1 + (|dv/dy| (1 + fy) + |dv/dx| (1 + fx)) / 127.5: the fp32 source coordinates (fy, fx) of the kernel
Every element must satisfy
    bf16 output:   |y - r| <= 2^-8 |r| + eps m        (one round-to-nearest of an fp32 result)
    fp32 output:   |y - r| <= eps m
and the relative L2 error of a bf16 output must be at most 2^-8.  Exact outputs must match bit for bit: the layout copies, the
zero-padded channels of every [.., 8] latent tensor, upsample_nearest_fwd, concat / split, nhwc8_to_latents, both casts (round to
nearest even, ties included), the elements dropout drops (the keep-mask restated with integer arithmetic below) and the rows of
dtok no id touches (they keep their preset).

Inputs (seed = crc32 of the launch id, drawn on the CPU): colsum rows with a per-column common mode of up to 30 standard
deviations; fan-in gradients that cancel (b ~ -a, c ~ -(a + b)); GELU inputs 3 N(0, 1) with at least 1% below -4; timesteps
999, 0, 1, 500 for the first four samples (distinct in every B > 1 launch); abar from oracle.leaves.ddpm_alphas_cumprod(); token
ids shaped like a padded prompt (BOS, a few ids, EOS repeated to L); accumulated outputs preset to nonzero values.  Element-wise
launches of more than PATTERN elements repeat one PATTERN-long draw (an odd length, so every lane of a vector meets every value);
their outputs are checked period by period.

eps, per output: the next power of two at or above 4x the largest ratio (check()) measured over the census and the sweeps of
tests/test_glue_step_gpu.py on one NVIDIA H100 80GB HBM3 at a 700 W power limit; 2^-22 (four fp32 unit roundoffs) where nothing
beyond one rounding was measured (ratio 0).  No kernel exceeded its bound; the float64 check found no defect in this family."""
import json
import math
import os
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LAUNCHES = os.path.join(HERE, "golden", "glue_launches.json")

U_BF16 = 2.0 ** -8
EPS = {                                   # measured max ratio (launch)
    "noise.y": 2.0 ** -22,          # 0         latents_to_nhwc8 1x4x16x32x32 add_noise
    "mse.loss": 2.0 ** -20,         # 1.78e-07  mse_loss_fwd 2x4x16x32x32
    "mse.dpred": 2.0 ** -22,        # 0         mse_loss_bwd 1x4x16x32x32
    "vel.loss": 2.0 ** -22,         # 3.72e-08  velocity_mse_loss_fwd 1x4x16x32x32
    "vel.dpred": 2.0 ** -23,        # 2.00e-08  velocity_mse_loss_bwd 4x4x1x64x64
    "temb.y": 2.0 ** -19,           # 2.53e-07  timestep_embedding sweep, t in [0, 999], dim 320
    "colsum.out": 2.0 ** -18,       # 7.37e-07  colsum S 1, P 17280, C 640
    "colsum_f32.out": 2.0 ** -20,   # 1.42e-07  colsum_f32 S 4, C 1280
    "upsample.dx": 2.0 ** -22,      # 0         upsample_nearest_bwd 16x16x16 -> 32x32, C 640
    "add.y": 2.0 ** -22,            # 0         add_bf16 n 5242880, 2 inputs
    "add_f32.y": 2.0 ** -22,        # 5.91e-08  add_f32 n 78848
    "scale.y": 2.0 ** -22,          # 0         scale_bf16 n 5242880, alpha 0.5 (synthetic)
    "dropout.y": 2.0 ** -22,        # 4.41e-08  dropout_scale_add n 315392, p 0.1, with base
    "embed.y": 2.0 ** -22,          # 0         embed_tokens 1x77, C 1024
    "embed.dtok": 2.0 ** -22,       # 5.96e-08  embed_tokens_bwd 1x77, C 1024, dtok and dpos
    "embed.dpos": 2.0 ** -22,       # 5.96e-08  embed_tokens_bwd 1x77, C 1024, dtok and dpos
    "gelu.y": 2.0 ** -23,           # 1.73e-08  gelu_bf16 n 315392, erf
    "gelu.dx": 2.0 ** -23,          # 2.33e-08  gelu_bwd n 315392, erf
    "vae.z": 2.0 ** -20,            # 1.45e-07  vae_sample 2x4 frames, 32x32
    "resize.y": 2.0 ** -21,         # 7.64e-08  frames_u8_to_nhwc8 4 frames 720x1280 -> 320x576
}
GELU_TAIL = (-4.0, 0.01)     # every GELU launch: at least 1% of its x below -4
PATTERN = (1 << 22) + 5      # element-wise launches above this many elements repeat one draw of this length
TIMESTEPS = (999, 0, 1, 500)
BOS, EOS = 49406, 49407
EPOCH_K = 0xD1342543DE82EF95
MASK64 = (1 << 64) - 1


def launches():
    with open(LAUNCHES) as f:
        return json.load(f)


def launch_id(r):
    fields = "-".join(f"{k}{json.dumps(v, separators=(',', ':')) if isinstance(v, list) else v}" for k, v in r.items() if k != "kind")
    return f'{r["kind"]}-{fields}'


def _gen(r):
    return torch.Generator().manual_seed(zlib.crc32(launch_id(r).encode()))


def n_drawn(r):
    """Elements drawn for an element-wise launch of n elements (the pattern repeats beyond PATTERN)."""
    return min(r["n"], PATTERN)


# ---------------------------------------------------------------------------------------------- inputs
def timesteps(B, g):
    if B <= len(TIMESTEPS):
        return torch.tensor(TIMESTEPS[:B], dtype=torch.int64)
    rest = torch.randperm(1000, generator=g)
    rest = rest[~torch.isin(rest, torch.tensor(TIMESTEPS))][:B - len(TIMESTEPS)]
    return torch.cat([torch.tensor(TIMESTEPS), rest]).to(torch.int64)


def prompt_ids(B, L, g):
    """BOS, 3..10 random ids, then EOS repeated to L, per prompt."""
    ids = torch.full((B, L), EOS, dtype=torch.int64)
    for b in range(B):
        k = int(torch.randint(3, 11, (1,), generator=g))
        ids[b, 0] = BOS
        ids[b, 1:1 + k] = torch.randint(0, BOS, (k,), generator=g)
    return ids


def _common_mode(g, lead, C):
    mu = (torch.rand(C, generator=g) * 2 - 1) * 30
    return torch.randn(*lead, C, generator=g) * (0.5 + torch.rand(C, generator=g)) + mu


def _tie_values(n, g):
    """fp32 values whose low 16 bits are random, 0x8000 (a tie) or 0 for a quarter of them each (and random signs / exponents)."""
    bits = torch.randint(0, 1 << 16, (n,), generator=g, dtype=torch.int64)
    hi = torch.randint(0x3000, 0x4F00, (n,), generator=g, dtype=torch.int64) | (torch.randint(0, 2, (n,), generator=g) << 15)
    sel = torch.randint(0, 4, (n,), generator=g)
    lo = torch.where(sel == 0, torch.full_like(bits, 0x8000), torch.where(sel == 1, torch.zeros_like(bits), bits))
    return ((hi << 16) | lo).to(torch.int32).view(torch.float32)


def make_inputs(r):
    """The launch's inputs, on the CPU."""
    g = _gen(r)
    k = r["kind"]
    out = {}
    if k in ("latents_to_nhwc8", "mse_loss_fwd", "mse_loss_bwd", "velocity_mse_loss_fwd", "velocity_mse_loss_bwd"):
        from oracle import leaves as L
        B, C, F, H, W = r["B"], r["C"], r["F"], r["H"], r["W"]
        x0 = torch.randn(B, C, F, H, W, generator=g)
        out["x0"] = x0
        if k == "latents_to_nhwc8" and not r["noise"]:
            return out
        out["noise"] = torch.randn(B, C, F, H, W, generator=g)
        out["abar"] = L.ddpm_alphas_cumprod().float().contiguous()
        out["t"] = timesteps(B, g)
        if k != "latents_to_nhwc8":
            pred = torch.randn(B * F, H, W, 8, generator=g)
            pred[..., C:] = 1e4   # padded channels: never read
            out["pred"] = pred.bfloat16()
            out["gout"] = torch.tensor(0.37)
    elif k == "nhwc8_to_latents":
        out["x"] = torch.randn(r["B"] * r["F"], r["H"], r["W"], 8, generator=g).bfloat16()
    elif k == "timestep_embedding":
        out["t"] = timesteps(r["B"], g)
    elif k == "colsum":
        out["x"] = _common_mode(g, (r["S"], r["P"]), r["C"]).bfloat16()
        out["preset"] = 1 + torch.randn(r["S"], r["C"], generator=g)
    elif k == "colsum_f32":
        out["x"] = _common_mode(g, (r["S"],), r["C"])
        out["preset"] = 1 + torch.randn(r["C"], generator=g)
    elif k == "upsample_nearest_fwd":
        out["x"] = torch.randn(r["N"], r["H"], r["W"], r["C"], generator=g).bfloat16()
    elif k == "upsample_nearest_bwd":
        out["dy"] = torch.randn(r["N"], r["Ho"], r["Wo"], r["C"], generator=g).bfloat16()
    elif k == "concat_channels":
        out["a"] = torch.randn(r["M"], r["Ca"], generator=g).bfloat16()
        out["b"] = torch.randn(r["M"], r["Cb"], generator=g).bfloat16()
    elif k == "split_channels":
        out["g"] = torch.randn(r["M"], r["Ct"], generator=g).bfloat16()
    elif k in ("add_bf16", "add_f32"):
        n = n_drawn(r)
        a = 4 * torch.randn(n, generator=g)
        b = -a * (0.9 + 0.2 * torch.rand(n, generator=g)) + 0.05 * torch.randn(n, generator=g)
        dt = torch.bfloat16 if k == "add_bf16" else torch.float32
        a, b = a.to(dt), b.to(dt)
        out["a"], out["b"] = a, b
        if k == "add_bf16" and r["inputs"] == 3:
            s = a.float() + b.float()
            out["c"] = (-s * (0.5 + torch.rand(n, generator=g)) + 0.01 * torch.randn(n, generator=g)).bfloat16()
    elif k == "scale_bf16":
        out["a"] = torch.randn(n_drawn(r), generator=g).bfloat16()
    elif k == "cast_f32_bf16":
        out["src"] = _tie_values(n_drawn(r), g)
    elif k == "cast_bf16_f32":
        out["src"] = _tie_values(n_drawn(r), g).bfloat16()
    elif k == "dropout_scale_add":
        n = r["n"]
        x = torch.randn(n, generator=g)
        out["x"] = (torch.sign(x) * (0.25 + x.abs())).bfloat16()
        if r["base"]:
            out["base"] = torch.randn(n, generator=g).bfloat16()
        out["seed"] = int(torch.randint(0, 1 << 62, (1,), generator=g)) * 3 + 1
        out["epoch"] = torch.tensor(int(torch.randint(1, 1 << 40, (1,), generator=g)), dtype=torch.int64)
    elif k in ("embed_tokens", "embed_tokens_bwd"):
        B, L, C, V = r["B"], r["L"], r["C"], r["vocab"]
        out["ids"] = prompt_ids(B, L, g)
        if k == "embed_tokens":
            out["tok"] = torch.randn(V, C, generator=g)
            out["pos"] = torch.randn(r["pos_rows"], C, generator=g)
        else:
            out["dy"] = torch.randn(B * L, C, generator=g).bfloat16()
            if r["dtok"]:
                out["dtok"] = 1 + torch.randn(V, C, generator=g)
            if r["dpos"]:
                out["dpos"] = 1 + torch.randn(r["pos_rows"], C, generator=g)
    elif k in ("gelu_bf16", "gelu_bwd"):
        out["x"] = (3 * torch.randn(r["n"], generator=g)).bfloat16()
        if k == "gelu_bwd":
            out["dy"] = (torch.randn(r["n"], generator=g) + 0.25).bfloat16()
    elif k == "vae_sample":
        B, F, h, w = r["B"], r["F"], r["h"], r["w"]
        mom = torch.randn(B * F, h, w, 8, generator=g)
        mom[..., 4:] = torch.rand(B * F, h, w, 4, generator=g) * 70 - 40   # logvar over [-40, 30]: both clamps
        out["moments"] = mom.bfloat16()
        out["eps"] = torch.randn(B, 4, F, h, w, generator=g)
    elif k == "frames_u8_to_nhwc8":
        out["frames"] = torch.randint(0, 256, (r["F"], r["H0"], r["W0"], 3), generator=g, dtype=torch.uint8)
    elif k == "frames_u8_to_nhwc8_ragged":
        clips = [torch.randint(0, 256, (F, H0, W0, 3), generator=g, dtype=torch.uint8) for F, H0, W0 in r["clips"]]
        off, rows = 0, []
        for c in clips:
            rows.append([off, *c.shape[:3]])
            off += c.numel()
        out["clips"] = clips
        out["packed"] = torch.cat([c.flatten() for c in clips])
        out["table"] = torch.tensor(rows, dtype=torch.int64)
    else:
        raise KeyError(k)
    return out


# ---------------------------------------------------------------------------------------------- float64 references
def _nhwc8(x5):
    """(B, C, F, H, W) -> [B*F, H, W, C] (no padding)."""
    B, C, F, H, W = x5.shape
    return x5.permute(0, 2, 3, 4, 1).reshape(B * F, H, W, C)


def _scales(inp):
    a = inp["abar"].double()[inp["t"]]
    return a.sqrt().view(-1, 1, 1, 1, 1), (1 - a).sqrt().view(-1, 1, 1, 1, 1)


def velocity(inp):
    """(v, m) of v = sqrt(abar_t) eps - sqrt(1 - abar_t) x0 (DDPMScheduler.get_velocity), (B, C, F, H, W)."""
    sa, sb = _scales(inp)
    n, x0 = inp["noise"].double(), inp["x0"].double()
    return sa * n - sb * x0, (sa * n).abs() + (sb * x0).abs()


def mix32(seed, idx):
    """splitmix64 finaliser of seed + idx * golden (mod 2^64), upper 32 bits, on numpy uint64 (wrapping arithmetic)."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + idx.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return (z ^ (z >> np.uint64(31))) >> np.uint64(32)


def keep_mask(n, p, seed, epoch):
    """Dropout keep-mask of element i: mix32(seed ^ epoch K, i) >= uint32(p 2^32), p as the fp32 the kernel receives."""
    s = (int(seed) ^ ((int(epoch) * EPOCH_K) & MASK64)) & MASK64
    thresh = int(float(np.float32(p)) * 4294967296.0)
    return torch.from_numpy(mix32(s, np.arange(n, dtype=np.uint64)) >= np.uint64(thresh))


def gelu_terms(x, quick):
    """(y, m_y, g = y', m_g) in float64."""
    if quick:
        s = torch.sigmoid(1.702 * x)
        y = x * s
        ds = s * (1 - s)
        g = s + 1.702 * x * ds
        d2 = 1.702 * ds * (2 + 1.702 * x * (1 - 2 * s))
        return y, y.abs() + x.abs() * ds * (1 + 1.702 * x.abs()), g, g.abs() + (d2.abs() + ds) * (1 + 1.702 * x.abs())
    phi = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
    y = x * cdf
    g = cdf + x * phi
    return y, y.abs() + x.abs(), g, g.abs() + 1 + x.abs() * phi * (1 + x * x)


def bilinear(frames, h, w, align_corners=False):
    """(v, m) of the resize of uint8 [F, H0, W0, 3] to [F, h, w, 3], v = bilinear / 127.5 - 1 (F.interpolate semantics,
    align_corners=False: source = (dst + 0.5) in / out - 0.5 clamped at 0)."""
    F_, H0, W0, _ = frames.shape

    def axis(n_out, n_in):
        d = torch.arange(n_out, dtype=torch.float64)
        if align_corners:
            f = d * ((n_in - 1) / (n_out - 1)) if n_out > 1 else d * 0
        else:
            f = ((d + 0.5) * (n_in / n_out) - 0.5).clamp_min(0)
        i0 = f.floor().long().clamp(max=n_in - 1)
        i1 = (i0 + 1).clamp(max=n_in - 1)
        return f, i0, i1, f - i0.double()

    fy, y0, y1, wy = axis(h, H0)
    fx, x0, x1, wx = axis(w, W0)
    p = frames.double()
    p00, p01 = p[:, y0][:, :, x0], p[:, y0][:, :, x1]
    p10, p11 = p[:, y1][:, :, x0], p[:, y1][:, :, x1]
    wx_, wy_ = wx.view(1, 1, -1, 1), wy.view(1, -1, 1, 1)
    top, bot = p00 + (p01 - p00) * wx_, p10 + (p11 - p10) * wx_
    v = (top + (bot - top) * wy_) / 127.5 - 1
    gx = (p01 - p00).abs() + (p11 - p10).abs()
    gy = (bot - top).abs()
    m = 1 + (gy * (1 + fy.view(1, -1, 1, 1)) + gx * (1 + fx.view(1, 1, -1, 1))) / 127.5
    return v, m


def _pad_zero(n5):
    return torch.zeros(n5, dtype=torch.float64)


def reference(r, inp):
    """{output: (r, m, mode)}: mode "bf16" / "f32" (bound) or "exact" (bit for bit; m unused).  Every [.., 8] output is split
    into its channels < C and its padded channels ("pad", exact zeros)."""
    k = r["kind"]
    if k == "latents_to_nhwc8":
        C = r["C"]
        if not r["noise"]:
            return {"y": (_nhwc8(inp["x0"]).bfloat16(), None, "exact"), "pad": (_pad_zero((r["B"] * r["F"], r["H"], r["W"], 8 - C)), None, "exact")}
        sa, sb = _scales(inp)
        x0, n = inp["x0"].double(), inp["noise"].double()
        return {"y": (_nhwc8(sa * x0 + sb * n), _nhwc8((sa * x0).abs() + (sb * n).abs()), "bf16"),
                "pad": (_pad_zero((r["B"] * r["F"], r["H"], r["W"], 8 - C)), None, "exact")}
    if k == "nhwc8_to_latents":
        B, C, F, H, W = r["B"], r["C"], r["F"], r["H"], r["W"]
        return {"out": (inp["x"].float().view(B, F, H, W, 8)[..., :C].permute(0, 4, 1, 2, 3).contiguous(), None, "exact")}
    if k in ("mse_loss_fwd", "mse_loss_bwd", "velocity_mse_loss_fwd", "velocity_mse_loss_bwd"):
        C = r["C"]
        p = inp["pred"].double()[..., :C]
        if k.startswith("velocity"):
            tgt, mt = velocity(inp)
            tgt, mt = _nhwc8(tgt), _nhwc8(mt)
        else:
            tgt = _nhwc8(inp["noise"].double())
            mt = tgt.abs()
        e, me = p - tgt, p.abs() + mt
        N = e.numel()
        pre = "vel" if k.startswith("velocity") else "mse"
        if k.endswith("fwd"):
            return {"loss": ((e * e).mean(), (me * me).mean(), "f32")}
        g = float(inp["gout"])
        return {"dpred": (2 * e * g / N, 2 * me * abs(g) / N, "bf16"), "pad": (_pad_zero(e.shape[:-1] + (8 - C,)), None, "exact"),
                "_pre": pre}
    if k == "timestep_embedding":
        half = r["dim"] // 2
        f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64) / half)
        a = inp["t"].double()[:, None] * f[None]
        m = 1 + a.abs()
        return {"y": (torch.cat([torch.cos(a), torch.sin(a)], -1), torch.cat([m, m], -1), "bf16")}
    if k == "colsum":
        x = inp["x"].double()
        pre = inp["preset"].double()
        return {"out": (pre + x.sum(1), pre.abs() + x.abs().sum(1), "f32")}
    if k == "colsum_f32":
        x = inp["x"].double()
        pre = inp["preset"].double()
        return {"out": (pre + x.sum(0), pre.abs() + x.abs().sum(0), "f32")}
    if k == "upsample_nearest_fwd":
        hi = torch.arange(r["Ho"]) * r["H"] // r["Ho"]
        wi = torch.arange(r["Wo"]) * r["W"] // r["Wo"]
        return {"y": (inp["x"][:, hi][:, :, wi], None, "exact")}
    if k == "upsample_nearest_bwd":
        N, H, W, Ho, Wo, C = (r[n] for n in ("N", "H", "W", "Ho", "Wo", "C"))
        hi = torch.arange(Ho) * H // Ho
        wi = torch.arange(Wo) * W // Wo
        idx = (hi[:, None] * W + wi[None, :]).flatten()
        dy = inp["dy"].double().view(N, Ho * Wo, C)
        dx = torch.zeros(N, H * W, C, dtype=torch.float64).index_add_(1, idx, dy)
        mx = torch.zeros(N, H * W, C, dtype=torch.float64).index_add_(1, idx, dy.abs())
        return {"dx": (dx.view(N, H, W, C), mx.view(N, H, W, C), "bf16")}
    if k == "concat_channels":
        return {"y": (torch.cat([inp["a"], inp["b"]], -1), None, "exact")}
    if k == "split_channels":
        return {"a": (inp["g"][:, :r["Ca"]].contiguous(), None, "exact"), "b": (inp["g"][:, r["Ca"]:].contiguous(), None, "exact")}
    if k in ("add_bf16", "add_f32"):
        ts = [inp[n].double() for n in ("a", "b", "c") if n in inp]
        return {"y": (sum(ts), sum(t.abs() for t in ts), "bf16" if k == "add_bf16" else "f32")}
    if k == "scale_bf16":
        y = float(np.float32(r["alpha"])) * inp["a"].double()
        return {"y": (y, y.abs(), "bf16")}
    if k == "cast_f32_bf16":
        return {"y": (inp["src"].bfloat16(), None, "exact")}
    if k == "cast_bf16_f32":
        return {"y": (inp["src"].float(), None, "exact")}
    if k == "dropout_scale_add":
        keep = keep_mask(r["n"], r["p"], inp["seed"], inp["epoch"])
        kf = float(np.float32(r["scale"])) / (1 - float(np.float32(r["p"])))
        x = inp["x"].double()
        base = inp["base"].double() if "base" in inp else torch.zeros_like(x)
        y = base + kf * x
        return {"y": (y[keep], base[keep].abs() + (kf * x[keep]).abs(), "bf16"),
                "dropped": ((inp["base"] if "base" in inp else torch.zeros(r["n"], dtype=torch.bfloat16))[~keep], None, "exact"),
                "_keep": keep}
    if k == "embed_tokens":
        ids = inp["ids"].clamp(0, r["vocab"] - 1).flatten()
        L = r["L"]
        tok, pos = inp["tok"].double()[ids], inp["pos"].double()[:L].repeat(r["B"], 1)
        return {"y": (tok + pos, tok.abs() + pos.abs(), "bf16")}
    if k == "embed_tokens_bwd":
        B, L, C, V = r["B"], r["L"], r["C"], r["vocab"]
        ids = inp["ids"].clamp(0, V - 1).flatten()
        dy = inp["dy"].double()
        out = {}
        if r["dtok"]:
            used = torch.unique(ids)
            pre = inp["dtok"].double()[used]
            s = torch.zeros(V, C, dtype=torch.float64).index_add_(0, ids, dy)[used]
            sa = torch.zeros(V, C, dtype=torch.float64).index_add_(0, ids, dy.abs())[used]
            untouched = torch.ones(V, dtype=torch.bool)
            untouched[used] = False
            out["dtok"] = (pre + s, pre.abs() + sa, "f32")
            out["dtok_untouched"] = (inp["dtok"][untouched], None, "exact")
            out["_used"] = used
        if r["dpos"]:
            pre = inp["dpos"].double()
            s, sa = pre.clone(), pre.abs()
            s[:L] += dy.view(B, L, C).sum(0)
            sa[:L] += dy.abs().view(B, L, C).sum(0)
            out["dpos"] = (s, sa, "f32")
        return out
    if k in ("gelu_bf16", "gelu_bwd"):
        y, my, g, mg = gelu_terms(inp["x"].double(), r["quick"])
        if k == "gelu_bf16":
            return {"y": (y, my, "bf16")}
        d = inp["dy"].double()
        return {"dx": (d * g, d.abs() * mg, "bf16")}
    if k == "vae_sample":
        B, F, h, w = r["B"], r["F"], r["h"], r["w"]
        mom = inp["moments"].double().view(B, F, h, w, 8)
        mean, lv = mom[..., :4].permute(0, 4, 1, 2, 3), mom[..., 4:].permute(0, 4, 1, 2, 3).clamp(-30.0, 20.0)
        sd, e = torch.exp(0.5 * lv), inp["eps"].double()
        s = float(np.float32(r["scale"]))
        return {"z": ((mean + sd * e) * s, (mean.abs() + sd * e.abs() * (1 + 0.5 * lv.abs())) * s, "f32")}
    if k == "frames_u8_to_nhwc8":
        v, m = bilinear(inp["frames"], r["h"], r["w"])
        return {"y": (v, m, "bf16"), "pad": (_pad_zero(v.shape[:-1] + (5,)), None, "exact")}
    if k == "frames_u8_to_nhwc8_ragged":
        vs = [bilinear(c, r["h"], r["w"]) for c in inp["clips"]]
        v, m = torch.cat([a for a, _ in vs]), torch.cat([b for _, b in vs])
        return {"y": (v, m, "bf16"), "pad": (_pad_zero(v.shape[:-1] + (5,)), None, "exact")}
    raise KeyError(k)


EPS_KEY = {"latents_to_nhwc8": "noise", "mse_loss_fwd": "mse", "mse_loss_bwd": "mse", "velocity_mse_loss_fwd": "vel",
           "velocity_mse_loss_bwd": "vel", "timestep_embedding": "temb", "colsum": "colsum", "colsum_f32": "colsum_f32",
           "upsample_nearest_bwd": "upsample", "add_bf16": "add", "add_f32": "add_f32", "scale_bf16": "scale",
           "dropout_scale_add": "dropout", "embed_tokens": "embed", "embed_tokens_bwd": "embed", "gelu_bf16": "gelu",
           "gelu_bwd": "gelu", "vae_sample": "vae", "frames_u8_to_nhwc8": "resize", "frames_u8_to_nhwc8_ragged": "resize"}


def eps_key(r, out):
    return f"{EPS_KEY[r['kind']]}.{out}"


# ---------------------------------------------------------------------------------------------- layout of the kernel outputs
def split_outputs(r, out):
    """The kernel's raw outputs {name: tensor} -> the tensors reference() describes (pad channels, kept / dropped elements, the
    touched and untouched rows of dtok)."""
    k = r["kind"]
    res = {}
    if k == "latents_to_nhwc8":
        C = r["C"]
        res = {"y": out["y"][..., :C], "pad": out["y"][..., C:]}
    elif k in ("mse_loss_bwd", "velocity_mse_loss_bwd"):
        C = r["C"]
        res = {"dpred": out["dpred"][..., :C], "pad": out["dpred"][..., C:]}
    elif k in ("frames_u8_to_nhwc8", "frames_u8_to_nhwc8_ragged"):
        res = {"y": out["y"][..., :3], "pad": out["y"][..., 3:]}
    else:
        res = dict(out)
    return res


# ---------------------------------------------------------------------------------------------- checks
def _coords(flat, shape):
    out = []
    for n in reversed(shape):
        out.append(flat % n)
        flat //= n
    return "(" + ", ".join(map(str, reversed(out))) + ")"


def _bits(t):
    t = t.contiguous()
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])


def check_exact(y, ref, what):
    ref = ref.to(y.device)
    if ref.dtype == torch.float64:
        ref = ref.to(y.dtype)
    assert tuple(y.shape) == tuple(ref.shape), (what, tuple(y.shape), tuple(ref.shape))
    assert y.dtype == ref.dtype, (what, y.dtype, ref.dtype)
    bad = _bits(y) != _bits(ref)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ in bits; first at {_coords(i, tuple(y.shape))}: "
                             f"y={float(y.flatten()[i])!r} r={float(ref.flatten()[i])!r}")
    return 0.0, 0.0


def check(y, r, m, key, rounded, what):
    """Asserts the per-element bound and the L2 bound of `y` against the float64 reference `r` with magnitude `m` (eps EPS[key]).
    Returns (ratio, relative L2 error): ratio = max |y - r| / m, for bf16 output max (|y - r| - 2^-8 |r|) / m."""
    r, m = r.to(y.device), m.to(y.device)
    assert tuple(y.shape) == tuple(r.shape), (what, tuple(y.shape), tuple(r.shape))
    eps = EPS[key]
    yd = y.double()
    err = (yd - r).abs()
    bound = eps * m + (U_BF16 * r.abs() if rounded else 0.0)
    ok = err <= bound
    l2 = float((yd - r).norm() / r.norm().clamp_min(1e-300))
    excess = (err - U_BF16 * r.abs()).clamp_min(0) if rounded else err
    ratio = float(torch.where(m > 0, excess / m.clamp_min(1e-300), torch.where(excess > 0, math.inf, 0.0)).nan_to_num(nan=math.inf).max()) \
        if y.numel() else 0.0
    if not bool(ok.all()):
        score = torch.where(ok, torch.full_like(err, -1.0), (err - bound) / bound.clamp_min(1e-300)).nan_to_num(nan=math.inf)
        i = int(score.flatten().argmax())
        yv, rv, mv, bv = (float(t.flatten()[i]) for t in (yd, r, m, bound))
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements out of bound; worst at {_coords(i, tuple(y.shape))}: "
                             f"y={yv!r} r={rv!r} m={mv!r} |y-r|={abs(yv - rv)!r} > bound {bv!r}; rel L2 {l2:.3e}")
    assert not rounded or l2 <= U_BF16, f"{what}: relative L2 error {l2:.3e} > {U_BF16:.3e}"
    return ratio, l2


def _periods(y, K):
    """A flat output of a launch whose input repeats with period K, cut into its periods (the last one may be short)."""
    flat = y.reshape(-1)
    return [flat[i:i + K] for i in range(0, flat.numel(), K)]


def assert_gelu_tail(x, what):
    lim, frac = GELU_TAIL
    got = float((x.double() < lim).double().mean())
    assert got >= frac, f"{what}: only {got:.2%} of x below {lim} (the inputs must exercise the negative tail of GELU)"


def check_outputs(r, inp, out, what, ref=None):
    """Checks every output of launch `r` ({name: tensor} as the kernel wrote it, on any device); returns {name: (ratio, l2)}."""
    if ref is None:
        ref = reference(r, inp)
    k = r["kind"]
    if k.startswith("gelu"):
        assert_gelu_tail(inp["x"], what)
    got = split_outputs(r, out)
    if k == "dropout_scale_add":
        keep = ref["_keep"].to(got["y"].device)
        got = {"y": got["y"][keep], "dropped": got["y"][~keep]}
    if k == "embed_tokens_bwd" and "dtok" in got:
        used = ref["_used"].to(got["dtok"].device)
        untouched = torch.ones(r["vocab"], dtype=torch.bool, device=used.device)
        untouched[used] = False
        got = dict(got, dtok=got["dtok"][used], dtok_untouched=got["dtok"][untouched])
    res = {}
    for name, val in ref.items():
        if name.startswith("_"):
            continue
        rv, m, mode = val
        y = got[name]
        periodic = "n" in r and y.numel() > rv.numel() and k not in ("dropout_scale_add",) and k not in ("gelu_bf16", "gelu_bwd")
        parts = _periods(y, rv.numel()) if periodic else [y]
        worst = (0.0, 0.0)
        for part in parts:
            n = part.numel()
            rr = rv.reshape(-1)[:n] if periodic else rv
            mm = (m.reshape(-1)[:n] if periodic else m) if m is not None else None
            if mode == "exact":
                one = check_exact(part, rr, f"{what} {name}")
            else:
                one = check(part, rr, mm, eps_key(r, name), mode == "bf16", f"{what} {name}")
            worst = max(worst, one)
        res[name] = worst
    return res


def old_metric(y, r):
    """max|y - r| / max|r|: the per-kernel tests' tolerance metric (they accept < 1e-2)."""
    return float((y.double() - r.to(y.device)).abs().max() / r.abs().max())
