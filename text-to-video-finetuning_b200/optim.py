"""Fused AdamW + global-norm gradient clipping on the flat parameter arena (SURVEY 8(f) row 1).

Reference: `torch.optim.AdamW` built at train.py:616-623, `accelerator.clip_grad_norm_(..., max_grad_norm)` at :868-876,
`optimizer.zero_grad()` at :879.  Here one optimizer step is three kernel launches per hyper-parameter set (csrc/optim.cu):
sum of squared gradients -> device-side scalars (step count, bias corrections, clip factor) -> update, which also writes the
bf16 compute shadow of every updated matrix (runtime.ParamArena.refresh_shadow is no longer needed per step) and zeroes the
gradient ranges it consumed (no per-step memset).  Nothing in `launch()` touches the host, so the optimizer is captured
into the CUDA graph of the training step; the learning rate reaches the device through `push_hyperparams()`.

Frozen parameters are never touched (torch semantics: grad None => skipped, no weight decay either).

`AdamW8bit` (`use_8bit_adam`, reference train.py:238-249) is the same step with blockwise 8-bit moments for tensors of at
least 4096 elements; its algorithm is stated on the class and on `dynamic_map`.

With `ema_decay` (`use_ema`), both keep an exponential moving average of the trained weights, updated by the same kernel
launch as the weights (diffusers' `EMAModel` with its default arguments; see `FusedAdamW`).
"""
import bisect
import contextlib
import math

import torch

from . import prims
from .runtime import _align

CHUNK = 1 << 16   # elements per chunk-table entry


def check_ema_decay(ema_decay):
    """The EMA decay cap as a float; ValueError unless it is finite and in [0, 1]."""
    d = float(ema_decay)
    if not (math.isfinite(d) and 0.0 <= d <= 1.0):
        raise ValueError(f"ema_decay = {ema_decay!r}: the EMA decay must be a finite number in [0, 1]")
    return d


class FusedAdamW(torch.optim.Optimizer):
    """ema_decay (None: no EMA): keep an fp32 exponential moving average of every trainable tensor, updated in the update
    kernel on the new weights while they are still in registers.  With k the step count after this step's increment,
    d_1 = 0 and d_k = min(ema_decay, k / (9 + k)), and ema -= (1 - d_k) * (ema - p): diffusers' `EMAModel.step` with its
    defaults (`(1 + s) / (10 + s)` with s = k - 1, no warm-up power, `min_decay` 0, `update_after_step` 0).  k is read on
    the device, so a replayed CUDA graph uses each step's decay.  The EMA is compact (the trainable tensors of this
    optimizer only, in arena order, each starting at a multiple of 64 elements) and starts as a copy of the weights; a frozen
    parameter's EMA is the parameter itself.  `ema_weights()` swaps it into the model."""

    def __init__(self, arena, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=None, ema_decay=None):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.arena = arena
        self.max_grad_norm = max_grad_norm
        dev = arena.master.device
        self.state_dev = torch.zeros(1, device=dev, dtype=torch.int64)     # [0] optimizer step count
        self.sq = torch.zeros(2, device=dev, dtype=torch.float64)          # [0] sum g^2 (running), [1] last gradient norm
        self._off = {id(p): o for p, o in zip(arena.params, arena.offsets)}
        for group in self.param_groups:
            for p in group["params"]:
                if id(p) not in self._off:
                    raise ValueError("FusedAdamW only drives parameters that live in the arena")
        self._alloc_state()
        self.ema_decay = None if ema_decay is None else check_ema_decay(ema_decay)
        self.ema = None if ema_decay is None else self._alloc_ema()
        self._sets = None
        self._build()

    def _alloc_state(self):
        self.exp_avg = torch.zeros_like(self.arena.master)
        self.exp_avg_sq = torch.zeros_like(self.arena.master)

    def _moments(self):
        """Name -> device tensor of the optimizer's moment state (what `state_dict` saves besides the step count)."""
        return {"exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq}

    def _saved(self):
        """_moments() plus the EMA when there is one: every tensor `state_dict` saves besides the step count."""
        return self._moments() if self.ema is None else dict(self._moments(), ema=self.ema)

    def state_tensors(self):
        """Every device tensor one step mutates besides the weights and gradients (a CUDA-graph capture snapshots them)."""
        return list(self._saved().values()) + [self.state_dev, self.sq]

    # ------------------------------------------------------------------------------------------------ EMA
    def _trainable_sorted(self):
        return sorted((p for g in self.param_groups for p in g["params"] if p.requires_grad), key=lambda q: self._off[id(q)])

    def _alloc_ema(self):
        """The compact EMA, a copy of the current trainable weights (alignment padding included, which the arena keeps at 0)."""
        master = self.arena.master
        self._ema_starts, self._ema_base, n = [], [], 0   # arena offset and EMA offset of each trainable tensor, arena order
        for p in self._trainable_sorted():
            self._ema_starts.append(self._off[id(p)])
            self._ema_base.append(n)
            n += _align(p.numel())
        ema = torch.empty(n, device=master.device, dtype=torch.float32)
        for a, e, b in zip(self._ema_starts, self._ema_base, self._ema_base[1:] + [n]):
            ema[e:b].copy_(master[a:a + b - e])
        return ema

    def _ema_rows(self, rows):
        """`rows` with the EMA offset of each row's first element appended.  A row spans arena-adjacent trainable tensors
        only, and those are adjacent in the EMA as well."""
        out = []
        for r in rows:
            i = bisect.bisect_right(self._ema_starts, r[0]) - 1
            out.append(tuple(r) + (self._ema_base[i] + r[0] - self._ema_starts[i],))
        return out

    @contextlib.contextmanager
    def ema_weights(self):
        """Within the `with` block the model holds the EMA weights (master and bf16 shadow); on exit the training weights
        and the EMA are swapped back, bit for bit.  Frozen parameters are left as they are."""
        if self.ema is None:
            raise RuntimeError("ema_weights() needs an optimizer built with ema_decay")
        ar = self.arena
        prims.ema_swap_chunks(ar.master, self.ema, ar.shadow, ar.n_mat, self._ema_swap)
        try:
            yield
        finally:
            prims.ema_swap_chunks(ar.master, self.ema, ar.shadow, ar.n_mat, self._ema_swap)

    # ------------------------------------------------------------------------------------------------ chunk tables
    @staticmethod
    def _key(group):
        return (float(group["lr"]), float(group["betas"][0]), float(group["betas"][1]), float(group["eps"]), float(group["weight_decay"]))

    def _runs(self, params):
        """Contiguous [a, b) ranges of the trainable parameters among `params` in arena order (alignment gaps between
        adjacent parameters hold zeros in master / grad / state and are swept along)."""
        spans = sorted((self._off[id(p)], self._off[id(p)] + _align(p.numel())) for p in params if p.requires_grad)
        runs = []
        for a, b in spans:
            if runs and runs[-1][1] == a:
                runs[-1][1] = b
            else:
                runs.append([a, b])
        return runs

    def _table(self, params):
        """Update-kernel rows (offset, length) over the trainable `params`, never straddling the matrix / vector boundary."""
        n_mat = self.arena.n_mat
        chunks = []
        for a, b in self._runs(params):
            for lo, hi in ((a, min(b, n_mat)), (max(a, n_mat), b)):
                pos = lo
                while pos < hi:
                    n = min(CHUNK, hi - pos)
                    chunks.append((pos, n))
                    pos += n
        return chunks

    def _build(self):
        """Groups with identical hyper-parameters form one set: one chunk table, one row of device hyper-parameters."""
        by_key = {}
        for gi, group in enumerate(self.param_groups):
            by_key.setdefault(self._key(group), []).append(gi)
        dev = self.arena.master.device
        sets = []
        for key, gis in by_key.items():
            params = [p for gi in gis for p in self.param_groups[gi]["params"]]
            chunks = self._table(params)
            if not chunks:
                continue
            # each table is built on the host and kept there next to its device copy (the host copy is what a table built
            # on the meta device can still be read from)
            host = torch.tensor(chunks, dtype=torch.int64)
            table = host.to(dev)
            sets.append({"groups": gis, "key": key, "chunks": table, "norm_chunks": table[:, :2].contiguous() if table.shape[1] > 2 else table,
                         "n": sum(c[1] for c in chunks), "chunks_host": host})
            if self.ema is not None:
                ema_host = torch.tensor(self._ema_rows(chunks), dtype=torch.int64)
                sets[-1]["ema_chunks"], sets[-1]["ema_chunks_host"] = ema_host.to(dev), ema_host
        if not sets:
            raise ValueError("FusedAdamW: no trainable parameters")
        if self.ema is not None:   # (arena offset, length, EMA offset) over every set: the rows ema_weights() swaps
            self._ema_swap = torch.cat([s["ema_chunks"][:, [0, 1, -1]] for s in sets]).contiguous()
        self._sets = sets
        self.hp_host = torch.zeros((len(sets), 5), dtype=torch.float32)
        if dev.type == "cuda":
            self.hp_host = self.hp_host.pin_memory()
        self.hp_in = torch.zeros((len(sets), 5), device=dev, dtype=torch.float32)
        self.hp = torch.zeros((len(sets), 8), device=dev, dtype=torch.float32)
        self.generation = getattr(self, "generation", 0) + 1   # graphs captured against an older table must be re-captured

    def covers_all_trainable(self):
        """True when every trainable parameter of the arena is updated (and therefore zeroed) by this optimizer."""
        mine = {id(p) for g in self.param_groups for p in g["params"]}
        return all(id(p) in mine for p in self.arena.params if p.requires_grad)

    @property
    def trainable_elements(self):
        return sum(s["n"] for s in self._sets)

    # ------------------------------------------------------------------------------------------------ step
    def push_hyperparams(self):
        """Host -> device copy of (lr, beta1, beta2, eps, weight_decay) per set (stream-ordered, before the step's kernels or
        the graph replay).  A scheduler that makes groups of one set diverge triggers a rebuild of the tables.  The check runs
        only when some group's hyper-parameters differ from the previous call's (a run with one group per tensor has
        ~1,500 groups, and this is host time on every optimizer step)."""
        seen = [(g["lr"], tuple(g["betas"]), g["eps"], g["weight_decay"]) for g in self.param_groups]
        if seen != getattr(self, "_hp_seen", None):
            self._check_sets()
            self._hp_seen = seen
        for i, s in enumerate(self._sets):
            g = self.param_groups[s["groups"][0]]
            self.hp_host[i, 0] = float(g["lr"])
            self.hp_host[i, 1], self.hp_host[i, 2] = float(g["betas"][0]), float(g["betas"][1])
            self.hp_host[i, 3], self.hp_host[i, 4] = float(g["eps"]), float(g["weight_decay"])
        self.hp_in.copy_(self.hp_host, non_blocking=True)

    def _check_sets(self):
        """Rebuild the tables when the groups of one set no longer share their hyper-parameters."""
        for s in self._sets:
            if any(self._key(self.param_groups[gi])[1:] != s["key"][1:] or
                   self.param_groups[gi]["lr"] != self.param_groups[s["groups"][0]]["lr"] for gi in s["groups"]):
                self._build()
                break

    def launch(self, zero_grad=True, grad_bf16=None):
        """The device-only part of one step (capturable): gradient norm, scalars, update.  grad_bf16: flat bf16 twin of the
        gradient buffer holding the all-reduced gradients (runtime.GradientBuckets.comm); the fp32 buffer is then only zeroed."""
        ar = self.arena
        if self.max_grad_norm is not None:
            for s in self._sets:
                prims.sqnorm_chunks(ar.grad, s["norm_chunks"], self.sq, grad_bf16)
        prims.adamw_prepare(self.hp_in, self.hp, self.state_dev, self.sq, self.max_grad_norm or 0.0)
        for i, s in enumerate(self._sets):
            self._update(s, self.hp[i], zero_grad, grad_bf16)

    def _update(self, s, hp_row, zero_grad, grad_bf16):
        ar = self.arena
        if self.ema is None:
            prims.adamw_chunks(ar.master, ar.grad, self.exp_avg, self.exp_avg_sq, ar.shadow, ar.n_mat, s["chunks"], hp_row, zero_grad, grad_bf16)
        else:
            prims.adamw_ema_chunks(ar.master, ar.grad, self.exp_avg, self.exp_avg_sq, ar.shadow, ar.n_mat, s["ema_chunks"], hp_row, self.ema,
                                   self.state_dev, self.ema_decay, zero_grad, grad_bf16)

    @torch.no_grad()
    def step(self, closure=None, zero_grad=True):
        loss = closure() if closure is not None else None
        self.push_hyperparams()
        self.launch(zero_grad)
        return loss

    def zero_grad(self, set_to_none=False):
        """Gradients live in the arena and are zeroed by the update kernel; an explicit call zeroes the whole flat buffer."""
        self.arena.zero_grads()

    @property
    def steps(self):
        return int(self.state_dev.item())

    def last_grad_norm(self):
        """Global gradient norm seen by the last step (device scalar, fp64); only maintained when clipping is on."""
        return self.sq[1]

    # ------------------------------------------------------------------------------------------------ checkpointing
    def state_dict(self):
        d = super().state_dict()
        d["fused"] = dict(self._saved(), step=self.steps)
        return d

    def load_state_dict(self, state_dict):
        fused = state_dict.pop("fused", None)
        super().load_state_dict(state_dict)
        if fused is not None:
            for name, t in self._saved().items():
                t.copy_(fused[name])
            self.state_dev.fill_(int(fused["step"]))


# ---------------------------------------------------------------------------------------------------- blockwise 8-bit AdamW
MIN_8BIT_SIZE = 4096   # tensors with fewer elements keep fp32 moments
QBLOCK = 256           # elements per quantisation block


def dynamic_map(signed):
    """The 256-entry dynamic-tree quantisation map of Dettmers et al., *8-bit Optimizers via Block-wise Quantization*
    (ICLR 2022), with bitsandbytes' `create_dynamic_map` defaults (7 exponent levels, 8 bits), as sorted fp32 values.

    A code's leading zero bits select a decade 10^(e-6), e = 0..6; the bits after the first one (the indicator) select one
    of 2^k linearly spaced fractions of that decade: the midpoints of `linspace(0.1, 1, 2^k + 1)`.  Signed (for m): one
    sign bit, so decade e holds 2^e fractions, each with both signs (2 * 127 values).  Unsigned (for v): decade e holds
    2^(e+1) fractions (254 values).  0 and 1 are added, so both maps hold 256 distinct entries, contain 0 and 1 exactly, and
    are densest near 0, where most normalised moments fall.  Computed in fp32 like the reference construction."""
    data = []
    for e in range(7):
        n = 2 ** e if signed else 2 ** (e + 1)
        bounds = torch.linspace(0.1, 1, n + 1, dtype=torch.float32)
        means = (bounds[:-1] + bounds[1:]) / 2.0
        data += ((10 ** (e - 6)) * means).tolist()
        if signed:
            data += (-(10 ** (e - 6)) * means).tolist()
    data += [0.0, 1.0]
    assert len(data) == 256
    return torch.tensor(sorted(data), dtype=torch.float32)


class AdamW8bit(FusedAdamW):
    """AdamW with blockwise 8-bit moments (bitsandbytes `AdamW8bit` defaults: block size 256, `min_8bit_size` 4096, no
    percentile clipping) on the flat arena; the reference builds `bitsandbytes.optim.AdamW8bit` for `use_8bit_adam`.

    A trainable tensor with fewer than MIN_8BIT_SIZE elements keeps fp32 m and v and gets exactly FusedAdamW's update.  A
    larger one is cut into blocks of QBLOCK consecutive elements from its first element; each block stores one uint8 code
    per element and one fp32 absmax per moment, m through the signed `dynamic_map`, v through the unsigned one.  Per element:
        g *= clip;  m = b1 * deq(m) + (1 - b1) * g;  v = b2 * deq(v) + (1 - b2) * g^2   with deq(c) = map[c] * absmax_old
        p *= 1 - lr * wd;  p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)          (the unquantised fp32 m and v)
    then per block absmax = max |m| (|v|) and code = the smallest i with m / absmax <= 0.5f * (map[i] + map[i+1]); a block
    whose absmax is 0 stores the code of 0.0.  The state is compact: it covers the trainable tensors only, in arena order,
    each tensor's 8-bit state starting at a multiple of QBLOCK.  One update launch per hyper-parameter set
    (csrc/optim.cu adamw8bit_chunks_kernel); the clipping norm and the device scalars are FusedAdamW's."""

    def _alloc_state(self):
        dev = self.arena.master.device
        self._layout, n8, n32 = {}, 0, 0   # id(param) -> (bits, state offset)
        params = [p for g in self.param_groups for p in g["params"] if p.requires_grad]
        for p in sorted(params, key=lambda q: self._off[id(q)]):
            n = _align(p.numel())
            if p.numel() >= MIN_8BIT_SIZE:
                self._layout[id(p)] = (8, n8)
                n8 += _align(n, QBLOCK)
            else:
                self._layout[id(p)] = (32, n32)
                n32 += n
        qmaps = torch.cat([dynamic_map(True), dynamic_map(False)])
        zero_m = int((qmaps[:256] == 0).nonzero()[0, 0])   # on the host map: a meta-device map has no values
        self.qmaps = qmaps.to(dev)
        self.code_m = torch.full((n8,), zero_m, device=dev, dtype=torch.uint8)
        self.code_v = torch.zeros(n8, device=dev, dtype=torch.uint8)   # the unsigned map starts at 0.0
        self.absmax_m = torch.zeros(n8 // QBLOCK, device=dev, dtype=torch.float32)
        self.absmax_v = torch.zeros(n8 // QBLOCK, device=dev, dtype=torch.float32)
        self.exp_avg32 = torch.zeros(n32, device=dev, dtype=torch.float32)
        self.exp_avg_sq32 = torch.zeros(n32, device=dev, dtype=torch.float32)

    def _moments(self):
        return {"code_m": self.code_m, "code_v": self.code_v, "absmax_m": self.absmax_m, "absmax_v": self.absmax_v,
                "exp_avg32": self.exp_avg32, "exp_avg_sq32": self.exp_avg_sq32}

    def state_bytes(self):
        return sum(t.numel() * t.element_size() for t in self._moments().values())

    def _table(self, params):
        """Rows (arena offset, length, state offset, bits): at most CHUNK elements, inside one tensor (CHUNK is a multiple of
        QBLOCK, so every 8-bit row but a tensor's last covers whole blocks)."""
        rows = []
        for p in sorted((p for p in params if p.requires_grad), key=lambda q: self._off[id(q)]):
            a, n = self._off[id(p)], _align(p.numel())
            bits, s = self._layout[id(p)]
            for lo in range(0, n, CHUNK):
                rows.append((a + lo, min(CHUNK, n - lo), s + lo, bits))
        return rows

    def _update(self, s, hp_row, zero_grad, grad_bf16):
        ar = self.arena
        if self.ema is None:
            prims.adamw8bit_chunks(ar.master, ar.grad, ar.shadow, ar.n_mat, s["chunks"], hp_row, self.qmaps, self.exp_avg32, self.exp_avg_sq32,
                                   self.code_m, self.code_v, self.absmax_m, self.absmax_v, zero_grad, grad_bf16)
        else:
            prims.adamw8bit_ema_chunks(ar.master, ar.grad, ar.shadow, ar.n_mat, s["ema_chunks"], hp_row, self.qmaps, self.exp_avg32,
                                       self.exp_avg_sq32, self.code_m, self.code_v, self.absmax_m, self.absmax_v, self.ema, self.state_dev,
                                       self.ema_decay, zero_grad, grad_bf16)
