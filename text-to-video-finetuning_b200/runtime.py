"""Step-level runtime: flat parameter arena (fp32 master / fp32 gradient / bf16 compute shadow), the single
data-parallel gradient all-reduce, and CUDA-graph capture of the whole forward+backward.

H100-first design notes
  * 80 GB of HBM per GPU holds three flat copies of a 1.4 B-parameter model (5.6 + 5.6 + 2.8 GB) with room to spare, and a
    flat layout turns per-step housekeeping into three kernels: one memset (zero grads), one cast (fp32 -> bf16 shadow
    in kernel layout) and ONE ncclAllReduce over NVLink/NVSwitch for the gradients (the north-star's only collective;
    the reference reaches NCCL implicitly through accelerate/DDP, train.py:661,861).
  * A step has ~4-5 thousand kernel launches; replaying it as a CUDA graph removes the host launch cost entirely.
"""
import os

import torch
import torch.distributed as dist

from . import ops, prims


def _align(n, a=64):
    return (n + a - 1) // a * a


def _has_shadow(p):
    """GEMM weights (rank >= 2) get a bf16 compute copy; a lookup table marked `_t2v_lookup` (an embedding, gathered from its
    fp32 master) is stored with the vectors instead, so no shadow is kept or rewritten for it."""
    return p.dim() >= 2 and not getattr(p, "_t2v_lookup", False)


class ParamArena:
    """Adopts a module's parameters into flat buffers.  Parameters keep their identity, shape, strides and names;
    only their storage moves.  `param.grad` becomes a view into the flat gradient buffer and matrix-like weights (not
    lookup tables) get a `_t2v_shadow` bf16 view in kernel layout ([Cout, KH, KW, Cin] / [out, 1, 1, in])."""

    def __init__(self, module, device=None, extra=()):
        # extra: parameters outside `module` to adopt as well (the text-encoder LoRA factors of a text-LoRA run)
        params = [p for p in module.parameters()]
        params += [p for p in extra if all(p is not q for q in params)]
        if not params:
            raise ValueError("module has no parameters")
        device = device or params[0].device
        for p in params:
            if p.dtype != torch.float32:
                raise ValueError("ParamArena expects fp32 master parameters (the reference keeps the UNet in fp32 under autocast)")
        # matrices first (they need a bf16 shadow), then vectors; inside each class the TRAINABLE parameters come first (in
        # registration order), so the gradients that have to cross NVLink form two compact spans - 29 M elements instead of
        # 1.44 B for a LoRA run - and a block's trainable matrices stay one contiguous range.
        mats = [p for p in params if _has_shadow(p)]
        vecs = [p for p in params if not _has_shadow(p)]
        mats = [p for p in mats if p.requires_grad] + [p for p in mats if not p.requires_grad]
        vecs = [p for p in vecs if p.requires_grad] + [p for p in vecs if not p.requires_grad]
        self.params = mats + vecs
        self._flags = [p.requires_grad for p in self.params]
        offs, off = [], 0
        for p in self.params:
            offs.append(off)
            off += _align(p.numel())
        self.total = off
        self.n_mat = sum(_align(p.numel()) for p in mats)
        t_mat = sum(_align(p.numel()) for p in mats if p.requires_grad)
        t_vec = sum(_align(p.numel()) for p in vecs if p.requires_grad)
        self.trainable_spans = [(0, t_mat), (self.n_mat, self.n_mat + t_vec)]   # what a data-parallel step has to all-reduce
        self.master = torch.zeros(self.total, device=device, dtype=torch.float32)
        self.grad = torch.zeros(self.total, device=device, dtype=torch.float32)
        self.shadow = torch.zeros(max(self.n_mat, 8), device=device, dtype=torch.bfloat16)
        with torch.no_grad():
            for p, o in zip(self.params, offs):
                n = p.numel()
                src = p.detach().to(device)
                phys = ops._phys(src) if _has_shadow(p) else src
                if not phys.is_contiguous():
                    raise ValueError("conv weights must be in channels_last memory format before adoption")
                self.master[o:o + n].copy_(phys.reshape(-1))
                view = torch.as_strided(self.master, p.shape, p.stride(), o)
                p.data = view
                # frozen parameters keep grad None, so optimizers skip them exactly as they do in the reference
                p.grad = torch.as_strided(self.grad, p.shape, p.stride(), o) if p.requires_grad else None
                if _has_shadow(p):
                    p._t2v_shadow = self.shadow[o:o + n].view(ops._phys(view).shape)
        self.offsets = offs
        self._attach_fused(module, {id(p): o for p, o in zip(self.params, offs)})
        self.refresh_shadow()

    def _attach_fused(self, module, off_of):
        """Attention projections registered back to back (to_q, to_k, to_v) are adjacent in the arena: expose them as
        one [3C, in] (self-attention) or [2C, ctx] (cross-attention K|V) matrix so they run as a single GEMM."""
        import torch.nn as nn
        for m in module.modules():
            if not all(type(getattr(m, a, None)) is nn.Linear for a in ("to_q", "to_k", "to_v")):
                continue
            ws = [m.to_q.weight, m.to_k.weight, m.to_v.weight]
            if any(w.dim() != 2 or id(w) not in off_of or m_.bias is not None for w, m_ in zip(ws, (m.to_q, m.to_k, m.to_v))):
                continue
            o = [off_of[id(w)] for w in ws]
            n = [w.numel() for w in ws]
            group = None
            if ws[0].shape == ws[1].shape == ws[2].shape and o[1] == o[0] + n[0] and o[2] == o[1] + n[1]:
                group = ("qkv", ws, o[0])
            elif ws[1].shape == ws[2].shape and o[2] == o[1] + n[1]:
                group = ("kv", ws[1:], o[1])
            if group is None:
                continue
            kind, params, start = group
            rows, cin = sum(w.shape[0] for w in params), params[0].shape[1]
            total = rows * cin
            m._t2v_fused = (kind, ops.FusedWeight(params, self.shadow[start:start + total].view(rows, 1, 1, cin),
                                                 self.grad[start:start + total].view(rows, 1, 1, cin)))

    def refresh_shadow(self):
        """fp32 master -> bf16 compute copy for every matrix parameter: one kernel over the flat buffer."""
        if self.n_mat:
            prims.cast_f32_bf16(self.master[:self.n_mat], self.shadow[:self.n_mat])

    def zero_grads(self):
        self.grad.zero_()

    def reattach_grads(self):
        """optimizer.zero_grad(set_to_none=True) drops the views; put them back (trainable parameters only: a frozen
        parameter's grad stays None, which is what makes torch optimizers skip it - no weight decay on frozen weights).
        Runs before every step: when every parameter still holds the gradient object set here last time, nothing is done."""
        views = getattr(self, "_grad_views", None)
        if views is not None and all(p.grad is v for p, v in zip(self.params, views)):
            return
        for p, o in zip(self.params, self.offsets):
            if not p.requires_grad:
                p.grad = None
            elif p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * o:
                p.grad = torch.as_strided(self.grad, p.shape, p.stride(), o)
        self._grad_views = [p.grad for p in self.params]

    def grad_norm(self):
        return self.grad.norm()

    def check_layout(self):
        """The trainable-first layout is fixed when the arena is built; flipping requires_grad afterwards needs a new arena."""
        if any(p.requires_grad != f for p, f in zip(self.params, self._flags)):
            raise RuntimeError("requires_grad changed after the parameter arena was built: rebuild the DataParallelStep")


def allreduce_gradients(arena, world_size=None, average=True):
    """The one collective of the step, un-overlapped form (T2V_NO_OVERLAP=1): all-reduce the trainable spans of the flat
    fp32 gradient buffer over NCCL (NVLink 5 / NVSwitch)."""
    if not (dist.is_available() and dist.is_initialized()):
        return None
    world_size = world_size or dist.get_world_size()
    if world_size == 1:
        return None
    for lo, hi in arena.trainable_spans:
        if hi > lo:
            view = arena.grad[lo:hi]
            if average:
                view.div_(world_size)
            dist.all_reduce(view, op=dist.ReduceOp.SUM, async_op=False)
    return None


class GradientBuckets:
    """Overlaps the gradient all-reduce with the backward pass.

    The flat gradient buffer holds the trainable weight matrices in registration order, so those of one top-level block
    (down_blocks.i / mid_block / up_blocks.i) are one contiguous range.  The model marks the input of every block
    (ops.grad_mark); when the backward pass reaches a mark, that block's range is complete and its all-reduce is issued
    asynchronously (NCCL runs it on its own stream, also inside a captured CUDA graph) while the rest of the backward keeps
    the SMs busy.  `finish()` reduces what is left of the trainable spans (stem, time embedding, all vectors, and the text-encoder LoRA
    factors, whose gradients are complete only once the text encoder's backward has run) and joins.

    compress (default on NCCL): gradients cross NVLink as bf16.  Each range is scaled by 1 / world and rounded into a flat
    bf16 twin of the gradient buffer (one pass, 6 B / parameter, overlapped like the collective itself), the SUM all-reduce
    runs on that twin - half the bytes on the wire - and the fused AdamW reads its gradient values straight from it
    (optim.FusedAdamW.launch(grad_bf16=...)), so nothing is widened back.  Accumulation across micro-steps stays fp32.
    Pieces of at most PIECE elements keep every collective short enough to pipeline behind the next block's backward."""

    PIECE = 1 << 26   # 64 Mi elements = 128 MiB of bf16 per collective

    def __init__(self, arena, module, group=None, compress=None):
        self.arena, self.module, self.group = arena, module, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        off_of = {id(p): o for p, o in zip(arena.params, arena.offsets)}
        ranges = {}
        for name, p in module.named_parameters():
            if p.dim() < 2 or id(p) not in off_of or not p.requires_grad:
                continue
            parts = name.split(".")
            key = ".".join(parts[:2]) if parts[0] in ("down_blocks", "up_blocks") else parts[0]
            lo, hi = off_of[id(p)], off_of[id(p)] + _align(p.numel())
            a, b = ranges.get(key, (lo, hi))
            ranges[key] = (min(a, lo), max(b, hi))
        self.ranges = {k: v for k, v in ranges.items() if k.startswith(("down_blocks.", "up_blocks.")) or k == "mid_block"}
        spans = sorted(self.ranges.values())
        for (a0, b0), (a1, b1) in zip(spans, spans[1:]):
            if b0 > a1:
                raise RuntimeError("block gradient ranges overlap: parameters are not laid out in registration order")
        self.armed = False
        self._done, self._works = set(), []
        nccl = dist.is_initialized() and dist.get_backend(group) == "nccl"
        if compress is None and os.environ.get("T2V_GRAD_COMPRESS") is not None:   # A/B switch: 0 = fp32 on the wire
            compress = os.environ["T2V_GRAD_COMPRESS"] not in ("0", "")
        self.compress = nccl if compress is None else bool(compress)
        self.comm = torch.zeros(arena.total, device=arena.grad.device, dtype=torch.bfloat16) if self.compress else None
        self._op = dist.ReduceOp.AVG if nccl else dist.ReduceOp.SUM
        self.bytes_on_wire = 0   # per-rank payload handed to the collectives of the last step

    def install(self):
        self.module._t2v_grad_hook = self.on_block_done

    def _reduce(self, a, b):
        while a < b:
            e = min(b, a + self.PIECE)
            if self.compress:
                view = self.comm[a:e]
                prims.scale_cast_f32_bf16(self.arena.grad[a:e], view, 1.0 / self.world)
                self._works.append(dist.all_reduce(view, op=dist.ReduceOp.SUM, group=self.group, async_op=True))
            else:
                view = self.arena.grad[a:e]
                if self._op == dist.ReduceOp.SUM:
                    view.div_(self.world)
                self._works.append(dist.all_reduce(view, op=self._op, group=self.group, async_op=True))
            self.bytes_on_wire += view.numel() * view.element_size()
            a = e

    def on_block_done(self, key):
        if not self.armed or key in self._done or key not in self.ranges:
            return
        if not self._done:
            self.bytes_on_wire = 0
        self._done.add(key)
        self._reduce(*self.ranges[key])

    def finish(self):
        """Reduce every part of the trainable spans no mark has covered, then make the current stream wait for all of it."""
        if not self._done:
            self.bytes_on_wire = 0
        covered = sorted(self.ranges[k] for k in self._done)
        for lo, hi in self.arena.trainable_spans:
            pos = lo
            for a, b in covered + [(hi, hi)]:
                a, b = max(a, lo), min(b, hi)
                if a > pos:
                    self._reduce(pos, min(a, hi))
                pos = max(pos, b)
                if pos >= hi:
                    break
        for w in self._works:
            w.wait()
        self.last_overlapped = len(self._done)   # blocks whose all-reduce started inside the backward pass
        self._works, self._done, self.armed = [], set(), False

    def widen(self):
        """compress mode without a fused optimizer: write the reduced gradients back into the fp32 buffer."""
        if self.compress:
            for lo, hi in self.arena.trainable_spans:
                if hi > lo:
                    prims.cast_bf16_f32(self.comm[lo:hi], self.arena.grad[lo:hi])


class GraphedStep:
    """Captures `fn(*static_inputs)` (forward + backward [+ optimizer] of one clip batch) into a CUDA graph and replays it.

    `fn` must be free of host synchronisation and allocate only through PyTorch's caching allocator (true for every
    Function in ops.py).  Inputs are copied into static buffers before each replay.  `snapshot`: tensors that `fn` mutates
    in place (weights, gradient buffer, optimizer state); they are saved before the warm-up / capture dry runs and restored
    afterwards, so building the graph does not advance training."""

    def __init__(self, fn, example_inputs, warmup=2, snapshot=()):
        self.fn = fn
        self.static_in = [x.clone() for x in example_inputs]
        saved = [t.clone() for t in snapshot]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self.static_out = fn(*self.static_in)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_out = fn(*self.static_in)
        with torch.no_grad():
            for t, s in zip(snapshot, saved):
                t.copy_(s)
        torch.cuda.synchronize()

    def __call__(self, *inputs):
        for dst, src in zip(self.static_in, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_out
