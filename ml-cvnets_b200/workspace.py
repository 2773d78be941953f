"""Per-model step workspace: ONE flat fp32 gradient buffer that the backward kernels write into directly, plus a persistent, once-per-step
zeroed arena for every statistics accumulator of the step (SURVEY.md 8f row 1, DESIGN.md "step execution").

Why: the reference's step (engine/training_engine.py:257-312) ends in ``clip_grad_norm_`` / ``optimizer.step`` / DDP's bucketed all-reduce,
all of which walk ~200 separate ``.grad`` tensors.  Here every ``p.grad`` is a VIEW of one flat buffer; the autograd functions of the
hot-path modules write their weight gradients into those views (they return ``None`` for the parameters), so

  * the optimizer tail is two launches over the flat buffer (``optim.FlatAdamW``),
  * the data-parallel exchange is an all-reduce of contiguous slices of that buffer, issued per bucket as soon as the backward of the
    modules inside the bucket has finished (overlapping the rest of the backward, like DDP's reducer; main_train.py:90-96),
  * the ~60 little zero-fills per step (fp64 BatchNorm / GroupNorm accumulators, atomically accumulated dW) collapse into two memsets.

Anything that does not know about the workspace still works: autograd accumulates into the same views (``p.grad += g``).
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib as L

ALIGN = 8  # every parameter starts at a multiple of 8 floats (32 B): the weight-gradient kernels use 16-byte vector reductions


class Arena:
    """Zero-initialised fp32 / fp64 scratch handed out in carves (accumulators, kernel-layout gradients), each 16-byte aligned.

    ``rec`` is the record ``[n32, n64]`` of one arena key: the most that earlier calls with that key carved.  The arena is one zeroed buffer
    per dtype of that size -- fresh per call, or a slice of a StepWorkspace zeroed by the step's single memset.  A carve that does not fit
    (no record yet, or a larger shape than before) gets a zeroed tensor of its own and raises the record, so the next call fits."""

    def __init__(self, rec: List[int], device=None, b32: Optional[torch.Tensor] = None, b64: Optional[torch.Tensor] = None):
        self.rec = rec
        self.b32 = torch.zeros(rec[0], device=device, dtype=torch.float32) if b32 is None else b32
        self.b64 = torch.zeros(rec[1], device=device, dtype=torch.float64) if b64 is None else b64
        self.used = [0, 0]  # elements carved so far, fp32 and fp64
        self.c32 = None

    def f32(self, *shape: int) -> torch.Tensor:
        return self._carve(0, self.b32, shape, 4)

    def f64(self, *shape: int) -> torch.Tensor:
        return self._carve(1, self.b64, shape, 2)

    def _carve(self, i: int, buf: torch.Tensor, shape, align: int) -> torch.Tensor:
        n, o = math.prod(shape), self.used[i]
        self.used[i] = end = o + (n + align - 1) // align * align
        self.rec[i] = max(self.rec[i], end)
        v = buf[o:o + n] if end <= buf.numel() else self._own(end - o, buf)[:n]
        return v.view(*shape)

    @staticmethod
    def _own(n: int, like: torch.Tensor) -> torch.Tensor:
        """The tensor of a carve that does not fit the buffer."""
        return torch.zeros(n, device=like.device, dtype=like.dtype)

    def cast(self):
        """fp64 statistics -> fp32 (ONE conversion kernel for the buffer); call after the last kernel that accumulates into them."""
        self.c32 = self.b64.float()

    def as_f32(self, v64: torch.Tensor) -> torch.Tensor:
        o = (v64.data_ptr() - self.b64.data_ptr()) // 8
        if 0 <= o < self.b64.numel():
            return self.c32[o:o + v64.numel()].view(v64.shape)
        return v64.float()  # a carve of its own


class StepWorkspace:
    def __init__(self, model: torch.nn.Module):
        self.params: List[torch.nn.Parameter] = [p for p in model.parameters() if p.requires_grad]
        assert self.params, "model has no trainable parameters"
        dev = self.params[0].device
        assert dev.type == "cuda", "StepWorkspace needs the model on a CUDA device"
        self.device = dev
        self.offsets: Dict[int, Tuple[int, int]] = {}
        o = 0
        for p in self.params:
            assert p.dtype == torch.float32, "parameters must be fp32 (bf16 kernel layouts are a cache, SURVEY.md 8b)"
            k = p.numel()
            self.offsets[id(p)] = (o, k)
            o += (k + ALIGN - 1) // ALIGN * ALIGN
        self.n = o
        self.flat_g = torch.zeros(o, device=dev, dtype=torch.float32)
        self._gviews: Dict[int, torch.Tensor] = {}
        for p in self.params:
            oo, k = self.offsets[id(p)]
            v = self.flat_g[oo:oo + k].view_as(p)
            self._gviews[id(p)] = v
            p.grad = v
        self.active = False           # True only inside TrainStep's forward/backward: modules then write gradients in place
        # batch mixing {mode, lambda, x1, y1, x2, y2} read by the stem gather and the loss (mode 0 = off); device-resident so that a captured
        # step follows per-iteration changes (engine.TrainStep.set_mix)
        self.mix = torch.zeros(6, device=dev, dtype=torch.float32)
        self.mix[1] = 1.0
        self._plan: Dict[tuple, Tuple[List[int], int, int, int, int]] = {}  # arena key -> (record, o32, n32, o64, n64) of its slice
        self._used = set()
        self._buf32 = self._buf64 = None
        self._cast_tables: Dict[tuple, Tuple[torch.Tensor, int, int]] = {}
        # data-parallel buckets
        self.group = None
        self.world = 1
        self.n_buckets = 1
        self._unit_bucket: Dict[Tuple[int, int], int] = {}  # module's flat range -> bucket (planned after the first step)
        self._bucket_range: List[Tuple[int, int]] = []
        self._bucket_count: List[int] = []
        self._bucket_left: List[int] = []
        self._bucket_fired: List[bool] = []
        self._plan_valid = False
        self._seen_units: List[Tuple[int, int]] = []
        self._units_done = 0
        self._works = []
        self.model = model
        for m in model.modules():
            object.__setattr__(m, "_ws", self)

    def __deepcopy__(self, memo):  # EMA deep-copies the model (cvnets/misc/averaging_utils.py:33): the copy has no workspace
        return None

    def detach(self):
        for m in self.model.modules():
            if getattr(m, "_ws", None) is self:
                object.__setattr__(m, "_ws", None)

    # ------------------------------------------------------------------------------------------------------------- gradients
    def gview(self, p: torch.Tensor) -> torch.Tensor:
        return self._gviews[id(p)]

    def has(self, p: torch.Tensor) -> bool:
        return id(p) in self._gviews

    # ----------------------------------------------------------------------------------------------------------------- arena
    def arena(self, key: tuple, rec: List[int]) -> Arena:
        """Scratch for one forward / backward of one module (``rec``: the key's record, see Arena): its slice of the step arena, planned
        from the records and zeroed by begin_step.  Until the slice is planned, or when a call outgrows it, the call's carves are tensors of
        their own and the next begin_step re-plans."""
        plan = self._plan.setdefault(key, (rec, 0, 0, 0, 0))
        if self._buf32 is None or key in self._used:
            return Arena(rec, self.device)
        self._used.add(key)
        _, o32, n32, o64, n64 = plan
        return Arena(rec, b32=self._buf32[o32:o32 + n32], b64=self._buf64[o64:o64 + n64])

    def _replan(self):
        o32 = o64 = 0
        new = {}
        for k, (rec, *_) in self._plan.items():
            n32, n64 = (rec[0] + 7) // 8 * 8, (rec[1] + 3) // 4 * 4  # 32-byte aligned slices
            new[k] = (rec, o32, n32, o64, n64)
            o32 += n32
            o64 += n64
        self._plan = new
        self._buf32 = torch.zeros(max(o32, 8), device=self.device, dtype=torch.float32)
        self._buf64 = torch.zeros(max(o64, 4), device=self.device, dtype=torch.float64)
        self._cast_tables.clear()

    def begin_step(self):
        """Zero the gradient buffer and the arena (two memset nodes), reset the per-step bookkeeping."""
        outgrown = any(r[0] > n32 or r[1] > n64 for r, _, n32, _, n64 in self._plan.values())
        if self._plan and (self._buf32 is None or outgrown):
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("StepWorkspace: run at least two eager steps before capturing the step in a CUDA graph")
            self._replan()
        self._used.clear()
        lib = L.load()
        st = torch.cuda.current_stream().cuda_stream
        lib.cvb_memset_zero(self.flat_g.data_ptr(), self.flat_g.numel() * 4, st)
        if self._buf32 is not None:
            lib.cvb_memset_zero(self._buf32.data_ptr(), self._buf32.numel() * 4, st)
            lib.cvb_memset_zero(self._buf64.data_ptr(), self._buf64.numel() * 8, st)
        self._units_done = 0
        self._works = []
        self._reset_bucket_state()

    # ------------------------------------------------------------------------------------------- fp64 statistics -> fp32 gradients
    def scatter64(self, key: tuple, pairs: Sequence[Tuple[torch.Tensor, torch.Tensor]]):
        """dst32[i] = float(src64[i]) for every (src, dst) pair in ONE launch; the descriptor table is cached once the arena is planned
        (all addresses are then static, which is what makes the step capturable)."""
        if not pairs:
            return
        cached = self._cast_tables.get(key)
        sig = tuple((s.data_ptr(), d.data_ptr(), s.numel()) for s, d in pairs)
        if cached is None or cached[3] != sig:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("StepWorkspace: descriptor table missing during capture (run two eager warm-up steps first)")
            descs = (L.cvb_cast_desc * len(pairs))()
            mx = 1
            for i, (s, d) in enumerate(pairs):
                assert s.dtype == torch.float64 and d.dtype == torch.float32 and s.numel() == d.numel() and s.is_contiguous() and d.is_contiguous()
                descs[i] = L.cvb_cast_desc(s.data_ptr(), d.data_ptr(), s.numel(), 0)
                mx = max(mx, s.numel())
            table = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).to(self.device)
            cached = (table, len(pairs), mx, sig)
            self._cast_tables[key] = cached
        from . import ops
        L.load().cvb_cast_f64_f32(cached[0].data_ptr(), cached[1], cached[2], torch.cuda.current_stream().cuda_stream)
        ops._count()

    # ---------------------------------------------------------------------------------------------- data-parallel gradient exchange
    def enable_ddp(self, group=None, n_buckets: int = 3):
        import torch.distributed as dist
        self.group = group
        self.world = dist.get_world_size(group)
        self.n_buckets = max(1, int(n_buckets))

    def unit_done(self, params: Sequence[torch.Tensor]):
        """Called at the end of a module's backward (after its side-stream weight gradients were joined): its gradients are final.
        Fires the all-reduce of every bucket whose modules are all done (whatever order autograd runs them in)."""
        if self.world == 1 or not self.active:
            return
        offs = [self.offsets[id(p)] for p in params if id(p) in self.offsets]
        if not offs:
            return
        lo = min(o for o, _ in offs)
        hi = max((o + k + ALIGN - 1) // ALIGN * ALIGN for o, k in offs)
        self._units_done += 1
        self._seen_units.append((lo, hi))
        b = self._unit_bucket.get((lo, hi))
        if b is None:
            self._plan_valid = False  # unknown module (first step, or the set of modules changed): exchange everything at the end, re-plan
            return
        if not self._plan_valid:
            return
        self._bucket_left[b] -= 1
        if self._bucket_left[b] == 0:
            self._allreduce(*self._bucket_range[b])
            self._bucket_fired[b] = True

    def _allreduce(self, lo: int, hi: int):
        import torch.distributed as dist
        if hi <= lo:
            return
        self._works.append(dist.all_reduce(self.flat_g[lo:hi], op=dist.ReduceOp.SUM, group=self.group, async_op=True))

    def _plan_buckets(self, units):
        """Contiguous flat ranges cut at module boundaries into ~equal-sized buckets (from the end of the buffer: the classifier's and the
        last stages' gradients are final first); a bucket fires when every module inside it has reported."""
        self._unit_bucket, self._bucket_range, self._bucket_count = {}, [], []
        units = sorted(set(units))
        pos = 0
        for lo, hi in units:  # the reporting modules must tile the whole buffer, else some gradient could arrive after its bucket went out
            if lo != pos:
                return
            pos = hi
        if pos != self.n:
            return
        target = self.n / self.n_buckets
        top, members = self.n, []
        for lo, hi in reversed(units):
            members.append((lo, hi))
            if (top - lo) >= target and len(self._bucket_range) < self.n_buckets - 1 or lo == 0:
                b = len(self._bucket_range)
                self._bucket_range.append((lo, top))
                self._bucket_count.append(len(members))
                for u in members:
                    self._unit_bucket[u] = b
                top, members = lo, []

    def _reset_bucket_state(self):
        self._bucket_left = list(self._bucket_count)
        self._bucket_fired = [False] * len(self._bucket_count)
        self._plan_valid = bool(self._bucket_count)
        self._seen_units = []

    def finish_reduce(self):
        """Everything not yet exchanged goes out now; then the current stream waits for all exchanges."""
        if self.world == 1:
            return
        if self._plan_valid and all(self._bucket_fired):
            pass
        elif not self._works:
            self._allreduce(0, self.n)
        else:  # a partially fired plan (should not happen: an unknown unit invalidates the plan before anything fires out of order)
            for b, fired in enumerate(self._bucket_fired):
                if not fired:
                    self._allreduce(*self._bucket_range[b])
        if not self._plan_valid or not self._bucket_count:
            self._plan_buckets(self._seen_units)
        for w in self._works:
            w.wait()
        self._works = []

    def broadcast_buffers(self, src: int = 0):
        """DDP(broadcast_buffers=True) semantics (SURVEY.md C2): BatchNorm running statistics follow rank ``src``."""
        import torch.distributed as dist
        if self.world == 1:
            return
        bufs = [b for b in self.model.buffers() if b.is_floating_point()]
        if not bufs:
            return
        if getattr(self, "_flat_buf", None) is None:
            n = sum(b.numel() for b in bufs)
            self._flat_buf = torch.empty(n, device=self.device, dtype=torch.float32)
            o = 0
            for b in bufs:
                k = b.numel()
                self._flat_buf[o:o + k].copy_(b.reshape(-1))
                b.data = self._flat_buf[o:o + k].view_as(b)  # buffers become views of one flat tensor (state_dict / modules see no change)
                o += k
        dist.broadcast(self._flat_buf, src=src, group=self.group)
