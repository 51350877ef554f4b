"""Host-buffer entry point of the hot path: what a caller holding HOST (pinned) arrays uses.

`ViewAttentionHostPlan` owns the device staging buffers for one problem shape and runs, per
call, H2D of every input -> fused forward -> fused backward -> D2H of every result, all on one
CUDA stream through the C ABI.  bench.py times this call for its `e2e` number (host<->device
copies inside the timed region).  Operator semantics are those of ops.view_attention
(modules.py:518 + pooling.py:285-300).

`ViewAttentionHostPipeline` keeps `depth` plans on `depth` CUDA streams: consecutive steps go to
alternating slots, so step k+1's H2D copies run on the copy-in engine while step k computes and
streams its results out on the copy-out engine (PCIe is full duplex; a single stream uses one
direction at a time).  Every step still moves all of its inputs and results.
"""
import torch

from . import _lib
from ._lib import launch


class ViewAttentionHostPlan:
    def __init__(self, N, V, R, C, G, dtype=torch.float32, idx_dtype=torch.int32, gating=True,
                 group_scaling=True, eps=1e-12, device="cuda"):
        self.N, self.V, self.R, self.C, self.G = N, V, R, C, G
        self.dtype, self.group_scaling, self.eps, self.gating = dtype, group_scaling, eps, gating
        d = torch.device(device)
        self.device = d
        e = lambda shape, dt: torch.empty(shape, dtype=dt, device=d)  # noqa: E731
        self.x = e((R, C), dtype)
        self.idx = e((V,), idx_dtype) if idx_dtype is not None else None
        self.compat = e((V, G), torch.float32)
        self.ptr = e((N + 1,), torch.int64)
        self.gout = e((N, C), dtype)
        self.gate = e((2, G), torch.float32) if gating else None      # [w; b]
        self.out = e((N, C), dtype)
        self.seg_max = e((N, G), torch.float32)
        self.seg_den = e((N, G), torch.float32)
        self.seg_arg = e((N, G), torch.int32)
        self.gx = e((V, C), dtype)
        self.gcompat = e((V, G), torch.float32)
        self.ggate = e((2, G), torch.float32) if gating else None
        # gate-gradient partials and the lane kernel's range queue
        self.ws = _lib.workspace(_lib.load().dva_view_attention_bwd_workspace_bytes(G), d)
        self.dcode = _lib.DTYPE_CODES[dtype]

    # -- device-resident pieces (bench.py's `value` times exactly these two calls) ---------------
    def forward_device(self, save_att=None):
        gw = self.gate[0] if self.gating else None
        gb = self.gate[1] if self.gating else None
        launch("dva_view_attention_fwd", self.device, self.x, self.idx,
               int(self.idx is not None and self.idx.dtype == torch.int64), self.compat, self.ptr, gw, gb, self.out,
               save_att, self.seg_max, self.seg_den, self.seg_arg, self.N, self.V, self.R, self.C, self.G,
               int(self.group_scaling), float(self.eps), self.dcode)

    def backward_device(self):
        gw = self.gate[0] if self.gating else None
        gb = self.gate[1] if self.gating else None
        launch("dva_view_attention_bwd", self.device, self.x, self.idx,
               int(self.idx is not None and self.idx.dtype == torch.int64), self.compat, self.ptr, gw, gb, self.gout,
               self.seg_max, self.seg_den, self.seg_arg, self.gx, self.gcompat, self.ggate, 0, self.N, self.V,
               self.R, self.C, self.G, int(self.group_scaling), self.dcode, self.ws, self.ws.numel())

    # -- host-buffer call ---------------------------------------------------------------------------
    def host_buffers(self, pin=True):
        """Allocate the pinned host arrays a caller would own: (inputs dict, outputs dict)."""
        def h(t):
            return torch.empty(t.shape, dtype=t.dtype, pin_memory=pin)
        ins = dict(x=h(self.x), compat=h(self.compat), ptr=h(self.ptr), gout=h(self.gout))
        if self.idx is not None:
            ins["idx"] = h(self.idx)
        if self.gating:
            ins["gate"] = h(self.gate)
        outs = dict(out=h(self.out), gx=h(self.gx), gcompat=h(self.gcompat))
        if self.gating:
            outs["ggate"] = h(self.ggate)
        return ins, outs

    def run_host(self, ins, outs):
        """H2D(all inputs) -> fwd -> bwd -> D2H(all results), asynchronously on the current stream.
        Returns (h2d_bytes, d2h_bytes)."""
        h2d = d2h = 0
        for k, host in ins.items():
            getattr(self, k).copy_(host, non_blocking=True)
            h2d += host.numel() * host.element_size()
        self.forward_device()
        self.backward_device()
        for k, host in outs.items():
            host.copy_(getattr(self, k), non_blocking=True)
            d2h += host.numel() * host.element_size()
        return h2d, d2h


class ViewAttentionHostPipeline:
    """`depth` independent ViewAttentionHostPlan slots, one CUDA stream each.

        pipe = ViewAttentionHostPipeline(2, N, V, R, C, G, ...)
        for step in steps:
            ev = pipe.submit(ins[step], outs[step % pipe.depth])   # returns at once
        pipe.drain()                                               # all results are in `outs`

    Results of a step are valid once its event completed; a slot's `outs` must not be reused
    by the caller before that.  Slot reuse on the device is ordered by the slot's stream."""

    def __init__(self, depth, *plan_args, first_plan=None, **plan_kwargs):
        assert depth >= 1
        self.depth = depth
        self.plans = [first_plan if (k == 0 and first_plan is not None)
                      else ViewAttentionHostPlan(*plan_args, **plan_kwargs) for k in range(depth)]
        dev = self.plans[0].device
        self.streams = [torch.cuda.Stream(device=dev) for _ in range(depth)]
        self._next = 0

    def submit(self, ins, outs, after_step=None):
        """Enqueue one full step (H2D, fwd, bwd, D2H) on the next slot; `after_step(plan)` runs on
        the slot's stream after the kernels (e.g. the gradient all-reduce).  Returns
        (event, h2d_bytes, d2h_bytes)."""
        k = self._next
        self._next = (k + 1) % self.depth
        plan, stream = self.plans[k], self.streams[k]
        stream.wait_stream(torch.cuda.current_stream(plan.device))
        with torch.cuda.stream(stream):
            h2d, d2h = plan.run_host(ins, outs)
            if after_step is not None:
                after_step(plan)
            ev = torch.cuda.Event()
            ev.record(stream)
        return ev, h2d, d2h

    def drain(self):
        cur = torch.cuda.current_stream(self.plans[0].device)
        for s in self.streams:
            cur.wait_stream(s)
