"""View-sharded multi-GPU plumbing (SURVEY.md section 8e): one process per GPU, `torch.distributed` (NCCL on the GPUs, gloo in
the CPU tests).  The path partitions by view — given the decoded Gaussians of a frame, project/bin/sort/blend of
different views are independent — so the only exchange steps are a broadcast of the decoded table from the frame
owner and a sum-reduction of its gradient.  The reference is single-GPU only (SURVEY.md section 2.4): nothing to match.

`FrameExchange` is the product API for those two steps: both run on a communication stream, double-buffered, so
that the broadcast of frame i+1 and the reduction of frame i's gradient overlap the render of the neighbouring
frames; only the frame OWNER touches its source (decoder output or a pinned host buffer) — the other ranks receive
the table over NVLink and never read theirs."""
from typing import List, Optional

import torch
import torch.distributed as dist


def views_of_rank(rank: int, world: int, n_views: int) -> List[int]:
    """Round-robin view partition: rank r renders views {v : v mod world == r}."""
    return list(range(rank, n_views, world))


def _active() -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def owner_broadcast(decoded: torch.Tensor, src: int = 0) -> torch.Tensor:
    """Broadcast the packed decoded-Gaussian table of a frame from its owner (in place; returns the tensor)."""
    if _active():
        dist.broadcast(decoded, src=src)
    return decoded


def reduce_grads(grad: torch.Tensor) -> torch.Tensor:
    """Sum dL/d(decoded table) over the ranks (each rank contributes its views); in place."""
    if _active():
        dist.all_reduce(grad, op=dist.ReduceOp.SUM)
    return grad


class FrameExchange:
    """Double-buffered exchange of one flat fp32 table per frame between the frame owner and the view shards.

        ex = FrameExchange(numel, device, owner=0)
        ex.post_input(0, source)                  # owner: source = decoder output or pinned host table; others: None
        for i in range(n):
            ex.take_input(i, static_in)           # main stream waits for frame i's table, copies it into the step's input
            if i + 1 < n: ex.post_input(i + 1, source)
            ... render forward + backward on the main stream, producing `grad` ...
            ex.post_grad(i, grad)                 # all-reduce of frame i's gradient on the communication stream
        ex.finish()                               # main stream waits for the last reduction
        ex.grad(i)                                # the reduced gradient of frame i (valid until frame i+2 is posted)

    On CPU (gloo, the unit tests) the streams degenerate to synchronous calls with the same ordering."""

    def __init__(self, numel: int, device, owner: int = 0, dtype=torch.float32):
        self.device = torch.device(device)
        self.owner = owner
        self.cuda = self.device.type == "cuda"
        self.rank = dist.get_rank() if _active() else 0
        self.world = dist.get_world_size() if _active() else 1
        self.inputs = [torch.empty(numel, dtype=dtype, device=self.device) for _ in range(2)]
        self.grads = [torch.empty(numel, dtype=dtype, device=self.device) for _ in range(2)]
        if self.cuda:
            self.comm = torch.cuda.Stream(device=self.device)
            self.h2d = torch.cuda.Stream(device=self.device)  # owner: host table -> device, beside the collectives
            ev = lambda: [torch.cuda.Event() for _ in range(2)]
            self.in_ready, self.in_free, self.g_ready, self.g_free = ev(), ev(), ev(), ev()
            self.h2d_done = ev()
        self.bytes_h2d = 0  # host bytes this rank copied in (owner only)

    def post_input(self, i: int, source: Optional[torch.Tensor], ready: Optional["torch.cuda.Event"] = None):
        """`ready`: event after which a device-resident `source` (the decoder output of frame i) may be read."""
        k = i & 1
        is_owner = self.rank == self.owner
        if is_owner and source is None:
            raise RuntimeError("the frame owner must provide the decoded table")
        if not self.cuda:
            if is_owner:
                self.bytes_h2d += source.numel() * source.element_size()
                self.inputs[k].copy_(source)
            owner_broadcast(self.inputs[k], self.owner)
            return
        if is_owner and source.device.type != "cuda":
            # a host table goes in on its own stream: the 22.8 MB PCIe copy of frame i+1 then runs beside the previous
            # frame's collectives instead of in front of them on the communication stream
            self.bytes_h2d += source.numel() * source.element_size()
            with torch.cuda.stream(self.h2d):
                if i >= 2:
                    self.h2d.wait_event(self.in_free[k])
                self.inputs[k].copy_(source, non_blocking=True)
                self.h2d_done[k].record(self.h2d)
        with torch.cuda.stream(self.comm):
            if i >= 2:
                self.comm.wait_event(self.in_free[k])
            if is_owner:  # only the owner reads its source; non-owners receive over NVLink
                if source.device.type != "cuda":
                    self.comm.wait_event(self.h2d_done[k])
                else:
                    if ready is not None:
                        self.comm.wait_event(ready)
                    self.inputs[k].copy_(source, non_blocking=True)
            owner_broadcast(self.inputs[k], self.owner)
            self.in_ready[k].record(self.comm)

    def take_input(self, i: int, dst: torch.Tensor):
        k = i & 1
        if not self.cuda:
            dst.copy_(self.inputs[k])
            return
        main = torch.cuda.current_stream(self.device)
        main.wait_event(self.in_ready[k])
        dst.copy_(self.inputs[k], non_blocking=True)
        self.in_free[k].record(main)

    def post_grad(self, i: int, grad: torch.Tensor):
        k = i & 1
        if not self.cuda:
            self.grads[k].copy_(grad)
            reduce_grads(self.grads[k])
            return
        main = torch.cuda.current_stream(self.device)
        if i >= 2:
            main.wait_event(self.g_free[k])
        self.grads[k].copy_(grad, non_blocking=True)
        self.g_ready[k].record(main)
        with torch.cuda.stream(self.comm):
            self.comm.wait_event(self.g_ready[k])
            reduce_grads(self.grads[k])
            self.g_free[k].record(self.comm)

    def grad(self, i: int) -> torch.Tensor:
        return self.grads[i & 1]

    # ---- zero-copy variant: the step reads inputs[i & 1] and writes its gradient into grads[i & 1] directly (one
    # captured graph per buffer parity), so neither table is copied on the device:
    #     ex.post_input(0, source)
    #     for i in range(n):
    #         ex.wait_input(i)                      # main stream: frame i's table has arrived in ex.inputs[i & 1]
    #         if i + 1 < n: ex.post_input(i + 1, source)
    #         ... step reading ex.inputs[i & 1], writing ex.grads[i & 1] ...
    #         ex.release_input(i)
    #         ex.post_grad_inplace(i)               # all-reduce of ex.grads[i & 1] on the communication stream
    #     ex.finish()
    def wait_input(self, i: int):
        """Main stream waits for frame i's table in inputs[i & 1] and for the reduction that last used grads[i & 1]."""
        if not self.cuda:
            return
        k = i & 1
        main = torch.cuda.current_stream(self.device)
        main.wait_event(self.in_ready[k])
        if i >= 2:
            main.wait_event(self.g_free[k])

    def release_input(self, i: int):
        if self.cuda:
            self.in_free[i & 1].record(torch.cuda.current_stream(self.device))

    def post_grad_inplace(self, i: int):
        k = i & 1
        if not self.cuda:
            reduce_grads(self.grads[k])
            return
        main = torch.cuda.current_stream(self.device)
        self.g_ready[k].record(main)
        with torch.cuda.stream(self.comm):
            self.comm.wait_event(self.g_ready[k])
            reduce_grads(self.grads[k])
            self.g_free[k].record(self.comm)

    def finish(self):
        if self.cuda:
            torch.cuda.current_stream(self.device).wait_stream(self.comm)
            torch.cuda.current_stream(self.device).wait_stream(self.h2d)
