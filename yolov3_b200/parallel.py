"""Data-parallel gradient exchange — the ONE collective on the path (SURVEY §8e, row a19).

The reference wraps the model in ``DistributedDataParallel`` (utils/torch_utils.py:60-72, train.py:323): one process
per GPU, each rank runs forward/backward on its shard, gradients are averaged with a bucketed NCCL all-reduce, and
``loss *= WORLD_SIZE`` (train.py:405-406) undoes the averaging because the loss is already scaled by the rank batch size.
Here every gradient lives in ONE flat fp32 buffer laid out in backward-completion order (``params.ParamStore``), and the
backward pass is cut into a few segments: ``DDP(model)`` makes ``TrainEngine.backward`` launch an NCCL all-reduce of a
segment's contiguous gradient range on a side stream as soon as that segment is enqueued, so the exchange of the deep layers
(90 % of the 248 MB) runs under the back-propagation of the shallow ones and only the last, small range is exposed.  No
packing / unpacking copies: NCCL reads and writes the gradient buffer in place, and the 1/world_size of the mean is folded
into the fused optimizer update (``optim.SGD``) or applied by ``DDP.finish()``.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def scale_loss(loss: torch.Tensor) -> torch.Tensor:
    """train.py:405-406: ``loss *= WORLD_SIZE`` (gradients are averaged between ranks afterwards)."""
    return loss * world_size()


def allreduce_gradients(params, average: bool = True, flat: torch.Tensor | None = None) -> torch.Tensor | None:
    """All-reduce (mean) the ``.grad`` of ``params`` across ranks in ONE flat buffer.  Returns the flat buffer so the
    caller can keep it alive / reuse it.  No-op for a single process."""
    ps = [p for p in params if p.grad is not None]
    w = world_size()
    if w == 1 or not ps:
        return flat
    n = sum(p.grad.numel() for p in ps)
    if flat is None or flat.numel() != n or flat.device != ps[0].grad.device:
        flat = torch.empty(n, dtype=torch.float32, device=ps[0].grad.device)
    off = 0
    for p in ps:
        k = p.grad.numel()
        flat[off:off + k].copy_(p.grad.reshape(-1))
        off += k
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    if average:
        flat.div_(w)
    off = 0
    for p in ps:
        k = p.grad.numel()
        p.grad.copy_(flat[off:off + k].view_as(p.grad))
        off += k
    return flat


class DDP:
    """``smart_DDP(model)`` (utils/torch_utils.py:60-72) for the GPU ``Model``: marks the model so that its training engine
    overlaps the bucketed gradient all-reduce with the backward pass, and broadcasts rank 0's parameters like DDP's
    constructor does (train.py:323).  ``forward`` / attribute access go to the wrapped model (``de_parallel`` not needed).

    ``no_sync()``: gradient accumulation without exchange, as torch's DDP.no_sync (the exchange must then happen on the last
    backward of the accumulation window, where the whole accumulated buffer is reduced)."""

    def __init__(self, model, broadcast=True):
        self.module = model
        self.world = world_size()
        self.require_sync = True
        self.pending_average = False  # True: the gradient buffer holds sums over ranks that still need the 1/world
        model.ddp = self
        if broadcast and self.world > 1:
            dist.broadcast(model.store().P, 0)  # one flat buffer: parameters AND BatchNorm buffers, like DDP's constructor

    def __call__(self, *a, **k):
        return self.module(*a, **k)

    def __getattr__(self, name):
        return getattr(self.__dict__["module"], name)

    def no_sync(self):
        ddp = self

        class _Ctx:
            def __enter__(self):
                ddp.require_sync = False

            def __exit__(self, *exc):
                ddp.require_sync = True

        return _Ctx()

    def finish(self):
        """For optimizers other than ``optim.SGD`` (which averages inside its update): turn the summed gradients into the mean."""
        if self.pending_average:
            self.module.store().G.div_(self.world)
            self.pending_average = False


def broadcast_parameters(params, src: int = 0):
    """DDP's constructor broadcast: every rank starts from rank ``src``'s parameters (train.py:323)."""
    if world_size() == 1:
        return
    for p in params:
        dist.broadcast(p.data, src)


def convert_sync_batchnorm(model):
    """``torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)`` of the reference's ``--sync-bn`` switch (train.py:270-272):
    the training engine all-reduces every BatchNorm's (sum, sum of squares) in the forward and (sum dz, sum dz*xhat) in the
    backward, so batch statistics cover all ranks' images.  gamma/beta gradients stay rank-local sums (the gradient
    all-reduce averages them like every other parameter), exactly as torch's SyncBatchNorm does under DDP."""
    model.sync_bn = True
    model._train_engines.clear()
    return model
