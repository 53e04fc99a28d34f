"""Data-parallel plumbing: one process per GPU, gradient buckets all-reduced over NCCL/NVLink (gloo in CPU tests).

Replaces the reference's single-process nn.DataParallel + replicate callback (sync_batchnorm/replicate.py:50-67,
train_generator.py:171-178): no parameter re-broadcast per forward, no scatter/gather, only a gradient all-reduce.
The hot path shards by samples, so the only exchange step is the gradient average (SURVEY.md §8e).

Two ways to drive it:
  * automatic (what the unchanged reference loops get): `GradBucketReducer.attach()` registers a post-accumulate-grad hook on
    every parameter.  When the last gradient of a bucket has been produced the bucket's all-reduce is launched
    asynchronously (it overlaps the rest of the backward pass); a callback queued on the autograd engine waits for the
    outstanding collectives when backward() returns, so `loss.backward(); optimizer.step()` (train_generator.py:314-322)
    is synchronised without any extra call.
  * explicit: `reduce()` after backward() — used inside CUDA-graph capture, where the bucket copies and the collectives are
    recorded on the capturing stream.
Gradients live in persistent flat buckets (p.grad becomes a view of its bucket: no torch.cat, no copy-back).
"""
import os

import torch
import torch.distributed as dist
import torch.nn as nn


def _world(group=None):
    if not (dist.is_available() and dist.is_initialized()):
        return 1
    return dist.get_world_size(group)


def broadcast_module_state(module, src=0, group=None):
    """Rank `src`'s parameters and buffers (BatchNorm running statistics, spectral-norm u/v) become everyone's: the
    replicas start identical, as nn.DataParallel's replicate() guarantees at every forward of the reference."""
    if _world(group) == 1:
        return 0
    n = 0
    with torch.no_grad():
        for t in list(module.parameters()) + list(module.buffers()):
            dist.broadcast(t.data, src=src, group=group)
            n += 1
    return n


def average_module_buffers(module, group=None):
    """Averages floating-point buffers (BatchNorm running_mean/var) over ranks and re-broadcasts the rest from rank 0 —
    call before saving a checkpoint so that the saved statistics describe the global batch, not rank 0's shard.  Not needed for a
    model whose BatchNorm layers are all SynchronizedBatchNorm2d: every rank updates them from the same global statistics."""
    w = _world(group)
    if w == 1:
        return
    with torch.no_grad():
        for b in module.buffers():
            if b.is_floating_point():
                dist.all_reduce(b.data, op=dist.ReduceOp.SUM, group=group)
                b.data.div_(w)
            else:
                dist.broadcast(b.data, src=0, group=group)


class GradBucketReducer:
    """Averages .grad of the given parameters across ranks in a few large flat buckets (default 64 MiB: on NVSwitch the
    cost is launch latency, not link count).  Buckets follow REVERSE registration order (the order gradients become
    ready).  Parameters that never receive a gradient (the reference's dead conv2.* branch, networks.py:131) are found on
    the first backward and skipped consistently on every rank (presence mask exchanged once)."""

    def __init__(self, params, bucket_bytes=64 << 20, group=None, wire_dtype=None):
        self.params = [p for p in params if p.requires_grad]
        self.bucket_bytes = bucket_bytes
        self.group = group
        env = os.environ.get("HRV_DDP_WIRE", "")
        self.wire_dtype = wire_dtype if wire_dtype is not None else (torch.bfloat16 if env == "bf16" else None)
        self._present = None
        self._buckets = None      # list of dicts: params, flat, views, pending
        self._slot = {}           # id(param) -> (bucket index, view)
        self._handles = []
        self._hooks = []
        self._callback_queued = False
        self.launched = 0         # collectives launched by the last backward (tests / bench read it)

    # ------------------------------------------------------------------ bucket construction
    def _build(self):
        world = _world(self.group)
        dev = self.params[0].device
        if self._present is None:
            mask = torch.tensor([1 if p.grad is not None else 0 for p in self.params], dtype=torch.int32, device=dev)
            if world > 1:
                dist.all_reduce(mask, op=dist.ReduceOp.MAX, group=self.group)
            self._present = mask.tolist()
        live = [p for p, has in zip(self.params, self._present) if has]
        groups, cur, cur_bytes = [], [], 0
        for p in reversed(live):
            nbytes = p.numel() * p.element_size()
            if cur and (cur_bytes + nbytes > self.bucket_bytes or p.dtype != cur[0].dtype):
                groups.append(cur)
                cur, cur_bytes = [], 0
            cur.append(p)
            cur_bytes += nbytes
        if cur:
            groups.append(cur)
        self._buckets = []
        for bi, ps in enumerate(groups):
            flat = torch.zeros(sum(p.numel() for p in ps), dtype=ps[0].dtype, device=dev)
            views, off = [], 0
            for p in ps:
                v = flat[off:off + p.numel()].view_as(p)
                views.append(v)
                self._slot[id(p)] = (bi, v)
                off += p.numel()
            wire = torch.empty_like(flat, dtype=self.wire_dtype) if (self.wire_dtype is not None and self.wire_dtype != flat.dtype) else None
            self._buckets.append({"params": ps, "flat": flat, "views": views, "wire": wire, "pending": len(ps)})

    def _adopt(self, p):
        """p.grad -> its bucket view (one device copy the first time after zero_grad(set_to_none=True); free afterwards)."""
        bi, v = self._slot[id(p)]
        g = p.grad
        if g is None:
            v.zero_()
        elif g.data_ptr() != v.data_ptr():
            v.copy_(g)
        p.grad = v
        return bi

    def _launch(self, bucket, async_op):
        world = _world(self.group)
        flat = bucket["flat"]
        buf = flat
        if bucket["wire"] is not None:
            bucket["wire"].copy_(flat)
            buf = bucket["wire"]
        backend = dist.get_backend(self.group)
        if backend == "nccl":
            h = dist.all_reduce(buf, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op)
            post = None
        else:  # gloo has no AVG
            h = dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group, async_op=async_op)
            post = world
        self.launched += 1
        return h, buf, post

    def _finish(self, bucket, buf, post):
        if post is not None:
            buf.div_(post)
        if buf is not bucket["flat"]:
            bucket["flat"].copy_(buf)

    # ------------------------------------------------------------------ explicit mode
    def reduce(self):
        """All-reduce every bucket now (after backward()).  Safe inside CUDA-graph capture once the communicator has been
        used outside of it.  Returns the number of buckets."""
        if _world(self.group) == 1 or not self.params:
            return 0
        if self._buckets is None:
            self._build()
        self.launched = 0
        for b in self._buckets:
            for p in b["params"]:
                self._adopt(p)
            _, buf, post = self._launch(b, async_op=False)
            self._finish(b, buf, post)
        return len(self._buckets)

    # ------------------------------------------------------------------ automatic mode (hooks)
    def attach(self):
        """Register the hooks; idempotent."""
        if self._hooks:
            return self
        for p in self.params:
            self._hooks.append(p.register_post_accumulate_grad_hook(self._on_grad))
        return self

    def detach(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []

    def _on_grad(self, p):
        if _world(self.group) == 1:
            return
        if not self._callback_queued:
            self._callback_queued = True
            self.launched = 0
            torch.autograd.Variable._execution_engine.queue_callback(self._finalize)
        if self._buckets is None:
            return  # first backward: the set of live parameters is not known yet -> everything happens in _finalize
        if id(p) not in self._slot:
            return
        bi = self._adopt(p)
        b = self._buckets[bi]
        b["pending"] -= 1
        if b["pending"] == 0:
            h, buf, post = self._launch(b, async_op=True)
            self._handles.append((h, b, buf, post))

    def _finalize(self):
        self._callback_queued = False
        if self._buckets is None:
            self.reduce()
            return
        done = set()
        for h, b, buf, post in self._handles:
            h.wait()  # NCCL: the current stream waits for the collective (no host block)
            self._finish(b, buf, post)
            done.add(id(b))
        self._handles = []
        for b in self._buckets:  # a bucket with parameters that got no gradient this time (unused branch): reduce it now
            if id(b) not in done and b["pending"] != len(b["params"]):
                for p in b["params"]:
                    self._adopt(p)
                _, buf, post = self._launch(b, async_op=False)
                self._finish(b, buf, post)
            b["pending"] = len(b["params"])


class DataParallelWithCallback(nn.Module):
    """Same name/constructor as sync_batchnorm.DataParallelWithCallback(module, device_ids=...) (train_generator.py:171-178).
    Under torchrun (WORLD_SIZE > 1, process group initialised — this wrapper initialises it from the environment if the
    script did not) it is a DDP-style wrapper: parameters/buffers are broadcast from rank 0 when wrapping, and gradients are
    averaged automatically during backward() (hooks).  With one process it is a transparent pass-through.  Modules without
    trainable parameters (the reference also wraps its loss modules) are passed through."""

    def __init__(self, module, device_ids=None, output_device=None, dim=0):
        super().__init__()
        self.module = module
        self.device_ids = device_ids
        self._reducer = None
        world_env = int(os.environ.get("WORLD_SIZE", "1"))
        if world_env > 1 and dist.is_available() and not dist.is_initialized():
            first = next(module.parameters(), None)
            backend = "nccl" if (first is None or first.is_cuda) and torch.cuda.is_available() else "gloo"
            dist.init_process_group(backend)
        if _world() > 1:
            params = [p for p in module.parameters() if p.requires_grad]
            broadcast_module_state(module)
            if params:
                self._reducer = GradBucketReducer(params).attach()
            if any(isinstance(m, SynchronizedBatchNorm2d) for m in module.modules()):
                syncbn_group()  # made here, at the same point on every rank (new_group is collective)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def reduce_gradients(self):
        """Explicit reduction (kept for callers that used it); a no-op when the hooks already did the work."""
        if self._reducer is None or self._reducer._hooks:
            return 0
        return self._reducer.reduce()


# ------------------------------------------------------------------------------------------------ synchronised BatchNorm

_SYNCBN_GROUP = [None, None]  # (default process group it was made from, the SyncBN group)


def syncbn_group():
    """The process group of SynchronizedBatchNorm2d's collectives, or None with one process (the layers then run the per-rank
    path, which is the same computation).  Same ranks as the default group but its own communicator: the gradient buckets are
    all-reduced asynchronously from hooks while backward() runs, and the statistics exchange must not queue behind them or depend
    on how the two interleave.  Made on first use; new_group is collective, so every rank reaches that point together."""
    if _world() == 1:
        return None
    default = dist.distributed_c10d._get_default_group()
    if _SYNCBN_GROUP[0] is not default:
        _SYNCBN_GROUP[1] = dist.new_group(ranks=list(range(dist.get_world_size())), backend=dist.get_backend())
        _SYNCBN_GROUP[0] = default
    return _SYNCBN_GROUP[1]


def syncbn_all_reduce(buf, group):
    """In-place sum of a SyncBN wire buffer (fp64, on the GPU) over `group`, ordered on the current stream.  NCCL reduces it on the
    device (and can be captured in a CUDA graph); gloo reduces in host memory, so the buffer is staged there."""
    if dist.get_backend(group) == "gloo":
        host = buf.cpu()
        dist.all_reduce(host, op=dist.ReduceOp.SUM, group=group)
        buf.copy_(host)
    else:
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)


class SynchronizedBatchNorm2d(nn.BatchNorm2d):
    """sync_batchnorm.SynchronizedBatchNorm2d: BatchNorm2d whose train-mode statistics cover the batch of every data-parallel rank.
    Same constructor defaults and state_dict as nn.BatchNorm2d, so checkpoints load either way.  Inside ConditionGenerator /
    ResBlock training each layer exchanges one fp64 buffer of per-channel sums per direction (hrviton_b200.autograd_tocg); with one
    process it runs exactly the nn.BatchNorm2d path.  Eval mode uses the running statistics (folded into the convolution).  The
    affine gradients stay per rank: the gradient average over ranks then equals torch.nn.SyncBatchNorm's."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True):
        super().__init__(num_features, eps=eps, momentum=momentum, affine=affine)

    def forward(self, input):
        if self.training and _world() > 1:
            raise NotImplementedError("a standalone SynchronizedBatchNorm2d has no synchronised kernel path: its statistics are exchanged "
                                      "inside ConditionGenerator / ResBlock training")
        return super().forward(input)


class SynchronizedBatchNorm1d(nn.BatchNorm1d):
    """Import parity with the reference's sync_batchnorm: no model here has 1-D BatchNorm, so using it raises."""

    def forward(self, input):
        raise NotImplementedError("SynchronizedBatchNorm1d is not implemented (only SynchronizedBatchNorm2d is)")


class SynchronizedBatchNorm3d(nn.BatchNorm3d):
    """Import parity with the reference's sync_batchnorm: no model here has 3-D BatchNorm, so using it raises."""

    def forward(self, input):
        raise NotImplementedError("SynchronizedBatchNorm3d is not implemented (only SynchronizedBatchNorm2d is)")


def convert_model(module):
    """sync_batchnorm.convert_model for 2-D BatchNorm: returns `module` with every nn.BatchNorm2d replaced by a SynchronizedBatchNorm2d
    that keeps its running statistics (the same buffers), affine parameters (copies) and train/eval mode.  A module wrapped in
    nn.DataParallel or DataParallelWithCallback comes back wrapped in a new DataParallelWithCallback (the old wrapper's gradient hooks
    are removed: they belong to parameters that have been replaced)."""
    if isinstance(module, (nn.DataParallel, DataParallelWithCallback)):
        if isinstance(module, DataParallelWithCallback) and module._reducer is not None:
            module._reducer.detach()
        return DataParallelWithCallback(convert_model(module.module), device_ids=module.device_ids)
    mod = module
    if isinstance(module, nn.BatchNorm2d) and not isinstance(module, SynchronizedBatchNorm2d):
        mod = SynchronizedBatchNorm2d(module.num_features, module.eps, module.momentum, module.affine)
        mod.running_mean = module.running_mean
        mod.running_var = module.running_var
        mod.num_batches_tracked = module.num_batches_tracked
        if module.affine:
            mod.weight = nn.Parameter(module.weight.detach().clone(), requires_grad=module.weight.requires_grad)
            mod.bias = nn.Parameter(module.bias.detach().clone(), requires_grad=module.bias.requires_grad)
        mod.train(module.training)
    for name, child in module.named_children():
        mod.add_module(name, convert_model(child))
    return mod
