"""Step loop mirror of /root/reference/unet3d/train/training_utils.py:20-112 (epoch_training / batch_loss /
_batch_loss), kept call-compatible so the reference's ``run_training`` can drive it, minus the per-step
``torch.cuda.empty_cache()`` (training_utils.py:46-47) and with non-blocking pinned H2D copies
(training_utils.py:89-91 copies synchronously from pageable memory).
"""
from __future__ import annotations

import time

import torch


class AverageMeter(object):
    """training_utils.py:156-178."""

    def __init__(self, name, fmt=":f"):
        self.name, self.fmt = name, fmt
        self.reset()

    def reset(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count

    def __str__(self):
        return ("{name} {val" + self.fmt + "} ({avg" + self.fmt + "})").format(**self.__dict__)


def _to_device(t: torch.Tensor) -> torch.Tensor:
    if t.is_cuda:
        return t
    return t.cuda(non_blocking=t.is_pinned())


def _batch_loss(model, images, target, criterion, inferer=None):
    """training_utils.py:101-112."""
    if inferer is not None:
        output = inferer(images, model).to(images.device)
    else:
        output = model(images)
    batch_size = images.size(0)
    loss = criterion(output, target)
    return loss, batch_size


def batch_loss(model, images, target, criterion, n_gpus=0, use_amp=None, inferer=None):
    """training_utils.py:88-98.  ``use_amp`` selects nothing here: precision is a model property."""
    if n_gpus is not None:
        images = _to_device(images)
        target = _to_device(target)
    return _batch_loss(model, images, target, criterion, inferer=inferer)


class GraphedTrainStep:
    """One training step -- forward, criterion, backward [, grad_sync], optimizer.step -- with the forward+loss+backward
    part captured ONCE as a CUDA graph and replayed (training_utils.py:59-72 is what it replaces; shapes are static and
    the plan is a fixed kernel list, so ~180 launches per step collapse into one graph launch).

    ``step(images, target)`` accepts host (pinned or pageable) or device tensors: they are copied straight into the
    graph's static input buffers (H2D lands in place, no staging copy) and the returned loss is the graph's static
    0-dim tensor (read it with ``.item()`` when needed).  The model runs in flat-gradient mode: every replay overwrites
    the ``.grad`` views of one persistent bucket, which ``grad_sync`` all-reduces in place.
    """

    def __init__(self, model, criterion, optimizer, images_shape, target_shape, target_dtype=torch.uint8, device=None,
                 grad_sync=None, warmup: int = 2, capture_error_mode: str = "global"):
        self.model, self.criterion, self.optimizer, self.grad_sync = model, criterion, optimizer, grad_sync
        self.graph_tail = None      # always None: bench.py reads it to report whether the exchange ran overlapped
        device = device or next(model.parameters()).device
        self.images = torch.zeros(tuple(images_shape), dtype=torch.float32, device=device)
        self.target = torch.zeros(tuple(target_shape), dtype=target_dtype, device=device)
        self.graph = None
        self.loss = None
        self.warmup = int(warmup)
        self.device = device
        # "global" (torch's default).  Observed with torch 2.11 (tools/graph_debug.py): "global" and "relaxed" capture the
        # step, "thread_local" does not -- autograd runs the backward of the step on its device worker thread, which may not
        # enqueue into a stream another thread is capturing in thread-local mode
        self.capture_error_mode = capture_error_mode

    def _capture(self):
        model = self.model
        model.train()
        model.use_flat_gradients(True)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(self.warmup):            # plan creation, workspace, table uploads, bucket: outside the capture
                self.optimizer.zero_grad(set_to_none=True)
                loss = self.criterion(model(self.images), self.target)
                loss.backward()
                # No autograd graph of the warm-up may outlive this line.  While one is alive it keeps the parameters'
                # AccumulateGrad nodes alive, and those remember the stream they were created on (this side stream); the
                # captured backward would reuse them, autograd would synchronise the capturing stream with that
                # non-capturing one, and the capture ends as cudaErrorStreamCaptureInvalidated (observed with
                # torch 2.11 and tools/graph_debug2.py: 'replica' fails, 'del_loss' captures).
                del loss
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        model._overwrite_grads = True
        self.graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(self.graph, capture_error_mode=self.capture_error_mode):
                self.loss = self.criterion(model(self.images), self.target)
                self.loss.backward()
        except Exception as e:
            self.graph = None
            self.loss = None
            raise RuntimeError(
                "GraphedTrainStep: CUDA-graph capture of the training step failed (%s).  A loss (or any tensor with a grad_fn) of "
                "an earlier eager step of this model that is still referenced makes autograd synchronise the capturing stream "
                "with the stream of that step: drop those references before the first graphed step." % (e,)) from e

    def step(self, images, target):
        if self.graph is None:
            self.images.copy_(images, non_blocking=True)
            self.target.copy_(target, non_blocking=True)
            self._capture()
        self.images.copy_(images, non_blocking=True)
        self.target.copy_(target, non_blocking=True)
        self.graph.replay()
        params = self.model.ordered_parameters()
        if params[0].grad is None:          # somebody ran zero_grad(set_to_none=True) since: re-bind the bucket views
            for p, v in zip(params, self.model._grad_views):
                if p.requires_grad:
                    p.grad = v
        if self.grad_sync is not None:
            self.grad_sync()
        self.optimizer.step()
        return self.loss

    __call__ = step

    def matches(self, images, target) -> bool:
        return tuple(images.shape) == tuple(self.images.shape) and tuple(target.shape) == tuple(self.target.shape)


class DevicePrefetcher:
    """Iterates a loader of ``{"image", "label"}`` items one batch ahead: the next batch's host->device copies run on a
    side stream while the current step computes (the reference copies synchronously from pageable memory on the compute
    stream: training_utils.py:89-91).  Pageable tensors still work, they just do not overlap.  ``transform`` (optional, e.g.
    an ``augment.Compose``) runs on each staged batch on the same side stream, after its copies."""

    _streams = {}    # one copy stream per device, kept across epochs (stream creation is not free)

    def __init__(self, loader, device, transform=None):
        self.loader, self.device, self.transform = loader, device, transform
        key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
        if key not in DevicePrefetcher._streams:
            DevicePrefetcher._streams[key] = torch.cuda.Stream(device=device)
        self.stream = DevicePrefetcher._streams[key]

    def __len__(self):
        return len(self.loader)

    def _stage(self, item):
        with torch.cuda.stream(self.stream):
            out = dict(item)
            for k in ("image", "label"):
                t = item[k]
                out[k] = t if t.is_cuda else t.to(self.device, non_blocking=True)
            if self.transform is not None:
                out = self.transform(out)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return out, ev

    def __iter__(self):
        it = iter(self.loader)
        try:
            nxt = self._stage(next(it))
        except StopIteration:
            return
        while nxt is not None:
            cur, ev = nxt
            try:
                nxt = self._stage(next(it))
            except StopIteration:
                nxt = None
            main = torch.cuda.current_stream(self.device)
            main.wait_event(ev)
            for k in ("image", "label"):
                cur[k].record_stream(main)
            yield cur


class _LaggedLoss:
    """Reads step i's loss while step i+1 is already queued: an async D2H into pinned memory + an event per step
    instead of ``loss.item()`` right after the launch (training_utils.py:63), which would drain the GPU every step."""

    _pinned = None   # the two pinned read-back slots and their events are process-wide: cudaHostAlloc per epoch is not free

    def __init__(self):
        if _LaggedLoss._pinned is None:
            _LaggedLoss._pinned = ([torch.zeros((), dtype=torch.float32).pin_memory() for _ in range(2)],
                                   [torch.cuda.Event(), torch.cuda.Event()])
        self.slots, self.events = _LaggedLoss._pinned
        self.pending = []   # (slot, batch_size)
        self.i = 0

    def push(self, loss, batch_size):
        k = self.i % 2
        self.i += 1
        self.slots[k].copy_(loss.detach(), non_blocking=True)
        self.events[k].record()
        self.pending.append((k, batch_size))

    def pop_ready(self, keep: int):
        out = []
        while len(self.pending) > keep:
            k, bs = self.pending.pop(0)
            self.events[k].synchronize()
            out.append((float(self.slots[k]), bs))
        return out


def _graphed_step_for(model, criterion, optimizer, images, target, grad_sync):
    cache = model.__dict__.setdefault("_graphed_steps", {})
    key = (tuple(images.shape), tuple(target.shape), target.dtype, id(criterion), id(optimizer), id(grad_sync))
    step = cache.get(key)
    if step is None:
        step = cache[key] = GraphedTrainStep(model, criterion, optimizer, images.shape, target.shape,
                                             target_dtype=target.dtype, grad_sync=grad_sync)
    return step


def epoch_training(train_loader, model, criterion, optimizer, epoch, n_gpus=None, print_frequency=1,
                   print_gpu_memory=False, scaler=None, samples_per_epoch=None, iteration=1, grad_sync=None,
                   use_cuda_graph=False, device_transform=None):
    """training_utils.py:20-85.  ``grad_sync`` (optional callable) runs between backward and optimizer.step:
    the data-parallel gradient all-reduce of ``parallel.GradAllReduce``.  ``use_cuda_graph``: replay the step through
    ``GraphedTrainStep`` (kept on the model across epochs) for every batch of the first batch's shape; other shapes,
    e.g. a short last batch, run eagerly.  On a GPU the loader is read one batch ahead (``DevicePrefetcher``) and the
    loss of step i is read back while step i+1 runs, so the only host syncs are one step behind the queue.
    ``device_transform`` (optional, e.g. the ``Compose`` of ``augment.build_device_transform``) runs on every staged training
    batch on the prefetcher's copy stream, overlapping the running step; it keeps each batch's shapes and dtypes."""
    graphed = None
    batch_time = AverageMeter("Time", ":6.3f")
    data_time = AverageMeter("Data", ":6.3f")
    losses = AverageMeter("Loss", ":.4e")
    model.train()
    on_gpu = n_gpus is not None and torch.cuda.is_available() and next(model.parameters()).is_cuda
    if device_transform is not None and not on_gpu:
        raise RuntimeError("epoch_training: device_transform needs the model on a CUDA device and n_gpus set")
    loader = DevicePrefetcher(train_loader, next(model.parameters()).device, device_transform) if on_gpu else train_loader
    lag = _LaggedLoss() if on_gpu else None
    end = time.time()
    batch_size = 0
    for i, item in enumerate(loader):
        images, target = item["image"], item["label"]
        data_time.update(time.time() - end)
        if use_cuda_graph and graphed is None:
            graphed = _graphed_step_for(model, criterion, optimizer, images, target, grad_sync)
        if graphed is not None and graphed.matches(images, target):
            loss, batch_size = graphed(images, target), images.size(0)
        else:
            optimizer.zero_grad()            # (in flat-gradient mode the eager backward re-binds the same bucket views)
            loss, batch_size = batch_loss(model, images, target, criterion, n_gpus=n_gpus, use_amp=scaler is not None)
            loss.backward()
            if grad_sync is not None:
                grad_sync()
            optimizer.step()
        if lag is not None:
            lag.push(loss, batch_size)
            for v, bs in lag.pop_ready(keep=1):
                losses.update(v, bs)
        else:
            losses.update(loss.item(), batch_size)
        del loss
        batch_time.update(time.time() - end)
        end = time.time()
        if print_frequency and i % print_frequency == 0:
            print("Epoch: [{}][{}/{}]\t{}\t{}\t{}".format(epoch, i + 1, len(train_loader), batch_time, data_time, losses))
        if samples_per_epoch and (i + 1) * batch_size >= samples_per_epoch:
            break
    if lag is not None:
        for v, bs in lag.pop_ready(keep=0):
            losses.update(v, bs)
    return losses.avg


def epoch_validation(val_loader, model, criterion, n_gpus, print_freq=1, use_amp=False, inferer=None):
    """training_utils.py:115-147."""
    losses = AverageMeter("Loss", ":.4e")
    model.eval()
    with torch.no_grad():
        for i, item in enumerate(val_loader):
            loss, batch_size = batch_loss(model, item["image"], item["label"], criterion, n_gpus=n_gpus, inferer=inferer)
            losses.update(loss.item(), batch_size)
    return losses.avg
