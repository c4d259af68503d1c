"""Host-side mirror of the reference's model interface for the U-Net path.

Mirrors (paths relative to /root/reference):
  * ``unet3d/models/pytorch/segmentation/unet.py:47-70``  UNet3D / AutocastUNet / AutoImplantUNet
  * ``unet3d/models/pytorch/autoencoder/variational.py:37-87`` ctor kwargs + forward contract
  * ``unet3d/models/build.py:9-64``  fetch_model_by_name / build_or_load_model / load_state_dict

The module keeps canonical fp32 parameters under the reference's state-dict keys (so reference checkpoints load and
checkpoints written here load into the reference), and runs forward/backward as ONE call each into libb200unet's
whole-network plan (hand-written sm_90a kernels).  There is no PyTorch-op fallback: on a non-CUDA tensor, or if
the library is missing, ``forward`` raises.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Dict, Optional, Sequence, Tuple

import torch
from torch import nn

from . import lib as _lib

_ACT = {None: 0, "sigmoid": 1, "softmax": 2}


class _Node(nn.Module):
    """Plain container used to reproduce the reference's dotted state-dict keys."""


def _register(root: nn.Module, key: str, param: nn.Parameter) -> None:
    parts = key.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Node())
        mod = mod._modules[p]
    mod.register_parameter(parts[-1], param)


class _Plan:
    """Owns one ``b200unet_plan`` + its workspace for a fixed (batch, D, H, W, precision, device)."""

    def __init__(self, desc: _lib.NetDesc, device: torch.device):
        self.lib = _lib.load_library()
        self.handle = C.c_void_p()
        _lib.check(self.lib.b200unet_plan_create(C.byref(desc), C.byref(self.handle)), "plan_create")
        self.n_params = self.lib.b200unet_plan_num_params(self.handle)
        self.ws_bytes = int(self.lib.b200unet_plan_workspace_bytes(self.handle))
        self.device = device
        self.workspace = None
        self.inference_only = bool(desc.inference_only)
        self.serial = 0          # forward passes issued with save_for_backward (see _UNetFunction.backward)
        self.packed_stamp = None  # (parameter pointers, sum of version counters) the workspace's packed weights were made from

    def ensure_workspace(self):
        if self.workspace is None:
            self.workspace = torch.empty(self.ws_bytes, dtype=torch.uint8, device=self.device)
        return self.workspace

    def param_spec(self):
        out = []
        shape = (C.c_int64 * 5)()
        buf = C.create_string_buffer(256)
        for i in range(self.n_params):
            nd = self.lib.b200unet_plan_param_info(self.handle, i, shape, buf, 256)
            out.append((buf.value.decode(), tuple(int(shape[k]) for k in range(nd))))
        return out

    def last_launches(self) -> int:
        return int(self.lib.b200unet_plan_last_launches(self.handle))

    def backward_parts(self) -> int:
        """2 when the backward schedule can run as two calls (``b200unet_plan_backward_part``), else 1 (0: forward-only plan)"""
        return int(self.lib.b200unet_plan_backward_parts(self.handle))

    def param_parts(self):
        """per parameter (state-dict order): the backward part after which its gradient is final"""
        if self.backward_parts() != 2:
            return [0] * self.n_params
        return [int(self.lib.b200unet_plan_param_backward_part(self.handle, i)) for i in range(self.n_params)]

    CATEGORIES = ("conv_fwd", "conv_dgrad", "conv_wgrad", "norm_act", "resample", "head", "weight_pack", "other")

    def algorithmic_macs(self):
        n = len(self.CATEGORIES)
        arr = (C.c_double * n)()
        _lib.check(self.lib.b200unet_plan_algorithmic_macs(self.handle, arr, n), "algorithmic_macs")
        return dict(zip(self.CATEGORIES, [float(v) for v in arr]))

    def profile_begin(self, max_launches: int) -> None:
        _lib.check(self.lib.b200unet_plan_profile_begin(self.handle, int(max_launches)), "profile_begin")

    def profile_dump(self, path: str) -> None:
        _lib.check(self.lib.b200unet_plan_profile_dump(self.handle, path.encode()), "profile_dump")

    def profile_end(self):
        n = len(self.CATEGORIES)
        ms = (C.c_double * n)()
        cnt = (C.c_int64 * n)()
        _lib.check(self.lib.b200unet_plan_profile_end(self.handle, ms, cnt, n), "profile_end")
        return {k: {"ms": float(m), "launches": int(c)} for k, m, c in zip(self.CATEGORIES, ms, cnt)}

    def __del__(self):
        try:
            if self.handle:
                self.lib.b200unet_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


def _ptr_array(tensors: Sequence[torch.Tensor]):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


class _UNetFunction(torch.autograd.Function):
    """forward+backward of the whole network as two library calls (a third one for the input gradient)."""

    @staticmethod
    def forward(ctx, model, x, drop, need_bwd, need_dx, *params):
        # need_bwd / need_dx are decided by the caller: inside Function.forward autograd's grad mode is always off.  need_dx
        # selects a plan created with input_grad (same parameter-gradient launches, plus the input-gradient ops)
        plan = model._plan_for(x, inference_only=not need_bwd, input_grad=need_dx)
        n, _, d, h, w = x.shape
        logits = torch.empty((n, model.n_outputs, d, h, w), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):   # the library launches on the current device's current stream
            ws = plan.ensure_workspace()
            pa = _ptr_array(params)
            # packed bf16 weights are reused while no parameter has been written (torch's tensor version counters) and the
            # storage is the same: tiled inference runs 9-27 forwards per volume on fixed weights
            stamp = (tuple(p.data_ptr() for p in params), sum(p._version for p in params))
            # (forward-only plans only: a training step always repacks, also inside a captured CUDA graph)
            flags = int(need_bwd) | (2 if (not need_bwd and plan.packed_stamp == stamp) else 0)
            _lib.check(plan.lib.b200unet_plan_forward(plan.handle, x.data_ptr(), pa, drop.data_ptr() if drop is not None else None,
                                                      flags, ws.data_ptr(), logits.data_ptr(), _lib.stream_ptr()),
                       "plan_forward")
            plan.packed_stamp = stamp
        model.launches_last_forward = plan.last_launches()
        if need_bwd:
            plan.serial += 1
        ctx.plan = plan
        ctx.need_dx = bool(need_dx)
        ctx.serial = plan.serial
        ctx.model = model
        ctx.save_for_backward(*params)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        plan = ctx.plan
        if plan.inference_only:
            raise RuntimeError("B200 UNet3D: backward through a forward that ran without gradients enabled")
        if ctx.serial != plan.serial:
            # the saved activations, GroupNorm statistics and the dropout mask live in ONE per-shape workspace: a later
            # forward of the same shape has overwritten what this backward needs
            raise RuntimeError("B200 UNet3D: backward of forward pass #%d, but forward pass #%d of the same input shape has "
                               "overwritten the saved activations since; run backward before the next same-shape forward "
                               "(one outstanding forward per input shape)" % (ctx.serial, plan.serial))
        params = ctx.saved_tensors
        model = ctx.model
        need_dx = ctx.need_dx and ctx.needs_input_grad[1]
        if need_dx and torch.is_grad_enabled():
            raise RuntimeError("B200 %s: double backward (create_graph=True) through the input gradient is not supported"
                               % type(model).__name__)
        dlogits = dlogits.contiguous().float()
        dx = None
        with torch.cuda.device(dlogits.device):
            grads, direct = model._grad_targets(params, plan)
            # the input gradient reads what the whole backward leaves in the workspace: never deferred
            if model._defer_backward_tail and direct and not need_dx and plan.backward_parts() == 2:
                # two-part backward (train.GraphedTrainStep with a gradient exchange): part 0 -- head, decoder, deepest encoder
                # level -- runs here; the caller runs the rest through finish_backward() after it has started the exchange of
                # the gradients that are final now (model.flat_gradient_bucket_parts()[0])
                _lib.check(plan.lib.b200unet_plan_backward_part(plan.handle, 0, dlogits.data_ptr(), _ptr_array(params), _ptr_array(grads),
                                                                plan.workspace.data_ptr(), _lib.stream_ptr()), "plan_backward_part(0)")
                model._backward_tail = (plan, dlogits, params, grads)
            else:
                _lib.check(plan.lib.b200unet_plan_backward(plan.handle, dlogits.data_ptr(), _ptr_array(params), _ptr_array(grads),
                                                           plan.workspace.data_ptr(), _lib.stream_ptr()), "plan_backward")
            model.launches_last_backward = plan.last_launches()
            if need_dx:
                n, _, d, h, w = dlogits.shape
                dx = torch.empty((n, model.n_features, d, h, w), dtype=torch.float32, device=dlogits.device)
                _lib.check(plan.lib.b200unet_plan_input_grad(plan.handle, dx.data_ptr(), plan.workspace.data_ptr(), _lib.stream_ptr()),
                           "plan_input_grad")
                model.launches_last_backward += plan.last_launches()
        if direct:                      # flat-bucket mode: the gradients already sit in the parameters' .grad views
            return (None, dx, None, None, None) + (None,) * len(params)
        return (None, dx, None, None, None) + tuple(grads)


class _PlanModel(nn.Module):
    """Shared machinery of the plan-backed models: canonical fp32 parameters under the reference's state-dict keys, a
    cache of whole-network plans keyed by input shape, gradient placement.  Subclasses provide ``_param_spec_cpu`` (ordered
    (key, shape) list), ``_net_desc`` (the library's network descriptor) and ``_init_tensor``."""

    def _setup(self, precision: Optional[str], deterministic: Optional[bool] = None) -> None:
        # deterministic: weight gradients reduced without floating-point atomics (per-split partial sums + fixed-order sum):
        # bit-identical gradients run to run at ~3 % of the step time; B200UNET_DETERMINISTIC=1 sets the default
        if deterministic is None:
            deterministic = os.environ.get("B200UNET_DETERMINISTIC", "0") == "1"
        self.deterministic = bool(deterministic)
        precision = precision or os.environ.get("B200UNET_PRECISION", "bf16")
        if precision not in ("bf16", "split"):
            raise ValueError("precision must be 'bf16' or 'split'")
        self.precision = precision
        self._plans: Dict[Tuple, _Plan] = {}
        self.launches_last_forward = 0
        self.launches_last_backward = 0
        self._forced_dropout_scale: Optional[torch.Tensor] = None
        self._flat_grads = False
        self._grad_bucket: Optional[torch.Tensor] = None
        self._grad_views = None
        self._bucket_split = None        # elements of the bucket that belong to part 0 of a two-part backward
        self._param_parts = None         # per parameter: backward part after which its gradient is final (from the plan)
        self._defer_backward_tail = False
        self._backward_tail = None
        self._keys = []
        spec = self._param_spec_cpu()
        shapes = dict(spec)
        for key, shape in spec:
            t = torch.empty(shape, dtype=torch.float32)
            self._init_tensor(key, t, shapes)
            _register(self, key, nn.Parameter(t))
            self._keys.append(key)

    def ordered_parameters(self):
        sd = dict(self.named_parameters())
        return [sd[k] for k in self._keys]

    # ------------------------------------------------------------------ plan cache
    def _plan_for(self, x: torch.Tensor, inference_only: bool = False, input_grad: bool = False) -> _Plan:
        n, _, d, h, w = x.shape
        key = (n, d, h, w, self.precision, x.device.index, bool(input_grad), bool(inference_only))
        plan = self._plans.get(key)
        if plan is None:
            desc = self._net_desc(n, d, h, w)
            desc.inference_only = int(bool(inference_only))
            desc.input_grad = int(bool(input_grad))
            desc.deterministic = int(self.deterministic and not inference_only)
            plan = _Plan(desc, x.device)
            spec = plan.param_spec()
            mine = [(k, tuple(p.shape)) for k, p in zip(self._keys, self.ordered_parameters())]
            if spec != mine:
                raise RuntimeError("libb200unet parameter spec does not match the module's state_dict")
            self._plans[key] = plan
        return plan

    # ------------------------------------------------------------------ gradient placement
    def use_flat_gradients(self, enabled: bool = True) -> None:
        """Write the parameter gradients straight into views of ONE persistent flat fp32 bucket (the parameters whose gradients are final first:
        ``flat_gradient_bucket_parts``) and
        bind them as ``p.grad``: no per-step allocation, and the data-parallel exchange (``parallel.GradAllReduce``)
        all-reduces the bucket in place without copies.  Backward then returns no gradients to autograd for the
        parameters (hooks on them do not fire)."""
        self._flat_grads = bool(enabled)
        if not enabled:
            self._grad_bucket = self._grad_views = self._bucket_split = None

    def flat_gradient_bucket(self) -> Optional[torch.Tensor]:
        return self._grad_bucket

    def flat_gradient_bucket_parts(self):
        """``(early, late)`` slices of the flat bucket: the gradients that are final after part 0 of a two-part backward (head,
        decoder, deepest encoder level: ~90 % of the parameters) and the rest.  ``None`` before the first flat-gradient backward."""
        if self._grad_bucket is None or self._bucket_split is None:
            return None
        return self._grad_bucket[:self._bucket_split], self._grad_bucket[self._bucket_split:]

    def _bucket_views(self, params, plan=None):
        if (self._grad_bucket is None or self._grad_bucket.device != params[0].device
                or self._grad_bucket.numel() != sum(p.numel() for p in params)):
            if self._param_parts is None:
                # the schedule's split point is a property of the architecture, not of the input shape: any training plan tells
                self._param_parts = plan.param_parts() if plan is not None else [0] * len(params)
            self._grad_bucket = torch.zeros(sum(p.numel() for p in params), dtype=torch.float32, device=params[0].device)
            # bucket layout: the parameters of part 0 first (state-dict order within a part), so that each part is one
            # contiguous slice for the exchange; the views stay in state-dict order
            views, off = [None] * len(params), 0
            for part in (0, 1):
                for i, p in enumerate(params):
                    if (self._param_parts[i] != 0) == bool(part):
                        views[i] = self._grad_bucket[off:off + p.numel()].view_as(p)
                        off += p.numel()
                if part == 0:
                    self._bucket_split = off
            self._grad_views = views
        return self._grad_views

    def finish_backward(self) -> None:
        """Runs part 1 of a deferred two-part backward (see ``_UNetFunction.backward``) on the current stream."""
        if self._backward_tail is None:
            raise RuntimeError("finish_backward: no deferred backward is pending")
        plan, dlogits, params, grads = self._backward_tail
        self._backward_tail = None
        with torch.cuda.device(dlogits.device):
            _lib.check(plan.lib.b200unet_plan_backward_part(plan.handle, 1, dlogits.data_ptr(), _ptr_array(params), _ptr_array(grads),
                                                            plan.workspace.data_ptr(), _lib.stream_ptr()), "plan_backward_part(1)")
        self.launches_last_backward += plan.last_launches()

    def _grad_targets(self, params, plan=None):
        """(tensors the library writes the gradients into, whether they are already bound as ``.grad``)."""
        if not self._flat_grads:
            return [torch.empty_like(p) for p in params], False
        views = self._bucket_views(params, plan)
        live = self.ordered_parameters()
        if all(p.grad is None for p in live):                       # the usual step: zero_grad(set_to_none=True) ran
            for p, v in zip(live, views):
                if p.requires_grad:
                    p.grad = v
            return views, True
        bound = all(p.grad is not None and p.grad.data_ptr() == v.data_ptr() for p, v in zip(live, views) if p.requires_grad)
        if bound and self._overwrite_grads:                         # CUDA-graph replay: every step overwrites .grad
            return views, True
        # gradient accumulation (an earlier backward's result is still in .grad): compute into fresh tensors and let
        # autograd add them
        return [torch.empty_like(p) for p in params], False

    _overwrite_grads = False   # set by train.GraphedTrainStep while it owns the step

    @staticmethod
    def _needs_backward(params, x: torch.Tensor) -> Tuple[bool, bool]:
        """(training plan: activations kept, iff autograd will ask for a backward; otherwise the forward-only plan,
        input gradient: the plan also produces d(loss)/d(x))"""
        need_dx = bool(torch.is_grad_enabled() and x.requires_grad)
        return bool(need_dx or (torch.is_grad_enabled() and any(p.requires_grad for p in params))), need_dx

    def _check_input(self, x: torch.Tensor, n_in: int) -> torch.Tensor:
        if not isinstance(x, torch.Tensor) or x.dim() != 5:
            raise ValueError("%s expects a 5-D tensor [N, C, D, H, W]" % type(self).__name__)
        if not x.is_cuda:
            raise RuntimeError("B200 %s runs only on CUDA tensors (no CPU fallback); got device %s" % (type(self).__name__, x.device))
        if x.shape[1] != n_in:
            raise ValueError("expected %d input channels, got %d" % (n_in, x.shape[1]))
        # MetaTensor -> plain view; as_subclass, contiguous and float stay on the autograd graph, so the input gradient
        # reaches the caller's tensor
        xp = x.as_subclass(torch.Tensor) if type(x) is not torch.Tensor else x
        xp = xp.contiguous().float()
        params = self.ordered_parameters()
        if params[0].device != xp.device:
            raise RuntimeError("model parameters are on %s but the input is on %s" % (params[0].device, xp.device))
        return xp


class UNet3D(_PlanModel):
    """Drop-in for the reference ``UNet3D`` (same ctor kwargs, same state_dict), H100-native arithmetic.

    Extra kwarg ``precision``: ``"bf16"`` (default; single-pass bf16 tensor-core operands, fp32 accumulate) or
    ``"split"`` (hi/lo bf16 operand split, three MMAs per product: the parity mode that meets 1e-3 vs fp32).
    ``B200UNET_PRECISION`` overrides the default.
    """

    def __init__(self, input_shape=None, n_features=1, base_width=32, encoder_blocks=None, decoder_blocks=None,
                 feature_dilation=2, downsampling_stride=2, interpolation_mode="trilinear", encoder_class=None,
                 decoder_class=None, n_outputs=1, layer_widths=None, decoder_mirrors_encoder=False, activation=None,
                 use_transposed_convolutions=False, kernel_size=3, precision: Optional[str] = None,
                 dropout: float = 0.2, norm_groups: int = 8, deterministic: Optional[bool] = None):
        super().__init__()
        if downsampling_stride != 2:
            raise NotImplementedError("B200 UNet3D: downsampling_stride=%r (only 2 is implemented)" % (downsampling_stride,))
        if interpolation_mode != "trilinear":
            raise NotImplementedError("B200 UNet3D: interpolation_mode=%r (only 'trilinear')" % (interpolation_mode,))
        if kernel_size != 3:
            raise NotImplementedError("B200 UNet3D: kernel_size=%r (only 3)" % (kernel_size,))
        if layer_widths is not None:
            raise NotImplementedError("B200 UNet3D: layer_widths is not supported (the reference's UNet3D also breaks on it)")
        if encoder_class is not None or decoder_class is not None:
            raise NotImplementedError("B200 UNet3D: custom encoder/decoder classes are not supported")
        if activation not in _ACT:
            raise ValueError("activation must be None, 'sigmoid' or 'softmax'")
        if encoder_blocks is None:
            encoder_blocks = [1, 2, 2, 4]                       # variational.py:44-45
        if decoder_mirrors_encoder:
            decoder_blocks = list(encoder_blocks)               # variational.py:71-74
        elif decoder_blocks is None:
            decoder_blocks = [1] * len(encoder_blocks)          # variational.py:75-76
        if len(decoder_blocks) != len(encoder_blocks):
            raise ValueError("decoder_blocks and encoder_blocks must have the same length")
        self.input_shape = input_shape
        self.n_features, self.n_outputs, self.base_width = int(n_features), int(n_outputs), int(base_width)
        self.encoder_blocks, self.decoder_blocks = [int(b) for b in encoder_blocks], [int(b) for b in decoder_blocks]
        self.feature_dilation = int(feature_dilation)
        self.use_transposed_convolutions = bool(use_transposed_convolutions)
        self.activation_name = activation
        self.dropout_p = float(dropout)                          # myronenko.py:85 (hard-wired 0.2 in the reference)
        self.norm_groups = int(norm_groups)
        self.dropout_width = self.base_width
        self._setup(precision, deterministic)                    # parameters under the reference's keys (SURVEY appendix B)

    @staticmethod
    def _init_tensor(key, t, shapes):
        """default torch init of the reference's modules (Conv3d: U(+-1/sqrt(fan_in)); GroupNorm: 1 / 0)"""
        if key.endswith("norm1.weight"):
            nn.init.ones_(t)
        elif key.endswith("norm1.bias"):
            nn.init.zeros_(t)
        else:
            wshape = shapes[key[:-5] + ".weight"] if key.endswith(".bias") else tuple(t.shape)
            fan_in = wshape[1] * wshape[2] * wshape[3] * wshape[4]   # torch default: weight.size(1) * k^3
            bound = 1.0 / math.sqrt(fan_in)
            nn.init.uniform_(t, -bound, bound)

    # ------------------------------------------------------------------ spec (pure python twin of plan.cu's)
    def _dec_widths(self, depth: int) -> Tuple[int, int]:
        n = len(self.encoder_blocks)
        if depth > 0:
            out_w = self.base_width * self.feature_dilation ** (depth - 1)
            in_w = out_w * self.feature_dilation
        else:
            out_w = in_w = self.base_width
        if depth != n - 1:
            in_w *= 2
        return in_w, out_w

    def _param_spec_cpu(self):
        spec = []

        def block(prefix, cin, cout):
            spec.append((prefix + ".conv1.norm1.weight", (cin,)))
            spec.append((prefix + ".conv1.norm1.bias", (cin,)))
            spec.append((prefix + ".conv1.conv.weight", (cout, cin, 3, 3, 3)))
            spec.append((prefix + ".conv2.norm1.weight", (cout,)))
            spec.append((prefix + ".conv2.norm1.bias", (cout,)))
            spec.append((prefix + ".conv2.conv.weight", (cout, cout, 3, 3, 3)))
            if cin != cout:
                spec.append((prefix + ".sample.weight", (cout, cin, 1, 1, 1)))

        n = len(self.encoder_blocks)
        widths = [self.base_width * self.feature_dilation ** i for i in range(n)]
        cin = self.n_features
        for li, nb in enumerate(self.encoder_blocks):
            for b in range(nb):
                block("encoder.layers.%d.blocks.%d" % (li, b), cin if b == 0 else widths[li], widths[li])
            cin = widths[li]
        for li in range(n - 1):
            spec.append(("encoder.downsampling_convolutions.%d.weight" % li, (widths[li], widths[li], 3, 3, 3)))
        for i, nb in enumerate(self.decoder_blocks):
            depth = n - 1 - i
            in_w, out_w = self._dec_widths(depth)
            planes = in_w if depth != 0 else out_w
            for b in range(nb):
                block("decoder.layers.%d.blocks.%d" % (i, b), in_w if b == 0 else planes, planes)
        for i in range(n - 1):
            in_w, out_w = self._dec_widths(n - 1 - i)
            if self.use_transposed_convolutions:
                spec.append(("decoder.upsampling_blocks.%d.weight" % i, (in_w, out_w, 3, 3, 3)))
                spec.append(("decoder.upsampling_blocks.%d.bias" % i, (out_w,)))
            else:
                spec.append(("decoder.pre_upsampling_blocks.%d.weight" % i, (out_w, in_w, 1, 1, 1)))
        spec.append(("final_convolution.weight", (self.n_outputs, self.base_width, 1, 1, 1)))
        return spec

    # ------------------------------------------------------------------ library descriptor
    def _net_desc(self, n, d, h, w) -> _lib.NetDesc:
        nd = _lib.NetDesc()
        nd.n_features, nd.n_outputs, nd.base_width = self.n_features, self.n_outputs, self.base_width
        nd.n_levels = len(self.encoder_blocks)
        for i, b in enumerate(self.encoder_blocks):
            nd.encoder_blocks[i] = b
        for i, b in enumerate(self.decoder_blocks):
            nd.decoder_blocks[i] = b
        nd.feature_dilation = self.feature_dilation
        nd.norm_groups = self.norm_groups
        nd.use_transposed_convolutions = int(self.use_transposed_convolutions)
        nd.activation = _ACT[self.activation_name]
        nd.split_precision = int(self.precision == "split")
        nd.batch, nd.depth, nd.height, nd.width = n, d, h, w
        return nd

    def set_dropout_scale(self, scale: Optional[torch.Tensor]) -> None:
        """Testing hook: force the (N, C0) Dropout3d channel scale used by the next training forwards."""
        self._forced_dropout_scale = scale

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        xp = self._check_input(x, self.n_features)
        params = self.ordered_parameters()
        drop = None
        if self.training and self.dropout_p > 0:
            if self._forced_dropout_scale is not None:
                drop = self._forced_dropout_scale.to(device=xp.device, dtype=torch.float32).contiguous()
            else:
                keep = (torch.rand((xp.shape[0], self.base_width), device=xp.device) >= self.dropout_p)
                drop = keep.float() / (1.0 - self.dropout_p)
        return _UNetFunction.apply(self, xp, drop, *self._needs_backward(params, xp), *params)


class AutocastUNet(UNet3D):
    """Reference: fp16 autocast wrapper (unet.py:53-58).  Here: the single-pass bf16 tensor-core mode."""

    def __init__(self, *args, **kwargs):
        kwargs.setdefault("precision", "bf16")
        super().__init__(*args, **kwargs)


class AutoImplantUNet(UNet3D):
    """unet.py:61-70: forward returns ``y - x``; ``test`` returns the plain network output."""

    def forward(self, x):
        y = super().forward(x)
        return y - x

    def test(self, x):
        return super().forward(x)


class DynUNet(_PlanModel):
    """Drop-in for ``monai.networks.nets.DynUNet`` as the reference's example configs instantiate it
    (examples/brats2020/brats2020_config.json:2-107, examples/sppin/sppin_config.json: ``getattr(unet3d.models.pytorch,
    "DynUNet")(**kwargs)`` through the ``from monai.networks.nets import *`` in unet3d/models/pytorch/__init__.py:1).

    MONAI's kwarg names; implemented: ``spatial_dims=3``, ``kernel_size`` all 3, ``strides`` [1, 2, 2, ...],
    ``upsample_kernel_size`` all 2 (transposed convolution with kernel = stride), instance norm (affine), LeakyReLU,
    ``res_block=False``, ``deep_supervision=False``, ``trans_bias=False``, ``dropout=None``; anything else raises.
    State-dict keys follow MONAI's module names (input_block / downsamples.N / bottleneck / upsamples.N / output_block);
    MONAI additionally exposes the same tensors a second time under ``skip_layers.*`` -- load such a checkpoint with
    ``strict=False`` (parity with MONAI itself is unpinned: it is absent from this image)."""

    def __init__(self, spatial_dims=3, in_channels=1, out_channels=1, kernel_size=None, strides=None, upsample_kernel_size=None,
                 filters=None, dropout=None, norm_name=("INSTANCE", {"affine": True}),
                 act_name=("leakyrelu", {"inplace": True, "negative_slope": 0.01}), deep_supervision=False, deep_supr_num=1,
                 res_block=False, trans_bias=False, precision: Optional[str] = None, deterministic: Optional[bool] = None):
        super().__init__()

        def triple(v):
            return [int(v)] * 3 if isinstance(v, int) else [int(e) for e in v]
        if spatial_dims != 3:
            raise NotImplementedError("B200 DynUNet: spatial_dims=%r (only 3)" % (spatial_dims,))
        if strides is None or kernel_size is None:
            raise ValueError("DynUNet needs kernel_size and strides")
        strides = [triple(v) for v in strides]
        kernel_size = [triple(v) for v in kernel_size]
        if upsample_kernel_size is None:
            upsample_kernel_size = strides[1:]
        upsample_kernel_size = [triple(v) for v in upsample_kernel_size]
        if len(kernel_size) != len(strides) or len(upsample_kernel_size) != len(strides) - 1:
            raise ValueError("length of kernel_size and strides should be the same, upsample_kernel_size one shorter")
        if any(k != [3, 3, 3] for k in kernel_size):
            raise NotImplementedError("B200 DynUNet: kernel_size must be 3 at every level")
        if strides[0] != [1, 1, 1] or any(v != [2, 2, 2] for v in strides[1:]):
            raise NotImplementedError("B200 DynUNet: strides must be [1, 2, 2, ...]")
        if any(v != [2, 2, 2] for v in upsample_kernel_size):
            raise NotImplementedError("B200 DynUNet: upsample_kernel_size must be 2 (= stride) at every level")
        norm = (norm_name if isinstance(norm_name, str) else norm_name[0]).lower()
        norm_kw = {} if isinstance(norm_name, str) else dict(norm_name[1])
        if norm != "instance" or not norm_kw.get("affine", False):
            raise NotImplementedError("B200 DynUNet: norm_name must be ('INSTANCE', {'affine': True})")
        act = (act_name if isinstance(act_name, str) else act_name[0]).lower()
        act_kw = {} if isinstance(act_name, str) else dict(act_name[1])
        if act not in ("leakyrelu", "relu"):
            raise NotImplementedError("B200 DynUNet: act_name %r (only leakyrelu / relu)" % (act_name,))
        if deep_supervision or res_block or trans_bias or dropout is not None:
            raise NotImplementedError("B200 DynUNet: deep_supervision / res_block / trans_bias / dropout are not implemented")
        if filters is None:
            filters = [min(2 ** (5 + i), 320) for i in range(len(strides))]      # MONAI's default for spatial_dims = 3
        filters = [int(f) for f in filters][:len(strides)]
        if len(filters) < len(strides):
            raise ValueError("length of filters should be no less than the length of strides")
        if not 2 <= len(filters) <= 8:
            raise NotImplementedError("B200 DynUNet: 2..8 levels")
        self.in_channels, self.out_channels = int(in_channels), int(out_channels)
        self.n_features, self.n_outputs = self.in_channels, self.out_channels
        self.filters = filters
        self.act_slope = float(act_kw.get("negative_slope", 0.01)) if act == "leakyrelu" else 0.0
        self._setup(precision, deterministic)

    def _param_spec_cpu(self):
        spec = []
        L = len(self.filters)
        F = self.filters

        def block(prefix, cin, cout):
            spec.append((prefix + ".conv1.conv.weight", (cout, cin, 3, 3, 3)))
            spec.append((prefix + ".conv2.conv.weight", (cout, cout, 3, 3, 3)))
            for n in ("norm1", "norm2"):
                spec.append((prefix + "." + n + ".weight", (cout,)))
                spec.append((prefix + "." + n + ".bias", (cout,)))
        for i in range(L):
            name = "input_block" if i == 0 else "bottleneck" if i == L - 1 else "downsamples.%d" % (i - 1)
            block(name, self.in_channels if i == 0 else F[i - 1], F[i])
        for u in range(L - 1):
            lo, hi = L - 1 - u, L - 2 - u
            spec.append(("upsamples.%d.transp_conv.conv.weight" % u, (F[lo], F[hi], 2, 2, 2)))
            block("upsamples.%d.conv_block" % u, 2 * F[hi], F[hi])
        spec.append(("output_block.conv.conv.weight", (self.out_channels, F[0], 1, 1, 1)))
        spec.append(("output_block.conv.conv.bias", (self.out_channels,)))
        return spec

    def _init_tensor(self, key, t, shapes):
        """MONAI DynUNet.initialize_weights: kaiming_normal_(a=0.01) on conv / transposed-conv weights, zero biases;
        InstanceNorm affine 1 / 0."""
        if ".norm" in key:
            (nn.init.ones_ if key.endswith("weight") else nn.init.zeros_)(t)
        elif key.endswith(".bias"):
            nn.init.zeros_(t)
        else:
            nn.init.kaiming_normal_(t, a=0.01)

    def _net_desc(self, n, d, h, w) -> _lib.NetDesc:
        nd = _lib.NetDesc()
        nd.arch = 1
        nd.n_features, nd.n_outputs = self.in_channels, self.out_channels
        nd.n_levels = len(self.filters)
        for i, f in enumerate(self.filters):
            nd.filters[i] = f
        nd.act_slope = self.act_slope
        nd.activation = 0
        nd.split_precision = int(self.precision == "split")
        nd.batch, nd.depth, nd.height, nd.width = n, d, h, w
        return nd

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        xp = self._check_input(x, self.in_channels)
        params = self.ordered_parameters()
        return _UNetFunction.apply(self, xp, None, *self._needs_backward(params, xp), *params)


_MODELS = {"UNet3D": UNet3D, "AutocastUNet": AutocastUNet, "AutoImplantUNet": AutoImplantUNet,
           "B200UNet3D": UNet3D, "DynUNet": DynUNet}


def fetch_model_by_name(model_name, *args, **kwargs):
    """build.py:9-13."""
    try:
        cls = _MODELS[model_name]
    except KeyError:
        raise ValueError("model name {} not supported".format(model_name))
    return cls(*args, **kwargs)


def match_tensor_sizes(fixed_tensor, moving_tensor):
    """build.py:54-64: tile then narrow every mismatching dim."""
    fixed_size = fixed_tensor.size()
    for dim in range(len(moving_tensor.size())):
        if fixed_size[dim] > moving_tensor.size()[dim]:
            reps = int(math.ceil(fixed_size[dim] / moving_tensor.size()[dim]))
            moving_tensor = torch.cat([moving_tensor] * reps, dim=dim)
        if fixed_size[dim] != moving_tensor.size()[dim]:
            moving_tensor = moving_tensor.narrow(dim=dim, start=0, length=fixed_size[dim])
    return moving_tensor


def match_state_dict_shapes(fixed_state_dict, moving_state_dict):
    """build.py:47-51."""
    for key in fixed_state_dict:
        if key in moving_state_dict and fixed_state_dict[key].size() != moving_state_dict[key].size():
            moving_state_dict[key] = match_tensor_sizes(fixed_state_dict[key], moving_state_dict[key])
    return moving_state_dict


def load_state_dict(model, state_dict, n_gpus, strict=False):
    """build.py:32-44 (the DataParallel retry branch is kept for wrapped models)."""
    try:
        if not strict:
            state_dict = match_state_dict_shapes(model.state_dict(), state_dict)
        model.load_state_dict(state_dict, strict=strict)
    except RuntimeError as error:
        if n_gpus > 1 and hasattr(model, "module"):
            if not strict:
                state_dict = match_state_dict_shapes(model.module.state_dict(), state_dict)
            model.module.load_state_dict(state_dict, strict=strict)
        else:
            raise error
    return model


def build_or_load_model(model_name, model_filename, n_gpus=0, strict=False, **kwargs):
    """build.py:16-29.  ``n_gpus > 1`` in ONE process is the reference's DataParallel branch; this path is one
    process per GPU (see ``parallel.py``), so here every n_gpus >= 1 places the replica on the current device."""
    model = fetch_model_by_name(model_name, **kwargs)
    if n_gpus > 0:
        model = model.cuda()
    if model_filename and os.path.exists(model_filename):
        if n_gpus > 0:
            state_dict = torch.load(model_filename)
        else:
            state_dict = torch.load(model_filename, map_location=torch.device("cpu"))
        model = load_state_dict(model, state_dict, n_gpus=n_gpus, strict=strict)
    return model
