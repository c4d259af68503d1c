"""CPU dry run of the host layer against a marshalling stub of libb200unet: every device-touching entry point is replaced
by a function that checks the argument COUNT and ctypes CONVERTIBILITY against the binding's declared signature and
returns success; the host-only entry points (plan creation, parameter spec, workspace sizes) stay real.  Catches what
otherwise only shows on the GPU box: wrong arity / argument order in a ctypes call, autograd plumbing (forward/backward
serial guard, flat gradient bucket, forward-only plans), the tiling loop of the inferer, the pre/post-processing wrappers.
No arithmetic is checked here (that is what the -m gpu tests are for)."""
import contextlib
import ctypes as C
import importlib

import pytest
import torch

HOST_ONLY = {"b200unet_version", "b200unet_last_error", "b200unet_plan_create", "b200unet_plan_destroy", "b200unet_plan_num_params",
             "b200unet_plan_param_info", "b200unet_plan_workspace_bytes", "b200unet_plan_last_launches", "b200unet_plan_algorithmic_macs",
             "b200unet_plan_backward_parts", "b200unet_plan_param_backward_part",
             "b200unet_head_bwd_scratch_bytes"}


class _FakeCuda(torch.Tensor):
    """a CPU tensor that claims to live on a CUDA device (only the entry checks of the host layer look at this flag)"""
    is_cuda = True


def fake(t):
    return t.as_subclass(_FakeCuda)


@pytest.fixture()
def stubbed(pkg, monkeypatch):
    L = pkg.lib
    real = L.load_library()
    calls = []

    class Stub:
        pass
    stub = Stub()
    for name, (res, argtypes) in list(L._SIGS.items()) + list(L._DIAG_SIGS.items()):
        if name in HOST_ONLY:
            setattr(stub, name, getattr(real, name))
            continue

        def make(name=name, argtypes=argtypes):
            def f(*args):
                assert len(args) == len(argtypes), "%s: %d arguments, signature has %d" % (name, len(args), len(argtypes))
                for i, (v, t) in enumerate(zip(args, argtypes)):
                    try:
                        t.from_param(v)
                    except Exception as e:  # noqa: BLE001
                        raise AssertionError("%s: argument %d (%r) does not convert to %s: %s" % (name, i, v, t, e))
                calls.append(name)
                return 0
            return f
        setattr(stub, name, make())
    monkeypatch.setattr(L, "_lib", stub)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(torch.cuda, "device", lambda *_a, **_k: contextlib.nullcontext())
    return calls


def _batch(n=1, c=4, o=3, s=16):
    x = fake(torch.randn(n, c, s, s, s))
    t = fake((torch.rand(n, o, s, s, s) > 0.5).to(torch.uint8))
    return x, t


def test_unet3d_training_and_inference_calls(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    crit = pkg.DiceLoss(sigmoid=True)
    x, t = _batch()
    model.train()
    out = model(x)
    assert out.shape == (1, 3, 16, 16, 16) and out.requires_grad
    loss = crit(fake(out), t)
    loss.backward()
    assert all(p.grad is not None and p.grad.shape == p.shape for p in model.parameters())
    assert stubbed.count("b200unet_plan_forward") == 1 and stubbed.count("b200unet_plan_backward") == 1
    assert "b200unet_dice_fwd" in stubbed and "b200unet_dice_bwd" in stubbed
    # forward-only plan under no_grad; the training plan is untouched
    with torch.no_grad():
        y = model(x)
    assert not y.requires_grad
    kinds = sorted(k[-1] for k in model._plans)
    assert kinds == [False, True]
    # one outstanding forward per shape
    o1 = model(x)
    o2 = model(x)
    o2.sum().backward()
    with pytest.raises(RuntimeError, match="overwritten the saved activations"):
        o1.sum().backward()
    with pytest.raises(RuntimeError):
        y.sum().backward()
    # soft (float) Dice targets take the fp32-target flag
    crit(fake(model(x)), fake(torch.rand(1, 3, 16, 16, 16))).backward()


def test_flat_gradient_bucket_binding(pkg, stubbed):
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    model.train()
    model.use_flat_gradients(True)
    x, _ = _batch()
    model(x).sum().backward()
    bucket = model.flat_gradient_bucket()
    lo, hi = bucket.data_ptr(), bucket.data_ptr() + 4 * bucket.numel()
    assert bucket.numel() == sum(p.numel() for p in model.parameters())
    assert all(lo <= p.grad.data_ptr() < hi for p in model.parameters())
    first = [p.grad.data_ptr() for p in model.parameters()]
    # accumulation: .grad still bound -> autograd adds fresh tensors into the views, pointers stay
    model(x).sum().backward()
    assert [p.grad.data_ptr() for p in model.parameters()] == first
    # the usual step: zero_grad(set_to_none) -> re-bound to the same views
    for p in model.parameters():
        p.grad = None
    model(x).sum().backward()
    assert [p.grad.data_ptr() for p in model.parameters()] == first
    sync = pkg.parallel.GradAllReduce(model.parameters(), model=model)
    sync()                                   # no process group: a no-op that must not raise
    # bucket layout: the parameters whose gradients part 0 of the two-part backward finishes (head, decoder, deepest encoder level)
    # form the leading slice, state-dict order within each slice; the views themselves stay in state-dict order
    early, late = model.flat_gradient_bucket_parts()
    assert early.data_ptr() == bucket.data_ptr() and early.numel() + late.numel() == bucket.numel() and late.numel() > 0
    plan = next(iter(model._plans.values()))
    parts = plan.param_parts()
    split = bucket.data_ptr() + 4 * early.numel()
    offs = {0: [], 1: []}
    for p, part in zip(model.ordered_parameters(), parts):
        assert (p.grad.data_ptr() < split) == (part == 0)
        offs[part].append(p.grad.data_ptr())
    assert offs[0] == sorted(offs[0]) and offs[1] == sorted(offs[1])
    assert not sync.supports_overlap and not sync._begun      # single process: begin() declines, finish() is the plain call
    sync.begin()
    sync.finish()


def test_deferred_backward_tail_calls(pkg, stubbed):
    """two-part backward marshalling: with the tail deferred the autograd backward issues part 0 only, finish_backward() part 1"""
    model = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    model.train()
    model.use_flat_gradients(True)
    x, _ = _batch()
    model._defer_backward_tail = True
    model(x).sum().backward()
    model._defer_backward_tail = False
    assert stubbed.count("b200unet_plan_backward_part") == 1 and stubbed.count("b200unet_plan_backward") == 0
    assert model._backward_tail is not None
    model.finish_backward()
    assert stubbed.count("b200unet_plan_backward_part") == 2 and model._backward_tail is None
    with pytest.raises(RuntimeError, match="no deferred backward"):
        model.finish_backward()
    # without the flat bucket the gradients go back through autograd: the backward cannot be deferred
    model2 = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    model2.train()
    model2._defer_backward_tail = True
    model2(x).sum().backward()
    assert model2._backward_tail is None and stubbed.count("b200unet_plan_backward") == 1


def test_dynunet_calls(pkg, stubbed):
    kw = dict(spatial_dims=3, in_channels=4, out_channels=3, kernel_size=[[3, 3, 3]] * 3, strides=[[1, 1, 1], [2, 2, 2], [2, 2, 2]],
              upsample_kernel_size=[[2, 2, 2]] * 2, filters=[8, 16, 24])
    model = pkg.DynUNet(**kw)
    x, t = _batch()
    model.train()
    pkg.DiceLoss(sigmoid=True)(fake(model(x)), t).backward()
    assert all(p.grad is not None for p in model.parameters())
    model.eval()
    with torch.no_grad():
        assert model(x).shape == (1, 3, 16, 16, 16)


def test_sliding_window_inferer_calls(pkg, stubbed):
    inf = pkg.SlidingWindowInferer(roi_size=(8, 8, 8), sw_batch_size=4, overlap=0.25, mode="gaussian")
    x = fake(torch.randn(2, 1, 12, 12, 20))
    with torch.no_grad():
        out = inf(x, lambda tiles: tiles + 1)
    assert out.shape == (2, 1, 12, 12, 20)
    n_tiles = 2 * 2 * 2 * 3                                                    # starts per axis: 12 -> [0, 4]; 20 -> [0, 6, 12]
    assert stubbed.count("b200unet_tiles_gather") == -(-n_tiles // 4) == stubbed.count("b200unet_tiles_scatter")
    assert stubbed.count("b200unet_tiles_count") == 1 and stubbed.count("b200unet_tiles_normalize") == 1
    inf(x, lambda tiles: tiles)                                                 # cached scan: no second count kernel
    assert stubbed.count("b200unet_tiles_count") == 1
    with pytest.raises(RuntimeError, match="inference-only"):
        w = torch.ones(1, requires_grad=True)
        inf(x, lambda tiles: tiles * w)


def test_prepost_calls(pkg, stubbed):
    lab = fake(torch.randint(0, 4, (1, 1, 6, 6, 6)).float())
    y = pkg.prepost.compile_one_hot_encoding(lab, n_labels=3, labels=[[1, 2, 3], [1, 3], 3])
    assert y.shape == (3, 6, 6, 6) and y.dtype == torch.uint8
    z = pkg.prepost.normalize_intensity(fake(torch.randn(4, 6, 6, 6)), nonzero=True, channel_wise=True)
    assert z.shape == (4, 6, 6, 6)
    p = fake(torch.rand(3, 6, 6, 6))
    assert pkg.prepost.convert_one_hot_to_label_map(p, [1, 2, 4], label_hierarchy=True).dtype == torch.int16
    assert pkg.prepost.convert_one_hot_to_label_map(p, [[1, 2], [4]], activation="sigmoid").shape == (2, 6, 6, 6)
    assert pkg.prepost.convert_one_hot_to_label_map_using_hierarchy(p, [1, 2, 4]).shape == (6, 6, 6)
    assert {"b200unet_one_hot", "b200unet_zscore", "b200unet_label_map"} <= set(stubbed)


def test_per_kernel_wrappers_marshal_fused_groupnorm(pkg, stubbed):
    """the thin wrappers tests/test_gpu_ops.py drives (conv3d, wgrad, GroupNorm, upsample, head, pack)"""
    L = pkg.lib
    a = L.Act(torch.zeros(1, 4, 8, 8, 8, dtype=torch.bfloat16))
    b = L.Act(torch.zeros(1, 4, 8, 8, 16, dtype=torch.bfloat16))
    w = torch.zeros(27, 16, 8, dtype=torch.bfloat16)
    st = torch.zeros(1, 16, 2, dtype=torch.float64)
    L.conv3d(a, w, None, 3, 1, b, 16, 8, res=b, stats=st, stats_ld=16, cls_mode=0)
    L.conv3d_wgrad(a, b, 3, 1, 8, 16, torch.zeros(27, 8, 16))
    coef = torch.zeros(1, 16, 4)
    L.gn_apply(b, b, st, None, None, 16, 8, coef, slope=0.01)
    L.gn_bwd(b, b, coef, st, None, 16, 8, b, torch.zeros(16), torch.zeros(16), add1=b)
    L.gn_bwd_finalize(st, coef, None, 1, 16, 16, 8, 1024, torch.zeros(1, 16, 2), None, None)
    L.head_bwd(b, torch.zeros(3, 16), 3, torch.zeros(1, 3, 4, 8, 8), b, torch.zeros(3, 16))
    L.pack_weights(torch.zeros(8, 16, 2, 2, 2), 4)
    assert {"b200unet_conv3d", "b200unet_gn_apply", "b200unet_gn_bwd", "b200unet_gn_bwd_finalize", "b200unet_head_bwd"} <= set(stubbed)
