"""MONAI UNet on the GPU (oracle/unet_oracle.py: PARITY UNPINNED, MONAI is absent): split-precision logits and every parameter
gradient (PReLU slopes, biases in front of the norms, residual convs) and the input gradient against fp64 autograd, the bf16
mode at looser bounds, the forward-only plan, deterministic gradients, the CUDA-graph step, and the new kernels (device-slope
PReLU forward / backward, the slope gradient's run-to-run repeatability, the logits unpack) element by element."""
import pytest
import torch

from oracle.unet_oracle import MonaiUNetConfig, make_unet_state_dict, unet_forward

pytestmark = pytest.mark.gpu
DEV = "cuda"
# those of test_gpu_segresnet.py's ReLU cases; the input gradient crosses every activation kink of the network once more than
# any parameter gradient, so it gets the gradient-norm bound with room for the flips of near-zero pre-activations
BOUNDS = dict(logits=1e-3, grad_norm=3e-2, cos=0.999, cos_small=0.995, dx=5e-2)
BF16_LOGITS = 5e-2


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def _kw(cfg):
    act = {"prelu": ("prelu", {"init": cfg.prelu_init}), "relu": "relu",
           "leakyrelu": ("leakyrelu", {"negative_slope": cfg.act_slope})}[cfg.act]
    return dict(in_channels=cfg.in_channels, out_channels=cfg.out_channels, channels=cfg.channels,
                strides=(2,) * (len(cfg.channels) - 1), num_res_units=cfg.num_res_units, bias=cfg.bias, act=act,
                norm=("instance", {"affine": cfg.norm_affine}))


def _setup(pkg, cfg, shape, precision="split", seed=0, deterministic=None):
    sd = make_unet_state_dict(cfg, seed=seed)
    m = pkg.UNet(precision=precision, deterministic=deterministic, **_kw(cfg)).to(DEV)
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn((shape[0], cfg.in_channels) + tuple(shape[1:]), generator=g, dtype=torch.float64)
    wl = torch.randn((shape[0], cfg.out_channels) + tuple(shape[1:]), generator=g, dtype=torch.float64)
    return m, sd, x, wl


def _reference(cfg, sd, x, wl, loss=None):
    """fp64 autograd of the oracle on the loss sum(out * wl), or loss(out): (logits, parameter gradients, input gradient)"""
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xr = x.clone().requires_grad_(True)
    out = unet_forward(xr, sd, cfg)
    ((out * wl).sum() if loss is None else loss(out)).backward()
    return out.detach(), {k: v.grad for k, v in sd.items()}, xr.grad


def _slope_noise_floor(cfg, sd, x, wl, ref_g, runs=2, loss=None):
    """largest change of each PReLU slope gradient over fp64 passes with every parameter perturbed by 2^-16 relative: a slope
    gradient sums z * g over the negative pre-activations of a whole layer, and the flips of near-zero z move it by far more
    than the split-precision rounding (the first residual unit of a 2-unit network moves by ~20 % in fp64 alone)"""
    floor = {k: 0.0 for k in ref_g if k.endswith(".adn.A.weight")}
    for t in range(runs):
        g = torch.Generator().manual_seed(100 + t)
        sd2 = {k: v * (1 + 2.0 ** -16 * torch.randn(v.shape, generator=g, dtype=torch.float64)) for k, v in sd.items()}
        _, g2, _ = _reference(cfg, sd2, x, wl, loss)
        for k in floor:
            floor[k] = max(floor[k], float((g2[k] - ref_g[k]).abs().max()))
    return floor


def _is_logits_conv(m, pre):
    return pre in ("model.2", "model.2.1.conv.unit0") and (pre == "model.2") == (m.num_res_units == 0)


def check_split_grads(m, ref_g, floor):
    """every parameter gradient of a split-precision step against fp64 (ref_g); floor: {PReLU slope key: its noise floor}.
    Returns the worst relative deviation of a gradient norm among the tensors held to the norm bound."""
    worst = 0.0
    for k, p in m.named_parameters():
        r = ref_g[k]
        g = p.grad.double().cpu()
        if k in floor:
            assert float((g - r).abs().max()) < 4 * floor[k] + BOUNDS["grad_norm"] * float(r.abs().max()), (k, g, r, floor[k])
            continue
        if k.endswith(".conv.bias") and not _is_logits_conv(m, k[:-len(".conv.bias")]):
            # in front of an instance norm: ~0, compared at an absolute bound scaled by the layer's weight gradient
            wn = float(ref_g[k[:-len("bias")] + "weight"].norm())
            assert float((g - r).abs().max()) < 1e-3 * wn + 1e-6, (k, g, r)
            assert bool((g != 0).any()), k   # the rounded per-channel sum, not zeros written in its place
            continue
        gn, rn = float(g.norm()), float(r.norm())
        worst = max(worst, abs(gn - rn) / (rn + 1e-30))
        assert abs(gn - rn) < BOUNDS["grad_norm"] * rn + 1e-12, (k, gn, rn)
        cos = float((g * r).sum() / (gn * rn + 1e-30))
        assert cos > (BOUNDS["cos_small"] if p.numel() <= 64 else BOUNDS["cos"]), (k, cos)
    return worst


CASES = [
    ("r0_prelu_bias", MonaiUNetConfig(1, 2, (8, 16, 32), 0, "prelu"), (2, 32, 32, 32)),
    ("r0_relu_nobias_affine", MonaiUNetConfig(4, 3, (16, 32, 64), 0, "relu", norm_affine=True, bias=False), (1, 32, 32, 32)),
    ("r1_leaky_bias", MonaiUNetConfig(1, 3, (8, 16, 32, 64), 1, "leakyrelu", act_slope=0.1), (1, 32, 48, 64)),
    ("r2_prelu_bias_affine", MonaiUNetConfig(4, 16, (16, 32, 64), 2, "prelu", prelu_init=0.1, norm_affine=True), (1, 32, 32, 32)),
    ("r2_prelu_nobias", MonaiUNetConfig(1, 1, (8, 16, 24), 2, "prelu", bias=False), (2, 32, 32, 32)),
    ("r1_relu_bias_equal_bottom", MonaiUNetConfig(4, 2, (16, 16), 1, "relu"), (1, 32, 32, 32)),
]


@pytest.mark.parametrize("name,cfg,shape", CASES, ids=[c[0] for c in CASES])
def test_unet_split_precision_matches_oracle(pkg, name, cfg, shape):
    m, sd, x, wl = _setup(pkg, cfg, shape)
    ref_out, ref_g, ref_dx = _reference(cfg, sd, x, wl)
    xg = x.float().to(DEV).requires_grad_(True)
    out = m(xg)
    (out * wl.float().to(DEV)).sum().backward()
    assert rel_l2(out.detach(), ref_out) < BOUNDS["logits"]
    assert rel_l2(xg.grad, ref_dx) < BOUNDS["dx"]
    floor = _slope_noise_floor(cfg, sd, x, wl, ref_g) if cfg.act == "prelu" else {}
    check_split_grads(m, ref_g, floor)
    # the forward-only plan computes the training plan's logits
    with torch.no_grad():
        out_inf = m(x.float().to(DEV))
    assert rel_l2(out_inf, out.detach()) < 1e-6


@pytest.mark.parametrize("name,cfg,shape", CASES[:3], ids=[c[0] for c in CASES[:3]])
def test_unet_bf16_mode_looser_bound(pkg, name, cfg, shape):
    m, sd, x, wl = _setup(pkg, cfg, shape, precision="bf16")
    with torch.no_grad():
        ref = unet_forward(x, sd, cfg)
        out = m(x.float().to(DEV))
    assert rel_l2(out, ref) < BF16_LOGITS
    # the last conv's fp32 accumulators reach the logits as hi + lo: bf16 mode does not round the logits to bf16 (a bf16-rounded
    # tensor would be representable in bf16 everywhere)
    assert float((out.bfloat16().float() == out).float().mean()) < 0.05


def test_unet_deterministic_gradients_bit_identical(pkg):
    cfg = MonaiUNetConfig(1, 2, (16, 32, 64), 2, "prelu", norm_affine=True)
    m, sd, x, wl = _setup(pkg, cfg, (2, 32, 32, 32), precision="bf16", deterministic=True)
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        (m(x.float().to(DEV)) * wl.float().to(DEV)).sum().backward()
        grads.append([p.grad.clone() for p in m.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def test_unet_graphed_step_matches_eager_and_sees_prelu_updates(pkg):
    from importlib import import_module
    train = import_module(pkg.__name__ + ".train")
    cfg = MonaiUNetConfig(1, 2, (16, 32, 64), 2, "prelu")
    shape = (2, 32, 32, 32)
    m, sd, x, wl = _setup(pkg, cfg, shape)
    xs, w = x.float().to(DEV), wl.float().to(DEV)

    def crit(out, t):
        return (out * t).sum()
    m.zero_grad(set_to_none=True)
    loss_e = crit(m(xs), w)
    loss_e.backward()
    eager = {k: p.grad.clone() for k, p in m.named_parameters()}
    loss_e = float(loss_e)
    m.zero_grad(set_to_none=True)
    slopes = [p for k, p in m.named_parameters() if k.endswith(".adn.A.weight")]
    others = [p for k, p in m.named_parameters() if not k.endswith(".adn.A.weight")]
    # plain SGD that moves only the PReLU slopes (the other parameters at lr 0)
    opt = torch.optim.SGD([{"params": others, "lr": 0.0}, {"params": slopes, "lr": 1e-4}])
    step = train.GraphedTrainStep(m, crit, opt, xs.shape, w.shape, target_dtype=torch.float32)
    loss_g = float(step(xs, w))
    assert abs(loss_g - loss_e) <= 1e-6 * abs(loss_e)
    for k, p in m.named_parameters():
        assert rel_l2(p.grad, eager[k]) < 1e-5, k
    # the step's optimizer update moved the slopes (slope -= lr * its gradient); the next replay must use the new values
    slope = dict(m.named_parameters())["model.0.conv.unit0.adn.A.weight"]
    expect = cfg.prelu_init - 1e-4 * float(eager["model.0.conv.unit0.adn.A.weight"])
    assert float(slope) == pytest.approx(expect, rel=1e-3, abs=1e-7) and float(slope) != cfg.prelu_init
    sd2 = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    ref = float((unet_forward(x, sd2, cfg) * wl).sum())
    loss_new = float(step(xs, w))
    ref_old = float((unet_forward(x, sd, cfg) * wl).sum())
    assert abs(loss_new - ref) < 1e-3 * (abs(ref) + 1.0)
    assert abs(loss_new - ref) < abs(loss_new - ref_old)


# ------------------------------------------------------------------------------------------------ the new kernels alone
def _act(pkg, t, split=True):
    return pkg.lib.Act.from_ncdhw(t, split=split)


# 72 and 264 channels: 252- and 231-thread blocks, whose last warp is partial
@pytest.mark.parametrize("c,with_add", [(8, False), (24, True), (3, True), (72, True), (264, False)])
def test_prelu_apply_and_bwd_against_fp64(pkg, c, with_add):
    L = pkg.lib
    g = torch.Generator().manual_seed(c)
    n, d, h, w = 2, 8, 12, 16
    x = torch.randn(n, c, d, h, w, generator=g, dtype=torch.float64) * 2 + 0.5
    add = torch.randn(n, c, d, h, w, generator=g, dtype=torch.float64)
    gy = torch.randn(n, c, d, h, w, generator=g, dtype=torch.float64)
    g2 = torch.randn(n, c, d, h, w, generator=g, dtype=torch.float64)
    gamma = 1 + 0.1 * torch.randn(c, generator=g, dtype=torch.float64)
    beta = 0.1 * torch.randn(c, generator=g, dtype=torch.float64)
    a = torch.tensor([0.3], dtype=torch.float64)
    xa = _act(pkg, x.float().to(DEV))
    cp = xa.c
    # the plans' inputs: x rounded to hi + lo
    xv = xa.value().permute(0, 4, 1, 2, 3)[:, :c].double().cpu()
    stats = torch.zeros(n, cp, 2, dtype=torch.float64, device=DEV)
    stats[:, :c, 0] = xv.sum((2, 3, 4)).to(DEV)
    stats[:, :c, 1] = (xv * xv).sum((2, 3, 4)).to(DEV)
    coef = torch.zeros(n, cp, 4, device=DEV)
    y = L.Act.empty(n, d, h, w, cp, split=True, device=DEV)
    adda = _act(pkg, add.float().to(DEV)) if with_add else None
    slope = a.float().to(DEV)
    L.prelu_apply(xa, y, stats, gamma.float().to(DEV), beta.float().to(DEV), c, c, coef, slope, add=adda)
    addv = adda.value().permute(0, 4, 1, 2, 3)[:, :c].double().cpu() if with_add else 0
    z = torch.nn.functional.group_norm(xv, c, gamma, beta, eps=1e-5)
    ref = torch.nn.functional.prelu(z, a) + addv
    assert rel_l2(y.to_ncdhw(c), ref) < 1e-4
    # backward: dz = (g1 + g2) * prelu'(z), dslope = sum_{z<0} z (g1 + g2), gsum = g1 + g2
    g1a, g2a = _act(pkg, gy.float().to(DEV)), _act(pkg, g2.float().to(DEV))
    gv = (g1a.value() + g2a.value()).permute(0, 4, 1, 2, 3)[:, :c].double().cpu()
    dz = L.Act.empty(n, d, h, w, cp, split=True, device=DEV)
    gs = L.Act.empty(n, d, h, w, cp, split=True, device=DEV)
    bstats = torch.zeros(n, cp, 2, dtype=torch.float64, device=DEV)
    dslope = torch.zeros(1, device=DEV)
    L.prelu_bwd(g1a, g2a, xa, coef, slope, dz, bstats, cp, dslope, gsum=gs)
    zz = z
    assert rel_l2(dz.to_ncdhw(c), torch.where(zz > 0, gv, gv * a)) < 1e-4
    assert rel_l2(gs.to_ncdhw(c), gv) < 1e-5
    ref_ds = float((torch.where(zz < 0, zz, torch.zeros_like(zz)) * gv).sum())
    assert abs(float(dslope) - ref_ds) < 1e-4 * (abs(ref_ds) + float((zz.clamp(max=0).abs() * gv.abs()).sum()) * 1e-3)
    # the slope gradient repeats bit for bit
    again = torch.zeros(1, device=DEV)
    L.prelu_bwd(g1a, g2a, xa, coef, slope, dz, torch.zeros_like(bstats), cp, again, gsum=gs)
    assert torch.equal(again, dslope)


@pytest.mark.parametrize("c,with_add,with_bias", [(1, False, True), (3, True, True), (16, True, False), (5, False, False)])
def test_logits_unpack_exact(pkg, c, with_add, with_bias):
    L = pkg.lib
    g = torch.Generator().manual_seed(c)
    n, d, h, w = 2, 4, 6, 10
    y = torch.randn(n, c, d, h, w, generator=g)
    r = torch.randn(n, c, d, h, w, generator=g)
    b = torch.randn(c, generator=g)
    ya = _act(pkg, y.to(DEV))
    ra = _act(pkg, r.to(DEV)) if with_add else None
    out = L.logits_unpack(ya, c, b.to(DEV) if with_bias else None, ra)
    yv = ya.value().permute(0, 4, 1, 2, 3)[:, :c]
    exp = yv + (b.to(DEV).view(1, c, 1, 1, 1) if with_bias else 0)
    if with_add:
        exp = exp + ra.value().permute(0, 4, 1, 2, 3)[:, :c]
    assert torch.equal(out, exp)
    # the backward's pack of dlogits into the padded layout: hi = bf16(x), lo = bf16(x - hi) on the real channels, zeros on the pad
    dl = torch.randn(n, c, d, h, w, generator=g).to(DEV)
    pa = L.Act.from_ncdhw(dl, split=True)
    nd = dl.permute(0, 2, 3, 4, 1)
    hi = nd.bfloat16()
    assert torch.equal(pa.hi[..., :c], hi) and torch.equal(pa.lo[..., :c], (nd - hi.float()).bfloat16())
    assert not pa.hi[..., c:].any() and not pa.lo[..., c:].any()


# (ci, co, input extents): an inner up layer of the spleen network, the conv-only top layer to 2 outputs, a 256 -> 128 bottom stage
@pytest.mark.parametrize("ci,co,dims,bias", [(48, 16, (8, 8, 8), True), (32, 2, (12, 8, 10), False), (256, 128, (6, 6, 6), True)])
def test_convt_output_padding_kind_three_directions(pkg, ci, co, dims, bias):
    """LAYER_CONVT_OP1 as the plan runs it: forward = zero insertion + a k3 s1 conv with the flipped pack (mode 2) and the bias,
    no forced-zero boundary; data gradient = a k3 s2 conv of dU with the mode-3 pack; weight gradient over the zero-inserted input,
    unpacked as mode 2.  Against fp64 autograd of ConvTranspose3d(k3, s2, p1, output_padding 1)."""
    import ctypes as C
    L = pkg.lib
    g = torch.Generator().manual_seed(ci + co)
    n = 1
    x = torch.randn(n, ci, *dims, generator=g)
    w = torch.randn(ci, co, 3, 3, 3, generator=g) / (ci * 27) ** 0.5
    b = torch.randn(co, generator=g) if bias else None
    fine = tuple(2 * e for e in dims)
    du = torch.randn(n, co, *fine, generator=g)
    xa, dua = _act(pkg, x.to(DEV)), _act(pkg, du.to(DEV))
    cip, cop = xa.c, dua.c
    z = L.Act.empty(n, *fine, cip, split=True, device=DEV)
    L.check(L.load_library().b200unet_zero_insert(C.byref(xa.ct()), C.byref(z.ct()), 0, 0, 0, L.stream_ptr()), "zero_insert")
    whi, wlo, _, _, _ = L.pack_weights(w.to(DEV), 2, split=True, cop=cop, cip=cip)
    y = L.Act.empty(n, *fine, cop, split=True, device=DEV)
    bp = torch.zeros(cop, device=DEV)
    if bias:
        bp[:co] = b.to(DEV)
    L.conv3d_ex(z, whi, wlo, 3, 1, y, cop, cip, ext=L.diag_ext(bias=bp))
    wdh, wdl, _, _, _ = L.pack_weights(w.to(DEV), 3, split=True, cop=cop, cip=cip)
    dx = L.Act.empty(n, *dims, cip, split=True, device=DEV)
    L.conv3d(dua, wdh, wdl, 3, 2, dx, cip, cop)
    acc = torch.zeros(27 * cip * cop, device=DEV)
    L.conv3d_wgrad(z, dua, 3, 1, cip, cop, acc)
    dw = torch.empty(ci, co, 3, 3, 3, device=DEV)
    L.check(L.load_library().b200unet_unpack_wgrad(acc.data_ptr(), co, ci, cop, cip, 27, 2, dw.data_ptr(), L.stream_ptr()), "unpack")
    xv = xa.value().permute(0, 4, 1, 2, 3)[:, :ci].double().cpu().requires_grad_(True)
    duv = dua.value().permute(0, 4, 1, 2, 3)[:, :co].double().cpu()
    w64 = w.double().requires_grad_(True)
    ref = torch.nn.functional.conv_transpose3d(xv, w64, b.double() if bias else None, stride=2, padding=1, output_padding=1)
    ref.backward(duv)
    assert rel_l2(y.to_ncdhw(co), ref.detach()) < 1e-4
    assert rel_l2(dx.to_ncdhw(ci), xv.grad) < 1e-4
    assert rel_l2(dw, w64.grad) < 1e-4
