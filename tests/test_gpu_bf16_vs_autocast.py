"""How accurate is the single-pass bf16 mode (what bench.py times)?  Measured side by side with torch's own bf16 autocast:
the oracle's functional graph of the reference model runs on the same GPU (a) in fp64 (ground truth; pinned to the CPU
oracle below), (b) under ``torch.autocast("cuda", dtype=torch.bfloat16)`` through cuDNN; this library runs in bf16 mode on
the same weights and inputs.  Per parameter tensor, the gradient error of this library must stay within a small factor of
autocast's error.

tools/bf16_grad_study.py prints the same comparison.  Bounds: whole gradient and logits <= 1.25x autocast, every tensor <= 2x
autocast + 5e-3, every gradient norm within 8 % of the truth."""
import pytest
import torch

from oracle import UNetConfig, make_state_dict, unet3d_forward, dice_loss

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _oracle_on_gpu(sd, x, t, cfg, dtype, autocast):
    sdr = {k: v.to(DEV, dtype).requires_grad_(True) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        out = unet3d_forward(sdr, x.to(DEV, dtype), cfg)
    loss = dice_loss(out.float() if autocast else out, t.to(DEV))
    loss.backward()
    return out.detach().double(), float(loss), {k: v.grad.double() for k, v in sdr.items()}


def test_gpu_fp64_graph_is_the_cpu_oracle():
    """the ground truth used below (oracle graph on cuda in fp64) against the CPU oracle in fp64"""
    cfg = UNetConfig(n_features=4, n_outputs=3, base_width=8)
    sd = make_state_dict(cfg, seed=0)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 4, 16, 16, 16, generator=g)
    t = (torch.rand(1, 3, 16, 16, 16, generator=g) > 0.7).to(torch.uint8)
    out_g, loss_g, grads_g = _oracle_on_gpu(sd, x, t, cfg, torch.float64, False)
    sdc = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    out_c = unet3d_forward(sdc, x.double(), cfg)
    loss_c = dice_loss(out_c, t)
    loss_c.backward()
    assert float((out_g.cpu() - out_c.detach()).norm() / out_c.detach().norm()) < 1e-10
    assert abs(loss_g - float(loss_c)) < 1e-12
    for k in sdc:
        assert float((grads_g[k].cpu() - sdc[k].grad).norm() / (sdc[k].grad.norm() + 1e-300)) < 1e-8, k


@pytest.mark.parametrize("bw,seed", [(16, 2), (32, 4)])
def test_bf16_mode_gradient_error_is_torch_autocast_class(pkg, bw, seed):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    kw = dict(n_features=4, n_outputs=3, base_width=bw)
    cfg = UNetConfig(**kw)
    sd = make_state_dict(cfg, seed=0)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 4, 64, 64, 64, generator=g)
    t = (torch.rand(1, 3, 64, 64, 64, generator=g) > 0.7).to(torch.uint8)
    ref_out, ref_loss, ref_g = _oracle_on_gpu(sd, x, t, cfg, torch.float64, False)
    ac_out, ac_loss, ac_g = _oracle_on_gpu(sd, x, t, cfg, torch.float32, True)

    model = pkg.UNet3D(precision="bf16", **kw).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.train()
    model.set_dropout_scale(torch.ones(1, bw))
    out = model(x.to(DEV))
    loss = pkg.DiceLoss(sigmoid=True)(out, t.to(DEV))
    loss.backward()
    ours_g = {k: p.grad.double() for k, p in model.named_parameters()}

    def rel(a, b):
        return float((a - b).norm() / (b.norm() + 1e-300))

    assert abs(float(loss) - ref_loss) < 1e-3 * abs(ref_loss)
    assert rel(out.detach().double(), ref_out) <= 1.25 * rel(ac_out, ref_out)
    num_o = num_a = den = 0.0
    ratios = []
    for k, r in ref_g.items():
        eo, ea = rel(ours_g[k], r), rel(ac_g[k], r)
        assert eo <= 2.0 * ea + 5e-3, (k, eo, ea)
        assert abs(float(ours_g[k].norm() / r.norm()) - 1.0) < 0.08, k
        ratios.append(eo / (ea + 1e-12))
        num_o += float((ours_g[k] - r).pow(2).sum())
        num_a += float((ac_g[k] - r).pow(2).sum())
        den += float(r.pow(2).sum())
    assert (num_o / den) ** 0.5 <= 1.25 * (num_a / den) ** 0.5
    assert sorted(ratios)[len(ratios) // 2] <= 1.25                # median per-tensor ratio (measured 0.90 .. 1.04)
