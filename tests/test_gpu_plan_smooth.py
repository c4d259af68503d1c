"""The whole-network UNet3D and DynUNet plans at activation slope 1 against fp64 autograd of the oracle, at bounds fixed from
the fp64 noise floor (tests/plan_smooth_cases.py): the loss, the logits, every parameter gradient by state-dict key and the
input gradient.  The ReLU plan tests (test_gpu_model.py, test_gpu_dynunet.py, ...) check the activation masks at loose
bounds; these rows check the plan's wiring -- concat slices, skip gradients, dropout scales, residual adds, up-sampling and
ConvT gradients, the head -- tightly enough that an error of a few percent in any one of them fails."""
import pytest
import torch

import plan_smooth_cases as P

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _check(name, got, ref, precision, fails):
    """rel-L2 of the tensor against its bound; in split precision also every logit / dx element against elem * rms(ref).
    Returns the rel-L2 error over the bound."""
    got, ref = got.double().cpu(), ref.double().cpu()
    if got.shape != ref.shape or not bool(torch.isfinite(got).all()):
        fails.append("%s: shape %s vs %s, finite %s" % (name, tuple(got.shape), tuple(ref.shape), bool(torch.isfinite(got).all())))
        return float("inf")
    err, bound = P.rel_l2(got, ref), P.bound_of(name, precision)
    diff = (got - ref).abs()
    i = int(diff.argmax())
    worst = "worst element %s: %.6e vs %.6e" % (tuple(int(v) for v in torch.unravel_index(torch.tensor(i), diff.shape)),
                                                 float(got.flatten()[i]), float(ref.flatten()[i]))
    if not err <= bound:
        fails.append("%s: rel-L2 %.3e > bound %.1e; %s" % (name, err, bound, worst))
    elem = P.BOUNDS[precision]["elem"]
    if elem is not None and name in ("logits", "dx"):
        rms = float(ref.pow(2).mean().sqrt())
        if not float(diff.max()) <= elem * rms:
            fails.append("%s: element error %.3e > %.0e * rms %.3e; %s" % (name, float(diff.max()), elem, rms, worst))
    return err / bound


def _train_step(pkg, model, x, t, input_grad):
    model.zero_grad(set_to_none=True)
    xd = x.to(DEV).requires_grad_(input_grad)
    out = model(xd)
    loss = pkg.DiceLoss(sigmoid=True)(out, t.to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    got = {"logits": out.detach(), "loss": loss.detach().reshape(1)}
    got.update({k: p.grad.detach().clone() for k, p in model.named_parameters()})
    if input_grad:
        got["dx"] = xd.grad.detach().clone()
    return got


@pytest.mark.parametrize("case", P.CASES, ids=lambda c: c.id)
def test_plan_matches_fp64_oracle_at_slope_1(pkg, case):
    sd, x, t, mask = P.inputs(case)
    ref = P.clean_reference(case)
    model = P.model_of(pkg, case).to(DEV)
    model.load_state_dict(sd, strict=True)
    if case.train:
        model.train()
        if mask is not None:
            model.set_dropout_scale(mask)
        got = _train_step(pkg, model, x, t, case.input_grad)
    else:
        model.eval()
        with torch.no_grad():
            got = {"logits": model(x.to(DEV))}
        torch.cuda.synchronize()
    assert sorted(got) == sorted(ref)
    fails = []
    ratios = {k: _check(k, got[k], ref[k], case.precision, fails) for k in ref}
    k = max(ratios, key=ratios.get)
    print("%s [%s]: largest error %s rel-L2 %.3e, bound %.1e (%.0f %% of it)"
          % (case.id, case.precision, k, ratios[k] * P.bound_of(k, case.precision), P.bound_of(k, case.precision), 100 * ratios[k]))
    assert not fails, "%s:\n  %s" % (case.id, "\n  ".join(fails))
    if case.deterministic:
        again = _train_step(pkg, model, x, t, case.input_grad)
        diff = [k for k in got if k != "logits" and k != "loss" and not torch.equal(got[k], again[k])]
        assert not diff, "a deterministic plan must repeat its gradients bit for bit: %r" % diff
