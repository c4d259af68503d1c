"""The C-ABI library: loads, exports every symbol include/b200unet.h declares, and its host-side planner (no GPU
needed: plan_create is pure host logic) reproduces the reference state-dict contract and rejects what it does not
implement with an error code instead of falling back."""
import ctypes as C
import os
import re

import pytest
import torch

from oracle import UNetConfig, unet3d_state_dict_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols(header="b200unet.h"):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200unet_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_exactly_the_declared_symbols(pkg):
    lib = pkg.lib.load_library()
    declared = _declared_symbols()
    assert len(declared) >= 30
    raw = C.CDLL(pkg.lib.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), "missing export: " + name
    assert set(pkg.lib.EXPORTED_SYMBOLS) == set(declared)      # the binding covers the whole header
    assert lib.b200unet_version() >= 100
    assert lib.b200unet_last_error() is not None


def test_library_exports_the_diagnostics_header(pkg):
    """include/b200unet_diag.h is bound by lib._DIAG_SIGS, outside the product surface"""
    pkg.lib.load_library()
    declared = _declared_symbols("b200unet_diag.h")
    raw = C.CDLL(pkg.lib.LIB_PATH)
    assert declared and all(hasattr(raw, name) for name in declared)
    assert set(pkg.lib._DIAG_SIGS) == set(declared)
    assert not set(declared) & set(pkg.lib.EXPORTED_SYMBOLS)


def test_library_is_sm90a_wgmma(pkg):
    """The shipped binary must contain Hopper warpgroup-MMA + TMA SASS."""
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", pkg.lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    assert "HGMMA" in sass and "UTMALDG" in sass and "UTMASTG" in sass
    assert "HMMA." not in sass.replace("HGMMA", "")            # no legacy mma.sync path


def _plan(pkg, n, d, h, w, **kw):
    net = pkg.UNet3D(**kw)
    return net, pkg.models._Plan(net._net_desc(n, d, h, w), torch.device("cpu"))


@pytest.mark.parametrize("kw", [
    dict(n_features=4, n_outputs=3, base_width=8),
    dict(n_features=4, n_outputs=3, base_width=32),
    dict(n_features=1, n_outputs=1, base_width=48, encoder_blocks=[1, 2, 2, 4, 4]),
    dict(n_features=2, n_outputs=2, base_width=16, encoder_blocks=[2, 2, 1], decoder_blocks=[1, 2, 2]),
    dict(n_features=4, n_outputs=3, base_width=8, decoder_mirrors_encoder=True),
])
def test_plan_param_spec_is_reference_state_dict(pkg, kw):
    net, plan = _plan(pkg, 1, 32, 32, 32, **kw)
    okw = {k: v for k, v in kw.items() if k != "decoder_mirrors_encoder"}
    if kw.get("decoder_mirrors_encoder"):
        okw["decoder_blocks"] = [1, 2, 2, 4]
    spec = unet3d_state_dict_spec(UNetConfig(**okw))
    assert plan.param_spec() == spec
    assert [(k, tuple(v.shape)) for k, v in net.state_dict().items()] == spec
    assert plan.ws_bytes > 0


def test_plan_rejects_unsupported_loudly(pkg):
    net = pkg.UNet3D(n_features=4, n_outputs=3, base_width=8)
    with pytest.raises(RuntimeError, match="must be even"):
        pkg.models._Plan(net._net_desc(1, 36, 32, 32), torch.device("cpu"))   # 36 -> 18 -> 9: odd before last level
    net12 = pkg.UNet3D(n_features=4, n_outputs=3, base_width=12)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        pkg.models._Plan(net12._net_desc(1, 32, 32, 32), torch.device("cpu"))


def test_workspace_fits_h100_for_headline_config(pkg):
    _, plan = _plan(pkg, 2, 128, 128, 128, n_features=4, n_outputs=3, base_width=32)
    assert plan.ws_bytes < 40 * 2 ** 30                          # 80 GB HBM3: room for the CUDA context, optimizer and inputs
    _, plan3 = _plan(pkg, 2, 160, 192, 128, n_features=4, n_outputs=3, base_width=32)
    assert plan3.ws_bytes < 60 * 2 ** 30
