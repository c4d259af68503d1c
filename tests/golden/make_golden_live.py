"""Generate tests/golden/live_reference.npz by running the UNMODIFIED reference UNet3D on CPU (fp64).

Needs the reference repository (oracle/ref_loader.py; B200UNET_REFERENCE_ROOT):   python tests/golden/make_golden_live.py
Stores, per case of tests/test_oracle_golden.py::test_oracle_matches_live_reference, the reference's state-dict spec and its
eval-mode logits (every 4th voxel per axis) for seeded weights and input, and the state-dict spec of the model
tests/test_host_logic.py::test_checkpoint_interchange_with_reference loads.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import UNetConfig, make_state_dict  # noqa: E402
from oracle.ref_loader import reference_unet3d  # noqa: E402

LIVE_CASES = [
    (dict(n_features=4, n_outputs=3, base_width=8), (1, 4, 16, 16, 16)),
    (dict(n_features=2, n_outputs=2, base_width=8, encoder_blocks=[1, 1, 2]), (2, 2, 16, 24, 16)),
    (dict(n_features=4, n_outputs=3, base_width=8, use_transposed_convolutions=True), (1, 4, 16, 16, 16)),
]
CHECKPOINT_KW = dict(n_features=4, n_outputs=3, base_width=8)
SUB = (slice(None), slice(None), slice(None, None, 4), slice(None, None, 4), slice(None, None, 4))   # stored logits sample


def main():
    out = {}
    for i, (kw, shape) in enumerate(LIVE_CASES):
        ref = reference_unet3d(**kw).double()
        sd = make_state_dict(UNetConfig(**kw), seed=3, dtype=torch.float64)
        ref.load_state_dict(sd, strict=True)
        ref.eval()
        x = torch.randn(shape, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
        with torch.no_grad():
            out["case%d_logits_sub4" % i] = ref(x)[SUB].numpy()
        out["case%d_keys" % i] = np.array(list(ref.state_dict()))
        out["case%d_shapes" % i] = np.array([str(tuple(v.shape)) for v in ref.state_dict().values()])
    ref = reference_unet3d(**CHECKPOINT_KW)
    out["checkpoint_keys"] = np.array(list(ref.state_dict()))
    out["checkpoint_shapes"] = np.array([str(tuple(v.shape)) for v in ref.state_dict().values()])
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "live_reference.npz"), **out)


if __name__ == "__main__":
    main()
