"""Generate tests/golden/multiclass.npz: the UNMODIFIED reference at class counts the 1..8-output head cannot serve.

Run in the build container (needs /root/reference):   python tests/golden/make_golden_multiclass.py
UNet3D cases run in fp64 on CPU exactly as make_golden.py runs them (train mode, the shared Dropout3d mask, Dice with
sigmoid); inputs and weights are regenerated from the seeds of recipe.py.  Per case: logits subsampled by 8 along each
spatial axis, norms of the logits and of every parameter gradient, Dice, and the full head weight gradient.  The
one-hot / label-map cases run the reference's own unet3d/utils/one_hot.py with 104 labels.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import UNetConfig, make_state_dict, dice_loss  # noqa: E402
from recipe import golden_inputs, dropout_mask  # noqa: E402

SHAPE = (1, 4, 32, 32, 32)
TRAIN_CASES = {"mc24": dict(n_features=4, n_outputs=24, base_width=8), "mc104": dict(n_features=4, n_outputs=104, base_width=8)}
SOFTMAX_CASE = ("mc24_softmax_eval", dict(n_features=4, n_outputs=24, base_width=8, activation="softmax"))
SUB8 = (slice(None), slice(None), slice(None, None, 8), slice(None, None, 8), slice(None, None, 8))
HEAD = "final_convolution.weight"

N_LABELS = 104
ONE_HOT_SHAPE, ONE_HOT_SEED = (1, 1, 6, 7, 8), 21          # label values 0..104
LABEL_MAP_SHAPE, LABEL_MAP_SEED = (N_LABELS, 5, 6, 7), 22
LABEL_MAP_CASES = {"lm104_argmax": dict(threshold=0.5), "lm104_hierarchy": dict(label_hierarchy=True, threshold=0.1)}


def one_hot_input():
    from recipe_prepost import label_map_input
    return label_map_input(ONE_HOT_SHAPE, list(range(N_LABELS + 1)), ONE_HOT_SEED)


def label_map_prediction():
    from recipe_prepost import prediction_input
    return prediction_input(LABEL_MAP_SHAPE, LABEL_MAP_SEED)


def labels():
    return list(range(1, N_LABELS + 1))


def _reference_model(kw):
    from oracle.ref_loader import reference_unet3d
    cfg = UNetConfig(**kw)
    model = reference_unet3d(**kw).double()
    model.load_state_dict(make_state_dict(cfg, seed=0, dtype=torch.float64), strict=True)
    return cfg, model


def run_train_case(kw):
    cfg, model = _reference_model(kw)
    x, t, g3 = golden_inputs(SHAPE, cfg.n_outputs)
    mask = dropout_mask(SHAPE[0], cfg.enc_widths()[0], cfg.dropout, g3)
    model.encoder.layers[0].dropout.forward = lambda inp: inp * mask.to(inp.dtype).view(inp.shape[0], inp.shape[1], 1, 1, 1)
    model.train()
    logits = model(x.double())
    loss = dice_loss(logits, t)
    loss.backward()
    grads = {k: p.grad.detach().numpy() for k, p in model.named_parameters()}
    return logits.detach(), loss.detach(), grads


def main():
    from make_golden_prepost import load_reference_one_hot
    out = {}
    for name, kw in TRAIN_CASES.items():
        logits, loss, grads = run_train_case(kw)
        keys = sorted(grads)
        out[name + "::logits_sub8"] = logits[SUB8].numpy().astype(np.float32)
        out[name + "::logits_norm"] = np.float64(logits.norm())
        out[name + "::dice"] = np.float64(loss)
        out[name + "::grad_keys"] = np.array(keys)
        out[name + "::grad_norms"] = np.array([np.linalg.norm(grads[k]) for k in keys])
        out[name + "::grad_head"] = grads[HEAD].astype(np.float32)
        print(name, "dice", float(loss), "|logits|", float(logits.norm()))
    name, kw = SOFTMAX_CASE
    _, model = _reference_model(kw)
    model.eval()
    x, _, _ = golden_inputs(SHAPE, kw["n_outputs"])
    with torch.no_grad():
        p = model(x.double())
    out[name + "::sub8"] = p[SUB8].numpy().astype(np.float32)
    out[name + "::norm"] = np.float64(p.norm())

    ref, MetaTensor = load_reference_one_hot()
    y = ref.compile_one_hot_encoding(MetaTensor(one_hot_input(), meta={}), n_labels=N_LABELS, labels=None, return_4d=False)
    out["one_hot104"] = np.packbits(torch.as_tensor(y).numpy().astype(np.uint8))
    out["one_hot104_shape"] = np.array(y.shape)
    for lname, lkw in LABEL_MAP_CASES.items():
        lm = ref.convert_one_hot_to_label_map(label_map_prediction(), labels=labels(), **lkw)
        out[lname] = torch.as_tensor(lm).numpy().astype(np.int16)
        print(lname, "labels present", np.unique(out[lname]).size)
    path = os.path.join(HERE, "multiclass.npz")
    np.savez_compressed(path, **out)
    print("->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
