"""The BraTS DynUNet workload (examples/brats2020/brats2020_config.json: plan_launches.BRATS_DYNUNET, batch 2, 4 x 128^3) with
the input gradient, and the routes of its convolutions on a 132-SM H100.  Its launches are plan_launches.dynunet's; the input
gradient adds one, the data gradient of input_block.conv1 into the packed 4(8)-channel input.  tests/test_dynunet_host.py holds
the tables to the library's route query, tests/test_gpu_dynunet_brats_size.py again on the device."""
import dataclasses

import plan_launches as P

BRATS = dataclasses.replace(P.BY_NAME["brats-dynunet"], input_grad=True)


def label(key):
    """a conv's label in the route tables: its state-dict key without ".conv.weight" """
    return key[:-len(".conv.weight")]


def route_table(L, split):
    """{label (".dgrad" for a data gradient): (kind, BN, KC, CTAs per SM)} of the workload's convolutions"""
    return P.route_table(L, BRATS, split, label)


def wgrad_route_table(L, split):
    """{label: (kind, K chunk, BN)} of the workload's weight gradients"""
    return P.wgrad_route_table(L, BRATS, split, label)


# (kind, BN, KC, CTAs per SM) per precision.  In bf16 the top level's 64 -> 64 convs and their data gradients run on the two-CTA
# (BN 64, KC 64) halo kernel, conv1 of the input block (4(8) -> 64) and the data gradient of the top concat conv (128 -> 64) on
# one-CTA halo tiles; split precision takes the per-tap kernel there, at one CTA per SM.  Every other layer routes the same in
# both: per-tap BN 128 tiles from 96 channels down, parity class 2 for the kernel-2 transposed convs, parity class 1 for the
# stride-2 data gradients.
_SAME = {
    "downsamples.0.conv1": ("tap", 128, 64, 1), "downsamples.0.conv2": ("tap", 128, 64, 1),
    "downsamples.1.conv1": ("tap", 128, 64, 1), "downsamples.1.conv2": ("tap", 128, 64, 1),
    "downsamples.2.conv1": ("tap", 128, 64, 1), "downsamples.2.conv2": ("tap", 128, 64, 1),
    "downsamples.3.conv1": ("tap", 128, 64, 1), "downsamples.3.conv2": ("tap", 128, 64, 1),
    "bottleneck.conv1": ("tap", 128, 64, 1), "bottleneck.conv2": ("tap", 128, 64, 1),
    "upsamples.0.transp_conv": ("class2", 64, 64, 1), "upsamples.0.conv_block.conv1": ("tap", 128, 64, 1),
    "upsamples.0.conv_block.conv2": ("tap", 128, 64, 1), "upsamples.1.transp_conv": ("class2", 64, 64, 1),
    "upsamples.1.conv_block.conv1": ("tap", 128, 64, 1), "upsamples.1.conv_block.conv2": ("tap", 128, 64, 1),
    "upsamples.2.transp_conv": ("class2", 64, 64, 1), "upsamples.2.conv_block.conv1": ("tap", 128, 64, 1),
    "upsamples.2.conv_block.conv2": ("tap", 128, 64, 1), "upsamples.3.transp_conv": ("class2", 64, 64, 1),
    "upsamples.3.conv_block.conv1": ("tap", 128, 64, 1), "upsamples.3.conv_block.conv2": ("tap", 128, 64, 1),
    "upsamples.4.transp_conv": ("class2", 64, 64, 1), "upsamples.4.conv_block.conv1": ("tap", 64, 64, 1),
    "upsamples.4.transp_conv.dgrad": ("tap", 128, 64, 1),
    "upsamples.3.conv_block.conv2.dgrad": ("tap", 128, 64, 1), "upsamples.3.conv_block.conv1.dgrad": ("tap", 128, 64, 1),
    "upsamples.3.transp_conv.dgrad": ("tap", 128, 64, 1),
    "upsamples.2.conv_block.conv2.dgrad": ("tap", 128, 64, 1), "upsamples.2.conv_block.conv1.dgrad": ("tap", 128, 64, 1),
    "upsamples.2.transp_conv.dgrad": ("tap", 128, 64, 1),
    "upsamples.1.conv_block.conv2.dgrad": ("tap", 128, 64, 1), "upsamples.1.conv_block.conv1.dgrad": ("tap", 128, 64, 1),
    "upsamples.1.transp_conv.dgrad": ("tap", 128, 64, 1),
    "upsamples.0.conv_block.conv2.dgrad": ("tap", 128, 64, 1), "upsamples.0.conv_block.conv1.dgrad": ("tap", 128, 64, 1),
    "upsamples.0.transp_conv.dgrad": ("tap", 128, 64, 1),
    "bottleneck.conv2.dgrad": ("tap", 128, 64, 1), "bottleneck.conv1.dgrad": ("class1", 64, 64, 1),
    "downsamples.3.conv2.dgrad": ("tap", 128, 64, 1), "downsamples.3.conv1.dgrad": ("class1", 64, 64, 1),
    "downsamples.2.conv2.dgrad": ("tap", 128, 64, 1), "downsamples.2.conv1.dgrad": ("class1", 64, 64, 1),
    "downsamples.1.conv2.dgrad": ("tap", 128, 64, 1), "downsamples.1.conv1.dgrad": ("class1", 64, 64, 1),
    "downsamples.0.conv2.dgrad": ("tap", 128, 64, 1), "downsamples.0.conv1.dgrad": ("class1", 64, 64, 1),
    "input_block.conv1.dgrad": ("tap", 16, 64, 2),
}
BRATS_ROUTES = {
    "bf16": dict(_SAME, **{
        "input_block.conv1": ("halo", 64, 16, 1), "input_block.conv2": ("halo", 64, 64, 2),
        "upsamples.4.conv_block.conv2": ("halo", 64, 64, 2), "upsamples.4.conv_block.conv2.dgrad": ("halo", 64, 64, 2),
        "upsamples.4.conv_block.conv1.dgrad": ("halo", 128, 64, 1), "input_block.conv2.dgrad": ("halo", 64, 64, 2),
    }),
    "split": dict(_SAME, **{
        "input_block.conv1": ("tap", 64, 16, 1), "input_block.conv2": ("tap", 64, 64, 1),
        "upsamples.4.conv_block.conv2": ("tap", 64, 64, 1), "upsamples.4.conv_block.conv2.dgrad": ("tap", 64, 64, 1),
        "upsamples.4.conv_block.conv1.dgrad": ("tap", 128, 64, 1), "input_block.conv2.dgrad": ("tap", 64, 64, 1),
    }),
}

# (kind, K chunk, BN) per precision: per-tap, K chunks of 64 and BN 128 from 96 output channels down (the 64-channel top level:
# BN 64; the 4(8)-channel input block conv1: K chunk 16).  In bf16 the 64 -> 64 convs of the top level run on halo tiles.
_WSAME = {
    "upsamples.4.conv_block.conv1": ("tap", 64, 64), "upsamples.4.transp_conv": ("tap", 64, 128),
    "upsamples.3.conv_block.conv2": ("tap", 64, 128), "upsamples.3.conv_block.conv1": ("tap", 64, 128),
    "upsamples.3.transp_conv": ("tap", 64, 128), "upsamples.2.conv_block.conv2": ("tap", 64, 128),
    "upsamples.2.conv_block.conv1": ("tap", 64, 128), "upsamples.2.transp_conv": ("tap", 64, 128),
    "upsamples.1.conv_block.conv2": ("tap", 64, 128), "upsamples.1.conv_block.conv1": ("tap", 64, 128),
    "upsamples.1.transp_conv": ("tap", 64, 128), "upsamples.0.conv_block.conv2": ("tap", 64, 128),
    "upsamples.0.conv_block.conv1": ("tap", 64, 128), "upsamples.0.transp_conv": ("tap", 64, 128),
    "bottleneck.conv2": ("tap", 64, 128), "bottleneck.conv1": ("tap", 64, 128),
    "downsamples.3.conv2": ("tap", 64, 128), "downsamples.3.conv1": ("tap", 64, 128),
    "downsamples.2.conv2": ("tap", 64, 128), "downsamples.2.conv1": ("tap", 64, 128),
    "downsamples.1.conv2": ("tap", 64, 128), "downsamples.1.conv1": ("tap", 64, 128),
    "downsamples.0.conv2": ("tap", 64, 128), "downsamples.0.conv1": ("tap", 64, 128),
    "input_block.conv1": ("tap", 16, 64),
}
BRATS_WGRAD_ROUTES = {
    "bf16": dict(_WSAME, **{"upsamples.4.conv_block.conv2": ("halo", 64, 64), "input_block.conv2": ("halo", 64, 64)}),
    "split": dict(_WSAME, **{"upsamples.4.conv_block.conv2": ("tap", 64, 64), "input_block.conv2": ("tap", 64, 64)}),
}
