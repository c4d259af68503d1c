"""The C5 inference network (bench.py: 1 channel, 5 levels [1, 2, 2, 4, 4], base_width 48, three 128^3 tiles per forward) and
the route of every forward convolution of its forward-only plan on a 132-SM H100, ``C5_ROUTES``, asserted by
tests/test_conv_routes_host.py and tests/test_gpu_c5_size.py through the library's route query (include/b200unet_diag.h)."""
import re

import bench
import plan_launches as P

C5 = dict(bench.CONFIGS["C5"]["model"])
C5_BATCH = bench.CONFIGS["C5"]["sw_batch"]
C5_ROI = tuple(bench.CONFIGS["C5"]["roi"])
C5_VOLUME = tuple(bench.CONFIGS["C5"]["volume"])
C5_OVERLAP = bench.CONFIGS["C5"]["overlap"]


def route_table(L, split):
    """{label: (kind, BN, KC, kchunks)} of the C5 forward (tests/plan_launches.py) from the library's route query; a label is the
    layer's state-dict name, with "+sample" when the launch adds the block's sample convolution"""
    out = {}
    for l in P.BY_NAME["C5"].launches():
        if l.kernel == "fwd":
            r = P.conv_route(L, l, split)
            out[re.sub(r"(\.conv)?\.weight$", "", l.key) + ("+sample" if l.key2 else "")] = \
                None if r is None else (r["kind"], r["bn"], r["kc"], r["kchunks"])
    return out


# the routes of the C5 forward (3 x 1 x 128^3, base_width 48) on a 132-SM H100, (kind, BN, KC, (K chunks of source 0, of the
# second source)) per precision
C5_ROUTES = {
    "bf16": {
        "encoder.layers.0.blocks.0.conv1": ("halo", 64, 16, (1, 0)),
        "encoder.layers.0.blocks.0.conv2+sample": ("halo", 64, 64, (1, 1)),
        "encoder.downsampling_convolutions.0": ("tap", 64, 64, (1, 0)),
        "encoder.layers.1.blocks.0.conv1": ("halo", 128, 64, (1, 0)),
        "encoder.layers.1.blocks.0.conv2+sample": ("tap", 128, 64, (2, 1)),
        "encoder.layers.1.blocks.1.conv1": ("tap", 128, 64, (2, 0)),
        "encoder.layers.1.blocks.1.conv2": ("tap", 128, 64, (2, 0)),
        "encoder.downsampling_convolutions.1": ("tap", 128, 64, (2, 0)),
        "encoder.layers.2.blocks.0.conv1": ("tap", 128, 64, (2, 0)),
        "encoder.layers.2.blocks.0.conv2+sample": ("tap", 128, 64, (3, 2)),
        "encoder.layers.2.blocks.1.conv1": ("tap", 128, 64, (3, 0)),
        "encoder.layers.2.blocks.1.conv2": ("tap", 128, 64, (3, 0)),
        "encoder.downsampling_convolutions.2": ("tap", 128, 64, (3, 0)),
        "encoder.layers.3.blocks.0.conv1": ("tap", 128, 64, (3, 0)),
        "encoder.layers.3.blocks.0.conv2+sample": ("tap", 128, 64, (6, 3)),
        "encoder.layers.3.blocks.1.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.1.conv2": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.2.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.2.conv2": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.3.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.3.conv2": ("tap", 128, 64, (6, 0)),
        "encoder.downsampling_convolutions.3": ("tap", 128, 64, (6, 0)),
        "encoder.layers.4.blocks.0.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.4.blocks.0.conv2+sample": ("tap", 128, 64, (12, 6)),
        "encoder.layers.4.blocks.1.conv1": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.1.conv2": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.2.conv1": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.2.conv2": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.3.conv1": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.3.conv2": ("tap", 128, 64, (12, 0)),
        "decoder.layers.0.blocks.0.conv1": ("tap", 128, 64, (12, 0)),
        "decoder.layers.0.blocks.0.conv2": ("tap", 128, 64, (12, 0)),
        "decoder.pre_upsampling_blocks.0": ("tap", 128, 64, (12, 0)),
        "decoder.layers.1.blocks.0.conv1": ("tap", 128, 64, (12, 0)),
        "decoder.layers.1.blocks.0.conv2": ("tap", 128, 64, (12, 0)),
        "decoder.pre_upsampling_blocks.1": ("tap", 128, 64, (12, 0)),
        "decoder.layers.2.blocks.0.conv1": ("tap", 128, 64, (6, 0)),
        "decoder.layers.2.blocks.0.conv2": ("tap", 128, 64, (6, 0)),
        "decoder.pre_upsampling_blocks.2": ("tap", 128, 64, (6, 0)),
        "decoder.layers.3.blocks.0.conv1": ("tap", 128, 64, (3, 0)),
        "decoder.layers.3.blocks.0.conv2": ("tap", 128, 64, (3, 0)),
        "decoder.pre_upsampling_blocks.3": ("tap", 64, 64, (3, 0)),
        "decoder.layers.4.blocks.0.conv1": ("tap", 64, 64, (2, 0)),
        "decoder.layers.4.blocks.0.conv2+sample": ("halo", 64, 64, (1, 2)),
    },
    # no halo mode for hi + lo operands: the per-tap kernel wherever bf16 takes the halo box
    "split": {
        "encoder.layers.0.blocks.0.conv1": ("tap", 64, 16, (1, 0)),
        "encoder.layers.0.blocks.0.conv2+sample": ("tap", 64, 64, (1, 1)),
        "encoder.downsampling_convolutions.0": ("tap", 64, 64, (1, 0)),
        "encoder.layers.1.blocks.0.conv1": ("tap", 128, 64, (1, 0)),
        "encoder.layers.1.blocks.0.conv2+sample": ("tap", 128, 64, (2, 1)),
        "encoder.layers.1.blocks.1.conv1": ("tap", 128, 64, (2, 0)),
        "encoder.layers.1.blocks.1.conv2": ("tap", 128, 64, (2, 0)),
        "encoder.downsampling_convolutions.1": ("tap", 128, 64, (2, 0)),
        "encoder.layers.2.blocks.0.conv1": ("tap", 128, 64, (2, 0)),
        "encoder.layers.2.blocks.0.conv2+sample": ("tap", 128, 64, (3, 2)),
        "encoder.layers.2.blocks.1.conv1": ("tap", 128, 64, (3, 0)),
        "encoder.layers.2.blocks.1.conv2": ("tap", 128, 64, (3, 0)),
        "encoder.downsampling_convolutions.2": ("tap", 128, 64, (3, 0)),
        "encoder.layers.3.blocks.0.conv1": ("tap", 128, 64, (3, 0)),
        "encoder.layers.3.blocks.0.conv2+sample": ("tap", 128, 64, (6, 3)),
        "encoder.layers.3.blocks.1.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.1.conv2": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.2.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.2.conv2": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.3.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.3.blocks.3.conv2": ("tap", 128, 64, (6, 0)),
        "encoder.downsampling_convolutions.3": ("tap", 128, 64, (6, 0)),
        "encoder.layers.4.blocks.0.conv1": ("tap", 128, 64, (6, 0)),
        "encoder.layers.4.blocks.0.conv2+sample": ("tap", 128, 64, (12, 6)),
        "encoder.layers.4.blocks.1.conv1": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.1.conv2": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.2.conv1": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.2.conv2": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.3.conv1": ("tap", 128, 64, (12, 0)),
        "encoder.layers.4.blocks.3.conv2": ("tap", 128, 64, (12, 0)),
        "decoder.layers.0.blocks.0.conv1": ("tap", 128, 64, (12, 0)),
        "decoder.layers.0.blocks.0.conv2": ("tap", 128, 64, (12, 0)),
        "decoder.pre_upsampling_blocks.0": ("tap", 128, 64, (12, 0)),
        "decoder.layers.1.blocks.0.conv1": ("tap", 128, 64, (12, 0)),
        "decoder.layers.1.blocks.0.conv2": ("tap", 128, 64, (12, 0)),
        "decoder.pre_upsampling_blocks.1": ("tap", 128, 64, (12, 0)),
        "decoder.layers.2.blocks.0.conv1": ("tap", 128, 64, (6, 0)),
        "decoder.layers.2.blocks.0.conv2": ("tap", 128, 64, (6, 0)),
        "decoder.pre_upsampling_blocks.2": ("tap", 128, 64, (6, 0)),
        "decoder.layers.3.blocks.0.conv1": ("tap", 128, 64, (3, 0)),
        "decoder.layers.3.blocks.0.conv2": ("tap", 128, 64, (3, 0)),
        "decoder.pre_upsampling_blocks.3": ("tap", 64, 64, (3, 0)),
        "decoder.layers.4.blocks.0.conv1": ("tap", 64, 64, (2, 0)),
        "decoder.layers.4.blocks.0.conv2+sample": ("tap", 64, 64, (1, 2)),
    },
}
