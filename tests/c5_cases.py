"""The C5 inference network (bench.py: 1 channel, 5 levels [1, 2, 2, 4, 4], base_width 48, three 128^3 tiles per forward) and
the convolution launches of the UNet3D plans, restated from plan.cu: build_unet3d.

``unet3d_conv_layers`` lists every convolution launch of a UNet3D plan with its route-query arguments; ``C5_ROUTES`` is the
route of every forward convolution of the C5 forward-only plan on a 132-SM H100, asserted by tests/test_conv_routes_host.py and
tests/test_gpu_c5_size.py through the library's route query (include/b200unet_diag.h)."""
import bench

C5 = dict(bench.CONFIGS["C5"]["model"])
C5_BATCH = bench.CONFIGS["C5"]["sw_batch"]
C5_ROI = tuple(bench.CONFIGS["C5"]["roi"])
C5_VOLUME = tuple(bench.CONFIGS["C5"]["volume"])
C5_OVERLAP = bench.CONFIGS["C5"]["overlap"]


def unet3d_conv_layers(n_features, base_width, dims, encoder_blocks=(1, 2, 2, 4), decoder_blocks=None, train=False):
    """(label, op, cin, cout, output extents, epilogue mode, cin2) of every convolution launch of a UNet3D plan with trilinear
    up-sampling (plan.cu: build_unet3d).  cin is the channel count of the source view (the packed input has its channels padded to
    a multiple of 8), cin2 that of a fused 1x1x1 second source.

    Forward: per residual block conv1 (3x3x3) and conv2 (3x3x3), which adds the block's `sample` 1x1x1 convolution of the block
    input as its second source when the width changes (otherwise the input as a residual); the stride-2 downsampling convolution
    of every level but the last; per decoder stage the blocks at the width the stage receives (the deeper stages read the 2C-channel
    concat buffer), then the `pre_upsampling_blocks` 1x1x1 convolution to the next width.  Training plans add the data gradients
    (build_block_bwd, emit_down_bwd): conv2 and conv1 through the GroupNorm + ReLU backward epilogue (mode 1), the sample
    convolution's, the stride-2 convolution's on parity classes and the pre-up-sampling convolution's."""
    L = len(encoder_blocks)
    decoder_blocks = list(decoder_blocks) if decoder_blocks is not None else [1] * L
    widths = [base_width << k for k in range(L)]
    ext = [tuple(d >> k for d in dims) for k in range(L)]
    out = []

    def block(pre, xc, cin_real, C, k):
        sample = xc if cin_real != C else 0
        out.append((pre + ".conv1", "k3s1", xc, C, ext[k], 0, 0))
        out.append((pre + ".conv2" + ("+sample" if sample else ""), "k3s1", C, C, ext[k], 0, sample))
        if train:
            out.append((pre + ".conv2.dgrad", "k3s1", C, C, ext[k], 1, 0))
            out.append((pre + ".conv1.dgrad", "k3s1", C, xc, ext[k], 1, 0))
            if sample and pre != "encoder.layers.0.blocks.0":
                out.append((pre + ".sample.dgrad", "k1", C, xc, ext[k], 0, 0))

    xc, cin_real = (n_features + 7) // 8 * 8, n_features
    for k in range(L):
        for b in range(encoder_blocks[k]):
            block("encoder.layers.%d.blocks.%d" % (k, b), xc, cin_real, widths[k], k)
            xc = cin_real = widths[k]
        if k + 1 < L:
            out.append(("encoder.downsampling_convolutions.%d" % k, "k3s2", widths[k], widths[k], ext[k + 1], 0, 0))
            if train:
                out.append(("encoder.downsampling_convolutions.%d.dgrad" % k, "class1", widths[k], widths[k], ext[k], 0, 0))
    for i in range(L - 1):
        depth = L - 1 - i
        in_w = widths[depth] if depth == L - 1 else 2 * widths[depth]
        for b in range(decoder_blocks[i]):
            block("decoder.layers.%d.blocks.%d" % (i, b), in_w, in_w, in_w, depth)
        out.append(("decoder.pre_upsampling_blocks.%d" % i, "k1", in_w, widths[depth - 1], ext[depth], 0, 0))
        if train:
            out.append(("decoder.pre_upsampling_blocks.%d.dgrad" % i, "k1", widths[depth - 1], in_w, ext[depth], 0, 0))
    xc = 2 * base_width
    for b in range(decoder_blocks[L - 1]):
        block("decoder.layers.%d.blocks.%d" % (L - 1, b), xc, xc, base_width, 0)
        xc = base_width
    return out


def conv_layers():
    """the forward convolutions of the C5 forward-only plan: batch 3 (sw_batch) of 128^3 tiles"""
    return unet3d_conv_layers(C5["n_features"], C5["base_width"], C5_ROI, C5["encoder_blocks"])


def route_table(L, split):
    """{label: (kind, BN, KC, kchunks)} of the C5 forward from the library's route query"""
    from conv_route_cases import conv_query
    out = {}
    for label, op, ci, co, ext, mode, ci2 in conv_layers():
        r = conv_query(L, op, ci, co, ext, split, mode, ci2, n=C5_BATCH)
        out[label] = None if r is None else (r["kind"], r["bn"], r["kc"], r["kchunks"])
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
