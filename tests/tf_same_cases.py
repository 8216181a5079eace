"""The launches of the TF "SAME" kernels (dfd_stem_im2col_pad, dfd_dwconv_fwd_pad, dfd_dwconv_bwd_pad) in the eight default
tf_efficientnet plans, and the kernel cases the GPU file runs for them. Shared by test_tf_efficientnet_cpu.py (the coverage
contract, no GPU) and test_tf_efficientnet_gpu.py.

The default plans are tf_efficientnet_b0..b7 at their default resolution (default_cfg input_size), in training form, at
PLAN_BATCH images. Each distinct launch is a (kernel, H, W, C, k, stride, pad_top, pad_left) shape. The GPU file runs every
one at CASE_BATCH images: a reduced batch, stated here. The kernels index every image the same way (the batch is the grid's
z extent, or the image-group stride of the fused backward), so the batch changes how many images a CTA walks, not which
pixels, taps or pads it touches; CASE_BATCH = 2 keeps the fp64 references of the 600² B7 layers small, and still gives the
fused backward two images per channel block on its smaller layers.
"""
from deepfake_detection_b200.arch import TF_ARCHS

PLAN_BATCH = 8
CASE_BATCH = 2
NEW_KERNELS = ("dfd_stem_im2col_pad", "dfd_dwconv_fwd_pad", "dfd_dwconv_bwd_pad")
DEFAULT_ARCHS = TF_ARCHS[:8]


def launch_shape(name, args):
    """(kernel, H, W, C, k, stride, pad_top, pad_left) of a planned launch of a new kernel"""
    if name == "dfd_stem_im2col_pad":
        _, _, N, Cin, H, W, k, s, pt, pl, Kp, dt = args
        return (name, H, W, Cin, k, s, pt, pl)
    if name == "dfd_dwconv_fwd_pad":
        H, W, C, k, s, pt, pl = args[6:13]
        return (name, H, W, C, k, s, pt, pl)
    if name == "dfd_dwconv_bwd_pad":
        H, W, C, k, s, pt, pl = args[15:22]
        return (name, H, W, C, k, s, pt, pl)
    raise KeyError(name)


def plan_shapes(arch, batch=PLAN_BATCH, H=None, W=None, **kw):
    """the distinct launch shapes of the new kernels in a plan-only training plan"""
    from deepfake_detection_b200.engine import Engine
    e = Engine(arch, batch, H, W, device="plan-only", **kw)
    out = []
    for _, name, args in e.fwd_ops + e.bwd_ops:
        if name in NEW_KERNELS:
            s = launch_shape(name, args)
            if s not in out:
                out.append(s)
    return out


def default_shapes():
    """{shape: [arch, ...]} over the eight default plans, in plan order"""
    out = {}
    for a in DEFAULT_ARCHS:
        for s in plan_shapes(a):
            out.setdefault(s, []).append(a)
    return out


# The distinct launch shapes of default_shapes(), written out so that collecting the GPU file builds no plan (building the
# eight plans allocates over a gigabyte of host memory); test_tf_efficientnet_cpu.py checks that this list equals the
# harvest. Comment: the sizes whose plans issue the launch.
DEFAULT_CASES = [
    ('dfd_stem_im2col_pad', 224, 224, 3, 3, 2, 0, 0),  # b0
    ('dfd_dwconv_fwd_pad', 112, 112, 96, 3, 2, 0, 0),  # b0
    ('dfd_dwconv_fwd_pad', 56, 56, 144, 5, 2, 1, 1),  # b0
    ('dfd_dwconv_fwd_pad', 28, 28, 240, 3, 2, 0, 0),  # b0
    ('dfd_dwconv_fwd_pad', 14, 14, 672, 5, 2, 1, 1),  # b0
    ('dfd_dwconv_bwd_pad', 14, 14, 672, 5, 2, 1, 1),  # b0
    ('dfd_dwconv_bwd_pad', 28, 28, 240, 3, 2, 0, 0),  # b0
    ('dfd_dwconv_bwd_pad', 56, 56, 144, 5, 2, 1, 1),  # b0
    ('dfd_dwconv_bwd_pad', 112, 112, 96, 3, 2, 0, 0),  # b0
    ('dfd_stem_im2col_pad', 240, 240, 3, 3, 2, 0, 0),  # b1
    ('dfd_dwconv_fwd_pad', 120, 120, 96, 3, 2, 0, 0),  # b1
    ('dfd_dwconv_fwd_pad', 60, 60, 144, 5, 2, 1, 1),  # b1
    ('dfd_dwconv_fwd_pad', 30, 30, 240, 3, 2, 0, 0),  # b1
    ('dfd_dwconv_bwd_pad', 30, 30, 240, 3, 2, 0, 0),  # b1
    ('dfd_dwconv_bwd_pad', 60, 60, 144, 5, 2, 1, 1),  # b1
    ('dfd_dwconv_bwd_pad', 120, 120, 96, 3, 2, 0, 0),  # b1
    ('dfd_stem_im2col_pad', 260, 260, 3, 3, 2, 0, 0),  # b2
    ('dfd_dwconv_fwd_pad', 130, 130, 96, 3, 2, 0, 0),  # b2
    ('dfd_dwconv_bwd_pad', 130, 130, 96, 3, 2, 0, 0),  # b2
    ('dfd_stem_im2col_pad', 300, 300, 3, 3, 2, 0, 0),  # b3
    ('dfd_dwconv_fwd_pad', 150, 150, 144, 3, 2, 0, 0),  # b3
    ('dfd_dwconv_fwd_pad', 38, 38, 288, 3, 2, 0, 0),  # b3
    ('dfd_dwconv_bwd_pad', 38, 38, 288, 3, 2, 0, 0),  # b3
    ('dfd_dwconv_bwd_pad', 150, 150, 144, 3, 2, 0, 0),  # b3
    ('dfd_stem_im2col_pad', 380, 380, 3, 3, 2, 0, 0),  # b4
    ('dfd_dwconv_fwd_pad', 190, 190, 144, 3, 2, 0, 0),  # b4
    ('dfd_dwconv_fwd_pad', 48, 48, 336, 3, 2, 0, 0),  # b4
    ('dfd_dwconv_fwd_pad', 24, 24, 960, 5, 2, 1, 1),  # b4
    ('dfd_dwconv_bwd_pad', 24, 24, 960, 5, 2, 1, 1),  # b4
    ('dfd_dwconv_bwd_pad', 48, 48, 336, 3, 2, 0, 0),  # b4
    ('dfd_dwconv_bwd_pad', 190, 190, 144, 3, 2, 0, 0),  # b4
    ('dfd_stem_im2col_pad', 456, 456, 3, 3, 2, 0, 0),  # b5
    ('dfd_dwconv_fwd_pad', 228, 228, 144, 3, 2, 0, 0),  # b5
    ('dfd_dwconv_fwd_pad', 114, 114, 240, 5, 2, 1, 1),  # b5
    ('dfd_dwconv_bwd_pad', 114, 114, 240, 5, 2, 1, 1),  # b5
    ('dfd_dwconv_bwd_pad', 228, 228, 144, 3, 2, 0, 0),  # b5
    ('dfd_stem_im2col_pad', 528, 528, 3, 3, 2, 0, 0),  # b6
    ('dfd_dwconv_fwd_pad', 264, 264, 192, 3, 2, 0, 0),  # b6
    ('dfd_dwconv_fwd_pad', 132, 132, 240, 5, 2, 1, 1),  # b6
    ('dfd_dwconv_fwd_pad', 66, 66, 432, 3, 2, 0, 0),  # b6
    ('dfd_dwconv_bwd_pad', 66, 66, 432, 3, 2, 0, 0),  # b6
    ('dfd_dwconv_bwd_pad', 132, 132, 240, 5, 2, 1, 1),  # b6
    ('dfd_dwconv_bwd_pad', 264, 264, 192, 3, 2, 0, 0),  # b6
    ('dfd_stem_im2col_pad', 600, 600, 3, 3, 2, 0, 0),  # b7
    ('dfd_dwconv_fwd_pad', 300, 300, 192, 3, 2, 0, 0),  # b7
    ('dfd_dwconv_fwd_pad', 150, 150, 288, 5, 2, 1, 1),  # b7
    ('dfd_dwconv_fwd_pad', 38, 38, 1344, 5, 2, 1, 1),  # b7
    ('dfd_dwconv_bwd_pad', 38, 38, 1344, 5, 2, 1, 1),  # b7
    ('dfd_dwconv_bwd_pad', 150, 150, 288, 5, 2, 1, 1),  # b7
    ('dfd_dwconv_bwd_pad', 300, 300, 192, 3, 2, 0, 0),  # b7
]


# Kernel cases of the GPU file beyond the default plans: non-square inputs whose pads differ between the axes (the
# layers of tf_efficientnet_b0 at 66x96, where H = 33 after the stem is odd and W = 48 even, and an H-even / W-odd layer).
EXTRA_CASES = [
    ("dfd_stem_im2col_pad", 66, 96, 3, 3, 2, 0, 0),         # both axes even: the plain asymmetric stem of a 66x96 input
    ("dfd_dwconv_fwd_pad", 33, 48, 96, 3, 2, 1, 0),         # stage 1 of tf_efficientnet_b0 at 66x96: pad_top != pad_left
    ("dfd_dwconv_bwd_pad", 33, 48, 96, 3, 2, 1, 0),
    ("dfd_dwconv_fwd_pad", 17, 24, 144, 5, 2, 2, 1),        # stage 2 there (k = 5, C = 144: 16-channel-pair lanes)
    ("dfd_dwconv_bwd_pad", 17, 24, 144, 5, 2, 2, 1),
    ("dfd_dwconv_fwd_pad", 28, 27, 240, 3, 2, 0, 1),        # H even, W odd: the other mixed form
    ("dfd_dwconv_bwd_pad", 28, 27, 240, 3, 2, 0, 1),
]
