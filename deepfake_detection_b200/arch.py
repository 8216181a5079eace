"""Architecture descriptions (host-side only) for the models on the hot path.

A *spec* is a plain description of the layer graph — channel counts, kernel sizes, strides and the
reference's parameter names — from which (a) the native engine lays out its HBM arenas and kernel
plan and (b) the CPU oracle (`oracle/model.py`) builds the same network out of torch fp32 ops.

This file restates the reference's arch-string decoder and stage builder for the variants that
BASELINE.json names; it builds no modules and owns no tensors.
  * EfficientNet arch strings / depth scaling: dfd/timm/models/efficientnet_builder.py:20-191
  * stage builder (stride only on the first block of a stage): efficientnet_builder.py:276-362
  * channel rounding: dfd/timm/models/efficientnet_blocks.py:55-69
  * SE width `make_divisible(block_in_chs * 0.25, 1)`: efficientnet_blocks.py:46-47,98
  * B0/B4 generator (stem 32, head 1280, 7 stages): dfd/timm/models/efficientnet.py:760-803,1078,1132
  * deepfake_v4 (stem 128, head 128, x2.0 / x3.1): efficientnet.py:806-851,1186-1192
  * tf_efficientnet_b0..b7 (+ _ap, _ns): the B0 generator with pad_type='same', efficientnet.py:1265-1530; TF "SAME"
    padding of the stride-2 convolutions, layers/padding.py `pad_same` / layers/conv2d_same.py
  * ResNet-18/50 layout: dfd/timm/models/resnet.py:115-260,280-468,472,523
  * ResNet-26/34/101/152, tv_*, wide_* (base_width 128) and ResNet-D (deep stem, downsample_avg): resnet.py:187,263-277,
    349-439,483-625
  * Xception: dfd/timm/models/xception.py (SeparableConv2d :58-69, Block :72-124, Xception :127-226)
  * SE-ResNets (seresnet18/34/50/101/152): dfd/timm/models/senet.py (SEModule :67-86, SEResNetBottleneck :141-163 with the
    stride on conv1, SEResNetBlock :190-223, SENet :226-396: layer0 7x7 s2 -> BN -> ReLU -> MaxPool2d(3, 2, ceil_mode=True),
    1x1 downsample, `last_linear`; entrypoints :399-461)
  * DenseNet-121/161/169/201: dfd/timm/models/densenet.py (_DenseLayer :37-56, _DenseBlock :59-65, _Transition :62-70,
    DenseNet :73-140, entrypoints :161-215)
"""
import math
import re
from dataclasses import dataclass, field
from typing import List, Optional, Tuple


def make_divisible(v, divisor=8, min_value=None):
    # efficientnet_blocks.py:55-61
    min_value = min_value or divisor
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


def round_channels(channels, multiplier=1.0, divisor=8, channel_min=None):
    # efficientnet_blocks.py:64-69
    if not multiplier:
        return channels
    channels *= multiplier
    return make_divisible(channels, divisor, channel_min)


def conv_out(h, k, s, p):
    return (h + 2 * p - k) // s + 1


def same_pad(i, k, s):
    """TF "SAME" padding of one axis of extent i (layers/padding.py get_same_padding / pad_same):
    (begin, end, output extent). The total is max((ceil(i/s) - 1)*s + k - i, 0); the begin side (top / left) gets half of
    it rounded down. At stride 1 (k odd) and over an odd extent at stride 2 that is the symmetric (k-1)/2; over an even
    extent at stride 2 the begin side gets one element less."""
    out = -(-i // s)
    total = max((out - 1) * s + k - i, 0)
    return total // 2, total - total // 2, out


# ----------------------------------------------------------------------------------------------
# EfficientNet
# ----------------------------------------------------------------------------------------------

@dataclass
class MBBlock:
    """One DepthwiseSeparableConv ('ds') or InvertedResidual ('ir') block."""
    name: str            # 'blocks.<stage>.<idx>'
    kind: str            # 'ds' | 'ir'
    cin: int
    cmid: int            # == cin for 'ds'
    cout: int
    k: int               # depthwise kernel size
    stride: int
    cse: int             # squeeze width (0 = no SE)
    has_residual: bool

    @property
    def pad(self):
        # symmetric PyTorch padding, layers/padding.py:12-14 (pad_type='' never selects Conv2dSame)
        return (self.k - 1) // 2


@dataclass
class EfficientNetSpec:
    arch: str
    in_chans: int
    stem: int
    blocks: List[MBBlock]
    head_in: int
    num_features: int
    num_classes: int
    input_size: Tuple[int, int, int]
    family: str = "efficientnet"
    global_pool: str = "avg"
    pad_type: str = ""           # '' (symmetric (k-1)/2) or 'same' (TF "SAME" on the stride-2 stem and depthwise convs)

    @property
    def pooled_features(self):
        """width of the pooled vector the classifier reads: num_features * feat_mult (adaptive_avgmax_pool.py:17-21)"""
        return self.num_features * pool_feat_mult(self.global_pool)


_EFFNET_ARCH_DEF = [
    "ds_r1_k3_s1_e1_c16_se0.25",
    "ir_r2_k3_s2_e6_c24_se0.25",
    "ir_r2_k5_s2_e6_c40_se0.25",
    "ir_r3_k3_s2_e6_c80_se0.25",
    "ir_r3_k5_s1_e6_c112_se0.25",
    "ir_r4_k5_s2_e6_c192_se0.25",
    "ir_r1_k3_s1_e6_c320_se0.25",
]


def _decode_block_str(s):
    ops = s.split("_")
    kind = ops[0]
    opt = {}
    for op in ops[1:]:
        m = re.split(r"(\d.*)", op)
        if len(m) >= 2:
            opt[m[0]] = m[1]
    return dict(kind=kind, repeat=int(opt["r"]), k=int(opt["k"]), stride=int(opt["s"]),
                exp=float(opt.get("e", 1)), c=int(opt["c"]), se=float(opt["se"]) if "se" in opt else 0.0)


def _efficientnet_spec(arch, channel_multiplier, depth_multiplier, stem_size, num_features,
                       in_chans, num_classes, input_size):
    stem = round_channels(stem_size, channel_multiplier, 8, None)
    blocks = []
    cin = stem
    for si, bs in enumerate(_EFFNET_ARCH_DEF):
        d = _decode_block_str(bs)
        # one block string per stage -> _scale_stage_depth reduces to ceil(r * depth_multiplier)
        repeat = int(math.ceil(d["repeat"] * depth_multiplier))
        for bi in range(repeat):
            stride = d["stride"] if bi == 0 else 1
            cout = round_channels(d["c"], channel_multiplier, 8, None)
            if d["kind"] == "ds":
                cmid = cin
            else:
                cmid = make_divisible(cin * d["exp"])
            cse = make_divisible(cin * d["se"], 1) if d["se"] > 0 else 0
            blocks.append(MBBlock(name="blocks.%d.%d" % (si, bi), kind=d["kind"], cin=cin, cmid=cmid,
                                  cout=cout, k=d["k"], stride=stride, cse=cse,
                                  has_residual=(cin == cout and stride == 1)))
            cin = cout
    return EfficientNetSpec(arch=arch, in_chans=in_chans, stem=stem, blocks=blocks, head_in=cin,
                            num_features=num_features, num_classes=num_classes, input_size=input_size)


# ----------------------------------------------------------------------------------------------
# ResNet
# ----------------------------------------------------------------------------------------------

@dataclass
class ResBlock:
    name: str            # 'layer<l>.<idx>'
    kind: str            # 'basic' | 'bottleneck'
    cin: int
    planes: int
    cout: int
    stride: int
    downsample: bool     # 1x1 conv (stride) + BN on the identity path
    width: int           # bottleneck width int(planes * base_width / 64), resnet.py:187 (== planes for a BasicBlock)
    avg_down: bool = False   # ResNet-D shortcut: AvgPool2d(2, stride, ceil_mode, count_include_pad=False) -> 1x1 conv -> BN
    cse: int = 0             # SENet: squeeze width cout // reduction of the block's SEModule (0: no SE)


@dataclass
class ResNetSpec:
    arch: str
    in_chans: int
    stem: int
    blocks: List[ResBlock]
    num_features: int
    num_classes: int
    input_size: Tuple[int, int, int]
    family: str = "resnet"
    global_pool: str = "avg"
    stem_type: str = ""          # '' (7x7 conv) or 'deep' (3x3 s2 -> 3x3 -> 3x3 of stem_width, stem_width, 64), resnet.py:365-379
    stem_width: int = 32
    # SE-ResNet (senet.py): an SEModule in every block, the bottleneck's stride on its 1x1 conv1, the stem pool
    # MaxPool2d(3, 2, ceil_mode=True) without padding, and the SENet key names (layer0.*, se_module.*, last_linear)
    se_reduction: int = 0
    stride_in_1x1: bool = False
    stem_pool: str = "p1"        # 'p1' (3x3 s2 padding 1) or 'ceil' (3x3 s2 padding 0, ceil mode)
    naming: str = "resnet"       # 'resnet' or 'senet'

    @property
    def pooled_features(self):
        return self.num_features * pool_feat_mult(self.global_pool)

    @property
    def stem_conv(self):
        return "layer0.conv1" if self.naming == "senet" else "conv1"

    @property
    def stem_bn(self):
        return "layer0.bn1" if self.naming == "senet" else "bn1"

    @property
    def cls_name(self):
        return "last_linear" if self.naming == "senet" else "fc"


def _resnet_spec(arch, kind, layers, in_chans, num_classes, input_size, base_width=64, stem_type="", avg_down=False):
    exp = 4 if kind == "bottleneck" else 1
    blocks = []
    cin = 64
    for li, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
        for bi in range(n):
            stride = 2 if (bi == 0 and li > 0) else 1
            cout = planes * exp
            blocks.append(ResBlock(name="layer%d.%d" % (li + 1, bi), kind=kind, cin=cin, planes=planes,
                                   cout=cout, stride=stride,
                                   downsample=(bi == 0 and (stride != 1 or cin != cout)),
                                   width=int(math.floor(planes * (base_width / 64))), avg_down=avg_down))
            cin = cout
    return ResNetSpec(arch=arch, in_chans=in_chans, stem=64, blocks=blocks, num_features=cin,
                      num_classes=num_classes, input_size=input_size, stem_type=stem_type)


def _senet_spec(arch, in_chans, num_classes):
    """SENet(block, layers, groups=1, reduction=16, inplanes=64, input_3x3=False, downsample_kernel_size=1,
    downsample_padding=0) of the seresnet* entrypoints (senet.py:399-461)"""
    kind, layers = _SENET_DEFS[arch]
    spec = _resnet_spec(arch, kind, layers, in_chans, num_classes, (3, 224, 224))
    for b in spec.blocks:
        b.cse = b.cout // 16
    spec.se_reduction, spec.stride_in_1x1, spec.stem_pool, spec.naming = 16, kind == "bottleneck", "ceil", "senet"
    return spec


def stem_pool_out(h, stem_pool):
    """extent after the ResNet stem's max-pool: 3x3 s2 p1, or SENet's 3x3 s2 p0 ceil mode (torch's pooling_output_shape)"""
    if stem_pool != "ceil":
        return conv_out(h, 3, 2, 1)
    o = (h - 3 + 1) // 2 + 1
    return o - 1 if (o - 1) * 2 >= h else o


# ----------------------------------------------------------------------------------------------
# Xception
# ----------------------------------------------------------------------------------------------

@dataclass
class XBlock:
    """One Xception `Block` (xception.py:72-124): separable convolutions, each followed by a BatchNorm, a max-pool 3x3 s2 p1
    at the end of a strided block and a 1x1 convolution + BN shortcut where the shape changes."""
    name: str            # 'block<i>'
    cin: int
    cout: int
    stride: int
    start_with_relu: bool
    seps: List[Tuple[int, int, int]]     # (rep index of the SeparableConv2d, cin, cout); its BN is at rep index + 1

    @property
    def skip(self):
        return self.cout != self.cin or self.stride != 1


@dataclass
class XceptionSpec:
    arch: str
    in_chans: int
    blocks: List[XBlock]
    num_features: int
    num_classes: int
    input_size: Tuple[int, int, int]
    family: str = "xception"
    global_pool: str = "avg"

    @property
    def pooled_features(self):
        return self.num_features * pool_feat_mult(self.global_pool)


def _xblock(i, cin, cout, reps, stride, start_with_relu=True, grow_first=True):
    """rep indices count the ReLU modules (xception.py:89-110): every separable convolution follows a ReLU, except the
    first one of a block that does not start with a ReLU (block1)"""
    chans = [(cin, cout)] + [(cout, cout)] * (reps - 1) if grow_first else [(cin, cin)] * (reps - 1) + [(cin, cout)]
    first = 1 if start_with_relu else 0
    seps = [(first + 3 * j, ci, co) for j, (ci, co) in enumerate(chans)]
    return XBlock("block%d" % i, cin, cout, stride, start_with_relu, seps)


def _xception_spec(arch, in_chans, num_classes):
    blocks = [_xblock(1, 64, 128, 2, 2, start_with_relu=False), _xblock(2, 128, 256, 2, 2), _xblock(3, 256, 728, 2, 2)]
    blocks += [_xblock(i, 728, 728, 3, 1) for i in range(4, 12)]
    blocks.append(_xblock(12, 728, 1024, 2, 2, grow_first=False))
    return XceptionSpec(arch=arch, in_chans=in_chans, blocks=blocks, num_features=2048, num_classes=num_classes,
                        input_size=(3, 299, 299))


def xception_extents(H, W):
    """feature-map extents of Xception at input H x W: [(h, w)] after conv1, conv2 and every block (xception.py:183-200):
    3x3 s2 p0, 3x3 p0, then (h - 1) // 2 + 1 per strided block (max-pool 3x3 s2 p1 and the 1x1 s2 shortcut agree)"""
    h, w = conv_out(H, 3, 2, 0), conv_out(W, 3, 2, 0)
    out = [(h, w)]
    h, w = conv_out(h, 3, 1, 0), conv_out(w, 3, 1, 0)
    out.append((h, w))
    for b in _xception_spec("xception", 3, 2).blocks:
        if b.stride != 1:
            h, w = conv_out(h, 3, 2, 1), conv_out(w, 3, 2, 1)
        out.append((h, w))
    return out


# ----------------------------------------------------------------------------------------------
# DenseNet
# ----------------------------------------------------------------------------------------------

@dataclass
class DenseNetSpec:
    """DenseNet-BC (densenet.py:73-140): stem conv0 7x7 s2 -> norm0 -> relu -> max-pool 3x3 s2 p1, dense blocks of layers
    (norm1, relu, 1x1 conv1 to bn_size * k, norm2, relu, 3x3 conv2 to k, concatenated), transitions (norm, relu, 1x1 conv
    halving the width, 2x2 average pool) between them, norm5 and the classifier."""
    arch: str
    in_chans: int
    growth: int
    init_features: int
    block_config: Tuple[int, ...]
    num_classes: int
    input_size: Tuple[int, int, int] = (3, 224, 224)
    bn_size: int = 4
    family: str = "densenet"
    global_pool: str = "avg"

    @property
    def block_widths(self):
        """[(input width C0, final width)] of every dense block"""
        out, c = [], self.init_features
        for n in self.block_config:
            out.append((c, c + n * self.growth))
            c = (c + n * self.growth) // 2
        return out

    @property
    def num_features(self):
        return self.block_widths[-1][1]

    @property
    def pooled_features(self):
        return self.num_features * pool_feat_mult(self.global_pool)


# arch -> (growth k, init features, block config), densenet.py:161-215
_DENSENET_DEFS = {
    "densenet121": (32, 64, (6, 12, 24, 16)),
    "densenet169": (32, 64, (6, 12, 32, 32)),
    "densenet201": (32, 64, (6, 12, 48, 32)),
    "densenet161": (48, 96, (6, 12, 36, 24)),
}
DENSENET_ARCHS = tuple(_DENSENET_DEFS)


def densenet_extents(H, W):
    """feature-map extents of a DenseNet at input H x W: [(h, w)] of the stem conv, then of every dense block (the stem
    pool 3x3 s2 p1, then a floor-mode 2x2 average pool per transition)"""
    h, w = conv_out(H, 7, 2, 3), conv_out(W, 7, 2, 3)
    out = [(h, w)]
    h, w = conv_out(h, 3, 2, 1), conv_out(w, 3, 2, 1)
    out.append((h, w))
    for _ in range(3):
        h, w = h // 2, w // 2
        out.append((h, w))
    return out


# ----------------------------------------------------------------------------------------------
# registry of the variants on the hot path
# ----------------------------------------------------------------------------------------------

GLOBAL_POOL_TYPES = ("avg", "max", "avgmax", "catavgmax")


def pool_feat_mult(pool_type):
    return 2 if pool_type == "catavgmax" else 1


def get_spec(arch, num_classes=2, in_chans=3, global_pool="avg"):
    """`global_pool`: the SelectAdaptivePool2d type behind the last feature map (efficientnet.py:297-300,
    resnet.py:407-409); 'catavgmax' doubles the classifier input."""
    if global_pool not in GLOBAL_POOL_TYPES:
        raise ValueError("Invalid pool type: %s" % (global_pool,))      # adaptive_avgmax_pool.py:82-84
    spec = _base_spec(arch, num_classes, in_chans)
    spec.global_pool = global_pool
    return spec


def _base_spec(arch, num_classes, in_chans):
    if arch == "efficientnet_b0":
        return _efficientnet_spec(arch, 1.0, 1.0, 32, 1280, in_chans, num_classes, (3, 224, 224))
    if arch == "efficientnet_b4":
        return _efficientnet_spec(arch, 1.4, 1.8, 32, round_channels(1280, 1.4, 8, None), in_chans,
                                  num_classes, (3, 380, 380))
    if arch == "efficientnet_deepfake_v4":
        # efficientnet.py:806-851: stem_size=128, num_features=round_channels(128, 2.0)
        return _efficientnet_spec(arch, 2.0, 3.1, 128, round_channels(128, 2.0, 8, None), in_chans,
                                  num_classes, (in_chans, 600, 600))
    if arch in TF_ARCHS:
        cm, dm, res = _TF_SCALING[int(arch[len("tf_efficientnet_b")])]
        spec = _efficientnet_spec(arch, cm, dm, 32, round_channels(1280, cm, 8, None), in_chans, num_classes, (3, res, res))
        spec.pad_type = "same"
        return spec
    if arch == "resnet18":
        return _resnet_spec(arch, "basic", (2, 2, 2, 2), in_chans, num_classes, (3, 224, 224))
    if arch == "resnet50":
        return _resnet_spec(arch, "bottleneck", (3, 4, 6, 3), in_chans, num_classes, (3, 224, 224))
    if arch in RESNET_ARCHS:
        kind, layers, base_width, deep = _RESNET_DEFS[arch]
        return _resnet_spec(arch, kind, layers, in_chans, num_classes, (3, 224, 224), base_width=base_width,
                            stem_type="deep" if deep else "", avg_down=deep)
    if arch in XCEPTION_ARCHS:
        return _xception_spec(arch, in_chans, num_classes)
    if arch in SENET_ARCHS:
        return _senet_spec(arch, in_chans, num_classes)
    if arch in DENSENET_ARCHS:
        k, c0, cfg = _DENSENET_DEFS[arch]
        return DenseNetSpec(arch=arch, in_chans=in_chans, growth=k, init_features=c0, block_config=cfg,
                            num_classes=num_classes)
    raise ValueError("arch %r is not on the native hot path (see SURVEY.md section 8)" % (arch,))


SUPPORTED_ARCHS = ("efficientnet_b0", "efficientnet_b4", "efficientnet_deepfake_v4", "resnet18", "resnet50")

# The rest of the dense ResNet registry (resnet.py:483-625): arch -> (block, layers, base_width, ResNet-D). ResNet-D is
# stem_type='deep', stem_width=32, avg_down=True (resnet26d, resnet50d); base_width=128 doubles the bottleneck width
# (wide_*). tv_* differ from resnet34 / resnet50 only in their default_cfg.
_RESNET_DEFS = {
    "resnet26": ("bottleneck", (2, 2, 2, 2), 64, False),
    "resnet34": ("basic", (3, 4, 6, 3), 64, False),
    "resnet101": ("bottleneck", (3, 4, 23, 3), 64, False),
    "resnet152": ("bottleneck", (3, 8, 36, 3), 64, False),
    "tv_resnet34": ("basic", (3, 4, 6, 3), 64, False),
    "tv_resnet50": ("bottleneck", (3, 4, 6, 3), 64, False),
    "wide_resnet50_2": ("bottleneck", (3, 4, 6, 3), 128, False),
    "wide_resnet101_2": ("bottleneck", (3, 4, 23, 3), 128, False),
    "resnet26d": ("bottleneck", (2, 2, 2, 2), 64, True),
    "resnet50d": ("bottleneck", (3, 4, 6, 3), 64, True),
}
RESNET_ARCHS = tuple(_RESNET_DEFS)

XCEPTION_ARCHS = ("xception",)      # xception.py:229-237

# SE-ResNets (senet.py:399-461): arch -> (block, layers). SE-ResNeXt and senet154 (grouped 3x3 convolutions) are not here.
_SENET_DEFS = {
    "seresnet18": ("basic", (2, 2, 2, 2)),
    "seresnet34": ("basic", (3, 4, 6, 3)),
    "seresnet50": ("bottleneck", (3, 4, 6, 3)),
    "seresnet101": ("bottleneck", (3, 4, 23, 3)),
    "seresnet152": ("bottleneck", (3, 8, 36, 3)),
}
SENET_ARCHS = tuple(_SENET_DEFS)

# TensorFlow-ported EfficientNets (efficientnet.py:1265-1530): the B0 generator with TF "SAME" padding and BatchNorm eps 1e-3.
# _ap (AdvProp) and _ns (Noisy Student) share the plain variant's layers; only their default_cfg differs (models.py).
# size -> (channel multiplier, depth multiplier, default resolution), efficientnet.py:112-195,1268-1350
_TF_SCALING = {0: (1.0, 1.0, 224), 1: (1.0, 1.1, 240), 2: (1.1, 1.2, 260), 3: (1.2, 1.4, 300),
               4: (1.4, 1.8, 380), 5: (1.6, 2.2, 456), 6: (1.8, 2.6, 528), 7: (2.0, 3.1, 600)}
TF_ARCHS = tuple("tf_efficientnet_b%d%s" % (i, suf) for suf in ("", "_ap", "_ns") for i in range(8))
# default_cfg pool_size / crop_pct per size (efficientnet.py:112-195)
TF_POOL_CROP = {0: ((7, 7), 0.875), 1: ((8, 8), 0.882), 2: ((9, 9), 0.890), 3: ((10, 10), 0.904),
                4: ((12, 12), 0.922), 5: ((15, 15), 0.934), 6: ((17, 17), 0.942), 7: ((19, 19), 0.949)}


def conv_pads(spec, H, W):
    """The padded convolutions of an EfficientNet spec at input H x W, in forward order: [(layer, k, stride, h, w,
    pad_top, pad_left, ho, wo)] for 'conv_stem' and every '<block>.conv_dw'. pad_type '' pads (k-1)/2 on every side;
    'same' pads as TF "SAME" (same_pad) per axis. The output extents agree either way."""
    out = []

    def add(name, k, s, h, w):
        if spec.pad_type == "same":
            pt, _, ho = same_pad(h, k, s)
            pl, _, wo = same_pad(w, k, s)
        else:
            pt = pl = (k - 1) // 2
            ho, wo = conv_out(h, k, s, pt), conv_out(w, k, s, pl)
        out.append((name, k, s, h, w, pt, pl, ho, wo))
        return ho, wo

    h, w = add("conv_stem", 3, 2, H, W)
    for b in spec.blocks:
        h, w = add(b.name + ".conv_dw", b.k, b.stride, h, w)
    return out


# ----------------------------------------------------------------------------------------------
# parameter / buffer naming in the reference's state_dict order
# ----------------------------------------------------------------------------------------------

def _bn_entries(prefix, c):
    return [(prefix + ".weight", (c,), "bn_w"), (prefix + ".bias", (c,), "bn_b"),
            (prefix + ".running_mean", (c,), "bn_rm"), (prefix + ".running_var", (c,), "bn_rv"),
            (prefix + ".num_batches_tracked", (), "bn_nbt")]


def _sep_entries(prefix, cin, cout):
    """SeparableConv2d (xception.py:58-69): depthwise 3x3 `conv1`, then 1x1 `pointwise`, neither with a bias"""
    return [(prefix + ".conv1.weight", (cin, 1, 3, 3), "dw_w"), (prefix + ".pointwise.weight", (cout, cin, 1, 1), "conv_w")]


def state_entries(spec):
    """[(name, shape, role)] in the reference's `state_dict()` order (params and buffers interleaved).

    role in {'conv_w', 'dw_w', 'bn_w', 'bn_b', 'bn_rm', 'bn_rv', 'bn_nbt', 'se_w', 'se_b', 'fc_w', 'fc_b'}.
    """
    out = []
    if spec.family == "efficientnet":
        out.append(("conv_stem.weight", (spec.stem, spec.in_chans, 3, 3), "conv_w"))
        out += _bn_entries("bn1", spec.stem)
        for b in spec.blocks:
            p = b.name
            if b.kind == "ir":
                out.append((p + ".conv_pw.weight", (b.cmid, b.cin, 1, 1), "conv_w"))
                out += _bn_entries(p + ".bn1", b.cmid)
                out.append((p + ".conv_dw.weight", (b.cmid, 1, b.k, b.k), "dw_w"))
                out += _bn_entries(p + ".bn2", b.cmid)
            else:
                out.append((p + ".conv_dw.weight", (b.cmid, 1, b.k, b.k), "dw_w"))
                out += _bn_entries(p + ".bn1", b.cmid)
            if b.cse:
                out.append((p + ".se.conv_reduce.weight", (b.cse, b.cmid, 1, 1), "se_w"))
                out.append((p + ".se.conv_reduce.bias", (b.cse,), "se_b"))
                out.append((p + ".se.conv_expand.weight", (b.cmid, b.cse, 1, 1), "se_w"))
                out.append((p + ".se.conv_expand.bias", (b.cmid,), "se_b"))
            if b.kind == "ir":
                out.append((p + ".conv_pwl.weight", (b.cout, b.cmid, 1, 1), "conv_w"))
                out += _bn_entries(p + ".bn3", b.cout)
            else:
                out.append((p + ".conv_pw.weight", (b.cout, b.cmid, 1, 1), "conv_w"))
                out += _bn_entries(p + ".bn2", b.cout)
        out.append(("conv_head.weight", (spec.num_features, spec.head_in, 1, 1), "conv_w"))
        out += _bn_entries("bn2", spec.num_features)
        out.append(("classifier.weight", (spec.num_classes, spec.pooled_features), "fc_w"))
        out.append(("classifier.bias", (spec.num_classes,), "fc_b"))
    elif spec.family == "densenet":
        c0, k = spec.init_features, spec.growth
        out.append(("features.conv0.weight", (c0, spec.in_chans, 7, 7), "conv_w"))
        out += _bn_entries("features.norm0", c0)
        for b, (cin, cend) in enumerate(spec.block_widths):
            for l in range(spec.block_config[b]):
                p = "features.denseblock%d.denselayer%d" % (b + 1, l + 1)
                c = cin + l * k
                out += _bn_entries(p + ".norm1", c)
                out.append((p + ".conv1.weight", (spec.bn_size * k, c, 1, 1), "conv_w"))
                out += _bn_entries(p + ".norm2", spec.bn_size * k)
                out.append((p + ".conv2.weight", (k, spec.bn_size * k, 3, 3), "conv_w"))
            if b + 1 < len(spec.block_config):
                p = "features.transition%d" % (b + 1)
                out += _bn_entries(p + ".norm", cend)
                out.append((p + ".conv.weight", (cend // 2, cend, 1, 1), "conv_w"))
        out += _bn_entries("features.norm5", spec.num_features)
        out.append(("classifier.weight", (spec.num_classes, spec.pooled_features), "fc_w"))
        out.append(("classifier.bias", (spec.num_classes,), "fc_b"))
    elif spec.family == "xception":
        out.append(("conv1.weight", (32, spec.in_chans, 3, 3), "conv_w"))
        out += _bn_entries("bn1", 32)
        out.append(("conv2.weight", (64, 32, 3, 3), "conv_w"))
        out += _bn_entries("bn2", 64)
        for b in spec.blocks:
            p = b.name
            if b.skip:      # registered before `rep` (xception.py:75-80)
                out.append((p + ".skip.weight", (b.cout, b.cin, 1, 1), "conv_w"))
                out += _bn_entries(p + ".skipbn", b.cout)
            for r, ci, co in b.seps:
                out += _sep_entries("%s.rep.%d" % (p, r), ci, co)
                out += _bn_entries("%s.rep.%d" % (p, r + 1), co)
        out += _sep_entries("conv3", 1024, 1536)
        out += _bn_entries("bn3", 1536)
        out += _sep_entries("conv4", 1536, spec.num_features)
        out += _bn_entries("bn4", spec.num_features)
        out.append(("fc.weight", (spec.num_classes, spec.pooled_features), "fc_w"))
        out.append(("fc.bias", (spec.num_classes,), "fc_b"))
    else:
        if spec.stem_type == "deep":
            # conv1 = Sequential(conv, bn, relu, conv, bn, relu, conv), resnet.py:370-377
            sw = spec.stem_width
            out.append(("conv1.0.weight", (sw, spec.in_chans, 3, 3), "conv_w"))
            out += _bn_entries("conv1.1", sw)
            out.append(("conv1.3.weight", (sw, sw, 3, 3), "conv_w"))
            out += _bn_entries("conv1.4", sw)
            out.append(("conv1.6.weight", (64, sw, 3, 3), "conv_w"))
        else:
            out.append((spec.stem_conv + ".weight", (64, spec.in_chans, 7, 7), "conv_w"))
        out += _bn_entries(spec.stem_bn, 64)
        for b in spec.blocks:
            p = b.name
            if b.kind == "basic":
                out.append((p + ".conv1.weight", (b.planes, b.cin, 3, 3), "conv_w"))
                out += _bn_entries(p + ".bn1", b.planes)
                out.append((p + ".conv2.weight", (b.cout, b.planes, 3, 3), "conv_w"))
                out += _bn_entries(p + ".bn2", b.cout)
            else:
                out.append((p + ".conv1.weight", (b.width, b.cin, 1, 1), "conv_w"))
                out += _bn_entries(p + ".bn1", b.width)
                out.append((p + ".conv2.weight", (b.width, b.width, 3, 3), "conv_w"))
                out += _bn_entries(p + ".bn2", b.width)
                out.append((p + ".conv3.weight", (b.cout, b.width, 1, 1), "conv_w"))
                out += _bn_entries(p + ".bn3", b.cout)
            if b.cse:
                # SEModule fc1 / fc2: 1x1 convolutions with a bias, registered after the last BN (senet.py:72-76,161,202)
                out.append((p + ".se_module.fc1.weight", (b.cse, b.cout, 1, 1), "se_w"))
                out.append((p + ".se_module.fc1.bias", (b.cse,), "se_b"))
                out.append((p + ".se_module.fc2.weight", (b.cout, b.cse, 1, 1), "se_w"))
                out.append((p + ".se_module.fc2.bias", (b.cout,), "se_b"))
            if b.downsample:
                # downsample_avg puts the pool (nn.Identity at stride 1: no keys) at index 0, resnet.py:263-277
                i = 1 if b.avg_down else 0
                out.append((p + ".downsample.%d.weight" % i, (b.cout, b.cin, 1, 1), "conv_w"))
                out += _bn_entries(p + ".downsample.%d" % (i + 1), b.cout)
        out.append((spec.cls_name + ".weight", (spec.num_classes, spec.pooled_features), "fc_w"))
        out.append((spec.cls_name + ".bias", (spec.num_classes,), "fc_b"))
    return out


def param_entries(spec):
    """[(name, shape, role)] of the learnable tensors, in `named_parameters()` order."""
    return [e for e in state_entries(spec) if e[2] not in ("bn_rm", "bn_rv", "bn_nbt")]


def is_no_decay(name, shape):
    # optim_factory.py:17: 1-D tensors and anything named *.bias get weight_decay = 0
    return len(shape) == 1 or name.endswith(".bias")
