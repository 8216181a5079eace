"""CPU oracle of the TensorFlow-ported EfficientNets (tf_efficientnet_b0..b7, _ap, _ns) - test infrastructure.

The tf_* models are the EfficientNet generator with two differences (dfd/timm/models/efficientnet.py:1265-1530):
  * TF "SAME" padding on every convolution (pad_type='same'). Where the padding can be static (stride 1, odd k) that is the
    usual symmetric (k-1)/2; the 3x3 stride-2 stem and the stride-2 depthwise convolutions pad from the input extent,
    per axis: total = max((ceil(i/s) - 1)*s + k - i, 0), total // 2 before (top / left), the rest after
    (layers/padding.py `pad_same`, layers/conv2d_same.py). Here that is restated as an explicit F.pad in front of an
    unpadded convolution.
  * BatchNorm eps 1e-3.

Everything else - BatchNorm, Swish, squeeze-excite, the 16-bit rounding points of `act_dtype`, losses and the optimizer step
- is oracle/model.py and oracle/train.py unchanged: `train_step` / `validate_step` run those with this forward in place of
theirs for specs with pad_type 'same'.
"""
import contextlib
import math

import torch.nn.functional as F

from oracle import model as OM
from oracle import train as OT

BN_EPS_TF = 1e-3


def same_pads(extent, k, s):
    """(before, after) zero padding of one axis under TF 'SAME'"""
    total = max((math.ceil(extent / s) - 1) * s + k - extent, 0)
    return total // 2, total - total // 2


def conv_same(x, w, stride, groups=1):
    k = w.shape[-1]
    pt, pb = same_pads(x.shape[2], k, stride)
    pl, pr = same_pads(x.shape[3], k, stride)
    return F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, stride=stride, groups=groups)


def _mb_block(x, sd, b, bn, act_dtype, taps, drop_mask=None):
    """oracle/model.py `_mb_block` with the depthwise convolution padded as TF 'SAME'"""
    q = OM.q
    p = b.name
    residual = x
    if b.kind == "ir":
        x = q(F.conv2d(x, sd[p + ".conv_pw.weight"]), act_dtype)
        if taps is not None:
            taps[p + ".conv_pw"] = x
        x = q(OM.swish(OM.batch_norm(x, sd, p + ".bn1", bn)), act_dtype)
        x = q(conv_same(x, sd[p + ".conv_dw.weight"], b.stride, groups=b.cmid), act_dtype)
        if taps is not None:
            taps[p + ".conv_dw"] = x
        x = OM.swish(OM.batch_norm(x, sd, p + ".bn2", bn))
        if b.cse:
            x = OM._squeeze_excite(x, sd, p)
        x = q(x, act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv_pwl.weight"]), act_dtype)
        if taps is not None:
            taps[p + ".conv_pwl"] = x
        x = OM.batch_norm(x, sd, p + ".bn3", bn)
    else:
        x = q(conv_same(x, sd[p + ".conv_dw.weight"], b.stride, groups=b.cmid), act_dtype)
        if taps is not None:
            taps[p + ".conv_dw"] = x
        x = OM.swish(OM.batch_norm(x, sd, p + ".bn1", bn))
        if b.cse:
            x = OM._squeeze_excite(x, sd, p)
        x = q(x, act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv_pw.weight"]), act_dtype)
        if taps is not None:
            taps[p + ".conv_pw"] = x
        x = OM.batch_norm(x, sd, p + ".bn2", bn)
    if b.has_residual:
        if drop_mask is not None and bn.training:
            x = x * drop_mask.view(-1, 1, 1, 1)
        x = x + residual
    x = q(x, act_dtype)
    if taps is not None:
        taps[p + ".out"] = x
    return x


def forward(spec, sd, x, bn=None, act_dtype=None, taps=None, drop_masks=None, dropout_mask=None):
    """oracle/model.py `efficientnet_forward` with the stem and the depthwise convolutions padded as TF 'SAME'"""
    assert spec.family == "efficientnet" and spec.pad_type == "same", spec.arch
    bn = bn or OM.BNState(eps=BN_EPS_TF)
    q = OM.q
    x = q(x, act_dtype, grad_too=False)
    x = q(conv_same(x, sd["conv_stem.weight"], 2), act_dtype)
    if taps is not None:
        taps["conv_stem"] = x
    x = q(OM.swish(OM.batch_norm(x, sd, "bn1", bn)), act_dtype)
    if taps is not None:
        taps["stem.out"] = x
    for b in spec.blocks:
        x = _mb_block(x, sd, b, bn, act_dtype, taps, None if drop_masks is None else drop_masks.get(b.name))
    x = q(F.conv2d(x, sd["conv_head.weight"]), act_dtype)
    if taps is not None:
        taps["conv_head"] = x
    x = OM.swish(OM.batch_norm(x, sd, "bn2", bn))
    x = x.mean((2, 3))
    if taps is not None:
        taps["pooled"] = x
    if dropout_mask is not None and bn.training:
        x = x * dropout_mask
    return F.linear(x, sd["classifier.weight"], sd["classifier.bias"])


@contextlib.contextmanager
def _routed():
    """oracle.train calls oracle.model.forward: send the 'same'-padded specs here while the block runs"""
    orig = OM.forward

    def fwd(spec, *a, **k):
        return (forward if getattr(spec, "pad_type", "") == "same" else orig)(spec, *a, **k)

    OM.forward = fwd
    try:
        yield
    finally:
        OM.forward = orig


def train_step(spec, sd, x, target, opt=None, smoothing=0.0, act_dtype=None, taps=None, bn_momentum=0.1):
    with _routed():
        return OT.train_step(spec, sd, x, target, opt, smoothing=smoothing,
                             bn=OM.BNState(training=True, momentum=bn_momentum, eps=BN_EPS_TF), act_dtype=act_dtype, taps=taps)


def validate_step(spec, sd, x, target, act_dtype=None):
    with _routed():
        return OT.validate_step(spec, sd, x, target, bn_eps=BN_EPS_TF, act_dtype=act_dtype)
