"""CPU ORACLE — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain torch-fp32 CPU restatement of the reference's train/validate step for every model family the native path runs
(EfficientNet incl. the TF "SAME"-padded ones, ResNet / ResNet-D / Wide ResNet / SE-ResNet, Xception).  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` / `--impl reference` legs may import this package, and only as
the checker / the CPU baseline — never as the thing shipped.  The product path (`deepfake_detection_b200`) must not import
it (tests/test_host_plan.py::test_no_oracle_on_product_path).

Parity pin: the reference has NO tests, golden vectors or fixtures of its own (SURVEY.md section 4/8c), so
this restatement is pinned against outputs of the reference itself: `oracle/mint_goldens.py` and `tools/mint_*_goldens.py`
import the unmodified reference (authoring container only), run it on seeded synthetic weights and inputs, and commit the
results under tests/golden/; tests/test_oracle_vs_reference_goldens.py checks this file against them on CPU, one run per
step fixture of tests/reference_steps.py's CPU_STEPS.

What each function follows (file:line under /root/reference):
  efficientnet_forward : dfd/timm/models/efficientnet.py:320-348
  _mb_block            : dfd/timm/models/efficientnet_blocks.py:177-194 (DS), :314-348 (IR)
  _squeeze_excite      : dfd/timm/models/efficientnet_blocks.py:104-110
  same_pads, conv_same : dfd/timm/models/layers/padding.py `pad_same`, layers/conv2d_same.py (pad_type 'same')
  swish                : dfd/timm/models/layers/activations.py:19-27 (x * sigmoid(x))
  resnet_forward       : dfd/timm/models/resnet.py:450-468, BasicBlock :150-175, Bottleneck :215-246, deep stem :365-377,
                         avg-pool shortcut :263-277; senet.py:291-300 (layer0), :94-114 / :141-163 / :206-223 (blocks)
  _se_module           : dfd/timm/models/senet.py:67-86
  _bn_drop             : dfd/timm/models/layers/drop.py:24-100 (DropBlock2d, DropPath)
  xception_forward     : dfd/timm/models/xception.py:58-124, :183-215
  global_pool          : dfd/timm/models/layers/adaptive_avgmax_pool.py:24-48
  batch norm           : torch.nn.BatchNorm2d semantics (biased var to normalise, unbiased var into
                         running_var, momentum 0.1, eps 1e-5 unless overridden, efficientnet_blocks.py:22-30;
                         eps 1e-3 for the TF EfficientNets, efficientnet.py:1265-1530)
  cross_entropy        : dfd/timm/loss/cross_entropy.py:20-36 and nn.CrossEntropyLoss (train.py:509-520)
  accuracy             : dfd/timm/utils.py:170-186

`act_dtype` (None | torch.bfloat16 | torch.float16): when set, every tensor that the native path stores
in 16-bit (conv outputs, block outputs, SE-gated activations, the network input) is rounded to that type
and back at the same point.  Arithmetic stays fp32.  This keeps the comparison with the CUDA path tight
enough to localise a wrong kernel; parity against the *reference* uses act_dtype=None.

Stochastic regularisation takes its masks INJECTED (torch's random stream cannot be reproduced by another implementation),
and applies them in training only:
  drop_masks   {"<block>": [N] floor(keep + u) / keep}: the drop-path factor of that block's residual branch
  dropout_mask [N, P] already divided by keep, on the pooled vector (Xception discards its dropout, xception.py:214-215)
  drop_block   {"<block>.bn<i>": [N, C, H, W] 0/1 block mask} behind that ResNet BatchNorm, formulas.drop_block_apply
"""
import math

import torch
import torch.nn.functional as F

from .formulas import drop_block_apply


class _QuantSTE(torch.autograd.Function):
    """Round-trip through a 16-bit type in forward AND backward (the native path stores activation
    gradients in 16-bit too)."""

    @staticmethod
    def forward(ctx, x, dt):
        ctx.dt = dt
        return x.to(dt).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dt).to(torch.float32), None


class _GradQ(torch.autograd.Function):
    """identity forward; the gradient is rounded to the 16-bit type (the native path stores it there)"""

    @staticmethod
    def forward(ctx, x, dt):
        ctx.dt = dt
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dt).to(torch.float32), None


def q(x, act_dtype, grad_too=True):
    if act_dtype is None:
        return x
    if grad_too:
        return _QuantSTE.apply(x, act_dtype)
    return x.to(act_dtype).to(torch.float32)


def swish(x):
    return x * torch.sigmoid(x)


def default_bn_eps(spec):
    """BatchNorm eps of `spec`'s reference model: 1e-3 for the TF-ported EfficientNets (pad_type 'same'), else 1e-5"""
    return 1e-3 if getattr(spec, "pad_type", "") == "same" else 1e-5


class BNState:
    """Holds bn hyper-parameters and whether running stats are updated (training) or used (eval)."""

    def __init__(self, training=True, momentum=0.1, eps=1e-5):
        self.training = training
        self.momentum = momentum
        self.eps = eps


def batch_norm(x, sd, prefix, bn):
    rm = sd[prefix + ".running_mean"]
    rv = sd[prefix + ".running_var"]
    if bn.training:
        nbt = sd.get(prefix + ".num_batches_tracked")
        if nbt is not None:
            nbt += 1
    return F.batch_norm(x, rm, rv, sd[prefix + ".weight"], sd[prefix + ".bias"], bn.training, bn.momentum, bn.eps)


def global_pool(x, pool_type="avg"):
    """[N, C, H, W] -> [N, P]: avg, max, avgmax = 0.5 * (avg + max), catavgmax = cat(avg, max) along the features"""
    if pool_type == "avg":
        return x.mean((2, 3))
    x_max = F.adaptive_max_pool2d(x, 1).flatten(1)
    if pool_type == "max":
        return x_max
    x_avg = F.adaptive_avg_pool2d(x, 1).flatten(1)
    if pool_type == "avgmax":
        return 0.5 * (x_avg + x_max)
    if pool_type == "catavgmax":
        return torch.cat((x_avg, x_max), 1)
    raise ValueError("Invalid pool type: %s" % (pool_type,))


def _head(x, sd, name, spec, bn, taps, dropout_mask):
    """global pool, F.dropout (the mask injected), then the classifier `name`"""
    x = global_pool(x, spec.global_pool)
    if taps is not None:
        taps["pooled"] = x
    if dropout_mask is not None and bn.training:
        x = x * dropout_mask
    return F.linear(x, sd[name + ".weight"], sd[name + ".bias"])


def forward(spec, sd, x, bn=None, act_dtype=None, taps=None, drop_masks=None, dropout_mask=None, drop_block=None):
    """x: [N, C, H, W] fp32 -> logits [N, num_classes] fp32. `sd` maps reference state_dict names to
    fp32 CPU tensors (parameters may require grad; running stats are updated in place when bn.training)."""
    if spec.family == "efficientnet":
        assert not drop_block, "DropBlock is a ResNet option"
        return efficientnet_forward(spec, sd, x, bn, act_dtype, taps, drop_masks, dropout_mask)
    if spec.family == "resnet":
        return resnet_forward(spec, sd, x, bn, act_dtype, taps, drop_masks, dropout_mask, drop_block)
    if spec.family == "xception":
        assert not (drop_masks or drop_block), "Xception has no drop path or DropBlock"
        return xception_forward(spec, sd, x, bn, act_dtype)
    raise ValueError("no oracle for model family %r" % (spec.family,))


# ------------------------------------------------------------------------------------------------
# EfficientNet
# ------------------------------------------------------------------------------------------------

def same_pads(extent, k, s):
    """(before, after) zero padding of one axis under TF 'SAME'"""
    total = max((math.ceil(extent / s) - 1) * s + k - extent, 0)
    return total // 2, total - total // 2


def conv_same(x, w, stride, groups=1):
    """TF 'SAME' convolution as an explicit F.pad in front of an unpadded convolution"""
    k = w.shape[-1]
    pt, pb = same_pads(x.shape[2], k, stride)
    pl, pr = same_pads(x.shape[3], k, stride)
    return F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, stride=stride, groups=groups)


def _squeeze_excite(x, sd, p):
    x_se = x.mean((2, 3), keepdim=True)
    x_se = F.conv2d(x_se, sd[p + ".se.conv_reduce.weight"], sd[p + ".se.conv_reduce.bias"])
    x_se = swish(x_se)
    x_se = F.conv2d(x_se, sd[p + ".se.conv_expand.weight"], sd[p + ".se.conv_expand.bias"])
    return x * torch.sigmoid(x_se)


def _conv_dw(x, sd, b, same):
    """the block's depthwise convolution; 'same' pads it with F.pad at every stride, as the TF models do"""
    w = sd[b.name + ".conv_dw.weight"]
    if same:
        return conv_same(x, w, b.stride, groups=b.cmid)
    return F.conv2d(x, w, stride=b.stride, padding=b.pad, groups=b.cmid)


def _mb_block(x, sd, b, bn, act_dtype, taps, drop_mask=None, same=False):
    """drop_mask: optional [N] tensor = floor(keep + U) / keep of drop_path (layers/drop.py:84-100), applied to the block's
    main path before the residual add (efficientnet_blocks.py:343-346)."""
    p = b.name
    residual = x
    if b.kind == "ir":
        x = q(F.conv2d(x, sd[p + ".conv_pw.weight"]), act_dtype)
        if taps is not None:
            taps[p + ".conv_pw"] = x
        # the native depthwise kernel stages its activated input in 16-bit shared memory (as apex AMP O1 casts
        # the conv input to half in the reference's GPU path): one more rounding point in emulation mode
        x = q(swish(batch_norm(x, sd, p + ".bn1", bn)), act_dtype)
        x = q(_conv_dw(x, sd, b, same), act_dtype)
        if taps is not None:
            taps[p + ".conv_dw"] = x
        x = swish(batch_norm(x, sd, p + ".bn2", bn))
        if b.cse:
            x = _squeeze_excite(x, sd, p)
        x = q(x, act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv_pwl.weight"]), act_dtype)
        if taps is not None:
            taps[p + ".conv_pwl"] = x
        x = batch_norm(x, sd, p + ".bn3", bn)
    else:
        x = q(_conv_dw(x, sd, b, same), act_dtype)
        if taps is not None:
            taps[p + ".conv_dw"] = x
        x = swish(batch_norm(x, sd, p + ".bn1", bn))
        if b.cse:
            x = _squeeze_excite(x, sd, p)
        x = q(x, act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv_pw.weight"]), act_dtype)
        if taps is not None:
            taps[p + ".conv_pw"] = x
        x = batch_norm(x, sd, p + ".bn2", bn)
    if b.has_residual:
        if drop_mask is not None and bn.training:
            x = x * drop_mask.view(-1, 1, 1, 1)
        x = x + residual
    x = q(x, act_dtype)
    if taps is not None:
        taps[p + ".out"] = x
    return x


def efficientnet_forward(spec, sd, x, bn=None, act_dtype=None, taps=None, drop_masks=None, dropout_mask=None):
    bn = bn or BNState(eps=default_bn_eps(spec))
    same = spec.pad_type == "same"
    x = q(x, act_dtype, grad_too=False)
    w = sd["conv_stem.weight"]
    x = q(conv_same(x, w, 2) if same else F.conv2d(x, w, stride=2, padding=1), act_dtype)
    if taps is not None:
        taps["conv_stem"] = x
    x = q(swish(batch_norm(x, sd, "bn1", bn)), act_dtype)
    if taps is not None:
        taps["stem.out"] = x
    for b in spec.blocks:
        x = _mb_block(x, sd, b, bn, act_dtype, taps, None if drop_masks is None else drop_masks.get(b.name), same)
    x = q(F.conv2d(x, sd["conv_head.weight"]), act_dtype)
    if taps is not None:
        taps["conv_head"] = x
    x = swish(batch_norm(x, sd, "bn2", bn))
    return _head(x, sd, "classifier", spec, bn, taps, dropout_mask)


# ------------------------------------------------------------------------------------------------
# ResNet, ResNet-D, Wide ResNet, SE-ResNet
# ------------------------------------------------------------------------------------------------

def _bn_drop(x, sd, name, bn, act_dtype, drop_block, gate=None):
    """BatchNorm `name`, then its DropBlock and the block's drop-path gate (training only)"""
    x = batch_norm(x, sd, name, bn)
    m = drop_block.get(name) if (drop_block and bn.training) else None
    g = gate if bn.training else None
    if m is None and g is None:
        return x
    if act_dtype is not None:
        x = _GradQ.apply(x, act_dtype)
    if m is not None:
        x = drop_block_apply(x, m)
    if g is not None:
        x = x * g.view(-1, 1, 1, 1)
    return x


def _se_module(z, sd, p):
    """SEModule.forward (senet.py:79-86): z * sigmoid(fc2(relu(fc1(mean_hw z))))"""
    s = z.mean((2, 3), keepdim=True)
    s = F.relu(F.conv2d(s, sd[p + ".se_module.fc1.weight"], sd[p + ".se_module.fc1.bias"]))
    gate = torch.sigmoid(F.conv2d(s, sd[p + ".se_module.fc2.weight"], sd[p + ".se_module.fc2.bias"]))
    return z * gate


def _res_stem(spec, sd, x, bn, act_dtype):
    """7x7 s2 conv (or the ResNet-D deep stem of three 3x3 convs), BN, ReLU, then the 3x3 s2 max-pool: padded ('p1') or,
    in SENet's layer0, unpadded in ceil mode ('ceil')"""
    if spec.stem_type == "deep":
        x = q(F.conv2d(x, sd["conv1.0.weight"], stride=2, padding=1), act_dtype)
        x = q(F.relu(batch_norm(x, sd, "conv1.1", bn)), act_dtype)
        x = q(F.conv2d(x, sd["conv1.3.weight"], padding=1), act_dtype)
        x = q(F.relu(batch_norm(x, sd, "conv1.4", bn)), act_dtype)
        x = q(F.conv2d(x, sd["conv1.6.weight"], padding=1), act_dtype)
    else:
        x = q(F.conv2d(x, sd[spec.stem_conv + ".weight"], stride=2, padding=3), act_dtype)
    x = q(F.relu(batch_norm(x, sd, spec.stem_bn, bn)), act_dtype)
    if spec.stem_pool == "ceil":
        return F.max_pool2d(x, kernel_size=3, stride=2, ceil_mode=True)
    return F.max_pool2d(x, kernel_size=3, stride=2, padding=1)


def _shortcut(b, sd, x, bn, act_dtype):
    p = b.name
    if not b.avg_down:
        x = q(F.conv2d(x, sd[p + ".downsample.0.weight"], stride=b.stride), act_dtype)
        return batch_norm(x, sd, p + ".downsample.1", bn)
    if b.stride != 1:
        x = q(F.avg_pool2d(x, 2, b.stride, ceil_mode=True, count_include_pad=False), act_dtype)
    x = q(F.conv2d(x, sd[p + ".downsample.1.weight"]), act_dtype)
    return batch_norm(x, sd, p + ".downsample.2", bn)


def _res_block(x, sd, b, bn, act_dtype, taps=None, drop_block=None, gate=None, spec=None):
    """one residual block. `spec` is the block's ResNetSpec: an SE-ResNet spec puts the bottleneck's stride on its 1x1 and
    rounds the shortcut BN output to 16 bit; None stands for a plain ResNet"""
    p = b.name
    residual = x
    senet = spec is not None and spec.naming == "senet"
    s1, s2 = (b.stride, 1) if spec is not None and spec.stride_in_1x1 else (1, b.stride)
    if b.kind == "basic":
        x = q(F.conv2d(x, sd[p + ".conv1.weight"], stride=b.stride, padding=1), act_dtype)
        x = q(F.relu(_bn_drop(x, sd, p + ".bn1", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], padding=1), act_dtype)
        x = _bn_drop(x, sd, p + ".bn2", bn, act_dtype, drop_block, gate)
        if b.cse:
            x = F.relu(x)           # SEResNetBlock applies the ReLU before the SE (senet.py:213-215)
    else:
        x = q(F.conv2d(x, sd[p + ".conv1.weight"], stride=s1), act_dtype)
        x = q(F.relu(_bn_drop(x, sd, p + ".bn1", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], stride=s2, padding=1), act_dtype)
        x = q(F.relu(_bn_drop(x, sd, p + ".bn2", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv3.weight"]), act_dtype)
        x = _bn_drop(x, sd, p + ".bn3", bn, act_dtype, drop_block, gate)
    if b.cse:
        x = _se_module(x, sd, p)
    if b.downsample:
        residual = _shortcut(b, sd, residual, bn, act_dtype)
        if senet:
            residual = q(residual, act_dtype)       # the SE-ResNet plan stores its shortcut BN output in 16 bit
    x = q(F.relu(x + residual), act_dtype)
    if taps is not None:
        taps[p + ".out"] = x
    return x


def resnet_forward(spec, sd, x, bn=None, act_dtype=None, taps=None, drop_masks=None, dropout_mask=None, drop_block=None):
    bn = bn or BNState()
    x = _res_stem(spec, sd, q(x, act_dtype, grad_too=False), bn, act_dtype)
    if taps is not None:
        taps["stem.out"] = x
    for b in spec.blocks:
        x = _res_block(x, sd, b, bn, act_dtype, taps, drop_block, None if drop_masks is None else drop_masks.get(b.name),
                       spec)
    return _head(x, sd, spec.cls_name, spec, bn, taps, dropout_mask)


# ------------------------------------------------------------------------------------------------
# Xception
# ------------------------------------------------------------------------------------------------
# With act_dtype set, every tensor the native plan stores in 16 bit is rounded at the same point: the stem convolution
# outputs and activations, each depthwise output (its input ReLU and BN applied in fp32, then the staged value rounded),
# each pointwise output, the shortcut convolution output and every block output. The pooled BN output of a strided block,
# like the head's BN + ReLU, stays fp32.
# Semantics pinned (xception.py): conv1 3x3 s2 p0, conv2 3x3 p0, each + BN + ReLU (:183-188); Block (:72-124): rep[0] is
# a NON-inplace ReLU, so the shortcut reads the block input before activation; block1 starts without a ReLU; strided
# blocks end with MaxPool2d(3, 2, 1) on the last BN output; x += skipbn(skip(inp)) or x += inp; conv3's depthwise reads
# block12's output with no activation (:201); dropout's result is discarded (:214-215).

def _sep(x, sd, prefix, act_dtype):
    """SeparableConv2d (:58-69): depthwise 3x3 p1, then 1x1, each output stored in 16 bit"""
    C = x.shape[1]
    d = q(F.conv2d(x, sd[prefix + ".conv1.weight"], padding=1, groups=C), act_dtype)
    return q(F.conv2d(d, sd[prefix + ".pointwise.weight"]), act_dtype)


def _xblock(x, sd, b, bn, act_dtype):
    p = b.name
    inp = x
    h = F.relu(x) if b.start_with_relu else x
    for j, (r, _, _) in enumerate(b.seps):
        if j:
            h = q(F.relu(h), act_dtype)          # the staged BN + ReLU of the next depthwise input
        y = _sep(h, sd, "%s.rep.%d" % (p, r), act_dtype)
        h = batch_norm(y, sd, "%s.rep.%d" % (p, r + 1), bn)
    if b.stride != 1:
        h = F.max_pool2d(h, 3, 2, 1)
    if b.skip:
        s = q(F.conv2d(inp, sd[p + ".skip.weight"], stride=b.stride), act_dtype)
        s = batch_norm(s, sd, p + ".skipbn", bn)
    else:
        s = inp
    return q(h + s, act_dtype)


def xception_forward(spec, sd, x, bn=None, act_dtype=None):
    bn = bn or BNState()
    x = q(x, act_dtype, grad_too=False)
    x = q(F.conv2d(x, sd["conv1.weight"], stride=2), act_dtype)
    x = q(F.relu(batch_norm(x, sd, "bn1", bn)), act_dtype)
    x = q(F.conv2d(x, sd["conv2.weight"]), act_dtype)
    x = q(F.relu(batch_norm(x, sd, "bn2", bn)), act_dtype)
    for b in spec.blocks:
        x = _xblock(x, sd, b, bn, act_dtype)
    x = _sep(x, sd, "conv3", act_dtype)
    x = q(F.relu(batch_norm(x, sd, "bn3", bn)), act_dtype)
    x = _sep(x, sd, "conv4", act_dtype)
    x = F.relu(batch_norm(x, sd, "bn4", bn))
    return _head(x, sd, "fc", spec, bn, None, None)


# ------------------------------------------------------------------------------------------------
# losses and metrics
# ------------------------------------------------------------------------------------------------

def cross_entropy(logits, target, smoothing=0.0):
    """Covers the reference's three losses: nn.CrossEntropyLoss (hard target, smoothing 0),
    LabelSmoothingCrossEntropy (cross_entropy.py:20-26) and SoftTargetCrossEntropy (:34-36, float target)."""
    logp = F.log_softmax(logits, dim=-1)
    if target.dtype.is_floating_point:
        return torch.sum(-target * logp, dim=-1).mean()
    nll = -logp.gather(dim=-1, index=target.unsqueeze(1)).squeeze(1)
    smooth = -logp.mean(dim=-1)
    return ((1.0 - smoothing) * nll + smoothing * smooth).mean()


def bce_two_class(logits, target, smoothing=0.0):
    """The sigmoid-BCE form the fused CUDA head computes (SURVEY.md section 8a row H2):
    with d = z1 - z0 and soft target t1, CE(z, t) == t1*softplus(-d) + (1-t1)*softplus(d)."""
    d = logits[:, 1] - logits[:, 0]
    if target.dtype.is_floating_point:
        t1 = target[:, 1]
    else:
        t1 = target.to(torch.float32) * (1.0 - smoothing) + 0.5 * smoothing
    return (t1 * F.softplus(-d) + (1.0 - t1) * F.softplus(d)).mean()


def accuracy_top1(logits, target):
    # utils.py:170-186 (soft targets: argmax of the target row, :177-178)
    if target.dtype.is_floating_point:
        target = target.argmax(dim=1)
    pred = logits.argmax(dim=1)
    return (pred == target).to(torch.float32).mean() * 100.0
