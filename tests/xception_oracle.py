"""CPU oracle of Xception (test infrastructure, like oracle/).

A restatement of dfd/timm/models/xception.py's forward and of the train / validate steps, from oracle/'s building blocks
(BatchNorm, losses, optimizers and the 16-bit storage emulation `q`). With act_dtype set, every tensor the native plan stores
in 16 bit is rounded at the same point: the stem convolution outputs and activations, each depthwise output (its input ReLU
and BN applied in fp32, then the staged value rounded), each pointwise output, the shortcut convolution output and every
block output. The pooled BN output of a strided block, like the head's BN + ReLU, stays fp32.

Semantics pinned (xception.py):
  * conv1 3x3 s2 p0, conv2 3x3 p0, each + BN + ReLU (:183-188);
  * Block (:72-124): rep[0] is a NON-inplace ReLU, so the shortcut reads the block input before activation; block1 starts
    without a ReLU; strided blocks end with MaxPool2d(3, 2, 1) on the last BN output; x += skipbn(skip(inp)) or x += inp;
  * conv3's depthwise reads block12's output with no activation (:201);
  * dropout's result is discarded (:214-215): drop_rate has no effect.
"""
import torch
import torch.nn.functional as F

from oracle import model as M
from oracle import train as OT

import gpool_oracle as GO


TAME = 0.2


def tame_state(spec, sd, factor=TAME):
    """scale the last BatchNorm gamma of every block's `rep` (the residual branch): see resnet_family_oracle.tame_state"""
    for b in spec.blocks:
        r = b.seps[-1][0] + 1
        k = "%s.rep.%d.weight" % (b.name, r)
        sd[k] = sd[k] * factor
    return sd


def _sep(x, sd, prefix, act_dtype):
    """SeparableConv2d (:58-69): depthwise 3x3 p1, then 1x1, each output stored in 16 bit"""
    q = M.q
    C = x.shape[1]
    d = q(F.conv2d(x, sd[prefix + ".conv1.weight"], padding=1, groups=C), act_dtype)
    return q(F.conv2d(d, sd[prefix + ".pointwise.weight"]), act_dtype)


def _block(x, sd, b, bn, act_dtype):
    q, p = M.q, b.name
    inp = x
    h = F.relu(x) if b.start_with_relu else x
    for j, (r, _, _) in enumerate(b.seps):
        if j:
            h = q(F.relu(h), act_dtype)          # the staged BN + ReLU of the next depthwise input
        y = _sep(h, sd, "%s.rep.%d" % (p, r), act_dtype)
        h = M.batch_norm(y, sd, "%s.rep.%d" % (p, r + 1), bn)
    if b.stride != 1:
        h = F.max_pool2d(h, 3, 2, 1)
    if b.skip:
        s = q(F.conv2d(inp, sd[p + ".skip.weight"], stride=b.stride), act_dtype)
        s = M.batch_norm(s, sd, p + ".skipbn", bn)
    else:
        s = inp
    return q(h + s, act_dtype)


def forward(spec, sd, x, bn=None, act_dtype=None):
    assert spec.family == "xception", spec.arch
    q = M.q
    bn = bn or M.BNState()
    x = q(x, act_dtype, grad_too=False)
    x = q(F.conv2d(x, sd["conv1.weight"], stride=2), act_dtype)
    x = q(F.relu(M.batch_norm(x, sd, "bn1", bn)), act_dtype)
    x = q(F.conv2d(x, sd["conv2.weight"]), act_dtype)
    x = q(F.relu(M.batch_norm(x, sd, "bn2", bn)), act_dtype)
    for b in spec.blocks:
        x = _block(x, sd, b, bn, act_dtype)
    x = _sep(x, sd, "conv3", act_dtype)
    x = q(F.relu(M.batch_norm(x, sd, "bn3", bn)), act_dtype)
    x = _sep(x, sd, "conv4", act_dtype)
    x = F.relu(M.batch_norm(x, sd, "bn4", bn))
    x = GO.global_pool(x, spec.global_pool)
    return F.linear(x, sd["fc.weight"], sd["fc.bias"])


def train_step(spec, sd, x, target, opt=None, smoothing=0.0, act_dtype=None):
    """oracle.train.train_step over `forward` above. `sd` tensors are updated in place."""
    params, _ = OT.split_state(spec, sd)
    for p in params.values():
        p.requires_grad_(True)
        p.grad = None
    logits = forward(spec, sd, x, M.BNState(training=True), act_dtype)
    loss = M.cross_entropy(logits, target, smoothing)
    prec1 = M.accuracy_top1(logits.detach(), target)
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in params.items()}
    for p in params.values():
        p.requires_grad_(False)
        p.grad = None
    if opt is not None:
        OT.optimizer_step(opt, params, grads)
    return dict(logits=logits.detach(), loss=loss.detach(), prec1=prec1, grads=grads)


@torch.no_grad()
def validate_step(spec, sd, x, target, act_dtype=None):
    logits = forward(spec, sd, x, M.BNState(training=False), act_dtype)
    return dict(logits=logits, loss=M.cross_entropy(logits, target, 0.0), prec1=M.accuracy_top1(logits, target))
