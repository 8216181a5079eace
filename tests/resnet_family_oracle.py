"""CPU oracle of the dense ResNet family beyond resnet18 / resnet50 (test infrastructure, like oracle/).

oracle/model.py's ResNet forward reads every convolution's shape from its weight, so the bottleneck width of the wide models
(resnet.py:187) and the deeper layouts need nothing new. What it does not restate is ResNet-D (resnet26d, resnet50d):
  * the deep stem, conv1 = Sequential(conv 3x3 s2, BN, ReLU, conv 3x3, BN, ReLU, conv 3x3), resnet.py:365-377;
  * the average-pool shortcut downsample_avg = [AvgPool2d(2, stride, ceil_mode=True, count_include_pad=False) (nn.Identity at
    stride 1), conv 1x1, BN], resnet.py:263-277.
This module restates the forward and the train / validate steps with both, from oracle/'s building blocks (BatchNorm, the
16-bit storage emulation `act_dtype`, losses, optimizers) and tests/resnet_drop_oracle.py's injected DropBlock / drop-path /
dropout masks. For a spec without them, and no masks, it is oracle.train.train_step's arithmetic.
"""
import torch
import torch.nn.functional as F

from oracle import model as M
from oracle import train as OT

import gpool_oracle as GO
import resnet_drop_oracle as RD


TAME = 0.2


def tame_state(spec, sd, factor=TAME):
    """scale the last BatchNorm gamma of every residual branch (engine_checks.run_parity(tame=True)): with gamma ~ 1 on every
    branch the synthetic-weight networks amplify 16-bit rounding by orders of magnitude, which no 16-bit path can be held to"""
    for b in spec.blocks:
        k = b.name + (".bn2.weight" if b.kind == "basic" else ".bn3.weight")
        sd[k] = sd[k] * factor
    return sd


def stem(spec, sd, x, bn, act_dtype):
    q = M.q
    if spec.stem_type == "deep":
        x = q(F.conv2d(x, sd["conv1.0.weight"], stride=2, padding=1), act_dtype)
        x = q(F.relu(M.batch_norm(x, sd, "conv1.1", bn)), act_dtype)
        x = q(F.conv2d(x, sd["conv1.3.weight"], padding=1), act_dtype)
        x = q(F.relu(M.batch_norm(x, sd, "conv1.4", bn)), act_dtype)
        x = q(F.conv2d(x, sd["conv1.6.weight"], padding=1), act_dtype)
    else:
        x = q(F.conv2d(x, sd["conv1.weight"], stride=2, padding=3), act_dtype)
    x = q(F.relu(M.batch_norm(x, sd, "bn1", bn)), act_dtype)
    return F.max_pool2d(x, kernel_size=3, stride=2, padding=1)


def shortcut(b, sd, x, bn, act_dtype):
    q, p = M.q, b.name
    if not b.avg_down:
        x = q(F.conv2d(x, sd[p + ".downsample.0.weight"], stride=b.stride), act_dtype)
        return M.batch_norm(x, sd, p + ".downsample.1", bn)
    if b.stride != 1:
        x = q(F.avg_pool2d(x, 2, b.stride, ceil_mode=True, count_include_pad=False), act_dtype)
    x = q(F.conv2d(x, sd[p + ".downsample.1.weight"]), act_dtype)
    return M.batch_norm(x, sd, p + ".downsample.2", bn)


def _res_block(x, sd, b, bn, act_dtype, drop_block, gate):
    """tests/resnet_drop_oracle.py's block (resnet.py:150-175, 215-246) with `shortcut` above"""
    q, p = M.q, b.name
    residual = x
    if b.kind == "basic":
        x = q(F.conv2d(x, sd[p + ".conv1.weight"], stride=b.stride, padding=1), act_dtype)
        x = q(F.relu(RD._bn_drop(x, sd, p + ".bn1", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], padding=1), act_dtype)
        x = RD._bn_drop(x, sd, p + ".bn2", bn, act_dtype, drop_block, gate)
    else:
        x = q(F.conv2d(x, sd[p + ".conv1.weight"]), act_dtype)
        x = q(F.relu(RD._bn_drop(x, sd, p + ".bn1", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], stride=b.stride, padding=1), act_dtype)
        x = q(F.relu(RD._bn_drop(x, sd, p + ".bn2", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv3.weight"]), act_dtype)
        x = RD._bn_drop(x, sd, p + ".bn3", bn, act_dtype, drop_block, gate)
    if b.downsample:
        residual = shortcut(b, sd, residual, bn, act_dtype)
    return q(F.relu(x + residual), act_dtype)


def forward(spec, sd, x, bn=None, act_dtype=None, drop_block=None, drop_masks=None, dropout_mask=None):
    assert spec.family == "resnet", spec.arch
    bn = bn or M.BNState()
    x = stem(spec, sd, M.q(x, act_dtype, grad_too=False), bn, act_dtype)
    for b in spec.blocks:
        x = _res_block(x, sd, b, bn, act_dtype, drop_block, None if drop_masks is None else drop_masks.get(b.name))
    x = GO.global_pool(x, spec.global_pool)
    if dropout_mask is not None and bn.training:
        x = x * dropout_mask
    return F.linear(x, sd["fc.weight"], sd["fc.bias"])


def train_step(spec, sd, x, target, opt=None, smoothing=0.0, act_dtype=None, drop_block=None, drop_masks=None,
               dropout_mask=None):
    """oracle.train.train_step over `forward` above. `sd` tensors are updated in place."""
    params, _ = OT.split_state(spec, sd)
    for p in params.values():
        p.requires_grad_(True)
        p.grad = None
    logits = forward(spec, sd, x, M.BNState(training=True), act_dtype, drop_block, drop_masks, dropout_mask)
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
