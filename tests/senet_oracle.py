"""CPU oracle of the SE-ResNets (seresnet18/34/50/101/152, dfd/timm/models/senet.py; test infrastructure, like oracle/).

What oracle/model.py's ResNet does not restate:
  * layer0: conv1 7x7 s2 p3 -> bn1 -> ReLU -> MaxPool2d(3, 2, ceil_mode=True) without padding (senet.py:291-300);
  * SEResNetBottleneck puts the stride on its 1x1 conv1, conv2 runs at stride 1 (:141-163); SEResNetBlock as BasicBlock;
  * every block ends in relu(se_module(z) + residual), z = bn3(conv3) in the bottleneck (:94-114) and relu(bn2(conv2)) in the
    basic block (:206-223); SEModule = avg-pool, fc1 (bias), ReLU, fc2 (bias), sigmoid, multiply (:67-86);
  * the classifier is `last_linear`, after F.dropout on the pooled vector (:386-391, the mask injected here).
Built from oracle/'s BatchNorm, 16-bit storage emulation `act_dtype`, losses and optimizers; rounding points where the native
plan stores 16-bit tensors (the SE gate and pooled vector are fp32 there, and so here).
"""
import torch
import torch.nn.functional as F

from oracle import model as M
from oracle import train as OT

import gpool_oracle as GO

TAME = 0.2


def tame_state(spec, sd, factor=TAME):
    """scale the last BatchNorm gamma of every residual branch (the SE scales that branch, it does not replace it)"""
    for b in spec.blocks:
        k = b.name + (".bn2.weight" if b.kind == "basic" else ".bn3.weight")
        sd[k] = sd[k] * factor
    return sd


def se_module(z, sd, p):
    """SEModule.forward (senet.py:79-86): z * sigmoid(fc2(relu(fc1(mean_hw z))))"""
    s = z.mean((2, 3), keepdim=True)
    s = F.relu(F.conv2d(s, sd[p + ".se_module.fc1.weight"], sd[p + ".se_module.fc1.bias"]))
    gate = torch.sigmoid(F.conv2d(s, sd[p + ".se_module.fc2.weight"], sd[p + ".se_module.fc2.bias"]))
    return z * gate


def stem(sd, x, bn, act_dtype):
    q = M.q
    x = q(F.conv2d(x, sd["layer0.conv1.weight"], stride=2, padding=3), act_dtype)
    x = q(F.relu(M.batch_norm(x, sd, "layer0.bn1", bn)), act_dtype)
    return F.max_pool2d(x, kernel_size=3, stride=2, ceil_mode=True)


def block(x, sd, b, bn, act_dtype):
    q, p = M.q, b.name
    residual = x
    if b.kind == "basic":
        x = q(F.conv2d(x, sd[p + ".conv1.weight"], stride=b.stride, padding=1), act_dtype)
        x = q(F.relu(M.batch_norm(x, sd, p + ".bn1", bn)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], padding=1), act_dtype)
        z = F.relu(M.batch_norm(x, sd, p + ".bn2", bn))        # SEResNetBlock applies the ReLU before the SE (senet.py:213-215)
    else:
        x = q(F.conv2d(x, sd[p + ".conv1.weight"], stride=b.stride), act_dtype)
        x = q(F.relu(M.batch_norm(x, sd, p + ".bn1", bn)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], padding=1), act_dtype)
        x = q(F.relu(M.batch_norm(x, sd, p + ".bn2", bn)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv3.weight"]), act_dtype)
        z = M.batch_norm(x, sd, p + ".bn3", bn)
    if b.downsample:
        residual = q(F.conv2d(residual, sd[p + ".downsample.0.weight"], stride=b.stride), act_dtype)
        residual = q(M.batch_norm(residual, sd, p + ".downsample.1", bn), act_dtype)
    return q(F.relu(se_module(z, sd, p) + residual), act_dtype)


def forward(spec, sd, x, bn=None, act_dtype=None, dropout_mask=None):
    assert spec.naming == "senet", spec.arch
    bn = bn or M.BNState()
    x = stem(sd, M.q(x, act_dtype, grad_too=False), bn, act_dtype)
    for b in spec.blocks:
        x = block(x, sd, b, bn, act_dtype)
    x = GO.global_pool(x, spec.global_pool)
    if dropout_mask is not None and bn.training:
        x = x * dropout_mask
    return F.linear(x, sd["last_linear.weight"], sd["last_linear.bias"])


def train_step(spec, sd, x, target, opt=None, smoothing=0.0, act_dtype=None, dropout_mask=None):
    """oracle.train.train_step over `forward` above. `sd` tensors are updated in place."""
    params, _ = OT.split_state(spec, sd)
    for p in params.values():
        p.requires_grad_(True)
        p.grad = None
    logits = forward(spec, sd, x, M.BNState(training=True), act_dtype, dropout_mask)
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
