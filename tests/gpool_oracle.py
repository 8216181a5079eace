"""CPU oracle of the selectable global pool (test infrastructure, like oracle/).

The reference builds `SelectAdaptivePool2d(pool_type=global_pool)` behind the last feature map (efficientnet.py:297-300,340,
resnet.py:407-409,464; layers/adaptive_avgmax_pool.py:24-48). oracle/model.py restates the reference at its default, 'avg';
this module restates the forward, train and validate steps with any pool type, from oracle/'s own building blocks (the
blocks, BatchNorm, Swish, 16-bit storage emulation, losses and optimizers), so everything but the pool is the same
arithmetic. tests/test_global_pool_cpu.py pins it to fixtures minted from the unmodified reference."""
import torch
import torch.nn.functional as F

from oracle import model as M
from oracle import train as OT


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


def forward(spec, sd, x, bn=None, act_dtype=None, dropout_mask=None):
    """oracle.model.forward with `spec.global_pool` behind the last feature map (no drop path: drop_path_rate = 0)"""
    bn = bn or M.BNState()
    x = M.q(x, act_dtype, grad_too=False)
    if spec.family == "efficientnet":
        x = M.q(F.conv2d(x, sd["conv_stem.weight"], stride=2, padding=1), act_dtype)
        x = M.q(M.swish(M.batch_norm(x, sd, "bn1", bn)), act_dtype)
        for b in spec.blocks:
            x = M._mb_block(x, sd, b, bn, act_dtype, None)
        x = M.q(F.conv2d(x, sd["conv_head.weight"]), act_dtype)
        x = global_pool(M.swish(M.batch_norm(x, sd, "bn2", bn)), spec.global_pool)
        if dropout_mask is not None and bn.training:
            x = x * dropout_mask            # F.dropout with the engine's mask (already / keep), efficientnet.py:346-347
        return F.linear(x, sd["classifier.weight"], sd["classifier.bias"])
    x = M.q(F.conv2d(x, sd["conv1.weight"], stride=2, padding=3), act_dtype)
    x = M.q(F.relu(M.batch_norm(x, sd, "bn1", bn)), act_dtype)
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    for b in spec.blocks:
        x = M._res_block(x, sd, b, bn, act_dtype, None)
    return F.linear(global_pool(x, spec.global_pool), sd["fc.weight"], sd["fc.bias"])


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
