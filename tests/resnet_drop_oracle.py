"""CPU oracle of the ResNet stochastic regularisation (test infrastructure, like oracle/).

The reference ResNet applies DropBlock2d(rate, 7, 0.25 / 1.0) behind every main-branch BatchNorm of layer3 / layer4, one
DropPath(drop_path_rate) to the main branch of every block, and F.dropout to the pooled vector (resnet.py:153-175,218-246,
385-404,466; layers/drop.py:24-100). torch's random stream cannot be reproduced by another implementation, so this module
restates the forward and train steps with the masks INJECTED, from oracle/'s own building blocks (BatchNorm, 16-bit storage
emulation, losses, optimizers): everything but the masks is oracle.model's arithmetic, and with no masks it is
oracle.train.train_step bit for bit. tests/test_resnet_drop_cpu.py pins it to fixtures minted from the unmodified reference.

Masks:
  drop_block  {"<block>.bn<i>": [N, C, H, W] 0/1 block mask}: x * m * (numel / (sum m + 1e-7)), drop.py:59-61
  drop_masks  {"<block>": [N] floor(keep + u) / keep}: the drop-path factor of that block's main branch
  dropout_mask [N, P] already divided by keep
"""
import torch
import torch.nn.functional as F

from oracle import model as M
from oracle import train as OT

import gpool_oracle as GO


def drop_block_gamma(H, W, rate, gamma_scale, block_size=7):
    """(gamma, clipped block size) exactly as drop_block_2d computes them (drop.py:36-42)"""
    cb = min(block_size, min(W, H))
    return gamma_scale * rate * (W * H) / cb ** 2 / ((W - block_size + 1) * (H - block_size + 1)), cb


def valid_block(H, W, cb):
    """drop.py:45-48: built on a [W, H] meshgrid and reshaped to [H, W] (scrambled for non-square maps)"""
    w_i, h_i = torch.meshgrid(torch.arange(W), torch.arange(H), indexing="ij")
    v = ((w_i >= cb // 2) & (w_i < W - (cb - 1) // 2)) & ((h_i >= cb // 2) & (h_i < H - (cb - 1) // 2))
    return torch.reshape(v, (1, 1, H, W)).float()


def seeds_from_noise(u, gamma, cb):
    """[N, C, H, W] 0/1 seed-keep mask from the uniform draws, in the reference's fp32 order (drop.py:51)"""
    H, W = u.shape[-2:]
    return ((2 - gamma - valid_block(H, W, cb) + u) >= 1).float()


def block_from_seeds(seeds, cb):
    """drop.py:52-56: min-pool of the seeds (the -inf padding of max_pool2d is ignored)"""
    return -F.max_pool2d(-seeds, kernel_size=cb, stride=1, padding=cb // 2)


def drop_block_apply(x, m):
    """drop.py:60-61"""
    return x * m * (m.numel() / (torch.sum(m) + 1e-7))


class _GradQ(torch.autograd.Function):
    """identity forward; the gradient is rounded to the 16-bit type (the native path stores it there)"""

    @staticmethod
    def forward(ctx, x, dt):
        ctx.dt = dt
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dt).to(torch.float32), None


def _gq(x, act_dtype):
    return x if act_dtype is None else _GradQ.apply(x, act_dtype)


def _bn_drop(x, sd, name, bn, act_dtype, drop_block, gate=None):
    """BatchNorm `name`, then its DropBlock and the block's drop-path gate (training only)"""
    x = M.batch_norm(x, sd, name, bn)
    m = drop_block.get(name) if (drop_block and bn.training) else None
    g = gate if bn.training else None
    if m is None and g is None:
        return x
    x = _gq(x, act_dtype)
    if m is not None:
        x = drop_block_apply(x, m)
    if g is not None:
        x = x * g.view(-1, 1, 1, 1)
    return x


def _res_block(x, sd, b, bn, act_dtype, drop_block, gate):
    """oracle.model._res_block with the masks (resnet.py:150-175, 215-246)"""
    q, p = M.q, b.name
    residual = x
    if b.kind == "basic":
        x = q(F.conv2d(x, sd[p + ".conv1.weight"], stride=b.stride, padding=1), act_dtype)
        x = q(F.relu(_bn_drop(x, sd, p + ".bn1", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], padding=1), act_dtype)
        x = _bn_drop(x, sd, p + ".bn2", bn, act_dtype, drop_block, gate)
    else:
        x = q(F.conv2d(x, sd[p + ".conv1.weight"]), act_dtype)
        x = q(F.relu(_bn_drop(x, sd, p + ".bn1", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv2.weight"], stride=b.stride, padding=1), act_dtype)
        x = q(F.relu(_bn_drop(x, sd, p + ".bn2", bn, act_dtype, drop_block)), act_dtype)
        x = q(F.conv2d(x, sd[p + ".conv3.weight"]), act_dtype)
        x = _bn_drop(x, sd, p + ".bn3", bn, act_dtype, drop_block, gate)
    if b.downsample:
        residual = q(F.conv2d(residual, sd[p + ".downsample.0.weight"], stride=b.stride), act_dtype)
        residual = M.batch_norm(residual, sd, p + ".downsample.1", bn)
    return q(F.relu(x + residual), act_dtype)


def forward(spec, sd, x, bn=None, act_dtype=None, drop_block=None, drop_masks=None, dropout_mask=None):
    """oracle.model.resnet_forward with injected DropBlock / drop-path / dropout masks (applied in training only)"""
    bn = bn or M.BNState()
    q = M.q
    x = q(x, act_dtype, grad_too=False)
    x = q(F.conv2d(x, sd["conv1.weight"], stride=2, padding=3), act_dtype)
    x = q(F.relu(M.batch_norm(x, sd, "bn1", bn)), act_dtype)
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
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


def engine_masks(eng):
    """the masks a native ResNet engine drew for its last training step, in this oracle's layout (CPU)"""
    db = {k: m.permute(0, 3, 1, 2).float().cpu() for k, (m, _) in eng.drop_block_masks.items()}
    dp = {k: g[:, 0].cpu().clone() for k, g in eng.drop_masks.items()}
    dm = eng.dropout_mask.cpu().clone() if eng.drop_rate > 0 else None
    return db, dp, dm
