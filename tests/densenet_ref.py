"""DenseNet restated in plain torch ops for the DenseNet tests: densenet.py's forward (_DenseLayer :37-56, _Transition :62-70,
DenseNet.forward_features / forward :130-140) with the dropout masks given (already divided by keep, as the native plan draws
them) and BatchNorm in training mode (batch statistics, running statistics updated with momentum 0.1 and the unbiased
variance) or eval mode. It is held to the reference's own steps by tests/test_densenet_cpu.py (fixtures of
tools/mint_densenet_goldens.py).

act_dtype (torch.float16 / torch.bfloat16) emulates the native plan's 16-bit storage: the weights of the convolutions, every
tensor the plan stores (convolution outputs, BN + ReLU outputs, the block buffers, the pooled transition input) and the
gradient of each of them are rounded to that type at the point the plan stores them, the transition pools before its
convolution as the plan does, and the block buffer's gradient is rounded after every layer's contribution is added. It is
the yardstick of the native gradients: the distance between this emulation and the exact step is what 16-bit storage alone
costs."""
import torch
import torch.nn.functional as F


class _Round(torch.autograd.Function):
    """value and gradient rounded to a 16-bit type (computation stays in the input's precision)"""

    @staticmethod
    def forward(ctx, x, dt):
        ctx.dt = dt
        return x.to(dt).to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dt).to(g.dtype), None


def _bn(x, sd, p, training, new_sd):
    rm, rv = sd[p + ".running_mean"].to(x).clone(), sd[p + ".running_var"].to(x).clone()
    y = F.batch_norm(x, rm, rv, sd[p + ".weight"].to(x), sd[p + ".bias"].to(x), training, 0.1, 1e-5)
    if new_sd is not None and training:
        new_sd[p + ".running_mean"], new_sd[p + ".running_var"] = rm.detach(), rv.detach()
    return y


def forward(spec, sd, x, training=True, masks=None, head_mask=None, new_sd=None, act_dtype=None):
    """logits of NCHW x; masks: {layer name: [N, H, W, k] keep mask / keep} (NHWC, as the plan stores them); new_sd: receives
    the updated running statistics"""
    q = (lambda t: _Round.apply(t, act_dtype)) if act_dtype is not None else (lambda t: t)
    W = (lambda n: sd[n].to(x).to(act_dtype).to(x.dtype) if act_dtype is not None else sd[n].to(x))
    x = q(F.conv2d(x, W("features.conv0.weight"), stride=2, padding=3))
    x = q(F.relu(_bn(x, sd, "features.norm0", training, new_sd)))
    x = q(F.max_pool2d(x, 3, 2, 1))
    for b, n in enumerate(spec.block_config):
        for l in range(n):
            p = "features.denseblock%d.denselayer%d" % (b + 1, l + 1)
            x = q(x)
            h = q(F.relu(_bn(x, sd, p + ".norm1", training, new_sd)))
            h = q(F.conv2d(h, W(p + ".conv1.weight")))
            h = q(F.relu(_bn(h, sd, p + ".norm2", training, new_sd)))
            h = q(F.conv2d(h, W(p + ".conv2.weight"), padding=1))
            if masks is not None and p in masks:
                h = q(h * masks[p].to(x).permute(0, 3, 1, 2))
            x = torch.cat([x, h], 1)
        x = q(x)
        if b + 1 < len(spec.block_config):
            p = "features.transition%d" % (b + 1)
            x = F.relu(_bn(x, sd, p + ".norm", training, new_sd))
            if act_dtype is not None:       # the plan's order: pool (stored), then the 1x1 convolution
                x = q(F.conv2d(q(F.avg_pool2d(x, 2, 2)), W(p + ".conv.weight")))
            else:
                x = F.avg_pool2d(F.conv2d(x, W(p + ".conv.weight")), 2, 2)
    x = F.relu(_bn(x, sd, "features.norm5", training, new_sd))
    x = x.mean((2, 3))
    if head_mask is not None:
        x = x * head_mask.to(x)
    return F.linear(x, W("classifier.weight") if act_dtype is None else sd["classifier.weight"].to(x),
                    sd["classifier.bias"].to(x))


def train_grads(spec, sd, x, y, masks=None, head_mask=None, dtype=torch.float64, act_dtype=None, loss_scale=1.0,
                new_sd=None):
    """(loss, logits, {param name: gradient}) of one training forward / backward with the mean cross-entropy; with act_dtype
    the loss is multiplied by loss_scale before the backward (the rounded gradients are those of the scaled loss) and the
    gradients divided by it afterwards"""
    params = {n: sd[n].to(device=x.device, dtype=dtype).clone().requires_grad_(True) for n in sd
              if not n.endswith(("running_mean", "running_var", "num_batches_tracked"))}
    full = dict(sd)
    full.update(params)
    logits = forward(spec, full, x.to(dtype), True, masks, head_mask, new_sd=new_sd, act_dtype=act_dtype)
    loss = F.cross_entropy(logits, y)
    (loss * loss_scale).backward()
    return float(loss.detach()), logits.detach(), {n: p.grad.detach() / loss_scale for n, p in params.items()}
