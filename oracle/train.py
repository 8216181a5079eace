"""CPU ORACLE — TEST INFRASTRUCTURE (see oracle/model.py header).

Restates one iteration of the reference's hot loop (dfd/runners/train.py:610-649) and the optimizers
of optim_factory.py:26-100, as plain torch-fp32 CPU arithmetic:

  sgd         : torch.optim.SGD(nesterov=True) as built by dfd/timm/optim/optim_factory.py:48-50
  adam        : torch.optim.Adam (optim_factory.py:51-53; L2 decay added to the gradient)
  adamw       : dfd/timm/optim/adamw.py:55-117 (decoupled decay first, :72)
  rmsproptf   : dfd/timm/optim/rmsprop_tf.py:57-122 (square_avg init ONES :80, eps inside sqrt :107,
                lr folded into the momentum buffer :112-114)
  radam       : dfd/timm/optim/radam.py:21-82 (N_sma / step size from the step and group 0's lr, :54-70, shared by every
                group through self.buffer; decoupled decay first with the tensor's own lr, :73-74; N_sma < 5: no denominator)
  adadelta    : torch.optim.Adadelta(rho 0.9), _single_tensor_adadelta (L2 decay into the gradient)
  rmsprop     : torch.optim.RMSprop(alpha 0.9), _single_tensor_rmsprop (square_avg from zeros, eps outside the sqrt)
  novograd    : dfd/timm/optim/novograd.py:24-77 (the constructor's decay, betas (0.95, 0.98) and eps; the first step of a
                freshly built optimizer re-initialises every tensor, :30-46)
  nvnovograd  : dfd/timm/optim/nvnovograd.py:59-117 (exp_avg_sq copied from the norm while it is 0, :96-99; the group's decay)
  param groups: optim_factory.py:11-38: with `single_group` every tensor gets `weight_decay` (filter_bias_and_bn=False);
                otherwise 1-D tensors and biases get 0, and NovoGrad, built with weight_decay=0 by the factory, decays
                nothing at all
  train_step  : train.py:621-637 (forward, loss, prec1, zero_grad, backward, step)
  validate_step : train.py:719-731
"""
import math

import torch

from deepfake_detection_b200.arch import is_no_decay, param_entries

from . import model as M

BASE_KINDS = ("sgd", "adam", "adamw", "rmsproptf")
EXT_KINDS = ("radam", "adadelta", "rmsprop", "novograd", "nvnovograd")
KINDS = BASE_KINDS + EXT_KINDS
DEFAULT_BETAS = {"radam": (0.9, 0.999), "novograd": (0.95, 0.98), "nvnovograd": (0.95, 0.98)}


class OptState:
    """Optimizer state keyed by parameter name (momentum_buffer / exp_avg / exp_avg_sq / square_avg / ...).
    weight_decay: as the optimizer receives it (for adamw and radam: already divided by the initial lr,
    optim_factory.py:29-33)."""

    def __init__(self, kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, eps=1e-8, betas=None, alpha=0.9, rho=0.9,
                 single_group=False):
        assert kind in KINDS, kind
        self.kind, self.lr, self.momentum, self.weight_decay, self.eps = kind, lr, momentum, weight_decay, eps
        self.betas = betas or DEFAULT_BETAS.get(kind, (0.9, 0.999))
        self.alpha, self.rho, self.single_group = alpha, rho, single_group
        self.lr_nodecay = None          # lr of group 0 when it differs from `lr` (RAdam's shared step size)
        self.step = 0
        self.state = {}
        self.initialized = False        # NovoGrad's _momentum_initialized (not part of its state_dict)

    def group_wd(self, name, p):
        return self.weight_decay if self.single_group or not is_no_decay(name, tuple(p.shape)) else 0.0


@torch.no_grad()
def optimizer_step(opt, params, grads, lrs=None):
    """params / grads: dict name -> tensor (named_parameters order). Updates params in place. `lrs` (optional): name -> lr."""
    opt.step += 1
    lr_of = (lambda n: lrs[n]) if lrs else (lambda n: opt.lr)
    if opt.kind == "novograd":
        _novograd(opt, params, grads, lr_of)
        return
    for name, p in params.items():
        g = grads[name]
        wd, lr = opt.group_wd(name, p), lr_of(name)
        st = opt.state.setdefault(name, {})
        if opt.kind == "sgd":
            if wd != 0:
                g = g.add(p, alpha=wd)
            if "momentum_buffer" not in st:
                buf = st["momentum_buffer"] = g.clone()
            else:
                buf = st["momentum_buffer"]
                buf.mul_(opt.momentum).add_(g)
            g = g.add(buf, alpha=opt.momentum)  # nesterov
            p.add_(g, alpha=-lr)
        elif opt.kind in ("adam", "adamw"):
            b1, b2 = opt.betas
            if opt.kind == "adamw":
                p.mul_(1 - lr * wd)
            elif wd != 0:
                g = g.add(p, alpha=wd)
            if "exp_avg" not in st:
                st["exp_avg"] = torch.zeros_like(p)
                st["exp_avg_sq"] = torch.zeros_like(p)
            st["exp_avg"].mul_(b1).add_(g, alpha=1 - b1)
            st["exp_avg_sq"].mul_(b2).addcmul_(g, g, value=1 - b2)
            bc1 = 1 - b1 ** opt.step
            bc2 = 1 - b2 ** opt.step
            denom = (st["exp_avg_sq"].sqrt() / math.sqrt(bc2)).add_(opt.eps)
            p.addcdiv_(st["exp_avg"], denom, value=-lr / bc1)
        elif opt.kind == "rmsproptf":
            if wd != 0:
                g = g.add(p, alpha=wd)
            if "square_avg" not in st:
                st["square_avg"] = torch.ones_like(p)
                st["momentum_buffer"] = torch.zeros_like(p)
            sq = st["square_avg"]
            sq.add_(g.pow(2) - sq, alpha=1 - opt.alpha)
            avg = sq.add(opt.eps).sqrt_()
            if opt.momentum > 0:
                buf = st["momentum_buffer"]
                buf.mul_(opt.momentum).addcdiv_(g, avg, value=lr)
                p.add_(-buf)
            else:
                p.addcdiv_(g, avg, value=-lr)
        elif opt.kind == "radam":
            b1, b2 = opt.betas
            if not st:
                st.update(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p))
            st["exp_avg_sq"].mul_(b2).addcmul_(g, g, value=1 - b2)
            st["exp_avg"].mul_(b1).add_(g, alpha=1 - b1)
            st["step"] += 1
            t = st["step"]
            lr0 = opt.lr_nodecay if opt.lr_nodecay is not None else opt.lr
            b2t = b2 ** t
            nmax = 2 / (1 - b2) - 1
            nsma = nmax - 2 * t * b2t / (1 - b2t)
            if nsma >= 5:
                ss = lr0 * math.sqrt((1 - b2t) * (nsma - 4) / (nmax - 4) * (nsma - 2) / nsma * nmax / (nmax - 2)) / (1 - b1 ** t)
            else:
                ss = lr0 / (1 - b1 ** t)
            if wd != 0:
                p.add_(p, alpha=-wd * lr)
            if nsma >= 5:
                p.addcdiv_(st["exp_avg"], st["exp_avg_sq"].sqrt().add_(opt.eps), value=-ss)
            else:
                p.add_(st["exp_avg"], alpha=-ss)
        elif opt.kind == "adadelta":
            if not st:
                st.update(square_avg=torch.zeros_like(p), acc_delta=torch.zeros_like(p))
            if wd != 0:
                g = g.add(p, alpha=wd)
            st["square_avg"].mul_(opt.rho).addcmul_(g, g, value=1 - opt.rho)
            std = st["square_avg"].add(opt.eps).sqrt_()
            delta = st["acc_delta"].add(opt.eps).sqrt_().div_(std).mul_(g)
            st["acc_delta"].mul_(opt.rho).addcmul_(delta, delta, value=1 - opt.rho)
            p.add_(delta, alpha=-lr)
        elif opt.kind == "rmsprop":
            if not st:
                st["square_avg"] = torch.zeros_like(p)
                if opt.momentum > 0:
                    st["momentum_buffer"] = torch.zeros_like(p)
            if wd != 0:
                g = g.add(p, alpha=wd)
            st["square_avg"].mul_(opt.alpha).addcmul_(g, g, value=1 - opt.alpha)
            avg = st["square_avg"].sqrt().add_(opt.eps)
            if opt.momentum > 0:
                st["momentum_buffer"].mul_(opt.momentum).addcdiv_(g, avg)
                p.add_(st["momentum_buffer"], alpha=-lr)
            else:
                p.addcdiv_(g, avg, value=-lr)
        else:  # nvnovograd
            b1, b2 = opt.betas
            if not st:
                st.update(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros([]))
            st["step"] += 1
            norm = torch.sum(torch.pow(g, 2))
            if st["exp_avg_sq"] == 0:
                st["exp_avg_sq"].copy_(norm)
            else:
                st["exp_avg_sq"].mul_(b2).add_(norm, alpha=1 - b2)
            gg = g / st["exp_avg_sq"].sqrt().add(opt.eps)
            if wd != 0:
                gg = gg.add(p, alpha=wd)
            st["exp_avg"].mul_(b1).add_(gg)
            p.add_(st["exp_avg"], alpha=-lr)


def _novograd(opt, params, grads, lr_of):
    b1, b2 = opt.betas
    eps, wd = opt.eps, (opt.weight_decay if opt.single_group else 0.0)
    if not opt.initialized:
        for name, p in params.items():
            g = grads[name]
            v = torch.norm(g) ** 2
            opt.state[name] = dict(step=0, v=v, m=g / (torch.sqrt(v) + eps) + wd * p, grad_ema=None)
        opt.initialized = True
    for name, p in params.items():
        st = opt.state[name]
        st["step"] += 1
        g = grads[name].clone()                      # the reference scales p.grad in place; the caller's gradient stays
        g2 = torch.norm(g) ** 2
        ge = g2 if st["grad_ema"] is None else st["grad_ema"] * b2 + g2 * (1. - b2)
        g *= 1.0 / (torch.sqrt(ge) + eps)
        g2 = torch.norm(g) ** 2
        st["v"] = b2 * st["v"] + (1. - b2) * g2
        st["m"] = b1 * st["m"] + (g / (torch.sqrt(st["v"]) + eps) + wd * p)
        st["grad_ema"] = ge
        t = st["step"]
        p.add_(st["m"], alpha=-(lr_of(name) * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)))


def split_state(spec, sd):
    """-> (params dict in named_parameters order, buffers dict)"""
    pnames = [n for n, _, _ in param_entries(spec)]
    params = {n: sd[n] for n in pnames}
    buffers = {n: t for n, t in sd.items() if n not in params}
    return params, buffers


def train_step(spec, sd, x, target, opt=None, smoothing=0.0, bn=None, act_dtype=None, taps=None,
               grad_hook=None, drop_masks=None, dropout_mask=None, drop_block=None):
    """One iteration of train.py:621-637 on CPU for any spec of `arch.get_spec`. `sd` tensors are updated in place.
    Without `bn`, BatchNorm trains with momentum 0.1 and the spec's eps (model.default_bn_eps).
    Returns dict(logits, loss, prec1, grads)."""
    params, _ = split_state(spec, sd)
    for p in params.values():
        p.requires_grad_(True)
        p.grad = None
    bn = bn or M.BNState(training=True, eps=M.default_bn_eps(spec))
    masks = dict(drop_masks=drop_masks, dropout_mask=dropout_mask, drop_block=drop_block)
    logits = M.forward(spec, sd, x, bn, act_dtype, taps, **{k: m for k, m in masks.items() if m is not None})
    loss = M.cross_entropy(logits, target, smoothing)
    prec1 = M.accuracy_top1(logits.detach(), target)
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in params.items()}
    for p in params.values():
        p.requires_grad_(False)
        p.grad = None
    if grad_hook is not None:
        grad_hook(grads)  # e.g. the DDP mean all-reduce
    if opt is not None:
        optimizer_step(opt, params, grads)
    return dict(logits=logits.detach(), loss=loss.detach(), prec1=prec1, grads=grads)


@torch.no_grad()
def validate_step(spec, sd, x, target, bn_eps=None, act_dtype=None):
    """`bn_eps`: None for the spec's own (model.default_bn_eps)"""
    bn = M.BNState(training=False, eps=M.default_bn_eps(spec) if bn_eps is None else bn_eps)
    logits = M.forward(spec, sd, x, bn, act_dtype)
    return dict(logits=logits, loss=M.cross_entropy(logits, target, 0.0), prec1=M.accuracy_top1(logits, target))
