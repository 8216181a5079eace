"""CPU restatement of the optimizers of optim_factory.py:26-100 beyond sgd / adam / adamw / rmsproptf, as plain torch-fp32 CPU
arithmetic (test infrastructure, like oracle/train.py, whose `optimizer_step` keeps the four original kinds):

  radam       dfd/timm/optim/radam.py:21-82 (N_sma / step size from the step and group 0's lr, :54-70, shared by every
              group through self.buffer; decoupled decay first with the tensor's own lr, :73-74; N_sma < 5: no denominator)
  adadelta    torch.optim.Adadelta(rho 0.9), _single_tensor_adadelta (L2 decay into the gradient)
  rmsprop     torch.optim.RMSprop(alpha 0.9), _single_tensor_rmsprop (square_avg from zeros, eps outside the sqrt)
  novograd    dfd/timm/optim/novograd.py:24-77 (the constructor's decay, betas (0.95, 0.98) and eps; the first step of a
              freshly built optimizer re-initialises every tensor, :30-46)
  nvnovograd  dfd/timm/optim/nvnovograd.py:59-117 (exp_avg_sq copied from the norm while it is 0, :96-99; the group's decay)

Parameter groups follow optim_factory.py:11-38: with `single_group` every tensor gets `weight_decay` (filter_bias_and_bn=False);
otherwise 1-D tensors and biases get 0, and NovoGrad, built with weight_decay=0 by the factory, decays nothing at all.
"""
import math

import torch

from deepfake_detection_b200.arch import is_no_decay
from oracle import train as OT

KINDS = ("radam", "adadelta", "rmsprop", "novograd", "nvnovograd")
DEFAULT_BETAS = {"radam": (0.9, 0.999), "novograd": (0.95, 0.98), "nvnovograd": (0.95, 0.98)}


class OptState:
    """weight_decay: as the optimizer receives it (for radam: already divided by the initial lr, optim_factory.py:29-33)"""

    def __init__(self, kind, lr=1e-3, momentum=0.9, weight_decay=1e-4, eps=1e-8, betas=None, alpha=0.9, rho=0.9,
                 single_group=False):
        assert kind in KINDS, kind
        self.kind, self.lr, self.momentum, self.weight_decay, self.eps = kind, lr, momentum, weight_decay, eps
        self.betas = betas or DEFAULT_BETAS.get(kind)
        self.alpha, self.rho, self.single_group = alpha, rho, single_group
        self.lr_nodecay = None          # lr of group 0 when it differs from `lr` (RAdam's shared step size)
        self.step = 0
        self.state = {}
        self.initialized = False        # NovoGrad's _momentum_initialized (not part of its state_dict)

    def group_wd(self, name, p):
        return self.weight_decay if self.single_group or not is_no_decay(name, tuple(p.shape)) else 0.0

    def novograd_wd(self):
        return self.weight_decay if self.single_group else 0.0


@torch.no_grad()
def optimizer_step(opt, params, grads, lrs=None):
    """params / grads: dict name -> tensor (named_parameters order). Updates params in place. `lrs` (optional): name -> lr."""
    if not isinstance(opt, OptState):
        return OT.optimizer_step(opt, params, grads)
    opt.step += 1
    lr_of = (lambda n: lrs[n]) if lrs else (lambda n: opt.lr)
    if opt.kind == "novograd":
        _novograd(opt, params, grads, lr_of)
        return
    for name, p in params.items():
        g = grads[name]
        wd, lr = opt.group_wd(name, p), lr_of(name)
        st = opt.state.setdefault(name, {})
        if opt.kind == "radam":
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
    eps, wd = opt.eps, opt.novograd_wd()
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


def train_step(spec, sd, x, target, opt, smoothing=0.0, act_dtype=None):
    """oracle.train.train_step with the optimizer of this module (same forward / loss / backward)"""
    out = OT.train_step(spec, sd, x, target, None, smoothing=smoothing, act_dtype=act_dtype)
    params, _ = OT.split_state(spec, sd)
    optimizer_step(opt, params, out["grads"])
    return out

