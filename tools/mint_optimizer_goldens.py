"""Mint the fixtures of the radam / adadelta / rmsprop / novograd / nvnovograd optimizers under tests/golden/ FROM THE
UNMODIFIED REFERENCE (CPU only, through oracle/ref_shims.py):

    python tools/mint_optimizer_goldens.py

optimizers_ext.json: the reference factory (dfd/timm/optim/optim_factory.py:26-100) on a toy module with two parameter
groups ([bias] without decay, [w, k] with it), weight_decay 1e-2 and opt_eps 1e-3, over 10 steps of fixed gradients, so that
RAdam crosses into its rectified steps (step 6 on). The lr of every group halves before step 5 (a scheduler update). `k`'s
gradient is all zero at step 1 (NvNovoGrad's exp_avg_sq == 0 branch, also at step 2). Extra runs:
  novograd_single   filter_bias_and_bn=False: one group, and NovoGrad's constructor decay is the weight decay
  radam_group_lrs   group 1's lr doubled: the step size of every group follows group 0's lr (radam.py:54-70)
Every run records the parameters after each step, the groups' weight decays, the final state_dict (tensors as lists) and,
for NovoGrad, the constructor decay the factory passed.

step_efficientnet_b0_radam.json, step_resnet18_nvnovograd.json: two train steps through the reference model, factory and
loss (tools/mint_multiclass_goldens.py's recipe, lr 1e-3, weight decay 1e-4).
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN, _args  # noqa: E402

KINDS = ("radam", "adadelta", "rmsprop", "novograd", "nvnovograd")
LR, WD, EPS, STEPS, LR_CHANGE = 1e-2, 1e-2, 1e-3, 10, 4


class Toy(torch.nn.Module):
    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(3)
        self.w = torch.nn.Parameter(torch.randn(5, 7, generator=g))
        self.bias = torch.nn.Parameter(torch.randn(7, generator=g))
        self.k = torch.nn.Parameter(torch.randn(4, 1, 3, 3, generator=g))


def toy_grads(step, gen):
    """the gradients of one step, in named_parameters order (draw order fixed), `k` zero at step 0"""
    out = {}
    for name, shape in (("w", (5, 7)), ("bias", (7,)), ("k", (4, 1, 3, 3))):
        out[name] = torch.randn(shape, generator=gen)
    out["k"] = out["k"] * 0 if step == 0 else out["k"]
    return out


def _state_json(opt, model):
    ids = {id(p): n for n, p in model.named_parameters()}
    out = {}
    for p, st in opt.state.items():
        out[ids[id(p)]] = {k: (v.reshape(-1).tolist() if torch.is_tensor(v) else v) for k, v in st.items()}
    return out


def run(kind, filter_bias_and_bn=True, group_lr_scale=None):
    from dfd.timm.optim import create_optimizer
    m = Toy()
    opt = create_optimizer(_args(opt=kind, lr=LR, weight_decay=WD, opt_eps=EPS), m, filter_bias_and_bn=filter_bias_and_bn)
    if group_lr_scale:
        for g, s in zip(opt.param_groups, group_lr_scale):
            g["lr"] *= s
    gen = torch.Generator().manual_seed(11)
    hist, lrs = [], []
    for step in range(STEPS):
        if step == LR_CHANGE:
            for g in opt.param_groups:
                g["lr"] *= 0.5
        grads = toy_grads(step, gen)
        for n, p in m.named_parameters():
            p.grad = grads[n].clone()
        lrs.append([g["lr"] for g in opt.param_groups])
        opt.step()
        hist.append({n: p.detach().reshape(-1).tolist() for n, p in m.named_parameters()})
    rec = dict(kind=kind, lr=LR, weight_decay=WD, eps=EPS, momentum=0.9, filter_bias_and_bn=filter_bias_and_bn,
               group_lr_scale=group_lr_scale, lrs=lrs, hist=hist,
               group_weight_decay=[g["weight_decay"] for g in opt.param_groups],
               group_sizes=[len(g["params"]) for g in opt.param_groups], state=_state_json(opt, m))
    if kind == "novograd":
        rec["ctor_weight_decay"] = opt._wd
    return rec


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    out = {k: run(k) for k in KINDS}
    out["novograd_single"] = run("novograd", filter_bias_and_bn=False)
    out["radam_group_lrs"] = run("radam", group_lr_scale=[1.0, 2.0])
    with open(os.path.join(GOLDEN, "optimizers_ext.json"), "w") as f:
        json.dump(out, f)
    print("optimizers_ext.json:", {k: (v["group_sizes"], v.get("ctor_weight_decay")) for k, v in out.items()})
    from mint_multiclass_goldens import mint_step_k
    mint_step_k("efficientnet_b0", 4, 64, 64, 2, opt_name="radam", tag="_radam")
    mint_step_k("resnet18", 4, 64, 64, 2, opt_name="nvnovograd", tag="_nvnovograd")


if __name__ == "__main__":
    main()
