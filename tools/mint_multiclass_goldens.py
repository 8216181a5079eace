"""Mint the K-class train-step fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only).

    python tools/mint_multiclass_goldens.py

The same recipe as oracle/mint_goldens.py's `mint_step` (synthetic weights of oracle/weights.py loaded into the
reference's own `create_model`, its own optimizers, losses and `accuracy`), with the class count as a parameter:

    step_efficientnet_b0_k5_ls.json            K = 5,    LabelSmoothingCrossEntropy(0.1), SGD
    step_efficientnet_b0_k5_soft_rmsprop.json  K = 5,    SoftTargetCrossEntropy (mixup-style targets), RMSpropTF
    step_resnet18_k1000.json                   K = 1000, nn.CrossEntropyLoss, SGD

Compact records (a few kB): logits as a summary (norm, sum, up to 32 sampled elements), and summaries of the gradients /
updated values of a fixed subset of tensors only - six parameters spread evenly over the network plus the classifier,
and three BatchNorm running statistics - rounded to 9 significant digits.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepfake_detection_b200.arch import get_spec  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN, _args  # noqa: E402
from oracle.weights import synth_batch, synth_state  # noqa: E402


def _r(v):
    return float("%.9g" % v)


def _summ(t, n=8):
    f = t.detach().reshape(-1).to(torch.float64)
    idx = torch.linspace(0, f.numel() - 1, steps=min(n, f.numel())).round().long()
    return dict(norm=_r(f.norm()), sum=_r(f.sum()), samples=[_r(v) for v in f[idx].tolist()], idx=idx.tolist())


def _pick(names, k):
    """k names spread evenly over the list, plus the last two (the classifier weight and bias for parameters)"""
    n = len(names)
    return [names[i] for i in sorted({round(j * (n - 1) / (k - 1)) for j in range(k)} | {n - 2, n - 1})]


def mint_step_k(arch, batch, H, W, num_classes, n_steps=2, smoothing=0.0, opt_name="sgd", soft=False, tag="",
                global_pool="avg"):
    from dfd.timm.loss import LabelSmoothingCrossEntropy, SoftTargetCrossEntropy
    from dfd.timm.models import create_model
    from dfd.timm.optim import create_optimizer
    from dfd.timm.utils import accuracy
    torch.manual_seed(0)
    spec = get_spec(arch, num_classes=num_classes, global_pool=global_pool)
    model = create_model(arch, num_classes=num_classes, global_pool=global_pool)
    model.load_state_dict(synth_state(spec, seed=7), strict=True)
    model.train()
    lr = 0.01 if opt_name == "sgd" else 1e-3
    wd = 1e-4
    optimizer = create_optimizer(_args(opt=opt_name, lr=lr, weight_decay=wd), model)
    if soft:
        loss_fn = SoftTargetCrossEntropy()
    elif smoothing > 0:
        loss_fn = LabelSmoothingCrossEntropy(smoothing)
    else:
        loss_fn = torch.nn.CrossEntropyLoss()
    params = dict(model.named_parameters())
    buffers = {k: b for k, b in model.named_buffers() if not k.endswith("num_batches_tracked")}
    pk, bk = _pick(list(params), 6), _pick([k for k in buffers if k.endswith("running_var")], 2)
    rec = dict(arch=arch, batch=batch, H=H, W=W, num_classes=num_classes, weight_seed=7, opt=opt_name, lr=lr,
               momentum=0.9, weight_decay=wd, smoothing=smoothing, soft=soft, torch=torch.__version__, steps=[])
    if global_pool != "avg":
        rec["global_pool"] = global_pool
    for step in range(n_steps):
        x, y = synth_batch(batch, 3, H, W, seed=1234 + step, soft=soft, num_classes=num_classes)
        out = model(x)
        loss = loss_fn(out, y)
        prec1 = accuracy(out, y, topk=(1,))
        optimizer.zero_grad()
        loss.backward()
        grads = {k: _summ(params[k].grad) for k in pk}
        optimizer.step()
        rec["steps"].append(dict(logits=_summ(out, 32), loss=float(loss), prec1=float(prec1), grads=grads,
                                 params={k: _summ(params[k]) for k in pk},
                                 buffers={k: _summ(buffers[k].float()) for k in bk}))
    model.eval()
    with torch.no_grad():
        x, y = synth_batch(batch, 3, H, W, seed=999, num_classes=num_classes)
        out = model(x)
        rec["eval"] = dict(logits=_summ(out, 32), loss=float(torch.nn.CrossEntropyLoss()(out, y)))
    name = "step_%s%s.json" % (arch, tag)
    with open(os.path.join(GOLDEN, name), "w") as f:
        json.dump(rec, f)
    print(name, "loss", [s["loss"] for s in rec["steps"]], "eval", rec["eval"]["loss"])


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    mint_step_k("efficientnet_b0", 4, 64, 64, 5, smoothing=0.1, tag="_k5_ls")
    mint_step_k("efficientnet_b0", 4, 64, 64, 5, soft=True, opt_name="rmsproptf", tag="_k5_soft_rmsprop")
    mint_step_k("resnet18", 2, 64, 64, 1000, tag="_k1000")


if __name__ == "__main__":
    main()
