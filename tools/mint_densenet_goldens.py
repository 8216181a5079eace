"""Mint the DenseNet fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only, through oracle/ref_shims.py):

    python tools/mint_densenet_goldens.py

densenet_state_keys.json
        counts and sha256 of the state_dict / named_parameters [name, shape] lists of densenet121 / 169 / 201 / 161
        (dfd/timm/models/densenet.py), num_classes 2, at in_chans 3, and of densenet121 at in_chans 12; densenet121's lists in
        full (tools/mint_tf_goldens.py `_entry`).
step_densenet121_72x88.json
        two SGD train steps + eval of densenet121 at batch 4, 72x88 (tools/mint_multiclass_goldens.py's `mint_step_k`,
        synthetic weights of oracle/weights.py): extents 36x44 -> 18x22 -> 9x11 -> 4x5 -> 2x2, so two transitions pool
        odd extents in floor mode.
step_densenet161_70x54.json
        one step + eval of densenet161 (growth 48) at batch 2, 70x54 (35x27 -> 18x14 -> 9x7 -> 4x3 -> 2x1).
step_densenet121_224.json
        one step + eval of densenet121 at batch 2, 224x224.
step_densenet121_drop_48.json
        one step of densenet121 with drop_rate 0.2 at batch 2, 48x48. Every F.dropout call of the reference is recorded: its
        keep mask, in call order (58 dense layers, then the classifier input), as packed bits in base64.
"""
import base64
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN  # noqa: E402

ARCHS = ("densenet121", "densenet169", "densenet201", "densenet161")


def mint_state_keys():
    from dfd.timm.models import create_model
    from mint_tf_goldens import _entry
    out = {a: _entry(create_model(a, num_classes=2), full=a == "densenet121") for a in ARCHS}
    out["densenet121@in_chans12"] = _entry(create_model("densenet121", num_classes=2, in_chans=12))
    with open(os.path.join(GOLDEN, "densenet_state_keys.json"), "w") as f:
        json.dump(out, f)
    print("densenet_state_keys.json:", len(out), "entries")


def mint_drop_step(batch=2, H=48, W=48, drop_rate=0.2):
    import torch.nn.functional as F
    from dfd.timm.models import create_model
    from dfd.timm.optim import create_optimizer
    from mint_multiclass_goldens import _args, _pick, _summ
    from deepfake_detection_b200.arch import get_spec
    from oracle.weights import synth_batch, synth_state
    torch.manual_seed(0)
    spec = get_spec("densenet121", num_classes=2)
    model = create_model("densenet121", num_classes=2, drop_rate=drop_rate)
    model.load_state_dict(synth_state(spec, seed=7), strict=True)
    model.train()
    optimizer = create_optimizer(_args(opt="sgd", lr=0.01, weight_decay=1e-4), model)
    masks, orig = [], F.dropout

    def recording_dropout(x, p=0.5, training=True, inplace=False):
        m = orig(torch.ones_like(x), p, training)        # the same draw F.dropout makes; m = keep / (1 - p)
        masks.append(m)
        return x * m

    F.dropout = recording_dropout
    try:
        x, y = synth_batch(batch, 3, H, W, seed=1234)
        out = model(x)
        loss = torch.nn.CrossEntropyLoss()(out, y)
        optimizer.zero_grad()
        loss.backward()
    finally:
        F.dropout = orig
    params = dict(model.named_parameters())
    pk = _pick(list(params), 6)
    grads = {k: _summ(params[k].grad) for k in pk}
    optimizer.step()
    rec = dict(arch="densenet121", batch=batch, H=H, W=W, num_classes=2, weight_seed=7, drop_rate=drop_rate, opt="sgd",
               lr=0.01, momentum=0.9, weight_decay=1e-4, torch=torch.__version__,
               masks=[dict(shape=list(m.shape), bits=base64.b64encode(np.packbits((m > 0).numpy().reshape(-1))).decode())
                      for m in masks],
               steps=[dict(logits=_summ(out, 32), loss=float(loss), grads=grads, params={k: _summ(params[k]) for k in pk})])
    with open(os.path.join(GOLDEN, "step_densenet121_drop_48.json"), "w") as f:
        json.dump(rec, f)
    print("step_densenet121_drop_48.json loss", float(loss), "masks", len(masks))


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    mint_state_keys()
    from mint_multiclass_goldens import mint_step_k
    mint_step_k("densenet121", 4, 72, 88, 2, tag="_72x88")
    mint_step_k("densenet161", 2, 70, 54, 2, n_steps=1, tag="_70x54")
    mint_step_k("densenet121", 2, 224, 224, 2, n_steps=1, tag="_224")
    mint_drop_step()


if __name__ == "__main__":
    main()
