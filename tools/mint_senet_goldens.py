"""Mint the SE-ResNet fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only, through oracle/ref_shims.py):

    python tools/mint_senet_goldens.py

senet_state_keys.json
        state_dict / named_parameters names and shapes of seresnet18/34/50/101/152 (dfd/timm/models/senet.py), num_classes 2,
        and seresnet50 at in_chans 12: the [name, shape] lists in full for seresnet18 and seresnet50, and for every entry their
        lengths and sha256 (tools/mint_tf_goldens.py `_entry`).
step_seresnet18_70x72.json
        two SGD train steps + eval of the reference seresnet18 at batch 4, 70x72 (tools/mint_multiclass_goldens.py's
        `mint_step_k`, synthetic weights of oracle/weights.py). The stem convolution gives 35x36: the ceil-mode stem pool makes
        17x18 of it where a padded pool would make 18x18, and clips its last window on the even axis.
step_seresnet50_64x64.json
        the same for seresnet50 at batch 4, 64x64.
step_seresnet101.json
        one step + eval of seresnet101 at batch 2, 64x64.
step_seresnet18_tame_70x72.json, step_seresnet50_tame_64x64.json, step_seresnet101_tame_64x64.json
        the same at batch 8 with the last BatchNorm gamma of every residual branch scaled by 0.2 (tests/senet_oracle.py
        `tame_state`, recorded as "tame"): the un-tamed steps amplify 16-bit rounding into changes of order one; these are the
        steps a 16-bit path is compared with.
Every model is built with drop_rate=0.0: SENet's default of 0.2 would draw dropout masks from torch's generator, which no other
implementation reproduces.
"""
import json
import os
import sys
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from deepfake_detection_b200.arch import SENET_ARCHS  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN  # noqa: E402

FULL = ("seresnet18", "seresnet50")


def mint_state_keys():
    from dfd.timm.models import create_model
    from mint_tf_goldens import _entry
    out = {a: _entry(create_model(a, num_classes=2), full=a in FULL) for a in SENET_ARCHS}
    out["seresnet50@in_chans12"] = _entry(create_model("seresnet50", num_classes=2, in_chans=12))
    with open(os.path.join(GOLDEN, "senet_state_keys.json"), "w") as f:
        json.dump(out, f)
    print("senet_state_keys.json:", len(out), "entries")


def mint_step(arch, batch, H, W, n_steps, tag, tame=False):
    """tools/mint_multiclass_goldens.py `mint_step_k` with create_model(..., drop_rate=0.0) and optionally the residual branches
    of the synthetic weights tamed"""
    import dfd.timm.models as RM
    import mint_multiclass_goldens as MM
    from senet_oracle import TAME, tame_state
    orig_create, orig_synth = RM.create_model, MM.synth_state
    RM.create_model = partial(orig_create, drop_rate=0.0)
    if tame:
        MM.synth_state = lambda spec, seed=0: tame_state(spec, orig_synth(spec, seed=seed))
    try:
        MM.mint_step_k(arch, batch, H, W, 2, n_steps=n_steps, tag=tag)
    finally:
        RM.create_model, MM.synth_state = orig_create, orig_synth
    path = os.path.join(GOLDEN, "step_%s%s.json" % (arch, tag))
    rec = json.load(open(path))
    rec["drop_rate"] = 0.0
    if tame:
        rec["tame"] = TAME
    with open(path, "w") as f:
        json.dump(rec, f)


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    mint_state_keys()
    mint_step("seresnet18", 4, 70, 72, 2, "_70x72")
    mint_step("seresnet50", 4, 64, 64, 2, "_64x64")
    mint_step("seresnet101", 2, 64, 64, 1, "")
    mint_step("seresnet18", 8, 70, 72, 2, "_tame_70x72", tame=True)
    mint_step("seresnet50", 8, 64, 64, 2, "_tame_64x64", tame=True)
    mint_step("seresnet101", 8, 64, 64, 1, "_tame_64x64", tame=True)


if __name__ == "__main__":
    main()
