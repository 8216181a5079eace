"""Mint the Xception fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only, through oracle/ref_shims.py):

    python tools/mint_xception_goldens.py

xception_state_keys.json
        state_dict / named_parameters names and shapes of xception (dfd/timm/models/xception.py), num_classes 2, at in_chans 3
        and 12: the [name, shape] lists in full and their lengths and sha256 (tools/mint_tf_goldens.py `_entry`).
step_xception_64x80.json
        two SGD train steps + eval of the reference xception at batch 4, 64x80 (tools/mint_multiclass_goldens.py's
        `mint_step_k`, synthetic weights of oracle/weights.py). The extents are 31x39 -> 29x37 -> 15x19 -> 8x10 -> 4x5 -> 2x3,
        so the max-pool windows of the strided blocks are clipped on odd extents.
step_xception_299.json
        one step + eval at batch 2, 299x299 (the model's own geometry).
step_xception_tame_64x80.json
        two steps + eval at batch 8, 64x80, with the last BatchNorm gamma of every block's `rep` scaled by 0.2
        (oracle/weights.py `tame_state`, recorded as "tame"): the un-tamed steps amplify 16-bit rounding into changes of
        order one; this is the step a 16-bit path is compared with.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN  # noqa: E402


def mint_state_keys():
    from dfd.timm.models import create_model
    from mint_tf_goldens import _entry
    out = {"xception": _entry(create_model("xception", num_classes=2), full=True),
           "xception@in_chans12": _entry(create_model("xception", num_classes=2, in_chans=12), full=True)}
    with open(os.path.join(GOLDEN, "xception_state_keys.json"), "w") as f:
        json.dump(out, f)
    print("xception_state_keys.json:", len(out), "entries")


def mint_tamed(batch, H, W, n_steps, tag):
    import mint_multiclass_goldens as MM
    from oracle.weights import TAME, tame_state
    orig = MM.synth_state
    MM.synth_state = lambda spec, seed=0: tame_state(spec, orig(spec, seed=seed))
    try:
        MM.mint_step_k("xception", batch, H, W, 2, n_steps=n_steps, tag=tag)
    finally:
        MM.synth_state = orig
    path = os.path.join(GOLDEN, "step_xception%s.json" % tag)
    rec = json.load(open(path))
    rec["tame"] = TAME
    with open(path, "w") as f:
        json.dump(rec, f)


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    mint_state_keys()
    from mint_multiclass_goldens import mint_step_k
    mint_step_k("xception", 4, 64, 80, 2, tag="_64x80")
    mint_step_k("xception", 2, 299, 299, 2, n_steps=1, tag="_299")
    mint_tamed(8, 64, 80, 2, "_tame_64x80")


if __name__ == "__main__":
    main()
