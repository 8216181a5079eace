"""Mint the fixtures of the dense ResNet family under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only, through
oracle/ref_shims.py):

    python tools/mint_resnet_family_goldens.py

resnet_family_state_keys.json
        state_dict / named_parameters names and shapes of resnet26, resnet34, resnet101, resnet152, tv_resnet34, tv_resnet50,
        wide_resnet50_2, wide_resnet101_2, resnet26d and resnet50d (resnet.py:483-625), num_classes 2, and resnet50d at
        in_chans 12: the [name, shape] lists in full for resnet26d and wide_resnet50_2, and for every entry their lengths and
        the sha256 of their compact JSON (json.dumps(..., separators=(",", ":"))).
step_resnet26d_72x88.json
        two SGD train steps + eval of the reference resnet26d at batch 4, 72x88 (tools/mint_multiclass_goldens.py's
        `mint_step_k`, synthetic weights of oracle/weights.py). The average-pool shortcuts pool 18x22 -> 9x11, 9x11 -> 5x6 and
        5x6 -> 3x3, so windows are clipped in both axes.
step_resnet50d.json, step_resnet34.json, step_wide_resnet50_2.json
        the same at batch 4, 64x64.
step_resnet101.json
        one step + eval at batch 2, 64x64.
step_resnet26d_tame_104x88.json, step_resnet34_tame_96.json, step_wide_resnet50_2_tame_96.json, step_resnet101_tame_96.json
        the same at batch 8 with the last BatchNorm gamma of every residual branch scaled by 0.2
        (tests/resnet_family_oracle.py `tame_state`, recorded as "tame"): resnet26d at 104x88 (pools 26x22 -> 13x11,
        13x11 -> 7x6 and 7x6 -> 4x3), the others at 96x96, resnet101 one step. The un-tamed steps above amplify 16-bit
        rounding into changes of order one; these are the steps a 16-bit path is compared with.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from deepfake_detection_b200.arch import RESNET_ARCHS  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN  # noqa: E402

FULL = ("resnet26d", "wide_resnet50_2")


def mint_state_keys():
    from dfd.timm.models import create_model
    from mint_tf_goldens import _entry
    out = {a: _entry(create_model(a, num_classes=2), full=a in FULL) for a in RESNET_ARCHS}
    out["resnet50d@in_chans12"] = _entry(create_model("resnet50d", num_classes=2, in_chans=12))
    with open(os.path.join(GOLDEN, "resnet_family_state_keys.json"), "w") as f:
        json.dump(out, f)
    print("resnet_family_state_keys.json:", len(out), "entries")


def mint_tamed(arch, batch, H, W, n_steps, tag):
    """tools/mint_multiclass_goldens.py `mint_step_k` with the residual branches of the synthetic weights tamed"""
    import mint_multiclass_goldens as MM
    from resnet_family_oracle import TAME, tame_state
    orig = MM.synth_state
    MM.synth_state = lambda spec, seed=0: tame_state(spec, orig(spec, seed=seed))
    try:
        MM.mint_step_k(arch, batch, H, W, 2, n_steps=n_steps, tag=tag)
    finally:
        MM.synth_state = orig
    path = os.path.join(GOLDEN, "step_%s%s.json" % (arch, tag))
    rec = json.load(open(path))
    rec["tame"] = TAME
    with open(path, "w") as f:
        json.dump(rec, f)


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    mint_state_keys()
    from mint_multiclass_goldens import mint_step_k
    mint_step_k("resnet26d", 4, 72, 88, 2, tag="_72x88")
    for arch in ("resnet50d", "resnet34", "wide_resnet50_2"):
        mint_step_k(arch, 4, 64, 64, 2)
    mint_step_k("resnet101", 2, 64, 64, 2, n_steps=1)
    mint_tamed("resnet26d", 8, 104, 88, 2, "_tame_104x88")
    mint_tamed("resnet34", 8, 96, 96, 2, "_tame_96")
    mint_tamed("wide_resnet50_2", 8, 96, 96, 2, "_tame_96")
    mint_tamed("resnet101", 8, 96, 96, 1, "_tame_96")


if __name__ == "__main__":
    main()
