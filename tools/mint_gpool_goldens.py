"""Mint the global-pool fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only).

    python tools/mint_gpool_goldens.py

Train steps, with the recipe of tools/mint_multiclass_goldens.py (synthetic weights of oracle/weights.py loaded into the
reference's own `create_model(..., global_pool=...)`, its own optimizers, losses and `accuracy`):

    step_efficientnet_b0_gp_max.json                 max,       K = 2, nn.CrossEntropyLoss, SGD
    step_efficientnet_b0_k5_gp_catavgmax_ls.json     catavgmax, K = 5, LabelSmoothingCrossEntropy(0.1), SGD
    step_resnet18_gp_avgmax.json                     avgmax,    K = 2, nn.CrossEntropyLoss, SGD

and state_keys_catavgmax.json: the reference's state_dict / named_parameters names and shapes of every native architecture
built with global_pool='catavgmax' (the classifier reads 2 x num_features), in the layout of state_keys.json.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))

from mint_multiclass_goldens import mint_step_k  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN  # noqa: E402


def mint_state_keys_catavgmax():
    from dfd.timm.models import create_model
    from dfd.timm.models.factory import create_deepfake_model_v4
    out = {}
    for arch in ("efficientnet_b0", "efficientnet_b4", "resnet18", "resnet50", "efficientnet_deepfake_v4"):
        if arch == "efficientnet_deepfake_v4":
            m = create_deepfake_model_v4(arch, num_classes=2, in_chans=12, global_pool="catavgmax")
        else:
            m = create_model(arch, num_classes=2, global_pool="catavgmax")
        out[arch] = dict(state=[[k, list(v.shape)] for k, v in m.state_dict().items()],
                         params=[[k, list(v.shape)] for k, v in m.named_parameters()],
                         n_params=sum(p.numel() for p in m.parameters()))
    with open(os.path.join(GOLDEN, "state_keys_catavgmax.json"), "w") as f:
        json.dump(out, f)
    print("state_keys_catavgmax.json:", {k: v["n_params"] for k, v in out.items()})


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    mint_step_k("efficientnet_b0", 4, 64, 64, 2, global_pool="max", tag="_gp_max")
    mint_step_k("efficientnet_b0", 4, 64, 64, 5, smoothing=0.1, global_pool="catavgmax", tag="_k5_gp_catavgmax_ls")
    mint_step_k("resnet18", 2, 64, 64, 2, global_pool="avgmax", tag="_gp_avgmax")
    mint_state_keys_catavgmax()


if __name__ == "__main__":
    main()
