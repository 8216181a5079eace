"""Mint the fixtures of the TensorFlow-ported EfficientNets under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only,
through oracle/ref_shims.py):

    python tools/mint_tf_goldens.py

tf_state_keys.json      state_dict / named_parameters names and shapes of all 24 tf_efficientnet_b0..b7 (+ _ap, _ns)
                        entrypoints (efficientnet.py:1265-1530), num_classes 2, and the tf_efficientnet_b7 at in_chans 12:
                        the [name, shape] lists in full for tf_efficientnet_b0, and for every entry their lengths and the
                        sha256 of their compact JSON (json.dumps(..., separators=(",", ":"))), which keeps the file small.
tf_pad_same.json        the (top, left) pad and the output extent of every Conv2dSame layer that pads dynamically (the
                        stride-2 stem and depthwise convolutions), recorded from the reference's own `pad_same`
                        (layers/padding.py) during a forward: every size at its default resolution, B0 at an odd size
                        (225², all extents odd) and at two non-square sizes (224x225, 66x96).
step_tf_efficientnet_b0_64x96.json, step_tf_efficientnet_b0_66x96.json
                        two SGD train steps of the reference tf_efficientnet_b0 (tools/mint_multiclass_goldens.py's
                        `mint_step_k`, synthetic weights of oracle/weights.py). At 64x96 every stride-2 extent is even in
                        both axes; at 66x96 H is asymmetric at the stem only (33 is odd) and W at every stride-2 layer.
tf_eval_b0_224.json     eval-mode logits of the reference tf_efficientnet_b0 at 224² (batch 4, weights synth_state(seed=7),
                        running statistics included), the full [4, 2] tensor.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from deepfake_detection_b200.arch import TF_ARCHS, get_spec  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN  # noqa: E402
from oracle.weights import synth_batch, synth_state  # noqa: E402

PAD_CASES = [(a, None, None) for a in TF_ARCHS[:8]] + [("tf_efficientnet_b0", 225, 225), ("tf_efficientnet_b0", 224, 225),
                                                      ("tf_efficientnet_b0", 66, 96)]


def _digest(entries):
    import hashlib
    return hashlib.sha256(json.dumps(entries, separators=(",", ":")).encode()).hexdigest()


def _entry(m, full=False):
    state = [[k, list(v.shape)] for k, v in m.state_dict().items()]
    params = [[k, list(v.shape)] for k, v in m.named_parameters()]
    out = dict(n_state=len(state), n_param_tensors=len(params), state_sha256=_digest(state), params_sha256=_digest(params),
               n_params=sum(p.numel() for p in m.parameters()))
    if full:
        out.update(state=state, params=params)
    return out


def mint_state_keys():
    from dfd.timm.models import create_model
    out = {a: _entry(create_model(a, num_classes=2), full=a == "tf_efficientnet_b0") for a in TF_ARCHS}
    out["tf_efficientnet_b7@in_chans12"] = _entry(create_model("tf_efficientnet_b7", num_classes=2, in_chans=12))
    with open(os.path.join(GOLDEN, "tf_state_keys.json"), "w") as f:
        json.dump(out, f)
    print("tf_state_keys.json:", len(out), "entries")


def mint_pad_same():
    """Conv2dSame.forward -> conv2d_same -> pad_same -> F.pad([left, right, top, bottom]): record the pad list of each call"""
    import importlib
    import torch.nn.functional as F
    from dfd.timm.models import create_model
    conv2d_same = importlib.import_module("dfd.timm.models.layers.conv2d_same")
    padding = importlib.import_module("dfd.timm.models.layers.padding")
    calls, orig_pad, orig_same = [], F.pad, padding.pad_same

    def rec_same(x, k, s, d=(1, 1)):
        calls.append(dict(h=int(x.shape[-2]), w=int(x.shape[-1]), k=int(k[0]), s=int(s[0]), pad=[0, 0, 0, 0]))
        return orig_same(x, k, s, d)

    def rec_pad(x, pad, *a, **kw):
        if calls and calls[-1]["pad"] == [0, 0, 0, 0]:
            calls[-1]["pad"] = [int(v) for v in pad]
        return orig_pad(x, pad, *a, **kw)

    out = []
    conv2d_same.pad_same, F.pad = rec_same, rec_pad
    try:
        for arch, H, W in PAD_CASES:
            m = create_model(arch, num_classes=2).eval()
            res = m.default_cfg["input_size"][1]
            H, W = H or res, W or res
            del calls[:]
            with torch.no_grad():
                y = m.forward_features(torch.zeros(1, 3, H, W))
            layers = []
            for c in calls:
                l_, r_, t_, b_ = c["pad"]
                layers.append(dict(k=c["k"], s=c["s"], h=c["h"], w=c["w"], top=t_, left=l_, bottom=b_, right=r_,
                                   ho=(c["h"] + t_ + b_ - c["k"]) // c["s"] + 1, wo=(c["w"] + l_ + r_ - c["k"]) // c["s"] + 1))
            out.append(dict(arch=arch, H=H, W=W, layers=layers, final=[int(y.shape[-2]), int(y.shape[-1])]))
            print(arch, H, W, [(d["top"], d["left"]) for d in layers])
    finally:
        conv2d_same.pad_same, F.pad = orig_same, orig_pad
    with open(os.path.join(GOLDEN, "tf_pad_same.json"), "w") as f:
        json.dump(out, f)


def mint_eval_logits():
    from dfd.timm.models import create_model
    arch = "tf_efficientnet_b0"
    m = create_model(arch, num_classes=2)
    m.load_state_dict(synth_state(get_spec(arch), seed=7), strict=True)
    m.eval()
    x, _ = synth_batch(4, 3, 224, 224, seed=4242)
    with torch.no_grad():
        logits = m(x)
    rec = dict(arch=arch, batch=4, H=224, W=224, weight_seed=7, input_seed=4242, torch=torch.__version__,
               logits=logits.tolist())
    with open(os.path.join(GOLDEN, "tf_eval_b0_224.json"), "w") as f:
        json.dump(rec, f)
    print("tf_eval_b0_224.json", rec["logits"])


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    if sys.argv[1:] == ["--state-keys"]:
        return mint_state_keys()
    mint_state_keys()
    mint_pad_same()
    mint_eval_logits()
    from mint_multiclass_goldens import mint_step_k
    mint_step_k("tf_efficientnet_b0", 4, 64, 96, 2, tag="_64x96")
    mint_step_k("tf_efficientnet_b0", 4, 66, 96, 2, tag="_66x96")


if __name__ == "__main__":
    main()
