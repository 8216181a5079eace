"""Pins oracle/ to the reference for class counts other than 2: the K-class fixtures under tests/golden/ were produced
by the UNMODIFIED reference (tools/mint_multiclass_goldens.py) and the oracle must reproduce them in fp32 on CPU, at the
tolerances of test_oracle_vs_reference_goldens.py (2e-4 relative on norms, samples to 5 x 2e-4 of the per-element scale;
25x looser after the first update; logits 1e-3, eval logits 5e-3).  The fixtures hold summaries (norm, sum, sampled
elements) of the logits and of a fixed subset of gradients, parameters and running statistics."""
import json
import os

import pytest
import torch

from deepfake_detection_b200.arch import get_spec
from oracle import model as OM
from oracle import train as OT
from oracle.weights import synth_batch, synth_state

RTOL = 2e-4
CASES = ["step_efficientnet_b0_k5_ls", "step_efficientnet_b0_k5_soft_rmsprop", "step_resnet18_k1000"]


def _check_summ(t, s, what, rtol=RTOL, floor=1e-7):
    f = t.detach().reshape(-1).to(torch.float64)
    assert float(f.norm()) == pytest.approx(s["norm"], rel=rtol, abs=floor * max(f.numel(), 1) ** 0.5), what + " norm"
    got = f[torch.tensor(s["idx"])]
    ref = torch.tensor(s["samples"], dtype=torch.float64)
    scale = max(s["norm"] / max(f.numel(), 1) ** 0.5, 1e-8)
    assert float((got - ref).abs().max()) <= 5 * rtol * scale + rtol * float(ref.abs().max()) + floor, what + " samples"


@pytest.mark.parametrize("case", CASES)
def test_k_class_train_steps_match_reference(case, golden_dir):
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    K = rec["num_classes"]
    torch.set_num_threads(8)
    spec = get_spec(rec["arch"], num_classes=K)
    sd = synth_state(spec, seed=rec["weight_seed"])
    opt = OT.OptState(kind=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"], eps=1e-8)
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i, soft=rec["soft"], num_classes=K)
        out = OT.train_step(spec, sd, x, y, opt, smoothing=rec["smoothing"])
        assert out["logits"].shape == (rec["batch"], K)
        _check_summ(out["logits"], st["logits"], "logits step %d" % i, rtol=1e-3)
        assert float(out["loss"]) == pytest.approx(st["loss"], rel=1e-4)
        assert float(out["prec1"]) == pytest.approx(st["prec1"], abs=1e-3)
        rt = RTOL * (1 if i == 0 else 25)
        gfloor = 1e-5 * max(v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 for k, v in st["grads"].items())
        for k, s in st["grads"].items():
            _check_summ(out["grads"][k], s, "grad %s step %d" % (k, i), rt, floor=gfloor)
        # adaptive optimizers turn a round-off (mathematically zero) gradient into an O(lr) update in both implementations
        noise = {k for k, v in st["grads"].items()
                 if v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 < 10 * gfloor} if rec["opt"] != "sgd" else set()
        if i == 0:
            skipped = set(noise)
        for k, s in st["params"].items():
            if k in skipped or k in noise:
                continue
            _check_summ(sd[k], s, "param %s step %d" % (k, i), rt)
        for k, s in st["buffers"].items():
            _check_summ(sd[k].float(), s, "buffer %s step %d" % (k, i), rt)
    x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=999, num_classes=K)
    ev = OT.validate_step(spec, sd, x, y)
    _check_summ(ev["logits"], rec["eval"]["logits"], "eval logits", rtol=5e-3)
    assert float(ev["loss"]) == pytest.approx(rec["eval"]["loss"], rel=2e-3)


def test_oracle_cross_entropy_is_k_general():
    """oracle/model.py::cross_entropy against torch's own losses at K = 5 and 1000 (hard, smoothed, soft targets)."""
    g = torch.Generator().manual_seed(0)
    for K in (5, 1000):
        z = torch.randn(16, K, generator=g, dtype=torch.float64) * 3
        y = torch.randint(0, K, (16,), generator=g)
        assert torch.allclose(OM.cross_entropy(z, y), torch.nn.functional.cross_entropy(z, y))
        assert torch.allclose(OM.cross_entropy(z, y, 0.1), torch.nn.functional.cross_entropy(z, y, label_smoothing=0.1))
        t = torch.softmax(torch.randn(16, K, generator=g, dtype=torch.float64), -1)
        assert torch.allclose(OM.cross_entropy(z, t), torch.nn.functional.cross_entropy(z, t))
