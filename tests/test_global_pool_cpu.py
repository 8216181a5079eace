"""Selectable global pooling (avg / max / avgmax / catavgmax) on the host side, without a GPU.

The pool oracle (tests/gpool_oracle.py) against oracle.train at 'avg' and against the global-pool fixtures minted from the UNMODIFIED reference (tools/mint_gpool_goldens.py) at the
tolerances of test_head_multiclass_cpu.py; the arch restatement against the reference's catavgmax state_dict names and
shapes; create_model / get_spec carrying the pool type; the plans of both families."""
import json
import os

import pytest
import torch

from deepfake_detection_b200.arch import SUPPORTED_ARCHS, get_spec, param_entries, state_entries
from oracle import train as OT
from oracle.weights import synth_batch, synth_state

import gpool_oracle as GO

from test_head_multiclass_cpu import RTOL, _check_summ

CASES = ["step_efficientnet_b0_gp_max", "step_efficientnet_b0_k5_gp_catavgmax_ls", "step_resnet18_gp_avgmax"]


@pytest.mark.parametrize("case", CASES)
def test_oracle_global_pool_steps_match_reference(case, golden_dir):
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    K, gp = rec["num_classes"], rec["global_pool"]
    torch.set_num_threads(8)
    spec = get_spec(rec["arch"], num_classes=K, global_pool=gp)
    sd = synth_state(spec, seed=rec["weight_seed"])
    opt = OT.OptState(kind=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"], eps=1e-8)
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i, soft=rec["soft"], num_classes=K)
        out = GO.train_step(spec, sd, x, y, opt, smoothing=rec["smoothing"])
        _check_summ(out["logits"], st["logits"], "logits step %d" % i, rtol=1e-3)
        assert float(out["loss"]) == pytest.approx(st["loss"], rel=1e-4)
        assert float(out["prec1"]) == pytest.approx(st["prec1"], abs=1e-3)
        rt = RTOL * (1 if i == 0 else 25)
        gfloor = 1e-5 * max(v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 for k, v in st["grads"].items())
        for k, s in st["grads"].items():
            _check_summ(out["grads"][k], s, "grad %s step %d" % (k, i), rt, floor=gfloor)
        for k, s in st["params"].items():
            _check_summ(sd[k], s, "param %s step %d" % (k, i), rt)
        for k, s in st["buffers"].items():
            _check_summ(sd[k].float(), s, "buffer %s step %d" % (k, i), rt)
    x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=999, num_classes=K)
    ev = GO.validate_step(spec, sd, x, y)
    _check_summ(ev["logits"], rec["eval"]["logits"], "eval logits", rtol=5e-3)


@pytest.mark.parametrize("arch", ["efficientnet_b0", "resnet18"])
def test_pool_oracle_at_avg_is_the_oracle(arch):
    """at 'avg' the pool oracle's train step is oracle.train.train_step bit for bit (16-bit emulation and dropout included)"""
    torch.set_num_threads(8)
    spec = get_spec(arch, num_classes=3)
    x, y = synth_batch(2, 3, 64, 64, seed=5, num_classes=3)
    mask = (torch.rand(2, spec.num_features, generator=torch.Generator().manual_seed(1)) > 0.3).float() / 0.7 \
        if spec.family == "efficientnet" else None
    outs = []
    for step in (OT.train_step, GO.train_step):
        sd = synth_state(spec, seed=7)
        outs.append((step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01), act_dtype=torch.bfloat16, dropout_mask=mask), sd))
    (a, sa), (b, sb) = outs
    assert torch.equal(a["logits"], b["logits"]) and torch.equal(a["loss"], b["loss"])
    assert all(torch.equal(a["grads"][k], b["grads"][k]) for k in a["grads"])
    assert all(torch.equal(sa[k], sb[k]) for k in sa)
    ev = [f(spec, sa, x, y, act_dtype=torch.bfloat16)["logits"] for f in (OT.validate_step, GO.validate_step)]
    assert torch.equal(ev[0], ev[1])


@pytest.mark.parametrize("arch", SUPPORTED_ARCHS)
def test_catavgmax_state_entries_match_reference(arch, golden_dir):
    ref = json.load(open(os.path.join(golden_dir, "state_keys_catavgmax.json")))[arch]
    spec = get_spec(arch, num_classes=2, in_chans=12 if arch == "efficientnet_deepfake_v4" else 3, global_pool="catavgmax")
    assert [[n, list(s)] for n, s, _ in state_entries(spec)] == ref["state"]
    assert [[n, list(s)] for n, s, _ in param_entries(spec)] == ref["params"]
    assert spec.pooled_features == 2 * spec.num_features


def test_oracle_global_pool_matches_torch_pooling():
    """gpool_oracle.global_pool is SelectAdaptivePool2d's arithmetic (adaptive_avgmax_pool.py:24-48)"""
    x = torch.randn(3, 16, 5, 7, dtype=torch.float64)
    avg, mx = torch.nn.functional.adaptive_avg_pool2d(x, 1).flatten(1), torch.nn.functional.adaptive_max_pool2d(x, 1).flatten(1)
    assert torch.equal(GO.global_pool(x, "avg"), x.mean((2, 3)))
    assert torch.equal(GO.global_pool(x, "max"), mx)
    assert torch.equal(GO.global_pool(x, "avgmax"), 0.5 * (avg + mx))
    assert torch.equal(GO.global_pool(x, "catavgmax"), torch.cat((avg, mx), 1))
    with pytest.raises(ValueError):
        GO.global_pool(x, "avgmaxc")


@pytest.mark.parametrize("gp", ["avg", "max", "avgmax", "catavgmax"])
@pytest.mark.parametrize("arch", ["efficientnet_b0", "resnet50"])
def test_create_model_carries_the_pool_type(arch, gp):
    from deepfake_detection_b200.models import create_model
    m = create_model(arch, num_classes=5, global_pool=gp)
    F = m.spec.num_features
    P = 2 * F if gp == "catavgmax" else F
    assert m.spec.global_pool == gp and m.spec.pooled_features == P
    assert m._engine_kwargs()["global_pool"] == gp
    cls = "classifier" if arch.startswith("efficientnet") else "fc"
    assert dict((n, s) for n, s, _ in state_entries(m.spec))[cls + ".weight"] == (5, P)
    if gp == "avg":
        assert state_entries(m.spec) == state_entries(get_spec(arch, num_classes=5))


def test_invalid_pool_type_is_rejected():
    from deepfake_detection_b200.models import create_deepfake_model_v4, create_model
    with pytest.raises(ValueError, match="Invalid pool type"):
        get_spec("efficientnet_b0", global_pool="avgmaxc")
    with pytest.raises(ValueError, match="Invalid pool type"):
        create_model("resnet18", global_pool="sum")
    with pytest.raises(ValueError, match="Invalid pool type"):
        create_deepfake_model_v4("efficientnet_deepfake_v4", num_classes=2, in_chans=12, global_pool="")


@pytest.mark.parametrize("arch", ["efficientnet_b0", "resnet50"])
def test_plans_of_every_pool_type(arch):
    """avg keeps the default plan op for op; the other types swap the pool forward / backward ops for the new entry points
    and size the head at P = feat_mult * F."""
    from deepfake_detection_b200.engine import Engine
    base = Engine(arch, 8, 224, 224, device="plan-only")
    names = lambda e: [n for _, n, _ in e.fwd_ops + e.bwd_ops]
    avg = Engine(arch, 8, 224, 224, device="plan-only", global_pool="avg")
    assert names(avg) == names(base) and avg.n_launch == base.n_launch
    for gp in ("max", "avgmax", "catavgmax"):
        e = Engine(arch, 8, 224, 224, device="plan-only", global_pool=gp)
        assert e.n_launch == base.n_launch
        swap = {"dfd_pool": "dfd_global_pool",
                "dfd_act_bwd": "dfd_act_bwd_gpool" if arch.startswith("efficientnet") else "dfd_act_bwd",
                "dfd_pool_bwd": "dfd_gpool_bwd"}
        diff = [(a, b) for a, b in zip(names(base), names(e)) if a != b]
        assert diff and all(swap[a] == b for a, b in diff), diff
        P = e.spec.pooled_features
        assert tuple(e.pooled.shape) == (8, P) and tuple(e.dpooled.shape) == (8, P)
        assert tuple(e.pool_argmax.shape) == (8, e.spec.num_features) and e.pool_argmax.dtype == torch.int32
