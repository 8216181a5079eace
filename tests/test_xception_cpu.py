"""Host logic of Xception, no GPU: the spec against the reference's state keys, the oracle (tests/xception_oracle.py) against
the reference's train steps, the model factory (default_cfg, init, the keyword arguments the reference refuses or drops) and
the plans. Fixtures: tools/mint_xception_goldens.py."""
import json
import math
import os
from collections import Counter

import pytest
import torch

import xception_oracle as XO
from deepfake_detection_b200 import _lib
from deepfake_detection_b200.arch import SUPPORTED_ARCHS, XCEPTION_ARCHS, get_spec, param_entries, state_entries, xception_extents
from deepfake_detection_b200.engine import Engine
from oracle import train as OT
from oracle.weights import synth_batch, synth_state
from test_resnet_family_cpu import _digest
from test_tf_efficientnet_cpu import RTOL, _check_summ

STEP_CASES = ["step_xception_64x80", "step_xception_299", "step_xception_tame_64x80"]


def test_registry_and_extents():
    assert XCEPTION_ARCHS == ("xception",) and "xception" not in SUPPORTED_ARCHS
    assert xception_extents(299, 299) == [(149, 149), (147, 147), (74, 74), (37, 37), (19, 19)] + [(19, 19)] * 8 + [(10, 10)]
    assert xception_extents(64, 80)[:5] + xception_extents(64, 80)[-1:] == [(31, 39), (29, 37), (15, 19), (8, 10), (4, 5), (2, 3)]


@pytest.mark.parametrize("key", ["xception", "xception@in_chans12"])
def test_spec_matches_reference_state_keys(key, golden_dir):
    ref = json.load(open(os.path.join(golden_dir, "xception_state_keys.json")))[key]
    spec = get_spec("xception", num_classes=2, in_chans=12 if key.endswith("12") else 3)
    state = [[n, list(s)] for n, s, _ in state_entries(spec)]
    params = [[n, list(s)] for n, s, _ in param_entries(spec)]
    assert state == ref["state"] and params == ref["params"]
    assert (len(state), len(params)) == (ref["n_state"], ref["n_param_tensors"]) == (276, 156)
    assert _digest(state) == ref["state_sha256"] and _digest(params) == ref["params_sha256"]
    assert sum(math.prod(s) for _, s, _ in param_entries(spec)) == ref["n_params"]
    if key == "xception":
        assert ref["n_params"] == 20811050


@pytest.mark.parametrize("case", STEP_CASES)
def test_oracle_matches_reference_steps(case, golden_dir):
    """tests/xception_oracle.py against the reference's own train steps and eval, at the ResNet family's fp32 tolerances"""
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    torch.set_num_threads(8)
    spec = get_spec(rec["arch"], num_classes=rec["num_classes"])
    sd = synth_state(spec, seed=rec["weight_seed"])
    if "tame" in rec:
        sd = XO.tame_state(spec, sd, rec["tame"])
    opt = OT.OptState(kind=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"], eps=1e-8)
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i)
        out = XO.train_step(spec, sd, x, y, opt)
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
    x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=999)
    ev = XO.validate_step(spec, sd, x, y)
    _check_summ(ev["logits"], rec["eval"]["logits"], "eval logits", rtol=5e-3)


# ---- factory ------------------------------------------------------------------------------------------------------------
def test_default_cfg_and_kwargs():
    from deepfake_detection_b200.models import create_model
    m = create_model("xception", num_classes=2, bn_eps=1e-3, bn_momentum=0.5, bn_tf=True, drop_path_rate=None,
                     drop_block_rate=None, drop_rate=0.5)
    cfg = m.default_cfg
    assert cfg["input_size"] == (3, 299, 299) and cfg["crop_pct"] == 0.8975 and cfg["interpolation"] == "bicubic"
    assert cfg["mean"] == cfg["std"] == (0.5, 0.5, 0.5) and cfg["first_conv"] == "conv1" and cfg["classifier"] == "fc"
    assert (m.bn_eps, m.bn_momentum) == (1e-5, 0.1)        # factory.py drops the BatchNorm arguments of non-EfficientNets
    for bad in (dict(drop_path_rate=0.1), dict(drop_block_rate=0.1), dict(drop_connect_rate=0.2)):
        with pytest.raises(TypeError):
            create_model("xception", num_classes=2, **bad)


def test_init_statistics():
    from deepfake_detection_b200.models import init_state_dict
    spec = get_spec("xception", num_classes=2)
    sd = init_state_dict(spec, seed=5)
    for name, C in {"block4.rep.1.conv1.weight": 728, "conv4.conv1.weight": 1536}.items():
        std = float(sd[name].std())
        assert std == pytest.approx(math.sqrt(2.0 / (9 * C)), rel=0.05), (name, std)      # fan_out = C * 9, not / groups
    assert float(sd["conv4.pointwise.weight"].std()) == pytest.approx(math.sqrt(2.0 / 2048), rel=0.02)
    r = 1.0 / math.sqrt(2048)
    assert all(float(sd[k].abs().max()) <= r for k in ("fc.weight", "fc.bias"))
    assert float(sd["fc.weight"].abs().max()) > 0.99 * r
    assert all(float(sd[n].min()) == 1.0 for n, _, role in state_entries(spec) if role == "bn_w")
    assert all(float(sd[n].abs().max()) == 0.0 for n, _, role in state_entries(spec) if role == "bn_b")


# ---- plans --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_chans", [3, 12])
@pytest.mark.parametrize("H,W", [(299, 299), (64, 80)])
def test_plan_census(H, W, in_chans):
    """every op passes _finish_plan's ABI check (the Engine constructor runs it); the launches per step"""
    e = Engine("xception", 2, H, W, device="plan-only", in_chans=in_chans)
    ops = [(n, a) for _, n, a in e.fwd_ops + e.bwd_ops]
    names = Counter(n for n, _ in ops)
    assert names["dfd_dwconv_fwd"] == 34
    assert names["dfd_dwconv_bwd"] + names["dfd_dwconv_bwd_relu"] == 34
    assert names["dfd_dwconv_bwd"] == 2          # block1's first (the activated stem output) and conv3's (block12's output)
    assert names["dfd_bn_maxpool_add"] == names["dfd_maxpool_bn_bwd_reduce"] == 4
    assert len([a for n, a in ops if n == "dfd_bn_act" and a[4] is not None]) == 8      # identity tails: bn(y) + x
    assert names["dfd_maxpool_fwd"] == names["dfd_maxpool_bwd"] == 0
    assert not [a for n, a in ops if n == "dfd_conv_tc" and 728 in (a[6], a[7])]
    assert not [a for n, a in ops if n == "dfd_conv1x1_dgrad_add" and 728 in (a[6], a[7])]
    assert [(a[6], a[7]) for n, a in ops if n == "dfd_conv_tc"] == [(64, 128), (128, 256)]
    assert names["dfd_stem_im2col"] == 1 and names["dfd_unpad_grad"] == 1 and names["dfd_unpack_grad"] == 1
    # depthwise forwards: no statistics, ReLU at load everywhere except block1's first and conv3's
    dws = [a for n, a in ops if n == "dfd_dwconv_fwd"]
    assert all(a[13] is None and a[14] is None for a in dws)
    assert sum(a[11] == _lib.ACT_RELU for a in dws) == 32
    assert sum(a[11] == _lib.ACT_RELU and a[1] is not None for a in dws) == 34 - 2 - 11     # inside a block, and conv4
    assert all(a[2] is None for n, a in ops if n == "dfd_dwconv_bwd_relu")                 # cA: gy is the pointwise dgrad


def test_eval_plan_drops_the_arg_max():
    e = Engine("xception", 1, 299, 299, device="plan-only")
    for fn, n, a in e.fwd_ops:
        if n == "dfd_bn_maxpool_add":
            assert e.launch_args(n, a, False)[7] is None and e.launch_args(n, a, True)[7] is not None


def test_sync_bn_refused():
    from deepfake_detection_b200 import ddp
    from deepfake_detection_b200.models import create_model
    with pytest.raises(_lib.NativeError):
        ddp.convert_syncbn_model(create_model("xception", num_classes=2))
