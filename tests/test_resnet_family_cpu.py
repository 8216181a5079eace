"""Host logic of the dense ResNet family (resnet26/34/101/152, tv_resnet34/50, wide_resnet50_2/101_2, resnet26d, resnet50d),
no GPU: the specs against the reference's state keys, the oracle (tests/resnet_family_oracle.py) against the reference's train
steps, the model factory's registry, default_cfg and init, and the plans. Fixtures: tools/mint_resnet_family_goldens.py."""
import hashlib
import json
import os
from collections import Counter

import pytest
import torch

import resnet_family_oracle as RO
from deepfake_detection_b200 import _lib
from deepfake_detection_b200.arch import RESNET_ARCHS, SUPPORTED_ARCHS, get_spec, param_entries, state_entries
from deepfake_detection_b200.engine import Engine
from oracle import train as OT
from oracle.weights import synth_batch, synth_state
from test_tf_efficientnet_cpu import RTOL, _check_summ

STEP_CASES = ["step_resnet26d_72x88", "step_resnet50d", "step_resnet34", "step_wide_resnet50_2", "step_resnet101",
              "step_resnet26d_tame_104x88", "step_resnet34_tame_96", "step_wide_resnet50_2_tame_96", "step_resnet101_tame_96"]


def _digest(entries):
    return hashlib.sha256(json.dumps(entries, separators=(",", ":")).encode()).hexdigest()


def test_registry():
    assert RESNET_ARCHS == ("resnet26", "resnet34", "resnet101", "resnet152", "tv_resnet34", "tv_resnet50", "wide_resnet50_2",
                            "wide_resnet101_2", "resnet26d", "resnet50d")
    assert not set(RESNET_ARCHS) & set(SUPPORTED_ARCHS)
    for a in ("resnet18", "resnet50"):
        spec = get_spec(a)
        assert spec.stem_type == "" and all(b.width == b.planes and not b.avg_down for b in spec.blocks)
    assert [b.width for b in get_spec("wide_resnet50_2").blocks if b.name.endswith(".0")] == [128, 256, 512, 1024]


@pytest.mark.parametrize("key", list(RESNET_ARCHS) + ["resnet50d@in_chans12"])
def test_specs_match_reference_state_keys(key, golden_dir):
    ref = json.load(open(os.path.join(golden_dir, "resnet_family_state_keys.json")))[key]
    arch, _, ic = key.partition("@in_chans")
    spec = get_spec(arch, num_classes=2, in_chans=int(ic or 3))
    state = [[n, list(s)] for n, s, _ in state_entries(spec)]
    params = [[n, list(s)] for n, s, _ in param_entries(spec)]
    if "state" in ref:          # written out in full: a mismatch shows the first differing entry
        assert state == ref["state"] and params == ref["params"]
    assert (len(state), len(params)) == (ref["n_state"], ref["n_param_tensors"])
    assert _digest(state) == ref["state_sha256"] and _digest(params) == ref["params_sha256"]
    n = 0
    for _, s, _ in param_entries(spec):
        k = 1
        for d in s:
            k *= d
        n += k
    assert n == ref["n_params"]


@pytest.mark.parametrize("case", STEP_CASES)
def test_oracle_matches_reference_steps(case, golden_dir):
    """tests/resnet_family_oracle.py against the reference's own train steps and eval, at the tolerances of
    test_oracle_vs_reference_goldens.py / test_tf_efficientnet_cpu.py"""
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    torch.set_num_threads(8)
    spec = get_spec(rec["arch"], num_classes=rec["num_classes"])
    sd = synth_state(spec, seed=rec["weight_seed"])
    if "tame" in rec:
        sd = RO.tame_state(spec, sd, rec["tame"])
    opt = OT.OptState(kind=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"], eps=1e-8)
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i)
        out = RO.train_step(spec, sd, x, y, opt)
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
    ev = RO.validate_step(spec, sd, x, y)
    _check_summ(ev["logits"], rec["eval"]["logits"], "eval logits", rtol=5e-3)


@pytest.mark.parametrize("in_chans", [3, 12])
@pytest.mark.parametrize("arch", RESNET_ARCHS)
def test_plan_builds_at_224(arch, in_chans):
    e = Engine(arch, 2, 224, 224, device="plan-only", in_chans=in_chans)
    names = Counter(n for _, n, _ in e.fwd_ops + e.bwd_ops)
    deep = arch.endswith("d")
    assert names["dfd_avgpool2_fwd"] == names["dfd_avgpool2_bwd_add"] == (3 if deep else 0)
    assert ("dfd_stem_fwd" in names) is False
    assert names["dfd_stem_im2col"] == 1 and names["dfd_unpad_grad"] == 1
    # every 3x3 with 64-multiple channels stays an implicit GEMM; the deep stem's two 32-channel 3x3s take im2col
    assert names["dfd_im2col"] == (4 if deep else 0)


def test_resnet50d_plan_pools_the_shortcut():
    e = Engine("resnet50d", 2, 224, 224, device="plan-only")
    ops = [(n, a) for _, n, a in e.fwd_ops + e.bwd_ops]
    pools = [a for n, a in ops if n == "dfd_avgpool2_fwd"]
    assert [(a[3], a[4], a[5]) for a in pools] == [(56, 56, 256), (28, 28, 512), (14, 14, 1024)]
    assert [(a[4], a[5], a[6]) for n, a in ops if n == "dfd_avgpool2_bwd_add"] == [(14, 14, 1024), (28, 28, 512), (56, 56, 256)]
    # no strided 1x1 downsample in any form: implicit conv / its weight gradient, gathered copy, col2im, strided dgrad-add
    assert not [a for n, a in ops if n == "dfd_conv_tc" and a[8] == 1]
    assert not [a for n, a in ops if n == "dfd_conv_wgrad_tc" and a[8] == 1]
    assert not [a for n, a in ops if n in ("dfd_im2col", "dfd_col2im") and a[6] == 1]
    assert all(a[8] == 1 for n, a in ops if n == "dfd_conv1x1_dgrad_add")      # layer1.0: stride-1 shortcut, no pool
    # every pooled 16-bit tensor feeds its downsample GEMM: the forward pool output is the GEMM's A operand
    fwd = [(n, a) for _, n, a in e.fwd_ops]
    for i, (n, a) in enumerate(fwd):
        if n == "dfd_avgpool2_fwd":
            assert fwd[i + 1][0] == "dfd_gemm_tn" and fwd[i + 1][1][0] == a[1]


def test_avgpool_bwd_adds_the_main_path_gradient():
    """the pooled shortcut's input gradient meets the main-path gradient (conv1's dgrad output) in the same pass"""
    e = Engine("resnet26d", 2, 72, 88, device="plan-only")
    bwd = [(n, a) for _, n, a in e.bwd_ops]
    for i, (n, a) in enumerate(bwd):
        if n != "dfd_avgpool2_bwd_add":
            continue
        dgrad = [b for m, b in bwd[:i] if m == "dfd_gemm_tn"]
        assert a[0] == dgrad[-1][2]         # pooled-grid gradient of the downsample GEMM
        assert a[1] == dgrad[-2][2]         # conv1's input gradient (main path)
        assert a[2] not in (a[0], a[1])


def test_deep_stem_plan():
    e = Engine("resnet50d", 2, 224, 224, device="plan-only")
    fwd = [n for _, n, _ in e.fwd_ops]
    assert fwd[:12] == ["dfd_stem_im2col", "dfd_gemm_tn", "dfd_bn_finalize", "dfd_bn_act",
                        "dfd_im2col", "dfd_gemm_tn", "dfd_bn_finalize", "dfd_bn_act",
                        "dfd_im2col", "dfd_gemm_tn", "dfd_bn_finalize", "dfd_bn_act"]
    assert fwd[12] == "dfd_maxpool_fwd"
    bwd = [n for _, n, _ in e.bwd_ops]
    tail = bwd[bwd.index("dfd_maxpool_bwd"):]
    # one ordered reduce for the stem's three weight gradients, then the two unpacks and the unpad
    assert tail.count("dfd_ordered_reduce") == 1 and tail[-4:] == ["dfd_ordered_reduce", "dfd_unpack_grad", "dfd_unpack_grad",
                                                                   "dfd_unpad_grad"]
    assert tail.count("dfd_col2im") == 2


@pytest.mark.parametrize("stem_impl", ["fwd", "direct"])
def test_deep_stem_refuses_other_stem_impls(stem_impl):
    with pytest.raises(ValueError, match="deep stem"):
        Engine("resnet26d", 2, 64, 64, device="plan-only", stem_impl=stem_impl)


def test_drop_block_sites_and_drop_path():
    for arch, n in (("resnet101", 78), ("resnet152", 117), ("resnet50d", 27), ("wide_resnet50_2", 27)):
        e = Engine(arch, 2, 224, 224, device="plan-only", drop_block_rate=0.1, drop_path_rate=0.1)
        assert len(e.drop_block_sites) == n
        assert len(e.drop_masks) == len(e.spec.blocks)
    e = Engine("wide_resnet50_2", 2, 224, 224, device="plan-only", drop_block_rate=0.1)
    assert e.drop_block_sites["layer3.0.bn1"][2] == 512 and e.drop_block_sites["layer3.0.bn3"][2] == 1024


@pytest.mark.parametrize("name", ["resnext50_32x4d", "resnext50d_32x4d", "resnext101_32x8d", "tv_resnext50_32x4d",
                                  "seresnext26d_32x4d", "seresnext50_32x4d", "ig_resnext101_32x8d", "ssl_resnet50",
                                  "swsl_resnet18", "ssl_resnext50_32x4d"])
def test_resnext_names_stay_unknown(name):
    from deepfake_detection_b200.models import create_model
    with pytest.raises(RuntimeError, match="Unknown model"):
        create_model(name, num_classes=2)


def test_default_cfg_and_init():
    from deepfake_detection_b200.models import NativeModel, init_state_dict
    bicubic = {"resnet26", "resnet26d", "resnet50d"}
    for a in RESNET_ARCHS:
        cfg = NativeModel(a, num_classes=2).default_cfg
        assert cfg["interpolation"] == ("bicubic" if a in bicubic else "bilinear"), a
        assert (cfg["first_conv"], cfg["classifier"], cfg["input_size"]) == ("conv1", "fc", (3, 224, 224))
    assert NativeModel("resnet18").default_cfg["interpolation"] == "bicubic"        # unchanged
    spec = get_spec("resnet50d", num_classes=2)
    sd = init_state_dict(spec, seed=3)
    assert list(sd) == [n for n, _, _ in state_entries(spec)]
    for n in ("conv1.0.weight", "conv1.3.weight", "conv1.6.weight", "layer2.0.downsample.1.weight"):
        w = sd[n]
        fan_out = w.shape[0] * w.shape[2] * w.shape[3]
        assert float(w.std()) == pytest.approx((2.0 / fan_out) ** 0.5, rel=0.15), n
    for b in spec.blocks:
        assert float(sd[b.name + ".bn3.weight"].abs().max()) == 0.0
    assert float(sd["conv1.1.weight"].min()) == 1.0 and float(sd["layer1.0.downsample.2.weight"].min()) == 1.0


def _shapes(e):
    """each op of a plan with its pointer operands left out"""
    from deepfake_detection_b200.engine import base_name
    out = []
    for _, n, a in e.fwd_ops + e.bwd_ops:
        codes = _lib.SIGNATURES.get(base_name(n), "")
        out.append((n, tuple(v for v, c in zip(a, codes) if c != "p" and not isinstance(v, (tuple, list)))))
    return out


def test_tv_resnet50_plan_equals_resnet50():
    """width == planes and no ResNet-D parts: tv_resnet50 (same layers as resnet50) plans the same launches"""
    a = Engine("resnet50", 2, 96, 96, device="plan-only")
    b = Engine("tv_resnet50", 2, 96, 96, device="plan-only")
    assert _shapes(a) == _shapes(b) and a.n_launch == b.n_launch
    assert _lib.SIGNATURES["dfd_avgpool2_fwd"] == "ppiiiiip" and _lib.SIGNATURES["dfd_avgpool2_bwd_add"] == "pppiiiiip"
