"""Host logic of the SE-ResNets, no GPU: the specs against the reference's state keys, the model factory (default_cfg, init,
the keyword arguments the reference refuses or drops) and the plans. Fixtures: tools/mint_senet_goldens.py; their train steps
are held by tests/reference_steps.py's tables."""
import json
import math
import os
from collections import Counter

import pytest
import torch

from deepfake_detection_b200 import _lib
from deepfake_detection_b200.arch import (RESNET_ARCHS, SENET_ARCHS, SUPPORTED_ARCHS, get_spec, param_entries, state_entries,
                                          stem_pool_out)
from deepfake_detection_b200.engine import Engine
from reference_steps import digest
N_STATE = {"seresnet18": 154, "seresnet34": 282, "seresnet50": 384, "seresnet101": 758, "seresnet152": 1132}


def test_registry_and_stem_pool():
    assert SENET_ARCHS == ("seresnet18", "seresnet34", "seresnet50", "seresnet101", "seresnet152")
    assert not set(SENET_ARCHS) & set(SUPPORTED_ARCHS + RESNET_ARCHS)
    # ceil mode without padding: 112 -> 56 (as the padded pool, windows shifted by one), 35 -> 17 (the padded pool gives 18),
    # 36 -> 18 with the last window clipped to two rows
    assert [stem_pool_out(h, "ceil") for h in (112, 35, 36, 3, 4)] == [56, 17, 18, 1, 2]
    assert [stem_pool_out(h, "p1") for h in (112, 35, 36)] == [56, 18, 18]
    for h in range(3, 80):
        ref = torch.nn.functional.max_pool2d(torch.zeros(1, 1, h, h), 3, 2, ceil_mode=True).shape[-1]
        assert stem_pool_out(h, "ceil") == ref


@pytest.mark.parametrize("key", list(SENET_ARCHS) + ["seresnet50@in_chans12"])
def test_spec_matches_reference_state_keys(key, golden_dir):
    ref = json.load(open(os.path.join(golden_dir, "senet_state_keys.json")))[key]
    arch = key.split("@")[0]
    spec = get_spec(arch, num_classes=2, in_chans=12 if key.endswith("12") else 3)
    state = [[n, list(s)] for n, s, _ in state_entries(spec)]
    params = [[n, list(s)] for n, s, _ in param_entries(spec)]
    if "state" in ref:
        assert state == ref["state"] and params == ref["params"]
    assert len(state) == ref["n_state"] == N_STATE[arch] and len(params) == ref["n_param_tensors"]
    assert digest(state) == ref["state_sha256"] and digest(params) == ref["params_sha256"]
    assert sum(math.prod(s) for _, s, _ in param_entries(spec)) == ref["n_params"]
    if key == "seresnet50":
        assert ref["n_params"] == 26043122
    se = [(n, s) for n, s, r in state_entries(spec) if r in ("se_w", "se_b")]
    assert len(se) == 4 * len(spec.blocks) and all(".se_module.fc" in n for n, _ in se)


def test_se_widths_and_strides():
    s18, s50 = get_spec("seresnet18"), get_spec("seresnet50")
    assert sorted({b.cse for b in s18.blocks}) == [4, 8, 16, 32]
    assert sorted({b.cse for b in s50.blocks}) == [16, 32, 64, 128]
    assert s50.stride_in_1x1 and not s18.stride_in_1x1 and s50.stem_pool == s18.stem_pool == "ceil"
    assert [b.name for b in s50.blocks if b.downsample] == ["layer1.0", "layer2.0", "layer3.0", "layer4.0"]


# ---- factory ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", SENET_ARCHS)
def test_default_cfg(arch):
    from deepfake_detection_b200.models import create_model
    m = create_model(arch, num_classes=2)
    cfg = m.default_cfg
    assert cfg["first_conv"] == "layer0.conv1" and cfg["classifier"] == "last_linear"
    assert cfg["interpolation"] == ("bicubic" if arch == "seresnet18" else "bilinear")
    assert cfg["input_size"] == (3, 224, 224) and cfg["pool_size"] == (7, 7) and cfg["crop_pct"] == 0.875
    assert cfg["mean"] == (0.485, 0.456, 0.406) and cfg["std"] == (0.229, 0.224, 0.225)


def test_factory_kwargs():
    from deepfake_detection_b200.models import create_model
    m = create_model("seresnet50", num_classes=2, bn_eps=1e-3, bn_momentum=0.5, bn_tf=True, drop_path_rate=None,
                     drop_block_rate=None)
    assert m.drop_rate == 0.2                               # SENet.__init__'s default
    assert (m.bn_eps, m.bn_momentum) == (1e-5, 0.1)         # factory.py drops the BatchNorm arguments of non-EfficientNets
    assert create_model("seresnet50", num_classes=2, drop_rate=0.0).drop_rate == 0.0
    for bad in (dict(drop_path_rate=0.1), dict(drop_block_rate=0.1), dict(drop_connect_rate=0.2), dict(inplanes=64)):
        with pytest.raises(TypeError):
            create_model("seresnet50", num_classes=2, **bad)
    with pytest.raises(ValueError, match="catavgmax"):
        create_model("seresnet18", num_classes=2, global_pool="catavgmax")
    for gp in ("max", "avgmax"):
        assert create_model("seresnet18", num_classes=2, global_pool=gp).spec.pooled_features == 512


def test_init_statistics():
    from deepfake_detection_b200.models import init_state_dict
    spec = get_spec("seresnet50", num_classes=2)
    sd = init_state_dict(spec, seed=5)
    for name, fan_out in {"layer0.conv1.weight": 64 * 49, "layer3.2.conv2.weight": 256 * 9, "layer4.0.conv3.weight": 2048,
                          "layer4.1.se_module.fc1.weight": 128, "layer4.1.se_module.fc2.weight": 2048}.items():
        assert float(sd[name].std()) == pytest.approx(math.sqrt(2.0 / fan_out), rel=0.05), name
    for name, fan_in in {"layer4.1.se_module.fc1.bias": 2048, "layer4.1.se_module.fc2.bias": 128}.items():
        r = 1.0 / math.sqrt(fan_in)
        assert float(sd[name].abs().max()) <= r and float(sd[name].abs().max()) > 0.5 * r, name
    r = 1.0 / math.sqrt(2048)
    assert all(float(sd[k].abs().max()) <= r for k in ("last_linear.weight", "last_linear.bias"))
    assert float(sd["last_linear.weight"].abs().max()) > 0.99 * r
    # no zero-init of the last BN gamma: every BN weight is 1, every BN bias 0
    assert all(float(sd[n].min()) == 1.0 for n, _, role in state_entries(spec) if role == "bn_w")
    assert all(float(sd[n].abs().max()) == 0.0 for n, _, role in state_entries(spec) if role == "bn_b")


# ---- plans --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gemm_impl", ["tc", "mma"])
@pytest.mark.parametrize("arch,H,W", [("seresnet18", 70, 72), ("seresnet50", 224, 224), ("seresnet50", 64, 64),
                                      ("seresnet101", 64, 64)])
def test_plan_census(arch, H, W, gemm_impl):
    """every op passes _finish_plan's ABI check (the Engine constructor runs it); the SE and stem launches per step"""
    e = Engine(arch, 2, H, W, device="plan-only", gemm_impl=gemm_impl, drop_rate=0.2)
    spec = e.spec
    nb = len(spec.blocks)
    ops = [(n, a) for _, n, a in e.fwd_ops + e.bwd_ops]
    names = Counter(n for n, _ in ops)
    assert names["dfd_pool_se_relu"] == names["dfd_relu_se_bwd_reduce"] == names["dfd_se_fc_wgrad"] == nb
    assert names["dfd_maxpool_ceil_fwd"] == names["dfd_maxpool_ceil_bwd"] == 1
    assert names["dfd_maxpool_fwd"] == names["dfd_maxpool_bwd"] == 0
    assert names["dfd_relu_bn_bwd_reduce"] == names["dfd_relu_bn_bwd_reduce_drop"] == 0
    assert names["dfd_mul_f32_train"] == 1             # the default dropout on the pooled vector
    tails = [a for n, a in ops if n == "dfd_bn_act" and a[4] is not None]
    assert len(tails) == nb and all(a[3] is not None and not isinstance(a[3], tuple) and a[10] == 2 for a in tails)
    # the last BN's input gradient: gm * gate + dpool / HW, no activation
    # the SE input: the bare BN output of a bottleneck, after the ReLU in a basic block (senet.py:213-215)
    act = _lib.ACT_RELU if spec.blocks[0].kind == "basic" else _lib.ACT_NONE
    assert all(a[9] == act for a in tails)
    assert all(a[13] == act for n, a in ops if n == "dfd_pool_se_relu")
    assert all(a[21] == act for n, a in ops if n == "dfd_relu_se_bwd_reduce")
    # the last BN's input gradient: (gm * gate + dpool / HW) * act'
    ab = [a for n, a in ops if n == "dfd_act_bwd" and a[6] is not None]
    assert len(ab) == nb and all(a[7] is not None and a[12] == act for a in ab)
    s1x1 = [b for b in spec.blocks if spec.stride_in_1x1 and b.stride != 1]
    assert len(s1x1) == (3 if spec.stride_in_1x1 else 0)
    if gemm_impl == "tc" and s1x1:
        strided_k1 = [a for n, a in ops if n == "dfd_conv_tc" and a[8] == 1 and a[9] == 2]
        assert len(strided_k1) == 2 * len(s1x1)        # conv1 and the downsample of each strided bottleneck
        assert names["dfd_conv1x1_dgrad_add"] == 2 * len(s1x1) + 1      # + layer1.0's stride-1 downsample
    assert not [a for n, a in ops if n == "dfd_conv_tc" and a[8] == 3 and a[9] == 2 and spec.stride_in_1x1]
    # the stem pool runs on the conv extent; the blocks start at the ceil-mode extent
    h1, w1 = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
    pf = [a for n, a in ops if n == "dfd_maxpool_ceil_fwd"][0]
    assert (pf[4], pf[5]) == (h1, w1)
    assert tuple(e.acts["stem.out"].shape[1:3]) == (stem_pool_out(h1, "ceil"), stem_pool_out(w1, "ceil"))


def test_eval_plan_keeps_the_gate():
    """the SE gate is computed in eval mode too (unlike the drop-path gate)"""
    e = Engine("seresnet18", 1, 224, 224, device="plan-only")
    for fn, n, a in e.fwd_ops:
        if n in ("dfd_pool_se_relu", "dfd_bn_act"):
            assert e.launch_args(n, a, False) == e.launch_args(n, a, True) is not None


@pytest.mark.parametrize("kw", [dict(drop_path_rate=0.1), dict(drop_block_rate=0.1)])
def test_engine_refuses_drop_path_and_drop_block(kw):
    with pytest.raises(ValueError):
        Engine("seresnet50", 2, 64, 64, device="plan-only", **kw)


def test_sync_bn_refused():
    from deepfake_detection_b200 import ddp
    from deepfake_detection_b200.models import create_model
    with pytest.raises(_lib.NativeError):
        ddp.convert_syncbn_model(create_model("seresnet50", num_classes=2))
