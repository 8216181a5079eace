"""DenseNet host logic without a GPU: the specs against densenet.py's parameter counts and key order, the factory rules, the
initialisation statistics, the plan-only builds in both gemm_impls with their launch census, and the fp64 restatement used by
the GPU tests against torch's own DenseNet layers built from the same weights."""
import math
from collections import Counter

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import densenet_ref as R
from deepfake_detection_b200.arch import DENSENET_ARCHS, SUPPORTED_ARCHS, get_spec, param_entries, state_entries
from reference_steps import check_summ, digest

# densenet.py at num_classes=2: state_dict entries, parameter tensors, parameters
TABLE = {"densenet121": (727, 364, 6955906), "densenet169": (1015, 508, 12487810),
         "densenet201": (1207, 604, 18096770), "densenet161": (967, 484, 26476418)}


@pytest.mark.parametrize("arch", DENSENET_ARCHS)
def test_spec_counts(arch):
    spec = get_spec(arch, num_classes=2)
    pe = param_entries(spec)
    assert (len(state_entries(spec)), len(pe), sum(math.prod(s) for _, s, _ in pe)) == TABLE[arch]
    assert arch not in SUPPORTED_ARCHS


def _torch_densenet_keys(spec, in_chans):
    """the key order of densenet.py's module tree, rebuilt from torch.nn modules with the same registration order"""
    feats = nn.Sequential()
    feats.add_module("conv0", nn.Conv2d(in_chans, spec.init_features, 7, 2, 3, bias=False))
    feats.add_module("norm0", nn.BatchNorm2d(spec.init_features))
    for b, (cin, cend) in enumerate(spec.block_widths):
        blk = nn.Sequential()
        for l in range(spec.block_config[b]):
            lay = nn.Sequential()
            c = cin + l * spec.growth
            lay.add_module("norm1", nn.BatchNorm2d(c))
            lay.add_module("conv1", nn.Conv2d(c, 4 * spec.growth, 1, bias=False))
            lay.add_module("norm2", nn.BatchNorm2d(4 * spec.growth))
            lay.add_module("conv2", nn.Conv2d(4 * spec.growth, spec.growth, 3, padding=1, bias=False))
            blk.add_module("denselayer%d" % (l + 1), lay)
        feats.add_module("denseblock%d" % (b + 1), blk)
        if b + 1 < len(spec.block_config):
            t = nn.Sequential()
            t.add_module("norm", nn.BatchNorm2d(cend))
            t.add_module("conv", nn.Conv2d(cend, cend // 2, 1, bias=False))
            feats.add_module("transition%d" % (b + 1), t)
    feats.add_module("norm5", nn.BatchNorm2d(spec.num_features))
    m = nn.Module()
    m.features = feats
    m.classifier = nn.Linear(spec.pooled_features, spec.num_classes)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


@pytest.mark.parametrize("arch,in_chans", [(a, 3) for a in DENSENET_ARCHS] + [("densenet121", 12)])
def test_state_keys_and_shapes(arch, in_chans):
    spec = get_spec(arch, num_classes=2, in_chans=in_chans)
    assert [(n, tuple(s)) for n, s, _ in state_entries(spec)] == _torch_densenet_keys(spec, in_chans)


def test_factory_rules_and_default_cfg():
    from deepfake_detection_b200.models import create_model
    m = create_model("densenet121", num_classes=2, bn_momentum=0.5, bn_eps=1e-3, bn_tf=True, drop_block_rate=None,
                     drop_path_rate=None)
    assert m.bn_momentum == 0.1 and m.bn_eps == 1e-5
    for k in ("drop_path_rate", "drop_block_rate"):
        with pytest.raises(TypeError):
            create_model("densenet121", num_classes=2, **{k: 0.1})
    cfg = m.default_cfg
    assert cfg["input_size"] == (3, 224, 224) and cfg["pool_size"] == (7, 7) and cfg["crop_pct"] == 0.875
    assert cfg["interpolation"] == "bicubic" and cfg["first_conv"] == "features.conv0" and cfg["classifier"] == "classifier"
    assert cfg["mean"] == (0.485, 0.456, 0.406) and cfg["std"] == (0.229, 0.224, 0.225)
    m = create_model("densenet161", num_classes=3, global_pool="catavgmax", drop_rate=0.2)
    assert m.spec.pooled_features == 2 * 2208 and m.drop_rate == 0.2
    with pytest.raises(RuntimeError):
        create_model("densenet264")


def test_init_statistics():
    from deepfake_detection_b200.models import init_state_dict
    spec = get_spec("densenet121", num_classes=2)
    sd = init_state_dict(spec, seed=0)
    for n in ("features.conv0.weight", "features.denseblock3.denselayer7.conv2.weight",
              "features.transition2.conv.weight"):
        w = sd[n]
        bound = 1.0 / math.sqrt(w[0].numel())
        assert float(w.abs().max()) <= bound and float(w.abs().max()) > 0.95 * bound
        assert abs(float(w.std()) - bound / math.sqrt(3)) < 0.05 * bound
    b = 1.0 / math.sqrt(1024)
    assert float(sd["classifier.weight"].abs().max()) <= b and float(sd["classifier.bias"].abs().max()) <= b
    assert bool((sd["features.norm5.weight"] == 1).all()) and bool((sd["features.norm5.bias"] == 0).all())


@pytest.mark.parametrize("arch", DENSENET_ARCHS)
@pytest.mark.parametrize("H,W", [(224, 224), (72, 88)])
@pytest.mark.parametrize("gemm_impl", ["tc", "mma"])
def test_plan_builds_and_census(arch, H, W, gemm_impl):
    from deepfake_detection_b200.engine import Engine
    e = Engine(arch, 2, H, W, device="plan-only", gemm_impl=gemm_impl)
    spec = e.spec
    L = sum(spec.block_config)
    fwd = Counter(n for _, n, _ in e.fwd_ops)
    bwd = Counter(n for _, n, _ in e.bwd_ops)
    assert fwd["dfd_bn_relu_ld"] == L and fwd["dfd_bn_relu_avgpool2"] == 3
    assert fwd["dfd_bn_finalize_ld"] == L + 4               # every norm1, the three transitions, norm5
    assert fwd["dfd_bn_finalize"] == L + 1                  # norm0 and every norm2 (statistics of their own)
    assert bwd["dfd_relu_bn_bwd_apply_add_ld"] == L and bwd["dfd_bn_relu_avgpool2_bwd_apply"] == 3
    assert bwd["dfd_unpack_grad"] == L
    if gemm_impl == "tc":
        assert fwd["dfd_conv3x3_narrow_tc"] == L and bwd["dfd_conv3x3_narrow_dgrad_tc"] == L
        assert bwd["dfd_conv_wgrad_tc"] == L
        assert fwd["dfd_copy_ld"] == 4                      # the stem pool and the three transitions into block prefixes
        assert not any("_mma" in n for n in fwd) and not any("_mma" in n for n in bwd)
    else:
        assert "dfd_conv3x3_narrow_tc" not in fwd and fwd["dfd_im2col"] == L and fwd["dfd_copy_ld"] == L + 4
    assert not any(n.endswith("_train") for n in fwd)        # no mask draw, no dropout launch at drop_rate 0
    assert sum(fwd.values()) == e.n_launch["fwd"] and sum(bwd.values()) == e.n_launch["bwd"]


def test_dropout_launches_only_with_drop_rate():
    from deepfake_detection_b200.engine import Engine
    e = Engine("densenet121", 2, 72, 88, device="plan-only", drop_rate=0.2)
    fwd = Counter(n for _, n, _ in e.fwd_ops)
    assert fwd["dfd_rng_masks_train"] == 1 and fwd["dfd_mul_f32_train"] == 1 and len(e.drop_masks) == 58
    assert fwd["dfd_copy_ld"] == 4 + 58
    e0 = Engine("densenet121", 2, 72, 88, device="plan-only", drop_rate=0.0)
    assert not e0.drop_masks and "dfd_rng_masks_train" not in Counter(n for _, n, _ in e0.fwd_ops)


def test_too_small_input_is_refused():
    from deepfake_detection_b200.engine import Engine
    with pytest.raises(ValueError):
        Engine("densenet121", 1, 24, 24, device="plan-only")


def test_restatement_matches_torch_modules():
    """tests/densenet_ref.py against the same network assembled from torch.nn layers in densenet.py's order (conv then pool in
    the transitions, dropout off)"""
    spec = get_spec("densenet121", num_classes=2)
    from deepfake_detection_b200.models import init_state_dict
    sd = {k: v.double() if v.is_floating_point() else v for k, v in init_state_dict(spec, seed=3).items()}
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 72, 88, generator=g, dtype=torch.float64)
    got = R.forward(spec, sd, x, training=False)
    W = lambda n: sd[n]

    def bn(t, p):
        return F.batch_norm(t, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False)
    h = F.max_pool2d(F.relu(bn(F.conv2d(x, W("features.conv0.weight"), stride=2, padding=3), "features.norm0")), 3, 2, 1)
    for b, n in enumerate(spec.block_config):
        for l in range(n):
            p = "features.denseblock%d.denselayer%d" % (b + 1, l + 1)
            z = F.conv2d(F.relu(bn(h, p + ".norm1")), W(p + ".conv1.weight"))
            z = F.conv2d(F.relu(bn(z, p + ".norm2")), W(p + ".conv2.weight"), padding=1)
            h = torch.cat([h, z], 1)
        if b < 3:
            p = "features.transition%d" % (b + 1)
            h = nn.AvgPool2d(2, 2)(F.conv2d(F.relu(bn(h, p + ".norm")), W(p + ".conv.weight")))
    ref = F.linear(F.adaptive_avg_pool2d(F.relu(bn(h, "features.norm5")), 1).flatten(1), W("classifier.weight"),
                   W("classifier.bias"))
    assert torch.allclose(got, ref, rtol=1e-9, atol=1e-12)


# ---- the reference's own numbers (tests/golden/, minted by tools/mint_densenet_goldens.py) ---------------------------------
def _golden(name):
    import json
    import os
    return json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name)))


@pytest.mark.parametrize("key", list(DENSENET_ARCHS) + ["densenet121@in_chans12"])
def test_state_keys_match_reference(key):
    ref = _golden("densenet_state_keys.json")[key]
    arch, _, ic = key.partition("@in_chans")
    spec = get_spec(arch, num_classes=2, in_chans=int(ic or 3))
    state = [[n, list(s)] for n, s, _ in state_entries(spec)]
    params = [[n, list(s)] for n, s, _ in param_entries(spec)]
    if "state" in ref:
        assert state == ref["state"] and params == ref["params"]
    assert digest(state) == ref["state_sha256"] and digest(params) == ref["params_sha256"]
    assert (len(state), len(params), sum(math.prod(s) for _, s in params)) == (ref["n_state"], ref["n_param_tensors"],
                                                                              ref["n_params"])


def _fixture_masks(rec, spec):
    import base64
    import numpy as np
    from deepfake_detection_b200.arch import densenet_extents
    keep = 1.0 - rec["drop_rate"]
    ms = [torch.from_numpy(np.unpackbits(np.frombuffer(base64.b64decode(m["bits"]), dtype=np.uint8))[:math.prod(m["shape"])]
                           .astype(np.float64)).view(m["shape"]) / keep for m in rec["masks"]]
    names = ["features.denseblock%d.denselayer%d" % (b + 1, l + 1) for b, n in enumerate(spec.block_config) for l in range(n)]
    assert len(ms) == len(names) + 1
    return {p: m.permute(0, 2, 3, 1) for p, m in zip(names, ms)}, ms[-1]


@pytest.mark.parametrize("name", ["step_densenet121_72x88.json", "step_densenet161_70x54.json", "step_densenet121_224.json",
                                  "step_densenet121_drop_48.json"])
def test_restatement_matches_reference_steps(name):
    """the restatement (fp32, as the reference ran), stepped with the oracle's SGD, against every recorded step of the
    reference at the tolerances of tests/test_oracle_vs_reference_goldens.py"""
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    torch.set_num_threads(8)
    rec = _golden(name)
    spec = get_spec(rec["arch"], num_classes=rec["num_classes"])
    sd = synth_state(spec, seed=rec["weight_seed"])
    masks, head = _fixture_masks(rec, spec) if "masks" in rec else (None, None)
    ost = OT.OptState(kind="sgd", lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"])
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i)
        new = {}
        loss, logits, grads = R.train_grads(spec, sd, x, y, masks=masks, head_mask=head, new_sd=new, dtype=torch.float32)
        assert loss == pytest.approx(st["loss"], rel=1e-4), (i, loss, st["loss"])
        check_summ(logits, st["logits"], "logits step %d" % i, 1e-3)
        rt = 2e-4 * (1 if i == 0 else 25)           # after the first update fp32 differences are amplified through BN
        gfloor = 1e-5 * max(v["norm"] / max(grads[k].numel(), 1) ** 0.5 for k, v in st["grads"].items())
        for n, s in st["grads"].items():
            check_summ(grads[n], s, "grad %s step %d" % (n, i), rt, floor=gfloor)
        params = {n: sd[n].clone() for n in grads}
        OT.optimizer_step(ost, params, grads)
        sd.update(params)
        sd.update(new)
        for n, s in st["params"].items():
            check_summ(sd[n], s, "param %s step %d" % (n, i), rt)
        for n, s in st.get("buffers", {}).items():
            check_summ(sd[n], s, "buffer %s step %d" % (n, i), rt)
    if "eval" in rec:
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=999)
        with torch.no_grad():
            check_summ(R.forward(spec, sd, x, training=False), rec["eval"]["logits"], "eval logits", 5e-3)
