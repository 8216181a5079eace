"""Host logic of the TensorFlow-ported EfficientNets (tf_efficientnet_b0..b7, _ap, _ns), no GPU: the specs against the
reference's state keys, the engine's TF "SAME" pads against the reference's own `pad_same`, the oracle against the reference's
eval logits, the model factory's BatchNorm and default_cfg rules, the plans (where they differ from the symmetric models and
where they must not), and the coverage contract of the GPU file's kernel cases. Fixtures: tools/mint_tf_goldens.py; their
train steps are held by tests/reference_steps.py's tables."""
import json
import os

import pytest
import torch

import tf_same_cases as TC
from deepfake_detection_b200 import _lib
from deepfake_detection_b200.arch import SUPPORTED_ARCHS, TF_ARCHS, conv_pads, get_spec, param_entries, state_entries
from deepfake_detection_b200.engine import Engine, base_name
from oracle import train as OT
from oracle.weights import synth_batch, synth_state
from reference_steps import digest


def test_tf_archs_are_the_24_entrypoints_and_supported_archs_unchanged():
    assert len(TF_ARCHS) == 24 and len(set(TF_ARCHS)) == 24
    assert {a[: len("tf_efficientnet_b0")] for a in TF_ARCHS} == {"tf_efficientnet_b%d" % i for i in range(8)}
    assert SUPPORTED_ARCHS == ("efficientnet_b0", "efficientnet_b4", "efficientnet_deepfake_v4", "resnet18", "resnet50")
    assert get_spec("efficientnet_b0").pad_type == "" and all(get_spec(a).pad_type == "same" for a in TF_ARCHS)


@pytest.mark.parametrize("key", list(TF_ARCHS) + ["tf_efficientnet_b7@in_chans12"])
def test_specs_match_reference_state_keys(key, golden_dir):
    ref = json.load(open(os.path.join(golden_dir, "tf_state_keys.json")))[key]
    arch, _, ic = key.partition("@in_chans")
    spec = get_spec(arch, num_classes=2, in_chans=int(ic or 3))
    state = [[n, list(s)] for n, s, _ in state_entries(spec)]
    params = [[n, list(s)] for n, s, _ in param_entries(spec)]
    if "state" in ref:          # tf_efficientnet_b0 in full: a mismatch shows the first differing entry
        assert state == ref["state"] and params == ref["params"]
    assert (len(state), len(params)) == (ref["n_state"], ref["n_param_tensors"])
    assert digest(state) == ref["state_sha256"] and digest(params) == ref["params_sha256"]
    n = 0
    for _, s, _ in param_entries(spec):
        k = 1
        for d in s:
            k *= d
        n += k
    assert n == ref["n_params"]


def _pad_case_id(c):
    return "%s-%dx%d" % (c["arch"], c["H"], c["W"])


_PAD_CASES = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tf_pad_same.json")))


@pytest.mark.parametrize("case", _PAD_CASES, ids=_pad_case_id)
def test_engine_pads_match_reference_pad_same(case):
    """every layer the reference pads dynamically (the stride-2 stem and depthwise convs; stride-1 'same' is static and
    symmetric) gets the reference's (top, left) pad and output extent in the plan"""
    e = Engine(case["arch"], 1, case["H"], case["W"], device="plan-only")
    assert e.conv_pads == conv_pads(e.spec, case["H"], case["W"])
    mine = [dict(k=k, s=s, h=h, w=w, top=pt, left=pl, ho=ho, wo=wo) for _, k, s, h, w, pt, pl, ho, wo in e.conv_pads if s == 2]
    ref = [{k: v for k, v in d.items() if k not in ("bottom", "right")} for d in case["layers"]]
    assert mine == ref
    for _, k, s, h, w, pt, pl, ho, wo in e.conv_pads:
        if s == 1:
            assert (pt, pl) == ((k - 1) // 2, (k - 1) // 2) and (ho, wo) == (h, w)
    last = e.conv_pads[-1]
    assert [last[7], last[8]] == case["final"]


def test_issue_pad_table_at_default_resolutions():
    """B0 @224: every stride-2 layer asymmetric; B4 @380 symmetric only at stage 2 (k5 at 95); B7 @600 only at stage 3"""
    def asym(arch):
        spec = get_spec(arch)
        r = spec.input_size[1]
        return [(n, pt, pl) for n, k, s, h, w, pt, pl, ho, wo in conv_pads(spec, r, r) if s == 2 and pt != (k - 1) // 2]
    assert [n for n, _, _ in asym("tf_efficientnet_b0")] == ["conv_stem", "blocks.1.0.conv_dw", "blocks.2.0.conv_dw",
                                                             "blocks.3.0.conv_dw", "blocks.5.0.conv_dw"]
    assert "blocks.2.0.conv_dw" not in [n for n, _, _ in asym("tf_efficientnet_b4")] and len(asym("tf_efficientnet_b4")) == 4
    assert "blocks.3.0.conv_dw" not in [n for n, _, _ in asym("tf_efficientnet_b7")] and len(asym("tf_efficientnet_b7")) == 4


def test_oracle_eval_logits_match_reference(golden_dir):
    rec = json.load(open(os.path.join(golden_dir, "tf_eval_b0_224.json")))
    spec = get_spec(rec["arch"])
    x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=rec["input_seed"])
    ev = OT.validate_step(spec, synth_state(spec, seed=rec["weight_seed"]), x, y)
    ref = torch.tensor(rec["logits"])
    assert torch.allclose(ev["logits"], ref, rtol=1e-4, atol=1e-5), (ev["logits"], ref)


def test_model_bn_and_default_cfg_rules():
    from deepfake_detection_b200.models import create_model
    m = create_model("tf_efficientnet_b3", num_classes=2)
    assert (m.bn_eps, m.bn_momentum) == (1e-3, 0.1)
    assert create_model("tf_efficientnet_b0", num_classes=2, bn_eps=1e-5).bn_eps == 1e-3       # the caller's value is overridden
    m = create_model("tf_efficientnet_b0", num_classes=2, bn_tf=True)
    assert (m.bn_eps, m.bn_momentum) == (1e-3, pytest.approx(0.01))
    assert create_model("tf_efficientnet_b0", num_classes=2, bn_momentum=0.05).bn_momentum == 0.05
    assert create_model("efficientnet_b0", num_classes=2).bn_eps == 1e-5
    want = {0: (224, (7, 7), 0.875), 1: (240, (8, 8), 0.882), 2: (260, (9, 9), 0.890), 3: (300, (10, 10), 0.904),
            4: (380, (12, 12), 0.922), 5: (456, (15, 15), 0.934), 6: (528, (17, 17), 0.942), 7: (600, (19, 19), 0.949)}
    for a in TF_ARCHS:
        c = create_model(a, num_classes=2).default_cfg
        r, pool, crop = want[int(a[len("tf_efficientnet_b")])]
        assert c["input_size"] == (3, r, r) and c["pool_size"] == pool and c["crop_pct"] == crop, a
        inception = a.endswith("_ap")
        assert c["mean"] == ((0.5,) * 3 if inception else (0.485, 0.456, 0.406)), a
        assert c["std"] == ((0.5,) * 3 if inception else (0.229, 0.224, 0.225)), a
        assert c["interpolation"] == "bicubic" and c["first_conv"] == "conv_stem" and c["classifier"] == "classifier"
    with pytest.raises(RuntimeError, match="Unknown model"):
        create_model("tf_efficientnet_b8", num_classes=2)
    with pytest.raises(_lib.NativeError):
        create_model("tf_efficientnet_b0", pretrained=True)


@pytest.mark.parametrize("arch,in_chans", [(a, 3) for a in TC.DEFAULT_ARCHS] + [("tf_efficientnet_b7", 12)])
def test_plan_only_engines_build_at_default_resolution(arch, in_chans):
    e = Engine(arch, 2, device="plan-only", in_chans=in_chans, bn_eps=1e-3)
    r = e.spec.input_size[1]
    assert (e.H, e.W) == (r, r) and e.x_in.shape == (2, in_chans, r, r)
    names = [n for _, n, _ in e.fwd_ops + e.bwd_ops]
    assert names.count("dfd_stem_im2col_pad") == 1 and "dfd_stem_im2col" not in names       # every default resolution is even
    n_asym = sum(1 for n, k, s, *_r in e.conv_pads[1:] if s == 2 and (_r[2], _r[3]) != ((k - 1) // 2,) * 2)
    assert names.count("dfd_dwconv_fwd_pad") == n_asym and names.count("dfd_dwconv_bwd_pad") == n_asym


def _norm(name, args):
    """a planned launch with every pointer argument reduced to NULL / non-NULL (two engines own different buffers)"""
    codes = _lib.SIGNATURES[base_name(name)]
    out = []
    for v, c in zip(args, codes):
        if isinstance(v, tuple) and v[0] == "TRAIN_ONLY":
            v = v[1]
        out.append(("ptr" if v else None) if c == "p" else v)
    return out


def test_b0_and_tf_b0_plans_differ_only_in_the_padded_launches():
    sym = Engine("efficientnet_b0", 4, 224, 224, device="plan-only", bn_eps=1e-3)
    tf = Engine("tf_efficientnet_b0", 4, 224, 224, device="plan-only", bn_eps=1e-3)
    pads = {n: (pt, pl) for n, k, s, h, w, pt, pl, ho, wo in tf.conv_pads}
    for part in ("fwd_ops", "bwd_ops"):
        a, b = getattr(sym, part), getattr(tf, part)
        assert len(a) == len(b)
        changed = []
        for (_, na, aa), (_, nb, ab) in zip(a, b):
            if na == nb:
                assert _norm(na, aa) == _norm(nb, ab), na
                continue
            assert nb == na + "_pad", (na, nb)
            changed.append(nb)
            x, y = _norm(na, aa), _norm(nb, ab)
            if na == "dfd_stem_im2col":
                assert x[:8] == y[:8] and x[8] == 1 and tuple(y[8:10]) == pads["conv_stem"] and x[9:] == y[10:]
            else:
                i = 11 if na == "dfd_dwconv_fwd" else 20
                assert x[:i] == y[:i] and x[i:] == y[i + 2:] and (y[i], y[i + 1]) in pads.values()
        # at 224 the stem and the stride-2 depthwise convs of stages 1, 2, 3 and 5 are asymmetric (0/1 for k3, 1/2 for k5)
        want = (["dfd_stem_im2col_pad"] + ["dfd_dwconv_fwd_pad"] * 4) if part == "fwd_ops" else ["dfd_dwconv_bwd_pad"] * 4
        assert changed == want


def test_tf_plan_at_all_odd_extents_issues_no_new_kernel():
    e = Engine("tf_efficientnet_b0", 2, 225, 225, device="plan-only")
    assert all(s == 1 or (pt, pl) == ((k - 1) // 2,) * 2 for _, k, s, h, w, pt, pl, ho, wo in e.conv_pads)
    names = {n for _, n, _ in e.fwd_ops + e.bwd_ops}
    assert not names & set(TC.NEW_KERNELS)


def test_padded_forward_marks_its_statistics_training_only():
    """the padded depthwise forward's batch statistics are training-only operands: NULL in eval mode, their pointers in
    training, every other argument as planned in both modes"""
    e = Engine("tf_efficientnet_b0", 2, 64, 96, device="plan-only")
    op = next((n, a) for _, n, a in e.fwd_ops if n == "dfd_dwconv_fwd_pad")
    ev = e.launch_args(op[0], op[1], False)
    assert ev[:-3] == tuple(op[1][:-3]) and ev[-3:] == (None, None, None)
    # training runs the op as planned: only the statistics are marked training-only, and they resolve to their pointers
    bn = e.bns["blocks.1.0.bn2"]
    assert op[1][-3:] == (("TRAIN_ONLY", bn.fsum), ("TRAIN_ONLY", bn.fsq), None)
    assert e.launch_args(op[0], op[1], True) == tuple(op[1][:-3]) + (bn.fsum, bn.fsq, None)


def test_gpu_cases_cover_every_new_launch_of_the_default_plans():
    """coverage contract: the GPU file runs one kernel case per distinct launch shape of the new kernels in the eight default
    training plans (at tf_same_cases.CASE_BATCH, a stated reduced batch), plus the non-square EXTRA_CASES"""
    shapes = TC.default_shapes()
    assert list(shapes) == TC.DEFAULT_CASES           # the written-out list the GPU file parametrises over is current
    assert set(k for k, *_ in shapes) == set(TC.NEW_KERNELS)
    import test_tf_efficientnet_gpu as G
    cases = set(G.KERNEL_CASES)
    missing = [s for s in shapes if s not in cases]
    assert not missing, missing
    assert all(s in cases for s in TC.EXTRA_CASES)
    # every new launch shape is a TF "SAME" pad the kernels accept: one short on the begin side over an even extent
    for name, H, W, C, k, s, pt, pl in cases:
        assert s == 2 and (pt, pl) != ((k - 1) // 2,) * 2
        assert pt == ((k - 1) // 2 if H % 2 else (k - 1) // 2 - 1) and pl == ((k - 1) // 2 if W % 2 else (k - 1) // 2 - 1)
    # the reduced batch of the GPU cases is stated, and smaller than the plans'
    assert G.CASE_BATCH == TC.CASE_BATCH < TC.PLAN_BATCH
