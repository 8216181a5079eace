"""-m gpu: the TensorFlow-ported EfficientNets on the native path.

  * every distinct launch of the TF "SAME" kernels in the eight default plans (tests/tf_same_cases.py, at its stated reduced
    batch) and the non-square cases, in bf16 and fp16, against fp64 torch (tests/tf_same_checks.py); at symmetric pads the
    new entry points equal the old ones bit for bit;
  * graph-captured tf_efficientnet_b0 Trainer steps (bf16; fp16 with dynamic loss scaling) against the oracle
    (tests/tf_same_oracle.py) and the reference's step fixtures, identical bits over two runs; one tf_efficientnet_b4 step at
    380² against the oracle;
  * the reference's eval logits of tf_efficientnet_b0 at 224², and the runner's train_epoch / validate on a tf model.
No test here reads the reference tree: the fixtures under tests/golden/ came from tools/mint_tf_goldens.py.
"""
import json
import os
from types import SimpleNamespace

import pytest
import torch

import tf_same_cases as TC

pytestmark = pytest.mark.gpu

CASE_BATCH = TC.CASE_BATCH
KERNEL_CASES = TC.DEFAULT_CASES + TC.EXTRA_CASES
RED = 2e-3          # fp32 reductions of 16-bit data (tests/gpu_checks.py)


def _tc():
    import tf_same_checks
    return tf_same_checks


def _dt(name):
    return torch.bfloat16 if name == "bf16" else torch.float16


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("case", KERNEL_CASES, ids=lambda c: "%s-%dx%dx%d-k%d-p%d%d" % (c[0][4:], c[1], c[2], c[3], c[4], c[6], c[7]))
def test_new_kernel_launch(case, dtype):
    name, H, W, C, k, s, pt, pl = case
    if name == "dfd_stem_im2col_pad":
        r = _tc().check_stem_im2col_pad(CASE_BATCH, C, H, W, k, s, pt, pl, dtype=_dt(dtype))
        assert r["nan"] == 0 and r["diff"] == 0.0 and r["pad_max"] == 0.0, r
        return
    r = _tc().check_dw_pad(CASE_BATCH, H, W, C, k, s, pt, pl, dtype=_dt(dtype), bwd=name == "dfd_dwconv_bwd_pad")
    assert r["nan"] == 0 and r["fwd_ulp"] <= 1.0 and r["sum_rel"] < RED and r["sq_rel"] < RED, r
    if name == "dfd_dwconv_bwd_pad":
        # input gradient: tanh.approx sigmoid (2^-11 relative) and 16-bit storage, as in tests/test_kernels_gpu.py::test_dwconv
        assert r["nan_b"] == 0 and r["dgrad_rel"] < 8e-3 and r["wgrad_rel"] < RED, r
        assert r["bs1_rel"] < RED and r["bs2_rel"] < RED and r["bwd_bitwise"], r


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("H,W,C,k", [(57, 57, 144, 5), (27, 33, 96, 3), (21, 21, 32, 3)])
def test_symmetric_pads_equal_the_symmetric_entry_points(H, W, C, k, dtype):
    """TF "SAME" over odd extents at stride 2 is the symmetric (k-1)/2: the new entry points then run the symmetric kernels and
    give the same bits"""
    pt = pl = (k - 1) // 2
    r = _tc().check_dw_pad(CASE_BATCH, H, W, C, k, 2, pt, pl, dtype=_dt(dtype))
    assert r["sym_fwd_mismatch"] == 0 and r["sym_bwd_mismatch"] == 0 and r["fwd_ulp"] <= 1.0, r
    s = _tc().check_stem_im2col_pad(CASE_BATCH, 3, H, W, 3, 2, 1, 1, dtype=_dt(dtype))
    assert s["sym_mismatch"] == 0 and s["diff"] == 0.0, s


# ---- whole steps --------------------------------------------------------------------------------------------------------
def _trainer(arch, batch, H, W, dtype, sd):
    from deepfake_detection_b200.trainer import Trainer
    tr = Trainer(arch, batch, H, W, dtype=dtype, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, bn_eps=1e-3)
    tr.engine.load_state_dict(sd)
    return tr


def _relerr(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _run_steps(arch, batch, H, W, dtype, steps):
    from deepfake_detection_b200.arch import get_spec
    from oracle.weights import synth_batch, synth_state
    spec = get_spec(arch)
    sd0 = synth_state(spec, seed=7)
    tr = _trainer(arch, batch, H, W, dtype, sd0)
    out = []
    for i in range(steps):
        x, y = synth_batch(batch, 3, H, W, seed=1234 + i)
        e = tr.engine
        scale = float(e.loss_scale_state[0])        # fp16: the gradient arena holds loss-scaled gradients (1 in bf16)
        loss, _ = tr.train_step(x.cuda(), y.cuda())
        torch.cuda.synchronize()
        out.append(dict(loss=float(loss), logits=e.logits.detach().cpu().clone(), scale=scale,
                        grads=e.grads32.detach().cpu().clone(), params=e.params32.detach().cpu().clone()))
    assert tr.use_graph and tr.n_captures >= 1
    return spec, sd0, tr, out


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("H,W", [(64, 96), (66, 96)])
def test_tf_b0_captured_steps_match_oracle_and_reference(H, W, dtype, golden_dir):
    import tf_same_oracle as TO
    from deepfake_detection_b200.arch import param_entries
    from oracle import train as OT
    from oracle.weights import synth_batch
    arch, batch = "tf_efficientnet_b0", 4
    spec, sd0, tr, runs = _run_steps(arch, batch, H, W, dtype, 2)
    _, _, _, runs2 = _run_steps(arch, batch, H, W, dtype, 2)
    for a, b in zip(runs, runs2):                    # order-deterministic gradients: two runs give identical bits
        assert torch.equal(a["logits"], b["logits"]) and torch.equal(a["grads"], b["grads"]) and torch.equal(a["params"], b["params"])
    # the oracle, with the activations rounded where the native path stores them
    sd = {k: v.clone() for k, v in sd0.items()}
    ost = OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    e = tr.engine
    emul_loss = []
    for i, r in enumerate(runs):
        x, y = synth_batch(batch, 3, H, W, seed=1234 + i)
        o = TO.train_step(spec, sd, x, y, ost, act_dtype=_dt(dtype))
        emul_loss.append(float(o["loss"]))
        # tests/test_engine_gpu.py's step tolerances for B0 (fp16 per step; bf16 as its emulation bound). Batch 4 is a chaotic
        # regime for bf16 storage after the first update (the oracle's own bf16 emulation moves the step-1 logits by tens of
        # percent): there bf16 step 1 is held to the loss only, as tests/test_engine_gpu.py does with its batch-4 fixture
        lrel = _relerr(r["logits"], o["logits"])
        if dtype == "fp16" or i == 0:
            assert lrel < (2e-2 if dtype == "fp16" else 6e-2) * (1 + i), (i, lrel)
        assert abs(r["loss"] - float(o["loss"])) < (3e-3 if dtype == "fp16" else 1e-2) * (1 + i), (i, r["loss"], float(o["loss"]))
        if i == 0:
            # gradients against the fp32 oracle, relative to the yardstick of tests/test_engine_gpu.py: how far the oracle's own
            # 16-bit emulation lands from fp32 (batch 4 at 64x96 normalises the last stages over few values per channel, so
            # 16-bit rounding alone moves the gradients by tens of percent, oracle included)
            o32 = TO.train_step(spec, {k: v.clone() for k, v in sd0.items()}, x, y, None)
            names = [n for n, _, _ in param_entries(spec)]
            gn = torch.cat([r["grads"][e.p_off[n][0]:e.p_off[n][0] + e.p_off[n][2]] for n in names]) / r["scale"]
            go, g32 = (torch.cat([oo["grads"][n].flatten() for n in names]) for oo in (o, o32))
            yard = _relerr(go, g32)
            assert _relerr(gn, g32) < 1.5 * yard + 3e-2, (_relerr(gn, g32), yard)
    # the reference's own fp32 steps (fixture): step 0 tightly, step 1 on the loss (tests/test_engine_gpu.py::test_golden_b0),
    # each widened by the distance of the oracle's 16-bit emulation from the fixture (the rounding any 16-bit path pays)
    rec = json.load(open(os.path.join(golden_dir, "step_tf_efficientnet_b0_%dx%d.json" % (H, W))))
    for i, (r, st) in enumerate(zip(runs, rec["steps"])):
        yard = abs(emul_loss[i] - st["loss"])
        assert abs(r["loss"] - st["loss"]) < (1e-2 if i == 0 else 5e-2) * abs(st["loss"]) + yard, (i, r["loss"], st["loss"], yard)
        if i == 0:
            f = r["logits"].double().flatten()
            ref = torch.tensor(st["logits"]["samples"], dtype=torch.float64)
            got = f[torch.tensor(st["logits"]["idx"])]
            assert float((got - ref).norm() / ref.norm()) < 7e-2, (got, ref)


def test_tf_b4_step_at_380_matches_oracle():
    """reduced batch (2): one fp16 step of the full-resolution B4 plan against the oracle"""
    import tf_same_oracle as TO
    from oracle import train as OT
    from oracle.weights import synth_batch
    spec, sd0, tr, runs = _run_steps("tf_efficientnet_b4", 2, 380, 380, "fp16", 1)
    x, y = synth_batch(2, 3, 380, 380, seed=1234)
    o = TO.train_step(spec, {k: v.clone() for k, v in sd0.items()}, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9,
                                                                                        weight_decay=1e-4), act_dtype=torch.float16)
    assert _relerr(runs[0]["logits"], o["logits"]) < 2e-2
    assert abs(runs[0]["loss"] - float(o["loss"])) < 5e-3


def test_eval_logits_match_reference_fixture(golden_dir):
    """the fixture weights in create_model('tf_efficientnet_b0') reproduce the reference's eval logits; the same weights under
    efficientnet_b0 with bn_eps=1e-3 (so only the padding differs) land clearly further away: the padding is what is tested.
    With these synthetic weights the logits barely depend on the input (the classifier bias dominates): the fp16 oracle is
    2.4e-5 of max|logit| from the fixture on the CPU and symmetric padding 3.8e-3, so the bounds are stated in max|logit|."""
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from oracle.weights import synth_batch, synth_state
    rec = json.load(open(os.path.join(golden_dir, "tf_eval_b0_224.json")))
    sd = synth_state(get_spec(rec["arch"]), seed=rec["weight_seed"])
    x, _ = synth_batch(rec["batch"], 3, 224, 224, seed=rec["input_seed"])
    ref = torch.tensor(rec["logits"], dtype=torch.float64)
    errs = {}
    for arch in ("tf_efficientnet_b0", "efficientnet_b0"):
        m = create_model(arch, num_classes=2, dtype="fp16", bn_eps=1e-3)
        m.load_state_dict(sd)
        m.eval()
        with torch.no_grad():
            out = m(x.cuda()).double().cpu()
        errs[arch] = float((out - ref).abs().max() / ref.abs().max())
    assert errs["tf_efficientnet_b0"] < 1.2e-3, errs
    assert errs["efficientnet_b0"] > 2.5e-3 and errs["efficientnet_b0"] > 3 * errs["tf_efficientnet_b0"], errs


def test_runner_train_epoch_and_validate_on_tf_model():
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch, validate
    from oracle.weights import synth_batch, synth_state

    class _Loader(list):
        mixup_enabled = False

    args = SimpleNamespace(opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0,
                           mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0,
                           log_interval=1, save_images=False, recovery_interval=0, tta=0, model="tf_efficientnet_b0")
    model = create_model("tf_efficientnet_b0", num_classes=2, dtype="fp16")
    model.load_state_dict(synth_state(get_spec("tf_efficientnet_b0"), seed=7))
    opt = create_optimizer(args, model)
    batches = _Loader((x.cuda(), y.cuda()) for x, y in (synth_batch(8, 3, 96, 96, seed=1234 + i) for i in range(2)))
    m = train_epoch(0, model, batches, opt, torch.nn.CrossEntropyLoss(), args)
    v = validate(model, batches, torch.nn.CrossEntropyLoss(), args)
    assert set(m) == {"loss", "prec1", "learning_rate"} and 0.0 < m["loss"] < 5.0, m
    assert 0.0 < v["loss"] < 5.0 and all(torch.isfinite(t).all() for t in model.state_dict().values() if t.is_floating_point()), v
