"""Pins oracle/ (the CPU restatement) to the reference: every fixture under tests/golden/ was produced by
the UNMODIFIED reference (oracle/mint_goldens.py, tools/mint_*_goldens.py); here the oracle must reproduce them in fp32 on CPU.
Tolerance: 2e-4 relative on norms / 1e-4 absolute+relative on samples (same fp32 arithmetic, possibly
different op ordering inside torch between the module and functional forms)."""
import glob
import importlib
import json
import os

import pytest
import torch

import reference_steps as RS
from deepfake_detection_b200.arch import get_spec
from oracle import model as OM
from oracle import train as OT
from oracle.weights import synth_batch, synth_state, tame_state
from reference_steps import DECAY_PER_LR, RTOL, check_summ


@pytest.mark.parametrize("case", RS.CPU_STEPS)
def test_oracle_matches_reference_steps(case, golden_dir):
    """oracle.train.train_step / validate_step, which read every field of the spec they are given, against the reference's
    own train steps and eval; what runs comes from the fixture's fields"""
    rec = RS.load(golden_dir, case)
    assert rec.get("drop_rate", 0.0) == 0.0
    K = rec.get("num_classes", 2)
    torch.set_num_threads(8)
    spec = get_spec(rec["arch"], num_classes=K, global_pool=rec.get("global_pool", "avg"))
    sd = synth_state(spec, seed=rec["weight_seed"])
    if "tame" in rec:
        sd = tame_state(spec, sd, rec["tame"])
    wd = rec["weight_decay"] / rec["lr"] if rec["opt"] in DECAY_PER_LR else rec["weight_decay"]
    opt = OT.OptState(kind=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=wd, eps=1e-8)
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i, soft=rec["soft"], num_classes=K)
        out = OT.train_step(spec, sd, x, y, opt, smoothing=rec["smoothing"])
        assert out["logits"].shape == (rec["batch"], K)
        if isinstance(st["logits"], list):
            ref = torch.tensor(st["logits"])
            assert torch.allclose(out["logits"], ref, rtol=1e-3, atol=1e-4 * float(ref.abs().max() + 1)), "logits step %d" % i
        else:
            check_summ(out["logits"], st["logits"], "logits step %d" % i, rtol=1e-3)
        assert float(out["loss"]) == pytest.approx(st["loss"], rel=1e-4)
        assert float(out["prec1"]) == pytest.approx(st["prec1"], abs=1e-3)
        # after the first update tiny fp32 differences are amplified through BN: loosen progressively
        rt = RTOL * (1 if i == 0 else 25)
        gfloor = 1e-5 * max(v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 for k, v in st["grads"].items())
        for k, s in st["grads"].items():
            check_summ(out["grads"][k], s, "grad %s step %d" % (k, i), rt, floor=gfloor)
        # adaptive optimizers normalise the gradient, so a mathematically-zero (round-off) gradient becomes an O(lr) random
        # update in BOTH implementations: such parameters carry no parity information
        noise = {k for k, v in st["grads"].items()
                 if v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 < 10 * gfloor} if rec["opt"] != "sgd" else set()
        for k, s in st["params"].items():
            if k not in noise:
                check_summ(sd[k], s, "param %s step %d" % (k, i), rt)
        for k, s in st["buffers"].items():
            check_summ(sd[k].float(), s, "buffer %s step %d" % (k, i), rt)
    x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=999, num_classes=K)
    ev = OT.validate_step(spec, sd, x, y)
    if isinstance(rec["eval"]["logits"], list):
        ref = torch.tensor(rec["eval"]["logits"])
        assert torch.allclose(ev["logits"], ref, rtol=5e-3, atol=5e-3 * float(ref.abs().max())), "eval logits"
    else:
        check_summ(ev["logits"], rec["eval"]["logits"], "eval logits", rtol=5e-3)
    assert float(ev["loss"]) == pytest.approx(rec["eval"]["loss"], rel=2e-3)


def test_every_step_fixture_is_checked_once(golden_dir):
    """each tests/golden/step_*.json is held by the table above or by one named test, never both; the native path's table
    is a subset of the oracle's"""
    on_disk = {os.path.basename(p)[:-len(".json")] for p in glob.glob(os.path.join(golden_dir, "step_*.json"))}
    cpu = RS.CPU_STEPS
    elsewhere = [c for c, _ in RS.ELSEWHERE]
    assert len(set(cpu)) == len(cpu) and len(set(elsewhere)) == len(elsewhere)
    assert not set(cpu) & set(elsewhere)
    assert set(cpu) | set(elsewhere) == on_disk, (on_disk - set(cpu) - set(elsewhere), set(cpu) | set(elsewhere) - on_disk)
    gpu = [c for c, _ in RS.GPU_STEPS]
    assert len(set(gpu)) == len(gpu) and set(gpu) <= set(cpu), set(gpu) - set(cpu)
    for case, o in RS.GPU_STEPS:
        assert o["kind"] in ("engine", "tamed") and o["dtypes"] and set(o["dtypes"]) <= {"bf16", "fp16"}, case
    for case, test in RS.ELSEWHERE:
        module, _, name = test.partition("::")
        assert name.startswith("test_") and callable(getattr(importlib.import_module(module), name, None)), (case, test)


def test_optimizers_match_reference(golden_dir):
    rec = json.load(open(os.path.join(golden_dir, "optimizers.json")))
    for name, r in rec.items():
        g0 = torch.Generator().manual_seed(3)
        params = {"w": torch.randn(5, 7, generator=g0), "bias": torch.randn(7, generator=g0),
                  "k": torch.randn(4, 1, 3, 3, generator=g0)}
        wd = r["weight_decay"] / r["lr"] if name in DECAY_PER_LR else r["weight_decay"]
        opt = OT.OptState(kind=name, lr=r["lr"], momentum=r["momentum"], weight_decay=wd, eps=r["eps"])
        g = torch.Generator().manual_seed(11)
        for step in range(3):
            grads = {k: torch.randn(p.shape, generator=g) for k, p in params.items()}
            OT.optimizer_step(opt, params, grads)
            for k, p in params.items():
                ref = torch.tensor(r["hist"][step][k])
                assert torch.allclose(p.reshape(-1), ref, rtol=1e-5, atol=1e-6), (name, step, k)


def test_bce_form_equals_two_class_ce():
    """SURVEY.md 8a H2: the fused head's sigmoid-BCE on z1-z0 is exactly the reference's softmax-CE."""
    g = torch.Generator().manual_seed(0)
    z = torch.randn(64, 2, generator=g) * 3
    y = torch.randint(0, 2, (64,), generator=g)
    for sm in (0.0, 0.1):
        assert torch.allclose(OM.bce_two_class(z, y, sm), OM.cross_entropy(z, y, sm), atol=1e-6)
    soft = torch.softmax(torch.randn(64, 2, generator=g), -1)
    assert torch.allclose(OM.bce_two_class(z, soft), OM.cross_entropy(z, soft), atol=1e-6)


def test_runner_config1_resnet18(golden_dir):
    """BASELINE config 1 (ResNet-18, batch 8, 224, world_size 1): the reference's own train_epoch/validate
    metrics and final weights, reproduced by the oracle's step restatement."""
    rec = json.load(open(os.path.join(golden_dir, "runner_config1_resnet18.json")))
    torch.set_num_threads(8)
    spec = get_spec("resnet18")
    sd = synth_state(spec, seed=7)
    opt = OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    losses, precs = [], []
    batches = [synth_batch(8, 3, 224, 224, seed=1234 + i) for i in range(2)]
    for x, y in batches:
        o = OT.train_step(spec, sd, x, y, opt)
        losses.append(float(o["loss"]))
        precs.append(float(o["prec1"]))
    assert sum(losses) / 2 == pytest.approx(rec["train"]["loss"], rel=1e-4)
    assert sum(precs) / 2 == pytest.approx(rec["train"]["prec1"], abs=1e-3)
    vl = [float(OT.validate_step(spec, sd, x, y)["loss"]) for x, y in batches]
    assert sum(vl) / 2 == pytest.approx(rec["validate"]["loss"], rel=2e-3)
    for k, s in rec["params"].items():
        check_summ(sd[k], s, "param " + k, 25 * RTOL)


def test_dropped_step_matches_reference(golden_dir):
    """Stochastic depth + classifier dropout (scripts/train.sh production flags): the oracle, given the masks the reference
    drew, reproduces the reference's logits / loss / gradients / updated weights; the per-block rates follow the linear
    ramp of efficientnet_builder.py (drop_path_rate * block_idx / n_blocks)."""
    rec = json.load(open(os.path.join(golden_dir, "step_efficientnet_b0_dropped.json")))
    torch.set_num_threads(8)
    spec = get_spec(rec["arch"])
    n_blocks = len(spec.blocks)
    for i, (name, rate) in enumerate(rec["block_rates"]):
        assert name == spec.blocks[i].name and rate == pytest.approx(rec["drop_path_rate"] * i / n_blocks, abs=1e-7)
    sd = synth_state(spec, seed=rec["weight_seed"])
    x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234)
    masks = {k: torch.tensor(v) for k, v in rec["drop_masks"].items()}
    assert set(masks) == {b.name for i, b in enumerate(spec.blocks) if b.has_residual and i > 0}
    opt = OT.OptState(kind="sgd", lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"])
    out = OT.train_step(spec, sd, x, y, opt, drop_masks=masks, dropout_mask=torch.tensor(rec["dropout_mask"]))
    ref = torch.tensor(rec["logits"])
    assert torch.allclose(out["logits"], ref, rtol=1e-3, atol=1e-4 * float(ref.abs().max() + 1))
    assert float(out["loss"]) == pytest.approx(rec["loss"], rel=1e-4)
    gfloor = 1e-5 * max(v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 for k, v in rec["grads"].items())
    for k, s in rec["grads"].items():
        check_summ(out["grads"][k], s, "grad " + k, RTOL, floor=gfloor)
    for k, s in rec["params"].items():
        check_summ(sd[k], s, "param " + k, RTOL)


def test_aux_formulas_match_reference(golden_dir):
    """drop_path (layers/drop.py:84-100), the prefetcher's normalisation (loader.py:229-253) and ModelEma.update
    (utils.py:329-340) as the formulas the native kernels implement (tests/gpu_checks.py compares the kernels with these)."""
    from oracle import formulas as OF
    rec = json.load(open(os.path.join(golden_dir, "aux_formulas.json")))
    d = rec["drop_path"]
    mask = OF.drop_path_mask(torch.tensor(d["u"]), d["drop_prob"])
    # the reference computes x.div(keep) * binary_mask, the oracle / kernels x * (binary_mask / keep): equal to one fp32 ulp
    assert torch.allclose(torch.tensor(d["x"]) * mask.view(-1, 1, 1, 1), torch.tensor(d["y"]), rtol=3e-7, atol=0)
    assert all(v == 0.0 or abs(v - 1.0 / (1.0 - d["drop_prob"])) < 1e-6 for v in mask.tolist())
    n = rec["normalize"]
    y = OF.normalize_u8(torch.tensor(n["x"], dtype=torch.uint8), n["mean"], n["std"], n["img_num"])
    assert torch.equal(y, torch.tensor(n["y"]))
    e = rec["ema"]
    ema = {k: torch.tensor(v, dtype=torch.int64 if k.endswith("num_batches_tracked") else torch.float32)
           for k, v in e["hist"][0]["model"].items()}
    # ModelEma starts as a copy of the model BEFORE the first in-place change: rebuild that state from step 0
    first = e["hist"][0]
    for k in ema:
        m0 = torch.tensor(first["model"][k], dtype=ema[k].dtype)
        e0 = torch.tensor(first["ema"][k], dtype=ema[k].dtype)
        ema[k] = ((e0.double() - (1 - e["decay"]) * m0.double()) / e["decay"]).to(ema[k].dtype) if ema[k].dtype.is_floating_point else None
    for step in e["hist"]:
        for k in ema:
            if ema[k] is None:
                continue
            mv = torch.tensor(step["model"][k])
            ema[k] = OF.ema_update(ema[k], mv, e["decay"])
            assert torch.allclose(ema[k], torch.tensor(step["ema"][k]), rtol=1e-5, atol=1e-6), k
    # integer buffers: float arithmetic, truncating copy_ (utils.py:339-340)
    a = OF.ema_update(torch.tensor([0], dtype=torch.int64), torch.tensor([7], dtype=torch.int64), 0.9)
    assert int(a) == int(first["ema"]["bn.num_batches_tracked"][0])
