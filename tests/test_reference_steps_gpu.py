"""-m gpu: the native path against the reference-minted step fixtures, one run per row of tests/reference_steps.py's GPU_STEPS
and dtype. Each statement's measured quantities are recorded (record_property).

  * kind "engine": Engine + ArenaOptimizer steps from the fixture's synthetic weights. Batch 4 at 64x64 with lr 0.01 is a
    chaotic regime for 16-bit storage (the oracle's own bf16 emulation moves the step-1 logits by ~0.4 relative): the
    fixture pins step 0 tightly (loss within 1e-2, logits within 7e-2) and later steps on the loss only;
  * kind "tamed": Trainer steps from a fixture whose residual branches are damped (oracle.weights.tame_state), so 16-bit
    storage stays a small perturbation. Step 0's logits and loss against the oracle's 16-bit emulation, its logits and
    gradients against the fp32 oracle within 1.5 x the emulation's own distance + a margin, every step's loss against the
    reference, the step-0 logits against the reference's samples. resnet101 in bf16 is the one case where the emulation
    itself moves the logits by more than the emulation bound (7.4e-2): there that bound is 1.5 x the emulation's distance."""
import pytest
import torch

import engine_checks as EC
import reference_steps as RS
from deepfake_detection_b200.arch import get_spec, param_entries
from deepfake_detection_b200.engine import Engine
from deepfake_detection_b200.optim import ArenaOptimizer
from oracle import train as OT
from oracle.weights import synth_batch, synth_state, tame_state

pytestmark = pytest.mark.gpu

TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
CASES = [(case, over, dtype) for case, over in RS.GPU_STEPS for dtype in over["dtypes"]]


@pytest.mark.parametrize("case,over,dtype", CASES, ids=["%s-%s" % (c, d) for c, _, d in CASES])
def test_native_matches_reference_steps(case, over, dtype, golden_dir, record_property):
    rec = RS.load(golden_dir, case)
    (_engine_steps if over["kind"] == "engine" else _tamed_steps)(rec, over, dtype, record_property)


def _engine_steps(rec, over, dtype, record_property):
    K, gp = rec.get("num_classes", 2), rec.get("global_pool", "avg")
    spec = get_spec(rec["arch"], num_classes=K, global_pool=gp)
    eng = Engine(rec["arch"], rec["batch"], rec["H"], rec["W"], num_classes=K, dtype=dtype, global_pool=gp)
    eng.load_state_dict(synth_state(spec, seed=rec["weight_seed"]))
    opt = ArenaOptimizer(eng, opt=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"])
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i, soft=rec["soft"], num_classes=K)
        EC.engine_step(eng, opt, x.cuda(), y.cuda(), rec["smoothing"])
        loss = float(eng.loss)
        record_property("loss_%d" % i, loss)
        tol = 1e-2 if i == 0 else over.get("loss_after", 5e-2)
        assert abs(loss - st["loss"]) < tol * abs(st["loss"]), (i, loss, st["loss"])
        if i == 0:
            s = st["logits"]
            got = eng.logits.flatten().cpu()
            if isinstance(s, list):
                err = EC.relerr(got, torch.tensor(s))
            else:
                err = EC.relerr(got[torch.tensor(s["idx"])], torch.tensor(s["samples"]))
            record_property("logits_rel_0", err)
            assert err < 7e-2, err
            if over.get("norm"):
                norm_err = abs(float(got.double().norm()) - s["norm"])
                record_property("logits_norm_abs_0", norm_err)
                assert norm_err < 7e-2 * s["norm"], (norm_err, s["norm"])
    if over.get("step_count"):
        assert opt.step_count == len(rec["steps"])


def _tamed_steps(rec, over, dtype, record_property):
    arch, batch, H, W = rec["arch"], rec["batch"], rec["H"], rec["W"]
    spec = get_spec(arch)
    sd0 = tame_state(spec, synth_state(spec, seed=rec["weight_seed"]), rec["tame"])
    tr, runs = EC.trainer_steps(arch, batch, H, W, dtype, len(rec["steps"]), sd0)
    sd = {k: v.clone() for k, v in sd0.items()}
    ost = OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    e = tr.engine
    for i, (r, st) in enumerate(zip(runs, rec["steps"])):
        x, y = synth_batch(batch, 3, H, W, seed=1234 + i)
        o = OT.train_step(spec, sd, x, y, ost, act_dtype=TDT[dtype])
        record_property("loss_%d" % i, r["loss"])
        if i == 0:
            o32 = OT.train_step(spec, {k: v.clone() for k, v in sd0.items()}, x, y, None)
            yard_logits = EC.relerr(o["logits"], o32["logits"])
            emul_logits, fp32_logits = EC.relerr(r["logits"], o["logits"]), EC.relerr(r["logits"], o32["logits"])
            bound = max(2e-2 if dtype == "fp16" else 6e-2, 1.5 * yard_logits)
            assert emul_logits < bound, (emul_logits, yard_logits)
            assert abs(r["loss"] - float(o["loss"])) < 5e-3, (r["loss"], float(o["loss"]))
            assert fp32_logits < 1.5 * yard_logits + 1e-2, (fp32_logits, yard_logits)
            names = [n for n, _, _ in param_entries(spec)]
            gn = torch.cat([r["grads"][e.p_off[n][0]:e.p_off[n][0] + e.p_off[n][2]] for n in names]) / r["scale"]
            go, g32 = (torch.cat([oo["grads"][n].flatten() for n in names]) for oo in (o, o32))
            yard = EC.relerr(go, g32)
            grads = EC.relerr(gn, g32)
            assert grads < 1.5 * yard + 3e-2, (grads, yard)
            f = r["logits"].double().flatten()
            ref = torch.tensor(st["logits"]["samples"], dtype=torch.float64)
            got = f[torch.tensor(st["logits"]["idx"])]
            samples = float((got - ref).norm() / ref.norm())
            assert samples < 1.5 * yard_logits + 2e-2, (got, ref)
            for k, v in dict(emul_loss_0=float(o["loss"]), yard_logits_0=yard_logits, emul_logits_rel_0=emul_logits,
                             fp32_logits_rel_0=fp32_logits, yard_grads_0=yard, grads_rel_0=grads, samples_rel_0=samples).items():
                record_property(k, v)
        assert abs(r["loss"] - st["loss"]) < (1e-2 if i == 0 else 5e-2) * abs(st["loss"]), (i, r["loss"], st["loss"])
