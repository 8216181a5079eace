"""-m gpu: the kernels at the launch shapes of the plans the runner builds besides the shipped training step
(tests/plan_variants.py harvests them on the CPU; tests/test_plan_variants_cpu.py holds the case list to it):
  * every launch of the test_img plan (efficientnet_deepfake_v4, batch 1, fp16, 600 x 600, eval form) at its exact shape;
  * every eval-form variant the training plans lack (the stats-less depthwise forward) in both 16-bit types, the eval
    BatchNorm finalisation at every channel count and the logits-only head at every (N, F) of the eval plans;
  * one case per (kernel, batch class, dtype) of the validation and short-batch plans that no case of
    tests/test_plan_launches_gpu.py runs, at the smallest launch of the class and never at a reduced batch.
The checkers and their tolerances are those of tests/test_plan_launches_gpu.py, unchanged; the two new ones state theirs.
Then end to end: test_img's model at its deployed shape against the oracle, and eval logits that do not depend on the batch.
"""
import os

import pytest
import torch

import plan_variants as PV
from test_plan_launches_gpu import CHECKERS as PLAN_CHECKERS, F32, _gc

pytestmark = pytest.mark.gpu


def _check_head_fwd(kw, dt):
    """the logits-only head of validate / test_img against fp64, test_head_loss's bound"""
    r = _gc().check_head(kw["N"], kw["F"], with_loss=False)
    assert r["nan"] == 0 and r["logits_rel"] < F32 * 5, str(r)


def _check_bn_finalize_eval(kw, dt):
    """the BatchNorm folded from running statistics. rstd within 1 fp32 ulp of fp64 1/sqrt(rv + eps), the bound the kernel's
    Newton step claims (bn_act.cu:176-178); scale within 2 ulp of fp64 gamma * rstd (rstd's ulp plus the product's rounding);
    shift within ulp(beta) + ulp(rm * scale) of fp64 beta - rm * scale, an absolute bound because that subtraction can cancel.
    The running statistics and num_batches_tracked keep every bit."""
    r = _gc().check_bn_finalize_eval(kw["C"])
    assert r["nan"] == 0 and r["mean_exact"] and r["state_kept"], str(r)
    assert r["rstd_ulp"] <= 1.0 and r["scale_ulp"] <= 2.0 and r["shift_ulp"] <= 1.0, str(r)


NEW_CHECKERS = {
    "head_fwd": _check_head_fwd,
    "bn_finalize_eval": _check_bn_finalize_eval,
}
CHECKERS = dict(PLAN_CHECKERS, **NEW_CHECKERS)

_CASES = PV.variant_cases()


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    torch.cuda.empty_cache()        # the GPU is shared: give back what the last case held


@pytest.mark.parametrize("case", _CASES, ids=[c.id for c in _CASES])
def test_plan_variant(case):
    CHECKERS[case.check](case.kw, case.dtype)


# ---- end to end ---------------------------------------------------------------------------------------------------------
def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def test_test_img_logits_at_the_deployed_shape():
    """test_img's plan (batch 1, fp16, 600 x 600, eval) from synthetic weights: its logits, not the softmax score, against the
    oracle's eval forward in fp16 emulation, to the eval bound of the end-to-end parity tests (2e-2 relative)"""
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    torch.set_num_threads(int(os.environ.get("DFD_ORACLE_THREADS", "32")))
    spec = get_spec("efficientnet_deepfake_v4", in_chans=12)
    sd = synth_state(spec, seed=7)
    m = create_model("efficientnet_deepfake_v4", num_classes=2, in_chans=12, dtype="fp16")
    m.load_state_dict(sd)
    m.eval()
    x, y = synth_batch(1, 12, 600, 600, seed=5)
    x16 = x.half()
    with torch.no_grad():
        logits = m(x16.cuda()).float().cpu()
    ev = OT.validate_step(spec, sd, x16.float(), y, act_dtype=torch.float16)
    assert _rel(logits, ev["logits"]) < 2e-2, (logits, ev["logits"])


# eval logits of the same images as one batch and as short batches: (architecture, resolution, dtype, batch)
INVARIANCE = [("efficientnet_b0", 224, "bf16", 256), ("efficientnet_b4", 380, "fp16", 128), ("resnet50", 224, "bf16", 256)]


def _batch_drift(arch, res, dtype, b):
    """per image, |logits(short batch) - logits(batch b)| / |logits(batch b)| for short batches of 1 and 3"""
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from oracle.weights import synth_batch, synth_state
    spec = get_spec(arch)
    m = create_model(arch, num_classes=2, dtype=dtype)
    m.load_state_dict(synth_state(spec, seed=7))
    m.eval()
    x, _ = synth_batch(b, 3, res, res, seed=11)
    x = x.cuda()
    with torch.no_grad():
        full = m(x).float().clone()
        out = []
        for n in (1, 3):
            part = m(x[:n]).float()
            out.append(float(((part - full[:n]).norm(dim=1) / full[:n].norm(dim=1)).max()))
    return max(out)


@pytest.mark.parametrize("arch,res,dtype,b", INVARIANCE, ids=[a for a, *_ in INVARIANCE])
def test_eval_logits_do_not_depend_on_the_batch(arch, res, dtype, b):
    """In eval mode BatchNorm applies running statistics, every GEMM row, depthwise pixel and head row is computed from its own
    image with a K order that does not depend on M, so the batch can change only the order of two fp32 sums: the pools' row
    chunking (592 / n CTAs per image) and, for B4 at odd n, the K blocking of the K = 32 pointwise GEMMs that lose their row
    pack. Such a reordering moves an fp32 sum by ~2^-24 of its size; what survives is the stored 16-bit values whose rounding
    it flips, by one storage ulp each, on a small fraction of the elements, independently and with either sign. So the
    logits move by much less than one storage ulp of their size: the bound is that ulp, 2^-8 for bf16 and 2^-11 for fp16.
    Measured on one H100 80GB HBM3 (400 W power limit), short batches 1 and 3 against the full batch: B0 bf16 4.3e-4,
    B4 fp16 4.6e-5, ResNet-50 0 (its only pool sums ReLU outputs of 16-bit values, which fp32 adds exactly)."""
    drift = _batch_drift(arch, res, dtype, b)
    assert drift < (2.0 ** -8 if dtype == "bf16" else 2.0 ** -11), drift
