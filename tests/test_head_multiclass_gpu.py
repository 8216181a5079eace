"""-m gpu: the K-class classifier head (every class count other than 2: tiled fp32 GEMMs + a per-image log-sum-exp pass).

Kernel level: dfd_head_fwd / dfd_head_bwd against torch in fp64 (logits, loss, dlogits, dW, db, dpooled within 1e-5
relative L2, exact correct count), the accumulate-into contract of dW / db, run-to-run bit identity, the device loss
scale and the out-of-range label.  End to end: the graph-replayed Trainer step against the CPU oracle, the native path
against the K-class reference fixtures, and the default 1000-class create_model through the runner."""
import json
import math
import os
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu


def _P(t):
    return t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _close(a, ref, rtol=1e-5, atol=1e-9):
    """relative L2 distance; `atol` (per element, RMS) only matters for an all-zero reference"""
    a, ref = a.double().flatten(), ref.double().flatten()
    err = float((a - ref).norm())
    return err <= rtol * float(ref.norm()) + atol * max(ref.numel(), 1) ** 0.5, (err, float(ref.norm()))


def _inputs(N, F, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    pooled = torch.randn(N, F, device="cuda", generator=g).abs()          # post-Swish pooled features are mostly >= 0
    W = torch.randn(K, F, device="cuda", generator=g) / math.sqrt(F)
    b = 0.1 * torch.randn(K, device="cuda", generator=g)
    y = torch.randint(0, K, (N,), device="cuda", generator=g)
    tf = torch.softmax(2 * torch.randn(N, K, device="cuda", generator=g), -1)
    return pooled, W, b, y, tf


def _ref(pooled, W, b, y, tf, mode, smoothing):
    """torch fp64: logits, mean loss, dlogits, dW, db, dpooled, correct count"""
    p = pooled.double().requires_grad_(True)
    W64, b64 = W.double().requires_grad_(True), b.double().requires_grad_(True)
    z = torch.nn.functional.linear(p, W64, b64)
    z.retain_grad()
    if mode == "soft":
        loss = torch.nn.functional.cross_entropy(z, tf.double())
        lab = tf.argmax(1)
    else:
        loss = torch.nn.functional.cross_entropy(z, y, label_smoothing=smoothing)
        lab = y
    loss.backward()
    correct = float((z.detach().argmax(1) == lab).sum())
    return dict(logits=z.detach(), loss=float(loss), dlogits=z.grad, dW=W64.grad, db=b64.grad, dpooled=p.grad, correct=correct)


def _native(pooled, W, b, y, tf, mode, smoothing, dW0=None, db0=None, loss_scale=1.0, loss_scale_dev=None):
    from deepfake_detection_b200 import _lib
    N, F = pooled.shape
    K = W.shape[0]
    logits = torch.full((N, K), float("nan"), device="cuda")
    dlog = torch.full((N, K), float("nan"), device="cuda")
    acc = torch.zeros(2, device="cuda")
    soft = mode == "soft"
    _lib.call("dfd_head_fwd", _P(pooled), _P(W), _P(b), _P(logits), N, F, K, None if soft else _P(y), _P(tf) if soft else None,
              smoothing, loss_scale, None if loss_scale_dev is None else _P(loss_scale_dev), _P(acc), _P(acc) + 4, _P(dlog), _st())
    dW = torch.zeros(K, F, device="cuda") if dW0 is None else dW0.clone()
    db = torch.zeros(K, device="cuda") if db0 is None else db0.clone()
    dpooled = torch.full((N, F), float("nan"), device="cuda")
    _lib.call("dfd_head_bwd", _P(dlog), _P(pooled), _P(W), _P(dW), _P(db), _P(dpooled), N, F, K, _st())
    torch.cuda.synchronize()
    return dict(logits=logits, loss=float(acc[0]), correct=float(acc[1]), dlogits=dlog, dW=dW, db=db, dpooled=dpooled)


MODES = (("hard", 0.0), ("smooth", 0.1), ("soft", 0.0))


@pytest.mark.parametrize("N", [1, 7, 64, 256])
@pytest.mark.parametrize("F", [256, 1280, 2048])
@pytest.mark.parametrize("K", [1, 3, 5, 17, 33, 1000, 1001])
def test_head_kernels_match_fp64(K, F, N):
    pooled, W, b, y, tf = _inputs(N, F, K, seed=K * 7919 + F * 31 + N)
    for mode, s in MODES:
        ref = _ref(pooled, W, b, y, tf, mode, s)
        out = _native(pooled, W, b, y, tf, mode, s)
        for k in ("logits", "dlogits", "dW", "db", "dpooled"):
            ok, info = _close(out[k], ref[k])
            assert ok, (mode, k, info)
        assert out["loss"] == pytest.approx(ref["loss"], rel=1e-5, abs=1e-7), mode
        assert out["correct"] == ref["correct"], mode
        # gradients are ADDED to what the arena holds
        dW0 = torch.randn(K, F, device="cuda") * float(ref["dW"].abs().max() + 1e-3)
        db0 = torch.randn(K, device="cuda") * float(ref["db"].abs().max() + 1e-3)
        acc = _native(pooled, W, b, y, tf, mode, s, dW0=dW0, db0=db0)
        assert _close(acc["dW"], dW0.double() + ref["dW"], atol=1e-7)[0], mode
        assert _close(acc["db"], db0.double() + ref["db"], atol=1e-7)[0], mode
        # run to run: bit-identical (no atomics, no split reductions)
        again = _native(pooled, W, b, y, tf, mode, s)
        for k in ("logits", "dlogits", "dW", "db", "dpooled"):
            assert torch.equal(out[k], again[k]), (mode, k)
        assert out["loss"] == again["loss"] and out["correct"] == again["correct"]


@pytest.mark.parametrize("mode,s", MODES)
def test_device_loss_scale_scales_dlogits_only(mode, s):
    N, F, K = 64, 1280, 1000
    pooled, W, b, y, tf = _inputs(N, F, K, seed=3)
    base = _native(pooled, W, b, y, tf, mode, s)
    dev = torch.tensor([1024.0], device="cuda")
    sc = _native(pooled, W, b, y, tf, mode, s, loss_scale=2.0, loss_scale_dev=dev)
    assert torch.equal(sc["logits"], base["logits"]) and sc["loss"] == base["loss"] and sc["correct"] == base["correct"]
    # a power-of-two scale is exact in fp32
    assert torch.equal(sc["dlogits"], base["dlogits"] * 2048.0)


@pytest.mark.parametrize("bad", [-1, 5, 1 << 40])
def test_out_of_range_label_gives_nan_loss_and_zero_row(bad):
    N, F, K = 7, 256, 5
    pooled, W, b, y, tf = _inputs(N, F, K, seed=11)
    y_bad = y.clone()
    y_bad[3] = bad
    out = _native(pooled, W, b, y_bad, tf, "smooth", 0.1)
    ref = _ref(pooled, W, b, y, tf, "smooth", 0.1)        # the same batch with a valid label in row 3
    assert math.isnan(out["loss"])
    assert torch.equal(out["dlogits"][3], torch.zeros(K, device="cuda"))
    keep = [i for i in range(N) if i != 3]
    assert _close(out["dlogits"][keep], ref["dlogits"][keep])[0]
    assert _close(out["logits"], ref["logits"])[0]
    hit3 = float(ref["logits"][3].argmax() == y[3])
    assert out["correct"] == ref["correct"] - hit3


@pytest.mark.parametrize("F,K", [(2048, 32), (1280, 26)])
def test_head_bwd_former_scratch_overrun_shapes(F, K):
    """N = 256 with K * F > 32768: the split-reduction backward this replaced wrote past its scratch here.  Two calls in a
    row accumulate two gradients; a second forward + backward is unaffected by the first."""
    from deepfake_detection_b200 import _lib
    N = 256
    pooled, W, b, y, tf = _inputs(N, F, K, seed=5)
    ref = _ref(pooled, W, b, y, tf, "hard", 0.0)
    dlog = ref["dlogits"].float().contiguous()
    dW, db = torch.zeros(K, F, device="cuda"), torch.zeros(K, device="cuda")
    for call in (1, 2):
        dpooled = torch.zeros(N, F, device="cuda")
        _lib.call("dfd_head_bwd", _P(dlog), _P(pooled), _P(W), _P(dW), _P(db), _P(dpooled), N, F, K, _st())
        torch.cuda.synchronize()
        assert _close(dpooled, ref["dpooled"])[0], call
        assert _close(dW, call * ref["dW"])[0], call
        assert _close(db, call * ref["db"])[0], call
    out = _native(pooled, W, b, y, tf, "hard", 0.0)
    assert _close(out["dW"], ref["dW"])[0] and out["correct"] == ref["correct"]


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def _relerr(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _tame(spec, sd):
    """resnet: damp the residual branches as tests/engine_checks.py does (gamma ~ 1 on every last BN makes a ReLU network's
    16-bit gradients chaotic); both implementations see the same weights"""
    if spec.family == "resnet":
        for b in spec.blocks:
            k = b.name + (".bn2.weight" if b.kind == "basic" else ".bn3.weight")
            sd[k] = sd[k] * 0.2
    return sd


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("arch,batch,res,K,smoothing", [("efficientnet_b0", 16, 96, 5, 0.1), ("efficientnet_b0", 16, 96, 1000, 0.0),
                                                        ("resnet18", 8, 96, 5, 0.1), ("resnet18", 8, 96, 1000, 0.0)])
def test_trainer_graph_step_matches_oracle(arch, batch, res, K, smoothing, dtype):
    """Three graph-replayed Trainer steps (one capture; the learning rate changes between steps) against the oracle's
    emulation of the same 16-bit storage; fp16 runs with dynamic loss scaling."""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.trainer import Trainer
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    spec = get_spec(arch, num_classes=K)
    sd0 = _tame(spec, synth_state(spec, seed=7))
    tr = Trainer(arch, batch, res, res, dtype=dtype, lr=0.01, smoothing=smoothing, num_classes=K, use_graph=True)
    tr.load_state_dict(sd0)
    assert tr.dynamic_scale == (dtype == "fp16")
    sd = {k: v.clone() for k, v in sd0.items()}
    ost = OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    tdt = torch.float16 if dtype == "fp16" else torch.bfloat16
    for i, lr in enumerate((0.01, 0.005, 0.02)):
        for gr in tr.optimizer.param_groups:
            gr["lr"] = lr
        ost.lr = lr
        x, y = synth_batch(batch, 3, res, res, seed=1234 + i, num_classes=K)
        loss, correct = tr.train_step(x.cuda(), y.cuda())
        torch.cuda.synchronize()
        o = OT.train_step(spec, sd, x, y, ost, smoothing=smoothing, act_dtype=tdt)
        lo = float(o["loss"])
        assert abs(float(loss) - lo) < (3e-3 if dtype == "fp16" else 1e-2) * (1 + i) * max(1.0, lo), (i, float(loss), lo)
        # the logits carry the 16-bit storage noise of the whole forward: 6.1e-2 measured for B0 bf16 K = 1000 at step 0
        assert _relerr(tr.engine.logits, o["logits"]) < (2e-2 if dtype == "fp16" else 8e-2) * (1 + i), i
        assert abs(float(correct) * 100.0 / batch - float(o["prec1"])) <= 100.0 / batch + 1e-6
    assert tr.n_captures == 1
    worst = max(_relerr(tr.engine.param_view(n), sd[n]) for n, shape, _ in param_entries(spec) if len(shape) > 1)
    assert worst < 3e-2, worst
    cls = "classifier.weight" if spec.family != "resnet" else "fc.weight"
    assert _relerr(tr.engine.param_view(cls), sd[cls]) < 1e-2


@pytest.mark.parametrize("case", ["step_efficientnet_b0_k5_ls", "step_efficientnet_b0_k5_soft_rmsprop", "step_resnet18_k1000"])
def test_native_against_k_class_reference_goldens(case, golden_dir):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.optim import ArenaOptimizer
    from oracle.weights import synth_batch, synth_state
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    K = rec["num_classes"]
    spec = get_spec(rec["arch"], num_classes=K)
    eng = Engine(rec["arch"], rec["batch"], rec["H"], rec["W"], num_classes=K, dtype="fp16")
    eng.load_state_dict(synth_state(spec, seed=rec["weight_seed"]))
    opt = ArenaOptimizer(eng, opt=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"])
    st_ = _st()
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i, soft=rec["soft"], num_classes=K)
        eng.set_input(x.cuda())
        eng.set_target(y.cuda())
        eng.zero_step_scratch(st_, grads=True)
        eng.forward(training=True)
        eng.head(True, smoothing=rec["smoothing"], soft=rec["soft"])
        eng.backward()
        opt.step()
        torch.cuda.synchronize()
        # the tolerances of test_engine_gpu.py::test_against_reference_goldens: step 0 tight, step 1 on the loss only
        assert abs(float(eng.loss) - st["loss"]) < (1e-2 if i == 0 else 5e-2) * abs(st["loss"]), (i, float(eng.loss), st["loss"])
        if i == 0:      # rel-L2 over the sampled logits (all of them at K = 5) and of the norm
            s = st["logits"]
            got = eng.logits.flatten().cpu()
            assert _relerr(got[torch.tensor(s["idx"])], torch.tensor(s["samples"])) < 7e-2
            assert abs(float(got.double().norm()) - s["norm"]) < 7e-2 * s["norm"]


def _runner_args(**kw):
    d = dict(opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0, mixup_off_epoch=0,
             num_classes=1000, smoothing=0.0, distributed=False, world_size=1, local_rank=0, log_interval=1, save_images=False,
             recovery_interval=0, tta=0, model="efficientnet_b0")
    d.update(kw)
    return SimpleNamespace(**d)


class _Loader(list):
    mixup_enabled = False


def test_default_1000_class_model_trains_and_validates():
    """create_model("efficientnet_b0") keeps the reference's default of 1000 classes; it trains through the fused
    train_epoch and evaluates through validate, matching the oracle's restatement of the same loop."""
    from deepfake_detection_b200 import loss as NL
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch, validate
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    model = create_model("efficientnet_b0", dtype="fp16")
    assert model.num_classes == 1000 and model.spec.num_classes == 1000
    spec = model.spec
    sd0 = synth_state(spec, seed=7)
    model.load_state_dict(sd0)
    args = _runner_args()
    opt = create_optimizer(args, model)
    batches = _Loader((x.cuda(), y.cuda()) for x, y in (synth_batch(16, 3, 96, 96, seed=1234 + i, num_classes=1000) for i in range(2)))
    m = train_epoch(0, model, batches, opt, NL.CrossEntropyLoss(), args)
    v = validate(model, batches, torch.nn.CrossEntropyLoss(), args)
    sd = {k: t.clone() for k, t in sd0.items()}
    ost = OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    losses = [float(OT.train_step(spec, sd, x.cpu(), y.cpu(), ost, act_dtype=torch.float16)["loss"]) for x, y in batches]
    vl = [float(OT.validate_step(spec, sd, x.cpu(), y.cpu(), act_dtype=torch.float16)["loss"]) for x, y in batches]
    assert abs(m["loss"] - sum(losses) / 2) < 2e-3 * sum(losses) / 2, (m, losses)
    assert abs(v["loss"] - sum(vl) / 2) < 5e-3 * sum(vl) / 2, (v, vl)
    got = model.state_dict()
    worst = max(_relerr(got[k], sd[k]) for k in sd if sd[k].dtype.is_floating_point and sd[k].dim() > 1)
    assert worst < 5e-3, worst


def test_fused_and_protocol_paths_agree_at_k5():
    """The fused head (deepfake_detection_b200.loss.LabelSmoothingCrossEntropy) and the protocol path (torch's own loss,
    gradient back through the autograd bridge into dfd_head_bwd) give the same loss and gradients."""
    from deepfake_detection_b200 import loss as NL
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch
    from oracle.weights import synth_batch, synth_state
    spec = get_spec("efficientnet_b0", num_classes=5)
    sd0 = synth_state(spec, seed=7)
    batches = _Loader([tuple(t.cuda() for t in synth_batch(16, 3, 96, 96, seed=1234, num_classes=5))])
    res = {}
    for flavour in ("protocol", "fused"):
        model = create_model("efficientnet_b0", num_classes=5, dtype="bf16")
        model.load_state_dict(sd0)
        args = _runner_args(num_classes=5, smoothing=0.1)
        opt = create_optimizer(args, model)
        tagged = NL.LabelSmoothingCrossEntropy(0.1)

        class Plain(torch.nn.Module):          # the same loss without the tags that select the fused path
            def forward(self, x, t):
                return tagged(x, t)

        m = train_epoch(0, model, batches, opt, Plain() if flavour == "protocol" else tagged, args)
        torch.cuda.synchronize()
        e = model.engine_for(16, 96, 96)
        res[flavour] = (m["loss"], e.dlogits.clone(), model.engine.grads32.clone())
    assert abs(res["protocol"][0] - res["fused"][0]) < 1e-5 * abs(res["fused"][0]), res
    # dL/dlogits: the fused kernel vs torch's autograd of the same loss, both fp32
    assert _relerr(res["protocol"][1], res["fused"][1]) < 1e-5
    # the rest of the backward is the same kernels; the last-bit differences of dL/dlogits pass through bf16 rounding of
    # every stored gradient (1.5e-2 measured over the whole arena)
    assert _relerr(res["protocol"][2], res["fused"][2]) < 3e-2
