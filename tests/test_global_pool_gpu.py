"""-m gpu: selectable global pooling (max / avgmax / catavgmax) on the H100.

Kernel level: dfd_global_pool against fp64 torch on the same fp32 activations (every type, both 16-bit types, Swish and
none, one-CTA-per-image and chunked batches), exact argmax, ties and NaN under torch's adaptive_max_pool2d rule, chunking
invariance, and the two backward kernels (dfd_gpool_bwd, dfd_act_bwd_gpool with its BatchNorm sums) against fp64
autograd. End to end: the avg columns of catavgmax against the avg model, the graph-replayed Trainer step against the
oracle, the native path against the reference fixtures, bit-identical reruns, classifier dropout at width 2F, and the
runner protocol (train_epoch / validate, ModelEma, checkpoints)."""
import json
import os
import tempfile
from types import SimpleNamespace

import pytest
import torch

from deepfake_detection_b200 import _lib

import gpool_oracle as GO

pytestmark = pytest.mark.gpu

PT = _lib.POOL_TYPES
TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
DT = {"bf16": _lib.DT_BF16, "fp16": _lib.DT_FP16}


def _P(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _unique_max_input(N, hw, C, dtype, seed):
    """y [N, hw, C] in (-2, 2) with one planted maximum per (n, c) at a known row: the max is unique after any monotone map"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = (torch.rand(N, hw, C, device="cuda", generator=g) * 4 - 2)
    am = torch.randint(0, hw, (N, C), device="cuda", generator=g)
    top = 3 + torch.rand(N, C, device="cuda", generator=g)
    y.scatter_(1, am.unsqueeze(1), top.unsqueeze(1))
    return y.to(dtype), am.int()


def _affine(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return 0.5 + torch.rand(C, device="cuda", generator=g), 0.2 * (torch.rand(C, device="cuda", generator=g) - 0.5)


def _act64(y, scale, shift, act):
    u = y.double() if scale is None else (y.float() * scale + shift).double()     # the kernel's fp32 FMA, then fp64
    return u * torch.sigmoid(u) if act == _lib.ACT_SWISH else u


def _pool64(a, pool_type):
    """a [N, hw, C] -> pooled [N, P] (fp64)"""
    avg, mx = a.mean(1), a.max(1).values
    return {"avg": avg, "max": mx, "avgmax": 0.5 * (avg + mx), "catavgmax": torch.cat((avg, mx), 1)}[pool_type]


def _gpool(y, scale, shift, N, hw, C, act, pool_type, dt, max_chunks=8):
    P = 2 * C if pool_type == "catavgmax" else C
    pooled = torch.full((N, P), float("nan"), device="cuda")
    am = torch.full((N, C), -7, dtype=torch.int32, device="cuda")
    _lib.call("dfd_global_pool", _P(y), _P(scale), _P(shift), _P(pooled), _P(am), N, hw, C, act, PT[pool_type], DT[dt],
              max_chunks, _st())
    return pooled, am


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("pool_type", ["avg", "max", "avgmax", "catavgmax"])
def test_global_pool_forward_against_fp64(pool_type, dt):
    seed = 0
    for N in (1, 3, 64, 256):
        for hw in (1, 4, 49, 144, 361):
            if N * hw > 256 * 49:
                continue
            for C in (256, 1280, 1792, 2048):
                seed += 1
                act = _lib.ACT_SWISH if seed % 2 else _lib.ACT_NONE
                y, am_ref = _unique_max_input(N, hw, C, TDT[dt], seed)
                scale, shift = _affine(C, seed) if act == _lib.ACT_SWISH else (None, None)
                pooled, am = _gpool(y, scale, shift, N, hw, C, act, pool_type, dt)
                torch.cuda.synchronize()
                ref = _pool64(_act64(y, scale, shift, act), pool_type)
                case = (N, hw, C, act)
                assert _rel(pooled, ref) < 1e-5, case
                assert torch.equal(am, am_ref), case


def test_global_pool_argmax_ties_and_nan_follow_torch():
    """exact ties -> the first row; a NaN wins and propagates (with several NaNs the last one, as torch's
    `val > max || isnan(val)` scan); the same through the chunked and the per-image launch"""
    N, hw, C = 3, 49, 256
    g = torch.Generator(device="cuda").manual_seed(5)
    y = torch.randint(-3, 4, (N, hw, C), device="cuda", generator=g).float()          # small integers: many exact ties
    y[:, :, :8] = -float("inf")                                                        # all -inf columns -> row 0
    y[0, 10, 9] = float("nan")
    y[1, 3, 17] = float("nan")
    y[1, 40, 17] = float("nan")
    y = y.to(torch.bfloat16)
    x = y.float().permute(0, 2, 1).reshape(N, C, 7, 7)
    mx, idx = torch.nn.functional.adaptive_max_pool2d(x.cpu(), 1, return_indices=True)
    for chunks in (1, 8):
        pooled, am = _gpool(y, None, None, N, hw, C, _lib.ACT_NONE, "max", "bf16", chunks)
        torch.cuda.synchronize()
        assert torch.equal(am.cpu().long(), idx.flatten(1)), chunks
        assert torch.allclose(pooled.cpu(), mx.flatten(1), rtol=0, atol=0, equal_nan=True)
        assert torch.isnan(pooled[0, 9]) and int(am[0, 9]) == 10
        assert torch.isnan(pooled[1, 17]) and int(am[1, 17]) == 40
        assert int(am[2, 0]) == 0 and pooled[2, 0] == -float("inf")


@pytest.mark.parametrize("pool_type", ["max", "avgmax", "catavgmax"])
def test_global_pool_chunking_is_bit_invariant(pool_type):
    """the chunked launch (several CTAs per image) and one CTA per image give the same bits; the mean columns are dfd_pool's
    bits at the same chunking"""
    for N, hw, C in ((1, 361, 512), (3, 49, 1280), (7, 144, 2048)):
        y, _ = _unique_max_input(N, hw, C, torch.bfloat16, 11)
        y[:, 5:9] = y[:, 0:1]                     # a few exact ties across chunk boundaries too
        scale, shift = _affine(C, 3)
        p1, a1 = _gpool(y, scale, shift, N, hw, C, _lib.ACT_SWISH, pool_type, "bf16", 1)
        p8, a8 = _gpool(y, scale, shift, N, hw, C, _lib.ACT_SWISH, pool_type, "bf16", 8)
        pa, _ = _gpool(y, scale, shift, N, hw, C, _lib.ACT_SWISH, "avg", "bf16", 8)
        ref = torch.empty(N, C, device="cuda")
        _lib.call("dfd_pool", _P(y), _P(scale), _P(shift), _P(ref), N, hw, C, _lib.ACT_SWISH, _lib.DT_BF16, None, 8, _st())
        torch.cuda.synchronize()
        assert torch.equal(a1, a8) and torch.equal(pa, ref)
        if pool_type == "catavgmax":
            assert torch.equal(p1[:, C:], p8[:, C:]) and torch.equal(p8[:, :C], ref)
        elif pool_type == "max":
            assert torch.equal(p1, p8)


def _dpooled(N, P, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(N, P, device="cuda", generator=g)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("pool_type", ["max", "avgmax", "catavgmax"])
def test_resnet_gpool_backward_against_autograd(pool_type, dt):
    for N, hw, C in ((2, 49, 2048), (5, 9, 512), (64, 49, 256)):
        y, am = _unique_max_input(N, hw, C, TDT[dt], 21)
        P = 2 * C if pool_type == "catavgmax" else C
        dp = _dpooled(N, P, 4)
        dout = torch.full((N, hw, C), float("nan"), device="cuda", dtype=TDT[dt])
        _lib.call("dfd_gpool_bwd", _P(dp), _P(am), _P(dout), N, hw, C, PT[pool_type], DT[dt], _st())
        x = y.double().requires_grad_(True)
        (_pool64(x, pool_type) * dp.double()).sum().backward()
        torch.cuda.synchronize()
        assert _rel(dout, x.grad) < (4e-3 if dt == "bf16" else 5e-4), (N, hw, C)
        assert torch.equal(dout, x.grad.to(TDT[dt])) or _rel(dout, x.grad.to(TDT[dt])) < 1e-2


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("pool_type", ["max", "avgmax", "catavgmax"])
def test_efficientnet_gpool_backward_against_autograd(pool_type, dt):
    """gu = d/du of <dpooled, pool(swish(u))>, u = scale*y + shift, and the BN backward sums of the stored gu"""
    for N, hw, C in ((4, 49, 1280), (3, 144, 1792), (16, 9, 256)):
        y, am_ref = _unique_max_input(N, hw, C, TDT[dt], 31)
        scale, shift = _affine(C, 8)
        g = torch.Generator(device="cuda").manual_seed(2)
        mean, rstd = 0.1 * torch.randn(C, device="cuda", generator=g), 0.5 + torch.rand(C, device="cuda", generator=g)
        pooled, am = _gpool(y, scale, shift, N, hw, C, _lib.ACT_SWISH, pool_type, dt)
        P = pooled.shape[1]
        dp = _dpooled(N, P, 6)
        gu = torch.full((N, hw, C), float("nan"), device="cuda", dtype=TDT[dt])
        s1 = torch.zeros(8 * C, dtype=torch.float64, device="cuda")
        s2 = torch.zeros(8 * C, dtype=torch.float64, device="cuda")
        _lib.call("dfd_act_bwd_gpool", _P(y), _P(scale), _P(shift), _P(mean), _P(rstd), _P(dp), _P(am), _P(gu), N, hw, C,
                  _lib.ACT_SWISH, PT[pool_type], DT[dt], _P(s1), _P(s2), None, _st())
        u = (y.float() * scale + shift).double().requires_grad_(True)
        (_pool64(u * torch.sigmoid(u), pool_type) * dp.double()).sum().backward()
        torch.cuda.synchronize()
        assert torch.equal(am, am_ref)
        assert _rel(gu, u.grad) < (4e-3 if dt == "bf16" else 5e-4), (N, hw, C)
        g16 = gu.double().reshape(-1, C)
        xhat = ((y.float() - mean) * rstd).double().reshape(-1, C)
        assert _rel(s1.view(8, C).sum(0), g16.sum(0)) < 1e-6
        assert _rel(s2.view(8, C).sum(0), (g16 * xhat).sum(0)) < 1e-6


@pytest.mark.parametrize("arch,N,res", [("efficientnet_b0", 8, 96), ("efficientnet_b0", 300, 64), ("resnet50", 4, 96)])
def test_catavgmax_avg_columns_equal_the_avg_model(arch, N, res):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.engine import Engine
    from oracle.weights import synth_batch, synth_state
    x, _ = synth_batch(N, 3, res, res, seed=77)
    pooled = {}
    for gp in ("avg", "catavgmax"):
        e = Engine(arch, N, res, res, dtype="bf16", global_pool=gp)
        e.load_state_dict(synth_state(get_spec(arch, global_pool=gp), seed=7))
        e.set_input(x.cuda())
        e.zero_step_scratch(_st(), grads=False)
        e.forward(training=True)
        torch.cuda.synchronize()
        pooled[gp] = e.pooled.clone()
        F = e.spec.num_features
    assert pooled["catavgmax"].shape == (N, 2 * F)
    assert torch.equal(pooled["catavgmax"][:, :F], pooled["avg"])


def _tame(spec, sd):
    if spec.family == "resnet":
        for b in spec.blocks:
            k = b.name + (".bn2.weight" if b.kind == "basic" else ".bn3.weight")
            sd[k] = sd[k] * 0.2
    return sd


@pytest.mark.parametrize("gp", ["max", "avgmax", "catavgmax"])
@pytest.mark.parametrize("arch,batch,res,dtype", [("efficientnet_b0", 16, 96, "bf16"), ("efficientnet_b0", 16, 96, "fp16"),
                                                  ("resnet18", 8, 96, "bf16"), ("resnet50", 8, 96, "fp16")])
def test_trainer_graph_step_matches_oracle(arch, batch, res, dtype, gp):
    """three graph-replayed Trainer steps against the oracle's 16-bit emulation, with the tolerances of
    test_head_multiclass_gpu.py::test_trainer_graph_step_matches_oracle. The learning rates are a tenth of that test's: with
    the synthetic weights a max-pooled network's loss jumps several-fold after one step at 0.01 (the reference fixtures show
    it too), and past that point the two implementations' 16-bit roundings, which can move an argmax to another row and
    with it a whole gradient entry, are amplified instead of compared."""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.trainer import Trainer
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    K = 5
    spec = get_spec(arch, num_classes=K, global_pool=gp)
    sd0 = _tame(spec, synth_state(spec, seed=7))
    tr = Trainer(arch, batch, res, res, dtype=dtype, lr=0.001, smoothing=0.1, num_classes=K, use_graph=True, global_pool=gp)
    tr.load_state_dict(sd0)
    sd = {k: v.clone() for k, v in sd0.items()}
    ost = OT.OptState(kind="sgd", lr=0.001, momentum=0.9, weight_decay=1e-4)
    for i, lr in enumerate((0.001, 0.0005, 0.002)):
        for gr in tr.optimizer.param_groups:
            gr["lr"] = lr
        ost.lr = lr
        x, y = synth_batch(batch, 3, res, res, seed=1234 + i, num_classes=K)
        loss, correct = tr.train_step(x.cuda(), y.cuda())
        torch.cuda.synchronize()
        o = GO.train_step(spec, sd, x, y, ost, smoothing=0.1, act_dtype=TDT[dtype])
        lo = float(o["loss"])
        assert abs(float(loss) - lo) < (3e-3 if dtype == "fp16" else 1e-2) * (1 + i) * max(1.0, lo), (i, float(loss), lo)
        assert _rel(tr.engine.logits, o["logits"]) < (2e-2 if dtype == "fp16" else 8e-2) * (1 + i), i
        assert abs(float(correct) * 100.0 / batch - float(o["prec1"])) <= 100.0 / batch + 1e-6
    assert tr.n_captures == 1
    worst = max(_rel(tr.engine.param_view(n), sd[n]) for n, shape, _ in param_entries(spec) if len(shape) > 1)
    # 3e-2 in the avg test; 4.9e-2 measured for ResNet-50 fp16 max, where every channel's gradient enters through one row
    assert worst < 6e-2, worst
    cls = "classifier.weight" if spec.family != "resnet" else "fc.weight"
    assert tuple(sd[cls].shape) == (K, spec.pooled_features)
    assert _rel(tr.engine.param_view(cls), sd[cls]) < 1e-2


@pytest.mark.parametrize("case", ["step_efficientnet_b0_gp_max", "step_efficientnet_b0_k5_gp_catavgmax_ls",
                                  "step_resnet18_gp_avgmax"])
def test_native_against_global_pool_reference_goldens(case, golden_dir):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.optim import ArenaOptimizer
    from oracle.weights import synth_batch, synth_state
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    K, gp = rec["num_classes"], rec["global_pool"]
    spec = get_spec(rec["arch"], num_classes=K, global_pool=gp)
    eng = Engine(rec["arch"], rec["batch"], rec["H"], rec["W"], num_classes=K, dtype="fp16", global_pool=gp)
    eng.load_state_dict(synth_state(spec, seed=rec["weight_seed"]))
    opt = ArenaOptimizer(eng, opt=rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"])
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i, soft=rec["soft"], num_classes=K)
        eng.set_input(x.cuda())
        eng.set_target(y.cuda())
        eng.zero_step_scratch(_st(), grads=True)
        eng.forward(training=True)
        eng.head(True, smoothing=rec["smoothing"], soft=rec["soft"])
        eng.backward()
        opt.step()
        torch.cuda.synchronize()
        # step 0 as test_engine_gpu.py::test_against_reference_goldens; step 1 follows an update whose gradient depends on
        # argmax choices that fp16 storage and the fp32 reference can resolve differently: the loss only, within 8 %
        assert abs(float(eng.loss) - st["loss"]) < (1e-2 if i == 0 else 8e-2) * abs(st["loss"]), (i, float(eng.loss), st["loss"])
        if i == 0:
            s = st["logits"]
            got = eng.logits.flatten().cpu()
            assert _rel(got[torch.tensor(s["idx"])], torch.tensor(s["samples"])) < 7e-2
            assert abs(float(got.double().norm()) - s["norm"]) < 7e-2 * s["norm"]


@pytest.mark.parametrize("arch,N", [("efficientnet_b0", 8), ("resnet18", 4)])
@pytest.mark.parametrize("gp", ["max", "catavgmax"])
def test_global_pool_steps_are_bit_identical(arch, N, gp):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.engine import Engine
    from oracle.weights import synth_batch, synth_state
    import engine_checks as EC
    spec = get_spec(arch, num_classes=2, global_pool=gp)
    sd0 = synth_state(spec, seed=7)
    x, y = synth_batch(N, 3, 96, 96, seed=1234)
    out = []
    for _ in range(2):
        eng = Engine(arch, N, 96, 96, dtype="bf16", global_pool=gp)
        eng.load_state_dict(sd0)
        EC.engine_step(eng, None, x.cuda(), y.cuda())
        out.append((eng.pooled.clone(), eng.pool_argmax.clone(), eng.logits.clone(), eng.grads32.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)


def test_catavgmax_dropout_matches_oracle():
    """classifier dropout acts on the [N, 2F] pooled vector; the oracle applies the engine's mask"""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.optim import ArenaOptimizer
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    import engine_checks as EC
    torch.manual_seed(123)
    spec = get_spec("efficientnet_b0", global_pool="catavgmax")
    sd0 = synth_state(spec, seed=7)
    N = 32
    eng = Engine("efficientnet_b0", N, 96, 96, dtype="fp16", drop_rate=0.35, global_pool="catavgmax")
    eng.load_state_dict(sd0)
    opt = ArenaOptimizer(eng, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    x, y = synth_batch(N, 3, 96, 96, seed=1234)
    EC.engine_step(eng, opt, x.cuda(), y.cuda())
    dmask = eng.dropout_mask.cpu().clone()
    assert dmask.shape == (N, 2 * spec.num_features)
    assert abs(float((dmask > 0).float().mean()) - 0.65) < 0.02
    sd = {k: v.clone() for k, v in sd0.items()}
    out = GO.train_step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4),
                        act_dtype=torch.float16, dropout_mask=dmask)
    assert abs(float(eng.loss) - float(out["loss"])) < 3e-3
    assert _rel(eng.logits, out["logits"]) < 2e-2
    pn = [n for n, _, _ in param_entries(spec)]
    gn = torch.cat([eng.grad_view(n).flatten().cpu() for n in pn])
    go = torch.cat([out["grads"][n].flatten() for n in pn])
    # test_boundary_gpu.py's dropout test holds the avg model to 5e-2; here the max half routes each channel's gradient
    # through one row, and a row the fp16 path ranks differently from the oracle moves that whole entry
    assert _rel(gn, go) < 1.2e-1


class _Loader(list):
    mixup_enabled = False


def _runner_args(**kw):
    d = dict(opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0, mixup_off_epoch=0,
             num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0, log_interval=1, save_images=False,
             recovery_interval=0, tta=0, model="efficientnet_b0")
    d.update(kw)
    return SimpleNamespace(**d)


def test_catavgmax_model_protocol():
    """train_epoch + validate on a catavgmax model; a ModelEma copy keeps the pool type; a [K, 2F] classifier checkpoint
    round-trips and an avg checkpoint is refused"""
    from deepfake_detection_b200 import loss as NL
    from deepfake_detection_b200.ema import ModelEma
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch, validate
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    model = create_model("efficientnet_b0", num_classes=2, dtype="fp16", global_pool="catavgmax")
    spec = model.spec
    sd0 = synth_state(spec, seed=7)
    model.load_state_dict(sd0)
    args = _runner_args(lr=0.001)        # see test_trainer_graph_step_matches_oracle for the learning rate
    opt = create_optimizer(args, model)
    batches = _Loader((x.cuda(), y.cuda()) for x, y in (synth_batch(16, 3, 96, 96, seed=1234 + i) for i in range(2)))
    m = train_epoch(0, model, batches, opt, NL.CrossEntropyLoss(), args)
    v = validate(model, batches, torch.nn.CrossEntropyLoss(), args)
    sd = {k: t.clone() for k, t in sd0.items()}
    ost = OT.OptState(kind="sgd", lr=0.001, momentum=0.9, weight_decay=1e-4)
    losses = [float(GO.train_step(spec, sd, x.cpu(), y.cpu(), ost, act_dtype=torch.float16)["loss"]) for x, y in batches]
    vl = [float(GO.validate_step(spec, sd, x.cpu(), y.cpu(), act_dtype=torch.float16)["loss"]) for x, y in batches]
    assert abs(m["loss"] - sum(losses) / 2) < 2e-3 * sum(losses) / 2, (m, losses)
    assert abs(v["loss"] - sum(vl) / 2) < 5e-3 * sum(vl) / 2, (v, vl)
    ema = ModelEma(model, decay=0.9)
    assert ema.ema.global_pool == "catavgmax" and ema.ema.spec.pooled_features == 2 * spec.num_features
    assert ema.ema.get_classifier().weight.shape == (2, 2 * spec.num_features)
    ema.ema.eval()
    with torch.no_grad():
        assert torch.equal(ema.ema(batches[0][0]), model.eval()(batches[0][0]))
    state = model.state_dict()
    assert tuple(state["classifier.weight"].shape) == (2, 2 * spec.num_features)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ckpt.pth.tar")
        torch.save({"state_dict": state}, path)
        m2 = create_model("efficientnet_b0", num_classes=2, dtype="fp16", global_pool="catavgmax", checkpoint_path=path)
        got = m2.state_dict()
        assert all(torch.equal(got[k].cpu(), state[k].cpu()) for k in state)
        with pytest.raises(Exception):
            create_model("efficientnet_b0", num_classes=2, dtype="fp16", checkpoint_path=path)
