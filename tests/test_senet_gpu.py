"""-m gpu: the SE-ResNets on the native path.

  * dfd_maxpool_ceil_fwd / _bwd against F.max_pool2d(3, 2, ceil_mode=True), its indices and its autograd, at even and odd
    extents with forced ties; dfd_pool_se_relu against the SEModule formula in fp64 at every (C, Cse, HW) of seresnet18 / 50,
    batch 1 (chunked) and 64; dfd_relu_se_bwd_reduce + dfd_act_bwd + the BatchNorm backward + dfd_se_fc_wgrad against fp64
    autograd of relu(se(bn(y)) + res); bf16 and fp16;
  * seresnet50 at batch 32, 224x224, from the reference init against the fp32 oracle; fp16 eval at batch 1; max / avgmax
    pooling; the default dropout; checkpoints and two engines bit for bit; the runner's train_epoch with an EMA update.
No test here reads the reference tree: the fixtures under tests/golden/ came from tools/mint_senet_goldens.py.
Their train steps are held by tests/test_reference_steps_gpu.py.
"""
import io
import os
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from deepfake_detection_b200.arch import get_spec

pytestmark = pytest.mark.gpu

TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
DT_CODE = {"bf16": 0, "fp16": 1}
ACT_NONE, ACT_RELU = 0, 2
EPS16 = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _call(name, *args):
    from deepfake_detection_b200 import _lib
    _lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else t.data_ptr()


# ---- ceil-mode stem pool ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("H,W", [(112, 112), (35, 36), (36, 35), (8, 9), (3, 4)])
def test_maxpool_ceil_fwd_bwd(H, W, dtype):
    dt, N, C = TDT[dtype], 3, 64
    g = torch.Generator(device="cuda").manual_seed(H * 100 + W)
    # ReLU output with many exact ties: small integers, zeros included
    x = torch.randint(0, 4, (N, H, W, C), device="cuda", generator=g).to(dt)
    ref, ind = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, ceil_mode=True, return_indices=True)
    Ho, Wo = ref.shape[2:]
    y = torch.full((N, Ho, Wo, C), float("nan"), device="cuda", dtype=dt)
    idx = torch.full((N, Ho, Wo, C), 255, device="cuda", dtype=torch.uint8)
    _call("dfd_maxpool_ceil_fwd", _p(x), _p(y), _p(idx), N, H, W, C, DT_CODE[dtype])
    dy = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dt)
    dx = torch.full_like(x, float("nan"))
    _call("dfd_maxpool_ceil_bwd", _p(dy), _p(idx), _p(dx), N, H, W, C, DT_CODE[dtype])
    torch.cuda.synchronize()
    assert torch.equal(y.float(), ref.permute(0, 2, 3, 1))
    # the arg-max byte (kh * 3 + kw) names torch's flat index: the first maximum in row-major window order
    oy = torch.arange(Ho, device="cuda").view(1, Ho, 1, 1)
    ox = torch.arange(Wo, device="cuda").view(1, 1, Wo, 1)
    flat = (2 * oy + idx.long() // 3) * W + 2 * ox + idx.long() % 3
    assert torch.equal(flat, ind.permute(0, 2, 3, 1))
    x64 = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    F.max_pool2d(x64, 3, 2, ceil_mode=True).backward(dy.permute(0, 3, 1, 2).double())
    gref = x64.grad.permute(0, 2, 3, 1)
    assert float(((dx.double() - gref).abs() - EPS16[dtype] * gref.abs()).max()) <= 1e-6


# ---- squeeze-excite forward ---------------------------------------------------------------------------------------------
_LAYER_HW = {"layer1": 56 * 56, "layer2": 28 * 28, "layer3": 14 * 14, "layer4": 7 * 7}      # at 224x224
SE_SHAPES = sorted({(b.cout, b.cse, _LAYER_HW[b.name.split(".")[0]]) for arch in ("seresnet18", "seresnet50")
                    for b in get_spec(arch).blocks})


def _se_params(C, Cse, g):
    Wr = (torch.randn(Cse, C, device="cuda", generator=g) * (2.0 / C) ** 0.5).float()
    br = (torch.randn(Cse, device="cuda", generator=g) * 0.1).float()
    We = (torch.randn(C, Cse, device="cuda", generator=g) * (2.0 / Cse) ** 0.5).float()
    be = (torch.randn(C, device="cuda", generator=g) * 0.1).float()
    return Wr, br, We, be


def _bn_operands(C, g):
    gamma = 1.0 + 0.2 * torch.randn(C, device="cuda", generator=g)
    beta = 0.2 * torch.randn(C, device="cuda", generator=g)
    return gamma, beta


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("N", [1, 64])
@pytest.mark.parametrize("C,Cse,HW", SE_SHAPES)
def test_pool_se_relu(C, Cse, HW, N, dtype):
    dt = TDT[dtype]
    g = torch.Generator(device="cuda").manual_seed(C * 7 + HW)
    y = torch.randn(N, HW, C, device="cuda", generator=g).to(dt)
    scale, shift = _bn_operands(C, g)
    Wr, br, We, be = _se_params(C, Cse, g)
    for act in (ACT_NONE, ACT_RELU):
        pooled = torch.full((N, C), float("nan"), device="cuda")
        gate = torch.full((N, C), float("nan"), device="cuda")
        _call("dfd_pool_se_relu", _p(y), _p(scale), _p(shift), _p(pooled), _p(Wr), _p(br), _p(We), _p(be), _p(gate), N, HW, C, Cse,
              act, DT_CODE[dtype], 8)
        torch.cuda.synchronize()
        z = y.double() * scale.double() + shift.double()
        if act == ACT_RELU:
            z = z.clamp_min(0)
        p64 = z.mean(1)
        gate64 = torch.sigmoid(F.relu(p64 @ Wr.double().t() + br.double()) @ We.double().t() + be.double())
        assert _rel(pooled, p64) < 1e-5 and float((gate.double() - gate64).abs().max()) < 1e-4, (act, _rel(pooled, p64))


# ---- block tail backward ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("N,HW,C,Cse,act", [(8, 56 * 56, 256, 16, ACT_NONE), (4, 14 * 14, 1024, 64, ACT_NONE),
                                            (2, 7 * 7, 2048, 128, ACT_NONE), (8, 28 * 28, 128, 8, ACT_RELU),
                                            (1, 7 * 7, 512, 32, ACT_RELU)])
def test_se_tail_backward(N, HW, C, Cse, act, dtype):
    """the plan's backward of out = relu(a * se(a) + res), a = act(bn(y)) (batch statistics): dfd_relu_se_bwd_reduce, dfd_act_bwd
    with the gate and dpool, dfd_bn_bwd_finalize / _apply and dfd_se_fc_wgrad, against fp64 autograd"""
    from deepfake_detection_b200 import _lib
    dt, S = TDT[dtype], _lib.lib().stat_slots
    g = torch.Generator(device="cuda").manual_seed(N * C + HW)
    y = torch.randn(N, HW, C, device="cuda", generator=g).to(dt)
    res = torch.randn(N, HW, C, device="cuda", generator=g).to(dt)
    gout = torch.randn(N, HW, C, device="cuda", generator=g).to(dt)
    gamma, beta = _bn_operands(C, g)
    Wr, br, We, be = _se_params(C, Cse, g)
    eps = 1e-5
    y64 = y.double()
    mean = y64.mean((0, 1))
    rstd = 1.0 / torch.sqrt(y64.var((0, 1), unbiased=False) + eps)
    scale = (gamma.double() * rstd).float()
    shift = (beta.double() - mean * gamma.double() * rstd).float()
    mean, rstd = mean.float(), rstd.float()
    pooled, gate = torch.zeros(N, C, device="cuda"), torch.zeros(N, C, device="cuda")
    out = torch.empty_like(y)
    _call("dfd_pool_se_relu", _p(y), _p(scale), _p(shift), _p(pooled), _p(Wr), _p(br), _p(We), _p(be), _p(gate), N, HW, C, Cse,
          act, DT_CODE[dtype], 8)
    _call("dfd_bn_act", _p(y), _p(scale), _p(shift), _p(gate), _p(res), _p(out), N, HW, C, act, 2, DT_CODE[dtype])
    gm, gz, dy = torch.empty_like(y), torch.empty_like(y), torch.empty_like(y)
    draw, d_e, dpool = (torch.zeros(N, C, device="cuda") for _ in range(3))
    r, d_rpre = torch.zeros(N, Cse, device="cuda"), torch.zeros(N, Cse, device="cuda")
    bs1, bs2 = torch.zeros(S, C, dtype=torch.float64, device="cuda"), torch.zeros(S, C, dtype=torch.float64, device="cuda")
    dgamma, dbeta = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    cA, cB, cC = (torch.zeros(C, device="cuda") for _ in range(3))
    dWr, dbr, dWe, dbe = (torch.zeros_like(t) for t in (Wr, br, We, be))
    _call("dfd_relu_se_bwd_reduce", _p(gout), None, _p(y), _p(out), _p(scale), _p(shift), _p(gm), _p(draw), _p(pooled), _p(Wr),
          _p(br), _p(We), _p(be), _p(d_e), _p(r), _p(d_rpre), _p(dpool), N, HW, C, Cse, act, DT_CODE[dtype])
    _call("dfd_act_bwd", _p(gm), _p(y), _p(scale), _p(shift), _p(mean), _p(rstd), _p(gate), _p(dpool), _p(gz), N, HW, C, act,
          DT_CODE[dtype], _p(bs1), _p(bs2), None)
    _call("dfd_bn_bwd_finalize", _p(bs1), _p(bs2), float(N * HW), _p(gamma), _p(mean), _p(rstd), _p(dgamma), _p(dbeta), _p(cA),
          _p(cB), _p(cC), C)
    _call("dfd_bn_bwd_apply", _p(gz), _p(y), None, _p(cA), _p(cB), _p(cC), _p(dy), N, HW, C, DT_CODE[dtype])
    _call("dfd_se_fc_wgrad", _p(d_e), _p(r), _p(d_rpre), _p(pooled), _p(dWr), _p(dbr), _p(dWe), _p(dbe), N, C, Cse)
    torch.cuda.synchronize()
    # fp64 autograd from the same 16-bit inputs
    leaves = [t.double().requires_grad_(True) for t in (y, res, gamma, beta, Wr, br, We, be)]
    y_, res_, gamma_, beta_, Wr_, br_, We_, be_ = leaves
    x = y_.reshape(N * HW, C)
    m = x.mean(0)
    v = ((x - m) ** 2).mean(0)
    a = ((x - m) / torch.sqrt(v + eps) * gamma_ + beta_).reshape(N, HW, C)
    if act == ACT_RELU:
        a = F.relu(a)
    s = torch.sigmoid(F.relu(a.mean(1) @ Wr_.t() + br_) @ We_.t() + be_)
    o = F.relu(a * s[:, None, :] + res_)
    o.backward(gout.double())
    tol = 3e-2 if dtype == "bf16" else 5e-3
    # gm is the gradient of the residual; it is exact up to the mask of the 16-bit output
    assert _rel(gm, res_.grad) < tol, _rel(gm, res_.grad)
    checks = dict(dy=(dy, y_.grad), dgamma=(dgamma, gamma_.grad), dbeta=(dbeta, beta_.grad), dWr=(dWr, Wr_.grad),
                  dbr=(dbr, br_.grad), dWe=(dWe, We_.grad), dbe=(dbe, be_.grad))
    bad = {k: _rel(a_, b_) for k, (a_, b_) in checks.items() if not _rel(a_, b_) < tol}
    assert not bad, bad


# ---- realistic size -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_seresnet50_batch32_224_reference_init(dtype, record_property):
    """seresnet50 at batch 32, 224x224, from the reference's initialisers: loss and updated weights within 1e-2 of the fp32
    oracle, or - where the oracle's own 16-bit emulation is already further than that from fp32 - within 1.5 x that distance
    (yard) + 1e-2. Which statement holds is recorded."""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    from oracle import train as OT
    from oracle.weights import synth_batch
    torch.set_num_threads(int(os.environ.get("DFD_ORACLE_THREADS", "32")))
    spec = get_spec("seresnet50")
    pn = [n for n, _, _ in param_entries(spec)]
    w0 = init_state_dict(spec, seed=11)
    x, y = synth_batch(32, 3, 224, 224, seed=1234)
    ref = {}
    for key, adt in (("fp32", None), ("emul", TDT[dtype])):
        sd = {k: v.clone() for k, v in w0.items()}
        out = OT.train_step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4), act_dtype=adt)
        ref[key] = dict(loss=float(out["loss"]), sd=sd)
    tr = Trainer("seresnet50", 32, 224, 224, dtype=dtype, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, use_graph=False)
    eng = tr.engine
    for _ in range(8):
        tr.load_state_dict(init_state_dict(spec, seed=11))
        tr.train_step(x.cuda(), y.cuda())
        torch.cuda.synchronize()
        if not tr.dynamic_scale or int(eng.flags[1]) == 1:
            break
    else:
        raise AssertionError("no fp16 step was applied")
    fp, em = ref["fp32"], ref["emul"]
    loss_rel = abs(float(eng.loss) - fp["loss"]) / abs(fp["loss"])
    yard_loss = abs(em["loss"] - fp["loss"]) / abs(fp["loss"])
    worst = max((_rel(eng.param_view(n), fp["sd"][n]), n) for n in pn)
    yard_w = max(_rel(em["sd"][n], fp["sd"][n]) for n in pn)
    plain = loss_rel <= 1e-2 and worst[0] <= 1e-2
    record_property("statement", "plain" if plain else "yard")
    print("seresnet50 b32 224 %s: loss_rel %.3e (yard %.3e) worst weight %.3e %s (yard %.3e): %s" %
          (dtype, loss_rel, yard_loss, worst[0], worst[1], yard_w, "<= 1e-2" if plain else "<= 1.5 yard + 1e-2"))
    assert plain or (loss_rel <= 1.5 * yard_loss + 1e-2 and worst[0] <= 1.5 * yard_w + 1e-2), (loss_rel, yard_loss, worst, yard_w)
    del eng, tr
    torch.cuda.empty_cache()


def test_eval_batch1_fp16():
    """the test_img path: eval at batch 1 in fp16 (chunked SE pools) from the reference's initialisers"""
    from oracle import train as OT
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model, init_state_dict
    from oracle.weights import synth_batch
    spec = get_spec("seresnet50")
    sd = init_state_dict(spec, seed=11)
    m = create_model("seresnet50", num_classes=2, dtype="fp16")
    m.load_state_dict(sd)
    m.eval()
    x, y = synth_batch(1, 3, 224, 224, seed=5)
    with torch.no_grad():
        got = m(x.cuda()).cpu()
        again = m(x.cuda()).cpu()
    ref = OT.validate_step(spec, sd, x, y)["logits"]
    emu = OT.validate_step(spec, sd, x, y, act_dtype=torch.float16)["logits"]
    assert torch.equal(got, again)
    assert _rel(got, emu) < 2e-2 and _rel(got, ref) < 1.5 * _rel(emu, ref) + 2e-2, (_rel(got, emu), _rel(got, ref), _rel(emu, ref))


@pytest.mark.parametrize("gp", ["max", "avgmax"])
def test_global_pool_step(gp):
    """--gp max / avgmax: one step of the tamed seresnet18 against the oracle's emulation and fp32"""
    from oracle import train as OT
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.trainer import Trainer
    from oracle.weights import synth_batch, synth_state, tame_state
    spec = get_spec("seresnet18", global_pool=gp)
    sd0 = tame_state(spec, synth_state(spec, seed=7))
    tr = Trainer("seresnet18", 8, 96, 96, dtype="bf16", opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, global_pool=gp)
    tr.engine.load_state_dict(sd0)
    x, y = synth_batch(8, 3, 96, 96, seed=1234)
    tr.train_step(x.cuda(), y.cuda())
    torch.cuda.synchronize()
    e = tr.engine
    pn = [n for n, _, _ in param_entries(spec)]
    em = OT.train_step(spec, {k: v.clone() for k, v in sd0.items()}, x, y, None, act_dtype=torch.bfloat16)
    fp = OT.train_step(spec, {k: v.clone() for k, v in sd0.items()}, x, y, None)
    yard_l = _rel(em["logits"], fp["logits"])
    assert _rel(e.logits, fp["logits"]) < 1.5 * yard_l + 1e-2, (_rel(e.logits, fp["logits"]), yard_l)
    gn = torch.cat([e.grad_view(n).flatten().cpu() for n in pn])
    gf, ge = (torch.cat([o["grads"][n].flatten() for n in pn]) for o in (fp, em))
    assert _rel(gn, gf) < 1.5 * _rel(ge, gf) + 3e-2, (_rel(gn, gf), _rel(ge, gf))


def test_default_dropout_matches_oracle():
    """create_model("seresnet50") trains with SENet's default drop_rate 0.2: the engine draws the mask on the pooled vector, and
    the step matches the oracle fed that mask"""
    from oracle import train as OT
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.models import create_model
    from oracle.weights import synth_batch, synth_state, tame_state
    spec = get_spec("seresnet50")
    sd0 = tame_state(spec, synth_state(spec, seed=7))
    model = create_model("seresnet50", num_classes=2)
    assert model.drop_rate == 0.2
    model.load_state_dict(sd0)
    model.train()
    x, y = synth_batch(8, 3, 96, 96, seed=1234)
    out = model(x.cuda())
    torch.nn.functional.cross_entropy(out, y.cuda()).backward()
    torch.cuda.synchronize()
    e = model.engine_for(8, 96, 96)
    mask = e.dropout_mask.cpu()
    keep = mask != 0
    assert 0 < int((~keep).sum()) < mask.numel() and torch.allclose(mask[keep], torch.full_like(mask[keep], 1 / 0.8))
    pn = [n for n, _, _ in param_entries(spec)]
    em = OT.train_step(spec, {k: v.clone() for k, v in sd0.items()}, x, y, None, act_dtype=torch.bfloat16, dropout_mask=mask)
    fp = OT.train_step(spec, {k: v.clone() for k, v in sd0.items()}, x, y, None, dropout_mask=mask)
    assert _rel(out.detach(), fp["logits"]) < 1.5 * _rel(em["logits"], fp["logits"]) + 1e-2
    gn = torch.cat([e.grad_view(n).flatten().cpu() for n in pn])
    gf, ge = (torch.cat([o["grads"][n].flatten() for n in pn]) for o in (fp, em))
    assert _rel(gn, gf) < 1.5 * _rel(ge, gf) + 3e-2, (_rel(gn, gf), _rel(ge, gf))


# ---- checkpoints and determinism -------------------------------------------------------------------------------------------
def test_checkpoint_round_trip_is_bit_exact():
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from oracle.weights import synth_batch, synth_state
    sd0 = synth_state(get_spec("seresnet50", num_classes=2), seed=3)
    m1 = create_model("seresnet50", num_classes=2)
    m1.load_state_dict(sd0)
    m1.eval()
    x, _ = synth_batch(4, 3, 96, 112, seed=77)
    with torch.no_grad():
        l1 = m1(x.cuda())
    buf = io.BytesIO()
    torch.save(m1.state_dict(), buf)
    buf.seek(0)
    sd = torch.load(buf)
    assert list(sd) == list(sd0) and all(torch.equal(sd[k].cpu(), sd0[k]) for k in sd0)
    m2 = create_model("seresnet50", num_classes=2)
    m2.load_state_dict(sd)
    m2.eval()
    with torch.no_grad():
        l2 = m2(x.cuda())
    assert torch.equal(l1, l2)


@pytest.mark.parametrize("arch,batch", [("seresnet50", 8), ("seresnet18", 2)])
def test_two_engines_agree_bit_for_bit(arch, batch):
    """batch 2: the SE pools and the tail backward split each image over several CTAs (fixed-slot partials)"""
    from deepfake_detection_b200.arch import get_spec
    from oracle.weights import synth_state
    from engine_checks import trainer_steps
    sd0 = synth_state(get_spec(arch), seed=7)
    runs = [trainer_steps(arch, batch, 96, 96, "bf16", 2, sd0)[1] for _ in range(2)]
    for a, b in zip(*runs):
        assert a["loss"] == b["loss"]
        assert torch.equal(a["logits"], b["logits"]) and torch.equal(a["grads"], b["grads"]) and torch.equal(a["params"], b["params"])


def test_runner_train_epoch_with_ema():
    """train_epoch's loop body over create_model("seresnet50", drop_rate=0.0) for two steps, against the oracle's two steps
    (tamed synthetic weights); then one EMA update"""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.ema import ModelEma
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state, tame_state

    class _Loader(list):
        mixup_enabled = False

    args = SimpleNamespace(opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0,
                           mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0,
                           log_interval=1, save_images=False, recovery_interval=0, tta=0, model="seresnet50")
    spec = get_spec("seresnet50")
    sd0 = tame_state(spec, synth_state(spec, seed=7))
    model = create_model("seresnet50", num_classes=2, drop_rate=0.0)
    model.load_state_dict(sd0)
    opt = create_optimizer(args, model)
    ema = ModelEma(model, decay=0.9)
    data = [synth_batch(16, 3, 96, 96, seed=1234 + i) for i in range(2)]
    m = train_epoch(0, model, _Loader((x.cuda(), y.cuda()) for x, y in data), opt, torch.nn.CrossEntropyLoss(), args,
                    model_ema=ema)
    pn = [n for n, _, _ in param_entries(spec)]
    res = {}
    for key, adt in (("emul", torch.bfloat16), ("fp32", None)):
        sd = {k: v.clone() for k, v in sd0.items()}
        ost = OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
        losses = [float(OT.train_step(spec, sd, x, y, ost, act_dtype=adt)["loss"]) for x, y in data]
        res[key] = (sum(losses) / 2, torch.cat([(sd[n] - sd0[n]).flatten() for n in pn]))
    got = model.state_dict()
    dn = torch.cat([(got[n].cpu() - sd0[n]).flatten() for n in pn])
    assert abs(m["loss"] - res["fp32"][0]) < 2e-2 * max(1.0, res["fp32"][0]), (m, res["fp32"][0], res["emul"][0])
    yard = _rel(res["emul"][1], res["fp32"][1])
    assert _rel(dn, res["fp32"][1]) < 1.5 * yard + 3e-2, (_rel(dn, res["fp32"][1]), yard)
    e = ema.ema.state_dict()
    k = "layer4.2.se_module.fc1.weight"
    assert not torch.equal(e[k].cpu(), sd0[k]) and not torch.equal(e[k].cpu(), got[k].cpu())
