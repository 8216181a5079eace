"""-m gpu: Xception on the native path.

  * the depthwise forward with a ReLU input (after a BN or alone) and the fused depthwise backward in its two ReLU modes
    against fp64 torch at Xception's shapes; the strided block tail (dfd_bn_maxpool_add) and its backward
    (dfd_maxpool_bn_bwd_reduce) against F.max_pool2d and its indices, with negative inputs and forced ties;
  * batch 32 at 299x299 from the reference init against the fp32 oracle; eval at batch 1 in fp16 (the test_img path);
  * drop_rate changes no bit; checkpoints round-trip bit for bit and two engines agree bit for bit; the runner's train_epoch
    with SGD and RMSpropTF and an EMA update.
No test here reads the reference tree: the fixtures under tests/golden/ came from tools/mint_xception_goldens.py.
Their train steps are held by tests/test_reference_steps_gpu.py.
"""
import io
import os
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
DT_CODE = {"bf16": 0, "fp16": 1}
DW_SHAPES = [(147, 64), (147, 128), (74, 128), (74, 256), (37, 256), (37, 728), (19, 728), (10, 1024), (10, 1536)]
POOL_SHAPES = [(147, 128), (74, 256), (37, 728), (19, 1024), (15, 64), (8, 256)]     # + 15 -> 8 -> 4: odd extents
ACT_RELU = 2


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _call(name, *args):
    from deepfake_detection_b200 import _lib
    _lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else t.data_ptr()


def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


# ---- depthwise kernels ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("bn", [True, False], ids=["bn_relu", "relu"])
@pytest.mark.parametrize("H,C", DW_SHAPES)
def test_dwconv_relu_fwd_bwd(H, C, bn, dtype):
    from deepfake_detection_b200 import _lib
    dt, N, W = TDT[dtype], 2, H
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(H * 10000 + C + bn)
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dt)
    w = (torch.randn(C, 9, device="cuda", generator=g) / 3).contiguous()
    scale = (torch.rand(C, device="cuda", generator=g) + 0.5) if bn else None
    shift = (torch.randn(C, device="cuda", generator=g) * 0.5) if bn else None
    mean = torch.randn(C, device="cuda", generator=g) * 0.1
    rstd = torch.rand(C, device="cuda", generator=g) + 0.5
    gy = torch.randn(N, H, W, C, device="cuda", generator=g).to(dt)
    add = None if bn else torch.randn(N, H, W, C, device="cuda", generator=g).to(dt)
    out = torch.full_like(x, float("nan"))
    _call("dfd_dwconv_fwd", x.data_ptr(), _p(scale), _p(shift), w.data_ptr(), out.data_ptr(), N, H, W, C, 3, 1, ACT_RELU,
          DT_CODE[dtype], None, None, None)
    S = L.stat_slots
    s1 = torch.zeros(S * C, dtype=torch.float64, device="cuda")
    s2 = torch.zeros(S * C, dtype=torch.float64, device="cuda")
    dW = torch.zeros(C, 9, device="cuda")
    gx = torch.full_like(x, float("nan"))
    _call("dfd_dwconv_bwd_relu", gy.data_ptr(), None, None, None, None, w.data_ptr(), x.data_ptr(), _p(scale), _p(shift),
          _p(mean) if bn else None, _p(rstd) if bn else None, _p(add), gx.data_ptr(), dW.data_ptr(), N, H, W, C, 3, 1,
          DT_CODE[dtype], _p(s1) if bn else None, _p(s2) if bn else None, None, 0, None)
    torch.cuda.synchronize()
    # fp64 reference over the staged 16-bit input a = round16(relu(scale*x + shift)) / relu(x)
    xf = x.float()
    a = (torch.relu(torch.addcmul(shift, xf, scale)) if bn else torch.relu(xf)).to(dt)
    a64, w64 = _nchw(a), w.view(C, 1, 3, 3).double()
    ref = F.conv2d(a64, w64, padding=1, groups=C).permute(0, 2, 3, 1)
    tol = 8e-3 if dtype == "bf16" else 1e-3
    assert _rel(out, ref) < tol, _rel(out, ref)
    gy64 = _nchw(gy)
    ga = torch.nn.grad.conv2d_input(a64.shape, w64, gy64, padding=1, groups=C).permute(0, 2, 3, 1)
    mask = (a.double() > 0).double()
    gref = ga * mask + (0 if add is None else add.double())
    assert _rel(gx, gref) < tol, _rel(gx, gref)
    assert bool(((gx.double() != 0) <= (mask > 0) if bn else torch.ones((), dtype=torch.bool, device="cuda")).all())
    dwref = torch.nn.grad.conv2d_weight(a64, w64.shape, gy64, padding=1, groups=C).view(C, 9)
    assert _rel(dW, dwref) < tol, _rel(dW, dwref)
    if bn:
        g16 = gx.double()
        xh = (x.double() - mean.double()) * rstd.double()
        assert _rel(s1.view(S, C).sum(0), g16.sum((0, 1, 2))) < 1e-5
        assert _rel(s2.view(S, C).sum(0), (g16 * xh).sum((0, 1, 2))) < 1e-5


# ---- strided block tail --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("H,C", POOL_SHAPES)
def test_bn_maxpool_add_and_backward(H, C, dtype):
    from deepfake_detection_b200 import _lib
    dt, N, W = TDT[dtype], 2, H + 1 if H % 2 else H - 1        # one odd and one even extent
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    g = torch.Generator(device="cuda").manual_seed(H * 7 + C)
    # quarter steps in [-4, 4]: many exact ties in every window; power-of-two scales of both signs keep scale*y + shift exact
    y = (torch.randint(-16, 17, (N, H, W, C), device="cuda", generator=g).float() / 4).to(dt)
    pick = lambda: torch.tensor([0.5, 1.0, 2.0, -1.0], device="cuda")[torch.randint(0, 4, (C,), device="cuda", generator=g)]
    scale, scale_s = pick(), pick()
    shift = torch.randint(-8, 9, (C,), device="cuda", generator=g).float() / 4
    shift_s = torch.randint(-8, 9, (C,), device="cuda", generator=g).float() / 4
    ys = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dt)
    out = torch.full((N, Ho, Wo, C), float("nan"), device="cuda", dtype=dt)
    idx = torch.full((N, Ho, Wo, C), 255, device="cuda", dtype=torch.uint8)
    _call("dfd_bn_maxpool_add", y.data_ptr(), scale.data_ptr(), shift.data_ptr(), ys.data_ptr(), scale_s.data_ptr(),
          shift_s.data_ptr(), out.data_ptr(), idx.data_ptr(), N, H, W, C, DT_CODE[dtype])
    u = (y.float() * scale + shift).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    pooled, ind = F.max_pool2d(u, 3, 2, 1, return_indices=True)
    ref = (pooled.detach().permute(0, 2, 3, 1) + (ys.float() * scale_s + shift_s)).to(dt)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    iy, ix = (ind // W).permute(0, 2, 3, 1), (ind % W).permute(0, 2, 3, 1)
    oy = torch.arange(Ho, device="cuda").view(1, Ho, 1, 1)
    ox = torch.arange(Wo, device="cuda").view(1, 1, Wo, 1)
    tap = (iy - (2 * oy - 1)) * 3 + (ix - (2 * ox - 1))
    assert torch.equal(idx.long(), tap)
    # eval mode: no arg-max, same output
    out2 = torch.full_like(out, float("nan"))
    _call("dfd_bn_maxpool_add", y.data_ptr(), scale.data_ptr(), shift.data_ptr(), ys.data_ptr(), scale_s.data_ptr(),
          shift_s.data_ptr(), out2.data_ptr(), None, N, H, W, C, DT_CODE[dtype])
    # backward through the pool + the BN-backward sums
    gy = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dt)
    mean = torch.randn(C, device="cuda", generator=g) * 0.1
    rstd = torch.rand(C, device="cuda", generator=g) + 0.5
    S = _lib.lib().stat_slots
    s1 = torch.zeros(S * C, dtype=torch.float64, device="cuda")
    s2 = torch.zeros(S * C, dtype=torch.float64, device="cuda")
    gx = torch.full_like(y, float("nan"))
    _call("dfd_maxpool_bn_bwd_reduce", gy.data_ptr(), idx.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
          gx.data_ptr(), N, H, W, C, DT_CODE[dtype], s1.data_ptr(), s2.data_ptr())
    pooled.backward(gy.float().permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    assert torch.equal(out2, out)
    gref = u.grad.permute(0, 2, 3, 1)
    eps = 2.0 ** -8 if dtype == "bf16" else 2.0 ** -11
    assert float(((gx.double() - gref.double()).abs() - eps * gref.double().abs()).max()) <= 1e-6
    g16 = gx.double()
    xh = (y.double() - mean.double()) * rstd.double()
    assert _rel(s1.view(S, C).sum(0), g16.sum((0, 1, 2))) < 1e-5
    assert _rel(s2.view(S, C).sum(0), (g16 * xh).sum((0, 1, 2))) < 1e-5


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_act_bwd_gpool_relu(dtype):
    """dfd_act_bwd_gpool with ACT_RELU (Xception's head under max / avgmax / catavgmax) against fp64 autograd"""
    from deepfake_detection_b200 import _lib
    dt, N, hw, C = TDT[dtype], 3, 100, 2048
    g = torch.Generator(device="cuda").manual_seed(3)
    y = torch.randn(N, hw, C, device="cuda", generator=g).to(dt)
    scale, shift = torch.rand(C, device="cuda", generator=g) + 0.5, torch.randn(C, device="cuda", generator=g) * 0.3
    mean, rstd = torch.randn(C, device="cuda", generator=g) * 0.1, torch.rand(C, device="cuda", generator=g) + 0.5
    S = _lib.lib().stat_slots
    for pool in ("max", "avgmax", "catavgmax"):
        pt = _lib.POOL_TYPES[pool]
        P = 2 * C if pool == "catavgmax" else C
        pooled = torch.zeros(N, P, device="cuda")
        am = torch.zeros(N, C, dtype=torch.int32, device="cuda")
        _call("dfd_global_pool", y.data_ptr(), scale.data_ptr(), shift.data_ptr(), pooled.data_ptr(), am.data_ptr(), N, hw, C,
              ACT_RELU, pt, DT_CODE[dtype], 8)
        dp = torch.randn(N, P, device="cuda", generator=g)
        gu = torch.full_like(y, float("nan"))
        s1 = torch.zeros(S * C, dtype=torch.float64, device="cuda")
        s2 = torch.zeros(S * C, dtype=torch.float64, device="cuda")
        _call("dfd_act_bwd_gpool", y.data_ptr(), scale.data_ptr(), shift.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
              dp.data_ptr(), am.data_ptr(), gu.data_ptr(), N, hw, C, ACT_RELU, pt, DT_CODE[dtype], s1.data_ptr(),
              s2.data_ptr(), None)
        torch.cuda.synchronize()
        u = (y.double() * scale.double() + shift.double()).requires_grad_(True)
        a = torch.relu(u)
        mx, av = a.max(1).values, a.mean(1)
        o = {"max": mx, "avgmax": 0.5 * (mx + av), "catavgmax": torch.cat([av, mx], 1)}[pool]
        (o * dp.double()).sum().backward()
        tol = 8e-3 if dtype == "bf16" else 1e-3
        assert _rel(gu, u.grad) < tol, (pool, _rel(gu, u.grad))
        assert _rel(s1.view(S, C).sum(0), gu.double().sum((0, 1))) < 1e-5


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_batch32_299_reference_init(dtype):
    """loss and updated weights within 1e-2 of the fp32 oracle from the reference's initialisers (batch 32, 299x299)"""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    from oracle import train as OT
    from oracle.weights import synth_batch
    torch.set_num_threads(int(os.environ.get("DFD_ORACLE_THREADS", "32")))
    spec = get_spec("xception")
    key = "_xception_oracle"
    if key not in globals():
        sd = {k: v.clone() for k, v in init_state_dict(spec, seed=11).items()}
        x, y = synth_batch(32, 3, 299, 299, seed=1234)
        out = OT.train_step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4))
        globals()[key] = dict(sd=sd, x=x, y=y, logits=out["logits"], loss=float(out["loss"]))
    o = globals()[key]
    pn = [n for n, _, _ in param_entries(spec)]
    tr = Trainer("xception", 32, 299, 299, dtype=dtype, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, use_graph=False)
    eng = tr.engine
    for _ in range(8):
        tr.load_state_dict(init_state_dict(spec, seed=11))
        tr.train_step(o["x"].cuda(), o["y"].cuda())
        torch.cuda.synchronize()
        if not tr.dynamic_scale or int(eng.flags[1]) == 1:
            break
    else:
        raise AssertionError("no fp16 step was applied")
    # tensors that start at zero (the BN biases) are left out of the worst-tensor statement, as in
    # tests/test_resnet_family_gpu.py::test_batch32_224_reference_init: after one step they hold -lr * their gradient, a
    # per-channel sum that the BatchNorms downstream nearly cancel
    w0 = init_state_dict(spec, seed=11)
    live = [n for n in pn if float(w0[n].abs().max()) > 0]
    worst = max((_rel(eng.param_view(n), o["sd"][n]), n) for n in live)
    glob = _rel(torch.cat([eng.param_view(n).flatten().cpu() for n in pn]), torch.cat([o["sd"][n].flatten() for n in pn]))
    loss_rel = abs(float(eng.loss) - o["loss"]) / abs(o["loss"])
    assert loss_rel < 1e-2 and worst[0] < 1e-2 and glob < 1e-2, (loss_rel, worst, glob)
    del eng, tr
    torch.cuda.empty_cache()


def test_eval_batch1_fp16_299():
    """the test_img path: eval at batch 1 in fp16 from the reference's initialisers, against the fp32 oracle and its fp16
    emulation (the synthetic weights of oracle/weights.py grow the activations beyond the fp16 range at 299x299)"""
    from oracle import train as OT
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model, init_state_dict
    from oracle.weights import synth_batch
    spec = get_spec("xception")
    sd = init_state_dict(spec, seed=11)
    m = create_model("xception", num_classes=2, dtype="fp16")
    m.load_state_dict(sd)
    m.eval()
    x, y = synth_batch(1, 3, 299, 299, seed=5)
    with torch.no_grad():
        got = m(x.cuda()).cpu()
        again = m(x.cuda()).cpu()
    ref = OT.validate_step(spec, sd, x, y)["logits"]
    emu = OT.validate_step(spec, sd, x, y, act_dtype=torch.float16)["logits"]
    assert torch.equal(got, again)
    assert _rel(got, emu) < 2e-2 and _rel(got, ref) < 1.5 * _rel(emu, ref) + 2e-2, (_rel(got, emu), _rel(got, ref), _rel(emu, ref))


def test_drop_rate_changes_nothing():
    from deepfake_detection_b200.arch import get_spec
    from engine_checks import trainer_steps
    from oracle.weights import synth_state
    sd0 = synth_state(get_spec("xception"), seed=7)
    a = trainer_steps("xception", 4, 64, 80, "bf16", 2, sd0)[1]
    b = trainer_steps("xception", 4, 64, 80, "bf16", 2, sd0, drop_rate=0.5)[1]
    for ra, rb in zip(a, b):
        assert ra["loss"] == rb["loss"] and torch.equal(ra["logits"], rb["logits"]) and torch.equal(ra["params"], rb["params"])


def test_two_engines_agree_bit_for_bit():
    from deepfake_detection_b200.arch import get_spec
    from engine_checks import trainer_steps
    from oracle.weights import synth_state
    sd0 = synth_state(get_spec("xception"), seed=7)
    runs = [trainer_steps("xception", 8, 96, 96, "bf16", 2, sd0)[1] for _ in range(2)]
    for a, b in zip(*runs):
        assert a["loss"] == b["loss"]
        assert torch.equal(a["logits"], b["logits"]) and torch.equal(a["grads"], b["grads"]) and torch.equal(a["params"], b["params"])


def test_checkpoint_round_trip_is_bit_exact():
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from oracle.weights import synth_batch, synth_state
    sd0 = synth_state(get_spec("xception", num_classes=2), seed=3)
    m1 = create_model("xception", num_classes=2)
    m1.load_state_dict(sd0)
    m1.eval()
    x, _ = synth_batch(2, 3, 96, 112, seed=77)
    with torch.no_grad():
        l1 = m1(x.cuda())
    buf = io.BytesIO()
    torch.save(m1.state_dict(), buf)
    buf.seek(0)
    sd = torch.load(buf)
    assert list(sd) == list(sd0) and all(torch.equal(sd[k].cpu(), sd0[k]) for k in sd0)
    m2 = create_model("xception", num_classes=2)
    m2.load_state_dict(sd)
    m2.eval()
    with torch.no_grad():
        l2 = m2(x.cuda())
    assert torch.equal(l1, l2)


@pytest.mark.parametrize("opt_name", ["sgd", "rmsproptf"])
def test_runner_train_epoch_with_ema(opt_name):
    """train_epoch's loop body over create_model("xception") for two steps, against the oracle's two steps (tamed synthetic
    weights); then one EMA update"""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.ema import ModelEma
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state, tame_state

    class _Loader(list):
        mixup_enabled = False

    lr = 0.01 if opt_name == "sgd" else 1e-3
    args = SimpleNamespace(opt=opt_name, lr=lr, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8 if opt_name == "sgd" else 1e-3,
                           prefetcher=True, mixup=0.0, mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False,
                           world_size=1, local_rank=0, log_interval=1, save_images=False, recovery_interval=0, tta=0,
                           model="xception")
    spec = get_spec("xception")
    sd0 = tame_state(spec, synth_state(spec, seed=7))
    model = create_model("xception", num_classes=2)
    model.load_state_dict(sd0)
    opt = create_optimizer(args, model)
    ema = ModelEma(model, decay=0.9)
    data = [synth_batch(8, 3, 96, 96, seed=1234 + i) for i in range(2)]
    m = train_epoch(0, model, _Loader((x.cuda(), y.cuda()) for x, y in data), opt, torch.nn.CrossEntropyLoss(), args,
                    model_ema=ema)
    pn = [n for n, _, _ in param_entries(spec)]
    res = {}
    for key, adt in (("emul", torch.bfloat16), ("fp32", None)):
        sd = {k: v.clone() for k, v in sd0.items()}
        ost = OT.OptState(kind=opt_name, lr=lr, momentum=0.9, weight_decay=1e-4, eps=args.opt_eps)
        losses = [float(OT.train_step(spec, sd, x, y, ost, act_dtype=adt)["loss"]) for x, y in data]
        res[key] = (sum(losses) / 2, torch.cat([(sd[n] - sd0[n]).flatten() for n in pn]))
    got = model.state_dict()
    dn = torch.cat([(got[n].cpu() - sd0[n]).flatten() for n in pn])
    assert abs(m["loss"] - res["fp32"][0]) < 2e-2 * max(1.0, res["fp32"][0]), (m, res["fp32"][0], res["emul"][0])
    yard = _rel(res["emul"][1], res["fp32"][1])
    assert _rel(dn, res["fp32"][1]) < 1.5 * yard + 3e-2, (_rel(dn, res["fp32"][1]), yard)
    e = ema.ema.state_dict()
    k = "block4.rep.4.pointwise.weight"
    assert not torch.equal(e[k].cpu(), sd0[k]) and not torch.equal(e[k].cpu(), got[k].cpu())
