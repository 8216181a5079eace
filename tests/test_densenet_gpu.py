"""-m gpu: DenseNet on the native path.

  * the narrow 3x3 convolution (dfd_conv3x3_narrow_tc) and its input gradient against fp64 torch on the same rounded inputs,
    in bf16 and fp16, for growth 32 and 48, at DenseNet's extents (ragged tiles at 9x11, 4x5, 2x2) and at the first and last
    channel slice of a block: channels outside the slice hold a sentinel that must come back bit for bit, and the slice's
    statistics match fp64 sums of the stored values;
  * the channel-slice kernels (prefix BN + ReLU, slice copy with mask and statistics, norm1's backward reduce and
    apply-and-add) and the fused transition (BN + ReLU + floor 2x2 average pool) with its backward;
  * whole train steps of the tc and the mma plans: the loss, the logits and EVERY parameter gradient against the exact (fp64)
    step of tests/densenet_ref.py (held to the reference's own steps on the CPU), each within 1.5 x the distance of the
    restatement's 16-bit emulation from the exact step + 1e-2; a drop_rate step with the native masks given to the
    restatement; batch 32 at 224x224 from the reference's initialisers with the loss and every updated weight within 1e-2;
    fp16 eval at batch 1, two runs bit for bit, a checkpoint round trip and the runner's train_epoch.
"""
import io

import pytest
import torch
import torch.nn.functional as F

import densenet_ref as R

pytestmark = pytest.mark.gpu

TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
DT_CODE = {"bf16": 0, "fp16": 1}
S = 8


def _rel(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _call(name, *args):
    from deepfake_detection_b200 import _lib
    _lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


def _p(t, off=0):
    return None if t is None else t.data_ptr() + off * t.element_size()


def _tol(dtype):
    return 1e-2 if dtype == "bf16" else 2e-3


# (N, H, W, Cin, k, C0, Ctot, slice offset): first and last slice of blocks of densenet121 / densenet161
NARROW = [(2, 56, 56, 128, 32, 64, 256, 64), (2, 56, 56, 128, 32, 64, 256, 224), (3, 9, 11, 128, 32, 256, 1024, 992),
          (4, 4, 5, 128, 32, 512, 1024, 512), (5, 2, 2, 128, 32, 512, 1024, 608), (2, 18, 22, 192, 48, 96, 384, 96),
          (2, 9, 11, 192, 48, 384, 2112, 2064), (3, 7, 7, 192, 48, 1056, 2208, 2160)]


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("N,H,W,Cin,k,C0,Ct,c0", NARROW)
def test_narrow_conv_fwd_and_dgrad(N, H, W, Cin, k, C0, Ct, c0, dtype):
    dt = TDT[dtype]
    g = torch.Generator(device="cuda").manual_seed(H * 1000 + c0 + k)
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).to(dt)
    w = (torch.randn(k, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)).to(dt)
    wpk = w.permute(0, 2, 3, 1).contiguous()                            # [k][kh][kw][Cin]
    sentinel = torch.tensor(-7.25, dtype=dt)
    y = torch.full((N, H, W, Ct), float(sentinel), device="cuda", dtype=dt)
    st = torch.zeros(2, S, Ct, dtype=torch.float64, device="cuda")
    _call("dfd_conv3x3_narrow_tc", _p(x), _p(wpk), _p(y, c0), N, H, W, Cin, k, Ct, DT_CODE[dtype], _p(st[0], c0), _p(st[1], c0), Ct)
    torch.cuda.synchronize()
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), padding=1).permute(0, 2, 3, 1)
    got = y[..., c0:c0 + k]
    assert _rel(got, ref) < _tol(dtype)
    outside = torch.cat([y[..., :c0], y[..., c0 + k:]], -1)
    assert bool((outside == sentinel).all())
    tot = st.sum(1)
    gd = got.double().reshape(-1, k)
    assert _rel(tot[0, c0:c0 + k], gd.sum(0)) < 1e-6 and _rel(tot[1, c0:c0 + k], (gd * gd).sum(0)) < 1e-6
    assert bool((tot[:, :c0] == 0).all()) and bool((tot[:, c0 + k:] == 0).all())
    # input gradient with the tap-flipped [Cin][kh'][kw'][k] weights
    dy = torch.randn(N, H, W, k, device="cuda", generator=g).to(dt)
    wD = w.flip(2, 3).permute(1, 2, 3, 0).contiguous()
    dx = torch.empty(N, H, W, Cin, device="cuda", dtype=dt)
    _call("dfd_conv3x3_narrow_dgrad_tc", _p(dy), _p(wD), _p(dx), N, H, W, Cin, k, DT_CODE[dtype])
    torch.cuda.synchronize()
    xr = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    F.conv2d(xr, w.double(), padding=1).backward(dy.permute(0, 3, 1, 2).double())
    assert _rel(dx, xr.grad.permute(0, 2, 3, 1)) < _tol(dtype)


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("M,C,Ct,k", [(2 * 56 * 56, 224, 256, 32), (3 * 9 * 11, 992, 1024, 32), (5 * 4 * 5, 2064, 2112, 48)])
def test_slice_kernels(M, C, Ct, k, dtype):
    """prefix BN + ReLU, the masked slice copy with statistics, norm1's backward reduce and apply-and-add"""
    dt, code = TDT[dtype], DT_CODE[dtype]
    g = torch.Generator(device="cuda").manual_seed(M + C)
    x = torch.randn(M, Ct, device="cuda", generator=g).to(dt)
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.3
    a = torch.empty(M, C, device="cuda", dtype=dt)
    _call("dfd_bn_relu_ld", _p(x), Ct, _p(scale), _p(shift), _p(a), M, C, code)
    torch.cuda.synchronize()
    assert _rel(a, torch.relu(x[:, :C].double() * scale.double() + shift.double())) < _tol(dtype)
    # slice copy with a dropout mask, statistics after the mask; channels outside the slice untouched
    src = torch.randn(M, k, device="cuda", generator=g).to(dt)
    mask = (torch.rand(M, k, device="cuda", generator=g) > 0.2).float() / 0.8
    dst = x.clone()
    st = torch.zeros(2, S, Ct, dtype=torch.float64, device="cuda")
    c0 = C - k
    _call("dfd_copy_ld", _p(src), k, _p(dst, c0), Ct, _p(mask), M, k, code, _p(st[0], c0), _p(st[1], c0), Ct)
    torch.cuda.synchronize()
    want = (src.float() * mask).to(dt)
    assert torch.equal(dst[:, c0:C], want)
    assert torch.equal(dst[:, :c0], x[:, :c0]) and torch.equal(dst[:, C:], x[:, C:])
    tot = st.sum(1)
    assert _rel(tot[0, c0:C], want.double().sum(0)) < 1e-6 and _rel(tot[1, c0:C], (want.double() ** 2).sum(0)) < 1e-6
    # norm1 backward: sums, then dx_prefix += cA * g' + cB * x + cC
    gr = torch.randn(M, C, device="cuda", generator=g).to(dt)
    mean = torch.randn(C, device="cuda", generator=g) * 0.1
    rstd = torch.rand(C, device="cuda", generator=g) + 0.5
    s = torch.zeros(2, S, C, dtype=torch.float64, device="cuda")
    _call("dfd_relu_bn_bwd_reduce_ld", _p(gr), _p(a), _p(x), Ct, _p(mean), _p(rstd), M, C, code, _p(s[0]), _p(s[1]))
    gm = torch.where(a.double() > 0, gr.double(), torch.zeros((), dtype=torch.float64, device="cuda"))
    xh = (x[:, :C].double() - mean.double()) * rstd.double()
    assert _rel(s[0].sum(0), gm.sum(0)) < 1e-5 and _rel(s[1].sum(0), (gm * xh).sum(0)) < 1e-5
    cA, cB, cC = (torch.randn(C, device="cuda", generator=g) for _ in range(3))
    gx = torch.randn(M, Ct, device="cuda", generator=g).to(dt)
    gx0 = gx.clone()
    _call("dfd_relu_bn_bwd_apply_add_ld", _p(gr), _p(a), _p(x), Ct, _p(cA), _p(cB), _p(cC), _p(gx), Ct, M, C, code)
    torch.cuda.synchronize()
    want = gx0[:, :C].double() + cA.double() * gm + cB.double() * x[:, :C].double() + cC.double()
    assert _rel(gx[:, :C], want) < _tol(dtype)
    assert torch.equal(gx[:, C:], gx0[:, C:])


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("N,H,W,C", [(2, 56, 56, 256), (3, 9, 11, 1024), (4, 18, 22, 512), (2, 5, 7, 2112)])
def test_transition_pool_and_backward(N, H, W, C, dtype):
    dt, code = TDT[dtype], DT_CODE[dtype]
    g = torch.Generator(device="cuda").manual_seed(N * H * W + C)
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dt)
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.3
    Ho, Wo = H // 2, W // 2
    y = torch.empty(N, Ho, Wo, C, device="cuda", dtype=dt)
    _call("dfd_bn_relu_avgpool2", _p(x), _p(scale), _p(shift), _p(y), N, H, W, C, code)
    xr = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    r = torch.relu(xr * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1))
    ref = F.avg_pool2d(r, 2, 2)
    torch.cuda.synchronize()
    assert _rel(y, ref.permute(0, 2, 3, 1)) < _tol(dtype)
    gp = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dt)
    mean = torch.randn(C, device="cuda", generator=g) * 0.1
    rstd = torch.rand(C, device="cuda", generator=g) + 0.5
    s = torch.zeros(2, S, C, dtype=torch.float64, device="cuda")
    _call("dfd_bn_relu_avgpool2_bwd_reduce", _p(gp), _p(x), _p(scale), _p(shift), _p(mean), _p(rstd), N, H, W, C, code,
          _p(s[0]), _p(s[1]))
    ref.backward(gp.permute(0, 3, 1, 2).double())
    gu = xr.grad / scale.double().view(1, -1, 1, 1)              # the gradient of the BN output
    xh = (xr.detach() - mean.double().view(1, -1, 1, 1)) * rstd.double().view(1, -1, 1, 1)
    torch.cuda.synchronize()
    assert _rel(s[0].sum(0), gu.sum((0, 2, 3))) < 1e-5 and _rel(s[1].sum(0), (gu * xh).sum((0, 2, 3))) < 1e-5
    cA, cB, cC = (torch.randn(C, device="cuda", generator=g) for _ in range(3))
    dx = torch.empty_like(x)
    _call("dfd_bn_relu_avgpool2_bwd_apply", _p(gp), _p(x), _p(scale), _p(shift), _p(cA), _p(cB), _p(cC), _p(dx), N, H, W, C, code)
    torch.cuda.synchronize()
    v = lambda t: t.double().view(1, -1, 1, 1)
    want = v(cA) * gu + v(cB) * xr.detach() + v(cC)
    assert _rel(dx, want.permute(0, 2, 3, 1)) < _tol(dtype)


# ---- whole steps --------------------------------------------------------------------------------------------------------
def _state(arch, seed):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import init_state_dict
    return init_state_dict(get_spec(arch), seed=seed)


def _batch(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, H, W, generator=g), torch.randint(0, 2, (n,), generator=g)


LOSS_SCALE = {"bf16": 1.0, "fp16": 1024.0}     # fp16 trains under a loss scale (the runner's dynamic scaling starts higher)


def _native_step(arch, batch, H, W, dtype, sd0, gemm_impl="tc", drop_rate=0.0, seed=1234):
    from deepfake_detection_b200.engine import Engine
    ls = LOSS_SCALE[dtype]
    e = Engine(arch, batch, H, W, dtype=dtype, gemm_impl=gemm_impl, drop_rate=drop_rate)
    e.load_state_dict(sd0)
    x, y = _batch(batch, H, W, seed)
    st = torch.cuda.current_stream().cuda_stream
    e.set_input(x.cuda())
    e.set_target(y.cuda())
    e.zero_step_scratch(st)
    e.forward(training=True, stream=st)
    e.head(True, loss_scale=ls, stream=st)
    e.backward(stream=st)
    torch.cuda.synchronize()
    grads = {n: e.grad_view(n).detach().cpu().double() / ls for n in e.param_names}
    return e, x, y, float(e.loss), e.logits.detach().cpu().clone(), grads


def _check_against_emulation(spec, sd0, x, y, dtype, loss, logits, grads, masks=None, head_mask=None):
    """the loss, the logits and all parameter gradients together within 1.5 x (distance of the 16-bit emulation from the exact
    step) + 1e-2 of the exact step; every gradient tensor within 2 x its own emulation distance + 0.1, which a wrong
    offset, a skipped or doubled addition or a mis-initialised buffer exceeds by far. classifier.bias, a two-element batch
    sum of softmax residuals that nearly cancel, is held by the joint statement only: its relative error is a different
    draw of the rounding noise in the native step and in the emulation."""
    ls = LOSS_SCALE[dtype]
    xc, yc = x.cuda(), y.cuda()
    rl, rlog, rg = R.train_grads(spec, sd0, xc, yc, masks=masks, head_mask=head_mask)
    el, elog, eg = R.train_grads(spec, sd0, xc, yc, masks=masks, head_mask=head_mask, act_dtype=TDT[dtype], loss_scale=ls)
    assert abs(loss - rl) < 1.5 * abs(el - rl) + 1e-2 * abs(rl), (loss, el, rl)
    assert _rel(logits, rlog) < 1.5 * _rel(elog, rlog) + 1e-2, (_rel(logits, rlog), _rel(elog, rlog))
    bad = []
    for n in rg:
        yard = _rel(eg[n], rg[n])
        if n != "classifier.bias" and not _rel(grads[n], rg[n]) < 2 * yard + 0.1:
            bad.append((n, _rel(grads[n], rg[n]), yard))
    names = list(rg)
    cat = lambda d: torch.cat([d[n].flatten().cpu() for n in names])
    yard = _rel(cat(eg), cat(rg))
    assert not bad and _rel(cat(grads), cat(rg)) < 1.5 * yard + 1e-2, (bad[:8], len(bad), _rel(cat(grads), cat(rg)), yard)


@pytest.mark.parametrize("gemm_impl", ["tc", "mma"])
@pytest.mark.parametrize("arch,batch,H,W", [("densenet121", 8, 72, 88), ("densenet161", 4, 70, 54)])
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_step_gradients_against_emulation(arch, batch, H, W, dtype, gemm_impl):
    """the whole backward, parameter by parameter, against the exact (fp64) step with the 16-bit emulation as the yardstick"""
    from deepfake_detection_b200.arch import get_spec
    sd0 = _state(arch, 11)
    e, x, y, loss, logits, grads = _native_step(arch, batch, H, W, dtype, sd0, gemm_impl)
    _check_against_emulation(get_spec(arch), sd0, x, y, dtype, loss, logits, grads)


def test_batch32_224_reference_init():
    """loss and every updated weight within 1e-2 of the exact step from the reference's initialisers (batch 32, 224x224,
    fp16 with the trainer's dynamic loss scaling, one SGD step)"""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.trainer import Trainer
    from oracle import train as OT
    spec = get_spec("densenet121")
    sd0 = _state("densenet121", 3)
    x, y = _batch(32, 224, 224, 1234)
    tr = Trainer("densenet121", 32, 224, 224, dtype="fp16", opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, use_graph=False)
    eng = tr.engine
    for _ in range(8):          # the dynamic scale starts at 65536 and halves on every overflowing (skipped) step
        tr.load_state_dict(sd0)
        loss, _ = tr.train_step(x.cuda(), y.cuda())
        torch.cuda.synchronize()
        if int(eng.flags[1]) == 1:
            break
    else:
        raise AssertionError("no fp16 step was applied")
    rl, _, rg = R.train_grads(spec, sd0, x.cuda(), y.cuda())
    pn = [n for n, _, _ in param_entries(spec)]
    params = {n: sd0[n].double().cuda() for n in pn}
    OT.optimizer_step(OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4), params, {n: rg[n] for n in pn})
    live = [n for n in pn if float(sd0[n].abs().max()) > 0]     # the BN biases start at zero: after one step they hold -lr * g
    worst = max((_rel(eng.param_view(n), params[n]), n) for n in live)
    glob = _rel(torch.cat([eng.param_view(n).flatten().cpu() for n in pn]), torch.cat([params[n].flatten().cpu() for n in pn]))
    loss_rel = abs(float(loss) - rl) / abs(rl)
    assert loss_rel < 1e-2 and worst[0] < 1e-2 and glob < 1e-2, (loss_rel, worst, glob)


def test_drop_rate_step_with_native_masks():
    from deepfake_detection_b200.arch import densenet_extents, get_spec
    sd0 = _state("densenet121", 7)
    e, x, y, loss, logits, grads = _native_step("densenet121", 8, 72, 88, "fp16", sd0, drop_rate=0.2)
    spec = get_spec("densenet121")
    ext = densenet_extents(72, 88)[1:]
    masks = {}
    for b, n in enumerate(spec.block_config):
        h, w = ext[b]
        for l in range(n):
            p = "features.denseblock%d.denselayer%d" % (b + 1, l + 1)
            masks[p] = e.drop_masks[p].double().view(8, h, w, spec.growth)
    kept = torch.cat([m.flatten() for m in masks.values()])
    assert 0.75 < float((kept > 0).double().mean()) < 0.85
    _check_against_emulation(spec, sd0, x, y, "fp16", loss, logits, grads, masks=masks, head_mask=e.dropout_mask.double())


def test_eval_batch1_fp16_and_checkpoint_round_trip():
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    sd0 = _state("densenet121", 2)
    m = create_model("densenet121", num_classes=2, dtype="fp16")
    m.load_state_dict(sd0)
    m.eval()
    x, _ = _batch(1, 224, 224, 9)
    with torch.no_grad():
        got = m(x.cuda()).cpu()
        again = m(x.cuda()).cpu()
    ref = R.forward(get_spec("densenet121"), {k: v.double() for k, v in sd0.items()}, x.double(), training=False)
    assert torch.equal(got, again)
    assert _rel(got, ref) < 2e-2, _rel(got, ref)
    buf = io.BytesIO()
    torch.save(m.state_dict(), buf)
    buf.seek(0)
    m2 = create_model("densenet121", num_classes=2, dtype="fp16")
    m2.load_state_dict(torch.load(buf))
    m2.eval()
    with torch.no_grad():
        assert torch.equal(m2(x.cuda()).cpu(), got)


def test_two_runs_bit_identical():
    sd0 = _state("densenet121", 4)
    a = _native_step("densenet121", 4, 72, 88, "bf16", sd0)
    b = _native_step("densenet121", 4, 72, 88, "bf16", sd0)
    assert a[3] == b[3] and torch.equal(a[4], b[4]) and all(torch.equal(a[5][n], b[5][n]) for n in a[5])


def test_train_epoch_sgd_with_ema():
    from types import SimpleNamespace
    from deepfake_detection_b200.ema import ModelEma
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch

    class _Loader(list):
        mixup_enabled = False

    for opt_name in ("sgd", "rmsproptf"):
        args = SimpleNamespace(opt=opt_name, lr=0.01, momentum=0.9, weight_decay=1e-4, opt_eps=1e-3, prefetcher=True, mixup=0.0,
                               mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0,
                               log_interval=1, save_images=False, recovery_interval=0, tta=0, model="densenet121")
        model = create_model("densenet121", num_classes=2)
        sd0 = {k: v.clone() for k, v in model.state_dict().items()}
        opt = create_optimizer(args, model)
        ema = ModelEma(model, decay=0.9)
        data = [_batch(8, 64, 64, 100 + i) for i in range(2)]
        out = train_epoch(0, model, _Loader((x.cuda(), y.cuda()) for x, y in data), opt, torch.nn.CrossEntropyLoss(), args,
                          model_ema=ema)
        assert torch.isfinite(torch.tensor(out["loss"]))
        k = "features.denseblock2.denselayer3.conv2.weight"
        got = model.state_dict()[k]
        assert not torch.equal(got.cpu(), sd0[k].cpu())
        assert not torch.equal(ema.ema.state_dict()[k].cpu(), got.cpu())
