"""-m gpu: ResNet DropBlock, drop path and classifier dropout on the H100.

Masks: dfd_drop_block_masks against the reference expression recomputed in torch from the kernel's own uniform draws (exact),
its kept count, the seed-drop rate inside the valid region, and fresh masks every step and every graph replay. Kernels: the
masked BN + ReLU forward, block tail and the two backward reductions against fp64 torch on the same rounded operands, in
bf16 and fp16, with bit-identical reruns. End to end: one training step of ResNet-18 / ResNet-50 with all three rates
against tests/resnet_drop_oracle.py given the engine's masks (the statements and thresholds of
test_engine_gpu.py::test_resnet_train_step_parity), and the runner protocol with ModelEma."""
from types import SimpleNamespace

import pytest
import torch

from deepfake_detection_b200 import _lib
from deepfake_detection_b200.engine_resnet import drop_block_desc

import resnet_drop_oracle as RO

pytestmark = pytest.mark.gpu

TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
DT = {"bf16": _lib.DT_BF16, "fp16": _lib.DT_FP16}


def _P(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rel(a, b, floor=0.0):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + floor + 1e-30))


def _draw(shapes, step, noise=True):
    """run dfd_drop_block_masks over sites (N, H, W, C, rate, gamma_scale) at generator step `step`"""
    state = torch.tensor([1234567, step], dtype=torch.int64, device="cuda")
    kept = torch.zeros(len(shapes), dtype=torch.int64, device="cuda")
    out, raw = [], b""
    for i, (N, H, W, C, rate, gs) in enumerate(shapes):
        gamma, cb = RO.drop_block_gamma(H, W, rate, gs)
        m = torch.full((N, H, W, C), 7, dtype=torch.uint8, device="cuda")
        u = torch.full((N, H, W, C), -1.0, device="cuda") if noise else None
        raw += drop_block_desc(_P(m), _P(u), _P(kept) + 8 * i, gamma, N, H, W, C, cb, 100 + i)
        out.append((m, u, gamma, cb))
    table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    _lib.call("dfd_drop_block_masks", _P(table), len(shapes), _P(state), _st())
    torch.cuda.synchronize()
    return out, kept.cpu()


SITES = [(4, 10, 10, 64, 0.2, 1.0), (3, 5, 5, 32, 0.5, 1.0), (2, 7, 7, 64, 0.3, 1.0), (4, 10, 14, 64, 0.2, 0.25),
         (2, 5, 7, 64, 0.2, 1.0), (16, 14, 14, 256, 0.1, 0.25), (2, 40, 33, 96, 0.3, 1.0), (8, 28, 28, 256, 0.1, 0.25)]


def test_drop_block_masks_match_reference_expression():
    """the block mask equals drop_block_2d's expression evaluated by torch on the kernel's noise; exact kept count; seeds
    only inside `valid`, at rate gamma within 4 sigma; another step draws other masks"""
    out, kept = _draw(SITES, 0)
    out2, _ = _draw(SITES, 1, noise=False)
    for (N, H, W, C, rate, gs), (m, u, gamma, cb), k, (m2, _, _, _) in zip(SITES, out, kept, out2):
        un = u.permute(0, 3, 1, 2).cpu()
        assert float(un.min()) >= 0.0 and float(un.max()) < 1.0
        seeds = RO.seeds_from_noise(un, gamma, cb)
        ref = RO.block_from_seeds(seeds, cb)
        got = m.permute(0, 3, 1, 2).cpu().float()
        assert torch.equal(got, ref), (H, W, C, gamma)
        assert int(k) == int(m.sum())
        valid = RO.valid_block(H, W, cb).expand_as(seeds).bool()
        dropped = seeds == 0
        assert not bool(dropped[~valid].any())
        n = int(valid.sum())
        if gamma <= 0 or n == 0:
            assert not bool(dropped.any())
        else:
            rate_got = float(dropped[valid].float().mean())
            sigma = (gamma * (1 - gamma) / n) ** 0.5
            assert abs(rate_got - gamma) < 4 * sigma + 1e-12, (H, W, gamma, rate_got, sigma)
            assert not torch.equal(m, m2)
    # the plan's table has no noise operand: the same masks without it
    again, kept_again = _draw(SITES, 0, noise=False)
    assert all(torch.equal(a[0], b[0]) for a, b in zip(out, again)) and torch.equal(kept, kept_again)


def _operands(N, hw, C, dt, seed, rate=0.3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    T = TDT[dt]
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    y = r(N, hw, C).to(T)
    res = r(N, hw, C).to(T)
    da = r(N, hw, C).to(T)
    g2 = r(N, hw, C).to(T)
    scale, shift = 0.5 + torch.rand(C, device="cuda", generator=g), 0.3 * r(C)
    mean, rstd = 0.2 * r(C), 0.5 + torch.rand(C, device="cuda", generator=g)
    mask = (torch.rand(N, hw, C, device="cuda", generator=g) > rate).to(torch.uint8)
    kept = mask.sum().view(1).to(torch.int64)
    gate = (torch.rand(N, 1, device="cuda", generator=g) > 0.2).float().expand(N, C).contiguous() / 0.8
    return dict(y=y, res=res, da=da, g2=g2, scale=scale, shift=shift, mean=mean, rstd=rstd, mask=mask, kept=kept, gate=gate)


def _ms64(o):
    s = torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(float(o["kept"]), dtype=torch.float32) + 1e-7) * o["mask"].numel()
    return o["mask"].double() * float(s)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("N,hw,C", [(4, 196, 256), (3, 25, 512), (2, 784, 64)])
def test_bn_act_drop(dt, N, hw, C):
    o = _operands(N, hw, C, dt, 1)
    ms = _ms64(o)
    u = (o["y"].float() * o["scale"] + o["shift"]).double()
    for res_mode, gate in ((0, None), (2, None), (2, o["gate"]), (0, o["gate"])):
        outs = []
        for _ in range(2):
            out = torch.full_like(o["y"], float("nan"))
            _lib.call("dfd_bn_act_drop", _P(o["y"]), _P(o["scale"]), _P(o["shift"]), _P(o["mask"]), _P(o["kept"]), o["mask"].numel(),
                      _P(gate), _P(o["res"]) if res_mode else None, _P(out), N, hw, C, res_mode, DT[dt], _st())
            outs.append(out)
        torch.cuda.synchronize()
        ref = u * ms
        if gate is not None:
            ref = ref * gate.double().view(N, 1, C)
        if res_mode:
            ref = ref + o["res"].double()
        ref = ref.clamp_min(0)
        assert torch.equal(outs[0], outs[1])
        err = float((outs[0].double() - ref).abs().max() / (ref.abs().max() + 1e-30))
        assert err < (2.0 ** -7 if dt == "bf16" else 2.0 ** -10), (res_mode, gate is not None, err)


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("N,hw,C", [(4, 196, 256), (3, 25, 512), (2, 784, 64)])
def test_act_bwd_drop(dt, N, hw, C):
    o = _operands(N, hw, C, dt, 2)
    ms = _ms64(o)
    u = o["y"].float() * o["scale"] + o["shift"]
    ref = o["da"].double() * ms * (u > 0).double()
    xhat = (o["y"].double() - o["mean"].double()) * o["rstd"].double()
    outs = []
    for _ in range(2):
        gu = torch.full_like(o["y"], float("nan"))
        s = torch.zeros(2, 8, C, dtype=torch.float64, device="cuda")
        _lib.call("dfd_act_bwd_drop", _P(o["da"]), _P(o["y"]), _P(o["scale"]), _P(o["shift"]), _P(o["mean"]), _P(o["rstd"]),
                  _P(o["mask"]), _P(o["kept"]), o["mask"].numel(), _P(gu), N, hw, C, DT[dt], _P(s[0]), _P(s[1]), _st())
        outs.append((gu, s.sum(1)))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0])
    gu, s = outs[0]
    err = float((gu.double() - ref).abs().max() / (ref.abs().max() + 1e-30))
    assert err < (2.0 ** -7 if dt == "bf16" else 2.0 ** -10), err
    g64 = gu.double()               # the sums are of the stored (rounded) gradient
    assert _rel(s[0], g64.sum((0, 1))) < 1e-5 and _rel(s[1], (g64 * xhat).sum((0, 1))) < 1e-5


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("N,hw,C", [(4, 196, 256), (3, 49, 2048), (2, 784, 64)])
def test_relu_bn_bwd_reduce_drop(dt, N, hw, C):
    o = _operands(N, hw, C, dt, 3)
    ms = _ms64(o)
    out = (o["res"].float() + 0.3).to(TDT[dt])         # the block output whose sign masks the gradient
    xhat = (o["y"].double() - o["mean"].double()) * o["rstd"].double()
    for use_mask, use_gate, use_g2 in ((True, True, True), (True, False, False), (False, True, True), (True, False, True)):
        outs = []
        for _ in range(2):
            gm = torch.full_like(o["y"], float("nan"))
            gd = torch.full_like(o["y"], float("nan"))
            s = torch.zeros(2, 8, C, dtype=torch.float64, device="cuda")
            _lib.call("dfd_relu_bn_bwd_reduce_drop", _P(o["da"]), _P(o["g2"]) if use_g2 else None, _P(o["y"]), _P(out), _P(gm),
                      _P(o["mask"]) if use_mask else None, _P(o["kept"]), o["mask"].numel(), _P(o["gate"]) if use_gate else None,
                      _P(gd), _P(o["mean"]), _P(o["rstd"]), N, hw, C, DT[dt], _P(s[0]), _P(s[1]), _st())
            outs.append((gm, gd, s.sum(1)))
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        gm, gd, s = outs[0]
        g = o["da"].float() + o["g2"].float() if use_g2 else o["da"].float()
        gm_ref = g.to(TDT[dt]).double() * (out.float() > 0).double()        # round16(g + g2), then the ReLU mask
        assert torch.equal(gm.double(), gm_ref), (use_mask, use_gate, use_g2)
        gd_ref = gm_ref * (ms if use_mask else 1.0) * (o["gate"].double().view(N, 1, C) if use_gate else 1.0)
        err = float((gd.double() - gd_ref).abs().max() / (gd_ref.abs().max() + 1e-30))
        assert err < (2.0 ** -7 if dt == "bf16" else 2.0 ** -10), err
        g64 = gd.double()
        assert _rel(s[0], g64.sum((0, 1))) < 1e-5 and _rel(s[1], (g64 * xhat).sum((0, 1))) < 1e-5


def _tame(spec, sd):
    """engine_checks.run_parity(tame=True): damp the residual branches of the synthetic weights"""
    for b in spec.blocks:
        k = b.name + (".bn2.weight" if b.kind == "basic" else ".bn3.weight")
        sd[k] = sd[k] * 0.2
    return sd


RATES = dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.2)


@pytest.mark.parametrize("arch,batch,res,dtype", [("resnet18", 8, 160, "fp16"), ("resnet50", 8, 160, "fp16"),
                                                  ("resnet18", 8, 160, "bf16"), ("resnet50", 32, 224, "bf16")])
def test_train_step_with_drop_matches_oracle(arch, batch, res, dtype):
    """one training step with all three rates against the drop oracle given the engine's masks (emulation and fp32), with the
    statements and thresholds of test_resnet_train_step_parity; then eval mode applies no mask"""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.optim import ArenaOptimizer
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    import engine_checks as EC
    spec = get_spec(arch)
    sd0 = _tame(spec, synth_state(spec, seed=7))
    eng = Engine(arch, batch, res, res, dtype=dtype, **RATES)
    eng.load_state_dict(sd0)
    opt = ArenaOptimizer(eng, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    x, y = synth_batch(batch, 3, res, res, seed=1234)
    EC.engine_step(eng, opt, x.cuda(), y.cuda())
    db, dp, dm = RO.engine_masks(eng)
    assert len(db) == (8 if arch == "resnet18" else 27) and len(dp) == len(spec.blocks)
    assert all(int(k) == int(m.sum()) for m, k in eng.drop_block_masks.values())
    pn = [n for n, _, _ in param_entries(spec)]
    rep = {}
    for key, adt in (("emul", TDT[dtype]), ("fp32", None)):
        sd = {k: v.clone() for k, v in sd0.items()}
        out = RO.train_step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4), act_dtype=adt,
                            drop_block=db, drop_masks=dp, dropout_mask=dm)
        tot = torch.cat([out["grads"][n].flatten() for n in pn])
        rep[key] = dict(logits=out["logits"], loss=float(out["loss"]), grads=tot, sd=sd)
    gn = torch.cat([eng.grad_view(n).flatten().cpu() for n in pn])
    em, fp = rep["emul"], rep["fp32"]
    yard_logits, yard_grads = _rel(em["logits"], fp["logits"]), _rel(em["grads"], fp["grads"])
    assert _rel(eng.logits, em["logits"]) < (2e-2 if dtype == "fp16" else 6e-2)
    assert abs(float(eng.loss) - em["loss"]) < 5e-3, (float(eng.loss), em["loss"])
    assert _rel(eng.logits, fp["logits"]) < 1.5 * yard_logits + 1e-2
    assert _rel(gn, fp["grads"]) < 1.5 * yard_grads + 3e-2, (_rel(gn, fp["grads"]), yard_grads)
    # eval: the validate path applies none of the masks
    xe, ye = synth_batch(batch, 3, res, res, seed=999)
    eng.set_input(xe.cuda())
    eng.forward(training=False)
    eng.head(False)
    torch.cuda.synchronize()
    ev = OT.validate_step(spec, em["sd"], xe, ye, act_dtype=TDT[dtype])
    assert _rel(eng.logits, ev["logits"]) < 5e-2


def test_graph_replays_draw_fresh_masks():
    """a captured Trainer step draws new masks on every replay, from one capture"""
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.trainer import Trainer
    from oracle.weights import synth_batch, synth_state
    spec = get_spec("resnet18")
    tr = Trainer("resnet18", 8, 160, 160, dtype="fp16", use_graph=True, **RATES)
    tr.load_state_dict(_tame(spec, synth_state(spec, seed=7)))
    seen = []
    for i in range(3):
        x, y = synth_batch(8, 3, 160, 160, seed=1234 + i)
        loss, _ = tr.train_step(x.cuda(), y.cuda())
        torch.cuda.synchronize()
        assert torch.isfinite(torch.as_tensor(float(loss)))
        e = tr.engine
        # all sites and blocks together: one block's gate alone (8 samples, keep 0.9) repeats across two steps with p = 0.9 ** 16 = 0.19
        seen.append((torch.cat([m.flatten() for m, _ in e.drop_block_masks.values()]),
                     torch.cat([g.flatten() for g in e.drop_masks.values()]), e.dropout_mask.clone()))
    assert tr.n_captures == 1
    for a, b in ((0, 1), (1, 2)):
        assert all(not torch.equal(u, v) for u, v in zip(seen[a], seen[b]))


class _Loader(list):
    mixup_enabled = False


def test_runner_and_ema_with_drop():
    """train_epoch + validate with a rate-configured ResNet-18 and ModelEma; eval logits equal an undropped plan's over the
    same weights"""
    from deepfake_detection_b200 import loss as NL
    from deepfake_detection_b200.ema import ModelEma
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch, validate
    from oracle.weights import synth_batch, synth_state
    model = create_model("resnet18", num_classes=2, dtype="fp16", **RATES)
    model.load_state_dict(_tame(model.spec, synth_state(model.spec, seed=7)))
    args = SimpleNamespace(opt="sgd", lr=0.001, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0,
                           mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0,
                           log_interval=1, save_images=False, recovery_interval=0, tta=0, model="resnet18")
    opt = create_optimizer(args, model)
    batches = _Loader((x.cuda(), y.cuda()) for x, y in (synth_batch(16, 3, 160, 160, seed=1234 + i) for i in range(2)))
    m = train_epoch(0, model, batches, opt, NL.CrossEntropyLoss(), args)
    v = validate(model, batches, torch.nn.CrossEntropyLoss(), args)
    assert m["loss"] > 0 and v["loss"] > 0
    e = model.engine_for(16, 160, 160)
    assert len(e.drop_block_masks) == 8 and len(e.drop_masks) == 8 and e.drop_rate == 0.2
    ema = ModelEma(model, decay=0.9)
    assert ema.ema.drop_block_rate == 0.2 and ema.ema.drop_path_rate == 0.1 and ema.ema.drop_rate == 0.2
    ema.ema.eval()
    model.eval()
    x = batches[0][0]
    with torch.no_grad():
        got = model(x)
        assert torch.equal(ema.ema(x), got)
    plain = Engine("resnet18", 16, 160, 160, dtype="fp16", share_from=model.engine)
    plain.set_input(x)
    plain.zero_step_scratch(_st(), grads=False)
    plain.forward(training=False)
    plain.head(False)
    torch.cuda.synchronize()
    assert torch.equal(plain.logits, got)
