"""-m gpu: radam / adadelta / rmsprop / novograd / nvnovograd on the H100.

- each kind over the whole arena of every shipped configuration (tests/plan_launches.py CONFIGS), through the Trainer's
  wiring (tests/update_phase.py), in bf16 and in fp16 with loss scaling, over three update phases against an fp64
  restatement with first-order rounding-error bounds; the middle fp16 step overflows and must change nothing;
- the per-tensor sums of squares against fp64, bit-identical across runs;
- captured Trainer steps against oracle/train.py (the reference's step fixtures are held by
  tests/test_reference_steps_gpu.py);
- one captured graph across a per-step lr schedule; state_dict round trips with torch's classes and between native
  optimizers; the runner.
"""
import math
from types import SimpleNamespace

import pytest
import torch

import update_phase as UP
from deepfake_detection_b200 import _lib
from deepfake_detection_b200.arch import get_spec, param_entries
from deepfake_detection_b200.engine import _ptr
from oracle import train as OT
from oracle.weights import synth_batch, synth_state

pytestmark = pytest.mark.gpu

TAGS = list(UP.GPU_BATCH)
KINDS = OT.EXT_KINDS
TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
U = 2.0 ** -24


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


_CACHE = {}


def _engine(tag, dtype):
    key = (tag, dtype)
    if key not in _CACHE:
        _CACHE.clear()
        torch.cuda.empty_cache()
        _CACHE[key] = UP.engine(tag, dtype, batch=UP.GPU_BATCH[tag])
    return _CACHE[key]


def _tensor_index(a):
    """element -> tensor index in arena order (-1 for the alignment padding between tensors)"""
    idx = torch.full((a.n_params,), -1, dtype=torch.long, device="cuda")
    for t, (o, _, k) in enumerate(a.p_off.values()):
        idx[o:o + k] = t
    return idx


def _seg_sum(x, idx, nt):
    out = torch.zeros(nt + 1, dtype=torch.float64, device=x.device)
    out.index_add_(0, idx + 1, x)
    return out[1:]


def _sqrt_err(x, Ex):
    """first-order error of sqrt(x) from an error Ex on x (bounded by sqrt(Ex) where x is tiny)"""
    return torch.minimum(Ex / (2 * x.sqrt()).clamp_min(1e-300), Ex.sqrt())


def _ref_step(kind, S, g, lr, lr0, wd, t, hp, T=None):
    """one fp64 step of the kernel's arithmetic on the flat range in S (p, a, b and error bounds Ep, Ea, Eb), with the fp32
    hyper-parameters the kernels receive. Every fp32 operation rounds within U; E_q collects the propagated input errors
    plus k U (sum of the magnitudes entering q) over the k roundings on q's path. T (layer-wise kinds): per-tensor fp64
    state and its bounds, `ti` the tensor of every element of the range, `n2` the sums of squares."""
    p, a, b, Ep, Ea, Eb = S["p"], S["a"], S["b"], S["Ep"], S["Ea"], S["Eb"]
    Eg = U * g.abs()
    eps = hp["eps"]
    if kind == "radam":
        b1, b2 = 0.9, 0.999
        fb1, fb2, ob1, ob2 = (_f32(x) for x in (b1, b2, 1 - b1, 1 - b2))
        vv = fb2 * b + ob2 * g * g
        Evv = fb2 * Eb + 2 * ob2 * g.abs() * Eg + 3 * U * (fb2 * b.abs() + ob2 * g * g)
        mm = fb1 * a + ob1 * g
        Emm = fb1 * Ea + ob1 * Eg + 2 * U * (fb1 * a.abs() + ob1 * g.abs())
        dec = _f32(-wd * lr)
        p1 = p + dec * p if wd else p
        Ep1 = Ep * (1 + abs(dec)) + 2 * U * p.abs() if wd else Ep
        b2t = b2 ** t
        nmax = 2 / (1 - b2) - 1
        nsma = nmax - 2 * t * b2t / (1 - b2t)
        if nsma >= 5:
            ss = _f32(lr0 * math.sqrt((1 - b2t) * (nsma - 4) / (nmax - 4) * (nsma - 2) / nsma * nmax / (nmax - 2)) / (1 - b1 ** t))
            den = vv.sqrt() + eps
            Eden = _sqrt_err(vv, Evv) + 2 * U * den
            r = mm / den
            Er = Emm / den + r.abs() * Eden / den + U * r.abs()
            d = ss * r
            Ed = ss * Er + 2 * U * d.abs()          # the device step size: double, rounded once to fp32 (its own U)
        else:
            ss = _f32(lr0 / (1 - b1 ** t))
            d = ss * mm
            Ed = ss * Emm + 2 * U * d.abs()
        S.update(p=p1 - d, a=mm, b=vv, Ep=Ep1 + Ed + U * (p1.abs() + d.abs()), Ea=Emm, Eb=Evv)
    elif kind in ("adadelta", "rmsprop"):
        rho = hp["rho"] if kind == "adadelta" else hp["alpha"]
        orho = 1.0 - rho                     # the kernels form 1 - rho in fp32, which is exact for rho = fp32(0.9)
        gg = wd * p + g
        Egg = wd * Ep + Eg + 2 * U * ((wd * p).abs() + g.abs())
        sa = rho * a + orho * gg * gg
        Esa = rho * Ea + 2 * orho * gg.abs() * Egg + 3 * U * (rho * a.abs() + orho * gg * gg)
        if kind == "adadelta":
            num, den = (b + eps).sqrt(), (sa + eps).sqrt()
            Enum, Eden = Eb / (2 * num) + 2 * U * num, Esa / (2 * den) + 2 * U * den
            q = num / den
            delta = q * gg
            Ed = (Enum / den + q * Eden / den) * gg.abs() + q * Egg + 3 * U * delta.abs()
            acc = rho * b + orho * delta * delta
            Eacc = rho * Eb + 2 * orho * delta.abs() * Ed + 3 * U * (rho * b.abs() + orho * delta * delta)
            S.update(p=p - lr * delta, a=sa, b=acc, Ep=Ep + lr * Ed + 2 * U * (p.abs() + lr * delta.abs()), Ea=Esa, Eb=Eacc)
        else:
            mom = hp["momentum"]
            avg = sa.sqrt() + eps
            Eavg = _sqrt_err(sa, Esa) + 2 * U * avg
            q = gg / avg
            Eq = Egg / avg + q.abs() * Eavg / avg + U * q.abs()
            bn = mom * b + q
            Ebn = mom * Eb + Eq + U * (mom * b.abs() + q.abs())
            S.update(p=p - lr * bn, a=sa, b=bn, Ep=Ep + lr * Ebn + 2 * U * (p.abs() + lr * bn.abs()), Ea=Esa, Eb=Ebn)
    elif kind == "nvnovograd":
        b1, b2 = _f32(0.95), _f32(0.98)
        ti = T["ti"]
        d, Ed = T["d"][ti], T["Ed"][ti]
        q = g / d
        gg = q + wd * p
        Egg = Eg / d + q.abs() * (Ed / d + U) + wd * Ep + 2 * U * (q.abs() + (wd * p).abs())
        mm = b1 * a + gg
        Emm = b1 * Ea + Egg + U * (b1 * a.abs() + gg.abs())
        S.update(p=p - lr * mm, a=mm, Ep=Ep + lr * Emm + 2 * U * (p.abs() + lr * mm.abs()), Ea=Emm)
    else:  # novograd
        b1, b2 = _f32(0.95), _f32(0.98)
        ti, fresh, wdn = T["ti"], T["fresh"], T["wd"]
        a0, ra0, a1, ra1 = T["a0"][ti], T["ra0"][ti], T["a1"][ti], T["ra1"][ti]
        dp = wdn * p
        if fresh:
            mp = g * a0 + dp
            Emp = g.abs() * a0 * (ra0 + U) + a0 * Eg + wdn * Ep + 2 * U * ((g * a0).abs() + dp.abs())
        else:
            mp, Emp = a, Ea
        mm = b1 * mp + g * a1 + dp
        Emm = b1 * Emp + g.abs() * a1 * (ra1 + U) + a1 * Eg + wdn * Ep + 3 * U * (b1 * mp.abs() + (g * a1).abs() + dp.abs())
        ss = _f32(lr * math.sqrt(1 - 0.98 ** t) / (1 - 0.95 ** t))
        S.update(p=p - ss * mm, a=mm, Ep=Ep + ss * Emm + 2 * U * (p.abs() + ss * mm.abs()), Ea=Emm)


def _tensor_step(kind, T, n2, hp, fresh):
    """the per-tensor scalars of the layer-wise kinds in fp64 with their relative / absolute bounds"""
    eps, b2 = hp["eps"], _f32(0.98)
    En2 = U * n2                                  # fp64 partials: one rounding, to fp32
    if kind == "nvnovograd":
        e, Ee = T["e"], T["Ee"]
        zero = e == 0
        e2 = torch.where(zero, n2, b2 * e + (1 - b2) * n2)
        Ee2 = torch.where(zero, En2, b2 * Ee + (1 - b2) * En2 + 3 * U * (b2 * e + (1 - b2) * n2))
        d = e2.sqrt() + eps
        T.update(e=e2, Ee=Ee2, d=d, Ed=_sqrt_err(e2, Ee2) + 2 * U * d)
        return
    if fresh:
        ge, Ege, v, Ev = n2, En2, n2, En2
        T["a0"] = 1 / (n2.sqrt() + eps)
        T["ra0"] = (_sqrt_err(n2, En2) + 2 * U * n2.sqrt()) / (n2.sqrt() + eps) + U
    else:
        ge = b2 * T["ge"] + (1 - b2) * n2
        Ege = b2 * T["Ege"] + (1 - b2) * En2 + 3 * U * ge
        v, Ev = T["v"], T["Ev"]
    sg = ge.sqrt() + eps
    r = 1 / sg
    rr = (_sqrt_err(ge, Ege) + 2 * U * sg) / sg + U                 # relative bound of r
    n2h = n2 * r * r
    rn = U + 2 * rr + 2 * U                                        # relative bound of n2h
    v2 = b2 * v + (1 - b2) * n2h
    Ev2 = b2 * Ev + (1 - b2) * n2h * rn + 3 * U * v2
    sv = v2.sqrt() + eps
    T.update(ge=ge, Ege=Ege, v=v2, Ev=Ev2, a1=r / sv, ra1=rr + (_sqrt_err(v2, Ev2) + 2 * U * sv) / sv + 2 * U)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dtype", UP.DTYPES)
@pytest.mark.parametrize("tag", TAGS)
def test_kind_at_arena_geometry(tag, dtype, kind):
    """three Trainer update phases over the whole arena (one lr per group, device lr / step / 1/scale / skip flag); in fp16 the
    middle step overflows and must leave weights, every state, the per-tensor scalars, the init flag and the step counter"""
    e = _engine(tag, dtype)
    a = e.arena
    tr = UP.make_trainer(e, kind)
    o = tr.optimizer
    n, nd = a.n_params, a.n_decay
    dt = TDT[dtype]
    a.flags.zero_()
    gen = torch.Generator(device="cuda").manual_seed(5)
    a.params32.copy_(torch.randn(n, device="cuda", generator=gen) * 0.05)
    hp = dict(momentum=_f32(UP.HYPER["momentum"]), eps=_f32(UP.HYPER["eps"]), alpha=_f32(UP.HYPER["alpha"]), rho=_f32(0.9))
    lr = {gi: _f32(g["lr"]) for gi, g in enumerate(o.param_groups)}
    wd = {gi: _f32(g["weight_decay"]) for gi, g in enumerate(o.param_groups)}
    rng = {0: (nd, n), 1: (0, nd)}
    layerwise = kind in ("novograd", "nvnovograd")
    ti = _tensor_index(a)
    nt = len(a.p_off)
    z = torch.zeros(n, dtype=torch.float64, device="cuda")
    S = {gi: dict(p=a.params32[lo:hi].double(), a=o.state_a[lo:hi].double(),
                  b=(o.state_b[lo:hi].double() if o.state_b is not None else z[lo:hi].clone()),
                  Ep=z[lo:hi].clone(), Ea=z[lo:hi].clone(), Eb=z[lo:hi].clone()) for gi, (lo, hi) in rng.items()}
    zt = torch.zeros(nt, dtype=torch.float64, device="cuda")
    T = dict(e=zt.clone(), Ee=zt.clone(), wd=_f32(o.novograd_wd) if kind == "novograd" else 0.0)

    def state_snapshot():
        ts = [a.params32, o.state_a, a.params16, o.step_dev] + ([o.state_b] if o.state_b is not None else [])
        if layerwise:
            ts += [o.lw_state, o.lw_flags, o.lw_coef]
        return [t.clone() for t in ts]

    # RAdam starts at step 4 so that the three phases cross from N_sma < 5 (step 5) into the rectified update (step 6)
    t0 = 4 if kind == "radam" else 0
    o.step_count = t0
    scaled = dtype == "fp16"
    t = t0
    for step in range(3):
        skip = scaled and step == 1
        g = torch.randn(n, device="cuda", generator=gen) * 0.01
        inv = float(a.loss_scale_state[1]) if scaled else 1.0
        a.grads32.copy_(g / inv)
        if skip:
            a.grads32[int(torch.randint(n, (1,), generator=gen, device="cuda"))] = float("inf")
            before = state_snapshot()
        o.push_hyper()
        tr._launch_step(False, "back")
        torch.cuda.synchronize()
        if skip:
            for x, y in zip(before, state_snapshot()):
                assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                                   y.view(torch.int32) if y.dtype == torch.float32 else y)
            assert float(a.loss_scale_state[0]) == 32768.0 and int(a.flags[0]) == 0
            continue
        t += 1
        gd = a.grads32.double() * inv
        if layerwise:
            n2 = _seg_sum(gd * gd * (ti >= 0), ti, nt)
            _tensor_step(kind, T, n2, hp, fresh=t == 1)
            T["fresh"] = t == 1
        for gi, (lo, hi) in rng.items():
            T["ti"] = ti[lo:hi].clamp_min(0)
            _ref_step(kind, S[gi], gd[lo:hi], lr[gi], lr[0], wd[gi], t, hp, T)
    assert int(o.step_dev) == t
    # the layer-wise kinds update the tensors' elements only, not the alignment padding between them
    inside = ti >= 0 if layerwise else slice(None)
    assert torch.equal(a.params16.view(torch.int16)[inside], a.params32.to(dt).view(torch.int16)[inside])
    if layerwise:
        got = o.lw_state[0].double()
        ref, bound = (T["v"], T["Ev"]) if kind == "novograd" else (T["e"], T["Ee"])
        assert bool(((got - ref).abs() <= 2 * bound + 1e-30).all()), "per-tensor state"
        assert int(o.lw_flags[0]) == (1 if kind == "novograd" else 0)
    for gi, (lo, hi) in rng.items():
        R = S[gi]
        mask = (ti[lo:hi] >= 0) if layerwise else torch.ones(hi - lo, dtype=torch.bool, device="cuda")
        for name, got, key in (("p", a.params32[lo:hi], "p"), ("state_a", o.state_a[lo:hi], "a")) + \
                ((("state_b", o.state_b[lo:hi], "b"),) if o.state_b is not None else ()):
            err = (got.double() - R[key]).abs()[mask]
            bound = 2 * R["E" + key][mask]
            bad = err > bound
            assert not bool(bad.any()), "%s group %d: %d elements out of bound, worst err %.3e (bound %.3e)" % (
                name, gi, int(bad.sum()), float(err.max()), float(bound[(err - bound).argmax()]))
        assert float(R["Ep"][mask].max()) < 1e-3 * float(R["p"][mask].abs().max())


@pytest.mark.parametrize("tag", ["b4", "r50"])
def test_tensor_sumsq_exact_and_reproducible(tag):
    """the per-tensor sums of squares of the whole gradient arena against fp64, twice, bit for bit"""
    e = _engine(tag, "fp16")
    a = e.arena
    tr = UP.make_trainer(e, "nvnovograd")
    o = tr.optimizer
    gen = torch.Generator(device="cuda").manual_seed(2)
    a.grads32.copy_(torch.randn(a.n_params, device="cuda", generator=gen) * 3e3)
    a.loss_scale_state[1] = 2.0 ** -10
    a.flags.zero_()
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    for _ in range(2):
        o.lw_sumsq.fill_(float("nan"))
        o.lw_partial.fill_(float("nan"))
        _lib.call("dfd_tensor_sumsq", _ptr(a.grads32), _ptr(o.lw_table), o.lw_nchunks, _ptr(o.lw_chunk0), len(a.p_off),
                  _ptr(o.lw_partial), _ptr(o.lw_sumsq), 1.0, o.gscale_dev, o.skip_flag, st)
        torch.cuda.synchronize()
        outs.append(o.lw_sumsq.clone())
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    gs = (a.grads32 * (2.0 ** -10)).double()
    ref = torch.stack([gs[off:off + k].square().sum() for off, _, k in a.p_off.values()])
    rel = ((outs[0].double() - ref).abs() / ref.clamp_min(1e-300))
    assert float(rel.max()) <= U * 1.01, float(rel.max())
    # a skipped step writes nothing
    a.flags[0] = 1
    o.lw_sumsq.fill_(7.0)
    _lib.call("dfd_tensor_sumsq", _ptr(a.grads32), _ptr(o.lw_table), o.lw_nchunks, _ptr(o.lw_chunk0), len(a.p_off),
              _ptr(o.lw_partial), _ptr(o.lw_sumsq), 1.0, o.gscale_dev, o.skip_flag, st)
    torch.cuda.synchronize()
    assert bool((o.lw_sumsq == 7.0).all())
    a.flags.zero_()


# ---- whole steps ------------------------------------------------------------------------------------------------------------
def _relerr(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("kind", KINDS)
def test_captured_trainer_against_oracle(kind):
    """two graph-captured fp16 Trainer steps of EfficientNet-B0 against the oracle with the same 16-bit activation rounding:
    the loss at the tolerance of the existing multi-class step tests, the weights' updates per tensor"""
    from deepfake_detection_b200.trainer import Trainer
    spec = get_spec("efficientnet_b0")
    sd0 = synth_state(spec, seed=7)
    lr = 1e-3
    tr = Trainer("efficientnet_b0", 16, 96, 96, dtype="fp16", opt=kind, lr=lr, weight_decay=1e-4, opt_eps=1e-3, use_graph=True)
    tr.load_state_dict(sd0)
    sd = {k: v.clone() for k, v in sd0.items()}
    ost = OT.OptState(kind, lr=lr, weight_decay=1e-4 / lr if kind == "radam" else 1e-4, eps=1e-3)
    for i in range(2):
        x, y = synth_batch(16, 3, 96, 96, seed=1234 + i)
        loss, _ = tr.train_step(x.cuda(), y.cuda())
        o = OT.train_step(spec, sd, x, y, ost, act_dtype=torch.float16)
        assert abs(float(loss) - float(o["loss"])) < 3e-3 * (1 + i) * max(1.0, float(o["loss"])), (i, float(loss))
    torch.cuda.synchronize()
    assert tr.n_captures == 1
    upd = [(n, _relerr(tr.engine.param_view(n) - sd0[n].cuda(), sd[n] - sd0[n])) for n, s, _ in param_entries(spec)
           if len(s) > 1 and float((sd[n] - sd0[n]).norm()) > 0]
    worst = sorted(upd, key=lambda t: -t[1])[:3]
    # 16-bit activations move the gradients by a few percent; an update taken with the wrong lr, decay or per-tensor
    # scalar is off by tens of percent
    assert sum(r for _, r in upd) / len(upd) < 5e-2 and worst[0][1] < 0.3, worst


def test_one_graph_survives_lr_schedule_for_every_kind():
    from deepfake_detection_b200.trainer import Trainer
    sd = synth_state(get_spec("efficientnet_b0"), seed=7)
    x, y = synth_batch(8, 3, 96, 96, seed=1)
    for kind in KINDS:
        tr = Trainer("efficientnet_b0", 8, 96, 96, dtype="fp16", opt=kind, lr=0.01, loss_scale="none")
        tr.load_state_dict(sd)
        snaps = []
        for lr in (0.01, 0.005, 0.0, 0.0):
            for g in tr.optimizer.param_groups:
                g["lr"] = lr
            tr.train_step(x.cuda(), y.cuda())
            torch.cuda.synchronize()
            snaps.append(tr.engine.params32.clone())
        assert tr.n_captures == 1 and tr._graph is not None, (kind, tr.n_captures)
        assert not torch.equal(snaps[0], snaps[1]), kind
        # lr 0 read from device memory by the replayed graph: every kind applies its lr at the weight update, and RAdam's
        # decay is scaled by it too, so the weights stop moving
        assert torch.equal(snaps[2], snaps[3]), kind
        assert tr.optimizer.step_count == 4, kind


# ---- checkpoints ------------------------------------------------------------------------------------------------------------
def _reference_class(kind, named, lr, wd, eps):
    """the reference's optimizer class over CPU tensors, with the factory's groups (the classes need no GPU)"""
    from deepfake_detection_b200.arch import is_no_decay
    nd = [p for n, p in named if is_no_decay(n, tuple(p.shape))]
    d = [p for n, p in named if not is_no_decay(n, tuple(p.shape))]
    groups = [{"params": nd, "weight_decay": 0.0}, {"params": d, "weight_decay": wd}]
    if kind == "adadelta":
        return torch.optim.Adadelta(groups, lr=lr, eps=eps)
    if kind == "rmsprop":
        return torch.optim.RMSprop(groups, lr=lr, alpha=0.9, eps=eps, momentum=0.9)
    pytest.skip("the reference's own class is not importable on the GPU machine")


@pytest.mark.parametrize("kind", ["adadelta", "rmsprop"])
def test_state_dict_round_trip_with_torch_classes(kind):
    """native -> torch.optim class (CPU) -> one more step equals the native continuing, and the reverse load"""
    from deepfake_detection_b200.trainer import Trainer
    spec = get_spec("efficientnet_b0")
    sd0 = synth_state(spec, seed=7)
    x, y = synth_batch(8, 3, 96, 96, seed=3)
    tr = Trainer("efficientnet_b0", 8, 96, 96, dtype="bf16", opt=kind, lr=0.01, opt_eps=1e-3, use_graph=False)
    tr.load_state_dict(sd0)
    for _ in range(2):
        tr.train_step(x.cuda(), y.cuda())
    torch.cuda.synchronize()
    osd = tr.optimizer.state_dict()
    e = tr.engine
    named = [(n, torch.nn.Parameter(e.param_view(n).detach().cpu().clone())) for n in tr.optimizer.param_groups[0]["params"] +
             tr.optimizer.param_groups[1]["params"]]
    ref = _reference_class(kind, named, 0.01, 1e-4, 1e-3)
    ref.load_state_dict({"state": {k: {kk: vv.cpu() for kk, vv in v.items()} for k, v in osd["state"].items()},
                         "param_groups": osd["param_groups"]})
    # one more native step with a known gradient
    g = torch.Generator(device="cuda").manual_seed(4)
    e.grads32.copy_(torch.randn(e.n_params, device="cuda", generator=g) * 1e-2)
    for (n, p) in named:
        o, s, k = e.p_off[n]
        p.grad = e.grads32[o:o + k].view(s).cpu().clone()
    tr.optimizer.step()
    ref.step()
    torch.cuda.synchronize()
    worst = max(_relerr(e.param_view(n), p) for n, p in named if p.dim() > 1)
    assert worst < 1e-5, worst
    assert int(ref.state_dict()["state"][0]["step"]) == tr.optimizer.step_count == 3
    # reverse: the torch class's state loads into a fresh native optimizer
    from deepfake_detection_b200.optim import ArenaOptimizer
    o2 = ArenaOptimizer(e, opt=kind, lr=0.01, eps=1e-3)
    o2.load_state_dict(ref.state_dict())
    for gi in range(2):
        for n in o2.param_groups[gi]["params"]:
            o, s, k = e.p_off[n]
            torch.testing.assert_close(o2.state_a[o:o + k].cpu(), tr.optimizer.state_a[o:o + k].cpu(), rtol=1e-5, atol=1e-9)
    assert o2.step_count == 3


@pytest.mark.parametrize("kind", ["novograd", "nvnovograd", "radam"])
def test_state_dict_round_trip_layerwise(kind):
    """native state_dict -> a fresh native optimizer: RAdam and NvNovoGrad continue exactly as the original; NovoGrad
    re-initialises on its first step after the load (the reference's _momentum_initialized is not saved), exactly as a
    freshly built NovoGrad does on the same gradient"""
    from deepfake_detection_b200.optim import ArenaOptimizer
    e = _engine("b0", "bf16").arena
    gen = torch.Generator(device="cuda").manual_seed(6)
    p0 = torch.randn(e.n_params, device="cuda", generator=gen) * 0.05
    grads = [torch.randn(e.n_params, device="cuda", generator=gen) * 1e-2 for _ in range(3)]
    e.params32.copy_(p0)
    o = ArenaOptimizer(e, opt=kind, lr=1e-2, eps=1e-3)
    for gr in grads[:2]:
        e.grads32.copy_(gr)
        o.step()
    sd = o.state_dict()
    w = e.params32.clone()
    e.grads32.copy_(grads[2])
    o.step()
    cont = e.params32.clone()
    e.params32.copy_(w)
    o2 = ArenaOptimizer(e, opt=kind, lr=1e-2, eps=1e-3)
    o2.load_state_dict(sd)
    assert o2.step_count == 2
    e.grads32.copy_(grads[2])
    o2.step()
    torch.cuda.synchronize()
    if kind != "novograd":
        # a state_dict holds the tensors' elements: compare those (RAdam also steps the alignment padding between them)
        inside = _tensor_index(e) >= 0
        assert torch.equal(e.params32[inside], cont[inside])
    else:
        fresh = ArenaOptimizer(e, opt=kind, lr=1e-2, eps=1e-3)
        got = e.params32.clone()
        e.params32.copy_(w)
        fresh.step()
        torch.cuda.synchronize()
        assert torch.equal(got, e.params32) and not torch.equal(got, cont)
        assert o2.step_count == 1 and int(o2.lw_flags[0]) == 1
    sd2 = o2.state_dict()
    assert set(sd2["state"][0]) == set(sd["state"][0])


# ---- the runner -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_runner_train_epoch(kind):
    from deepfake_detection_b200 import loss as NL
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch

    class Loader(list):
        mixup_enabled = False

    args = SimpleNamespace(opt=kind, lr=1e-3, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0,
                           mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0,
                           log_interval=1, recovery_interval=0, tta=0)
    model = create_model("efficientnet_b0", num_classes=2, dtype="bf16")
    model.load_state_dict(synth_state(get_spec("efficientnet_b0"), seed=7))
    opt = create_optimizer(args, model)
    w0 = model.engine.params32.clone()
    train = Loader((x.cuda(), y.cuda()) for x, y in (synth_batch(8, 3, 96, 96, seed=60 + i) for i in range(3)))
    m = train_epoch(0, model, train, opt, NL.CrossEntropyLoss(), args)
    torch.cuda.synchronize()
    assert math.isfinite(m["loss"]) and not torch.equal(w0, model.engine.params32)
    assert bool(torch.isfinite(model.engine.params32).all()) and opt.step_count == 3

