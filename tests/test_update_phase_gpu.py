"""-m gpu: the update half of the training step at the arenas of the shipped configurations (tests/plan_launches.py CONFIGS),
in bf16 and in fp16 with dynamic loss scaling: the optimizer kernels against an fp64 restatement of oracle.train's
optimizer_step, every derived weight layout bit for bit against its definition, the loss-scale kernels against the contract,
the EMA, and a captured step that meets a later plan over the same arena."""
import math

import pytest
import torch

import update_phase as UP
from deepfake_detection_b200 import _lib
from deepfake_detection_b200.engine import _ptr

pytestmark = pytest.mark.gpu

TAGS = list(UP.GPU_BATCH)
TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
U = 2.0 ** -24                      # unit roundoff of fp32

# kernel of the update phase -> the test here that runs it at the arena's element counts with the Trainer's pointers
# (tests/test_update_phase_cpu.py holds this table to the launches of the shipped plans)
RUNS = {
    "dfd_set_floats": "test_optimizer_at_arena_geometry",
    "dfd_sgd_step": "test_optimizer_at_arena_geometry",
    "dfd_adam_step": "test_optimizer_at_arena_geometry",
    "dfd_rmsprop_tf_step": "test_optimizer_at_arena_geometry",
    "dfd_opt_tick": "test_optimizer_at_arena_geometry",
    "dfd_check_finite": "test_check_finite_full_arena",
    "dfd_update_loss_scale": "test_update_loss_scale_contract",
    "dfd_transpose_weights": "test_derived_layouts_exact",
    "dfd_repack_weights": "test_derived_layouts_exact",
    "dfd_pad_weight": "test_derived_layouts_exact",
    "dfd_blockdiag_weights": "test_derived_layouts_exact",
    "dfd_ema_update": "test_ema_at_arena_size",
}


def st():
    return torch.cuda.current_stream().cuda_stream


_CACHE = {}


def _engine(tag, dtype):
    """the configuration's plan at GPU_BATCH (one kept alive at a time: the parametrisations below group by configuration)"""
    key = (tag, dtype)
    if key not in _CACHE:
        _CACHE.clear()
        torch.cuda.empty_cache()
        _CACHE[key] = UP.engine(tag, dtype, batch=UP.GPU_BATCH[tag])
    return _CACHE[key]


def _bits(t):
    return t.view(torch.int16)


# ---- derived layouts ----------------------------------------------------------------------------------------------------------
def check_derived_layouts(a):
    """every derived 16-bit layout of arena `a` equals its definition built from round16(params32), bit for bit. The expected
    values come from the fp32 master weights, never from the current contents of a source buffer (a block-diagonal copy of a
    transposed or padded weight refreshed before its source would pass a comparison against the source). Returns the number
    of layouts compared."""
    dt = a.tdtype
    w16 = a.params32.to(dt)
    assert torch.equal(_bits(a.params16), _bits(w16)), "params16 != round16(params32)"

    def W(name):
        o, s, n = a.p_off[name]
        return w16[o:o + n].view(s)

    nchk = 0
    for name, (o, O, I) in a.t_off.items():
        assert torch.equal(_bits(a.paramsT16[o:o + O * I].view(I, O)), _bits(W(name).reshape(O, I).t().contiguous())), name
        nchk += 1
    stem = {}
    for key, wpad in getattr(a, "_stem_reg", {}).items():
        name, O, taps, Kp = key
        ref = torch.zeros(O, Kp, dtype=dt, device=w16.device)
        ref[:, :taps] = W(name).reshape(O, taps)
        assert torch.equal(_bits(wpad.view(O, Kp)), _bits(ref)), key
        stem[key] = ref
        nchk += 1
    by_t = {o: n for n, (o, _, _) in a.t_off.items()}
    by_p = {a.p_off[n][0]: n for n in a.p_off}
    for (B, Nn, K, pack), t in getattr(a, "_bd_reg", {}).items():
        buf, where = UP._where(a, B)
        if buf == "params16":
            src = W(by_p[where]).reshape(Nn, K)
        elif buf == "paramsT16":
            n = by_t[where]
            src = W(n).reshape(a.t_off[n][1], a.t_off[n][2]).t()
        else:
            src = stem[where]
        assert tuple(src.shape) == (Nn, K)
        ref = torch.block_diag(*([src.float()] * pack)).to(dt)
        assert torch.equal(_bits(t.view(pack * Nn, pack * K)), _bits(ref)), (buf, where, Nn, K, pack)
        nchk += 1
    for name, O, I, k, d in UP.repack_entries(a):
        w = W(name)                                                    # [O, I, k, k]
        n = O * I * k * k
        assert torch.equal(_bits(a.wpack16[d:d + n]), _bits(w.permute(0, 2, 3, 1).reshape(-1))), name
        assert torch.equal(_bits(a.wpackT16[d:d + n]), _bits(w.permute(2, 3, 1, 0).reshape(-1))), name
        assert torch.equal(_bits(a.wpackD16[d:d + n]), _bits(w.flip(2, 3).permute(1, 2, 3, 0).reshape(-1))), name
        nchk += 1
    return nchk


def _nan_fill_derived(a):
    for t in [a.params16, a.paramsT16] + list(getattr(a, "_bd_reg", {}).values()) + list(getattr(a, "_stem_reg", {}).values()):
        t.fill_(float("nan"))
    if getattr(a, "_rtable_count", 0):
        for t in (a.wpack16, a.wpackT16, a.wpackD16):
            t.fill_(float("nan"))


@pytest.mark.parametrize("dtype", UP.DTYPES)
@pytest.mark.parametrize("tag", TAGS)
def test_derived_layouts_exact(tag, dtype):
    e = _engine(tag, dtype)
    a = e.arena
    g = torch.Generator(device="cuda").manual_seed(11)
    a.params32.copy_(torch.randn(a.n_params, device="cuda", generator=g) * 0.1)
    a.grads32.copy_(torch.randn(a.n_params, device="cuda", generator=g))
    _nan_fill_derived(a)
    tr = UP.make_trainer(e, "sgd")
    tr.optimizer.push_hyper()
    tr._launch_step(False, "back")
    torch.cuda.synchronize()
    n = check_derived_layouts(a)
    assert n >= len(a.t_off) + 1


# ---- the optimizer at the arena geometry ----------------------------------------------------------------------------------
def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _bc_rel(b, t):
    """relative error bound of the fp32 bias correction 1 - powf(b, t) (powf within the 4 ulps CUDA documents, the subtraction
    then rounded at most once): it is amplified by b^t / (1 - b^t)"""
    bt = b ** t
    return 8 * U * bt / (1 - bt) + U


def _ref_step(kind, S, g, lr, wd, t, hp):
    """one fp64 step of oracle.train.optimizer_step (sgd = nesterov, adam / adamw, rmsproptf) on the flat range held in S
    (dict of fp64 tensors p, a, b and their first-order error bounds Ep, Ea, Eb), with the fp32 hyper-parameters the kernels
    receive.

    Error bound: every fp32 operation of the kernel rounds its result to within U = 2^-24 relative (an fma once). Writing A_q for
    the sum of the magnitudes of the terms that make up a quantity q, a computed q carries E_q = (errors of its inputs, scaled by
    the partial derivatives) + k U A_q, with k the number of roundings on q's path. Propagated through the three steps this is a
    first-order bound on |kernel - fp64| per element; the tests allow twice it, which covers the second-order terms. For the
    weights it comes to a few fp32 ulps of |p| + |update|, the magnitudes entering the final fma; Adam adds the error of its fp32
    bias corrections (_bc_rel), which the device computes with powf."""
    p, a, b = S["p"], S["a"], S["b"]
    Ep, Ea, Eb = S["Ep"], S["Ea"], S["Eb"]
    mom = hp["momentum"]
    if kind == "sgd":
        gg = wd * p + g
        Agg = (wd * p).abs() + g.abs()
        Egg = wd * Ep + 2 * U * Agg
        buf = mom * a + gg
        Abuf = mom * a.abs() + Agg
        Ebuf = mom * Ea + Egg + U * Abuf
        upd = mom * buf + gg
        Eupd = mom * Ebuf + Egg + U * (mom * Abuf + Agg)
        pn = p - lr * upd
        S.update(p=pn, a=buf, Ep=Ep + lr * Eupd + U * (p.abs() + lr * (mom * Abuf + Agg)), Ea=Ebuf)
    elif kind in ("adam", "adamw"):
        b1, b2, eps = hp["b1"], hp["b2"], hp["eps"]
        if kind == "adamw":
            c = 1 - lr * wd
            p1, Ep1 = p * c, Ep * c + 3 * U * p.abs()
            gg, Egg = g, U * g.abs()
        else:
            p1, Ep1 = p, Ep
            gg = wd * p + g
            Egg = wd * Ep + 2 * U * ((wd * p).abs() + g.abs())
        mm = b1 * a + (1 - b1) * gg
        Emm = b1 * Ea + (1 - b1) * Egg + 2 * U * (b1 * a.abs() + (1 - b1) * gg.abs())
        vv = b2 * b + (1 - b2) * gg * gg
        Evv = b2 * Eb + (1 - b2) * 2 * gg.abs() * Egg + 3 * U * vv
        bc1, bc2s = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
        rb1, rb2 = _bc_rel(b1, t), 0.5 * _bc_rel(b2, t) + U
        sq = vv.sqrt()
        Esq = torch.minimum(Evv / (2 * sq).clamp_min(1e-300), Evv.sqrt()) + U * sq
        den = sq / bc2s + eps
        Eden = Esq / bc2s + (sq / bc2s) * (rb2 + U) + U * den
        r = mm / den
        Er = Emm / den + r.abs() * Eden / den + U * r.abs()
        d = (lr / bc1) * r
        Ed = (lr / bc1) * (Er + r.abs() * (rb1 + 2 * U))
        pn = p1 - d
        S.update(p=pn, a=mm, b=vv, Ep=Ep1 + Ed + U * (p1.abs() + d.abs()), Ea=Emm, Eb=Evv)
    else:
        alpha, eps = hp["alpha"], hp["eps"]
        gg = wd * p + g
        Egg = wd * Ep + 2 * U * ((wd * p).abs() + g.abs())
        s = a + (1 - alpha) * (gg * gg - a)
        Es = Ea + (1 - alpha) * 2 * gg.abs() * Egg + 3 * U * (a.abs() + gg * gg)
        avg = (s + eps).sqrt()
        Eavg = torch.minimum(Es / (2 * avg), Es.sqrt()) + 2 * U * avg
        q = lr * gg / avg
        Eq = lr * Egg / avg + q.abs() * Eavg / avg + 2 * U * q.abs()
        bn = mom * b + q
        Ebn = mom * Eb + Eq + U * (mom * b.abs() + q.abs())
        pn = p - bn
        S.update(p=pn, a=s, b=bn, Ep=Ep + Ebn + U * (p.abs() + bn.abs()), Ea=Es, Eb=Ebn)


@pytest.mark.parametrize("opt", UP.OPTS)
@pytest.mark.parametrize("dtype", UP.DTYPES)
@pytest.mark.parametrize("tag", TAGS)
def test_optimizer_at_arena_geometry(tag, dtype, opt):
    """three Trainer update phases over the whole arena (both ranges, one lr per group, the device lr / step counter / 1/scale
    / skip flag); under fp16 loss scaling the middle step meets a non-finite gradient and must change nothing"""
    e = _engine(tag, dtype)
    a = e.arena
    tr = UP.make_trainer(e, opt)
    o = tr.optimizer
    n, nd = a.n_params, a.n_decay
    dt = TDT[dtype]
    a.flags.zero_()
    gen = torch.Generator(device="cuda").manual_seed(5)
    a.params32.copy_(torch.randn(n, device="cuda", generator=gen) * 0.05)
    hp = dict(momentum=_f32(UP.HYPER["momentum"]), eps=_f32(UP.HYPER["eps"]), alpha=_f32(UP.HYPER["alpha"]),
              b1=_f32(0.9), b2=_f32(0.999))
    lr = {gi: _f32(g["lr"]) for gi, g in enumerate(o.param_groups)}
    wd = {gi: _f32(g["weight_decay"]) for gi, g in enumerate(o.param_groups)}
    rng = {0: (nd, n), 1: (0, nd)}
    assert o.param_groups[0]["_ranges"] == [rng[0]] and o.param_groups[1]["_ranges"] == [rng[1]] and wd[0] == 0 and wd[1] > 0
    z = torch.zeros(n, dtype=torch.float64, device="cuda")
    S = {gi: dict(p=a.params32[lo:hi].double(), a=o.state_a[lo:hi].double(),
                  b=(o.state_b[lo:hi].double() if o.state_b is not None else z[lo:hi].clone()),
                  Ep=z[lo:hi].clone(), Ea=z[lo:hi].clone(), Eb=z[lo:hi].clone()) for gi, (lo, hi) in rng.items()}
    scaled = dtype == "fp16"
    t = 0
    for step in range(3):
        skip = scaled and step == 1
        g = torch.randn(n, device="cuda", generator=gen) * 0.01
        inv = float(a.loss_scale_state[1]) if scaled else 1.0
        a.grads32.copy_(g / inv)                                       # the scaled gradient the backward leaves behind
        if skip:
            a.grads32[int(torch.randint(n, (1,), generator=gen, device="cuda"))] = float("inf")
            before = [t_.clone() for t_ in (a.params32, o.state_a, a.params16, o.step_dev)] + \
                     ([o.state_b.clone()] if o.state_b is not None else [])
        o.push_hyper()
        tr._launch_step(False, "back")
        torch.cuda.synchronize()
        if skip:
            after = [a.params32, o.state_a, a.params16, o.step_dev] + ([o.state_b] if o.state_b is not None else [])
            for x, y in zip(before, after):
                assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x, y.view(torch.int32) if y.dtype == torch.float32 else y)
            assert float(a.loss_scale_state[0]) == 32768.0 and int(a.flags[0]) == 0
            continue
        t += 1
        gd = a.grads32.double() * inv
        for gi, (lo, hi) in rng.items():
            _ref_step(o.kind, S[gi], gd[lo:hi], lr[gi], wd[gi], t, hp)
    if o.kind in ("adam", "adamw"):
        assert int(o.step_dev) == t
    assert torch.equal(_bits(a.params16), _bits(a.params32.to(dt)))
    for gi, (lo, hi) in rng.items():
        R = S[gi]
        for name, got, key in (("p", a.params32[lo:hi], "p"), ("state_a", o.state_a[lo:hi], "a")) + \
                ((("state_b", o.state_b[lo:hi], "b"),) if o.state_b is not None else ()):
            err = (got.double() - R[key]).abs()
            bound = 2 * R["E" + key]
            bad = err > bound
            assert not bool(bad.any()), "%s group %d: %d elements out of bound, worst err %.3e at %d (bound %.3e)" % (
                name, gi, int(bad.sum()), float(err.max()), int((err - bound).argmax()), float(bound[(err - bound).argmax()]))
        # the bound is tight enough that a range updated with the other group's lr or weight decay falls outside it
        assert float(R["Ep"].max()) < 1e-3 * float(R["p"].abs().max())


# ---- loss scaling ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", TAGS)
def test_check_finite_full_arena(tag):
    a = _engine(tag, "fp16").arena
    n, nd = a.n_params, a.n_decay
    gen = torch.Generator(device="cpu").manual_seed(3)
    a.grads32.copy_(torch.randn(n, device="cuda") * 1e3)
    flag = a.flags[0:1]
    flag.zero_()
    _lib.call("dfd_check_finite", _ptr(a.grads32), n, _ptr(a.flags, 0), st())
    torch.cuda.synchronize()
    assert int(flag) == 0
    idx = [0, n - 1, int(torch.randint(0, nd, (1,), generator=gen)), int(torch.randint(nd, n, (1,), generator=gen))]
    for bad in (float("inf"), float("-inf"), float("nan")):
        for i in idx:
            keep = a.grads32[i].clone()
            a.grads32[i] = bad
            _lib.call("dfd_check_finite", _ptr(a.grads32), n, _ptr(a.flags, 0), st())
            torch.cuda.synchronize()
            assert int(flag) == 1, (bad, i)
            flag.zero_()
            a.grads32[i] = keep
    a.grads32[n // 2] = 3.4e38                        # finite but above the 3e38 overflow threshold
    _lib.call("dfd_check_finite", _ptr(a.grads32), n, _ptr(a.flags, 0), st())
    torch.cuda.synchronize()
    assert int(flag) == 1
    flag.zero_()


def test_update_loss_scale_contract():
    """halve on overflow (floor 1), double after `interval` clean steps (cap 2^24), clear the flag, write 1/scale"""
    flags = torch.zeros(2, dtype=torch.int32, device="cuda")
    state = torch.zeros(2, dtype=torch.float32, device="cuda")
    for interval, scale0, good0, script in (
            (2000, 65536.0, 1997, [0, 0, 0, 0, 1, 0, 0]),                     # doubling at the Trainer's interval
            (3, 4.0, 0, [1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 0]),                # floor at 1, then doubling again
            (2, 2.0 ** 23, 0, [0, 0, 0, 0, 0, 0, 1, 0, 0])):                   # cap at 2^24
        state.copy_(torch.tensor([scale0, 0.0]))
        flags.copy_(torch.tensor([0, good0], dtype=torch.int32))
        scale, good = torch.tensor(scale0, dtype=torch.float32), good0
        for f in script:
            flags[0] = f
            _lib.call("dfd_update_loss_scale", _ptr(flags, 0), _ptr(state, 0), _ptr(flags, 1), interval, _ptr(state, 1), st())
            if f:
                scale, good = torch.clamp(scale * 0.5, min=1.0), 0
            else:
                good += 1
                if good >= interval:
                    scale, good = torch.clamp(scale * 2.0, max=2.0 ** 24), 0
            s = state.cpu()
            fl = flags.cpu()
            assert float(s[0]) == float(scale) and int(fl[1]) == good and int(fl[0]) == 0, (interval, f, s, fl)
            assert float(s[1]) == float(1.0 / scale)


@pytest.mark.parametrize("opt", ("adam", "sgd"))
def test_fp16_graph_skips_overflow_and_resumes(opt):
    """an fp16 Trainer replaying its captured step meets an overflow: weights, optimizer state, p16 and Adam's step counter stay
    bit-identical, the scale halves; the next clean replay applies"""
    from deepfake_detection_b200.trainer import Trainer
    from oracle.weights import synth_batch, synth_state
    from deepfake_detection_b200.arch import get_spec
    tr = Trainer("efficientnet_b0", 8, 96, 96, dtype="fp16", opt=opt, lr=0.01, use_graph=True)
    tr.load_state_dict(synth_state(get_spec("efficientnet_b0"), seed=7))
    x, y = synth_batch(8, 3, 96, 96, seed=1)
    x, y = x.cuda(), y.cuda()
    e, o = tr.engine, tr.optimizer
    for _ in range(2):
        tr.train_step(x, y)
    torch.cuda.synchronize()

    def snap():
        return [t.clone() for t in (e.params32, o.state_a, e.params16, e.paramsT16, o.step_dev)] + \
               ([o.state_b.clone()] if o.state_b is not None else [])
    before = snap()
    e.loss_scale_state.copy_(torch.tensor([3.0e38, 1.0 / 3.0e38]))       # the backward overflows
    tr.train_step(x, y)
    torch.cuda.synchronize()
    assert tr.n_captures == 1
    for u, v in zip(before, snap()):
        assert torch.equal(u.view(torch.int16) if u.element_size() == 2 else u, v.view(torch.int16) if v.element_size() == 2 else v)
    assert float(e.loss_scale_state[0]) == _f32(3.0e38) / 2 and int(e.flags[0]) == 0 and int(e.flags[1]) == 0
    e.loss_scale_state.copy_(torch.tensor([1024.0, 1.0 / 1024.0]))
    tr.train_step(x, y)
    torch.cuda.synchronize()
    assert not torch.equal(e.params32, before[0]) and int(e.flags[1]) == 1
    if opt == "adam":
        assert int(o.step_dev) == int(before[4]) + 1
    assert torch.equal(_bits(e.params16), _bits(e.params32.half())) and tr.n_captures == 1


# ---- EMA ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", TAGS)
def test_ema_at_arena_size(tag):
    """ModelEma.update over whole arenas: params and running statistics per element against fp64 ema*d + (1-d)*model within
    the two roundings of the kernel, the int64 num_batches_tracked exactly as the reference's float arithmetic truncates them"""
    src = _engine(tag, "bf16").arena
    dst = UP.arena(tag, "bf16")
    gen = torch.Generator(device="cuda").manual_seed(9)
    decay = 0.9998
    for t in (src.params32, dst.params32, src.buffers32, dst.buffers32):
        t.copy_(torch.randn(t.numel(), device="cuda", generator=gen))
    nb = src.nbt.numel()
    src.nbt.copy_(torch.randint(3, 300000, (nb,), device="cuda", generator=gen))
    dst.nbt.copy_(src.nbt - torch.randint(0, 3, (nb,), device="cuda", generator=gen))
    dst.nbt[:3] = src.nbt[:3]
    before = [t.clone() for t in (dst.params32, dst.buffers32, dst.nbt)]
    UP.ema_update(dst, src, decay)
    torch.cuda.synchronize()
    d = _f32(decay)
    for got, e0, m in ((dst.params32, before[0], src.params32), (dst.buffers32, before[1], src.buffers32)):
        ref = e0.double() * d + (1 - d) * m.double()
        bound = 3 * U * (e0.double().abs() * d + (1 - d) * m.double().abs())
        assert bool(((got.double() - ref).abs() <= bound).all())
    ref_nbt = (before[2].cpu() * decay + (1. - decay) * src.nbt.cpu()).long()      # dfd/timm/utils.py:336-340, on int64
    assert torch.equal(dst.nbt.cpu(), ref_nbt)


# ---- a later plan over the same arena (the captured step's lifecycle) -----------------------------------------------------
def _eval_logits(e, x):
    s = st()
    e.set_input(x)
    e.zero_step_scratch(s, grads=False)
    e.forward(training=False, stream=s)
    e.head(False, stream=s)
    torch.cuda.synchronize()
    return e.logits.clone()


@pytest.mark.parametrize("dtype", UP.DTYPES)
def test_captured_step_after_a_later_plan(dtype):
    """B0 at 98x98: a batch-6 plan needs pack-2 block-diagonal copies where batch 8 uses pack 4. Built between replays, it must
    make the captured step re-capture: every layout is refreshed at the next steps and the batch-6 plan evaluates the trained
    weights exactly as a freshly built model does"""
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.trainer import Trainer
    from oracle.weights import synth_batch, synth_state
    tr = Trainer("efficientnet_b0", 8, 98, 98, dtype=dtype, lr=0.05, use_graph=True)
    tr.load_state_dict(synth_state(get_spec("efficientnet_b0"), seed=7))
    x, y = synth_batch(8, 3, 98, 98, seed=2)
    x, y = x.cuda(), y.cuda()
    for _ in range(2):
        tr.train_step(x, y)
    n_before = len(tr.engine._bd_reg)
    e6 = Engine("efficientnet_b0", 6, 98, 98, dtype=dtype, share_from=tr.engine)
    assert len(tr.engine._bd_reg) > n_before
    for _ in range(2):
        tr.train_step(x, y)
    torch.cuda.synchronize()
    assert tr.n_captures == 2
    check_derived_layouts(tr.engine)
    x6 = x[:6].to(e6.tdtype)
    got = _eval_logits(e6, x6)
    fresh = Engine("efficientnet_b0", 6, 98, 98, dtype=dtype)
    fresh.load_state_dict(tr.state_dict())
    assert torch.equal(got, _eval_logits(fresh, x6))


def test_runner_validate_between_epochs():
    """the runner's flow: fused train_epoch at batch 8, validate at batch 6 (a new plan over the shared arena), train_epoch,
    validate; the layouts of the model and of its EMA stay exact and the captured step re-captured once"""
    from types import SimpleNamespace
    from deepfake_detection_b200 import loss as NL
    from deepfake_detection_b200.ema import ModelEma
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch, validate
    from oracle.weights import synth_batch, synth_state
    from deepfake_detection_b200.arch import get_spec

    class Loader(list):
        mixup_enabled = False

    args = SimpleNamespace(opt="sgd", lr=0.05, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0,
                           mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0,
                           log_interval=1, recovery_interval=0, tta=0)
    model = create_model("efficientnet_b0", num_classes=2, dtype="bf16")
    model.load_state_dict(synth_state(get_spec("efficientnet_b0"), seed=7))
    opt = create_optimizer(args, model)
    ema = ModelEma(model, decay=0.9)
    train = Loader((x.cuda(), y.cuda()) for x, y in (synth_batch(8, 3, 98, 98, seed=40 + i) for i in range(2)))
    val = Loader((x.cuda(), y.cuda()) for x, y in (synth_batch(6, 3, 98, 98, seed=50 + i) for i in range(2)))
    for epoch in range(2):
        train_epoch(epoch, model, train, opt, NL.CrossEntropyLoss(), args, model_ema=ema)
        validate(model, val, torch.nn.CrossEntropyLoss(), args)
        validate(ema.ema, val, torch.nn.CrossEntropyLoss(), args, log_suffix=" (EMA)")
    torch.cuda.synchronize()
    (tr,) = model.__dict__["_trainers"].values()
    assert tr.n_captures == 2
    check_derived_layouts(model.engine)
    check_derived_layouts(ema.ema.engine)
    assert len(ema.ema.engine._bd_reg) > 0
