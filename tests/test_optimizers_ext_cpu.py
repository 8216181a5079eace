"""radam / adadelta / rmsprop / novograd / nvnovograd without a GPU: the CPU restatement (tests/optim_ext_oracle.py) against
the fixtures minted from the unmodified reference (tools/mint_optimizer_goldens.py), the factory's names, groups and decay
rules on the native optimizer, and the C-ABI launches of each kind's update phase on plan-only engines of every shipped
configuration."""
import json
import os
from types import SimpleNamespace

import pytest
import torch

import optim_ext_oracle as OX
import plan_launches as PL
import update_phase as UP
from deepfake_detection_b200 import _lib
from deepfake_detection_b200.arch import get_spec
from deepfake_detection_b200.optim import LW_CHUNK, ArenaOptimizer, create_optimizer
from oracle import train as OT
from oracle.weights import synth_batch, synth_state

RTOL = 2e-4
KINDS = OX.KINDS
STEP_KERNEL = {"radam": "dfd_radam_step", "adadelta": "dfd_adadelta_step", "rmsprop": "dfd_rmsprop_step",
               "novograd": "dfd_novograd_step", "nvnovograd": "dfd_nvnovograd_step"}


def _toy():
    g0 = torch.Generator().manual_seed(3)
    return {"w": torch.randn(5, 7, generator=g0), "bias": torch.randn(7, generator=g0), "k": torch.randn(4, 1, 3, 3, generator=g0)}


def _toy_grads(step, gen):
    out = {n: torch.randn(s, generator=gen) for n, s in (("w", (5, 7)), ("bias", (7,)), ("k", (4, 1, 3, 3)))}
    if step == 0:
        out["k"] = out["k"] * 0
    return out


def _run_oracle(r):
    kind = r["kind"]
    wd = r["weight_decay"] / r["lr"] if kind == "radam" else r["weight_decay"]
    opt = OX.OptState(kind, lr=r["lr"], momentum=r["momentum"], weight_decay=wd, eps=r["eps"],
                      single_group=not r["filter_bias_and_bn"])
    params = _toy()
    gen = torch.Generator().manual_seed(11)
    for step, lrs in enumerate(r["lrs"]):
        # group 0 = [bias] (no decay), group 1 = [w, k]; one group when the factory did not split
        by_name = {"bias": lrs[0], "w": lrs[-1], "k": lrs[-1]}
        opt.lr, opt.lr_nodecay = lrs[-1], lrs[0]
        OX.optimizer_step(opt, params, _toy_grads(step, gen), lrs=by_name)
        yield step, params, opt


@pytest.mark.parametrize("run", list(KINDS) + ["novograd_single", "radam_group_lrs"])
def test_oracle_matches_reference_optimizers(run, golden_dir):
    r = json.load(open(os.path.join(golden_dir, "optimizers_ext.json")))[run]
    # NovoGrad's ||ghat||^2 is the reference's own second norm here (the device forms it from ||g||^2): same arithmetic
    for step, params, opt in _run_oracle(r):
        for k, p in params.items():
            ref = torch.tensor(r["hist"][step][k])
            assert torch.allclose(p.reshape(-1), ref, rtol=RTOL, atol=RTOL * float(ref.abs().max())), (run, step, k)
    assert len(r["hist"]) >= 8
    # the final state, key for key, against the reference's state_dict
    for name, st in r["state"].items():
        for key, v in st.items():
            if key == "step":                    # an int, or a 0-d tensor for the torch.optim classes
                assert (v if isinstance(v, int) else int(v[0])) == len(r["hist"]), (run, key)
                continue
            ref = torch.tensor(v, dtype=torch.float32).reshape(-1)
            got = opt.state[name][key].reshape(-1).float()
            assert torch.allclose(got, ref, rtol=RTOL, atol=RTOL * float(ref.abs().max()) + 1e-12), (run, name, key)


def test_reference_decay_rules(golden_dir):
    rec = json.load(open(os.path.join(golden_dir, "optimizers_ext.json")))
    assert rec["novograd"]["ctor_weight_decay"] == 0.0 and rec["novograd"]["group_weight_decay"] == [0.0, 1e-2]
    assert rec["novograd_single"]["ctor_weight_decay"] == 1e-2 and rec["novograd_single"]["group_sizes"] == [3]
    assert rec["radam"]["group_weight_decay"] == [0.0, pytest.approx(1e-2 / 1e-2)]       # divided by the initial lr
    assert rec["nvnovograd"]["state"]["k"]["exp_avg_sq"] != [0.0]                        # the zero-gradient start was left


@pytest.mark.parametrize("case", ["step_efficientnet_b0_radam", "step_resnet18_nvnovograd"])
def test_oracle_train_steps_match_reference(case, golden_dir):
    from test_oracle_vs_reference_goldens import _check_summ
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    torch.set_num_threads(8)
    spec = get_spec(rec["arch"], num_classes=rec["num_classes"])
    sd = synth_state(spec, seed=rec["weight_seed"])
    wd = rec["weight_decay"] / rec["lr"] if rec["opt"] == "radam" else rec["weight_decay"]
    opt = OX.OptState(rec["opt"], lr=rec["lr"], momentum=rec["momentum"], weight_decay=wd, eps=1e-8)
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i, num_classes=rec["num_classes"])
        out = OX.train_step(spec, sd, x, y, opt)
        assert float(out["loss"]) == pytest.approx(st["loss"], rel=1e-4)
        rt = RTOL * (1 if i == 0 else 25)
        gfloor = 1e-5 * max(v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 for k, v in st["grads"].items())
        for k, s in st["grads"].items():
            _check_summ(out["grads"][k], s, "grad %s step %d" % (k, i), rt, floor=gfloor)
        # an adaptive optimizer turns a round-off gradient into an O(lr) update in both implementations: no parity there
        noise = {k for k, v in st["grads"].items() if v["norm"] / max(out["grads"][k].numel(), 1) ** 0.5 < 10 * gfloor}
        for k, s in st["params"].items():
            if k not in noise:
                _check_summ(sd[k], s, "param %s step %d" % (k, i), rt)


# ---- the factory on the native optimizer ---------------------------------------------------------------------------------
def _arena(arch="efficientnet_b0"):
    from deepfake_detection_b200.engine import Engine
    return Engine(arch, 1, device="plan-only", params_only=True)


def _args(opt, **kw):
    d = dict(opt=opt, lr=1e-2, momentum=0.9, weight_decay=1e-4, opt_eps=1e-3)
    d.update(kw)
    return SimpleNamespace(**d)


@pytest.mark.parametrize("kind", KINDS)
def test_factory_groups_and_decay(kind):
    a = _arena()
    o = create_optimizer(_args(kind.upper() if kind == "radam" else kind), a)
    assert o.kind == kind and [len(g["_ranges"]) for g in o.param_groups] == [1, 1]
    wd = o.param_groups[1]["weight_decay"]
    assert o.param_groups[0]["weight_decay"] == 0.0
    assert wd == pytest.approx(1e-4 / 1e-2 if kind == "radam" else 1e-4)        # optim_factory.py:29-33
    assert all(g["eps"] == 1e-3 for g in o.param_groups)
    if kind in ("novograd", "nvnovograd"):
        assert o.param_groups[0]["betas"] == (0.95, 0.98)
        assert o.lw_nchunks == sum(-(-k // LW_CHUNK) for _, _, k in a.p_off.values())
        assert sum(o.lw_range_chunks[r][1] for r in o.lw_range_chunks) == o.lw_nchunks
    if kind == "novograd":
        assert o.novograd_wd == 0.0                                                 # the factory split the groups
    assert (o.state_b is None) == (kind in ("novograd", "nvnovograd"))
    single = create_optimizer(_args(kind), a, filter_bias_and_bn=False)
    assert len(single.param_groups) == 1 and single.param_groups[0]["weight_decay"] == wd
    if kind == "novograd":
        assert single.novograd_wd == pytest.approx(1e-4)
    none = create_optimizer(_args(kind, weight_decay=0.0), a)
    assert len(none.param_groups) == 1 and none.param_groups[0]["weight_decay"] == 0.0


def test_rmsprop_without_momentum_has_no_buffer():
    o = create_optimizer(_args("rmsprop", momentum=0.0), _arena())
    assert o.state_b is None and "momentum_buffer" not in o.state_dict()["state"][0]


@pytest.mark.parametrize("bad", ["nadam", "lookahead_radam", "lookahead_novograd", "lookahead_sgd", "fusedsgd", "fusedadam",
                                 "fusedlamb", "fusednovograd", "adagrad"])
def test_still_refused(bad):
    with pytest.raises(ValueError) as ex:
        create_optimizer(_args(bad), _arena())
    assert "radam" in str(ex.value) and "nvnovograd" in str(ex.value)


def test_state_dict_keys_and_types():
    """the reference's state keys, shapes and types (0-d `step` tensors for the torch.optim classes)"""
    a = _arena()
    keys = {"radam": {"step", "exp_avg", "exp_avg_sq"}, "adadelta": {"step", "square_avg", "acc_delta"},
            "rmsprop": {"step", "square_avg", "momentum_buffer"}, "novograd": {"step", "v", "m", "grad_ema"},
            "nvnovograd": {"step", "exp_avg", "exp_avg_sq"}}
    for kind in KINDS:
        sd = create_optimizer(_args(kind), a).state_dict()
        names = [n for g in create_optimizer(_args(kind), a).param_groups for n in g["params"]]
        for i, st in sd["state"].items():
            assert set(st) == keys[kind], kind
            shape = a.p_off[names[i]][1]
            for k, v in st.items():
                if k == "step":
                    assert (torch.is_tensor(v) and v.dim() == 0) == (kind in ("adadelta", "rmsprop")), kind
                elif k in ("v", "grad_ema") or (kind == "nvnovograd" and k == "exp_avg_sq"):
                    assert v.dim() == 0, (kind, k)
                else:
                    assert tuple(v.shape) == shape, (kind, k)


def test_hyper_signature():
    a = _arena()
    for kind in KINDS:
        o = create_optimizer(_args(kind), a)
        sig = o.hyper_signature()
        o.param_groups[0]["lr"] = 0.5
        assert o.hyper_signature() == sig                    # the lr is read from the device
        o.param_groups[1]["eps"] = 0.5
        assert o.hyper_signature() != sig
    o = create_optimizer(_args("adadelta"), a)
    sig = o.hyper_signature()
    o.param_groups[0]["rho"] = 0.5
    assert o.hyper_signature() != sig
    o = create_optimizer(_args("novograd"), a)
    sig = o.hyper_signature()
    o.novograd_wd = 0.1
    assert o.hyper_signature() != sig


# ---- the launches of the update phase ---------------------------------------------------------------------------------
def _record(monkeypatch, tag, dtype, opt):
    """the C-ABI calls of one Trainer update phase (lr push, finite check, optimizer, loss scale, refresh)"""
    calls = []
    monkeypatch.setattr(_lib, "call", lambda name, *args: calls.append(PL._split(name, args[:-1])))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: SimpleNamespace(cuda_stream=0))
    tr = UP.make_trainer(UP.engine(tag, dtype, device="plan-only"), opt)
    tr.optimizer.push_hyper()
    tr._launch_step(False, "back")
    monkeypatch.undo()
    return calls, tr


@pytest.mark.parametrize("tag", [t for t, *_ in PL.CONFIGS])
def test_update_launches_of_every_kind(monkeypatch, tag):
    """one update launch per arena range with the Trainer's pointers: gscale_dev and skip under loss scaling only; the step
    counter ticks for every kind; the layer-wise kinds add one norm and one per-tensor launch, whose table covers the arena"""
    for dtype in UP.DTYPES:
        scaled = "pp" if dtype == "fp16" else "00"
        for kind in KINDS:
            calls, tr = _record(monkeypatch, tag, dtype, kind)
            names = [c.kernel for c in calls]
            step = [c for c in calls if c.kernel == STEP_KERNEL[kind]]
            ptrs = {"radam": "pppp" + scaled + "pppp", "adadelta": "pppp" + scaled + "pp", "rmsprop": "pppp" + scaled + "pp",
                    "novograd": "pppppp" + scaled + "ppp", "nvnovograd": "ppppp" + scaled + "pp"}[kind]
            assert [c.ptrs for c in step] == [ptrs, ptrs], (tag, dtype, kind, [c.ptrs for c in step])
            assert names.count("dfd_opt_tick") == 1 and names.index("dfd_opt_tick") < names.index(STEP_KERNEL[kind])
            assert ("dfd_check_finite" in names) == (dtype == "fp16")
            o = tr.optimizer
            e = tr.engine
            if kind in ("novograd", "nvnovograd"):
                (norm,) = [c for c in calls if c.kernel == "dfd_tensor_sumsq"]
                assert norm.ptrs == "ppppp" + scaled
                assert norm.shape[0] == o.lw_nchunks and norm.shape[1] == len(e.p_off)
                prep = "dfd_novograd_prepare" if kind == "novograd" else "dfd_nvnovograd_prepare"
                assert names.count(prep) == 1 and names.index("dfd_tensor_sumsq") < names.index(prep) < \
                    names.index(STEP_KERNEL[kind])
                # the chunk counts of the two ranges cover the table, decay range first
                assert [c.shape[0] for c in step] == [o.lw_range_chunks[(e.n_decay, e.n_params)][1],
                                                      o.lw_range_chunks[(0, e.n_decay)][1]]
                raw = o.lw_table.numpy().view("<i8").reshape(-1, 2)
                offs, lens, ts = raw[:, 0], raw[:, 1] & 0xFFFFFFFF, raw[:, 1] >> 32
                assert int(lens.max()) <= LW_CHUNK and int(lens.sum()) == sum(k for _, _, k in e.p_off.values())
                for t, (name, (off, _, k)) in enumerate(e.p_off.items()):
                    sel = ts == t
                    assert int(offs[sel].min()) == off and int((offs[sel] + lens[sel]).max()) == off + k, name
            else:
                assert "dfd_tensor_sumsq" not in names
                assert [c.shape[0] for c in step] == [e.n_params - e.n_decay, e.n_decay]


def test_existing_kinds_launch_as_before(monkeypatch):
    """sgd / adam / adamw / rmsproptf: no layer-wise launches, the tick only for Adam"""
    for kind in UP.OPTS:
        calls, _ = _record(monkeypatch, "b0", "bf16", kind)
        names = [c.kernel for c in calls]
        assert "dfd_tensor_sumsq" not in names and ("dfd_opt_tick" in names) == (kind in ("adam", "adamw"))


def test_oracle_keeps_the_original_kinds():
    """optim_ext_oracle.optimizer_step hands the four original kinds to oracle.train unchanged"""
    params = _toy()
    ref = {k: v.clone() for k, v in params.items()}
    g = _toy_grads(1, torch.Generator().manual_seed(1))
    OX.optimizer_step(OT.OptState(kind="adamw", lr=1e-2, weight_decay=1.0), params, g)
    OT.optimizer_step(OT.OptState(kind="adamw", lr=1e-2, weight_decay=1.0), ref, g)
    assert all(torch.equal(params[k], ref[k]) for k in params)


def test_arena_optimizer_default_betas_unchanged():
    a = _arena()
    for kind in ("adam", "adamw", "radam"):
        assert ArenaOptimizer(a, opt=kind).param_groups[0]["betas"] == (0.9, 0.999)
