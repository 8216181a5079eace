"""CPU: ResNet DropBlock / drop path / dropout.

The drop oracle (tests/resnet_drop_oracle.py) is oracle.train bit for bit when no mask is given, reproduces the reference's
drop_block_2d exactly (including the scrambled valid region of non-square maps and negative gamma), and is held to train
steps minted from the unmodified reference with its recorded masks. The plan-only engines: all rates 0 is today's plan;
rates > 0 add the mask generators and switch exactly the DropBlock sites and block tails to the masked kernels; the shapes on
which the reference's DropBlock fails are refused."""
import base64
import json
import os
import zlib

import numpy as np
import pytest
import torch

from deepfake_detection_b200.arch import get_spec, param_entries
from deepfake_detection_b200.engine import Engine
from oracle import train as OT
from oracle.weights import synth_batch, synth_state

import resnet_drop_oracle as RO

RATES = dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.2)
NEW_OPS = {"dfd_drop_block_masks_train", "dfd_memset_async_train", "dfd_rng_masks_train", "dfd_rng_tick_train",
           "dfd_mul_f32_train", "dfd_mul_f32", "dfd_bn_act_drop", "dfd_act_bwd_drop", "dfd_relu_bn_bwd_reduce_drop"}


def _f32(s):
    return torch.from_numpy(np.frombuffer(base64.b64decode(s), dtype="<f4").copy())


def _idx(s):
    return torch.from_numpy(np.frombuffer(zlib.decompress(base64.b64decode(s)), dtype="<i4").astype(np.int64)).cumsum(0)


def _zeros_mask(shape, packed):
    m = torch.ones(int(np.prod(shape)))
    m[_idx(packed)] = 0.0
    return m.view(shape)


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
def test_no_mask_is_oracle_train_bit_for_bit(arch):
    spec = get_spec(arch)
    sd0 = synth_state(spec, seed=7)
    x, y = synth_batch(2, 3, 64, 64, seed=1234)
    for adt in (None, torch.bfloat16):
        a = {k: v.clone() for k, v in sd0.items()}
        b = {k: v.clone() for k, v in sd0.items()}
        oa = OT.train_step(spec, a, x, y, OT.OptState(kind="sgd", lr=0.01), act_dtype=adt)
        ob = RO.train_step(spec, b, x, y, OT.OptState(kind="sgd", lr=0.01), act_dtype=adt)
        assert torch.equal(oa["logits"], ob["logits"]) and torch.equal(oa["loss"], ob["loss"])
        assert all(torch.equal(oa["grads"][n], ob["grads"][n]) for n in oa["grads"])
        assert all(torch.equal(a[n], b[n]) for n in a)


def test_drop_block_formulas_reproduced_exactly(golden_dir):
    rec = json.load(open(os.path.join(golden_dir, "drop_block_formulas.json")))
    n_neg = n_dropped = 0
    for c in rec["cases"]:
        H, W = c["H"], c["W"]
        shape = rec["shape"] + [H, W]
        x, u, out = _f32(c["x"]).view(shape), _f32(c["noise"]).view(shape), _f32(c["out"]).view(shape)
        gamma, cb = RO.drop_block_gamma(H, W, c["drop_prob"], c["gamma_scale"], c["block_size"])
        m = RO.block_from_seeds(RO.seeds_from_noise(u, gamma, cb), cb)
        assert torch.equal(RO.drop_block_apply(x, m), out), (H, W, c["gamma_scale"])
        n_neg += gamma < 0
        n_dropped += bool((m == 0).any())
        if gamma < 0:
            assert torch.equal(out, x * (m.numel() / (m.sum() + 1e-7)))       # nothing dropped
    assert n_neg == 2 and n_dropped >= 4          # 5 x 7 at both gamma scales
    # the non-square valid region is the reference's scrambled one, not the centred rectangle
    v = RO.valid_block(10, 14, 7)[0, 0]
    centred = torch.zeros(10, 14)
    centred[3:7, 3:11] = 1
    assert not torch.equal(v, centred) and int(v.sum()) == int(centred.sum())


def _check_summ(t, s, rtol, what):
    f = t.detach().reshape(-1).double()
    assert abs(float(f.norm()) - s["norm"]) <= rtol * abs(s["norm"]) + 1e-7 * f.numel() ** 0.5, what + " norm"
    got = f[torch.tensor(s["idx"])]
    ref = torch.tensor(s["samples"], dtype=torch.float64)
    assert float((got - ref).abs().max()) <= rtol * (float(ref.abs().max()) + abs(s["norm"]) / f.numel() ** 0.5) + 1e-7, what


@pytest.mark.parametrize("case", ["step_resnet18_drop_160", "step_resnet18_drop_160x224", "step_resnet50_drop_160"])
def test_drop_oracle_matches_reference_steps(case, golden_dir):
    """the reference's recorded masks through the drop oracle: step 0 on logits, loss, gradients and updated values, step 1
    (after an update) on the loss. The reference's drop path divides by keep where the oracle (and the native path)
    multiplies by a mask holding 1 / keep; that last-bit difference is amplified on the way back through ResNet-50's 16
    Bottlenecks (loss and classifier gradients agree to 1e-6, the stem gradient to 0.6 %), hence its looser gradient bound"""
    rec = json.load(open(os.path.join(golden_dir, case + ".json")))
    spec = get_spec(rec["arch"])
    sd = synth_state(spec, seed=rec["weight_seed"])
    ost = OT.OptState(kind="sgd", lr=rec["lr"], momentum=rec["momentum"], weight_decay=rec["weight_decay"])
    for i, st in enumerate(rec["steps"]):
        x, y = synth_batch(rec["batch"], 3, rec["H"], rec["W"], seed=1234 + i)
        db = {}
        for name, d in st["drop_block"].items():
            H, W = d["shape"][-2:]
            gs = 0.25 if name.startswith("layer3") else 1.0
            _, cb = RO.drop_block_gamma(H, W, rec["drop_block_rate"], gs)
            db[name] = RO.block_from_seeds(_zeros_mask(d["shape"], d["zeros"]), cb)
        dp = {k: torch.tensor(v) for k, v in st["drop_masks"].items()}
        dm = _zeros_mask(st["dropout_shape"], st["dropout_zeros"]) / (1.0 - rec["drop_rate"])
        out = RO.train_step(spec, sd, x, y, ost, drop_block=db, drop_masks=dp, dropout_mask=dm)
        assert abs(float(out["loss"]) - st["loss"]) < (1e-4 if i == 0 else 2e-2) * max(1.0, abs(st["loss"])), (i, float(out["loss"]))
        if i == 0:
            _check_summ(out["logits"], st["logits"], 1e-3, "logits")
            for k, s in st["grads"].items():
                _check_summ(out["grads"][k], s, 2e-3 if rec["arch"] == "resnet18" else 1e-2, "grad " + k)
            for k, s in st["params"].items():
                _check_summ(sd[k], s, 1e-4 if rec["arch"] == "resnet18" else 1e-2, "param " + k)


def _ops(e):
    return [n for _, n, _ in e.fwd_ops], [n for _, n, _ in e.bwd_ops]


@pytest.mark.parametrize("arch,n_sites", [("resnet18", 8), ("resnet50", 27)])
def test_plans(arch, n_sites):
    base = Engine(arch, 4, 224, 224, device="plan-only")
    f0, b0 = _ops(base)
    assert not (set(f0) | set(b0)) & NEW_OPS
    for kw in (dict(drop_rate=0.0, drop_path_rate=0.0, drop_block_rate=0.0), dict(drop_block_rate=None)):
        assert _ops(Engine(arch, 4, 224, 224, device="plan-only", **kw)) == (f0, b0)
    e = Engine(arch, 4, 224, 224, device="plan-only", **RATES)
    f1, b1 = _ops(e)
    spec = get_spec(arch)
    assert len(e.drop_block_masks) == n_sites and list(e.drop_masks) == [b.name for b in spec.blocks]
    assert all(s.split(".")[0] in ("layer3", "layer4") for s in e.drop_block_masks)
    assert f1[:4] == ["dfd_memset_async_train", "dfd_drop_block_masks_train", "dfd_rng_masks_train", "dfd_rng_tick_train"]
    assert f1.count("dfd_bn_act_drop") == n_sites and f1.count("dfd_mul_f32_train") == 1 and b1.count("dfd_mul_f32") == 1
    assert b1.count("dfd_relu_bn_bwd_reduce_drop") == len(spec.blocks)
    assert b1.count("dfd_act_bwd_drop") == n_sites - sum(1 for b in spec.blocks if b.name.split(".")[0] in ("layer3", "layer4"))
    # the rest of the plan is unchanged: the masked kernels take the place of their plain forms, no pass is added
    plain = {"dfd_bn_act_drop": "dfd_bn_act", "dfd_act_bwd_drop": "dfd_act_bwd", "dfd_relu_bn_bwd_reduce_drop": "dfd_relu_bn_bwd_reduce"}
    strip = lambda ops: [plain.get(n, n) for n in ops if n not in ("dfd_memset_async_train", "dfd_drop_block_masks_train",
                                                                    "dfd_rng_masks_train", "dfd_rng_tick_train",
                                                                    "dfd_mul_f32_train", "dfd_mul_f32")]
    assert strip(f1) == f0 and strip(b1) == b0
    # drop path alone: the gate goes through dfd_bn_act's (gate, residual + ReLU) form, no DropBlock site
    d = Engine(arch, 4, 160, 160, device="plan-only", drop_path_rate=0.1)
    fd, bd = _ops(d)
    assert "dfd_drop_block_masks_train" not in fd and not d.drop_block_masks and "dfd_bn_act_drop" not in fd
    assert bd.count("dfd_relu_bn_bwd_reduce_drop") == len(spec.blocks)


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
def test_drop_block_shapes(arch):
    """the reference's DropBlock divides by zero at (W-6)(H-6) == 0 and fails on an even clipped block size"""
    for res in (64, 96, 192):
        with pytest.raises(ValueError, match="DropBlock at layer"):
            Engine(arch, 2, res, res, device="plan-only", drop_block_rate=0.1)
        Engine(arch, 2, res, res, device="plan-only", drop_rate=0.1, drop_path_rate=0.1)     # no DropBlock: no limit
    for res in (160, 224):
        Engine(arch, 2, res, res, device="plan-only", drop_block_rate=0.1)
    e = Engine(arch, 2, 160, 224, device="plan-only", drop_block_rate=0.1)
    gam = {k: v[3] for k, v in e.drop_block_sites.items()}
    assert all(g < 0 for k, g in gam.items() if e.drop_block_sites[k][:2] == (5, 7))     # (7-6)(5-6) < 0, nothing dropped
    assert all(g > 0 for k, g in gam.items() if e.drop_block_sites[k][:2] == (10, 14))


def test_factory_accepts_the_rates():
    from deepfake_detection_b200.models import create_model
    import copy
    m = create_model("resnet50", num_classes=2, **RATES)
    assert (m.drop_rate, m.drop_path_rate, m.drop_block_rate) == (0.2, 0.1, 0.2)
    kw = m._engine_kwargs()
    assert kw["drop_block_rate"] == 0.2 and kw["drop_path_rate"] == 0.1 and kw["drop_rate"] == 0.2
    assert create_model("resnet18", drop_block_rate=None).drop_block_rate == 0.0
    c = copy.deepcopy(m)
    assert (c.drop_rate, c.drop_path_rate, c.drop_block_rate) == (0.2, 0.1, 0.2)
