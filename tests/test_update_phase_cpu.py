"""The update half of the training step without a GPU: a later plan over the same arena can register derived weight layouts,
and a captured train step must then be re-captured; every kernel the update phase launches, at every configuration's arena,
is run by tests/test_update_phase_gpu.py at the same element counts and pointer pattern, or excluded with a reason."""
from types import SimpleNamespace

import pytest
import torch

import plan_launches as PL
import update_phase as UP
from deepfake_detection_b200 import _lib


# ---- a second plan over the same arena -------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch,res,n1,n2,added", [("efficientnet_b0", 98, 8, 6, 8), ("efficientnet_b4", 380, 32, 13, 4)])
def test_later_plan_registers_new_layouts(arch, res, n1, n2, added):
    """the row-pack factor follows M = N*H*W: a plan of another batch size needs block-diagonal copies of other pack"""
    from deepfake_detection_b200.engine import Engine
    a = Engine(arch, n1, res, res, device="plan-only")
    before = dict(a._bd_reg)
    Engine(arch, n2, res, res, device="plan-only", share_from=a)
    new = [k for k in a._bd_reg if k not in before]
    assert len(before) > 0 and len(new) == added, (len(before), new)
    old_packs = {(B, Nn, K): pack for (B, Nn, K, pack) in before}
    for B, Nn, K, pack in new:          # the same weights, packed by a smaller factor
        assert (B, Nn, K) in old_packs and pack < old_packs[(B, Nn, K)]


def _plan_trainer(arch, n, res):
    from deepfake_detection_b200.engine import Engine
    return UP.make_trainer(Engine(arch, n, res, res, device="plan-only"), "sgd", use_graph=True)


def test_graph_signature_changes_when_a_later_plan_adds_layouts():
    """the captured step refreshes the layouts registered at capture time through a table that a later registration frees:
    the signature that decides re-capture must move"""
    from deepfake_detection_b200.engine import Engine
    tr = _plan_trainer("efficientnet_b0", 8, 98)
    sig = tr._graph_signature(False)
    Engine("efficientnet_b0", 6, 98, 98, device="plan-only", share_from=tr.engine)
    assert tr._graph_signature(False) != sig


def test_graph_signature_kept_when_a_later_plan_adds_nothing():
    """a plan that needs no new layout (B0 at 96x96 keeps every pack) does not force a re-capture"""
    from deepfake_detection_b200.engine import Engine
    tr = _plan_trainer("efficientnet_b0", 8, 96)
    n = len(tr.engine._bd_reg)
    sig = tr._graph_signature(False)
    Engine("efficientnet_b0", 6, 96, 96, device="plan-only", share_from=tr.engine)
    assert len(tr.engine._bd_reg) == n and tr._graph_signature(False) == sig


def test_resnet_layouts_bump_the_generation():
    from deepfake_detection_b200.engine import Engine
    a = Engine("resnet18", 1, device="plan-only", params_only=True)
    g = a.layout_gen
    Engine("resnet18", 2, 64, 64, device="plan-only", share_from=a)
    g2 = a.layout_gen
    assert g2 > g and a._rtable_count > 0 and len(a._stem_reg) == 1
    Engine("resnet18", 2, 64, 64, device="plan-only", share_from=a)          # nothing new: same generation
    assert a.layout_gen == g2


# ---- the coverage contract ---------------------------------------------------------------------------------------------------
def _record(monkeypatch, tag, dtype, opt, batch=None):
    """the C-ABI calls of one update phase (the Trainer's part after backward, zero_grad, the lr push and the EMA update) of
    the configuration's plan at `batch`, as plan_launches.Launch tuples"""
    calls = []
    monkeypatch.setattr(_lib, "call", lambda name, *args: calls.append(PL._split(name, args[:-1])))   # the stream last
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: SimpleNamespace(cuda_stream=0))
    eng = UP.engine(tag, dtype, batch=batch, device="plan-only")
    tr = UP.make_trainer(eng, opt)
    tr.optimizer.push_hyper()
    tr._launch_step(False, "back")
    tr.optimizer.zero_grad()
    UP.ema_update(UP.arena(tag, dtype, device="plan-only"), eng.arena, 0.9998)
    monkeypatch.undo()
    return calls


def _gpu_runs():
    """kernel -> the test of tests/test_update_phase_gpu.py that runs it (its RUNS table)"""
    import ast
    import os
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_update_phase_gpu.py")).read()
    node = next(n.value for n in ast.parse(src).body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "RUNS")
    return {k.value: v.value for k, v in zip(node.keys, node.values)}, {n.name for n in ast.parse(src).body
                                                                          if isinstance(n, ast.FunctionDef)}


@pytest.mark.parametrize("tag", [t for t, *_ in PL.CONFIGS])
def test_every_update_kernel_runs_on_the_gpu_at_the_shipped_geometry(monkeypatch, tag):
    """the GPU file runs the update phase through the same wiring (update_phase.make_trainer / ema_update) at GPU_BATCH: its
    launches must be exactly the shipped batch's, kernel for kernel, element count for element count, pointer for pointer"""
    runs, tests = _gpu_runs()
    assert set(runs.values()) <= tests and not set(runs) & set(UP.EXCLUDED)
    for dtype in UP.DTYPES:
        for opt in UP.OPTS:
            shipped = _record(monkeypatch, tag, dtype, opt)
            kernels = {la.kernel for la in shipped}
            assert not kernels - set(runs) - set(UP.EXCLUDED), (dtype, opt, sorted(kernels - set(runs) - set(UP.EXCLUDED)))
            step = {"sgd": "dfd_sgd_step", "adam": "dfd_adam_step", "adamw": "dfd_adam_step", "rmsproptf": "dfd_rmsprop_tf_step"}[opt]
            # one launch per arena range, with the Trainer's pointers: (p, g, state(s)), gscale_dev and skip under loss scaling
            # only, p16, lr_dev (and Adam's step_dev)
            scaled = "pp" if dtype == "fp16" else "00"
            ptrs = {"sgd": "ppp" + scaled + "pp", "rmsproptf": "pppp" + scaled + "pp"}.get(opt, "pppp" + scaled + "ppp")
            assert [la.ptrs for la in shipped if la.kernel == step] == [ptrs, ptrs]
            assert ("dfd_check_finite" in kernels) == ("dfd_update_loss_scale" in kernels) == (dtype == "fp16")
            assert ("dfd_opt_tick" in kernels) == (opt in ("adam", "adamw"))
            assert _record(monkeypatch, tag, dtype, opt, batch=UP.GPU_BATCH[tag]) == shipped


@pytest.mark.parametrize("tag", [t for t, *_ in PL.CONFIGS])
def test_gpu_batch_registers_the_shipped_layouts(tag):
    for dtype in UP.DTYPES:
        got = UP.layout_keys(UP.engine(tag, dtype, batch=UP.GPU_BATCH[tag], device="plan-only"))
        assert got == UP.shipped_layout_keys(tag, dtype)
    bd, stem, rep = UP.shipped_layout_keys(tag, PL.config_dtype(tag))
    # every configuration has a padded stem weight; EfficientNet has block-diagonal copies, ResNet packed k x k weights
    assert len(stem) == 1
    assert (len(rep) > 0) == tag.startswith("r") and (len(bd) > 0) == (not tag.startswith("r"))
