"""The coverage contract of tests/test_plan_variants_gpu.py, without a GPU: every kernel the runner's other plans (test_img,
validation, short batches) launch is checked there or excluded with a reason; the test_img plan runs launch for launch; every
eval-form variant and every (kernel, batch class, dtype) has a case, at a batch that was not reduced; Engine._run issues what
Engine.launch_args gives; and the facts that motivated these cases are still in the plans."""
import ast
import os
from types import SimpleNamespace

import pytest

import plan_launches as PL
import plan_variants as PV

HERE = os.path.dirname(os.path.abspath(__file__))


def _checker_names(fname, var):
    tree = ast.parse(open(os.path.join(HERE, fname)).read())
    node = next(n.value for n in tree.body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == var)
    return {k.value for k in node.keys}


def _why_kernel(w):
    return w[1].kernel if w[0] == "test_img" else w[1]


def _all_launches():
    for p in PV.plans():
        for la in PV.launches(p):
            yield p, la


def test_plan_set():
    ps = PV.plans()
    assert ps[0] == PV.Plan("test_img", "dfv4", 1, "fp16", False)
    for tag, _, b, _, dt, _ in PL.CONFIGS:
        ns = {(p.batch, p.training) for p in ps if p.tag == tag and p.dtype == dt}
        assert {(b, False), (2 * b, False)} <= ns
        assert all({(n, True), (n, False)} <= ns for n in set(PV.SHORT + (b - 1,)) - {b}), (tag, ns)


def test_every_checker_exists():
    keys = _checker_names("test_plan_launches_gpu.py", "CHECKERS") | _checker_names("test_plan_variants_gpu.py", "NEW_CHECKERS")
    assert set(PV.EVAL_CHECKED.values()) <= keys and {c.check for c in PV.variant_cases()} <= keys


def test_every_kernel_is_checked_or_excluded():
    unknown = {la.kernel for _, la in _all_launches() if not PV.is_checked(la) and la.kernel not in PL.EXCLUDED}
    assert not unknown, "kernels launched by a plan with neither a GPU case nor a stated exclusion: %s" % sorted(unknown)
    # the eval form of the BatchNorm finalisation has a checker; only the training form stays with test_kernels_gpu
    assert any(la.kernel == "dfd_bn_finalize" and PV.is_checked(la) for _, la in _all_launches())


def test_test_img_plan_runs_launch_for_launch_in_fp16():
    tp = PV.test_img_plan()
    cases = [c for c in PV.variant_cases() if any(w[0] == "test_img" for w in c.why)]
    missing = []
    for la in PV.launches(tp):
        if not PV.is_checked(la):
            continue
        check, kw, dt, _ = PV.case_of(la, "fp16", tp)
        if not any(("test_img", la) in c.why and c.check == check and c.kw == kw and c.dtype == dt for c in cases):
            missing.append(la)
    assert not missing, missing[:5]
    assert all(c.dtype in ("fp16", "fp32") for c in cases)


def _covered():
    """(kernel, batch class, dtype) and (kernel, pointer mask, dtype) that the cases of both GPU files run"""
    classes, masks = set(PV.shipped_classes()), set()
    for c in PV.variant_cases():
        for w in c.why:
            kernel = _why_kernel(w)
            classes.add((kernel, PV.batch_class(kernel, c.check, c.kw), c.dtype))
            if w[0] == "test_img":
                masks.add((w[1].kernel, w[1].ptrs, c.dtype))
            elif w[0] == "eval":
                masks.add((w[1], w[2], c.dtype))
    return classes, masks


def test_every_batch_class_has_a_case():
    classes, _ = _covered()
    missing = set()
    for p, la in _all_launches():
        if PV.is_checked(la):
            check, kw, dt, cls = PV.case_of(la, p.dtype, p)
            if (la.kernel, cls, dt) not in classes:
                missing.add((la.kernel, cls, dt))
    assert not missing, sorted(missing, key=str)[:5]


def test_every_eval_variant_runs_in_both_dtypes():
    _, masks = _covered()
    shipped = PV.shipped_masks()
    missing = set()
    for p, la in _all_launches():
        if not p.training and PV.is_checked(la) and (la.kernel, la.ptrs) not in shipped:
            check = PV.case_of(la, p.dtype, p)[0]
            for d in (("fp32",) if check in PV.FP32 else ("bf16", "fp16")):
                if (la.kernel, la.ptrs, d) not in masks:
                    missing.add((la.kernel, la.ptrs, d))
    assert not missing, sorted(missing)
    # the stats-less depthwise forward is one of them, and its case asserts the bit-identity with the stats run
    assert any(c.check == "dwconv" and c.kw.get("stats") is False for c in PV.variant_cases())


def test_eval_head_and_finalize_at_every_shape():
    cases = PV.variant_cases()
    have = {(c.check, tuple(sorted(c.kw.items()))) for c in cases}
    for p, la in _all_launches():
        if la.kernel in PV.EVAL_CHECKED and PV.is_checked(la):
            check, kw, _, _ = PV.case_of(la, p.dtype, p)
            assert (check, tuple(sorted(kw.items()))) in have, la
    assert {c.kw["N"] for c in cases if c.check == "head_fwd"} >= {2 * b for _, _, b, _, _, _ in PL.CONFIGS}


def test_cases_run_a_planned_launch_at_its_batch():
    """no case is reduced: each runs the exact kwargs of a launch of the plan set (class cases: of their class)"""
    exact = {}
    for p, la in _all_launches():
        if PV.is_checked(la):
            check, kw, dt, cls = PV.case_of(la, p.dtype, p)
            exact.setdefault(PL._key(check, kw, None), set()).add((la.kernel, cls))
    for c in PV.variant_cases():
        got = exact.get(PL._key(c.check, c.kw, None))
        assert got is not None, c.id
        for w in c.why:
            if w[0] == "class":
                assert (w[1], w[2]) in got, (c.id, w)
        assert "reducedN" not in c.id


def test_case_ids_unique():
    ids = [c.id for c in PV.variant_cases()]
    assert len(ids) == len(set(ids))


# ---- Engine._run issues what Engine.launch_args gives ------------------------------------------------------------------------
@pytest.mark.parametrize("arch,kw", [("efficientnet_b0", dict(drop_rate=0.2, drop_path_rate=0.2)),
                                     ("resnet50", dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.1))])
def test_run_issues_what_launch_args_gives(monkeypatch, arch, kw):
    """the C-ABI calls of plan-only eval and training forwards (recorded in place of the kernels) are the plan's ops through
    launch_args; eval mode passes no batch statistics, no training-only operand and runs no `_train` op; a second eval
    forward finalises no BatchNorm"""
    import torch
    from deepfake_detection_b200.engine import Engine
    eng = Engine(arch, 2, 64 if arch == "efficientnet_b0" else 160, device="plan-only", **kw)
    calls = []

    def rec(name):
        return lambda *a: (calls.append((name, tuple(a[:-1]))), 0)[1]

    ops = [(rec(n), n, a) for _, n, a in eng.fwd_ops]
    eng.fwd_ops = ops
    eng._plan_only = False
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: SimpleNamespace(cuda_stream=0))

    def want(training):
        out = []
        for _, n, a in ops:
            a = eng.launch_args(n, a, training)
            if a is not None:
                out.append((n, tuple(a)))
        return out

    eng.forward(training=False, stream=0)
    ev = list(calls)
    assert ev == want(False)
    assert not any(n.endswith("_train") for n, _ in ev) and any(n.endswith("_train") for _, n, _ in ops)
    assert not any(isinstance(v, (tuple, str)) for _, a in ev for v in a)
    fin = [a for n, a in ev if n.startswith("dfd_bn_finalize")]
    assert fin and all(a[0] is None and a[1] is None and a[10] == 0 for a in fin)
    assert all(a[-3:] == (None, None, None) for n, a in ev if n in ("dfd_gemm_tn", "dfd_gemm_tn_rowpack", "dfd_dwconv_fwd", "dfd_conv_tc"))
    del calls[:]
    eng.forward(training=False, stream=0)
    assert calls == [c for c in ev if not c[0].startswith("dfd_bn_finalize")]
    del calls[:]
    eng.forward(training=True, stream=0)
    assert calls == want(True) and any(n.endswith("_train") for n, _ in calls)
    assert not any(isinstance(v, (tuple, str)) for _, a in calls for v in a)


# ---- the facts that motivated these cases ----------------------------------------------------------------------------------
def test_test_img_plan_is_new():
    la = PV.launches(PV.test_img_plan())
    fwd = [x for x in la if x.kernel != "dfd_head_fwd"]
    assert len(fwd) == 107 and sum(la[x] for x in fwd) == 549
    shipped = {x for x, _ in PL.harvest()}
    assert not any(x in shipped for x in la)


def test_b4_runs_a_plain_k32_gemm_at_odd_batches():
    for n in (1, 3, 5, 7, 13, 127):
        for training in (True, False):
            assert any(la.kernel == "dfd_gemm_tn" and la.shape[2] == 32 for la in PL.plan_launches("b4", n, training, "fp16")), n
    assert not any(la.kernel == "dfd_gemm_tn" and la.shape[2] == 32 for la in PL.plan_launches("b4"))


def test_r50_at_13_has_a_half_empty_image_tile():
    hits = [la for la in PL.plan_launches("r50", 13, True, "bf16") if la.kernel == "dfd_conv_tc"
            and PL.conv_patch(la.shape[1], la.shape[2], la.shape[5], la.shape[6], la.shape[0])[2] == 2]
    assert hits and all(la.shape[0] % 2 == 1 for la in hits)


def test_some_pool_runs_one_cta_per_image():
    big = [(p, la) for p, la in _all_launches() if la.kernel == "dfd_pool" and la.shape[0] >= 296]
    assert big and all(PV.pool_geom(la.shape[2], la.shape[1], la.shape[0], la.shape[-1])[3] for _, la in big)
    assert all(la.shape[0] < 296 for la, _ in PL.harvest() if la.kernel == "dfd_pool")


def test_no_shipped_depthwise_forward_lacks_stats():
    masks = {la.ptrs for la, _ in PL.harvest() if la.kernel == "dfd_dwconv_fwd"}
    assert masks == {"ppppppp0", "p00pppp0"}, masks
