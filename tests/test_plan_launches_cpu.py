"""The coverage contract of tests/test_plan_launches_gpu.py, without a GPU: every kernel the shipped training plans launch is
checked there or excluded with a reason, every launch of a checked kernel has its case under the tiering rules, and the launch
shapes that motivated the per-launch tests are still in the plans."""
from collections import Counter

import pytest

import plan_launches as PL


def _cases():
    return PL.gpu_cases()


def _covered():
    """(Launch, dtype) -> the cases that list it"""
    out = {}
    for c in _cases():
        for la in c.launches:
            out.setdefault(la, []).append(c)
    return out


def test_harvest_sizes():
    sizes = {tag: len(PL.plan_launches(tag)) for tag, *_ in PL.CONFIGS}
    assert all(n > 90 for n in sizes.values()), sizes
    assert len(PL.harvest()) > 900, len(PL.harvest())


def test_every_planned_kernel_is_checked_or_excluded():
    kernels = {la.kernel for la, _ in PL.harvest()}
    unknown = kernels - set(PL.CHECKED) - set(PL.EXCLUDED)
    assert not unknown, "kernels launched by a plan with neither a GPU case nor a stated exclusion: %s" % sorted(unknown)
    assert not set(PL.CHECKED) & set(PL.EXCLUDED)
    assert all(PL.EXCLUDED.values())


def test_every_checker_exists():
    import ast
    import os
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_plan_launches_gpu.py")).read()
    tree = ast.parse(src)
    names = next(node.value for node in tree.body if isinstance(node, ast.Assign) and getattr(node.targets[0], "id", "") == "CHECKERS")
    keys = {k.value for k in names.keys}
    assert set(PL.CHECKED.values()) <= keys and {c.check for c in _cases()} <= keys


def _same_launch(case, la):
    """the case runs exactly this launch's shape (or at a reduced batch, stated in its id)"""
    check, kw, n_full, _ = PL._case_of(*la)
    if check != case.check:
        return False
    want = {k: v for k, v in kw.items() if k not in PL._COUNTS}
    got = {k: v for k, v in case.kw.items() if k not in PL._COUNTS}
    if case.n_full is not None:
        assert "reducedN%d" % case.n_full in case.id and case.kw["N"] < case.n_full == want["N"], case
        want["N"] = got["N"]
    return want == got


def test_every_contraction_launch_runs_at_its_shape_in_its_dtype():
    cov = _covered()
    missing = []
    for (la, dt), tags in PL.harvest().items():
        if la.kernel not in PL.CONTRACTION:
            continue
        cs = [c for c in cov.get((la, dt), []) if c.dtype == dt and _same_launch(c, (la, dt))]
        if not cs:
            missing.append((la, dt, tags))
    assert not missing, missing[:5]


def test_every_contraction_class_runs_in_the_other_dtype():
    classes = {}
    for (la, dt), _ in PL.harvest().items():
        if la.kernel in PL.CONTRACTION:
            classes.setdefault((la.kernel, PL._case_of(la, dt)[3]), set()).add(dt)
    have = set()
    for c in _cases():
        for la in c.launches:
            if la[0] == "class":
                have.add((la[1], la[2], c.dtype))
    missing = [(k, cls, dt) for (k, cls), dts in classes.items() for dt in ("bf16", "fp16") if dt not in dts and (k, cls, dt) not in have]
    assert not missing, missing[:5]


def test_every_bandwidth_shape_runs_in_both_dtypes():
    cov = _covered()
    missing = []
    for (la, dt), _ in PL.harvest().items():
        if la.kernel not in PL.BANDWIDTH:
            continue
        want = {"fp32"} if PL.CHECKED[la.kernel] in ("se_fc", "head") else {"bf16", "fp16"}
        got = {c.dtype for c in cov.get((la, dt), []) if _same_launch(c, (la, dt))}
        if not want <= got:
            missing.append((la, dt, want - got))
    assert not missing, missing[:5]


def test_row_kernel_cases_keep_the_whole_launch():
    """a per-row kernel's case keeps every argument that can select its instantiation: all non-pointer arguments but the
    dtype, and the pointer-presence mask; and the checker implements that kernel"""
    import gpu_checks
    for (la, dt), _ in PL.harvest().items():
        if PL.CHECKED.get(la.kernel) != "row":
            continue
        check, kw, _, _ = PL._case_of(la, dt)
        assert la.kernel in gpu_checks.ROW_KERNELS, la
        assert (kw["N"], kw["HW"], kw["C"]) == la.shape[:3] and len(kw["args"]) == len(la.shape) - 4 and kw["ptrs"] == la.ptrs, la


def test_resnet_elementwise_variants_have_cases():
    """the ResNet path's own instantiations: BN + ReLU, residual add then ReLU, ReLU backward, the affine-free pool"""
    runs = {(c.kw["kernel"], c.kw["args"], c.kw["ptrs"], c.dtype) for c in _cases() if c.check == "row"}
    for dt in ("bf16", "fp16"):
        assert any(k == "dfd_bn_act" and a[0] == 2 for k, a, _, d in runs if d == dt)
        assert any(k == "dfd_bn_act" and a[1] == 2 for k, a, _, d in runs if d == dt)
        assert any(k == "dfd_act_bwd" and a[0] == 2 for k, a, _, d in runs if d == dt)
        assert any(k == "dfd_act_bwd" and p[0] == "0" for k, a, p, d in runs if d == dt)
        assert any(k == "dfd_pool" and a[0] == 0 and p[1] == "0" for k, a, p, d in runs if d == dt)


def test_exact_batch_kept_where_split_counts_follow_it():
    """the weight-gradient split count and the depthwise backward's part count depend on the batch: at least one case per
    kernel runs the plan's own batch and asserts the plan's count"""
    cases = _cases()
    assert any(c.check == "wgrad" and "splits" in c.kw and c.n_full is None for c in cases)
    assert any(c.check == "dwconv" and "ws_bytes" in c.kw and c.n_full is None for c in cases)
    # and every exact-shape case asserts the count of its launch
    for c in cases:
        for la in c.launches:
            if la[0] != "class" and la[0].kernel in ("dfd_gemm_wgrad", "dfd_dwconv_bwd", "dfd_conv_wgrad_tc") and c.n_full is None:
                assert ("splits" in c.kw) or ("ws_bytes" in c.kw), c.id


def test_case_ids_unique_and_reductions_stated():
    ids = [c.id for c in _cases()]
    assert len(ids) == len(set(ids))
    for c in _cases():
        assert (c.n_full is None) == ("reducedN" not in c.id)
        assert c.n_full is None or c.kw["N"] < c.n_full


# ---- the facts that motivated the per-launch tests ------------------------------------------------------------------------
def test_b0_has_a_pack8_rowpack_launch():
    assert any(la.kernel == "dfd_gemm_tn_rowpack" and la.shape[3] == 8 for la in PL.plan_launches("b0"))
    packs = {la.shape[3] for tag in ("b0", "b4") for la in PL.plan_launches(tag) if la.kernel == "dfd_gemm_tn_rowpack"}
    assert {2, 4, 8} <= packs, packs


def test_b4_runs_cpw8_depthwise_at_190():
    hits = [la for la in PL.plan_launches("b4") if la.kernel in ("dfd_dwconv_fwd", "dfd_dwconv_bwd")
            and la.shape[1:3] == (190, 190) and PL.dw_cpw(la.shape[3]) == 8]
    assert {la.kernel for la in hits} == {"dfd_dwconv_fwd", "dfd_dwconv_bwd"}, hits
    assert PL.config_dtype("b4") == "fp16"


def test_some_depthwise_launch_has_tw32_and_cpw32():
    assert any(la.kernel == "dfd_dwconv_fwd" and PL.dw_tile(*la.shape[1:3], la.shape[4], la.shape[5])[0] == 32
               and PL.dw_cpw(la.shape[3]) == 32 for (la, _) in PL.harvest())


@pytest.mark.parametrize("tag", [t for t, *_ in PL.CONFIGS])
def test_stem_runs_through_im2col_and_the_tensor_core_gemm(tag):
    ks = Counter(la.kernel for la in PL.plan_launches(tag))
    assert ks["dfd_stem_im2col"] == 1 and ks["dfd_unpad_grad"] == 1 and "dfd_stem_fwd" not in ks, ks
    im = next(la for la in PL.plan_launches(tag) if la.kernel == "dfd_stem_im2col")
    N, Cin, H, W, k, s, pad, Kp = im.shape[:8]
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    # the plain tensor-core GEMM, or its row-packed form where Kp is small (Kp = 32: four rows per TMA row)
    assert any(la.kernel in ("dfd_gemm_tn", "dfd_gemm_tn_rowpack") and la.shape[0] == N * Ho * Wo and la.shape[2] == Kp
               for la in PL.plan_launches(tag))
