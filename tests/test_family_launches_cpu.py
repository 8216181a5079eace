"""The coverage contract of tests/test_family_launches_gpu.py, without a GPU: every kernel the model families' training plans
launch is checked there or excluded with a reason, every launch of a checked kernel has its case (or a shipped case runs its
key) under plan_launches' tiering, every mode argument of a launch is what its case runs, and the launch patterns that
motivated the cases are still in the plans."""
import pytest

import family_launches as FL
import plan_launches as PL


def _cases():
    return FL.gpu_cases()


def _runs(la, dt, plan):
    """the (check, kwargs without counts, dtype) keys that run this launch at its shape: its own case (the batch as the case
    runs it) or a shipped one"""
    check, kw, n_full, _ = FL.case_of(la, dt, plan)
    kw, _ = FL._sized(check, kw, n_full)
    return PL._key(check, kw, "fp32" if check in FL.FP32 else dt)


def _keys():
    return {PL._key(c.check, c.kw, c.dtype) for c in _cases()} | FL.shipped_keys()


def _plan_of(tags):
    return FL.plan_launches(tags[0])


def test_table_and_harvest_sizes():
    assert [t for t in FL.tags() if t in {c[0] for c in PL.CONFIGS}] == []
    assert all(c not in PL.CONFIGS for c in FL.FAMILY_CONFIGS)          # the shipped table is not extended
    sizes = {t: len(FL.plan_launches(t)) for t in FL.tags()}
    assert all(n > 90 for n in sizes.values()), sizes


def test_every_planned_kernel_is_checked_or_excluded():
    kernels = {la.kernel for la, _ in FL.harvest()}
    unknown = kernels - set(FL.CHECKED) - set(FL.EXCLUDED)
    assert not unknown, "kernels launched by a family plan with neither a GPU case nor a stated exclusion: %s" % sorted(unknown)
    assert not set(FL.CHECKED) & set(FL.EXCLUDED) and all(FL.EXCLUDED.values())


def test_every_checker_exists():
    import ast
    import os
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_family_launches_gpu.py")).read()
    call = next(node.value for node in ast.parse(src).body if isinstance(node, ast.Assign) and getattr(node.targets[0], "id", "") == "CHECKERS")
    own = {k.arg for k in call.keywords}
    shipped = set(PL.CHECKED.values()) | {"head_fwd", "bn_finalize_eval"}
    assert {c.check for c in _cases()} <= own | shipped


def test_every_contraction_launch_runs_at_its_shape_in_its_dtype():
    keys = _keys()
    missing = [(la, dt) for (la, dt), tgs in FL.harvest().items() if la.kernel in FL.CONTRACTION and _runs(la, dt, _plan_of(tgs)) not in keys]
    assert not missing, missing[:5]


def test_every_contraction_class_runs_in_the_other_dtype():
    have, classes = set(), {}
    for (la, dt), tgs in FL.harvest().items():
        if la.kernel in FL.CONTRACTION:
            classes.setdefault((la.kernel, FL.case_of(la, dt, _plan_of(tgs))[3]), set()).add(dt)
    for c in _cases():
        have |= {(la[1], la[2], c.dtype) for la in c.launches if la[0] == "class"}
    shipped = {(la[1], la[2], c.dtype) for c in PL.gpu_cases() for la in c.launches if la[0] == "class"}
    shipped |= {(la.kernel, PL._case_of(la, dt)[3], dt) for la, dt in PL.harvest() if la.kernel in PL.CONTRACTION}
    missing = [(k, cls, dt) for (k, cls), dts in classes.items() for dt in ("bf16", "fp16")
               if dt not in dts and (k, cls, dt) not in have | shipped]
    assert not missing, missing[:5]


def test_every_bandwidth_shape_runs_in_both_dtypes():
    keys = _keys()
    missing = []
    for (la, dt), tgs in FL.harvest().items():
        if la.kernel not in FL.BANDWIDTH:
            continue
        check, kw, n_full, _ = FL.case_of(la, dt, _plan_of(tgs))
        kw, _ = FL._sized(check, kw, n_full)
        for d in (("fp32",) if check in FL.FP32 else ("bf16", "fp16")):
            if PL._key(check, kw, d) not in keys:
                missing.append((la, d))
    assert not missing, missing[:5]


def test_row_kernel_cases_keep_the_whole_launch():
    import gpu_checks
    for (la, dt), tgs in FL.harvest().items():
        if FL.CHECKED.get(la.kernel) != "row":
            continue
        check, kw, _, _ = FL.case_of(la, dt, _plan_of(tgs))
        assert la.kernel in gpu_checks.ROW_KERNELS, la
        assert (kw["N"], kw["HW"], kw["C"]) == la.shape[:3] and len(kw["args"]) == len(la.shape) - 4 and kw["ptrs"] == la.ptrs, la


def test_exact_batch_cases_assert_split_and_part_counts():
    cases = _cases()
    assert any(c.check == "dwconv_relu" and "ws_bytes" in c.kw and c.n_full is None for c in cases)
    assert any(c.check == "dw_pad" and "ws_bytes" in c.kw and c.n_full is None for c in cases)
    for c in cases:
        for la in c.launches:
            if la[0] not in ("class", "eval", "odd") and c.n_full is None and la[0].kernel in (
                    "dfd_gemm_wgrad", "dfd_dwconv_bwd", "dfd_dwconv_bwd_relu", "dfd_dwconv_bwd_pad", "dfd_conv_wgrad_tc"):
                assert ("splits" in c.kw) or ("ws_bytes" in c.kw), c.id


def test_case_ids_unique_and_reductions_stated():
    ids = [c.id for c in _cases()]
    assert len(ids) == len(set(ids))
    shipped = {c.id for c in PL.gpu_cases()}
    assert not set(ids) & shipped
    for c in _cases():
        assert (c.n_full is None) == ("reducedN" not in c.id)
        assert c.n_full is None or c.kw["N"] < c.n_full


def test_case_of_reproduces_every_mode_argument():
    """every harvested launch (training plans, and the batch-1 eval plans) runs a case whose checker issues the launch's
    own mode arguments: activation, BatchNorm input, statistics, arg-max bytes, added gradient, second gradient source"""
    bad = []
    seen = [(la, dt, _plan_of(tgs)) for (la, dt), tgs in FL.harvest().items()]
    seen += [(la, FL.EVAL_DTYPE, FL.eval_plan(t)) for t in FL.tags() for la in FL.eval_plan(t)]
    for la, dt, plan in seen:
        modes = FL.launch_modes(la)
        if modes is None or not FL.is_checked(la):
            continue
        check, kw, _, _ = FL.case_of(la, dt, plan)
        if modes not in FL.case_modes(la, check, kw):
            bad.append((la, check, kw))
    assert not bad, bad[:5]


def test_unmodelled_mode_arguments_raise():
    xc = [la for la in FL.plan_launches("xc") if la.kernel == "dfd_dwconv_fwd"]
    la = xc[0]
    for shape, ptrs in ((la.shape[:6] + (3,) + la.shape[7:], la.ptrs), (la.shape[:6] + (1,) + la.shape[7:], "p00pp000"),
                        (la.shape[:6] + (0,) + la.shape[7:], "ppppp000")):
        with pytest.raises((KeyError, AssertionError)):
            FL.case_of(PL.Launch(la.kernel, shape, ptrs), "bf16", FL.plan_launches("xc"))
    bwd = next(la for la in FL.plan_launches("xc") if la.kernel == "dfd_dwconv_bwd_relu")
    with pytest.raises(AssertionError):            # a folded BatchNorm backward (cA) is not a form the ReLU kernels run
        FL.case_of(bwd._replace(ptrs=bwd.ptrs[:2] + "p" + bwd.ptrs[3:]), "bf16", FL.plan_launches("xc"))


# ---- the facts that motivated the cases -----------------------------------------------------------------------------------
def test_xception_issues_relu_depthwise_with_and_without_bn():
    fwd = {(la.shape[6], la.ptrs[1]) for la in FL.plan_launches("xc") if la.kernel == "dfd_dwconv_fwd"}
    assert {(2, "p"), (2, "0")} <= fwd, fwd
    bwd = {(la.ptrs[7], la.ptrs[11]) for la in FL.plan_launches("xc") if la.kernel == "dfd_dwconv_bwd_relu"}
    assert {("p", "0"), ("0", "p"), ("0", "0")} <= bwd, bwd


def test_xception_conv2_im2col_has_pad_0():
    im = [la.shape for la in FL.plan_launches("xc") if la.kernel == "dfd_im2col"]
    assert any(s[4] == 3 and s[6] == 0 and s[1] == 149 for s in im), im
    assert any(s[3] == 728 and s[4] == 1 and s[5] == 2 for s in im), im


def test_xception_block_tails_cover_odd_and_even_extents():
    hs = sorted({la.shape[1] for la in FL.plan_launches("xc") if la.kernel == "dfd_bn_maxpool_add"}, reverse=True)
    assert hs == [147, 74, 37, 19], hs
    assert any(la.ptrs[7] == "0" for la in FL.eval_plan("xc") if la.kernel == "dfd_bn_maxpool_add")


def test_seresnet_se_activation():
    se18 = {la.shape[4] for la in FL.plan_launches("se18") if la.kernel == "dfd_pool_se_relu"}
    se50 = {la.shape[4] for la in FL.plan_launches("se50") if la.kernel == "dfd_pool_se_relu"}
    assert se18 == {2} and se50 == {0}, (se18, se50)
    masks = {la.ptrs[1] for la in FL.plan_launches("se50") if la.kernel == "dfd_relu_se_bwd_reduce"}
    assert masks == {"p", "0"}, masks


@pytest.mark.parametrize("tag", ["r50d", "r26d"])
def test_resnet_d_average_pool_extents(tag):
    for k in ("dfd_avgpool2_fwd", "dfd_avgpool2_bwd_add"):
        assert sorted({la.shape[1] for la in FL.plan_launches(tag) if la.kernel == k}) == [14, 28, 56]
    assert any(la.kernel == "dfd_im2col" and la.shape[1] == 112 and la.shape[3] == 32 and la.shape[6] == 1 for la in FL.plan_launches(tag))


@pytest.mark.parametrize("tag", ["tfb0", "tfb4"])
def test_tf_plans_issue_the_pad_entry_points(tag):
    ks = {la.kernel for la in FL.plan_launches(tag)}
    assert {"dfd_dwconv_fwd_pad", "dfd_dwconv_bwd_pad", "dfd_stem_im2col_pad"} <= ks, ks
    assert "dfd_stem_im2col" not in ks


def test_families_without_new_shapes_cost_nothing():
    for tag in ("r34", "r101"):
        keys = {_runs(la, dt, FL.plan_launches(tag)) for (la, dt), tgs in FL.harvest().items() if tag in tgs and la.kernel in FL.CHECKED}
        assert keys <= FL.shipped_keys(), sorted(keys - FL.shipped_keys())[:3]
