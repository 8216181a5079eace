"""The kernel launches of the model families' training plans (ResNet-34/101, Wide ResNet, ResNet-D, SE-ResNet, Xception and the
TF EfficientNets), harvested on the CPU as tests/plan_launches.py harvests the shipped plans, and their GPU cases.

FAMILY_CONFIGS lists each family at the geometry its README / DESIGN timings use. The cases follow plan_launches' tiering,
batch reduction (MAX_ELEMS, `reducedN<full>` ids) and `_key`s; a case whose key a shipped case (plan_launches.gpu_cases())
already runs is dropped, so a family that launches only shipped shapes (resnet34, resnet101) costs nothing but stays under
the contract. Besides the training plans, each family's eval form at batch 1 in fp16 (the `test_img` path) contributes one
case per (kernel, pointer mask) that no training plan issues, in both 16-bit types, and the logits-only head and the eval
BatchNorm finalisation at every new (N, F) and channel count. The short-batch and `-vb` validation plans of these families
are not covered here: tests/plan_variants.py builds those for the shipped configurations only.

tests/test_family_launches_cpu.py holds the cases to the plans; tests/test_family_launches_gpu.py runs them.
"""
import functools
from collections import OrderedDict

import plan_launches as PL
import plan_variants as PV

# (tag, arch, batch, resolution, dtype, extra Engine kwargs)
FAMILY_CONFIGS = [
    ("r34", "resnet34", 256, 224, "bf16", {}),
    ("r101", "resnet101", 256, 224, "bf16", {}),
    ("wrn50", "wide_resnet50_2", 256, 224, "bf16", {}),
    ("r50d", "resnet50d", 256, 224, "bf16", {}),
    ("r26d", "resnet26d", 256, 224, "bf16", {}),
    ("se50", "seresnet50", 256, 224, "bf16", {}),
    ("se18", "seresnet18", 256, 224, "bf16", {}),
    ("xc", "xception", 64, 299, "bf16", {}),
    ("tfb0", "tf_efficientnet_b0", 256, 224, "bf16", {}),
    ("tfb4", "tf_efficientnet_b4_ns", 128, 380, "fp16", {}),
]
PL.TABLES["family"] = FAMILY_CONFIGS

EVAL_BATCH, EVAL_DTYPE = 1, "fp16"

# kernels only these plans launch -> their checker (tests/family_checks.py, tests/tf_same_checks.py)
CONTRACTION = dict(PL.CONTRACTION, **{
    "dfd_dwconv_bwd_relu": "dwconv_relu",
    "dfd_dwconv_fwd_pad": "dw_pad",
    "dfd_dwconv_bwd_pad": "dw_pad",
    "dfd_stem_im2col_pad": "stem_pad",
})
BANDWIDTH = dict(PL.BANDWIDTH, **{
    "dfd_bn_maxpool_add": "bn_maxpool",
    "dfd_maxpool_bn_bwd_reduce": "bn_maxpool",
    "dfd_maxpool_ceil_fwd": "maxpool_ceil",
    "dfd_maxpool_ceil_bwd": "maxpool_ceil",
    "dfd_pool_se_relu": "pool_se_relu",
    "dfd_relu_se_bwd_reduce": "relu_se_bwd",
    "dfd_se_fc_wgrad": "se_fc_wgrad",
    "dfd_avgpool2_fwd": "avgpool2",
    "dfd_avgpool2_bwd_add": "avgpool2",
    "dfd_im2col": "im2col",
    "dfd_col2im": "im2col",
})
CHECKED = dict(CONTRACTION, **BANDWIDTH)
EXCLUDED = dict(PL.EXCLUDED)
FP32 = ("se_fc", "head", "se_fc_wgrad", "head_fwd", "bn_finalize_eval")
# the plans pool even extents only (56 / 28 / 14): one more case per channel count clips the last window row and column
ODD_EXTENT = 15          # the avgpool2 case at an odd extent (a clipped last window) at each plan channel count


def tags():
    return [c[0] for c in FAMILY_CONFIGS]


def config_dtype(tag):
    return next(c[4] for c in FAMILY_CONFIGS if c[0] == tag)


def plan_launches(tag, batch=None, training=True, dtype=None):
    return PL.plan_launches(tag, batch, training, dtype, table="family")


@functools.lru_cache(maxsize=None)
def harvest():
    """OrderedDict (Launch, dtype) -> tags of the family configurations that issue it"""
    out = OrderedDict()
    for tag in tags():
        for la in plan_launches(tag):
            out.setdefault((la, config_dtype(tag)), []).append(tag)
    return out


def _tf_pads(plan):
    return any(la.kernel in ("dfd_dwconv_fwd_pad", "dfd_stem_im2col_pad") for la in plan)


def case_of(la, dtype, plan):
    """(check, kwargs, n_full, dispatch class) of a launch of `plan` (the launches of the plan that issues it): the family
    kernels here, the rest through plan_launches._case_of. An argument pattern no checker runs raises."""
    k, s, p = la.kernel, la.shape, la.ptrs
    if k in ("dfd_dwconv_fwd_pad", "dfd_dwconv_bwd_pad"):
        # the stride-2 stage of an inverted-residual block: BN + Swish input (mode 1, BN backward folded into gy)
        N, H, W, C, kk, st, pt, pl = s[:8]
        if k == "dfd_dwconv_fwd_pad":
            assert s[8] == 1 and p[1:5] == "pppp" and p[5] == p[6] and p[7] == "0", la
            return "dw_pad", dict(N=N, H=H, W=W, C=C, k=kk, s=st, pt=pt, pl=pl, stats=p[5] == "p"), N, \
                ("dw_pad_fwd", PL.dw_cpw(C), kk, pt, pl)
        assert p == "ppppppppppp0ppppp0", la
        return "dw_pad", dict(N=N, H=H, W=W, C=C, k=kk, s=st, pt=pt, pl=pl, stats=True, ws_bytes=s[9]), N, \
            ("dw_pad_bwd", PL.dw_cpw(C), PL.dw_bwd_tile(H, W), kk, pt, pl)
    if k == "dfd_stem_im2col_pad":
        N, Cin, H, W, kk, st, pt, pl = s[:8]
        return "stem_pad", dict(N=N, Cin=Cin, H=H, W=W, k=kk, s=st, pt=pt, pl=pl), N, ("stem_pad", Cin, kk, pt, pl)
    if k == "dfd_unpad_grad" and _tf_pads(plan):
        # the TF stem's weight gradient: the stem GEMM case at the symmetric pad runs the same GEMMs (same M, Cout and Kp at
        # an even extent) and dfd_unpad_grad
        im = next(x for x in plan if x.kernel == "dfd_stem_im2col_pad")
        N, Cin, H, W, kk, st, pt, pl, Kp = im.shape[:9]
        cout, pack = PL._stem_gemm_form(N, Cin, H, W, kk, st, (kk - 1) // 2, Kp, plan)
        return "stem_gemm", dict(N=N, Cin=Cin, H=H, W=W, Cout=cout, k=kk, s=st, pad=(kk - 1) // 2, pack=pack), N, ("stem", Cin, kk, pack)
    if k in ("dfd_bn_maxpool_add", "dfd_maxpool_bn_bwd_reduce"):
        # the forward with the arg-max bytes (training) or without (eval); the backward reads them
        assert p[:7] == "ppppppp" and (k == "dfd_bn_maxpool_add" or p == "p" * 8), la
        idx = k == "dfd_maxpool_bn_bwd_reduce" or p[7] == "p"
        return "bn_maxpool", dict(N=s[0], H=s[1], W=s[2], C=s[3], idx=idx), s[0], None
    if k in ("dfd_maxpool_ceil_fwd", "dfd_maxpool_ceil_bwd"):
        assert p == "ppp", la
        return "maxpool_ceil", dict(N=s[0], H=s[1], W=s[2], C=s[3]), s[0], None
    if k == "dfd_pool_se_relu":
        assert p == "p" * 9, la
        N, HW, C, Cse, act, _, chunks = s
        return "pool_se_relu", dict(N=N, HW=HW, C=C, Cse=Cse, act=act, max_chunks=chunks), N, None
    if k == "dfd_relu_se_bwd_reduce":
        assert p[0] == "p" and p[2:] == "p" * 15, la
        N, HW, C, Cse, act, _ = s
        return "relu_se_bwd", dict(N=N, HW=HW, C=C, Cse=Cse, act=act, two=p[1] == "p"), N, None
    if k == "dfd_se_fc_wgrad":
        assert p == "p" * 8, la
        return "se_fc_wgrad", dict(N=s[0], C=s[1], Cse=s[2]), None, None
    if k in ("dfd_avgpool2_fwd", "dfd_avgpool2_bwd_add"):
        # the forward does not say whether its backward adds: its case runs the backward with `add`, as the plan does
        add = k == "dfd_avgpool2_fwd" or p[1] == "p"
        assert p in ("pp", "ppp", "p0p"), la
        return "avgpool2", dict(N=s[0], H=s[1], W=s[2], C=s[3], add=add), s[0], None
    if k in ("dfd_im2col", "dfd_col2im"):
        N, H, W, C, kk, st, pad = s[:7]
        if k == "dfd_im2col":       # with the add of the plan's col2im at this geometry (none if it has no col2im there)
            assert p == "pp", la
            add = any(x.kernel == "dfd_col2im" and x.shape == s and x.ptrs[1] == "p" for x in plan)
        else:
            assert p in ("ppp", "p0p"), la
            add = p[1] == "p"
        return "im2col", dict(N=N, H=H, W=W, C=C, k=kk, s=st, pad=pad, add=add), N, None
    return PL._case_of(la, dtype, plan)


def _elems(check, kw):
    """elements of the operands one case allocates per image (see plan_launches._elems)"""
    if check in ("dwconv_relu", "dw_pad"):
        return PL._elems("dwconv", kw)
    if check == "stem_pad":
        return PL._elems("stem_gemm", dict(kw, pad=kw["pt"], Cout=0))
    if check in ("bn_maxpool", "maxpool_ceil"):
        return 2 * kw["H"] * kw["W"] * kw["C"] + 4 * ((kw["H"] + 1) // 2) * ((kw["W"] + 1) // 2) * kw["C"]
    if check == "pool_se_relu":
        return 2 * kw["HW"] * kw["C"]
    if check == "relu_se_bwd":
        return 5 * kw["HW"] * kw["C"]
    if check == "avgpool2":
        return 3 * kw["H"] * kw["W"] * kw["C"]
    if check == "im2col":
        ho = (kw["H"] + 2 * kw["pad"] - kw["k"]) // kw["s"] + 1
        wo = (kw["W"] + 2 * kw["pad"] - kw["k"]) // kw["s"] + 1
        return 3 * kw["H"] * kw["W"] * kw["C"] + 2 * ho * wo * kw["k"] ** 2 * kw["C"]
    return PL._elems(check, kw)


def _sized(check, kw, n_full):
    if n_full is None:
        return kw, None
    tn = PL.conv_patch(kw["H"], kw["W"], kw["k"], kw["stride"], n_full)[2] if check == "conv" else 1
    n = PL._fit_n(n_full, _elems(check, kw), PL.MAX_ELEMS, tn)
    if n == n_full:
        return kw, None
    return {k: v for k, v in dict(kw, N=n).items() if k not in PL._COUNTS}, n_full


@functools.lru_cache(maxsize=None)
def shipped_keys():
    return {PL._key(c.check, c.kw, c.dtype) for c in PL.gpu_cases()} | {PL._key(c.check, c.kw, c.dtype) for c in PV.variant_cases()}


def eval_plan(tag):
    return plan_launches(tag, EVAL_BATCH, False, EVAL_DTYPE)


def variant(la):
    """what selects a launch's code path besides its shape: the kernel, its pointer mask and its mode arguments"""
    return la.kernel, la.ptrs, launch_modes(la)


@functools.lru_cache(maxsize=None)
def training_variants():
    return {variant(la) for la, _ in PL.harvest()} | {variant(la) for la, _ in harvest()}


def is_checked(la):
    if la.kernel == "dfd_bn_finalize":
        return la.shape[3] == 0          # the eval form; the training form stays excluded as in plan_launches.EXCLUDED
    return la.kernel in CHECKED or la.kernel in PV.EVAL_CHECKED


@functools.lru_cache(maxsize=None)
def gpu_cases():
    """list of plan_launches.Case, the shipped harness's tiering over the family plans (see the module docstring); `launches`
    lists what each case stands for: (Launch, dtype), ("class", kernel, class), ("eval", kernel, ptrs) or ("odd", kernel)"""
    cases = OrderedDict()
    shipped = shipped_keys()

    def add(check, kw, n_full, dtype, why):
        kw, reduced = _sized(check, kw, n_full)
        key = PL._key(check, kw, dtype)
        if key in shipped:
            return
        if key not in cases:
            cases[key] = PL.Case(None, check, dict(kw), dtype, [], reduced)
        cases[key].kw.update({k: v for k, v in kw.items() if k in PL._COUNTS})
        cases[key].launches.append(why)

    other = {"bf16": "fp16", "fp16": "bf16"}
    classes, band = OrderedDict(), []
    for (la, dtype), tgs in harvest().items():
        if la.kernel not in CHECKED:
            continue
        check, kw, n_full, cls = case_of(la, dtype, plan_launches(tgs[0]))
        if la.kernel in CONTRACTION:
            add(check, kw, n_full, dtype, (la, dtype))
            size = _elems(check, kw) * (n_full or 1) + kw.get("M", 0) * (kw.get("K", 0) + kw.get("N", 0) + kw.get("Nw", 0) + kw.get("Kw", 0))
            best = classes.get((la.kernel, cls, other[dtype]))
            if best is None or size < best[0]:
                classes[(la.kernel, cls, other[dtype])] = (size, check, kw, n_full)
        elif check in FP32:
            add(check, kw, None, "fp32", (la, dtype))
        else:
            band.append((check, kw, n_full, la, dtype))
    for (kernel, cls, dt), (_, check, kw, n_full) in classes.items():
        add(check, {k: v for k, v in kw.items() if k not in PL._COUNTS}, n_full, dt, ("class", kernel, cls))
    band.sort(key=lambda b: -b[1].get("HW", b[1].get("H", 0) * b[1].get("W", 0)))
    for check, kw, n_full, la, dtype in band:
        for dt in (dtype, other[dtype]):
            add(check, kw, n_full, dt, (la, dtype))
    # the average pool at an odd extent (clipped last windows, count without padding) at each of the plans' channel counts
    for C in sorted({kw["C"] for check, kw, _, _, _ in band if check == "avgpool2"}):
        for dt in ("bf16", "fp16"):
            add("avgpool2", dict(N=8, H=ODD_EXTENT, W=ODD_EXTENT + 2, C=C, add=True), None, dt, ("odd", "dfd_avgpool2_fwd"))
    # the eval form at batch 1 in fp16: variants (kernel, pointer mask, mode arguments) no training plan issues, in both 16-bit
    # types; the logits-only head and the eval BatchNorm finalisation at every shape
    trained = training_variants()
    for tag in tags():
        plan = eval_plan(tag)
        for la in plan:
            if not is_checked(la):
                continue
            check, kw, _, _ = case_of(la, EVAL_DTYPE, plan)
            if check in ("head_fwd", "bn_finalize_eval"):
                add(check, kw, None, "fp32", ("eval", la.kernel, la.ptrs))
            elif variant(la) not in trained:
                for dt in (("fp32",) if check in FP32 else ("bf16", "fp16")):
                    add(check, kw, None, dt, ("eval", la.kernel, la.ptrs))
    out = []
    for (check, _, dtype), c in cases.items():
        parts = ["%s=%s" % (k, str(v).replace(" ", "")) for k, v in c.kw.items() if k not in PL._COUNTS]
        if c.n_full is not None:
            parts.append("reducedN%d" % c.n_full)
        out.append(c._replace(id="%s-%s-%s" % (check, dtype, ",".join(parts))))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# mode arguments: what a launch selects, and what its case runs
# ---------------------------------------------------------------------------------------------------------------------------
def launch_modes(la):
    """the arguments of a launch that select what the kernel computes (activation, BatchNorm input, optional operands), or
    None for a kernel without such arguments"""
    k, s, p = la.kernel, la.shape, la.ptrs
    if k == "dfd_dwconv_fwd":
        return ("act", s[6], "bn", p[1] == "p", "stats", p[5] == "p")
    if k == "dfd_dwconv_fwd_pad":
        return ("act", s[8], "bn", p[1] == "p", "stats", p[5] == "p")
    if k in ("dfd_dwconv_bwd", "dfd_dwconv_bwd_relu"):
        return ("bn", p[7] == "p", "add", p[11] == "p")
    if k == "dfd_bn_maxpool_add":
        return ("idx", p[7] == "p")
    if k == "dfd_col2im":
        return ("add", p[1] == "p")
    if k == "dfd_avgpool2_bwd_add":
        return ("add", p[1] == "p")
    if k in ("dfd_conv_tc", "dfd_gemm_tn", "dfd_gemm_tn_rowpack"):
        return ("stats", p[3] == "p")
    if k == "dfd_pool_se_relu":
        return ("act", s[4], "chunks", s[6])
    if k == "dfd_relu_se_bwd_reduce":
        return ("act", s[4], "g2", p[1] == "p")
    if BANDWIDTH.get(k) == "row":
        n_dt = {"dfd_pool": 4}.get(k, len(s) - 1)
        return ("args", tuple(v for i, v in enumerate(s[3:], 3) if i != n_dt), "ptrs", p)
    return None


def case_modes(la, check, kw):
    """the set of launch_modes that the checker `check` runs with these kwargs, for this launch's kernel"""
    k = la.kernel
    if k == "dfd_dwconv_fwd":
        if check == "dwconv_relu":
            return {("act", 2, "bn", kw["bn"], "stats", False)}
        act = 1 if kw["affine"] else 0
        return {("act", act, "bn", kw["affine"], "stats", st) for st in ((True, False) if not kw.get("stats", True) else (True,))}
    if k == "dfd_dwconv_fwd_pad":
        return {("act", 1, "bn", True, "stats", st) for st in ((True, False) if not kw["stats"] else (True,))}
    if k == "dfd_dwconv_bwd":
        return {("bn", kw["affine"], "add", kw["add"])}
    if k == "dfd_dwconv_bwd_relu":
        return {("bn", kw["bn"], "add", kw["add"])}
    if k == "dfd_bn_maxpool_add":
        return {("idx", kw["idx"])}
    if k in ("dfd_col2im", "dfd_avgpool2_bwd_add"):
        return {("add", kw["add"])}
    if k == "dfd_conv_tc":
        return {("stats", True), ("stats", False)}        # check_conv_implicit runs both forms
    if k in ("dfd_gemm_tn", "dfd_gemm_tn_rowpack"):
        return {("stats", kw["with_stats"])}
    if k == "dfd_pool_se_relu":
        return {("act", kw["act"], "chunks", kw["max_chunks"])}
    if k == "dfd_relu_se_bwd_reduce":
        return {("act", kw["act"], "g2", kw["two"])}
    if check == "row":
        return {("args", kw["args"], "ptrs", kw["ptrs"])}
    return set()
