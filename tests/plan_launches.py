"""The kernel launches of the shipped training plans, harvested on the CPU (plan-only engines: the built library, no GPU).

`harvest()` builds the call plan of every configuration in CONFIGS and returns its distinct launches: the kernel name, the
non-pointer arguments in ABI order (`shape`), which pointer operands are present (`ptrs`, 'p' or '0' per pointer argument:
it selects kernel variants, e.g. the depthwise backward's mode 0 / mode 1) and the 16-bit type the configuration trains in.
Pointers are told from shape arguments by the ctypes signature codes of `_lib.SIGNATURES` ('p'), never by Python type: a
device pointer is a plain int in the plan.

`gpu_cases()` turns the launches into the GPU checks of tests/test_plan_launches_gpu.py (tiering: see its docstring);
tests/test_plan_launches_cpu.py holds the two to each other.
"""
import functools
from collections import OrderedDict, namedtuple

from deepfake_detection_b200 import _lib
from deepfake_detection_b200.engine import base_name

# (tag, arch, batch, resolution, dtype, extra Engine kwargs): BASELINE configs 2/3 (B0; the per-GPU batch of the DDP config is
# also 256), config 5 (B4 fp16), config 4 (ResNet-50), ResNet-18, and the production model of test_production_model_gpu.py
CONFIGS = [
    ("b0", "efficientnet_b0", 256, 224, "bf16", {}),
    ("b4", "efficientnet_b4", 128, 380, "fp16", {}),
    ("r50", "resnet50", 256, 224, "bf16", {}),
    ("r18", "resnet18", 256, 224, "bf16", {}),
    ("dfv4", "efficientnet_deepfake_v4", 3, 600, "bf16", {"in_chans": 12}),
]

# configuration tables by name: tests/family_launches.py registers the model families' table as "family"
TABLES = {"shipped": CONFIGS}

Launch = namedtuple("Launch", "kernel shape ptrs")


def _split(name, args):
    codes = _lib.SIGNATURES[name]
    assert len(codes) == len(args) + 1, (name, codes, args)       # the trailing code is the stream
    shape, ptrs = [], ""
    for v, c in zip(args, codes):
        if isinstance(v, tuple) and v[0] == "TRAIN_ONLY":             # a training-only operand: present in the training step
            v = v[1]
        if c == "p":
            ptrs += "0" if v is None else "p"
        else:
            shape.append(1 if v == "TRAINING" else v)
    return Launch(name, tuple(shape), ptrs)


@functools.lru_cache(maxsize=2)         # the training and the eval harvest of one plan share its engine
def _plan_engine(tag, batch, dtype, table="shipped"):
    from deepfake_detection_b200.engine import Engine
    _, arch, b, res, dt, kw = next(c for c in TABLES[table] if c[0] == tag)
    return Engine(arch, batch or b, res, res, device="plan-only", dtype=dtype or dt, **kw)


@functools.lru_cache(maxsize=None)
def plan_launches(tag, batch=None, training=True, dtype=None, table="shipped"):
    """OrderedDict Launch -> number of times one step issues it, for one configuration of TABLES[table] (at another batch /
    16-bit type when given). Training: the forward and backward plan as built. Eval: the forward ops as Engine.launch_args
    rewrites them for eval mode, then the logits-only head (Engine.head(False))."""
    eng = _plan_engine(tag, batch, dtype, table)
    out = OrderedDict()

    def add(la):
        out[la] = out.get(la, 0) + 1

    for _, name, args in list(eng.fwd_ops) + (list(eng.bwd_ops) if training else []):
        if name.startswith("ALLREDUCE"):
            continue
        if not training:
            args = eng.launch_args(name, args, False)
            if args is None:
                continue
        add(_split(base_name(name), args))
    if not training:
        real = _lib.call
        _lib.call = lambda name, *args: add(_split(name, args[:-1]))          # the stream last
        try:
            eng.head(False, stream=0)
        finally:
            _lib.call = real
    return out


def config_dtype(tag):
    return next(c[4] for c in CONFIGS if c[0] == tag)


@functools.lru_cache(maxsize=None)
def harvest():
    """OrderedDict (Launch, dtype) -> tags of the configurations that issue it (deduplicated across fwd / bwd / configs)"""
    out = OrderedDict()
    for tag, *_ in CONFIGS:
        for la in plan_launches(tag):
            out.setdefault((la, config_dtype(tag)), []).append(tag)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------------
# kernel -> checker of tests/gpu_checks.py that runs it (through tests/test_plan_launches_gpu.py)
CONTRACTION = {
    "dfd_gemm_tn": "gemm",
    "dfd_gemm_tn_rowpack": "gemm",
    "dfd_gemm_wgrad": "wgrad",
    "dfd_dwconv_fwd": "dwconv",
    "dfd_dwconv_bwd": "dwconv",
    "dfd_conv_tc": "conv",
    "dfd_conv_wgrad_tc": "conv",
    "dfd_conv_dgrad_s2_tc": "conv",
    "dfd_conv1x1_dgrad_add": "conv1x1_dgrad_add",
    "dfd_stem_im2col": "stem_gemm",
    "dfd_unpad_grad": "stem_gemm",
}
# The per-row kernels run with the launch's own argument pattern (activation, residual mode, chunk count, which optional
# operands are present): those select the kernel instantiation (e.g. bn_act.cu:855), so a case keeps all of them
BANDWIDTH = {
    "dfd_bn_act": "row",
    "dfd_act_bwd": "row",
    "dfd_bn_bwd_reduce": "row",
    "dfd_bn_bwd_apply": "row",
    "dfd_pool": "row",
    "dfd_se_bwd_reduce": "row",
    "dfd_relu_bn_bwd_reduce": "relu_bn_bwd_reduce",
    "dfd_maxpool_fwd": "maxpool",
    "dfd_maxpool_bwd": "maxpool",
    "dfd_se_fc_fwd": "se_fc",
    "dfd_se_fc_bwd": "se_fc",
    "dfd_head_bwd": "head",
}
CHECKED = dict(CONTRACTION, **BANDWIDTH)

# kernels of the plans that have no per-launch case here, and why
EXCLUDED = {
    "dfd_memset_async": "cudaMemsetAsync of a gradient buffer; no kernel of ours",
    "dfd_bn_finalize": "one thread per channel (shape = C only): test_kernels_gpu's test_bn_chain / test_fused_bn_finalize",
    "dfd_bn_bwd_finalize": "one thread per channel (shape = C only): test_kernels_gpu's test_bn_chain / test_fused_bn_finalize",
    "dfd_ordered_reduce": "runs inside every wgrad, dwconv and conv case at that launch's split / part count",
    "dfd_unpack_grad": "permutation of the packed conv weight gradient: runs inside every conv case",
    "dfd_add_inplace": "elementwise residual add: checked bit for bit inside check_relu_bn_bwd_reduce(two=True)",
    "dfd_pool_bwd": "broadcast of dpooled / HW: check_maxpool_relu_pool checks it exactly",
}

# Operands of one case (inputs and outputs together) above this many elements: the batch is reduced (see _fit_n)
MAX_ELEMS = 512 * 2 ** 20

Case = namedtuple("Case", "id check kw dtype launches n_full")


def _n_class(N, tn):
    """the smallest batch >= tn with the same remainder modulo the image-stacking factor tn"""
    return tn + N % tn if tn > 1 else 1


def _fit_n(N, per_image, limit, tn=1):
    """largest batch <= N with per_image * batch <= limit, keeping N mod tn (the last M tile of stacked images)"""
    if N * per_image <= limit:
        return N
    n = max(int(limit // per_image), _n_class(N, tn))
    while tn > 1 and n % tn != N % tn:
        n -= 1
    return max(n, _n_class(N, tn))


def conv_patch(H, W, k, s, N):
    """output patch (TW, TH, TN) of dfd_conv_tc's M tile: gemm_tc.cu:729-738 (not exported)"""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    TW = Wo if Wo <= 128 else 128
    max_th = max(128 // TW, 1)
    ty = (Ho + max_th - 1) // max_th
    TH = (Ho + ty - 1) // ty
    TN = 128 // (TW * TH) if (TH == Ho and TW == Wo) else 1
    return TW, TH, max(1, min(TN, N))


def dw_tile(H, W, k, s):
    """forward tile (TW, TH) of the depthwise kernels: dwconv.cu:787-790 (fill_geom, not exported)"""
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    TW = 8 if Wo <= 8 else (16 if (Wo <= 16 or s == 2) else 32)
    TH = Ho if Ho < 8 else 8
    if s == 2 and k == 5 and Ho >= 8:
        TH = 4
    return TW, TH


def dw_bwd_tile(H, W):
    """tile (TW, TH) of the depthwise backward, which partitions the INPUT pixels: dwconv.cu:785-788 with input_space"""
    return (8 if W <= 8 else (16 if W <= 16 else 32)), (H if H < 8 else 8)


def dw_cpw(C):
    """channel pairs per warp sub-strip: half of the exported channels per CTA"""
    return _lib.lib().cdll.dfd_dwconv_block_channels(C) // 2


def _case_of(la, dtype, plan=None):
    """(check, kwargs, n_full, dispatch class) exercising this launch; kwargs at the full batch. `plan`: the launches of the
    plan that issues it (default: the shipped training plans)"""
    k, s = la.kernel, la.shape
    if k == "dfd_gemm_tn":
        M, N, K = s[0], s[1], s[2]
        bn = N if N <= 128 else 128
        bn = (bn + 15) // 16 * 16
        cls = ("tc", 64 if bn <= 64 else 128, N % bn != 0, K % 64 != 0)       # gemm_tc.cu:688,769 (MMA N template, n tail)
        return "gemm", dict(impl="tc", M=M, K=K, N=N, with_stats=la.ptrs[3] == "p"), None, cls
    if k == "dfd_gemm_tn_rowpack":
        M, N, K, pack = s[0], s[1], s[2], s[3]
        return "gemm", dict(impl="rowpack%d" % pack, M=M, K=K, N=N, with_stats=la.ptrs[3] == "p"), None, ("rowpack", pack, N > 64)
    if k == "dfd_gemm_wgrad":
        M, Nw, Kw, nbytes = s[0], s[1], s[2], s[4]
        return "wgrad", dict(M=M, Nw=Nw, Kw=Kw, splits=nbytes // (4 * Nw * Kw)), None, ("wgrad", Kw >= 128, Kw % 16 != 0, Nw > 128)
    if k == "dfd_dwconv_fwd":
        # act_in and the BatchNorm operands together select the staged input (dwconv.cu:891-895): raw, BN + Swish, BN + ReLU or
        # ReLU only; any other pattern is a form no checker runs
        assert la.ptrs[2] == la.ptrs[1] and la.ptrs[3:5] == "pp" and la.ptrs[6] == la.ptrs[5], la
        assert la.ptrs[7] == "0" or la.ptrs[5] == "p", la
        form = {(0, "0"): "raw", (1, "p"): "bn_swish", (2, "p"): "bn_relu", (2, "0"): "relu"}[(s[6], la.ptrs[1])]
        if form in ("bn_relu", "relu"):
            return _dw_relu_case(la)
    if k in ("dfd_dwconv_fwd", "dfd_dwconv_bwd"):
        N, H, W, C, kk, st = s[:6]
        affine = (s[6] == 1) if k == "dfd_dwconv_fwd" else la.ptrs[7] == "p"
        # mode 0 (raw input) adds the residual gradient when `add` is given; the forward does not say which, so its case runs
        # the backward with it (the plan's add-less mode-0 launches have cases of their own)
        add = not affine and (k == "dfd_dwconv_fwd" or la.ptrs[11] == "p")
        kw = dict(N=N, H=H, W=W, C=C, k=kk, s=st, affine=affine, add=add)
        if k == "dfd_dwconv_fwd" and la.ptrs[5] == "0":        # the eval form: no batch statistics, no finalisation
            kw["stats"] = False
        if k == "dfd_dwconv_fwd":
            return "dwconv", kw, N, ("dw_fwd", dw_cpw(C), dw_tile(H, W, kk, st), kk, st, affine)
        kw["ws_bytes"] = s[7]
        return "dwconv", kw, N, ("dw_bwd", dw_cpw(C), dw_bwd_tile(H, W), kk, st, affine, add)
    if k == "dfd_dwconv_bwd_relu":
        return _dw_relu_case(la)
    if k in ("dfd_conv_tc", "dfd_conv_wgrad_tc"):
        # dfd_conv_tc with statistics or without (the eval form, and the stride-1 input gradient): check_conv_implicit runs
        # both and holds them to the same bits
        assert k != "dfd_conv_tc" or la.ptrs in ("ppppp0", "pppppp", "ppp000"), la
        N, H, W, Cin, Cout, kk, st = s[:7]
        kw = dict(N=N, H=H, W=W, Cin=Cin, Cout=Cout, k=kk, stride=st)
        if k == "dfd_conv_wgrad_tc":
            kw["splits"] = s[8] // (4 * Cout * kk * kk * Cin)
        return "conv", kw, N, ("conv", conv_patch(H, W, kk, st, N), st, kk)
    if k == "dfd_conv_dgrad_s2_tc":
        N, H, W, Cin, Cout = s[:5]
        return "conv", dict(N=N, H=H, W=W, Cin=Cin, Cout=Cout, k=3, stride=2), N, ("conv", conv_patch(H, W, 3, 2, N), 2, 3)
    if k == "dfd_conv1x1_dgrad_add":
        N, H, W, Cin, Cout, st = s[:6]
        return "conv1x1_dgrad_add", dict(N=N, H=H, W=W, Cin=Cin, Cout=Cout, stride=st), N, ("c1x1", st)
    if k == "dfd_stem_im2col":
        N, Cin, H, W, kk, st, pad, Kp = s[:8]
        cout, pack = _stem_gemm_form(N, Cin, H, W, kk, st, pad, Kp, plan)
        return "stem_gemm", dict(N=N, Cin=Cin, H=H, W=W, Cout=cout, k=kk, s=st, pad=pad, pack=pack), N, ("stem", Cin, kk, pack)
    if k == "dfd_unpad_grad":            # the stem case of the configuration that issues it
        if plan is None:
            tag = next(t for t, *_ in CONFIGS if config_dtype(t) == dtype and la in plan_launches(t))
            plan = plan_launches(tag)
        return _case_of(next(x for x in plan if x.kernel == "dfd_stem_im2col"), dtype, plan)
    if CHECKED.get(k) == "row":
        # every non-pointer argument after (n, hw, C) but the dtype (the last one, except before dfd_pool's chunk count)
        n_dt = {"dfd_pool": 4}.get(k, len(s) - 1)
        args = tuple(v for i, v in enumerate(s[3:], 3) if i != n_dt)
        return "row", dict(kernel=k, N=s[0], HW=s[1], C=s[2], args=args, ptrs=la.ptrs), s[0], None
    if k == "dfd_relu_bn_bwd_reduce":
        return "relu_bn_bwd_reduce", dict(N=s[0], HW=s[1], C=s[2], two=la.ptrs[1] == "p"), s[0], None
    if k in ("dfd_maxpool_fwd", "dfd_maxpool_bwd"):
        return "maxpool", dict(N=s[0], H=s[1], W=s[2], C=s[3]), s[0], None
    if k in ("dfd_se_fc_fwd", "dfd_se_fc_bwd"):
        return "se_fc", dict(N=s[0], C=s[1], Cse=s[2]), None, None
    if k == "dfd_head_bwd":
        assert s[2] == 2, la                 # the 2-class head of the shipped configurations (check_head)
        return "head", dict(N=s[0], F=s[1]), None, None
    if k == "dfd_head_fwd":                  # logits only (validate / test_img): no target, loss, count or dlogits
        assert s[2] == 2 and la.ptrs == "pppp" + "0" * 6, la
        return "head_fwd", dict(N=s[0], F=s[1]), None, None
    if k == "dfd_bn_finalize":               # eval form: scale / shift from the running statistics
        assert s[3] == 0 and la.ptrs[:2] == "00", la
        return "bn_finalize_eval", dict(C=s[4]), None, None
    raise KeyError(k)


def _dw_relu_case(la):
    """the depthwise pair of a separable convolution whose input passes a ReLU (dwconv.cu:571-575): `bn` = the input is
    relu(scale*x + shift) (mode 2, BN-backward sums of gx), else relu(x) (mode 3, the identity-path gradient `add` when given).
    The forward does not say whether its backward adds: its case runs the backward with `add` in mode 3."""
    s, p = la.shape, la.ptrs
    N, H, W, C, kk, st = s[:6]
    if la.kernel == "dfd_dwconv_fwd":
        bn = p[1] == "p"
        assert p[5:8] == "000", la                     # no statistics: the ReLU forward rejects them (dwconv.cu:892)
        kw = dict(N=N, H=H, W=W, C=C, k=kk, s=st, bn=bn, add=not bn)
        return "dwconv_relu", kw, N, ("dw_relu_fwd", dw_cpw(C), dw_tile(H, W, kk, st), bn)
    assert la.kernel == "dfd_dwconv_bwd_relu", la
    # gy is the gradient of the depthwise output itself: no folded BatchNorm backward (yout, cA, cB, cC absent), no fin
    bn = p[7] == "p"
    assert p[:5] == "p0000" and p[5:7] == "pp" and p[7:11] == ("pppp" if bn else "0000") and p[12:14] == "pp", la
    assert p[14:16] == ("pp" if bn else "00") and p[16] == "p" and p[17] == "0" and not (bn and p[11] == "p"), la
    kw = dict(N=N, H=H, W=W, C=C, k=kk, s=st, bn=bn, add=p[11] == "p", ws_bytes=s[7])
    return "dwconv_relu", kw, N, ("dw_relu_bwd", dw_cpw(C), dw_bwd_tile(H, W), bn, p[11] == "p")


def _stem_gemm_form(N, Cin, H, W, k, s, pad, Kp, plan=None):
    """(Cout, pack) of the stem GEMM the plan runs on these columns: pack 1 = dfd_gemm_tn, else dfd_gemm_tn_rowpack"""
    M = N * ((H + 2 * pad - k) // s + 1) * ((W + 2 * pad - k) // s + 1)
    # the first such GEMM in plan order is the stem's (it follows the im2col); an eval plan's writes no statistics
    for launches in ([plan] if plan is not None else [plan_launches(tag) for tag, *_ in CONFIGS]):
        for la in launches:
            if la.kernel in ("dfd_gemm_tn", "dfd_gemm_tn_rowpack") and la.shape[0] == M and la.shape[2] == Kp and \
                    (la.ptrs[3] == "p" or plan is not None):
                return la.shape[1], (la.shape[3] if la.kernel == "dfd_gemm_tn_rowpack" else 1)
    raise KeyError((N, Cin, H, k))


def _elems(check, kw):
    """elements of the operands one case allocates per image (inputs + outputs of the kernels it runs)"""
    if check == "dwconv":
        pad = (kw["k"] - 1) // 2
        ho = (kw["H"] + 2 * pad - kw["k"]) // kw["s"] + 1
        wo = (kw["W"] + 2 * pad - kw["k"]) // kw["s"] + 1
        return 2 * kw["C"] * (kw["H"] * kw["W"] + ho * wo)
    if check == "conv":
        pad = (kw["k"] - 1) // 2
        ho = (kw["H"] + 2 * pad - kw["k"]) // kw["stride"] + 1
        wo = (kw["W"] + 2 * pad - kw["k"]) // kw["stride"] + 1
        # x, y, dy, dx and the im2col columns [Ho*Wo, k*k*Cin] of the bit-identity cross-check
        return 2 * (kw["H"] * kw["W"] * kw["Cin"] + ho * wo * kw["Cout"]) + ho * wo * kw["k"] ** 2 * kw["Cin"]
    if check == "conv1x1_dgrad_add":
        ho, wo = (kw["H"] - 1) // kw["stride"] + 1, (kw["W"] - 1) // kw["stride"] + 1
        return 2 * kw["H"] * kw["W"] * kw["Cin"] + ho * wo * kw["Cout"]
    if check == "stem_gemm":
        ho = (kw["H"] + 2 * kw["pad"] - kw["k"]) // kw["s"] + 1
        wo = (kw["W"] + 2 * kw["pad"] - kw["k"]) // kw["s"] + 1
        kp = (kw["Cin"] * kw["k"] ** 2 + 7) // 8 * 8
        return kw["Cin"] * kw["H"] * kw["W"] + ho * wo * (kp + kw["Cout"])
    if check in ("row", "relu_bn_bwd_reduce"):
        return 4 * kw["HW"] * kw["C"]
    if check == "maxpool":
        return 2 * kw["H"] * kw["W"] * kw["C"]
    return 0


def _sized(check, kw, n_full):
    """the case's kwargs with the batch reduced where the operands or the fp64 reference would exceed the budget"""
    if n_full is None:
        return kw, None
    tn = 1
    if check == "conv":              # the conv's M tiles stack tn whole images (gemm_tc.cu:736-738): keep N mod tn
        tn = conv_patch(kw["H"], kw["W"], kw["k"], kw["stride"], n_full)[2]
    n = _fit_n(n_full, _elems(check, kw), MAX_ELEMS, tn)
    if n == n_full:
        return kw, None
    # split / part counts follow the batch: only asserted at the exact shape
    return {k: v for k, v in dict(kw, N=n).items() if k not in _COUNTS}, n_full


_COUNTS = ("splits", "ws_bytes")      # asserted by a case, not part of what it runs


def _key(check, kw, dtype):
    return (check, tuple(sorted((k, v) for k, v in kw.items() if k not in _COUNTS)), dtype)


@functools.lru_cache(maxsize=None)
def gpu_cases():
    """list of Case: every contraction launch at its shape in its configuration's dtype, one case per dispatch class in the
    other dtype (the smallest launch of the class), one bandwidth case per distinct shape in each dtype (largest HW first)"""
    cases = OrderedDict()

    def add(check, kw, n_full, dtype, launch):
        kw, reduced = _sized(check, kw, n_full)
        key = _key(check, kw, dtype)
        if key not in cases:
            cases[key] = Case(None, check, dict(kw), dtype, [], reduced)
        cases[key].kw.update({k: v for k, v in kw.items() if k in _COUNTS})
        cases[key].launches.append(launch)

    other = {"bf16": "fp16", "fp16": "bf16"}
    classes = OrderedDict()
    band = []
    for (la, dtype), _ in harvest().items():
        if la.kernel not in CHECKED:
            continue
        check, kw, n_full, cls = _case_of(la, dtype)
        if la.kernel in CONTRACTION:
            add(check, kw, n_full, dtype, (la, dtype))
            size = _elems(check, kw) * (n_full or 1) + kw.get("M", 0) * (kw.get("K", 0) + kw.get("N", 0) + kw.get("Nw", 0) + kw.get("Kw", 0))
            best = classes.get((la.kernel, cls, other[dtype]))
            if best is None or size < best[0]:
                classes[(la.kernel, cls, other[dtype])] = (size, check, kw, n_full)
        elif check in ("se_fc", "head"):         # fp32 kernels: once per shape
            add(check, kw, None, "fp32", (la, dtype))
        else:
            band.append((check, kw, n_full, la, dtype))
    for (kernel, cls, dt), (_, check, kw, n_full) in classes.items():
        kw = {k: v for k, v in kw.items() if k not in _COUNTS}
        add(check, kw, n_full, dt, ("class", kernel, cls))
    band.sort(key=lambda b: -b[1].get("HW", b[1].get("H", 0) * b[1].get("W", 0)))
    for check, kw, n_full, la, dtype in band:
        for dt in (dtype, other[dtype]):
            add(check, kw, n_full, dt, (la, dtype))
    out = []
    for (check, _, dtype), c in cases.items():
        parts = ["%s=%s" % (k, str(v).replace(" ", "")) for k, v in c.kw.items() if k not in _COUNTS]
        if c.n_full is not None:
            parts.append("reducedN%d" % c.n_full)
        out.append(c._replace(id="%s-%s-%s" % (check, dtype, ",".join(parts))))
    return out
