"""The plans the runner builds besides the shipped training step, harvested on the CPU (plan-only engines), and their GPU cases.

`NativeModel.engine_for(n, h, w)` builds one plan per input shape, and `validate` / `test_img` run the forward in eval form
(Engine.launch_args). PLANS lists the set:
  * test_img: efficientnet_deepfake_v4 at batch 1, fp16, 600 x 600, eval (runners/test.py);
  * validation: every configuration in eval form at its batch and at twice it (the `-vb` multiplier);
  * short batches: every configuration, training and eval, at n in SHORT and b - 1 (the short last validation batch, and the
    short last training batch that the fused DDP path gives its own plan).

`batch_class` names the N-dependent dispatch decisions of a launch: where the library exports no rule it is restated here from
the .cu source (cited), as plan_launches.conv_patch / dw_tile do. `variant_cases()` turns the plans into the GPU checks of
tests/test_plan_variants_gpu.py; tests/test_plan_variants_cpu.py holds the two to each other:
  * every launch of the test_img plan at its exact shape in fp16;
  * every eval-form variant (kernel, pointer mask) that the shipped training plans lack, in both 16-bit types;
  * one case per (kernel, batch class, dtype) that no case of tests/test_plan_launches_gpu.py runs, at the smallest launch of
    that class, never at a reduced batch (the batch is what such a case tests);
  * the logits-only head at every (N, F) of the eval plans, the eval BatchNorm finalisation at every channel count.
"""
import functools
from collections import OrderedDict, namedtuple

import plan_launches as PL
from deepfake_detection_b200 import _lib

SMS = 132                           # DFD_SMS, common.cuh:143
ROWRED_WS_FLOATS = 4 << 20          # bn_act.cu:28
ROWRED_TICKETS = 65536              # bn_act.cu:29
SMALL_WS_FLOATS = 1 << 20           # se_head_optim.cu:19

SHORT = (1, 2, 3, 5, 7, 13)

Plan = namedtuple("Plan", "id tag batch dtype training")


@functools.lru_cache(maxsize=None)
def plans():
    out = [Plan("test_img", "dfv4", 1, "fp16", False)]
    for tag, _, b, _, dt, _ in PL.CONFIGS:
        out += [Plan("val", tag, n, dt, False) for n in (b, 2 * b)]
        for n in sorted(set(SHORT + (b - 1,)) - {b}):
            out += [Plan("short", tag, n, dt, True), Plan("short", tag, n, dt, False)]
    return tuple(out)


def launches(p):
    return PL.plan_launches(p.tag, p.batch, p.training, p.dtype)


def test_img_plan():
    return plans()[0]


# ---------------------------------------------------------------------------------------------------------------------------
# batch classes
# ---------------------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def make_geom(C, hw, n, target=SMS * 6, max_threads=256):
    """(RY, threads, chunks) of the per-row kernels: bn_act.cu:80-98"""
    V = C // 8
    RY = 1 if V >= max_threads else max_threads // V
    if max_threads > 256 and target > 1:
        target = target * 256 // max_threads
    RY = max(min(RY, 64, hw), 1)
    chunks = max(min(_cdiv(target, n), _cdiv(hw, RY)), 1)
    rpb = _cdiv(_cdiv(hw, chunks), RY) * RY
    return RY, V * RY, _cdiv(hw, rpb)


def row_maxt(hw, reduces_per_image):
    """bn_act.cu:74-79 (without the DFD_ROW_MAXT override)"""
    return 512 if reduces_per_image and hw >= 784 else 256


def pool_geom(C, hw, n, max_chunks):
    """(RY, threads, chunks, one CTA per image because n >= 296, scratch fallback): bn_act.cu:1088-1100"""
    chunked = max_chunks > 1 and n < 296 and n <= ROWRED_TICKETS
    RY, thr, chunks = make_geom(C, hw, n, 592 if chunked else 1, row_maxt(hw, True))
    if not chunked:
        chunks = 1
    if chunks > max_chunks and chunks > 1:
        rpb = _cdiv(_cdiv(hw, max_chunks), RY) * RY
        chunks = _cdiv(hw, rpb)
    fallback = chunks * n * C > ROWRED_WS_FLOATS
    return RY, thr, 1 if fallback else chunks, n >= 296, fallback


def se_bwd_geom(C, hw, n):
    """the same for dfd_se_bwd_reduce: bn_act.cu:1222-1223"""
    RY, thr, chunks = make_geom(C, hw, n, 1 if n >= 296 else 592, row_maxt(hw, True))
    fallback = chunks * n * C > ROWRED_WS_FLOATS or n > ROWRED_TICKETS
    if fallback:
        RY, thr, chunks = make_geom(C, hw, n, 1, row_maxt(hw, True))
    return RY, thr, chunks, n >= 296, fallback


# the geometry each per-row kernel launches with (bn_act.cu: dfd_bn_act :1061, dfd_act_bwd :1267, dfd_bn_bwd_reduce :1169,
# dfd_bn_bwd_apply :1208, dfd_relu_bn_bwd_reduce :1197)
_ROW_GEOM = {
    "dfd_bn_act": lambda C, hw, n: make_geom(C, hw, n, SMS * 6, row_maxt(hw, False)),
    "dfd_act_bwd": lambda C, hw, n: make_geom(C, hw, n),
    "dfd_bn_bwd_reduce": lambda C, hw, n: make_geom(C, hw, n, SMS * 6, row_maxt(hw, False)),
    "dfd_bn_bwd_apply": lambda C, hw, n: make_geom(C, hw, n),
    "dfd_relu_bn_bwd_reduce": lambda C, hw, n: make_geom(C, hw, n, SMS * 6, row_maxt(hw, False)),
}


def _row_class(kernel, N, HW, C, args=()):
    if kernel == "dfd_pool":
        RY, thr, chunks, big, fb = pool_geom(C, HW, N, args[1])
    elif kernel == "dfd_se_bwd_reduce":
        RY, thr, chunks, big, fb = se_bwd_geom(C, HW, N)
    else:
        (RY, thr, chunks), big, fb = _ROW_GEOM[kernel](C, HW, N), False, False
    return ("row", RY, thr, chunks > 1, big, fb)


def _tc_tiles(M, N):
    """M x N tiles of the tensor-core GEMM: gemm_tc.cu:769-771 (BLOCK_M 128, block_n = N rounded to 16, at most 128)"""
    return _cdiv(M, 128) * _cdiv(N, 128 if N > 128 else (N + 15) // 16 * 16)


def _gemm_class(M, N, pack, stats):
    """the row pack chosen (dfd_gemm_tn_rowpack runs M / pack rows of N * pack columns, gemm_tc.cu:823), an M tail tile, more
    tiles than SMs (the persistent grid, gemm_tc.cu:701-702), and the statistics epilogue"""
    M, N = M // pack, N * pack
    return ("gemm", pack, M % 128 != 0, _tc_tiles(M, N) > SMS, stats)


def batch_class(kernel, check, kw):
    """the N-dependent decisions that select code paths in the launch a case runs (`check`, `kw` as plan_launches._case_of)"""
    L = _lib.lib().cdll
    if check == "gemm":
        pack = 1 if kw["impl"] == "tc" else int(kw["impl"][len("rowpack"):])
        return _gemm_class(kw["M"], kw["N"], pack, kw["with_stats"])
    if check == "wgrad":
        return ("wgrad", kw["M"] % 128 != 0, L.dfd_gemm_wgrad_splits(kw["M"], kw["Nw"], kw["Kw"]))
    if check == "stem_gemm":
        M = kw["N"] * ((kw["H"] + 2 * kw["pad"] - kw["k"]) // kw["s"] + 1) * ((kw["W"] + 2 * kw["pad"] - kw["k"]) // kw["s"] + 1)
        Kp = (kw["Cin"] * kw["k"] ** 2 + 7) // 8 * 8
        return _gemm_class(M, kw["Cout"], kw["pack"], True) + (L.dfd_gemm_wgrad_splits(M, kw["Cout"], Kp),)
    if check == "conv":
        N, k, s = kw["N"], kw["k"], kw["stride"]
        TN = PL.conv_patch(kw["H"], kw["W"], k, s, N)[2]
        return ("conv", TN, N % TN != 0, L.dfd_conv_wgrad_splits(N, kw["H"], kw["W"], kw["Cin"], kw["Cout"], k, s))
    if check == "conv1x1_dgrad_add":
        M = kw["N"] * ((kw["H"] - 1) // kw["stride"] + 1) * ((kw["W"] - 1) // kw["stride"] + 1)
        return _gemm_class(M, kw["Cin"], 1, False)
    if check == "dwconv":
        # image groups of the backward: parts = tiles x groups (dwconv.cu:936-942,948-956)
        N, H, W = kw["N"], kw["H"], kw["W"]
        TW, TH = PL.dw_bwd_tile(H, W)
        groups = L.dfd_dwconv_bwd_parts(N, H, W, kw["C"], kw["k"], kw["s"]) // (_cdiv(W, TW) * _cdiv(H, TH))
        return ("dw", _cdiv(N, groups) > 1, kw.get("stats", True))
    if check == "row":
        return _row_class(kw["kernel"], kw["N"], kw["HW"], kw["C"], kw["args"])
    if check == "relu_bn_bwd_reduce":
        return _row_class("dfd_relu_bn_bwd_reduce", kw["N"], kw["HW"], kw["C"])
    if check == "head":
        # image splits of the 2-class weight gradient: se_head_optim.cu:875
        return ("head", 16 if kw["N"] >= 64 else (4 if kw["N"] >= 8 else 1))
    if check == "se_fc":
        # image splits of the SE weight gradient: se_head_optim.cu:833-836
        bx, N = _cdiv(kw["C"] * kw["Cse"], 128), kw["N"]
        ns = 16 if N >= 64 else (4 if N >= 8 else 1)
        while ns > 1 and (bx * ns > 2368 or ns * bx * 128 * 4 > SMALL_WS_FLOATS):
            ns >>= 1
        return ("se_fc", ns)
    return (check,)          # maxpool (one thread per output element), head_fwd, bn_finalize_eval: nothing follows N


# ---------------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------------
# kernels of these plans that the shipped training plans do not launch, and their checkers (tests/test_plan_variants_gpu.py)
EVAL_CHECKED = {"dfd_head_fwd": "head_fwd", "dfd_bn_finalize": "bn_finalize_eval"}
FP32 = ("se_fc", "head", "head_fwd", "bn_finalize_eval")

Case = namedtuple("Case", "id check kw dtype why")


def is_checked(la):
    """the training form of dfd_bn_finalize (batch statistics) stays excluded as in plan_launches.EXCLUDED"""
    if la.kernel == "dfd_bn_finalize":
        return la.shape[3] == 0
    return la.kernel in PL.CHECKED or la.kernel in EVAL_CHECKED


def case_of(la, dtype, p):
    """(check, kw, dtype the case runs in, batch class) of a launch of plan p, at its exact shape"""
    check, kw, _, _ = PL._case_of(la, dtype, launches(p))
    return check, kw, "fp32" if check in FP32 else dtype, batch_class(la.kernel, check, kw)


def size_of(check, kw):
    """elements a case allocates (the order in which the smallest launch of a class is chosen)"""
    return PL._elems(check, kw) * kw.get("N", 1) + kw.get("M", 0) * (kw.get("K", 0) + kw.get("N", 0) + kw.get("Nw", 0) + kw.get("Kw", 0))


@functools.lru_cache(maxsize=None)
def shipped_classes():
    """(kernel, batch class, dtype) that a case of tests/test_plan_launches_gpu.py runs"""
    out = set()
    for c in PL.gpu_cases():
        for la in c.launches:
            kernel = la[1] if la[0] == "class" else la[0].kernel
            out.add((kernel, batch_class(kernel, c.check, c.kw), c.dtype))
    return out


@functools.lru_cache(maxsize=None)
def shipped_masks():
    return {(la.kernel, la.ptrs) for la, _ in PL.harvest()}


@functools.lru_cache(maxsize=None)
def variant_cases():
    """list of Case; `why` lists what each case stands for: ("test_img", Launch), ("eval", kernel, ptrs), ("class", kernel,
    batch class), ("shape", kernel)"""
    cases = OrderedDict()

    def add(check, kw, dtype, why):
        key = PL._key(check, kw, dtype)
        if key not in cases:
            cases[key] = Case(None, check, dict(kw), dtype, [])
        cases[key].kw.update({k: v for k, v in kw.items() if k in PL._COUNTS})
        cases[key].why.append(why)

    tp = test_img_plan()
    have, masks = set(shipped_classes()), shipped_masks()
    for la in launches(tp):
        if is_checked(la):
            check, kw, dt, cls = case_of(la, tp.dtype, tp)
            add(check, kw, dt, ("test_img", la))
            have |= {(la.kernel, cls, dt), (la.kernel, la.ptrs, dt)}
    best = OrderedDict()            # class / eval variant -> (size, check, kw, dtype)

    def keep(key, check, kw, dt):
        size = size_of(check, kw)
        if key not in best or size < best[key][0]:
            best[key] = (size, check, kw, dt)

    for p in plans():
        for la in launches(p):
            if not is_checked(la):
                continue
            check, kw, dt, cls = case_of(la, p.dtype, p)
            if check in ("head_fwd", "bn_finalize_eval"):
                add(check, kw, dt, ("shape", la.kernel))
                continue
            if not p.training and (la.kernel, la.ptrs) not in masks:
                for d in ((dt,) if dt == "fp32" else ("bf16", "fp16")):
                    if (la.kernel, la.ptrs, d) not in have:
                        keep(("eval", la.kernel, la.ptrs, d), check, kw, d)
            if (la.kernel, cls, dt) not in have:
                keep(("class", la.kernel, cls, dt), check, kw, dt)
    for key, (_, check, kw, dt) in best.items():
        add(check, kw, dt, key[:-1])
    out = []
    for (check, _, dtype), c in cases.items():
        parts = ["%s=%s" % (k, str(v).replace(" ", "")) for k, v in c.kw.items() if k not in PL._COUNTS]
        out.append(c._replace(id="%s-%s-%s" % (check, dtype, ",".join(parts))))
    return out
