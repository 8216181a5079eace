"""Host logic without a GPU: the C-ABI library loads and exports every symbol include/dfd_b200.h declares, the
ctypes signature table agrees with the header, and the engine's call plan (arenas, pointer arithmetic, argument
lists) builds for the BASELINE configurations."""
import os
import re

import pytest

from deepfake_detection_b200 import _lib
from deepfake_detection_b200.arch import get_spec, param_entries

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _protos():
    hdr = open(os.path.join(ROOT, "include", "dfd_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return re.findall(r"\b(?:int|const char\*)\s+(dfd_\w+)\s*\(([^)]*)\)\s*;", hdr)


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    names = [n for n, _ in _protos()]
    assert len(names) >= 30
    for n in names:
        assert hasattr(L.cdll, n), n
    assert L.cdll.dfd_abi_version() == 1
    assert L.stat_slots == 8


def test_ctypes_signatures_match_header():
    for name, params in _protos():
        if name == "dfd_last_error":
            continue
        codes = ""
        if params.strip() != "void":
            for p in params.split(","):
                p = p.strip()
                codes += "p" if "*" in p else "l" if "long long" in p else "f" if p.startswith("float") else \
                    "d" if p.startswith("double") else "i"
        assert _lib.SIGNATURES[name] == codes, name


@pytest.mark.parametrize("arch,batch,res", [("efficientnet_b0", 2, 64), ("efficientnet_b4", 1, 76),
                                             ("efficientnet_b0", 4, 224)])
def test_engine_plan_builds(arch, batch, res):
    from deepfake_detection_b200.engine import Engine
    eng = Engine(arch, batch, res, res, device="plan-only")
    spec = get_spec(arch)
    n = sum(int(__import__("math").prod(s)) for _, s, _ in param_entries(spec))
    assert eng.n_params >= n
    assert set(eng.p_off) == {e[0] for e in param_entries(spec)}
    assert eng.n_launch["fwd"] > 100 and eng.n_launch["bwd"] > 150
    # arena offsets never overlap
    spans = sorted((o, o + k) for o, _, k in eng.p_off.values())
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))


def test_no_oracle_on_product_path():
    """The product package must never import oracle/ (or fall back to torch compute)."""
    pkg = os.path.join(ROOT, "deepfake_detection_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def test_bench_native_arm_does_not_touch_the_oracle():
    """bench.py may execute oracle/ only on its cpu_baseline / --impl reference leg (run_reference)."""
    src = open(os.path.join(ROOT, "bench.py")).read()
    end = min(src.index("def cpu_baseline"), src.index("def run_reference"))
    native = src[src.index("def run_native"):end]
    assert src.index("def run_native") < end
    # the only mention allowed is the call into cpu_baseline(), which lives outside this function
    assert not re.search(r"(from|import)\s+oracle", native)


def test_row_pack_rule():
    """small-K pointwise convs are read `pack` rows at a time; pack must divide M and only applies below 64 channels"""
    from deepfake_detection_b200.engine import Engine
    assert Engine._row_pack(3211264, 16) == 4 and Engine._row_pack(802816, 24) == 8 and Engine._row_pack(3211264, 32) == 4
    assert Engine._row_pack(200704, 40) == 2 and Engine._row_pack(50176, 80) == 1 and Engine._row_pack(12544, 1152) == 1
    assert Engine._row_pack(802816 + 4, 24) == 4 and Engine._row_pack(7, 16) == 1        # halves until it divides M
    for M in (49, 50, 52, 56):
        for K in (8, 16, 24, 32, 40, 48, 56):
            assert M % Engine._row_pack(M, K) == 0


def test_plan_uses_the_fused_and_packed_kernels():
    """EfficientNet-B0 plan: every expansion block's depthwise backward is ONE fused launch, small-K pointwise convs go
    through the row-packed GEMM with block-diagonal weights registered for refresh, weight gradients use the tensor-core kernel."""
    from deepfake_detection_b200.engine import Engine
    eng = Engine("efficientnet_b0", 4, 224, 224, device="plan-only")
    names_f = [op[1] for op in eng.fwd_ops]
    names_b = [op[1] for op in eng.bwd_ops]
    assert names_b.count("dfd_dwconv_bwd") == 16 and "dfd_dwconv_wgrad" not in names_b and "dfd_dwconv_dgrad" not in names_b
    assert names_f.count("dfd_gemm_tn_rowpack") >= 5 and names_b.count("dfd_gemm_tn_rowpack") >= 4
    assert names_b.count("dfd_gemm_wgrad") == 33 and "dfd_gemm_wgrad_mma" not in names_b
    reg = eng._bd_reg
    assert len(reg) == names_f.count("dfd_gemm_tn_rowpack") + names_b.count("dfd_gemm_tn_rowpack")
    for (B, Nn, K, pack), t in reg.items():
        assert t.numel() == pack * Nn * pack * K and (4 * 224 * 224 // 4) % 1 == 0
    # a second plan over the same weights (other batch size) shares the registry of the owner
    eng2 = Engine("efficientnet_b0", 2, 224, 224, device="plan-only", share_from=eng)
    assert eng2.params32 is eng.params32 and not hasattr(eng2, "_bd_reg") and len(eng._bd_reg) >= len(reg)
    # an arena-only engine (what NativeModel.engine / the optimizer hold) owns weights but no plan and no activations
    ar = Engine("efficientnet_b0", 1, device="plan-only", params_only=True)
    assert ar.params_only and ar.fwd_ops == [] and not hasattr(ar, "acts") and ar.n_params == eng.n_params
    eng3 = Engine("efficientnet_b0", 2, 64, 64, device="plan-only", share_from=ar)
    assert eng3.arena is ar and eng3.grads32 is ar.grads32 and len(ar._bd_reg) > 0 and len(ar._stem_reg) == 1


def test_resnet_plan_validation_checks_argument_types(monkeypatch):
    """a ResNet plan is held to the ABI table's argument codes, not only to its argument counts"""
    from deepfake_detection_b200.engine import Engine
    _lib.lib()              # bind the library with the real table first: the patched one must only reach the plan check
    codes = _lib.SIGNATURES["dfd_bn_finalize"]
    monkeypatch.setitem(_lib.SIGNATURES, "dfd_bn_finalize", codes[:2] + "l" + codes[3:])   # the float count no longer fits
    with pytest.raises(AssertionError, match="does not fit code 'l'"):
        Engine("resnet18", 2, 64, 64, device="plan-only")


def test_resnet_eval_forward_passes_no_statistics_to_the_implicit_conv():
    """dfd_conv_tc writes batch statistics in training only: an eval forward passes NULL for them, so it does not accumulate
    them. No producer is planned with a finalisation descriptor: a dfd_bn_finalize launch of its own follows it"""
    from deepfake_detection_b200.engine import Engine
    eng = Engine("resnet50", 2, 160, 160, device="plan-only")
    convs = [a for _, n, a in eng.fwd_ops if n == "dfd_conv_tc"]
    assert len(convs) == 16 + 3          # every 3x3 convolution and the three strided 1x1 downsamples
    for a in convs:
        train, ev = eng.launch_args("dfd_conv_tc", a, True), eng.launch_args("dfd_conv_tc", a, False)
        assert ev[:-3] == train[:-3] and ev[-3:] == (None, None, None)
        assert train[-3] and train[-2] and train[-1] is None


def test_package_reads_no_environment():
    """what a plan launches follows from the Engine / Trainer arguments alone: no module of the package reads the
    environment (the kernels' own launch-geometry overrides under csrc/ are C code)"""
    pkg = os.path.join(ROOT, "deepfake_detection_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"\b(environ|getenv)\b", src), f


# environment variables that earlier versions of the plan builders, the Trainer and the DDP reducer read, each at a
# non-default value
RETIRED_VARIABLES = dict(DFD_NONDET="1", DFD_WGRAD_MMA="1", DFD_NO_ROWPACK="1", DFD_SE_FUSED="1", DFD_DW_SPLIT_BWD="1",
                         DFD_NO_IMPLICIT_CONV="1", DFD_NO_IMPLICIT_WGRAD="1", DFD_NO_IMPLICIT_S2="1",
                         DFD_NO_IMPLICIT_S2_DGRAD="1", DFD_NO_DGRAD_ADD="1", DFD_NO_RELU_FUSE="1", DFD_DDP_SPLIT_GRAPH="1",
                         DFD_DDP_BUCKET_MB="1")


@pytest.mark.parametrize("fused_finalize", ["1", "gemm"])
def test_retired_environment_variables_leave_the_plan_alone(monkeypatch, fused_finalize):
    """plan-only engines built with every retired variable set issue the same launches as without them"""
    from plan_launches import _split
    from deepfake_detection_b200.engine import Engine, base_name

    def launches(arch, H, W, kw):
        eng = Engine(arch, 2, H, W, device="plan-only", **kw)
        return [(n, _split(base_name(n), a)) for _, n, a in eng.fwd_ops + eng.bwd_ops]

    configs = [("efficientnet_b0", 64, 64, dict(drop_rate=0.2, drop_path_rate=0.2)),
               ("tf_efficientnet_b0", 66, 96, {}),
               ("resnet50", 160, 160, dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.1)),
               ("resnet18", 64, 64, dict(gemm_impl="mma"))]
    for name in list(RETIRED_VARIABLES) + ["DFD_FUSED_FINALIZE"]:
        monkeypatch.delenv(name, raising=False)
    plain = [launches(*c) for c in configs]
    for name, value in dict(RETIRED_VARIABLES, DFD_FUSED_FINALIZE=fused_finalize).items():
        monkeypatch.setenv(name, value)
    for c, ref in zip(configs, plain):
        assert launches(*c) == ref, c[0]


def test_resnet_refuses_sync_bn_over_several_ranks(monkeypatch):
    """the ResNet plan has no synchronised BatchNorm: over more than one rank it refuses, instead of running rank-local
    statistics; on one rank sync_bn is plain BatchNorm, as in torch"""
    import torch.distributed as dist
    from deepfake_detection_b200.engine import Engine
    Engine("resnet18", 2, 64, 64, device="plan-only", sync_bn=True)
    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda *a, **k: 2)
    for kw in (dict(), dict(params_only=True)):
        with pytest.raises(_lib.NativeError, match="sync_bn over 2 ranks"):
            Engine("resnet18", 2, 64, 64, device="plan-only", sync_bn=True, **kw)
    eng = Engine("efficientnet_b0", 2, 64, 64, device="plan-only", sync_bn=True)
    assert eng.sync_world == 2 and any(n == "dfd_bn_finalize_sync" for _, n, _ in eng.fwd_ops)


def test_resnet_stem_gemm_is_never_row_packed():
    """one input channel gives the ResNet stem GEMM K = 56; the ResNet plan keeps the plain GEMM there"""
    from deepfake_detection_b200.engine import Engine
    eng = Engine("resnet18", 2, 64, 64, device="plan-only", in_chans=1)
    names = [n for _, n, _ in eng.fwd_ops + eng.bwd_ops]
    assert "dfd_gemm_tn_rowpack" not in names and not getattr(eng, "_bd_reg", None)
