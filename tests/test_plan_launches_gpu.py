"""-m gpu: the kernels at the launch shapes of the shipped training plans (tests/plan_launches.py harvests them on the CPU).

Tiering (tests/test_plan_launches_cpu.py holds the case list to it):
  * contraction kernels (GEMMs, weight gradients, depthwise and dense convolutions, the stem): every distinct launch in its
    configuration's dtype, and one case per dispatch class in the other 16-bit type;
  * bandwidth kernels (BatchNorm / activation / pool / SE chain, ReLU-BN reduce, max-pool): one case per distinct launch in
    each 16-bit type, largest HW first. A per-row kernel's case keeps the launch's whole argument pattern (activation,
    residual mode, chunk count, which optional operands are present), which selects the kernel instantiation. The fp32 SE
    FCs and the 2-class head run once per shape.
A case runs the exact launch shape unless its operands exceed tests/plan_launches.MAX_ELEMS elements; then only the batch is
reduced (kept modulo the conv's image stacking) and the id says `reducedN<full>`. Split / part counts that follow the batch (dfd_gemm_wgrad_splits, dfd_conv_wgrad_splits,
dfd_dwconv_bwd_parts via the workspace size) are asserted equal to the plan's wherever the case runs the exact shape.

Tolerances are those of tests/gpu_checks.py / tests/test_kernels_gpu.py, unchanged: OUT16 = 2^-7 scaled max error of a bf16
output (2^-9 for the fp16 tensor-core GEMM, whose storage rounding is 4x finer), RED = 2e-3 rel-L2 of fp32 reductions of 16-bit
data, 1e-4 for fp32-accumulated weight gradients against fp64, and test_dwconv_fp16's bounds for the fp16 depthwise conv. One
bound is replaced: the depthwise forward on a BN + Swish input is held to the element-wise bound derived in
gpu_checks.check_dwconv (`fwd_ulp`), because the scaled 2^-7 bound does not follow from that arithmetic at 10^8 samples.
fp16 is held to fp16 precision, not to these bf16 bounds (bf16 assertions unchanged):
  * the tensor-core contractions (conv forward, the stride-1 / stride-2 input gradients, the GEMM + col2im input gradient,
    dfd_conv1x1_dgrad_add) to OUT_FP16_GEMM = 2^-9 scaled against fp64, as the fp16 GEMM;
  * the bandwidth kernels (the row kernels' 16-bit outputs, the max-pool gradient, the depthwise input gradient in each mode,
    the raw-input depthwise forward) to the element-wise bounds of tests/gpu_checks.py (`*_ulp` <= 1);
  * each of these also on the kernel's own output rounded through bf16, which must violate it (`*_bf16trip`): the check
    resolves a 16-bit path that rounds through bf16, which the bf16 bounds cannot.
Failure messages carry the whole result dict (str(r): pytest shortens a dict operand).
Every output buffer starts as NaN (an accumulated one from a known base), so an element that is never written fails.
"""
import pytest
import torch

import plan_launches as PL

pytestmark = pytest.mark.gpu

OUT16 = 2.0 ** -7
OUT_FP16_GEMM = 2.0 ** -9
RED = 2e-3
F32 = 2e-5

TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _gc():
    import gpu_checks
    return gpu_checks


def fp16_ulp(r, key):
    """an fp16 output within its element-wise bound, and the same output rounded through bf16 outside it"""
    assert r[key] <= 1.0 and r[key + "_bf16trip"] > 1.0, (key, str(r))


def fp16_scaled(r, key):
    """an fp16 tensor-core output within the fp16 GEMM's scaled bound, and the same output rounded through bf16 outside it"""
    assert r[key] < OUT_FP16_GEMM and r[key + "_bf16trip"] > OUT_FP16_GEMM, (key, str(r))


def _check_gemm(kw, dt):
    r = _gc().check_gemm(kw["impl"], kw["M"], kw["K"], kw["N"], dtype=TDT[dt], with_stats=kw["with_stats"])
    assert r["nan"] == 0 and r["out_max"] < (OUT_FP16_GEMM if dt == "fp16" else OUT16), str(r)
    if kw["with_stats"]:
        assert r["sum_rel"] < RED and r["sq_rel"] < RED, str(r)


def _check_wgrad(kw, dt):
    r = _gc().check_wgrad(kw["M"], kw["Nw"], kw["Kw"], dtype=TDT[dt], impl="dfd_gemm_wgrad", det=True)
    assert r["bitwise"] and r["rel"] < 1e-4 and r["vs_atomic"] < 1e-5, str(r)
    if "splits" in kw:
        assert r["splits"] == kw["splits"], (r["splits"], kw["splits"])


def _check_dwconv(kw, dt):
    """stats=False (the eval form of the forward): also the stats-less launch, bit for bit the output of the stats run"""
    stats = kw.get("stats", True)
    r = _gc().check_dwconv(kw["N"], kw["H"], kw["W"], kw["C"], kw["k"], kw["s"], dtype=TDT[dt], affine=kw["affine"], add=kw["add"],
                           stats=stats)
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fused_nan"] == 0 and r["det_nan"] == 0, str(r)
    assert stats or r["nostats_mismatch"] == 0, str(r)
    if dt == "fp16":      # test_dwconv_fp16's bounds
        assert r["fwd_rel"] < 2e-3 and r["dgrad_rel"] < 4e-3 and r["wgrad_rel"] < RED, str(r)
    else:
        assert r["dgrad_rel"] < 8e-3 and r["wgrad_rel"] < RED, str(r)
    # the activated input (BN + Swish) meets the element-wise bound derived in check_dwconv; a raw input only the output rounding
    assert r["fwd_ulp"] <= 1.0 if kw["affine"] else r["fwd_max"] < OUT16, str(r)
    if dt == "fp16":
        fp16_ulp(r, "dgrad_ulp")
        if not kw["affine"]:
            fp16_ulp(r, "fwd_ulp")
    assert r["sum_rel"] < RED and r["sq_rel"] < RED, str(r)
    assert r["fused_gx_diff"] == 0.0 and r["fused_wgrad_rel"] < RED, str(r)
    assert r["det_bitwise"] and r["det_vs_atomic"] < 1e-5 and r["det_gx_diff"] == 0.0, str(r)
    if kw["affine"]:
        assert r["bs1_rel"] < RED and r["bs2_rel"] < RED and r["fused_bs1_rel"] < RED and r["fused_bs2_rel"] < RED, str(r)
        assert r["det_bs1_rel"] < RED and r["det_bs2_rel"] < RED, str(r)
    if "ws_bytes" in kw:
        assert r["ws_bytes"] == kw["ws_bytes"], (r["ws_bytes"], kw["ws_bytes"])


def _check_conv(kw, dt):
    k, s = kw["k"], kw["stride"]
    r = _gc().check_conv_implicit(kw["N"], kw["H"], kw["W"], kw["Cin"], kw["Cout"], k, dtype=TDT[dt], stride=s)
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fwd_max"] < OUT16 and r["vs_im2col_mismatch"] == 0, str(r)
    assert r["nostats_mismatch"] == 0, str(r)
    assert r["sum_rel"] < 1e-6 and r["sq_rel"] < 1e-6, str(r)
    assert r["dgrad_rel"] < 6e-3, str(r)
    if s == 2 and k == 3:
        assert r["dgrad_vs_col2im"] < 8e-3, str(r)
    if dt == "fp16":
        fp16_scaled(r, "fwd_max")
        if s == 1 or k == 3:
            fp16_scaled(r, "dgrad_max")
        if s == 2 and k == 3:
            fp16_scaled(r, "col2im_dgrad_max")
    assert r["wgrad_rel"] < 1e-4 and r["wgrad_det_bitwise"] and r["wgrad_det_vs_atomic"] < 1e-5, str(r)
    if "splits" in kw:
        assert r["wgrad_splits"] == kw["splits"], (r["wgrad_splits"], kw["splits"])


def _check_conv1x1_dgrad_add(kw, dt):
    r = _gc().check_conv1x1_dgrad_add(kw["N"], kw["H"], kw["W"], kw["Cin"], kw["Cout"], kw["stride"], dtype=TDT[dt])
    assert r["nan"] == 0 and r["mismatch"] == 0 and r["rel"] < 6e-3, str(r)
    if dt == "fp16":        # the TMA reduction store adds in fp16 in L2
        fp16_scaled(r, "out_max")


def _check_stem_gemm(kw, dt):
    r = _gc().check_stem_gemm(kw["N"], kw["Cin"], kw["H"], kw["W"], kw["Cout"], kw["k"], kw["s"], kw["pad"], dtype=TDT[dt],
                              pack=kw["pack"])
    assert r["wpad_diff"] == 0.0 and r["wpad_tail"] == 0.0 and r["cols_nan"] == 0 and r["cols_tail"] == 0.0, str(r)
    assert r["cols_diff"] == 0.0, str(r)
    assert r["nan"] == 0 and r["fwd_max"] < (OUT_FP16_GEMM if dt == "fp16" else OUT16), str(r)
    assert r["sum_rel"] < RED and r["sq_rel"] < RED, str(r)
    assert r["wgrad_nan"] == 0 and r["wgrad_rel"] < 1e-4 and r["wgrad_bitwise"], str(r)


def _check_row(kw, dt):
    """the launch's own variant: 16-bit outputs to OUT16, the BatchNorm backward sums of the stored values to 1e-5 (as
    test_bn_chain's reduce bounds), fp32 pools and SE reductions of 16-bit data to RED, chunked pools bit-reproducible"""
    r = _gc().check_row_kernel(kw["kernel"], kw["N"], kw["HW"], kw["C"], kw["args"], kw["ptrs"], dtype=TDT[dt])
    assert r["nan"] == 0, str(r)
    assert r.get("out_max", 0.0) < OUT16, str(r)
    if dt == "fp16" and "out_max" in r:
        fp16_ulp(r, "out_ulp")
    assert r.get("s1_rel", 0.0) < 1e-5 and r.get("s2_rel", 0.0) < 1e-5, str(r)
    assert r.get("pool_rel", 0.0) < RED and r.get("repro", True) and r.get("draw_rel", 0.0) < RED, str(r)
    assert {"out_max", "s1_rel", "pool_rel", "draw_rel"} & set(r), str(r)


def _check_relu_bn_bwd_reduce(kw, dt):
    r = _gc().check_relu_bn_bwd_reduce(kw["N"], kw["HW"], kw["C"], dtype=TDT[dt], two=kw["two"])
    assert r["gm_mismatch"] == 0 and r["s1_rel"] < 1e-6 and r["s2_rel"] < 1e-6 and r["s1_ref"] < 1e-5 and r["s2_ref"] < 1e-5, str(r)


def _check_maxpool(kw, dt):
    r = _gc().check_maxpool_relu_pool(kw["N"], kw["H"], kw["W"], kw["C"], dtype=TDT[dt])
    assert r["fwd_exact"] == 0 and r["bwd_rel"] < 3e-3 and r["relu_mismatch"] == 0 and r["pool_bwd_rel"] < 1e-6, str(r)
    if dt == "fp16":
        fp16_ulp(r, "bwd_ulp")


def _check_head(kw, dt):
    """2-class classifier head at the plan's (N, F), hard labels (test_head_loss's bounds)"""
    r = _gc().check_head(kw["N"], kw["F"])
    assert r["correct_diff"] == 0 and max(v for k, v in r.items() if k != "correct_diff") < F32 * 5, str(r)


def _check_se_fc(kw, dt):
    r = _gc().check_se_fc(kw["N"], kw["C"], kw["Cse"])
    assert max(r.values()) < F32 * 5, str(r)


CHECKERS = {
    "gemm": _check_gemm,
    "wgrad": _check_wgrad,
    "dwconv": _check_dwconv,
    "conv": _check_conv,
    "conv1x1_dgrad_add": _check_conv1x1_dgrad_add,
    "stem_gemm": _check_stem_gemm,
    "row": _check_row,
    "head": _check_head,
    "relu_bn_bwd_reduce": _check_relu_bn_bwd_reduce,
    "maxpool": _check_maxpool,
    "se_fc": _check_se_fc,
}

_CASES = PL.gpu_cases()


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    torch.cuda.empty_cache()        # the GPU is shared: give back what the last (large) case held


@pytest.mark.parametrize("case", _CASES, ids=[c.id for c in _CASES])
def test_plan_launch(case):
    CHECKERS[case.check](case.kw, case.dtype)
