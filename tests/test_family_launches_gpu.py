"""-m gpu: the kernels at the launch shapes of the model families' plans (tests/family_launches.py harvests them on the CPU;
tests/test_family_launches_cpu.py holds the case list to them).

The shipped harnesses' checkers run unchanged (test_plan_variants_gpu.CHECKERS: test_plan_launches_gpu's with its
tolerances, and the eval head and BatchNorm finalisation); the kernels only these
plans launch have their own checkers in tests/family_checks.py and tests/tf_same_checks.py, with the bounds below:
  * OUT16 (2^-7 scaled) for a 16-bit output that one rounding makes: the max-pool tails, the gathered gradients, the average
    pool, col2im;
  * exact: the arg-max bytes (first maximum in row-major window order), the ceil-mode pool's output, im2col (a copy), the
    ReLU masks (taken on the staged 16-bit value), the SE tail's masked gradient, the stats-free / idx-free forms against the
    full ones, and every output of two launches of a fixed-slot or order-deterministic reduction;
  * RED for fp32 reductions of 16-bit data (pools, dL/dgate), 1e-5 for BatchNorm-backward sums of the stored gradient (as
    test_bn_chain), F32 * 5 for the fp32 SE chains and weight gradients, and the depthwise bounds of _check_dwconv.
Every output starts as NaN (an accumulated one from a known base).
"""
import pytest
import torch

import family_launches as FL
import test_plan_launches_gpu as TPL
import test_plan_variants_gpu as TPV

pytestmark = pytest.mark.gpu

OUT16, RED, F32 = TPL.OUT16, TPL.RED, TPL.F32
TDT = TPL.TDT


def _fc():
    import family_checks
    return family_checks


def _check_dwconv_relu(kw, dt):
    r = _fc().check_dwconv_relu(kw["N"], kw["H"], kw["W"], kw["C"], kw["k"], kw["s"], dtype=TDT[dt], bn=kw["bn"], add=kw["add"])
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fwd_ulp"] <= 1.0, str(r)
    assert r["mask_mismatch"] == 0 and r.get("edge_zeros", 1) > 0, str(r)
    if dt == "fp16":      # test_dwconv_fp16's bounds, as _check_dwconv
        assert r["dgrad_rel"] < 4e-3 and r["wgrad_rel"] < RED, str(r)
    else:
        assert r["dgrad_rel"] < 8e-3 and r["wgrad_rel"] < RED, str(r)
    assert r["det_bitwise"] and r["det_vs_atomic"] < 1e-5 and r["det_gx_diff"] == 0.0, str(r)
    if kw["bn"]:
        assert r["s1_rel"] < 1e-5 and r["s2_rel"] < 1e-5, str(r)
    if "ws_bytes" in kw:
        assert r["ws_bytes"] == kw["ws_bytes"], (r["ws_bytes"], kw["ws_bytes"])


def _check_bn_maxpool(kw, dt):
    r = _fc().check_bn_maxpool(kw["N"], kw["H"], kw["W"], kw["C"], dtype=TDT[dt])
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["out_max"] < OUT16 and r["noidx_mismatch"] == 0, str(r)
    assert r["idx_mismatch"] == 0 and r["tied_windows"] > 0, str(r)
    assert r["bwd_max"] < OUT16 and r["s1_rel"] < 1e-5 and r["s2_rel"] < 1e-5, str(r)


def _check_maxpool_ceil(kw, dt):
    r = _fc().check_maxpool_ceil(kw["N"], kw["H"], kw["W"], kw["C"], dtype=TDT[dt])
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fwd_mismatch"] == 0 and r["idx_mismatch"] == 0, str(r)
    assert r["bwd_max"] < OUT16, str(r)


def _check_pool_se_relu(kw, dt):
    r = _fc().check_pool_se_relu(kw["N"], kw["HW"], kw["C"], kw["Cse"], kw["act"], kw["max_chunks"], dtype=TDT[dt])
    assert r["nan"] == 0 and r["pool_rel"] < RED and r["gate_rel"] < F32 * 5 and r["repro"], str(r)


def _check_relu_se_bwd(kw, dt):
    r = _fc().check_relu_se_bwd(kw["N"], kw["HW"], kw["C"], kw["Cse"], kw["act"], kw["two"], dtype=TDT[dt])
    assert r["nan"] == 0 and r["gm_mismatch"] == 0 and r["draw_rel"] < RED and r["repro"], str(r)
    assert max(r[k] for k in ("d_e_rel", "r_rel", "d_rpre_rel", "dpool_rel", "dWr_rel", "dbr_rel", "dWe_rel", "dbe_rel")) < F32 * 5, str(r)


def _check_se_fc_wgrad(kw, dt):
    r = _fc().check_se_fc_wgrad(kw["N"], kw["C"], kw["Cse"])
    assert r["repro"] and max(v for k, v in r.items() if k != "repro") < F32 * 5, str(r)


def _check_avgpool2(kw, dt):
    r = _fc().check_avgpool2(kw["N"], kw["H"], kw["W"], kw["C"], add=kw["add"], dtype=TDT[dt])
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fwd_max"] < OUT16 and r["bwd_max"] < OUT16, str(r)


def _check_im2col(kw, dt):
    r = _fc().check_im2col(kw["N"], kw["H"], kw["W"], kw["C"], kw["k"], kw["s"], kw["pad"], add=kw["add"], dtype=TDT[dt])
    assert r["nan"] == 0 and r["cols_mismatch"] == 0 and r["nan_b"] == 0 and r["col2im_max"] < OUT16, str(r)


def _check_dw_pad(kw, dt):
    """test_tf_efficientnet_gpu's statements for the SAME-padded depthwise pair, at the plan's shape; the eval form bit for bit"""
    import tf_same_checks
    r = tf_same_checks.check_dw_pad(kw["N"], kw["H"], kw["W"], kw["C"], kw["k"], kw["s"], kw["pt"], kw["pl"], dtype=TDT[dt],
                                    stats=kw["stats"])
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fwd_ulp"] <= 1.0 and r.get("nostats_mismatch", 0) == 0, str(r)
    assert r["sum_rel"] < RED and r["sq_rel"] < RED and r["bwd_bitwise"], str(r)
    assert r.get("sym_fwd_mismatch", 0) == 0 and r.get("sym_bwd_mismatch", 0) == 0, str(r)
    assert r["dgrad_rel"] < (4e-3 if dt == "fp16" else 8e-3) and r["wgrad_rel"] < RED, str(r)
    assert r["bs1_rel"] < RED and r["bs2_rel"] < RED, str(r)
    if "ws_bytes" in kw:
        assert r["ws_bytes"] == kw["ws_bytes"], (r["ws_bytes"], kw["ws_bytes"])


def _check_stem_pad(kw, dt):
    import tf_same_checks
    r = tf_same_checks.check_stem_im2col_pad(kw["N"], kw["Cin"], kw["H"], kw["W"], kw["k"], kw["s"], kw["pt"], kw["pl"], dtype=TDT[dt])
    assert r["diff"] == 0.0 and r["nan"] == 0 and r["pad_max"] == 0.0 and r.get("sym_mismatch", 0) == 0, str(r)


CHECKERS = dict(TPV.CHECKERS, dwconv_relu=_check_dwconv_relu, bn_maxpool=_check_bn_maxpool, maxpool_ceil=_check_maxpool_ceil,
                pool_se_relu=_check_pool_se_relu, relu_se_bwd=_check_relu_se_bwd, se_fc_wgrad=_check_se_fc_wgrad,
                avgpool2=_check_avgpool2, im2col=_check_im2col, dw_pad=_check_dw_pad, stem_pad=_check_stem_pad)

_CASES = FL.gpu_cases()


@pytest.fixture(autouse=True)
def _free_between_cases():
    yield
    torch.cuda.empty_cache()        # the GPU is shared: give back what the last (large) case held


@pytest.mark.parametrize("case", _CASES, ids=[c.id for c in _CASES])
def test_family_launch(case):
    CHECKERS[case.check](case.kw, case.dtype)
