"""-m gpu: every C-ABI kernel against plain PyTorch fp32 on the same rounded inputs (see tests/gpu_checks.py for
the tolerance rationale: OUT16 = 2^-7 scaled max error for 16-bit outputs, RED = 2e-3 rel-L2 for fp32 reductions)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

OUT16 = 2.0 ** -7
RED = 2e-3
F32 = 2e-5


def _gc():
    import gpu_checks
    return gpu_checks


GEMM_SHAPES = [(1000, 16, 96), (4096 + 37, 24, 144), (777, 1152, 320), (5000, 320, 1280), (130, 40, 24), (50176, 80, 480),
               (300, 64, 64), (128, 64, 16), (256 * 49, 672, 192)]


@pytest.mark.parametrize("M,K,N", GEMM_SHAPES)
def test_gemm_tcgen05(M, K, N):
    r = _gc().check_gemm("tc", M, K, N)
    assert r["nan"] == 0 and r["out_max"] < OUT16 and r["sum_rel"] < RED and r["sq_rel"] < RED, r


@pytest.mark.parametrize("M,K,N,pack", [(1000, 16, 96, 4), (4096 + 38, 24, 144, 2), (50176, 32, 32, 2), (3 * 1001, 16, 32, 3),
                                        (25088 * 4, 16, 96, 4), (8, 32, 16, 2)])
def test_gemm_tcgen05_rowpack(M, K, N, pack):
    """small-K pointwise conv: packed rows against the block-diagonal weight == the plain product, statistics folded"""
    r = _gc().check_gemm("rowpack%d" % pack, M, K, N)
    assert r["nan"] == 0 and r["out_max"] < OUT16 and r["sum_rel"] < RED and r["sq_rel"] < RED, r


def test_gemm_tcgen05_fp16():
    r = _gc().check_gemm("tc", 3000, 144, 40, dtype=torch.float16)
    assert r["nan"] == 0 and r["out_max"] < 2.0 ** -9 and r["sum_rel"] < RED, r


@pytest.mark.parametrize("M,K,N", GEMM_SHAPES[:5])
def test_gemm_mma(M, K, N):
    r = _gc().check_gemm("mma", M, K, N, with_add=(N == 24))
    assert r["nan"] == 0 and r["out_max"] < OUT16 and r["sum_rel"] < RED and r["sq_rel"] < RED, r


@pytest.mark.parametrize("M,Nw,Kw", [(5000, 96, 16), (12345, 144, 24), (3000, 1152, 192), (777, 320, 1280), (64, 24, 144)])
def test_wgrad(M, Nw, Kw):
    assert _gc().check_wgrad(M, Nw, Kw)["rel"] < 1e-4


@pytest.mark.parametrize("M,Nw,Kw", [(5000, 96, 16), (12345, 144, 24), (3000, 1152, 192), (777, 320, 1280), (64, 24, 144),
                                     (50176, 672, 112), (130, 40, 240), (4096, 128, 128), (70, 8, 8)])
def test_wgrad_tcgen05(M, Nw, Kw):
    """MN-major wgmma weight gradient (operands straight from NHWC rows) against fp64"""
    assert _gc().check_wgrad(M, Nw, Kw, impl="dfd_gemm_wgrad")["rel"] < 1e-4


@pytest.mark.parametrize("M,Nw,Kw", [(50176, 672, 112), (12544, 1280, 320), (3211264 // 8, 96, 16), (130, 40, 240), (70, 8, 8),
                                     (12544, 512, 4608)])
def test_wgrad_tcgen05_deterministic(M, Nw, Kw):
    """order-deterministic mode (split partials in fixed workspace slots + dfd_ordered_reduce in split order): two runs agree
    bit for bit, the result matches fp64 and the atomic flush"""
    r = _gc().check_wgrad(M, Nw, Kw, impl="dfd_gemm_wgrad", det=True)
    assert r["bitwise"] and r["rel"] < 1e-4 and r["vs_atomic"] < 1e-5, r


def test_wgrad_tcgen05_fp16():
    assert _gc().check_wgrad(3000, 144, 40, dtype=torch.float16, impl="dfd_gemm_wgrad")["rel"] < 1e-4


@pytest.mark.parametrize("N,H,W,C,k,s,aff", [(2, 16, 16, 32, 3, 1, True), (2, 17, 19, 96, 3, 2, True), (2, 14, 14, 144, 5, 1, True),
                                              (2, 15, 15, 240, 5, 2, True), (3, 7, 7, 1152, 5, 1, True), (2, 40, 40, 32, 3, 1, False),
                                              (1, 33, 33, 24, 3, 1, False), (2, 56, 56, 144, 5, 2, True)])
def test_dwconv(N, H, W, C, k, s, aff):
    r = _gc().check_dwconv(N, H, W, C, k, s, affine=aff)
    assert r["nan"] == 0 and r["nan_b"] == 0, r
    assert r["fwd_max"] < OUT16 and r["sum_rel"] < RED and r["sq_rel"] < RED, r
    assert r["dgrad_rel"] < 8e-3 and r["wgrad_rel"] < RED, r      # tanh.approx sigmoid: 2^-11 relative
    # fused dgrad + wgrad pass: the same input gradient bit for bit, the same reductions
    assert r["fused_nan"] == 0 and r["fused_gx_diff"] == 0.0 and r["fused_wgrad_rel"] < RED, r
    if aff:
        assert r["bs1_rel"] < RED and r["bs2_rel"] < RED, r
        assert r["fused_bs1_rel"] < RED and r["fused_bs2_rel"] < RED, r


def test_dwconv_fp16():
    """also the fp16 element-wise bounds, each violated by the same output rounded through bf16 (test_plan_launches_gpu)"""
    import test_plan_launches_gpu as TPL
    r = _gc().check_dwconv(2, 14, 14, 80, 3, 1, dtype=torch.float16)
    assert r["fwd_rel"] < 2e-3 and r["dgrad_rel"] < 4e-3 and r["wgrad_rel"] < RED, r
    assert r["fwd_ulp"] <= 1.0, r
    TPL.fp16_ulp(r, "dgrad_ulp")


@pytest.mark.parametrize("N,Cin,H,W,k,s,pad", [(2, 3, 32, 32, 3, 2, 1), (3, 3, 37, 45, 3, 2, 1), (2, 3, 64, 64, 7, 2, 3), (1, 4, 19, 23, 3, 1, 1)])
def test_stem_im2col(N, Cin, H, W, k, s, pad):
    r = _gc().check_stem_im2col(N, Cin, H, W, k, s, pad)
    assert r["nan"] == 0 and r["diff"] == 0.0 and r["pad_max"] == 0.0, r


@pytest.mark.parametrize("N,HW,C", [(3, 64, 32), (2, 49, 1152), (4, 200, 144), (2, 1000, 16)])
def test_bn_chain(N, HW, C):
    r = _gc().check_bn_chain(N, HW, C)
    assert r["nan"] == 0 and r["nbt"] == 1, r
    assert r["rm_rel"] < 1e-5 and r["rv_rel"] < 1e-5, r
    assert r["gate_max"] < OUT16 and r["res_max"] < OUT16 and r["pool_rel"] < RED, r
    assert r["pool_chunk_rel"] < RED and r["pool_chunk_repro"] == 0.0, r       # several CTAs per image, still reproducible
    assert r["dy_rel"] < 1e-2 and r["dgamma_rel"] < 5e-3 and r["dbeta_rel"] < 5e-3, r
    assert r["reduce1_rel"] < 1e-5 and r["reduce2_rel"] < 1e-5 and r["draw_rel"] < RED, r


@pytest.mark.parametrize("kind", ["gemm", "gemm_rowpack", "dwconv_fwd", "act_bwd", "bn_bwd_reduce", "dwconv_bwd"])
def test_fused_bn_finalize(kind):
    """the last CTA of the statistics-producing kernel finalises the BatchNorm: same vectors as the standalone finalise launch
    (the fp64 slot sums may differ in their last bit with the order of the atomics: 1e-6 relative covers it)"""
    r = _gc().check_fused_finalize(kind)
    assert r["max_diff"] < 1e-6 and r["ticket_at_rest"] and r.get("nbt", 2) == 2, r


@pytest.mark.parametrize("N,C,Cse", [(5, 144, 6), (3, 1152, 48)])
def test_se_fc(N, C, Cse):
    r = _gc().check_se_fc(N, C, Cse)
    assert max(r.values()) < F32 * 5, r


@pytest.mark.parametrize("N,HW,C,Cse,dtype", [(5, 196, 144, 6, torch.bfloat16), (3, 49, 1152, 48, torch.bfloat16),
                                               (300, 64, 32, 8, torch.float16), (2, 3136, 96, 4, torch.bfloat16),
                                               (3, 361, 3840, 160, torch.float16)])
def test_se_fused_launches(N, HW, C, Cse, dtype):
    """dfd_pool_se / dfd_se_bwd_chain (the CTA that completes an image's reduction runs its FC chain) == the separate kernels"""
    r = _gc().check_se_fused(N, HW, C, Cse, dtype)
    assert r["pool_equal"] and r["gate_equal"] and r["draw_equal"] and r["pool_rel"] < RED and r["bwd_rel"] < 1e-5, r


@pytest.mark.parametrize("kw", [dict(), dict(smoothing=0.1), dict(soft=True)])
def test_head_loss(kw):
    r = _gc().check_head(16, 1280, **kw)
    assert r["correct_diff"] == 0 and max(v for k, v in r.items() if k != "correct_diff") < F32 * 5, r


@pytest.mark.parametrize("kind", ["sgd", "adam", "adamw", "rmsproptf"])
def test_optimizer(kind):
    r = _gc().check_optimizer(kind)
    assert r["rel"] < F32 and r["p16_rel"] == 0.0, r


def test_transpose():
    assert _gc().check_transpose()["mismatch"] == 0


@pytest.mark.parametrize("N,H,W,Cin,Cout,k,s", [(2, 14, 14, 64, 64, 3, 1), (2, 15, 17, 64, 128, 3, 2), (1, 9, 9, 128, 40, 3, 1),
                                                   (2, 12, 12, 64, 256, 1, 2)])
def test_conv_dense(N, H, W, Cin, Cout, k, s):
    r = _gc().check_conv_dense(N, H, W, Cin, Cout, k, s)
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fwd_max"] < OUT16 and r["dgrad_rel"] < 6e-3 and r["wgrad_rel"] < 1e-4, r


# the resnet50 / resnet18 stride-1 3x3 shapes (56 / 28 / 14 / 7: patch = 2 / 4 / 7 rows of an image, two stacked 7x7 images with
# an odd batch), ragged extents that do not divide into patches, a second N tile (Cout 512 > 256), 5x5
@pytest.mark.parametrize("N,H,W,Cin,Cout,k", [(2, 56, 56, 64, 64, 3), (3, 28, 28, 128, 128, 3), (3, 14, 14, 256, 256, 3),
                                                 (5, 7, 7, 512, 512, 3), (2, 13, 20, 64, 128, 3), (1, 9, 130, 64, 64, 3),
                                                 (2, 11, 11, 128, 64, 5)])
def test_conv_implicit(N, H, W, Cin, Cout, k):
    r = _gc().check_conv_implicit(N, H, W, Cin, Cout, k)
    assert r["nan"] == 0 and r["nan_b"] == 0 and r["fwd_max"] < OUT16 and r["dgrad_rel"] < 6e-3, r
    assert r["sum_rel"] < 1e-6 and r["sq_rel"] < 1e-6 and r["vs_im2col_mismatch"] == 0, r
    assert r["wgrad_rel"] < 1e-4 and r["wgrad_det_bitwise"] and r["wgrad_det_vs_atomic"] < 1e-5, r


# stride 2 (TMA element strides): the three strided 3x3 convolutions of resnet50 / resnet18 (56 -> 28, 28 -> 14, 14 -> 7), odd
# extents, and k = 1 stride 2 = the strided downsample convolution without its gather
@pytest.mark.parametrize("N,H,W,Cin,Cout,k", [(2, 56, 56, 128, 128, 3), (3, 28, 28, 256, 256, 3), (5, 14, 14, 512, 512, 3),
                                                 (2, 15, 21, 64, 128, 3), (3, 56, 56, 256, 512, 1), (2, 13, 9, 64, 64, 1)])
def test_conv_implicit_stride2(N, H, W, Cin, Cout, k):
    r = _gc().check_conv_implicit(N, H, W, Cin, Cout, k, stride=2)
    assert r["nan"] == 0 and r["fwd_max"] < OUT16 and r["sum_rel"] < 1e-6 and r["sq_rel"] < 1e-6 and r["vs_im2col_mismatch"] == 0, r
    if k == 3:      # the strided input gradient: four parity-class implicit GEMMs; every dx element written (no NaN left), fp64 autograd
        assert r["nan_b"] == 0 and r["dgrad_rel"] < 6e-3 and r["dgrad_vs_col2im"] < 8e-3, r
    assert r["wgrad_rel"] < 1e-4 and r["wgrad_det_bitwise"] and r["wgrad_det_vs_atomic"] < 1e-5, r


@pytest.mark.parametrize("N,H,W,Cin,Cout,stride", [(3, 56, 56, 64, 256, 1), (2, 56, 56, 256, 512, 2), (5, 14, 14, 1024, 2048, 2),
                                                      (2, 13, 9, 64, 128, 2)])
def test_conv1x1_dgrad_add(N, H, W, Cin, Cout, stride):
    r = _gc().check_conv1x1_dgrad_add(N, H, W, Cin, Cout, stride)
    assert r["nan"] == 0 and r["mismatch"] == 0 and r["rel"] < 6e-3, r


def test_conv_implicit_fp16():
    import test_plan_launches_gpu as TPL
    r = _gc().check_conv_implicit(2, 14, 14, 64, 128, 3, dtype=torch.float16)
    assert r["nan"] == 0 and r["fwd_max"] < OUT16 and r["dgrad_rel"] < 6e-3 and r["vs_im2col_mismatch"] == 0, r
    TPL.fp16_scaled(r, "fwd_max")        # fp16 precision (the fp16 GEMM's bound), violated by the output rounded through bf16
    TPL.fp16_scaled(r, "dgrad_max")
    assert r["wgrad_rel"] < 1e-4 and r["wgrad_det_bitwise"], r


@pytest.mark.parametrize("N,HW,C,two", [(3, 49, 2048, False), (2, 3136, 256, True), (5, 196, 64, True), (2, 784, 512, False)])
def test_relu_bn_bwd_reduce(N, HW, C, two):
    r = _gc().check_relu_bn_bwd_reduce(N, HW, C, two=two)
    assert r["gm_mismatch"] == 0 and r["s1_rel"] < 1e-6 and r["s2_rel"] < 1e-6 and r["s1_ref"] < 1e-5 and r["s2_ref"] < 1e-5, r


@pytest.mark.parametrize("N,H,W,C", [(2, 16, 16, 64), (3, 15, 13, 64)])
def test_maxpool_relu_pool(N, H, W, C):
    r = _gc().check_maxpool_relu_pool(N, H, W, C)
    # bwd: an input that is the arg-max of several windows receives a SUM of gradients, rounded once to 16 bit
    assert r["fwd_exact"] == 0 and r["bwd_rel"] < 3e-3 and r["relu_mismatch"] == 0 and r["pool_bwd_rel"] < 1e-6, r
