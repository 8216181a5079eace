"""-m gpu: fp16 overflow and subnormal stores of the kernels whose fp16 outputs carry loss-scaled gradients.

Dynamic loss scaling relies on a 16-bit gradient store that overflows producing +-inf (dfd_check_finite then skips the step),
and on a small gradient being stored as an fp16 subnormal rather than flushed. Each kernel runs once per mode at a small
plan-like shape on operands scaled so that:
  * overflow: a known fraction of the fp64 reference lies beyond the fp16 range. Every element whose reference rounds to
    +-inf (|ref| >= 65520 by more than its element-wise bound) is +-inf with the reference's sign, never a saturated +-65504;
  * underflow: a known fraction of the fp64 reference lies in [2^-24, 2^-14). Those elements meet the element-wise bound of
    tests/gpu_checks.py including TINY16 / 2; a flush to zero is off by up to 2^-14.
The fp32 reductions of an overflowed launch (BatchNorm-backward sums) are not asserted.
"""
import struct

import pytest
import torch
import torch.nn.functional as F

import gpu_checks as GC
from deepfake_detection_b200 import _lib

pytestmark = pytest.mark.gpu

F16 = torch.float16
D = GC.DT[F16]
P, st, nchw, nhwc = GC.P, GC.st, GC.nchw, GC.nhwc
HALF_MAX_RND = 65520.0          # the smallest magnitude that rounds to inf in fp16
MODES = ("overflow", "underflow")


def _f16(x):
    """x as fp16 operands, kept finite (a scaled sample beyond the fp16 range would make the reference itself inf)"""
    return x.clamp(-60000, 60000).to(F16)


def _nan(*shape, dtype=F16):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def _range(out, ref, bound, mode, min_frac=0.01, inner=None):
    """inner: (value, bound) of an intermediate 16-bit store that the output is the sum of (dfd_conv1x1_dgrad_add stores the
    input gradient, then adds it to the main path): where that store overflows, the sum is inf with its sign"""
    out, ref, bound = out.double(), ref.double(), bound.double()
    assert bool(torch.isfinite(ref).all())          # finite operands: every inf in the output is the kernel's own store
    if mode == "overflow":
        sel = ref.abs() >= HALF_MAX_RND + bound
        sign = torch.sign(ref)
        band = (ref.abs() - HALF_MAX_RND).abs() < bound
        if inner is not None:
            v, vb = inner
            isel = v.abs() >= HALF_MAX_RND + vb
            band = (band | ((v.abs() - HALF_MAX_RND).abs() < vb)) & ~isel
            sel = (sel | isel) & ~band
            sign = torch.where(isel, torch.sign(v), sign)
        frac = float(sel.double().mean())
        wrong = sel & ~(torch.isinf(out) & (torch.sign(out) == sign))
        sat = sel & (out.abs() == 65504.0)
        assert frac >= min_frac and int(wrong.sum()) == 0 and int(sat.sum()) == 0, \
            dict(frac=frac, wrong=int(wrong.sum()), saturated=int(sat.sum()))
        # below the threshold (by more than the bound) the store is finite and within the bound
        fin = ~sel & ~band
        assert bool(torch.isfinite(out[fin]).all())
        assert GC.ulp_ratio(out[fin], ref[fin], bound[fin]) <= 1.0
    else:
        sel = (ref.abs() >= 2.0 ** -24) & (ref.abs() < 2.0 ** -14)
        frac = float(sel.double().mean())
        ratio = GC.ulp_ratio(out[sel], ref[sel], bound[sel])
        assert frac >= min_frac and ratio <= 1.0, dict(frac=frac, ratio=ratio, zeros=int((out[sel] == 0).sum()))


def _gen(seed=0):
    return torch.Generator(device="cuda").manual_seed(seed)


def _scales(mode, big, small):
    return big if mode == "overflow" else small


# ---- tensor-core input gradients -----------------------------------------------------------------------------------------
def _packed(w):
    Cout, Cin, k, _ = w.shape
    wp = torch.zeros(Cout * k * k * Cin, device="cuda", dtype=F16)
    wpT, wpD = torch.zeros_like(wp), torch.zeros_like(wp)
    table = torch.frombuffer(bytearray(struct.pack("<QQQQiiii", P(w), P(wp), P(wpT), P(wpD), Cout, Cin, k, 0)),
                             dtype=torch.uint8).cuda()
    _lib.call("dfd_repack_weights", P(table), 1, D, st())
    return wp, wpT, wpD


def _conv_dgrad_ref(dy, w, H, W, stride):
    """fp64 input gradient of the padded k x k convolution and the same sum over |w| |dy| (NHWC)"""
    N, Cin, k = dy.shape[0], w.shape[1], w.shape[2]
    shape, pad = (N, Cin, H, W), (k - 1) // 2
    ref = torch.nn.grad.conv2d_input(shape, w.double(), nchw(dy.double()), stride=stride, padding=pad)
    mag = torch.nn.grad.conv2d_input(shape, w.double().abs(), nchw(dy.double()).abs(), stride=stride, padding=pad)
    return nhwc(ref), nhwc(mag)


def _tc_bound(ref, mag, K):
    return GC.elem_bound(ref, F16, GC.acc_term(mag, K))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stride", [1, 2])
def test_conv_dgrad_range(mode, stride):
    """dfd_conv_tc as the stride-1 input gradient (tap-flipped weights), dfd_conv_dgrad_s2_tc for stride 2"""
    g = _gen(1)
    N, H, W, Cin, Cout, k = 2, 14, 14, 64, 64, 3
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    a, b = _scales(mode, (600.0, 4.0), (2.0 ** -10, 2.0 ** -10))
    dy = _f16((torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g) * a))
    w = _f16((torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * b))
    _, _, wpD = _packed(w)
    dx = _nan(N, H, W, Cin)
    if stride == 1:
        _lib.call("dfd_conv_tc", P(dy), P(wpD), P(dx), N, H, W, Cout, Cin, k, 1, D, None, None, None, st())
    else:
        _lib.call("dfd_conv_dgrad_s2_tc", P(dy), P(wpD), P(dx), N, H, W, Cin, Cout, D, st())
    torch.cuda.synchronize()
    ref, mag = _conv_dgrad_ref(dy, w, H, W, stride)
    _range(dx, ref, _tc_bound(ref, mag, k * k * Cout), mode)


@pytest.mark.parametrize("mode", MODES)
def test_conv1x1_dgrad_add_range(mode):
    """dfd_conv1x1_dgrad_add: the input gradient stored to 16 bits, then added to the main-path gradient by the TMA reduction
    store in fp16 (two roundings: out_term of the gradient besides that of the sum)"""
    g = _gen(2)
    N, H, W, Cin, Cout, stride = 2, 14, 14, 64, 128, 2
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    a, b, m = _scales(mode, (500.0, 8.0, 1000.0), (2.0 ** -10, 2.0 ** -10, 2.0 ** -17))
    dy = _f16((torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g) * a))
    w = _f16((torch.randn(Cout, Cin, device="cuda", generator=g) * b))
    wT = w.t().contiguous()
    main = _f16((torch.randn(N, H, W, Cin, device="cuda", generator=g) * m))
    got = main.clone()
    _lib.call("dfd_conv1x1_dgrad_add", P(dy), P(wT), P(got), N, H, W, Cin, Cout, stride, D, st())
    torch.cuda.synchronize()
    dg = (dy.double().reshape(-1, Cout) @ w.double()).reshape(N, Ho, Wo, Cin)
    dmag = (dy.double().abs().reshape(-1, Cout) @ w.double().abs()).reshape(N, Ho, Wo, Cin)
    ref, mag, inner = main.double(), main.double().abs(), torch.zeros_like(main, dtype=torch.float64)
    ref[:, ::stride, ::stride] += dg
    mag[:, ::stride, ::stride] += dmag
    inner[:, ::stride, ::stride] = GC.out_term(dg, F16) + GC.acc_term(dmag, Cout)
    dg_full, dgb_full = torch.zeros_like(ref), torch.zeros_like(ref)
    dg_full[:, ::stride, ::stride], dgb_full[:, ::stride, ::stride] = dg, GC.acc_term(dmag, Cout) + GC.U_OUT[F16] * dg.abs()
    _range(got, ref, GC.elem_bound(ref, F16, inner) + GC.acc_term(mag, Cout), mode, inner=(dg_full, dgb_full))


@pytest.mark.parametrize("mode", MODES)
def test_gemm_col2im_range(mode):
    """dfd_gemm_tn (the column gradient dy W^T) and dfd_col2im (the overlapping column terms summed), each store on its own"""
    g = _gen(3)
    N, H, W, C, Cout, k, s, pad = 2, 14, 14, 64, 64, 3, 2, 1
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    M = N * Ho * Wo
    a, b = _scales(mode, (2000.0, 8.0), (2.0 ** -10, 2.0 ** -10))
    dy = _f16((torch.randn(M, Cout, device="cuda", generator=g) * a))
    wT = _f16((torch.randn(k * k * C, Cout, device="cuda", generator=g) * b))
    dcols = _nan(M, k * k * C)
    _lib.call("dfd_gemm_tn", P(dy), P(wT), P(dcols), M, k * k * C, Cout, D, None, None, None, st())
    torch.cuda.synchronize()
    ref = dy.double() @ wT.double().t()
    _range(dcols, ref, _tc_bound(ref, dy.double().abs() @ wT.double().abs().t(), Cout), mode)
    # col2im on finite column terms scaled to the range edge
    c = _scales(mode, 30000.0, 2.0 ** -17)
    cols = _f16((torch.randn(M, k * k * C, device="cuda", generator=g) * c))
    add = _f16((torch.randn(N, H, W, C, device="cuda", generator=g) * c))
    dx = _nan(N, H, W, C)
    _lib.call("dfd_col2im", P(cols), P(add), P(dx), N, H, W, C, k, s, pad, D, st())
    torch.cuda.synchronize()
    dc = cols.double().view(N, Ho * Wo, k * k, C).permute(0, 3, 2, 1).reshape(N, C * k * k, Ho * Wo)
    ref = nhwc(F.fold(dc, (H, W), k, padding=pad, stride=s)) + add.double()
    mag = nhwc(F.fold(dc.abs(), (H, W), k, padding=pad, stride=s)) + add.double().abs()
    _range(dx, ref, GC.sum_bound(ref, mag, -(-k // s) ** 2 + 1, F16), mode)


# ---- bandwidth kernels ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("act", [1, 2])
def test_act_bwd_range(mode, act):
    """dfd_act_bwd (Swish, ReLU) with the gate and the pooled gradient: gu = (da * gate + dpool / hw) * act'(u)"""
    g = _gen(4)
    N, HW, C = 4, 196, 64
    y = _f16((torch.randn(N, HW, C, device="cuda", generator=g) * 1.5 + 0.3))
    scale, shift = GC._bn_params(C, g)
    mean = 0.1 * torch.randn(C, device="cuda", generator=g)
    rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
    gate = torch.sigmoid(torch.randn(N, C, device="cuda", generator=g))
    a, p = _scales(mode, (40000.0, 60000.0 * HW), (2.0 ** -16, 2.0 ** -16 * HW))
    da = _f16((torch.randn(N, HW, C, device="cuda", generator=g) * a))
    dpool = torch.randn(N, C, device="cuda", generator=g) * p
    gu = _nan(N, HW, C)
    s1, s2 = GC.stat_buf(C), GC.stat_buf(C)
    _lib.call("dfd_act_bwd", P(da), P(y), P(scale), P(shift), P(mean), P(rstd), P(gate), P(dpool), P(gu), N, HW, C, act, D,
              P(s1), P(s2), None, st())
    torch.cuda.synchronize()
    gin = da.double() * gate.double().unsqueeze(1) + dpool.double().unsqueeze(1) / HW
    gmag = (da.double() * gate.double().unsqueeze(1)).abs() + dpool.double().abs().unsqueeze(1) / HW
    ref, bound = GC.act_bwd_bound(GC._u32(y, scale, shift).double(), act, gin, gmag, F16)
    _range(gu, ref, bound, mode)


@pytest.mark.parametrize("mode", MODES)
def test_bn_bwd_apply_range(mode):
    """dfd_bn_bwd_apply: dy = fmaf(cA, g, fmaf(cB, y, cC))"""
    g = _gen(5)
    N, HW, C = 4, 196, 64
    gr = _f16(torch.randn(N, HW, C, device="cuda", generator=g))
    y = _f16(torch.randn(N, HW, C, device="cuda", generator=g))
    f = _scales(mode, 40000.0, 2.0 ** -16)
    cA = (1.0 + 0.1 * torch.randn(C, device="cuda", generator=g)) * f
    cB = 0.5 * torch.randn(C, device="cuda", generator=g) * f
    cC = 0.1 * torch.randn(C, device="cuda", generator=g) * f
    dy = _nan(N, HW, C)
    _lib.call("dfd_bn_bwd_apply", P(gr), P(y), None, P(cA), P(cB), P(cC), P(dy), N, HW, C, D, st())
    torch.cuda.synchronize()
    ref = cA.double() * gr.double() + cB.double() * y.double() + cC.double()
    mag = (cA.double() * gr.double()).abs() + (cB.double() * y.double()).abs() + cC.double().abs()
    _range(dy, ref, GC.sum_bound(ref, mag, 2, F16), mode)


@pytest.mark.parametrize("mode", MODES)
def test_dwconv_bwd_range(mode):
    """dfd_dwconv_bwd (MODE 1: gu = dgrad * swish'(u)) on a dy tile staged from a scaled gradient (cB = cC = 0)"""
    g = _gen(6)
    N, H, W, C, k, s = 2, 14, 14, 64, 5, 1
    pad = (k - 1) // 2
    x = _f16(torch.randn(N, H, W, C, device="cuda", generator=g))
    w = (torch.randn(C, 1, k, k, device="cuda", generator=g) * _scales(mode, 2.0, 2.0 ** -8)).contiguous()
    scale, shift = GC._bn_params(C, g)
    gy = _f16((torch.randn(N, H, W, C, device="cuda", generator=g) * _scales(mode, 15000.0, 2.0 ** -12)))
    yout = _f16(torch.randn(N, H, W, C, device="cuda", generator=g))
    cA, cB, cC = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    mean = 0.1 * torch.randn(C, device="cuda", generator=g)
    rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
    gx, dW = _nan(N, H, W, C), torch.zeros_like(w)
    b1, b2 = GC.stat_buf(C), GC.stat_buf(C)
    _lib.call("dfd_dwconv_bwd", P(gy), P(yout), P(cA), P(cB), P(cC), P(w), P(x), P(scale), P(shift), P(mean), P(rstd), None,
              P(gx), P(dW), N, H, W, C, k, s, D, P(b1), P(b2), None, 0, None, st())
    torch.cuda.synchronize()
    ga, mag = GC.dw_input_grad64(GC.staged_dy(gy, yout, cA, cB, cC, F16), w, H, W, k, s, (pad,) * 4)
    u = GC._u32(x, scale, shift).double()
    d, err = GC.swish_grad64(u), GC.swish_grad_err(u)
    ref = ga * d
    acc = GC.acc_term(mag, k * k + 1)
    _range(gx, ref, GC.elem_bound(ref, F16, acc * (d.abs() + err), GC.swish_bwd_term(u, ga.abs() + acc)), mode)


@pytest.mark.parametrize("mode", MODES)
def test_maxpool_bwd_range(mode):
    """dfd_maxpool_bwd: the gradients of the (at most 2 x 2) windows whose arg-max a pixel is, summed; small-integer inputs
    so that pixels win several windows"""
    g = _gen(7)
    N, H, W, C = 4, 28, 28, 64
    x = _f16(torch.randint(0, 3, (N, H, W, C), device="cuda", generator=g))
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = _nan(N, Ho, Wo, C)
    idx = torch.zeros(N * Ho * Wo * C, dtype=torch.uint8, device="cuda")
    _lib.call("dfd_maxpool_fwd", P(x), P(out), P(idx), N, H, W, C, D, st())
    mag_g = _scales(mode, 50000.0, 2.0 ** -17)
    sign = torch.randint(0, 2, (N, Ho, Wo, C), device="cuda", generator=g).float() * 2 - 1
    gy = _f16(((0.6 + 0.4 * torch.rand(N, Ho, Wo, C, device="cuda", generator=g)) * mag_g * sign))
    gx = _nan(N, H, W, C)
    _lib.call("dfd_maxpool_bwd", P(gy), P(idx), P(gx), N, H, W, C, D, st())
    torch.cuda.synchronize()
    xr = nchw(x.double()).requires_grad_(True)
    y = F.max_pool2d(xr, 3, 2, 1)
    ref, = torch.autograd.grad(y, xr, nchw(gy.double()), retain_graph=True)
    mag, = torch.autograd.grad(y, xr, nchw(gy.double()).abs())
    ref, mag = nhwc(ref), nhwc(mag)
    _range(gx, ref, GC.sum_bound(ref, mag, 4, F16), mode, min_frac=0.005)


@pytest.mark.parametrize("mode", MODES)
def test_avgpool2_bwd_add_range(mode):
    """dfd_avgpool2_bwd_add: dx = fmaf(dy, 1 / count, add)"""
    g = _gen(8)
    N, H, W, C = 4, 15, 17, 64
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    f = _scales(mode, 40000.0, 2.0 ** -16)
    dy = _f16((torch.randn(N, Ho, Wo, C, device="cuda", generator=g) * f))
    add = _f16((torch.randn(N, H, W, C, device="cuda", generator=g) * f))
    dx = _nan(N, H, W, C)
    _lib.call("dfd_avgpool2_bwd_add", P(dy), P(add), P(dx), N, H, W, C, D, st())
    torch.cuda.synchronize()
    xr = torch.zeros(N, C, H, W, device="cuda", dtype=torch.float64, requires_grad=True)
    yp = F.avg_pool2d(xr, 2, 2, ceil_mode=True, count_include_pad=False)
    gd, = torch.autograd.grad(yp, xr, nchw(dy.double()))
    ref = nhwc(gd) + add.double()
    mag = nhwc(gd).abs() + add.double().abs()
    _range(dx, ref, GC.sum_bound(ref, mag, 1, F16), mode)
