"""The element-wise 16-bit error bounds of tests/gpu_checks.py, rehearsed on the CPU: at a few representative shapes an fp64
reference rounded once to fp16 meets each bound (ratio <= 1), the same reference rounded through bf16 violates it, the Swish
bounds hold for a sigmoid off by the documented worst-case tanh.approx error, and a planted kernel-style bug (a dropped tap,
one channel's scale applied twice, an extra 16-bit rounding, a gather that keeps one window) violates it. So each bound
resolves fp16 precision and admits the kernel's own arithmetic before any GPU case relies on it."""
import torch
import torch.nn.functional as F

import gpu_checks as GC

F16, BF16 = torch.float16, torch.bfloat16


def _gen(seed=0):
    return torch.Generator().manual_seed(seed)


def _r16(x):
    return x.to(F16)


def _trip(x):
    return x.to(BF16).to(F16)


def _sig_perturbed(u, sign):
    """sigmoid_fast with tanh.approx off by its documented worst case (2^-10.987 relative), in the direction `sign`"""
    t = torch.tanh(u / 2)
    return 0.5 * t * (1 + sign * GC.E_TANH) + 0.5


def _swish_grad_from(s, u):
    return s + u * s - u * s * s


# ---- depthwise 5x5 stride 2 input gradient, Swish input (MODE 1) --------------------------------------------------------
def _dw_case():
    g = _gen(1)
    N, H, W, C, k, s, pad = 2, 15, 13, 16, 5, 2, 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    x = torch.randn(N, H, W, C, generator=g).to(F16)
    w = torch.randn(C, 1, k, k, generator=g) / k
    scale = 1.0 + 0.2 * torch.randn(C, generator=g)
    shift = 0.3 * torch.randn(C, generator=g)
    gy = (0.1 * torch.randn(N, Ho, Wo, C, generator=g)).to(F16)
    yout = torch.randn(N, Ho, Wo, C, generator=g).to(F16)
    cA = 1.0 + 0.1 * torch.randn(C, generator=g)
    cB = 0.05 * torch.randn(C, generator=g)
    cC = 0.01 * torch.randn(C, generator=g)
    dy = GC.staged_dy(gy, yout, cA, cB, cC, F16)
    ga, mag = GC.dw_input_grad64(dy, w, H, W, k, s, (pad,) * 4)
    u = GC._u32(x, scale, shift).double()
    return dict(dy=dy, w=w, H=H, W=W, k=k, s=s, pad=pad, ga=ga, mag=mag, u=u, x=x, scale=scale, shift=shift)


def test_dw_dgrad_swish_bound():
    c = _dw_case()
    ga, mag, u, k = c["ga"], c["mag"], c["u"], c["k"]
    ref = ga * GC.swish_grad64(u)
    once, trip = GC.dw_dgrad_bound(_r16(ref), ga, mag, k, F16, u=u)
    assert once <= 1.0 and trip > 1.0, (once, trip)
    _, trip_bf = GC.dw_dgrad_bound(_trip(ref), ga, mag, k, F16, u=u)
    assert trip_bf > 1.0
    # the kernel's sigmoid off by the worst-case tanh.approx error, either way, still within the bound
    for sign in (1.0, -1.0):
        d = _swish_grad_from(_sig_perturbed(u, sign), u)
        r, _ = GC.dw_dgrad_bound(_r16(ga * d), ga, mag, k, F16, u=u)
        assert r <= 1.0, (sign, r)
    # one tap dropped from the transposed convolution
    w_bug = c["w"].clone().reshape(-1, k * k)
    w_bug[:, 7] = 0
    ga_bug, _ = GC.dw_input_grad64(c["dy"], w_bug, c["H"], c["W"], k, c["s"], (c["pad"],) * 4)
    r, _ = GC.dw_dgrad_bound(_r16(ga_bug * GC.swish_grad64(u)), ga, mag, k, F16, u=u)
    assert r > 1.0, r
    # one channel's scale applied twice to the pre-activation
    scale2 = c["scale"].clone()
    u_bug = u.clone()
    u_bug[..., 3] = GC._u32(c["x"][..., 3], scale2[3] * scale2[3], c["shift"][3]).double()
    r, _ = GC.dw_dgrad_bound(_r16(ga * GC.swish_grad64(u_bug)), ga, mag, k, F16, u=u)
    assert r > 1.0, r


def test_dw_dgrad_add_bound():
    """MODE 0: the input gradient plus the residual gradient, rounded once; an extra 16-bit rounding of the sum's first
    operand is visible where the two cancel"""
    c = _dw_case()
    add = torch.randn(*c["ga"].shape, generator=_gen(2)).to(F16)
    ga, mag, k = c["ga"], c["mag"], c["k"]
    ref = ga + add.double()
    once, trip = GC.dw_dgrad_bound(_r16(ref), ga, mag, k, F16, add=add)
    assert once <= 1.0 and trip > 1.0, (once, trip)
    r, _ = GC.dw_dgrad_bound(_r16(_r16(ga).double() + add.double()), ga, mag, k, F16, add=add)
    assert r > 1.0, r


# ---- row kernel: BatchNorm + Swish * gate + residual, and its backward ---------------------------------------------------
def _row_case():
    g = _gen(3)
    N, HW, C = 4, 300, 32
    y = (torch.randn(N, HW, C, generator=g) * 1.5 + 0.3).to(F16)
    scale = 1.0 + 0.2 * torch.randn(C, generator=g)
    shift = 0.3 * torch.randn(C, generator=g)
    gate = torch.sigmoid(torch.randn(N, C, generator=g)).double().unsqueeze(1)
    r = torch.randn(N, HW, C, generator=g).to(F16)
    u = GC._u32(y, scale, shift).double()
    return y, scale, shift, gate, r, u


def test_bn_act_swish_gate_residual_bound():
    y, scale, shift, gate, r, u = _row_case()
    ref, bound = GC.bn_act_bound(u, 1, gate, r, 1, F16)
    assert GC.ulp_ratio(_r16(ref), ref, bound) <= 1.0
    assert GC.ulp_ratio(_trip(ref), ref, bound) > 1.0
    for sign in (1.0, -1.0):
        out = u * _sig_perturbed(u, sign) * gate + r.double()
        assert GC.ulp_ratio(_r16(out), ref, bound) <= 1.0, sign
    # one channel's scale applied twice
    u_bug = u.clone()
    u_bug[..., 5] = GC._u32(y[..., 5], scale[5] * scale[5], shift[5]).double()
    out = GC.swish64(u_bug) * gate + r.double()
    assert GC.ulp_ratio(_r16(out), ref, bound) > 1.0
    # the residual-add variant without an activation, with the gated value rounded to 16 bits before the add
    ref0, bound0 = GC.bn_act_bound(u, 0, gate, r, 1, F16)
    out = _r16(u * gate).double() + r.double()
    assert GC.ulp_ratio(_r16(ref0), ref0, bound0) <= 1.0
    assert GC.ulp_ratio(_r16(out), ref0, bound0) > 1.0


def test_act_bwd_swish_bound():
    y, scale, shift, gate, r, u = _row_case()
    g = _gen(4)
    da = (0.1 * torch.randn(*y.shape, generator=g)).to(F16).double()
    dpool = 0.1 * torch.randn(y.shape[0], 1, y.shape[2], generator=g).double()
    gin = da * gate + dpool / y.shape[1]
    gmag = (da * gate).abs() + dpool.abs() / y.shape[1]
    ref, bound = GC.act_bwd_bound(u, 1, gin, gmag, F16)
    assert GC.ulp_ratio(_r16(ref), ref, bound) <= 1.0
    assert GC.ulp_ratio(_trip(ref), ref, bound) > 1.0
    for sign in (1.0, -1.0):
        d = _swish_grad_from(_sig_perturbed(u, sign), u)
        assert GC.ulp_ratio(_r16(gin * d), ref, bound) <= 1.0, sign
    # the activation derivative rounded to 16 bits before the product
    out = gin * _r16(GC.swish_grad64(u)).double()
    assert GC.ulp_ratio(_r16(out), ref, bound) > 1.0
    # the gate left out of one channel
    gin_bug = gin.clone()
    gin_bug[..., 2] = da[..., 2] + dpool[..., 2] / y.shape[1]
    assert GC.ulp_ratio(_r16(gin_bug * GC.swish_grad64(u)), ref, bound) > 1.0


# ---- max-pool window sum: the gradient gathered over the windows whose arg-max a pixel is ----------------------------------
def test_maxpool_bwd_bound():
    g = _gen(5)
    N, H, W, C = 2, 15, 15, 16
    x = torch.randint(0, 4, (N, H, W, C), generator=g).to(F16)        # small integers: ties, the first maximum decides
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    gy = torch.randn(N, Ho, Wo, C, generator=g).to(F16)
    pool = lambda t: F.max_pool2d(t, 3, 2, 1)
    xr = GC.nchw(x.double()).requires_grad_(True)
    pooled, ind = F.max_pool2d(xr, 3, 2, 1, return_indices=True)
    pooled.backward(GC.nchw(gy.double()))
    ref = GC.nhwc(xr.grad)
    once = GC.maxpool_bwd_bound(_r16(ref), x, gy, pool, F16)
    assert once[0] <= 1.0 and once[1] > 1.0, once
    # a gather that keeps one window's gradient instead of the sum (last writer wins)
    flat = torch.zeros(N, C, H * W, dtype=torch.float64)
    flat.scatter_(2, ind.view(N, C, -1), GC.nchw(gy.double()).view(N, C, -1))
    bug = GC.nhwc(flat.view(N, C, H, W))
    assert int((ref != bug).sum()) > 0
    assert GC.maxpool_bwd_bound(_r16(bug), x, gy, pool, F16)[0] > 1.0


# ---- col2im: overlapping column terms summed once --------------------------------------------------------------------------
def test_col2im_bound():
    g = _gen(6)
    N, H, W, C, k, s, pad = 2, 9, 11, 16, 3, 1, 1
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    dcols = torch.randn(N, C * k * k, Ho * Wo, generator=g).to(F16).double()
    add = torch.randn(N, C, H, W, generator=g).to(F16).double()
    ref = F.fold(dcols, (H, W), k, padding=pad, stride=s) + add
    mag = F.fold(dcols.abs(), (H, W), k, padding=pad, stride=s) + add.abs()
    n = -(-k // s) ** 2 + 1
    bound = GC.sum_bound(ref, mag, n, F16)
    assert GC.ulp_ratio(_r16(ref), ref, bound) <= 1.0
    assert GC.ulp_ratio(_trip(ref), ref, bound) > 1.0
    # one tap dropped
    d_bug = dcols.view(N, C, k * k, -1).clone()
    d_bug[:, :, 4] = 0
    bug = F.fold(d_bug.view(N, C * k * k, -1), (H, W), k, padding=pad, stride=s) + add
    assert GC.ulp_ratio(_r16(bug), ref, bound) > 1.0
    # every partial sum rounded to 16 bits (a 16-bit accumulator)
    acc = add.clone()
    cols = dcols.view(N, C, k, k, Ho, Wo)
    for kh in range(k):
        for kw in range(k):
            t = torch.zeros(N, C, H + 2 * pad, W + 2 * pad, dtype=torch.float64)
            t[:, :, kh:kh + Ho, kw:kw + Wo] = cols[:, :, kh, kw]
            acc = _r16(acc + t[:, :, pad:pad + H, pad:pad + W]).double()
    assert GC.ulp_ratio(acc.to(F16), ref, bound) > 1.0


def test_swish_grad_err_covers_the_sigmoid_error():
    """swish_grad_err against the derivative formed from a sigmoid off by exactly the documented bound, over a dense grid"""
    u = torch.linspace(-40, 40, 200001, dtype=torch.float64)
    exact = GC.swish_grad64(u)
    for sign in (1.0, -1.0):
        s = torch.sigmoid(u) + sign * (GC.E_SIG - 2.0 ** -24)
        err = (_swish_grad_from(s, u) - exact).abs()
        assert bool((err <= GC.swish_grad_err(u)).all())
