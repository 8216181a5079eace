"""GPU checks of the kernels that only the model families' plans launch (Xception, SE-ResNet, ResNet-D), against fp64 torch
on the same rounded 16-bit operands, in the bound style of tests/gpu_checks.py. Each check runs the plan's own pointer mask
and mode arguments, starts every output as NaN (an accumulated one from a known base) and returns {metric: value}; the
thresholds live in tests/test_family_launches_gpu.py."""
import struct

import torch
import torch.nn.functional as F

from deepfake_detection_b200 import _lib
from gpu_checks import (DT, P, TINY16, U_OUT, ULP_IN, _bn_params, _u32, dw_dgrad_bound, dw_input_grad64, maxerr_scaled,
                        maxpool_bwd_bound, nchw, nhwc, ratio_pair, relerr, st, stat_buf, sum_bound)

ACT_NONE, ACT_RELU = 0, 2


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def _bits_equal(a, b):
    return bool(torch.equal(a.view(torch.int16), b.view(torch.int16))) if a.element_size() == 2 else bool(torch.equal(a, b))


# ---- depthwise convolution with a ReLU input (Xception's separable convolutions) ---------------------------------------
def check_dwconv_relu(N, H, W, C, k, s, dtype=torch.bfloat16, bn=True, add=False, seed=0):
    """dfd_dwconv_fwd with act_in = ReLU and dfd_dwconv_bwd_relu, as the Xception plan issues them: bn = the staged input is
    round16(relu(scale*x + shift)) (backward mode 2: gx = dgrad * 1[a > 0] and the BN-backward sums of the stored gx), else
    relu(x) (mode 3: gx = dgrad * 1[x > 0] (+ add)). gy is the depthwise output's gradient itself (no folded BatchNorm
    backward). The backward runs twice in its order-deterministic form (workspace + dfd_ordered_reduce, as the plan runs it)
    and once with the atomic flush.
    The first 8 channels of a BN input have scale 2^-4, shift 0 and inputs of a few 16-bit subnormal steps, so that
    scale*x + shift is positive in fp32 but rounds to zero in the 16-bit type: the mask must be taken on the staged value."""
    assert k == 3 and s == 1, "the ReLU depthwise kernels run k = 3, stride 1 (dwconv.cu:1050)"
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
    w = (torch.randn(C, k * k, device="cuda", generator=g) / k).contiguous()
    scale, shift = _bn_params(C, g) if bn else (None, None)
    if bn and C >= 16:
        steps = torch.randint(-15, 16, (N, H, W, 8), device="cuda", generator=g).double()
        x[..., :8] = (steps * TINY16[dtype]).to(dtype)
        scale[:8], shift[:8] = 2.0 ** -4, 0.0
    out = _nan(N, H, W, C, dtype=dtype)
    _lib.call("dfd_dwconv_fwd", P(x), P(scale), P(shift), P(w), P(out), N, H, W, C, k, s, ACT_RELU, d, None, None, None, st())
    torch.cuda.synchronize()
    # the staged input, exactly as the kernel rounds it
    a = (torch.relu(_u32(x, scale, shift)) if bn else torch.relu(x.float())).to(dtype)
    a64, w64 = nchw(a.double()), w.view(C, 1, k, k).double()
    ref = F.conv2d(a64, w64, padding=(k - 1) // 2, groups=C)
    res = dict(nan=int(torch.isnan(out.float()).sum()))
    # gpu_checks.check_dwconv's element-wise bound without its Swish term (the reference stages the same rounded input), plus
    # half the 16-bit spacing below the normal range: the seeded channels' outputs are subnormal, where the output rounding
    # is off by up to TINY16 / 2 absolutely (fp32 keeps these products and sums to 2^-149)
    mag = F.conv2d(a64.abs(), w64.abs(), padding=(k - 1) // 2, groups=C)
    bound = U_OUT[dtype] * ref.abs() + (ULP_IN[dtype] + 2.0 ** -20) * mag + TINY16[dtype] / 2
    res["fwd_ulp"] = float(((nchw(out.double()) - ref).abs() / (bound + 1e-30)).max())
    del mag, bound, ref
    if bn and C >= 16:      # the seeded channels: fp32-positive inputs that the 16-bit staging turns into zeros
        res["edge_zeros"] = int(((_u32(x, scale, shift)[..., :8] > 0) & (a[..., :8] == 0)).sum())
    gy = (torch.randn(N, H, W, C, device="cuda", generator=g) * 0.1).to(dtype)
    addt = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype) if add else None
    mean = 0.1 * torch.randn(C, device="cuda", generator=g)
    rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
    parts = _lib.lib().cdll.dfd_dwconv_bwd_parts(N, H, W, C, k, s)
    cw = _lib.lib().cdll.dfd_dwconv_block_channels(C)
    cbs = (C + cw - 1) // cw
    ws = _nan(cbs, parts, cw * k * k)
    runs = []
    for det in (True, True, False):
        gx, dW = _nan(N, H, W, C, dtype=dtype), torch.zeros(C, k * k, device="cuda")
        s1, s2 = (stat_buf(C), stat_buf(C)) if bn else (None, None)
        _lib.call("dfd_dwconv_bwd_relu", P(gy), None, None, None, None, P(w), P(x), P(scale), P(shift), P(mean) if bn else None,
                  P(rstd) if bn else None, P(addt), P(gx), P(dW), N, H, W, C, k, s, d, P(s1), P(s2), P(ws) if det else None,
                  ws.numel() * 4 if det else 0, None, st())
        if det:
            raw = b"".join(struct.pack("<QQqqii", P(ws) + cb * parts * cw * k * k * 4, P(dW) + cb * cw * k * k * 4,
                                       min(cw, C - cw * cb) * k * k, cw * k * k, parts, 0) for cb in range(cbs))
            table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
            _lib.call("dfd_ordered_reduce", P(table), cbs, P(dW), (cw * k * k // 4 + 7) // 8 if parts > 64 else 1, st())
        torch.cuda.synchronize()
        runs.append((gx, dW, s1, s2))
    (gx, dW, s1, s2), (gx2, dW2, _, _), (gxa, dWa, _, _) = runs
    res.update(nan_b=int(torch.isnan(gx.float()).sum()), ws_bytes=ws.numel() * 4,
               det_bitwise=_bits_equal(gx, gx2) and bool(torch.equal(dW, dW2)), det_vs_atomic=relerr(dW, dWa),
               det_gx_diff=float((gx.float() - gxa.float()).abs().max()))
    gy64 = nchw(gy.double())
    ga = nhwc(torch.nn.grad.conv2d_input(a64.shape, w64, gy64, padding=(k - 1) // 2, groups=C))
    mask = a.double() > 0                 # the 16-bit staged value (mode 3: x itself, a = relu(x) exactly)
    base = addt.double() if add else torch.zeros_like(ga)
    gref = torch.where(mask, ga + base, base)
    res["dgrad_rel"] = relerr(gx.double(), gref)
    # element-wise (gpu_checks.dw_dgrad_bound, MODES 2 / 3): gy is staged as stored, the mask is exact
    ga64, mag64 = dw_input_grad64(gy, w, H, W, k, s, (1, 1, 1, 1))
    res["dgrad_ulp"], res["dgrad_ulp_bf16trip"] = dw_dgrad_bound(gx, ga64, mag64, k, dtype, add=addt, mask=mask)
    del ga64, mag64
    # the mask, exactly: off it gx is the added gradient (or zero) bit for bit; on it (without `add`, which can absorb a
    # small dgrad in the rounding) gx is not zero where the dgrad is not
    off = ~mask & (gx.double() != base)
    lost = mask & (gx.double() == 0) & (ga.abs() > 1e-6 * float(ga.pow(2).mean().sqrt())) if not add else torch.zeros(())
    res["mask_mismatch"] = int(off.sum()) + int(lost.sum())
    res["wgrad_rel"] = relerr(dW.double(), torch.nn.grad.conv2d_weight(a64, w64.shape, gy64, padding=(k - 1) // 2, groups=C).view(C, k * k))
    if bn:
        gxd = gx.double()
        xhat = (x.double() - mean.double()) * rstd.double()
        res["s1_rel"] = relerr(s1.sum(0), gxd.sum((0, 1, 2)))
        res["s2_rel"] = relerr(s2.sum(0), (gxd * xhat).sum((0, 1, 2)))
    return res


# ---- Xception's strided block tail ---------------------------------------------------------------------------------------
def _tie_inputs(shape, C, dtype, g):
    """16-bit input whose even channels hold quarter steps in [-4, 4] (exact ties in every window) under power-of-two scales
    of both signs and quarter shifts (scale*y + shift exact), and whose odd channels are plain normal samples"""
    y = torch.randn(*shape, C, device="cuda", generator=g)
    q = torch.randint(-16, 17, (*shape, C), device="cuda", generator=g).float() / 4
    even = (torch.arange(C, device="cuda") % 2 == 0)
    y = torch.where(even, q, y).to(dtype)
    scale, shift = _bn_params(C, g)
    pick = torch.tensor([0.5, 1.0, 2.0, -1.0], device="cuda")[torch.randint(0, 4, (C,), device="cuda", generator=g)]
    scale = torch.where(even, pick, scale)
    shift = torch.where(even, torch.randint(-8, 9, (C,), device="cuda", generator=g).float() / 4, shift)
    return y, scale, shift


def check_bn_maxpool(N, H, W, C, dtype=torch.bfloat16, seed=0):
    """dfd_bn_maxpool_add (out = maxpool3x3s2p1(scale*y + shift) + scale_s*ys + shift_s) with and without the arg-max bytes,
    and dfd_maxpool_bn_bwd_reduce (the gather of gy by the arg-max and the BN-backward sums). Reference: torch's max_pool2d on
    the fp32 values the kernel forms (first maximum in row-major window order, -inf padding), sums in fp64."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y, scale, shift = _tie_inputs((N, H, W), C, dtype, g)
    ys = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dtype)
    scale_s, shift_s = _bn_params(C, g)
    out, out2 = _nan(N, Ho, Wo, C, dtype=dtype), _nan(N, Ho, Wo, C, dtype=dtype)
    idx = torch.full((N, Ho, Wo, C), 255, device="cuda", dtype=torch.uint8)
    _lib.call("dfd_bn_maxpool_add", P(y), P(scale), P(shift), P(ys), P(scale_s), P(shift_s), P(out), P(idx), N, H, W, C, d, st())
    _lib.call("dfd_bn_maxpool_add", P(y), P(scale), P(shift), P(ys), P(scale_s), P(shift_s), P(out2), None, N, H, W, C, d, st())
    torch.cuda.synchronize()
    u = nchw(_u32(y, scale, shift)).requires_grad_(True)
    pooled, ind = F.max_pool2d(u, 3, 2, 1, return_indices=True)
    ref = nhwc(pooled.detach().double()) + ys.double() * scale_s.double() + shift_s.double()
    res = dict(nan=int(torch.isnan(out.float()).sum()), out_max=maxerr_scaled(out, ref), noidx_mismatch=int(not _bits_equal(out, out2)))
    # bn_act.cu:1251-1259: the maximum of the fp32 u's (exact, the reference's values), + fmaf(ys, scale_s, shift_s), one store
    sc_mag = nhwc(pooled.detach().double()).abs() + (ys.double() * scale_s.double()).abs() + shift_s.double().abs()
    res["out_ulp"], res["out_ulp_bf16trip"] = ratio_pair(out, ref, sum_bound(ref, sc_mag, 2, dtype))
    iy, ix = nhwc(ind // W), nhwc(ind % W)
    oy = torch.arange(Ho, device="cuda").view(1, Ho, 1, 1)
    ox = torch.arange(Wo, device="cuda").view(1, 1, Wo, 1)
    tap = (iy - (2 * oy - 1)) * 3 + (ix - (2 * ox - 1))
    res["idx_mismatch"] = int((idx.long() != tap).sum())
    # windows whose maximum occurs more than once: the first-maximum rule decides their arg-max
    with torch.no_grad():
        up = pooled.detach()
        upad = F.pad(u.detach(), (1, 1, 1, 1), value=float("-inf"))
        cnt = torch.zeros(up.shape, device="cuda", dtype=torch.uint8)
        for kh in range(3):
            for kw in range(3):
                cnt += upad[:, :, kh:kh + 2 * Ho - 1:2, kw:kw + 2 * Wo - 1:2] == up
        res["tied_windows"] = int((cnt > 1).sum())
        del up, upad, cnt
    gy = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dtype)
    mean = 0.1 * torch.randn(C, device="cuda", generator=g)
    rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
    s1, s2 = stat_buf(C), stat_buf(C)
    gx = _nan(N, H, W, C, dtype=dtype)
    _lib.call("dfd_maxpool_bn_bwd_reduce", P(gy), P(idx), P(y), P(mean), P(rstd), P(gx), N, H, W, C, d, P(s1), P(s2), st())
    pooled.backward(nchw(gy.float()))
    torch.cuda.synchronize()
    gref = nhwc(u.grad.double())
    gxd = gx.double()
    xhat = (y.double() - mean.double()) * rstd.double()
    res["bwd_ulp"], res["bwd_ulp_bf16trip"] = maxpool_bwd_bound(gx, nhwc(u.detach()), gy, lambda t: F.max_pool2d(t, 3, 2, 1), dtype)
    res.update(nan_b=int(torch.isnan(gx.float()).sum()), bwd_max=maxerr_scaled(gx, gref),
               s1_rel=relerr(s1.sum(0), gxd.sum((0, 1, 2))), s2_rel=relerr(s2.sum(0), (gxd * xhat).sum((0, 1, 2))))
    return res


# ---- SE-ResNet stem pool ---------------------------------------------------------------------------------------------------
def check_maxpool_ceil(N, H, W, C, dtype=torch.bfloat16, seed=0):
    """dfd_maxpool_ceil_fwd / _bwd (3x3, stride 2, no padding, ceil mode: the last window clipped) against F.max_pool2d on a
    ReLU output of small integers (exact ties, zeros included): output and arg-max exact, the gathered gradient rounded once"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    x = torch.randint(0, 4, (N, H, W, C), device="cuda", generator=g).to(dtype)
    xr = nchw(x.float()).requires_grad_(True)
    ref, ind = F.max_pool2d(xr, 3, 2, ceil_mode=True, return_indices=True)
    Ho, Wo = ref.shape[2:]
    y = _nan(N, Ho, Wo, C, dtype=dtype)
    idx = torch.full((N, Ho, Wo, C), 255, device="cuda", dtype=torch.uint8)
    _lib.call("dfd_maxpool_ceil_fwd", P(x), P(y), P(idx), N, H, W, C, d, st())
    gy = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dtype)
    gx = _nan(N, H, W, C, dtype=dtype)
    _lib.call("dfd_maxpool_ceil_bwd", P(gy), P(idx), P(gx), N, H, W, C, d, st())
    ref.backward(nchw(gy.float()))
    torch.cuda.synchronize()
    oy = torch.arange(Ho, device="cuda").view(1, Ho, 1, 1)
    ox = torch.arange(Wo, device="cuda").view(1, 1, Wo, 1)
    flat = (2 * oy + idx.long() // 3) * W + 2 * ox + idx.long() % 3
    bwd_ulp = maxpool_bwd_bound(gx, x, gy, lambda t: F.max_pool2d(t, 3, 2, ceil_mode=True), dtype)
    return dict(bwd_ulp=bwd_ulp[0], bwd_ulp_bf16trip=bwd_ulp[1],fwd_mismatch=int((y.float() != nhwc(ref.detach())).sum()), idx_mismatch=int((flat != nhwc(ind)).sum()),
                clipped=int((H - 3) % 2 == 1) + int((W - 3) % 2 == 1), bwd_max=maxerr_scaled(gx, nhwc(xr.grad.double())),
                nan=int(torch.isnan(y.float()).sum()), nan_b=int(torch.isnan(gx.float()).sum()))


# ---- SE-ResNet squeeze-excite tail ---------------------------------------------------------------------------------------
def _se_params(C, Cse, g):
    Wr = torch.randn(Cse, C, device="cuda", generator=g) * (2.0 / C) ** 0.5
    br = torch.randn(Cse, device="cuda", generator=g) * 0.1
    We = torch.randn(C, Cse, device="cuda", generator=g) * (2.0 / Cse) ** 0.5
    be = torch.randn(C, device="cuda", generator=g) * 0.1
    return Wr, br, We, be


def _act(u, act):
    return u.clamp_min(0) if act == ACT_RELU else u


def check_pool_se_relu(N, HW, C, Cse, act, max_chunks, dtype=torch.bfloat16, seed=0):
    """dfd_pool_se_relu at the plan's (N, HW, C, Cse, act, max_chunks): pooled = mean_hw act(scale*y + shift) against fp64; the
    gate sigmoid(We relu(Wr p + br) + be) against the fp64 chain on the kernel's own pooled vector; two launches bit for bit
    (the chunk partials sit in fixed slots and are added in chunk order)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype)
    scale, shift = _bn_params(C, g)
    Wr, br, We, be = _se_params(C, Cse, g)
    outs = []
    for _ in range(2):
        pooled, gate = _nan(N, C), _nan(N, C)
        _lib.call("dfd_pool_se_relu", P(y), P(scale), P(shift), P(pooled), P(Wr), P(br), P(We), P(be), P(gate), N, HW, C, Cse, act,
                  DT[dtype], max_chunks, st())
        torch.cuda.synchronize()
        outs.append((pooled, gate))
    (pooled, gate), (pooled2, gate2) = outs
    p64 = _act(_u32(y, scale, shift).double(), act).mean(1)
    pk = pooled.double()
    gate64 = torch.sigmoid(torch.relu(pk @ Wr.double().t() + br.double()) @ We.double().t() + be.double())
    return dict(pool_rel=relerr(pooled, p64), gate_rel=relerr(gate, gate64), repro=bool(torch.equal(pooled, pooled2) and torch.equal(gate, gate2)),
                nan=int(torch.isnan(pooled).sum() + torch.isnan(gate).sum()))


def _se_bwd_chain64(draw, pooled, Wr, br, We, be, rmask):
    """fp64 SEModule backward chain from dL/dgate: (d_e, r, d_rpre, dpool); rmask: the ReLU mask of r' pre-activation"""
    rpre = pooled @ Wr.t() + br
    r = rpre.clamp_min(0)
    gt = torch.sigmoid(r @ We.t() + be)
    d_e = draw * gt * (1 - gt)
    d_rpre = (d_e @ We) * rmask
    return d_e, r, d_rpre, d_rpre @ Wr


def check_relu_se_bwd(N, HW, C, Cse, act, two, dtype=torch.bfloat16, seed=0):
    """dfd_relu_se_bwd_reduce with the plan's mask (g2 present or absent) and act, then dfd_se_fc_wgrad on its outputs:
    gm = round16(g + g2) * (out > 0) bit for bit; draw = sum_hw gm * act(scale*y + shift) against fp64; d_e, r, d_rpre, dpool
    against the fp64 chain on the kernel's own draw (d_rpre under the kernel's ReLU mask of r, i.e. r > 0, whose values are
    checked themselves); the SE weight gradients against fp64 on the kernel's vectors; every output of two launches bit for bit"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    gr = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype)
    g2 = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype) if two else None
    y = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype)
    out = torch.relu(torch.randn(N, HW, C, device="cuda", generator=g)).to(dtype)
    scale, shift = _bn_params(C, g)
    pooled = torch.rand(N, C, device="cuda", generator=g)
    Wr, br, We, be = _se_params(C, Cse, g)
    base = [torch.randn(*t.shape, device="cuda", generator=g) for t in (Wr, br, We, be)]
    runs = []
    for _ in range(2):
        gm = _nan(N, HW, C, dtype=dtype)
        v = dict(draw=_nan(N, C), d_e=_nan(N, C), r=_nan(N, Cse), d_rpre=_nan(N, Cse), dpool=_nan(N, C))
        _lib.call("dfd_relu_se_bwd_reduce", P(gr), P(g2), P(y), P(out), P(scale), P(shift), P(gm), P(v["draw"]), P(pooled), P(Wr),
                  P(br), P(We), P(be), P(v["d_e"]), P(v["r"]), P(v["d_rpre"]), P(v["dpool"]), N, HW, C, Cse, act, d, st())
        wg = [b.clone() for b in base]
        _lib.call("dfd_se_fc_wgrad", P(v["d_e"]), P(v["r"]), P(v["d_rpre"]), P(pooled), *[P(t) for t in wg], N, C, Cse, st())
        torch.cuda.synchronize()
        runs.append((gm, v, wg))
    (gm, v, wg), (gm2, v2, wg2) = runs
    gs = (gr.float() + g2.float()).to(dtype) if two else gr
    gm_ref = torch.where(out.float() > 0, gs, torch.zeros_like(gs))
    res = dict(gm_mismatch=int((gm.view(torch.int16) != gm_ref.view(torch.int16)).sum()),
               nan=sum(int(torch.isnan(t.float()).sum()) for t in [gm] + list(v.values())),
               repro=_bits_equal(gm, gm2) and all(torch.equal(v[k], v2[k]) for k in v) and all(torch.equal(a, b) for a, b in zip(wg, wg2)))
    a = _act(_u32(y, scale, shift).double(), act)
    res["draw_rel"] = relerr(v["draw"], (gm_ref.double() * a).sum(1))
    d64 = [t.double() for t in (Wr, br, We, be)]
    d_e, r, d_rpre, dpool = _se_bwd_chain64(v["draw"].double(), pooled.double(), *d64, (v["r"] > 0).double())
    res.update(d_e_rel=relerr(v["d_e"], d_e), r_rel=relerr(v["r"], r), d_rpre_rel=relerr(v["d_rpre"], d_rpre), dpool_rel=relerr(v["dpool"], dpool))
    res.update(_wgrad_errs(wg, base, v["d_e"], v["r"], v["d_rpre"], pooled))
    return res


def _wgrad_errs(wg, base, d_e, r, d_rpre, pooled):
    """the SE parameter gradients that dfd_se_fc_wgrad added to `base`, against fp64 sums over the images"""
    ref = (d_rpre.double().t() @ pooled.double(), d_rpre.double().sum(0), d_e.double().t() @ r.double(), d_e.double().sum(0))
    return {k: relerr(w.double() - b.double(), rf) for k, w, b, rf in zip(("dWr_rel", "dbr_rel", "dWe_rel", "dbe_rel"), wg, base, ref)}


def check_se_fc_wgrad(N, C, Cse, seed=0):
    """dfd_se_fc_wgrad (accumulating into the gradient arena) at the plan's (N, C, Cse): its four gradients against fp64, two
    launches bit for bit (the image-split partials are added in a fixed order)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d_e, pooled = torch.randn(N, C, device="cuda", generator=g), torch.rand(N, C, device="cuda", generator=g)
    r = torch.relu(torch.randn(N, Cse, device="cuda", generator=g))
    d_rpre = torch.randn(N, Cse, device="cuda", generator=g) * (r > 0)
    base = [torch.randn(*s, device="cuda", generator=g) for s in ((Cse, C), (Cse,), (C, Cse), (C,))]
    runs = []
    for _ in range(2):
        wg = [b.clone() for b in base]
        _lib.call("dfd_se_fc_wgrad", P(d_e), P(r), P(d_rpre), P(pooled), *[P(t) for t in wg], N, C, Cse, st())
        torch.cuda.synchronize()
        runs.append(wg)
    res = _wgrad_errs(runs[0], base, d_e, r, d_rpre, pooled)
    res["repro"] = all(torch.equal(a, b) for a, b in zip(*runs))
    return res


# ---- ResNet-D average-pool shortcut ----------------------------------------------------------------------------------------
def check_avgpool2(N, H, W, C, add=True, dtype=torch.bfloat16, seed=0):
    """dfd_avgpool2_fwd / dfd_avgpool2_bwd_add against fp64 F.avg_pool2d(2, 2, ceil_mode=True, count_include_pad=False) and its
    autograd (+ the main-path gradient `add` as the plan passes it, or none): each output a sum of <= 4 16-bit terms times
    1 / count, rounded once"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
    y = _nan(N, Ho, Wo, C, dtype=dtype)
    _lib.call("dfd_avgpool2_fwd", P(x), P(y), N, H, W, C, d, st())
    dy = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dtype)
    addt = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype) if add else None
    dx = _nan(N, H, W, C, dtype=dtype)
    _lib.call("dfd_avgpool2_bwd_add", P(dy), P(addt), P(dx), N, H, W, C, d, st())
    torch.cuda.synchronize()
    xr = nchw(x.double()).requires_grad_(True)
    ref = F.avg_pool2d(xr, 2, 2, ceil_mode=True, count_include_pad=False)
    ref.backward(nchw(dy.double()))
    gref = nhwc(xr.grad) + (addt.double() if add else 0.0)
    res = dict(fwd_max=maxerr_scaled(y, nhwc(ref.detach())), bwd_max=maxerr_scaled(dx, gref),
               nan=int(torch.isnan(y.float()).sum()), nan_b=int(torch.isnan(dx.float()).sum()))
    # bn_act.cu:1159-1179: <= 4 terms summed in fp32, times 1 / count (1, 2 or 4: exact); bn_act.cu:1206: one fmaf
    with torch.no_grad():
        fref = nhwc(ref.detach())
        fmag = nhwc(F.avg_pool2d(xr.detach().abs(), 2, 2, ceil_mode=True, count_include_pad=False))
        res["fwd_ulp"], res["fwd_ulp_bf16trip"] = ratio_pair(y, fref, sum_bound(fref, fmag, 4, dtype))
        bmag = nhwc(xr.grad).abs() + (addt.double().abs() if add else 0.0)
        res["bwd_ulp"], res["bwd_ulp_bf16trip"] = ratio_pair(dx, gref, sum_bound(gref, bmag, 1, dtype))
    return res


# ---- dense convolutions through im2col ---------------------------------------------------------------------------------------
def check_im2col(N, H, W, C, k, s, pad, add=False, dtype=torch.bfloat16, seed=0):
    """dfd_im2col (a copy: bit for bit against F.unfold) and dfd_col2im (the sum of at most k^2 16-bit column terms, plus
    `add` or none, rounded once) at the plan's (k, stride, pad)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
    cols = _nan(N * Ho * Wo, k * k * C, dtype=dtype)
    _lib.call("dfd_im2col", P(x), P(cols), N, H, W, C, k, s, pad, d, st())
    torch.cuda.synchronize()
    res = dict(nan=int(torch.isnan(cols.float()).sum()))
    # F.unfold orders a column (c, kh, kw); the kernel's row is (kh, kw, c)
    diff = 0
    per = max(1, (64 << 20) // (C * k * k * Ho * Wo))
    for n0 in range(0, N, per):
        n1 = min(N, n0 + per)
        ref = F.unfold(nchw(x[n0:n1]), k, padding=pad, stride=s).view(n1 - n0, C, k * k, Ho * Wo).permute(0, 3, 2, 1)
        got = cols[n0 * Ho * Wo:n1 * Ho * Wo].view(n1 - n0, Ho * Wo, k * k, C)
        diff += int((got.view(torch.int16) != ref.contiguous().view(torch.int16)).sum())
        del ref
    res["cols_mismatch"] = diff
    dcols = torch.randn(N * Ho * Wo, k * k * C, device="cuda", generator=g).to(dtype)
    addt = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype) if add else None
    dx = _nan(N, H, W, C, dtype=dtype)
    _lib.call("dfd_col2im", P(dcols), P(addt), P(dx), N, H, W, C, k, s, pad, d, st())
    torch.cuda.synchronize()
    gref = torch.zeros(N, C, H, W, device="cuda", dtype=torch.float64)
    for n0 in range(0, N, per):
        n1 = min(N, n0 + per)
        dc = dcols[n0 * Ho * Wo:n1 * Ho * Wo].view(n1 - n0, Ho * Wo, k * k, C).permute(0, 3, 2, 1).reshape(n1 - n0, C * k * k, Ho * Wo)
        gref[n0:n1] = F.fold(dc.double(), (H, W), k, padding=pad, stride=s)
    gref = nhwc(gref) + (addt.double() if add else 0.0)
    res.update(col2im_max=maxerr_scaled(dx, gref), nan_b=int(torch.isnan(dx.float()).sum()))
    # conv_dense.cu:50-71: add, then every overlapping column term (ceil(k/s)^2 at most) summed in fp32, one store
    gmag = torch.zeros(N, C, H, W, device="cuda", dtype=torch.float64)
    for n0 in range(0, N, per):
        n1 = min(N, n0 + per)
        dc = dcols[n0 * Ho * Wo:n1 * Ho * Wo].view(n1 - n0, Ho * Wo, k * k, C).permute(0, 3, 2, 1).reshape(n1 - n0, C * k * k, Ho * Wo)
        gmag[n0:n1] = F.fold(dc.double().abs(), (H, W), k, padding=pad, stride=s)
    gmag = nhwc(gmag) + (addt.double().abs() if add else 0.0)
    n = -(-k // s) ** 2 + 1
    res["col2im_ulp"], res["col2im_ulp_bf16trip"] = ratio_pair(dx, gref, sum_bound(gref, gmag, n, dtype))
    return res
