"""GPU checks of the TF "SAME" kernels against fp64 torch (F.pad in front of an unpadded convolution, and autograd) on the
same rounded operands, in the bound style of tests/gpu_checks.py. Each check returns {metric: value}; the thresholds live in
tests/test_tf_efficientnet_gpu.py."""
import struct

import torch
import torch.nn.functional as F

from deepfake_detection_b200 import _lib
from gpu_checks import DT, P, nchw, relerr, st, stat_buf


def _same_pads(extent, k, s):
    total = max((-(-extent // s) - 1) * s + k - extent, 0)
    return total // 2, total - total // 2


def _ordered_reduce(ws, dW, C, k, parts, cw):
    cbs = (C + cw - 1) // cw
    raw = b"".join(struct.pack("<QQqqii", P(ws) + cb * parts * cw * k * k * 4, P(dW) + cb * cw * k * k * 4,
                               min(cw, C - cw * cb) * k * k, cw * k * k, parts, 0) for cb in range(cbs))
    table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    _lib.call("dfd_ordered_reduce", P(table), cbs, P(dW), (cw * k * k // 4 + 7) // 8 if parts > 64 else 1, st())


def check_dw_pad(N, H, W, C, k, s, pt, pl, dtype=torch.bfloat16, seed=0, bwd=True, stats=True):
    """dfd_dwconv_fwd_pad (BN + Swish input, statistics) and dfd_dwconv_bwd_pad (mode 1, order-deterministic workspace + the
    ordered reduce, as the training plan runs them) against fp64 torch. At symmetric pads also the symmetric entry points,
    which must give the same bits (`sym_*_mismatch`). Two runs of the backward give the same bits (`bwd_bitwise`).
    stats=False: also the eval form of the forward (no statistics), which must store the same bits (`nostats_mismatch`)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    ho_, wo_ = -(-H // s), -(-W // s)
    pb, pa = _same_pads(H, k, s)
    qb, qa = _same_pads(W, k, s)
    assert (pb, qb) == (pt, pl), (pb, qb, pt, pl)
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
    w = (torch.randn(C, 1, k, k, device="cuda", generator=g) * (1.0 / k)).contiguous()
    scale = 1.0 + 0.2 * torch.randn(C, device="cuda", generator=g)
    shift = 0.3 * torch.randn(C, device="cuda", generator=g)
    out = torch.full((N, ho_, wo_, C), float("nan"), device="cuda", dtype=dtype)
    s1, s2 = stat_buf(C), stat_buf(C)
    _lib.call("dfd_dwconv_fwd_pad", P(x), P(scale), P(shift), P(w), P(out), N, H, W, C, k, s, pt, pl, 1, d, P(s1), P(s2), None, st())
    torch.cuda.synchronize()
    res = dict(nan=int(torch.isnan(out.float()).sum()))
    if not stats:
        o2 = torch.full_like(out, float("nan"))
        _lib.call("dfd_dwconv_fwd_pad", P(x), P(scale), P(shift), P(w), P(o2), N, H, W, C, k, s, pt, pl, 1, d, None, None, None, st())
        torch.cuda.synchronize()
        res["nostats_mismatch"] = int((o2.view(torch.int16) != out.view(torch.int16)).sum())
        del o2
    sym = (pt, pl) == ((k - 1) // 2, (k - 1) // 2)
    if sym:
        o2, t1, t2 = torch.full_like(out, float("nan")), stat_buf(C), stat_buf(C)
        _lib.call("dfd_dwconv_fwd", P(x), P(scale), P(shift), P(w), P(o2), N, H, W, C, k, s, 1, d, P(t1), P(t2), None, st())
        torch.cuda.synchronize()
        res["sym_fwd_mismatch"] = int((o2.view(torch.int16) != out.view(torch.int16)).sum())
        del o2
    # fp64 reference on the same rounded operands: a = round16(swish(scale*x + shift)), F.pad, unpadded depthwise conv.
    xr = nchw(x.double()).requires_grad_(True)
    u = xr * scale.double().view(1, C, 1, 1) + shift.double().view(1, C, 1, 1)
    a = u * torch.sigmoid(u)
    a_q = a + (a.to(dtype).double() - a).detach()          # value rounded to the 16-bit type, gradient straight through
    wr = w.double().clone().requires_grad_(True)
    padding = (pl, qa, pt, pa)
    ref = F.conv2d(F.pad(a_q, padding), wr, stride=s, groups=C)
    # bound of gpu_checks.check_dwconv (there in fp32, here fp64): output half-ulp, the staged input's rounding and the
    # tanh.approx sigmoid (2^-11 absolute), fp32 accumulation of <= 25 taps
    u_out, ulp_in = (2.0 ** -8, 2.0 ** -7) if dtype == torch.bfloat16 else (2.0 ** -11, 2.0 ** -10)
    with torch.no_grad():
        mag = F.conv2d(F.pad(a_q.abs(), padding), w.double().abs(), stride=s, groups=C)
        bound = u_out * ref.abs() + (ulp_in + 2.0 ** -20) * mag
        bound += (1 + ulp_in) * 2.0 ** -11 * F.conv2d(F.pad(u.abs(), padding), w.double().abs(), stride=s, groups=C)
        res["fwd_ulp"] = float(((nchw(out.double()) - ref).abs() / (bound + 1e-30)).max())
        del mag, bound
    of = out.double()
    res["sum_rel"] = relerr(s1.sum(0), of.sum((0, 1, 2)))
    res["sq_rel"] = relerr(s2.sum(0), (of * of).sum((0, 1, 2)))
    if not bwd:
        return res
    gy = (torch.randn(N, ho_, wo_, C, device="cuda", generator=g) * 0.1).to(dtype)
    cA = 1.0 + 0.1 * torch.randn(C, device="cuda", generator=g)
    cB = 0.05 * torch.randn(C, device="cuda", generator=g)
    cC = 0.01 * torch.randn(C, device="cuda", generator=g)
    mean = 0.1 * torch.randn(C, device="cuda", generator=g)
    rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
    dy = (cA * gy.float() + cB * out.float() + cC).to(dtype).double()       # the kernel stages dy rounded to the 16-bit type
    ref.backward(nchw(dy))
    parts = _lib.lib().cdll.dfd_dwconv_bwd_parts(N, H, W, C, k, s)
    cw = _lib.lib().cdll.dfd_dwconv_block_channels(C)
    cbs = (C + cw - 1) // cw

    def run(entry, pads):
        gx = torch.full((N, H, W, C), float("nan"), device="cuda", dtype=dtype)
        dW = torch.zeros_like(w)
        b1, b2 = stat_buf(C), stat_buf(C)
        ws = torch.full((cbs, parts, cw * k * k), float("nan"), device="cuda")
        _lib.call(entry, P(gy), P(out), P(cA), P(cB), P(cC), P(w), P(x), P(scale), P(shift), P(mean), P(rstd), None, P(gx), P(dW),
                  N, H, W, C, k, s, *pads, d, P(b1), P(b2), P(ws), ws.numel() * 4, None, st())
        _ordered_reduce(ws, dW, C, k, parts, cw)
        torch.cuda.synchronize()
        return gx, dW, b1, b2

    gx, dW, b1, b2 = run("dfd_dwconv_bwd_pad", (pt, pl))
    gx2, dW2, _, _ = run("dfd_dwconv_bwd_pad", (pt, pl))
    res["bwd_bitwise"] = bool(torch.equal(dW, dW2)) and bool(torch.equal(gx.view(torch.int16), gx2.view(torch.int16)))
    del gx2, dW2
    if sym:
        gx3, dW3, _, _ = run("dfd_dwconv_bwd", ())
        res["sym_bwd_mismatch"] = int((gx3.view(torch.int16) != gx.view(torch.int16)).sum()) + int((dW3 != dW).sum())
        del gx3, dW3
    res["nan_b"] = int(torch.isnan(gx.float()).sum())
    res["ws_bytes"] = cbs * parts * cw * k * k * 4
    # xr.grad = scale * (dgrad * swish'(u)); the kernel stores gu = dgrad * swish'(u), rounded to the 16-bit type
    gu_ref = xr.grad / scale.double().view(1, C, 1, 1)
    res["dgrad_rel"] = relerr(nchw(gx.double()), gu_ref)
    res["wgrad_rel"] = relerr(dW.double(), wr.grad)
    gxd = gx.double()
    xhat = (x.double() - mean.double()) * rstd.double()
    res["bs1_rel"] = relerr(b1.sum(0), gxd.sum((0, 1, 2)))
    res["bs2_rel"] = relerr(b2.sum(0), (gxd * xhat).sum((0, 1, 2)))
    return res


def check_stem_im2col_pad(N, Cin, H, W, k, s, pt, pl, dtype=torch.bfloat16, seed=0):
    """im2col rows of the TF-'SAME'-padded NCHW image: exact against F.unfold(F.pad(x)); at symmetric pads also bit-equal to
    dfd_stem_im2col"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g).to(dtype)
    taps = Cin * k * k
    Kp = (taps + 7) // 8 * 8
    ho_, wo_ = -(-H // s), -(-W // s)
    pb, pa = _same_pads(H, k, s)
    qb, qa = _same_pads(W, k, s)
    assert (pb, qb) == (pt, pl)
    cols = torch.full((N * ho_ * wo_, Kp), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_stem_im2col_pad", P(x), P(cols), N, Cin, H, W, k, s, pt, pl, Kp, DT[dtype], st())
    torch.cuda.synchronize()
    ref = F.unfold(F.pad(x.float(), (pl, qa, pt, pa)), k, stride=s).transpose(1, 2).reshape(N * ho_ * wo_, taps)
    res = dict(diff=float((cols[:, :taps].float() - ref).abs().max()), nan=int(torch.isnan(cols.float()).sum()),
               pad_max=float(cols[:, taps:].float().abs().max()) if Kp > taps else 0.0)
    if (pt, pl) == ((k - 1) // 2, (k - 1) // 2):
        c2 = torch.full_like(cols, float("nan"))
        _lib.call("dfd_stem_im2col", P(x), P(c2), N, Cin, H, W, k, s, (k - 1) // 2, Kp, DT[dtype], st())
        torch.cuda.synchronize()
        res["sym_mismatch"] = int((c2.view(torch.int16) != cols.view(torch.int16)).sum())
    return res
