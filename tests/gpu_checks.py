"""GPU parity checks of every C-ABI kernel against plain PyTorch fp32 arithmetic ON THE SAME ROUNDED INPUTS.
Each check returns {metric: value}; thresholds live in the pytest wrappers (tests/test_kernels_gpu.py).
Shared by tools/gpu_diag.py, which runs them all without stopping at the first failure.

Tolerances (written here once): tensors stored in bf16 carry 2^-9 relative rounding per element, so
  * max |err| <= 2^-7 * (|ref| + scale)   for 16-bit outputs (scale = rms of the reference tensor),
  * rel-L2 <= 2e-3                        for fp32 reductions (statistics, weight gradients) of bf16 data,
  * 1e-5 relative for pure fp32 kernels (optimizers, SE FCs, head).
"""
import math

import torch
import torch.nn.functional as F

from deepfake_detection_b200 import _lib

DT = {torch.bfloat16: 0, torch.float16: 1}


def P(t):
    return None if t is None else t.data_ptr()


def st():
    return torch.cuda.current_stream().cuda_stream


def relerr(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def maxerr_scaled(a, b):
    """max |a-b| / (|b| + rms(b))"""
    a, b = a.double(), b.double()
    scale = b.pow(2).mean().sqrt() + 1e-30
    return float(((a - b).abs() / (b.abs() + scale)).max())


# ---- element-wise error bounds ---------------------------------------------------------------------------------------------
# A 16-bit output is held to |out - ref| <= bound element by element, the bound a sum of named terms, each traced to a step of
# the kernel's arithmetic. The reference rounds where the kernel rounds (16-bit staged operands, the fp32 fmaf of u), so the
# terms cover only what the kernel does in fp32 and its final store. The helpers work on CPU and GPU tensors alike.
#
# half an ulp of the 16-bit output (relative), the largest relative ulp of a 16-bit input, the smallest positive 16-bit value
U_OUT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
ULP_IN = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}
TINY16 = {torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24}
# sigmoid_fast (common.cuh:97) = fmaf(tanh.approx(x / 2), 0.5, 0.5): tanh.approx.f32 has at most 2^-10.987 relative error
# (PTX ISA) and |tanh| <= 1, halved by the fmaf, plus the fmaf's own fp32 rounding (2^-24, as s <= 1): absolute on s
E_TANH = 2.0 ** -10.987
E_SIG = 0.5 * E_TANH + 2.0 ** -24
# the scaled bound of the fp16 tensor-core contractions (the fp16 GEMM's, tests/test_plan_launches_gpu.OUT_FP16_GEMM)
OUT_FP16_TC = 2.0 ** -9


def ulp_ratio(out, ref, bound):
    """max |out - ref| / bound (<= 1: every element within its bound)"""
    return float(((out.double() - ref.double()).abs() / (bound.double() + 1e-300)).max())


def bf16_trip(out):
    """the output rounded through bf16 and back: what a kernel that rounds through bf16 somewhere would store"""
    return out.to(torch.bfloat16).to(out.dtype)


def out_term(ref, dtype):
    """the kernel's one rounding of its fp32 result to the 16-bit output: half an ulp, or half the subnormal spacing"""
    return U_OUT[dtype] * ref.double().abs() + TINY16[dtype] / 2


def in_term(mag, dtype):
    """an operand rounded to 16 bits at a point where the reference cannot round it identically: one ulp of |operand| * |weight|"""
    return ULP_IN[dtype] * mag


def acc_term(mag, n=16):
    """an fp32 evaluation of a short sum or chain of n operations (taps, pool windows, col2im overlaps, the fmaf's of a row
    kernel): at most n roundings of 2^-24 of the partial sums, each <= mag = the same sum of absolute values; 2^-20 for n <= 16"""
    return max(n, 16) * 2.0 ** -24 * mag


def swish64(u):
    return u * torch.sigmoid(u)


def swish_grad64(u):
    s = torch.sigmoid(u)
    return s * (1 + u * (1 - s))


def swish_fwd_term(u, mult):
    """act_fwd<SWISH>(u) = u * sigmoid_fast(u) (common.cuh:102): |u| E_SIG from the sigmoid, 2^-24 |swish| from the product;
    times mult = |what the activation is multiplied by| (gate, weight)"""
    return (u.abs() * E_SIG + 2.0 ** -24 * swish64(u).abs()) * mult


def swish_grad_err(u):
    """|act_bwd<SWISH>(u) - swish'(u)|: d(s) = fmaf(s, fmaf(-u, s, u), s) = s + u s - u s^2 (common.cuh:110) with s off by
    delta, |delta| <= E_SIG: d(s + delta) - d(s) = delta (1 + u (1 - 2 s)) - u delta^2; the two fmaf's round to fp32 at
    2^-24 (|s u (1 - s)| + |d|) <= 2^-23 (s + |s u (1 - s)|)"""
    s = torch.sigmoid(u)
    return (1 + u * (1 - 2 * s)).abs() * E_SIG + u.abs() * E_SIG ** 2 + 2.0 ** -23 * (s + (s * u * (1 - s)).abs())


def swish_bwd_term(u, mult):
    """a gradient of magnitude mult times act_bwd<SWISH>(u)"""
    return swish_grad_err(u) * mult


def elem_bound(ref, dtype, *terms):
    """out_term + the error of the fp32 value before the store (1 + U_OUT: the store's rounding is relative to that value)"""
    b = out_term(ref, dtype)
    for t in terms:
        b = b + (1 + U_OUT[dtype]) * t
    return b


def ratio_pair(out, ref, bound):
    """(ratio of the output, ratio of the output rounded through bf16) on the same reference and bound"""
    return ulp_ratio(out, ref, bound), ulp_ratio(bf16_trip(out), ref, bound)


def _scaled_pair(out, ref, to_nchw=True):
    """maxerr_scaled of a 16-bit NHWC output (to_nchw: against an NCHW reference) against an fp64 reference, and of the output
    rounded through bf16"""
    if to_nchw:
        out = nchw(out)
    return maxerr_scaled(out.double(), ref), maxerr_scaled(bf16_trip(out).double(), ref)


def maxpool_bwd_bound(gx, x, gy, pool, dtype):
    """a max-pool's gathered gradient (dfd_maxpool_bwd, dfd_maxpool_ceil_bwd, dfd_maxpool_bn_bwd_reduce; conv_dense.cu:271-293,
    bn_act.cu:1296-1314): the fp32 sum of the <= 4 window gradients routed to a pixel, rounded once. Reference: fp64 autograd
    of `pool` on the values the kernel compared (NHWC x; same windows, same first-maximum rule), and the same routing of |gy|
    for the sum's magnitude. Returns (ratio, ratio of the output rounded through bf16)."""
    xr = nchw(x.double()).requires_grad_(True)
    y = pool(xr)
    ref, = torch.autograd.grad(y, xr, nchw(gy.double()), retain_graph=True)
    mag, = torch.autograd.grad(y, xr, nchw(gy.double()).abs())
    ref, mag = nhwc(ref), nhwc(mag)
    return ratio_pair(gx, ref, sum_bound(ref, mag, 4, dtype))


def bn_act_bound(u, act, gt, r, res_mode, dtype):
    """(reference, bound) of dfd_bn_act (bn_act.cu:233-246): act(u) [* gate] [+ res] [relu], every step in fp32 (relu is
    1-Lipschitz), one 16-bit store. u: the fp32 fmaf(y, scale, shift) in fp64; gt: the gate broadcast (or 1); r: the residual
    or None. Terms: the fp32 steps over |act(u) gate| + |res|, and for Swish the tanh.approx term on |u gate|."""
    a = _act_ref(u, act)[0] * gt
    ref, mag = a, a.abs()
    if r is not None:
        ref, mag = ref + r.double(), mag + r.double().abs()
    if res_mode == 2:
        ref = ref.clamp_min(0)
    terms = [acc_term(mag, 4)] + ([swish_fwd_term(u, gt.abs())] if act == 1 else [])
    return ref, elem_bound(ref, dtype, *terms)


def act_bwd_bound(u, act, gin, gmag, dtype):
    """(reference, bound) of dfd_act_bwd (bn_act.cu:879-884): gin = fmaf(da, gate, dpool * inv_hw) in fp32 (gmag = |da gate| +
    |dpool| / hw), times act_bwd(u) (Swish: the tanh.approx term of swish_grad_err on |gin|), one 16-bit store"""
    dact = _act_ref(u, act)[1]
    ref = gin * dact
    gacc = acc_term(gmag, 4)
    derr = swish_grad_err(u) if act == 1 else torch.zeros_like(u)
    terms = [gacc * (dact.abs() + derr)] + ([swish_bwd_term(u, gmag + gacc)] if act == 1 else [])
    return ref, elem_bound(ref, dtype, *terms)


def sum_bound(ref, mag, n, dtype):
    """a short fp32 sum of n stored terms (pool windows, col2im overlaps, an added gradient) rounded once to 16 bits"""
    return elem_bound(ref, dtype, acc_term(mag, n))


def _u32(y, scale, shift):
    """fmaf(y, scale, shift) as the kernels form it: the product of a 16-bit and an fp32 value is exact in fp64, the sum is
    rounded to fp32 (the fp64 rounding in between changes the result only at an exact fp32 tie)"""
    return (y.double() * scale.double() + shift.double()).float()


def staged_dy(gy, yout, cA, cB, cC, dtype):
    """the gradient tile the depthwise backward stages (dwconv.cu stage_grad_tile): round16(fmaf(cA, gy, fmaf(cB, yout, cC))),
    in fp64 (exact products, each fmaf rounded to fp32 as the kernel rounds it)"""
    inner = (cB.double() * yout.double() + cC.double()).float()
    return (cA.double() * gy.double() + inner.double()).float().to(dtype).double()


def dw_input_grad64(dy, w, H, W, k, s, pads):
    """the depthwise input gradient in fp64 and the same sum over |w| |dy| (NHWC): dy [N, Ho, Wo, C], w [C, k*k] or
    [C, 1, k, k], pads (top, bottom, left, right) of the forward"""
    N, C = dy.shape[0], dy.shape[3]
    pt, pb, pl, pr = pads
    shape = (N, C, H + pt + pb, W + pl + pr)
    w64, d64 = w.double().reshape(C, 1, k, k), nchw(dy.double())
    ga = torch.nn.grad.conv2d_input(shape, w64, d64, stride=s, groups=C)[:, :, pt:pt + H, pl:pl + W]
    mag = torch.nn.grad.conv2d_input(shape, w64.abs(), d64.abs(), stride=s, groups=C)[:, :, pt:pt + H, pl:pl + W]
    return nhwc(ga), nhwc(mag)


def dw_dgrad_bound(gx, ga, mag, k, dtype, u=None, add=None, mask=None):
    """element-wise bound of a depthwise input gradient (dwconv.cu dwconv_bwd_kernel / dwconv_dgrad_kernel): the fp32 sum of
    k*k taps of the staged dy (acc_term over mag), then
      u given (MODE 1): gu = round16(acc * act_bwd<SWISH>(u)) - the tanh.approx term on |acc| and the product's rounding;
      mask given (MODES 2, 3): round16(acc * mask (+ add));  else (MODE 0): round16(acc (+ add)).
    Returns (ratio, ratio of the output rounded through bf16)."""
    if u is not None:
        d, err = swish_grad64(u), swish_grad_err(u)
        ref = ga * d
        acc = acc_term(mag, k * k + 1)
        bound = elem_bound(ref, dtype, acc * (d.abs() + err), swish_bwd_term(u, ga.abs() + acc))
    else:
        m = mask.double() if mask is not None else 1.0
        ref = ga * m + (add.double() if add is not None else 0.0)
        bound = elem_bound(ref, dtype, acc_term(mag * m + (add.double().abs() if add is not None else 0.0), k * k + 1))
    return ratio_pair(gx, ref, bound)


def slots():
    return _lib.lib().stat_slots


def stat_buf(C, dev="cuda"):
    return torch.zeros(slots(), C, dtype=torch.float64, device=dev)


def nhwc(x):  # [N,C,H,W] -> [N,H,W,C] contiguous
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------------------------
def check_gemm(impl, M, K, N, dtype=torch.bfloat16, with_stats=True, with_add=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
    B = (torch.randn(N, K, device="cuda", generator=g) * (1.0 / math.sqrt(K))).to(dtype)
    C = torch.full((M, N), float("nan"), device="cuda", dtype=dtype)
    add = (torch.randn(M, N, device="cuda", generator=g)).to(dtype) if with_add else None
    s1, s2 = (stat_buf(N), stat_buf(N)) if with_stats else (None, None)
    if impl == "tc":
        assert not with_add
        _lib.call("dfd_gemm_tn", P(A), P(B), P(C), M, N, K, DT[dtype], P(s1), P(s2), None, st())
    elif impl.startswith("rowpack"):
        # small-K path: block-diagonal weight built on the device, `pack` rows of A per TMA row
        import struct
        pack = int(impl[len("rowpack"):])
        Bd = torch.full((pack * N, pack * K), float("nan"), device="cuda", dtype=dtype)
        table = torch.frombuffer(bytearray(struct.pack("<QQiiii", P(B), P(Bd), N, K, pack, 0)), dtype=torch.uint8).cuda()
        _lib.call("dfd_blockdiag_weights", P(table), 1, DT[dtype], st())
        _lib.call("dfd_gemm_tn_rowpack", P(A), P(Bd), P(C), M, N, K, pack, DT[dtype], P(s1), P(s2), None, st())
    else:
        _lib.call("dfd_gemm_tn_mma", P(A), P(B), P(C), P(add), M, N, K, DT[dtype], P(s1), P(s2), st())
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    if with_add:
        ref = ref.to(dtype).float() + add.float()
    out = dict(out_max=maxerr_scaled(C.float(), ref), out_rel=relerr(C.float(), ref), nan=int(torch.isnan(C.float()).sum()))
    if with_stats:
        cf = C.double()
        out["sum_rel"] = relerr(s1.sum(0), cf.sum(0))
        out["sq_rel"] = relerr(s2.sum(0), (cf * cf).sum(0))
    return out


def check_wgrad(M, Nw, Kw, dtype=torch.bfloat16, seed=0, impl="dfd_gemm_wgrad_mma", det=False):
    """det: the order-deterministic flush of dfd_gemm_wgrad (workspace given): also returns whether two launches agree bit
    for bit and the distance to the atomic flush"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    G = (torch.randn(M, Nw, device="cuda", generator=g) * 0.3).to(dtype)
    X = (torch.randn(M, Kw, device="cuda", generator=g)).to(dtype)
    dW = torch.zeros(Nw, Kw, device="cuda")
    out = {}
    if impl == "dfd_gemm_wgrad":
        if not det:
            _lib.call(impl, P(G), P(X), P(dW), M, Nw, Kw, DT[dtype], None, 0, st())
        else:
            import struct
            splits = _lib.lib().cdll.dfd_gemm_wgrad_splits(M, Nw, Kw)
            ws = torch.full((splits, Nw, Kw), float("nan"), device="cuda")
            again = torch.zeros(Nw, Kw, device="cuda")
            for dst in (dW, again):
                _lib.call(impl, P(G), P(X), P(dst), M, Nw, Kw, DT[dtype], P(ws), ws.numel() * 4, st())
                table = torch.frombuffer(bytearray(struct.pack("<QQqqii", P(ws), P(dst), Nw * Kw, Nw * Kw, splits, 0)), dtype=torch.uint8).cuda()
                _lib.call("dfd_ordered_reduce", P(table), 1, P(dst), min(1024, (Nw * Kw // 4 + 255) // 256), st())
                torch.cuda.synchronize()
            atomic = torch.zeros(Nw, Kw, device="cuda")
            _lib.call(impl, P(G), P(X), P(atomic), M, Nw, Kw, DT[dtype], None, 0, st())
            torch.cuda.synchronize()
            out["bitwise"] = bool(torch.equal(dW, again))
            out["vs_atomic"] = relerr(dW, atomic)
            out["splits"] = splits
    else:
        _lib.call(impl, P(G), P(X), P(dW), M, Nw, Kw, DT[dtype], st())
    torch.cuda.synchronize()
    ref = G.double().t() @ X.double()
    out["rel"] = relerr(dW, ref)
    return out


def _bn_params(C, g):
    scale = 1.0 + 0.2 * torch.randn(C, device="cuda", generator=g)
    shift = 0.3 * torch.randn(C, device="cuda", generator=g)
    return scale, shift


def check_dwconv(N, H, W, C, k, s, dtype=torch.bfloat16, affine=True, seed=0, fwd_impl="dfd_dwconv_fwd", add=True, stats=True):
    """fwd + dgrad (both modes) + wgrad against F.conv2d autograd on the rounded operands. add (mode 0 only): the residual
    gradient added to the input gradient, as in a DS block with a skip connection. stats=False: also the eval form of the
    forward (no statistics, no finalisation), which must store the same output bit for bit (`nostats_mismatch`)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    pad = (k - 1) // 2
    x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
    w = (torch.randn(C, 1, k, k, device="cuda", generator=g) * (1.0 / k)).contiguous()
    scale, shift = _bn_params(C, g)
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    out = torch.full((N, Ho, Wo, C), float("nan"), device="cuda", dtype=dtype)
    s1, s2 = stat_buf(C), stat_buf(C)
    act = 1 if affine else 0
    _lib.call(fwd_impl, P(x), P(scale) if affine else None, P(shift) if affine else None, P(w), P(out), N, H, W, C,
              k, s, act, DT[dtype], P(s1), P(s2), None, st())
    torch.cuda.synchronize()
    nostats = {}
    if not stats:
        out_e = torch.full_like(out, float("nan"))
        _lib.call(fwd_impl, P(x), P(scale) if affine else None, P(shift) if affine else None, P(w), P(out_e), N, H, W, C,
                  k, s, act, DT[dtype], None, None, None, st())
        torch.cuda.synchronize()
        nostats["nostats_mismatch"] = int((out_e.view(torch.int16) != out.view(torch.int16)).sum())
        del out_e
    # reference (fp32, same rounding points: activated input rounded to `dtype`)
    xr = nchw(x.float()).requires_grad_(True)
    if affine:
        u = xr * scale.view(1, C, 1, 1) + shift.view(1, C, 1, 1)
        a = u * torch.sigmoid(u)
    else:
        a = xr
    a_q = a + (a.to(dtype).float() - a).detach()          # straight-through rounding (value rounded, gradient 1)
    wr = w.clone().requires_grad_(True)
    ref = F.conv2d(a_q, wr, stride=s, padding=pad, groups=C)
    res = dict(fwd_max=maxerr_scaled(nchw(out.float()), ref.detach()), fwd_rel=relerr(nchw(out.float()), ref.detach()),
               nan=int(torch.isnan(out.float()).sum()), **nostats)
    # Element-wise bound of the forward (fwd_ulp <= 1). The kernel's Swish is u * sigmoid_fast(u) with
    # sigmoid_fast = fmaf(tanh.approx(u/2), 0.5, 0.5) (common.cuh:97). tanh.approx.f32 has at most 2^-10.98 relative error and
    # |tanh| <= 1, so the sigmoid is off by < 2^-11 ABSOLUTE and the kernel's activation a' by e = |u| 2^-11 (relative to a this
    # is unbounded for negative u). Both a' and the reference's a are then rounded to the 16-bit type:
    # |rnd(a') - rnd(a)| <= e + ulp(max(|a|, |a'|)) <= e + ulp_in (|a| + e), with ulp_in the largest relative ulp (2^-7 bf16,
    # 2^-10 fp16). Summed over the taps, with the output half-ulp u_out (2^-8 bf16, 2^-11 fp16) and 2^-20 for both fp32
    # accumulations of <= 25 taps (and the reference's own fp32 Swish):
    #   |out - ref| <= u_out |ref| + (ulp_in + 2^-20) sum_taps |w a| + (1 + ulp_in) 2^-11 sum_taps |w u|
    # The scaled 2^-7 (|ref| + rms) bound does not follow from this arithmetic and fails once cancelling sums are sampled 10^8
    # times; a wrong tap, channel or tile is off by a whole |w a| term and fails this one.
    u_out, ulp_in = U_OUT[dtype], ULP_IN[dtype]
    with torch.no_grad():
        mag = F.conv2d(a_q.detach().abs(), w.abs(), stride=s, padding=pad, groups=C)
        bound = u_out * ref.detach().abs() + (ulp_in + 2.0 ** -20) * mag
        if affine:
            bound += (1 + ulp_in) * 2.0 ** -11 * F.conv2d(u.detach().abs(), w.abs(), stride=s, padding=pad, groups=C)
        res["fwd_ulp"] = float(((nchw(out.float()) - ref.detach()).abs() / (bound + 1e-30)).max())
        del mag, bound
        if not affine:      # a raw input is read as stored: no staging rounding, only the taps' fp32 sum and the store (fp64)
            x64, w64 = nchw(x.double()), w.double()
            ref64 = F.conv2d(x64, w64, stride=s, padding=pad, groups=C)
            mag64 = F.conv2d(x64.abs(), w64.abs(), stride=s, padding=pad, groups=C)
            res["fwd_ulp"], res["fwd_ulp_bf16trip"] = ratio_pair(nchw(out), ref64, elem_bound(ref64, dtype, acc_term(mag64, k * k)))
            del x64, ref64, mag64
    of = out.double()
    res["sum_rel"] = relerr(s1.sum(0), of.sum((0, 1, 2)))
    res["sq_rel"] = relerr(s2.sum(0), (of * of).sum((0, 1, 2)))
    # backward: gy is the gradient w.r.t. the BN output behind the conv; dy = cA*gy + cB*yout + cC
    gy = (torch.randn(N, Ho, Wo, C, device="cuda", generator=g) * 0.1).to(dtype)
    cA = 1.0 + 0.1 * torch.randn(C, device="cuda", generator=g)
    cB = 0.05 * torch.randn(C, device="cuda", generator=g)
    cC = 0.01 * torch.randn(C, device="cuda", generator=g)
    dy = (cA * gy.float() + cB * out.float() + cC).to(dtype).float()
    ref.backward(nchw(dy))
    # the input gradient's element-wise bound (dgrad_ulp <= 1) in fp64 on the dy tile exactly as the kernel stages it
    ga64, mag64 = dw_input_grad64(staged_dy(gy, out, cA, cB, cC, dtype), w, H, W, k, s, (pad, pad, pad, pad))
    dW = torch.zeros_like(w)
    _lib.call("dfd_dwconv_wgrad", P(x), P(scale) if affine else None, P(shift) if affine else None, P(gy), P(out), P(cA), P(cB),
              P(cC), P(dW), N, H, W, C, k, s, DT[dtype], st())
    torch.cuda.synchronize()
    res["wgrad_rel"] = relerr(dW, wr.grad)
    gx = torch.full((N, H, W, C), float("nan"), device="cuda", dtype=dtype)
    if affine:
        mean = 0.1 * torch.randn(C, device="cuda", generator=g)
        rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
        b1, b2 = stat_buf(C), stat_buf(C)
        _lib.call("dfd_dwconv_dgrad", P(gy), P(out), P(cA), P(cB), P(cC), P(w), P(x), P(scale), P(shift), P(mean), P(rstd), None,
                  P(gx), N, H, W, C, k, s, 1, DT[dtype], P(b1), P(b2), st())
        torch.cuda.synchronize()
        # xr.grad is d/dx of the whole chain = scale * (dgrad * swish'(u)); the kernel emits gu = dgrad*swish'(u)
        gu_ref = xr.grad / scale.view(1, C, 1, 1)
        res["dgrad_max"] = maxerr_scaled(nchw(gx.float()), gu_ref)
        res["dgrad_rel"] = relerr(nchw(gx.float()), gu_ref)
        res["dgrad_ulp"], res["dgrad_ulp_bf16trip"] = dw_dgrad_bound(gx, ga64, mag64, k, dtype, u=_u32(x, scale, shift).double())
        gxd = gx.double()
        xhat = (x.double() - mean.double()) * rstd.double()
        res["bs1_rel"] = relerr(b1.sum(0), gxd.sum((0, 1, 2)))
        res["bs2_rel"] = relerr(b2.sum(0), (gxd * xhat).sum((0, 1, 2)))
        # the fused pass (dgrad mode 1 + wgrad over one staged dy tile) must reproduce both
        gx2 = torch.full((N, H, W, C), float("nan"), device="cuda", dtype=dtype)
        dW2 = torch.zeros_like(w)
        c1, c2 = stat_buf(C), stat_buf(C)
        _lib.call("dfd_dwconv_bwd", P(gy), P(out), P(cA), P(cB), P(cC), P(w), P(x), P(scale), P(shift), P(mean), P(rstd), None,
                  P(gx2), P(dW2), N, H, W, C, k, s, DT[dtype], P(c1), P(c2), None, 0, None, st())
        torch.cuda.synchronize()
        res["fused_gx_diff"] = float((gx2.float() - gx.float()).abs().max())
        res["fused_nan"] = int(torch.isnan(gx2.float()).sum())
        res["fused_wgrad_rel"] = relerr(dW2, wr.grad)
        res["fused_bs1_rel"] = relerr(c1.sum(0), gxd.sum((0, 1, 2)))
        res["fused_bs2_rel"] = relerr(c2.sum(0), (gxd * xhat).sum((0, 1, 2)))
        det = _dwconv_bwd_det(lambda t, ws, nbytes, gxo, d1, d2: _lib.call(
            "dfd_dwconv_bwd", P(gy), P(out), P(cA), P(cB), P(cC), P(w), P(x), P(scale), P(shift), P(mean), P(rstd), None,
            P(gxo), P(t), N, H, W, C, k, s, DT[dtype], P(d1), P(d2), P(ws), nbytes, None, st()), w, dW2, gx, N, H, W, C, k, s, True)
        stats = det.pop("stats")
        res["det_bs1_rel"] = max(relerr(d1.sum(0), gxd.sum((0, 1, 2))) for d1, _ in stats)
        res["det_bs2_rel"] = max(relerr(d2.sum(0), (gxd * xhat).sum((0, 1, 2))) for _, d2 in stats)
        res.update(det)
    else:
        addt = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype) if add else None
        _lib.call("dfd_dwconv_dgrad", P(gy), P(out), P(cA), P(cB), P(cC), P(w), None, None, None, None, None, P(addt), P(gx), N, H,
                  W, C, k, s, 0, DT[dtype], None, None, st())
        torch.cuda.synchronize()
        ref_gx = xr.grad + nchw(addt.float()) if add else xr.grad
        res["dgrad_max"] = maxerr_scaled(nchw(gx.float()), ref_gx)
        res["dgrad_rel"] = relerr(nchw(gx.float()), ref_gx)
        res["dgrad_ulp"], res["dgrad_ulp_bf16trip"] = dw_dgrad_bound(gx, ga64, mag64, k, dtype, add=addt)
        # fused pass, mode 0 (input consumed as is, residual gradient added when given)
        gx2 = torch.full((N, H, W, C), float("nan"), device="cuda", dtype=dtype)
        dW2 = torch.zeros_like(w)
        _lib.call("dfd_dwconv_bwd", P(gy), P(out), P(cA), P(cB), P(cC), P(w), P(x), None, None, None, None, P(addt), P(gx2), P(dW2),
                  N, H, W, C, k, s, DT[dtype], None, None, None, 0, None, st())
        torch.cuda.synchronize()
        res["fused_gx_diff"] = float((gx2.float() - gx.float()).abs().max())
        res["fused_nan"] = int(torch.isnan(gx2.float()).sum())
        res["fused_wgrad_rel"] = relerr(dW2, wr.grad)
        det = _dwconv_bwd_det(lambda t, ws, nbytes, gxo, d1, d2: _lib.call(
            "dfd_dwconv_bwd", P(gy), P(out), P(cA), P(cB), P(cC), P(w), P(x), None, None, None, None, P(addt), P(gxo), P(t),
            N, H, W, C, k, s, DT[dtype], None, None, P(ws), nbytes, None, st()), w, dW2, gx, N, H, W, C, k, s, False)
        det.pop("stats")
        res.update(det)
    res["nan_b"] = int(torch.isnan(gx.float()).sum())
    return res


def _dwconv_bwd_det(launch, w, dW_atomic, gx_ref, N, H, W, C, k, s, with_stats):
    """order-deterministic mode of dfd_dwconv_bwd (partials in fixed workspace slots + dfd_ordered_reduce, as the training plan
    runs it), launched twice, each into its own NaN-filled input gradient: the weight gradients agree bit for bit, and with the
    atomic flush to fp32 round-off; the input gradient equals the two-pass dfd_dwconv_dgrad's (gx_ref) bit for bit, with every
    element written; also the workspace size in bytes, and (with_stats) each run's BatchNorm backward sums"""
    import struct
    parts = _lib.lib().cdll.dfd_dwconv_bwd_parts(N, H, W, C, k, s)
    cw = _lib.lib().cdll.dfd_dwconv_block_channels(C)
    cbs = (C + cw - 1) // cw
    ws = torch.full((cbs, parts, cw * k * k), float("nan"), device="cuda")
    dW3 = [torch.zeros_like(w), torch.zeros_like(w)]
    gx_diff, gx_nan, stats = 0.0, 0, []
    for t in dW3:
        gxo = torch.full_like(gx_ref, float("nan"))
        d1, d2 = (stat_buf(C), stat_buf(C)) if with_stats else (None, None)
        launch(t, ws, ws.numel() * 4, gxo, d1, d2)
        stats.append((d1, d2))
        raw = b"".join(struct.pack("<QQqqii", P(ws) + cb * parts * cw * k * k * 4, P(t) + cb * cw * k * k * 4,
                                   min(cw, C - cw * cb) * k * k, cw * k * k, parts, 0) for cb in range(cbs))
        table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
        _lib.call("dfd_ordered_reduce", P(table), cbs, P(t), (cw * k * k // 4 + 7) // 8 if parts > 64 else 1, st())
        torch.cuda.synchronize()
        gx_nan += int(torch.isnan(gxo.float()).sum())
        gx_diff = max(gx_diff, float((gxo.float() - gx_ref.float()).abs().max()))
        del gxo
    return dict(det_bitwise=bool(torch.equal(dW3[0], dW3[1])), det_vs_atomic=relerr(dW3[0], dW_atomic), ws_bytes=ws.numel() * 4,
                det_gx_diff=gx_diff, det_nan=gx_nan, stats=stats)


def check_stem_gemm(N, Cin, H, W, Cout, k, s, pad, dtype=torch.bfloat16, seed=0, pack=1):
    """the stem as the training plan runs it: dfd_stem_im2col -> dfd_pad_weight -> the tensor-core GEMM with
    the BatchNorm statistics (pack 1: dfd_gemm_tn; else dfd_gemm_tn_rowpack on the block-diagonal copy of the padded weight,
    the plan's form for small Kp) -> order-deterministic dfd_gemm_wgrad into the Kp-padded gradient -> dfd_unpad_grad. im2col
    exact against F.unfold; output and weight gradient against fp64 products of the same rounded operands."""
    import struct
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g).to(dtype)
    taps = Cin * k * k
    Kp = (taps + 7) // 8 * 8
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    M = N * Ho * Wo
    w = (torch.randn(Cout, taps, device="cuda", generator=g) / math.sqrt(taps)).to(dtype)
    wpad = torch.full((Cout, Kp), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_pad_weight", P(w), P(wpad), Cout, taps, Kp, d, st())
    cols = torch.full((M, Kp), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_stem_im2col", P(x), P(cols), N, Cin, H, W, k, s, pad, Kp, d, st())
    y = torch.full((M, Cout), float("nan"), device="cuda", dtype=dtype)
    s1, s2 = stat_buf(Cout), stat_buf(Cout)
    if pack == 1:
        _lib.call("dfd_gemm_tn", P(cols), P(wpad), P(y), M, Cout, Kp, d, P(s1), P(s2), None, st())
    else:
        Bd = torch.full((pack * Cout, pack * Kp), float("nan"), device="cuda", dtype=dtype)
        table = torch.frombuffer(bytearray(struct.pack("<QQiiii", P(wpad), P(Bd), Cout, Kp, pack, 0)), dtype=torch.uint8).cuda()
        _lib.call("dfd_blockdiag_weights", P(table), 1, d, st())
        _lib.call("dfd_gemm_tn_rowpack", P(cols), P(Bd), P(y), M, Cout, Kp, pack, d, P(s1), P(s2), None, st())
    torch.cuda.synchronize()
    res = dict(wpad_diff=float((wpad[:, :taps].float() - w.float()).abs().max()), wpad_tail=float(wpad[:, taps:].float().abs().max()) if Kp > taps else 0.0,
               cols_nan=int(torch.isnan(cols).sum()), cols_tail=float(cols[:, taps:].float().abs().max()) if Kp > taps else 0.0)
    # im2col, exact; chunked over images so that the fp32 unfold stays small
    diff = 0.0
    per = max(1, (64 << 20) // (taps * Ho * Wo))
    for n0 in range(0, N, per):
        n1 = min(N, n0 + per)
        ref = F.unfold(x[n0:n1].float(), k, padding=pad, stride=s).transpose(1, 2).reshape(-1, taps)
        diff = max(diff, float((cols[n0 * Ho * Wo:n1 * Ho * Wo, :taps].float() - ref).abs().max()))
        del ref
    res["cols_diff"] = diff
    ref_y = cols[:, :taps].double() @ w.double().t()
    res.update(fwd_max=maxerr_scaled(y.float(), ref_y), nan=int(torch.isnan(y).sum()))
    del ref_y
    yd = y.double()
    res["sum_rel"] = relerr(s1.sum(0), yd.sum(0))
    res["sq_rel"] = relerr(s2.sum(0), (yd * yd).sum(0))
    del yd
    gy = (torch.randn(M, Cout, device="cuda", generator=g) * 0.1).to(dtype)
    splits = _lib.lib().cdll.dfd_gemm_wgrad_splits(M, Cout, Kp)
    ws = torch.full((splits, Cout, Kp), float("nan"), device="cuda")
    gws = []
    base = torch.randn(Cout, taps, device="cuda", generator=g)        # dfd_unpad_grad accumulates into the gradient arena
    for _ in range(2):
        gpad = torch.zeros(Cout, Kp, device="cuda")
        gw = base.clone()
        _lib.call("dfd_gemm_wgrad", P(gy), P(cols), P(gpad), M, Cout, Kp, d, P(ws), ws.numel() * 4, st())
        table = torch.frombuffer(bytearray(struct.pack("<QQqqii", P(ws), P(gpad), Cout * Kp, Cout * Kp, splits, 0)), dtype=torch.uint8).cuda()
        _lib.call("dfd_ordered_reduce", P(table), 1, P(gpad), min(1024, (Cout * Kp // 4 + 255) // 256), st())
        _lib.call("dfd_unpad_grad", P(gpad), P(gw), Cout, taps, Kp, st())
        torch.cuda.synchronize()
        gws.append(gw)
    res["wgrad_rel"] = relerr(gws[0].double() - base.double(), gy.double().t() @ cols[:, :taps].double())
    res["wgrad_bitwise"] = bool(torch.equal(gws[0], gws[1]))
    res["wgrad_nan"] = int(torch.isnan(gws[0]).sum())
    res["splits"] = splits
    return res


def check_stem_im2col(N, Cin, H, W, k, s, pad, dtype=torch.bfloat16, seed=0):
    """im2col rows of the NCHW image in (ci, kh, kw) order, K zero-padded to a multiple of 8: exact against F.unfold"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g).to(dtype)
    taps = Cin * k * k
    Kp = (taps + 7) // 8 * 8
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    cols = torch.full((N * Ho * Wo, Kp), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_stem_im2col", P(x), P(cols), N, Cin, H, W, k, s, pad, Kp, DT[dtype], st())
    torch.cuda.synchronize()
    ref = F.unfold(x.float(), k, padding=pad, stride=s).transpose(1, 2).reshape(N * Ho * Wo, taps)
    return dict(diff=float((cols[:, :taps].float() - ref).abs().max()), pad_max=float(cols[:, taps:].float().abs().max()) if Kp > taps else 0.0,
                nan=int(torch.isnan(cols.float()).sum()))


def check_bn_chain(N, HW, C, dtype=torch.bfloat16, seed=0):
    """colstats -> bn_finalize -> bn_act(+gate,+res) / pool, then act_bwd -> bn_bwd_finalize -> bn_bwd_apply,
    against torch.nn.functional.batch_norm + swish autograd (train mode, running-stat EMA included)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = (torch.randn(N, HW, C, device="cuda", generator=g) * 1.5 + 0.3).to(dtype)
    gamma = 1.0 + 0.1 * torch.randn(C, device="cuda", generator=g)
    beta = 0.1 * torch.randn(C, device="cuda", generator=g)
    rm = 0.05 * torch.randn(C, device="cuda", generator=g)
    rv = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
    rm_ref, rv_ref = rm.clone(), rv.clone()
    nbt = torch.zeros(1, dtype=torch.int64, device="cuda")
    s1, s2 = stat_buf(C), stat_buf(C)
    scale, shift, mean, rstd = (torch.zeros(C, device="cuda") for _ in range(4))
    d = DT[dtype]
    _lib.call("dfd_colstats", P(y), N, HW, C, d, P(s1), P(s2), st())
    _lib.call("dfd_bn_finalize", P(s1), P(s2), float(N * HW), P(gamma), P(beta), P(rm), P(rv), P(nbt), 0.1, 1e-5, 1, C, P(scale),
              P(shift), P(mean), P(rstd), st())
    gate = torch.sigmoid(torch.randn(N, C, device="cuda", generator=g))
    a2 = torch.full((N, HW, C), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_bn_act", P(y), P(scale), P(shift), P(gate), None, P(a2), N, HW, C, 1, 0, d, st())
    res_t = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype)
    o_res = torch.full((N, HW, C), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_bn_act", P(y), P(scale), P(shift), None, P(res_t), P(o_res), N, HW, C, 0, 1, d, st())
    pooled = torch.zeros(N, C, device="cuda")
    _lib.call("dfd_pool", P(y), P(scale), P(shift), P(pooled), N, HW, C, 1, d, None, 0, st())
    # chunked variant (several CTAs per image, partial sums added in a fixed order): same means, bit-reproducible
    pooled_c = [torch.full((N, C), float("nan"), device="cuda") for _ in range(2)]
    partial = torch.full((8 * N * C,), float("nan"), device="cuda")
    for pc in pooled_c:
        _lib.call("dfd_pool", P(y), P(scale), P(shift), P(pc), N, HW, C, 1, d, P(partial), 8, st())
    torch.cuda.synchronize()
    # reference
    yr = y.float().permute(0, 2, 1).reshape(N, C, HW, 1).requires_grad_(True)
    gr = gamma.clone().requires_grad_(True)
    br = beta.clone().requires_grad_(True)
    u = F.batch_norm(yr, rm_ref, rv_ref, gr, br, True, 0.1, 1e-5)
    sw = u * torch.sigmoid(u)
    res = dict(
        rm_rel=relerr(rm, rm_ref), rv_rel=relerr(rv, rv_ref), nbt=int(nbt.item()),
        gate_max=maxerr_scaled(a2.float().permute(0, 2, 1), (sw.squeeze(-1) * gate.unsqueeze(-1)).detach()),
        res_max=maxerr_scaled(o_res.float().permute(0, 2, 1), (u.squeeze(-1) + res_t.float().permute(0, 2, 1)).detach()),
        pool_rel=relerr(pooled, sw.mean((2, 3)).detach()), pool_chunk_rel=relerr(pooled_c[0], sw.mean((2, 3)).detach()),
        pool_chunk_repro=float((pooled_c[0] - pooled_c[1]).abs().max()))
    # backward: gu = (da*gate + dpool/HW) * swish'(u); then BN backward
    da = (torch.randn(N, HW, C, device="cuda", generator=g) * 0.1).to(dtype)
    dpool = torch.randn(N, C, device="cuda", generator=g) * 0.1
    gu = torch.full((N, HW, C), float("nan"), device="cuda", dtype=dtype)
    b1, b2 = stat_buf(C), stat_buf(C)
    _lib.call("dfd_act_bwd", P(da), P(y), P(scale), P(shift), P(mean), P(rstd), P(gate), P(dpool), P(gu), N, HW, C, 1, d, P(b1), P(b2), None, st())
    dgamma, dbeta, cA, cB, cC = (torch.zeros(C, device="cuda") for _ in range(5))
    _lib.call("dfd_bn_bwd_finalize", P(b1), P(b2), float(N * HW), P(gamma), P(mean), P(rstd), P(dgamma), P(dbeta), P(cA), P(cB), P(cC), C, st())
    dy = torch.full((N, HW, C), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_bn_bwd_apply", P(gu), P(y), None, P(cA), P(cB), P(cC), P(dy), N, HW, C, d, st())
    # also the two-pass reduce variant used for un-activated BN outputs
    c1, c2 = stat_buf(C), stat_buf(C)
    _lib.call("dfd_bn_bwd_reduce", P(da), P(y), None, P(mean), P(rstd), N, HW, C, d, P(c1), P(c2), None, st())
    draw = torch.zeros(N, C, device="cuda")
    _lib.call("dfd_se_bwd_reduce", P(da), P(y), P(scale), P(shift), P(draw), N, HW, C, d, st())
    torch.cuda.synchronize()
    loss = (sw * gate.view(N, C, 1, 1) * da.float().permute(0, 2, 1).unsqueeze(-1)).sum() + (sw.mean((2, 3)) * dpool).sum()
    loss.backward()
    res["dy_max"] = maxerr_scaled(dy.float().permute(0, 2, 1), yr.grad.squeeze(-1))
    res["dy_rel"] = relerr(dy.float().permute(0, 2, 1), yr.grad.squeeze(-1))
    res["dgamma_rel"] = relerr(dgamma, gr.grad)
    res["dbeta_rel"] = relerr(dbeta, br.grad)
    xhat = (y.double() - mean.double()) * rstd.double()
    res["reduce1_rel"] = relerr(c1.sum(0), da.double().sum((0, 1)))
    res["reduce2_rel"] = relerr(c2.sum(0), (da.double() * xhat).sum((0, 1)))
    res["draw_rel"] = relerr(draw, (da.float().permute(0, 2, 1) * sw.squeeze(-1).detach()).sum(2))
    res["nan"] = int(torch.isnan(dy.float()).sum() + torch.isnan(a2.float()).sum())
    return res


ROW_KERNELS = ("dfd_bn_act", "dfd_act_bwd", "dfd_pool", "dfd_bn_bwd_reduce", "dfd_bn_bwd_apply", "dfd_se_bwd_reduce")


def _act_ref(u, act):
    """act(u) and act'(u) in fp64 (DFD_ACT_NONE / SWISH / RELU)"""
    if act == 1:
        s = torch.sigmoid(u)
        return u * s, s * (1 + u * (1 - s))
    if act == 2:
        return u.clamp_min(0), (u > 0).double()
    return u, torch.ones_like(u)


def check_row_kernel(kernel, N, HW, C, args, ptrs, dtype=torch.bfloat16, seed=0):
    """One launch of a per-row BatchNorm / activation / pool / SE kernel exactly as a plan issues it: `args` are its non-pointer
    arguments after (n, hw, C) with the dtype left out, `ptrs` its pointer-presence mask ('p' / '0' per pointer argument, ABI
    order; see tests/plan_launches.py), so the activation, residual mode and optional operands select the same instantiation.
    Reference: fp64 on the same rounded operands, with u = scale*y + shift rounded to fp32 once (the kernel's fmaf)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    has = lambda i: ptrs[i] == "p"
    y = (torch.randn(N, HW, C, device="cuda", generator=g) * 1.5 + 0.3).to(dtype)
    scale, shift = _bn_params(C, g)
    mean = 0.1 * torch.randn(C, device="cuda", generator=g)
    rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
    gate = torch.sigmoid(torch.randn(N, C, device="cuda", generator=g))
    yd = y.double()
    xhat = (yd - mean.double()) * rstd.double()
    res = {}

    def u_of(with_scale):
        return (yd * scale.double() + shift.double()).float().double() if with_scale else yd

    def sums(v):
        return v.sum((0, 1)), (v * xhat).sum((0, 1))

    if kernel == "dfd_bn_act":
        act, res_mode = args[0], args[1]
        r = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype) if has(4) else None
        out = torch.full_like(y, float("nan"))
        _lib.call(kernel, P(y), P(scale) if has(1) else None, P(shift) if has(2) else None, P(gate) if has(3) else None,
                  P(r), P(out), N, HW, C, act, res_mode, d, st())
        torch.cuda.synchronize()
        u = u_of(has(1))
        gt = gate.double().unsqueeze(1) if has(3) else torch.ones((), dtype=torch.float64, device="cuda")
        ref, bound = bn_act_bound(u, act, gt, r if res_mode else None, res_mode, dtype)
        res.update(out_max=maxerr_scaled(out.float(), ref), nan=int(torch.isnan(out.float()).sum()))
        res["out_ulp"], res["out_ulp_bf16trip"] = ratio_pair(out, ref, bound)
    elif kernel == "dfd_act_bwd":
        act = args[0]
        da = (torch.randn(N, HW, C, device="cuda", generator=g) * 0.1).to(dtype) if has(0) else None
        dpool = torch.randn(N, C, device="cuda", generator=g) * 0.1 if has(7) else None
        gu = torch.full_like(y, float("nan"))
        s1, s2 = (stat_buf(C), stat_buf(C)) if has(9) else (None, None)
        _lib.call(kernel, P(da), P(y), P(scale), P(shift), P(mean), P(rstd), P(gate) if has(6) else None, P(dpool), P(gu), N, HW, C,
                  act, d, P(s1), P(s2), None, st())
        torch.cuda.synchronize()
        gin = torch.zeros_like(yd)
        if has(0):
            gin = da.double() * (gate.double().unsqueeze(1) if has(6) else 1.0)
        if has(7):
            gin = gin + dpool.double().unsqueeze(1) / HW
        gmag = gin.abs() if not has(7) else (gin - dpool.double().unsqueeze(1) / HW).abs() + dpool.double().abs().unsqueeze(1) / HW
        ref, bound = act_bwd_bound(u_of(True), act, gin, gmag, dtype)
        res.update(out_max=maxerr_scaled(gu.float(), ref), nan=int(torch.isnan(gu.float()).sum()))
        res["out_ulp"], res["out_ulp_bf16trip"] = ratio_pair(gu, ref, bound)
        if has(9):      # the BatchNorm backward sums of the STORED gradient
            r1, r2 = sums(gu.double())
            res.update(s1_rel=relerr(s1.sum(0), r1), s2_rel=relerr(s2.sum(0), r2))
    elif kernel == "dfd_pool":
        act, chunks = args[0], args[1]
        pooled = [torch.full((N, C), float("nan"), device="cuda") for _ in range(2)]
        for t in pooled:
            _lib.call(kernel, P(y), P(scale) if has(1) else None, P(shift) if has(2) else None, P(t), N, HW, C, act, d, None, chunks, st())
        torch.cuda.synchronize()
        ref = _act_ref(u_of(has(1)), act)[0].mean(1)
        res.update(pool_rel=relerr(pooled[0], ref), repro=bool(torch.equal(pooled[0], pooled[1])), nan=int(torch.isnan(pooled[0]).sum()))
    elif kernel == "dfd_bn_bwd_reduce":
        gr = (torch.randn(N, HW, C, device="cuda", generator=g) * 0.1).to(dtype)
        out = torch.relu(torch.randn(N, HW, C, device="cuda", generator=g)).to(dtype) if has(2) else None
        s1, s2 = stat_buf(C), stat_buf(C)
        _lib.call(kernel, P(gr), P(y), P(out), P(mean), P(rstd), N, HW, C, d, P(s1), P(s2), None, st())
        torch.cuda.synchronize()
        gm = gr.double() * ((out.double() > 0).double() if has(2) else 1.0)
        r1, r2 = sums(gm)
        res.update(s1_rel=relerr(s1.sum(0), r1), s2_rel=relerr(s2.sum(0), r2), nan=0)
    elif kernel == "dfd_bn_bwd_apply":
        gr = (torch.randn(N, HW, C, device="cuda", generator=g) * 0.1).to(dtype)
        out = torch.relu(torch.randn(N, HW, C, device="cuda", generator=g)).to(dtype) if has(2) else None
        cA = 1.0 + 0.1 * torch.randn(C, device="cuda", generator=g)
        cB = 0.05 * torch.randn(C, device="cuda", generator=g)
        cC = 0.01 * torch.randn(C, device="cuda", generator=g)
        dy = torch.full_like(y, float("nan"))
        _lib.call(kernel, P(gr), P(y), P(out), P(cA), P(cB), P(cC), P(dy), N, HW, C, d, st())
        torch.cuda.synchronize()
        gm = gr.double() * ((out.double() > 0).double() if has(2) else 1.0)
        ref = cA.double() * gm + cB.double() * yd + cC.double()
        res.update(out_max=maxerr_scaled(dy.float(), ref), nan=int(torch.isnan(dy.float()).sum()))
        # bn_bwd_apply_kernel (bn_act.cu:606): two fp32 fmaf's, one 16-bit store
        mag = (cA.double() * gm).abs() + (cB.double() * yd).abs() + cC.double().abs()
        res["out_ulp"], res["out_ulp_bf16trip"] = ratio_pair(dy, ref, elem_bound(ref, dtype, acc_term(mag, 2)))
    elif kernel == "dfd_se_bwd_reduce":
        da = (torch.randn(N, HW, C, device="cuda", generator=g) * 0.1).to(dtype)
        draw = torch.full((N, C), float("nan"), device="cuda")
        _lib.call(kernel, P(da), P(y), P(scale), P(shift), P(draw), N, HW, C, d, st())
        torch.cuda.synchronize()
        ref = (da.double() * _act_ref(u_of(True), 1)[0]).sum(1)
        res.update(draw_rel=relerr(draw, ref), nan=int(torch.isnan(draw).sum()))
    else:
        raise KeyError(kernel)
    return res


def check_se_fc(N, C, Cse, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    pooled = torch.randn(N, C, device="cuda", generator=g)
    Wr = (torch.randn(Cse, C, device="cuda", generator=g) / math.sqrt(C)).requires_grad_(True)
    br = (0.1 * torch.randn(Cse, device="cuda", generator=g)).requires_grad_(True)
    We = (torch.randn(C, Cse, device="cuda", generator=g) / math.sqrt(Cse)).requires_grad_(True)
    be = (0.1 * torch.randn(C, device="cuda", generator=g)).requires_grad_(True)
    gate = torch.zeros(N, C, device="cuda")
    _lib.call("dfd_se_fc_fwd", P(pooled), P(Wr), P(br), P(We), P(be), P(gate), N, C, Cse, st())
    pr = pooled.clone().requires_grad_(True)
    r = F.linear(pr, Wr, br)
    r = r * torch.sigmoid(r)
    ref = torch.sigmoid(F.linear(r, We, be))
    draw = torch.randn(N, C, device="cuda", generator=g)
    ref.backward(draw)
    d_e, dpool = torch.zeros(N, C, device="cuda"), torch.zeros(N, C, device="cuda")
    rr, drp = torch.zeros(N, Cse, device="cuda"), torch.zeros(N, Cse, device="cuda")
    dWr, dbr, dWe, dbe = torch.zeros_like(Wr), torch.zeros_like(br), torch.zeros_like(We), torch.zeros_like(be)
    _lib.call("dfd_se_fc_bwd", P(draw), P(pooled), P(Wr), P(br), P(We), P(be), P(d_e), P(rr), P(drp), P(dpool), P(dWr), P(dbr), P(dWe),
              P(dbe), N, C, Cse, st())
    torch.cuda.synchronize()
    return dict(gate_rel=relerr(gate, ref.detach()), dpool_rel=relerr(dpool, pr.grad), dWr_rel=relerr(dWr, Wr.grad),
                dbr_rel=relerr(dbr, br.grad), dWe_rel=relerr(dWe, We.grad), dbe_rel=relerr(dbe, be.grad))


def _fin_desc(s1, s2, gamma, beta, rm, rv, nbt, scale, shift, mean, rstd, ticket, count, C, momentum=0.1, eps=1e-5):
    """BnFinDesc (csrc/bn_finalize.cuh) on the device"""
    import struct
    raw = struct.pack("<12Qddffii", P(s1), P(s2), P(gamma), P(beta), P(rm), P(rv), P(nbt), P(scale), P(shift), P(mean), P(rstd),
                      P(ticket), 1.0 / count, count / (count - 1.0), momentum, eps, C, 0)
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()


def _bfin_desc(s1, s2, gamma, mean, rstd, dgamma, dbeta, cA, cB, cC, ticket, count, C):
    import struct
    raw = struct.pack("<11Qdii", P(s1), P(s2), P(gamma), P(mean), P(rstd), P(dgamma), P(dbeta), P(cA), P(cB), P(cC), P(ticket),
                      1.0 / count, C, 0)
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()


def check_fused_finalize(kind, dtype=torch.bfloat16, seed=0):
    """The BatchNorm finalisation done by the LAST CTA of the kernel that produced the statistics == the standalone
    dfd_bn_finalize / dfd_bn_bwd_finalize launch on the same statistics (bit for bit: same device function, same fp64 sums up to
    the order of the slot atomics), twice in a row (the ticket returns to zero), running statistics included."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = DT[dtype]
    out = {}
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")

    def vecs(C, n):
        return [torch.zeros(C, device="cuda") for _ in range(n)]

    if kind in ("gemm", "gemm_rowpack", "dwconv_fwd"):
        if kind == "dwconv_fwd":
            N, H, W, C, k, s_ = 3, 19, 17, 96, 3, 1
            x = torch.randn(N, H, W, C, device="cuda", generator=g).to(dtype)
            w = (torch.randn(C, 1, k, k, device="cuda", generator=g) / k).contiguous()
            sc, sh = _bn_params(C, g)
            y = torch.empty(N, H, W, C, device="cuda", dtype=dtype)
            count = N * H * W
            launch = lambda a, b, fin: _lib.call("dfd_dwconv_fwd", P(x), P(sc), P(sh), P(w), P(y), N, H, W, C, k, s_, 1, d, P(a), P(b), fin, st())
        else:
            M, K, C = 5000, 32 if kind == "gemm_rowpack" else 144, 96
            A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
            B = (torch.randn(C, K, device="cuda", generator=g) / math.sqrt(K)).to(dtype)
            y = torch.empty(M, C, device="cuda", dtype=dtype)
            count = M
            if kind == "gemm":
                launch = lambda a, b, fin: _lib.call("dfd_gemm_tn", P(A), P(B), P(y), M, C, K, d, P(a), P(b), fin, st())
            else:
                import struct
                pack = 4
                Bd = torch.zeros(pack * C, pack * K, device="cuda", dtype=dtype)
                table = torch.frombuffer(bytearray(struct.pack("<QQiiii", P(B), P(Bd), C, K, pack, 0)), dtype=torch.uint8).cuda()
                _lib.call("dfd_blockdiag_weights", P(table), 1, d, st())
                launch = lambda a, b, fin: _lib.call("dfd_gemm_tn_rowpack", P(A), P(Bd), P(y), M, C, K, pack, d, P(a), P(b), fin, st())
        gamma = 1.0 + 0.1 * torch.randn(C, device="cuda", generator=g)
        beta = 0.1 * torch.randn(C, device="cuda", generator=g)
        res = []
        for fused in (True, False):
            rm, rv = torch.full((C,), 0.05, device="cuda"), torch.full((C,), 1.1, device="cuda")
            nbt = torch.zeros(1, dtype=torch.int64, device="cuda")
            o = vecs(C, 4)
            for rep in range(2):
                s1, s2 = stat_buf(C), stat_buf(C)
                if fused:
                    desc = _fin_desc(s1, s2, gamma, beta, rm, rv, nbt, *o, ticket, float(count), C)
                    launch(s1, s2, P(desc))
                else:
                    launch(s1, s2, None)
                    _lib.call("dfd_bn_finalize", P(s1), P(s2), float(count), P(gamma), P(beta), P(rm), P(rv), P(nbt), 0.1, 1e-5, 1, C,
                              P(o[0]), P(o[1]), P(o[2]), P(o[3]), st())
                torch.cuda.synchronize()
            res.append([t.clone() for t in o] + [rm, rv, nbt.float()])
        out["max_diff"] = max(float((a - b).abs().max() / (b.abs().max() + 1e-30)) for a, b in zip(res[0], res[1]))
        out["nbt"] = int(res[0][6])
    else:
        N, HW, C = 3, 77, 144
        y = (torch.randn(N, HW, C, device="cuda", generator=g) * 1.5).to(dtype)
        da = (0.1 * torch.randn(N, HW, C, device="cuda", generator=g)).to(dtype)
        sc, sh = _bn_params(C, g)
        mean = 0.1 * torch.randn(C, device="cuda", generator=g)
        rstd = 1.0 + 0.1 * torch.rand(C, device="cuda", generator=g)
        gamma = 1.0 + 0.1 * torch.randn(C, device="cuda", generator=g)
        gu = torch.empty(N, HW, C, device="cuda", dtype=dtype)
        count = N * HW
        if kind == "act_bwd":
            launch = lambda a, b, fin: _lib.call("dfd_act_bwd", P(da), P(y), P(sc), P(sh), P(mean), P(rstd), None, None, P(gu), N, HW, C, 1, d,
                                                 P(a), P(b), fin, st())
        elif kind == "bn_bwd_reduce":
            launch = lambda a, b, fin: _lib.call("dfd_bn_bwd_reduce", P(da), P(y), None, P(mean), P(rstd), N, HW, C, d, P(a), P(b), fin, st())
        else:       # dwconv_bwd (mode 1)
            Nn, H, W, k, s_ = 3, 14, 14, 5, 1
            C = 144
            x = torch.randn(Nn, H, W, C, device="cuda", generator=g).to(dtype)
            w = (torch.randn(C, 1, k, k, device="cuda", generator=g) / k).contiguous()
            gy = (0.1 * torch.randn(Nn, H, W, C, device="cuda", generator=g)).to(dtype)
            yo = torch.randn(Nn, H, W, C, device="cuda", generator=g).to(dtype)
            cv = [torch.rand(C, device="cuda", generator=g) + 0.5 for _ in range(3)]
            gx, dW = torch.empty_like(x), torch.zeros_like(w)
            count = Nn * H * W
            launch = lambda a, b, fin: _lib.call("dfd_dwconv_bwd", P(gy), P(yo), P(cv[0]), P(cv[1]), P(cv[2]), P(w), P(x), P(sc), P(sh),
                                                 P(mean), P(rstd), None, P(gx), P(dW), Nn, H, W, C, k, s_, d, P(a), P(b), None, 0, fin, st())
        res = []
        for fused in (True, False):
            o = vecs(C, 5)
            for rep in range(2):
                s1, s2 = stat_buf(C), stat_buf(C)
                if fused:
                    desc = _bfin_desc(s1, s2, gamma, mean, rstd, *o, ticket, float(count), C)
                    launch(s1, s2, P(desc))
                else:
                    launch(s1, s2, None)
                    _lib.call("dfd_bn_bwd_finalize", P(s1), P(s2), float(count), P(gamma), P(mean), P(rstd), P(o[0]), P(o[1]), P(o[2]),
                              P(o[3]), P(o[4]), C, st())
                torch.cuda.synchronize()
            res.append([t.clone() for t in o])
        out["max_diff"] = max(float((a - b).abs().max() / (b.abs().max() + 1e-30)) for a, b in zip(res[0], res[1]))
    out["ticket_at_rest"] = int(ticket) == 0
    return out


def check_se_fused(N, HW, C, Cse, dtype=torch.bfloat16, seed=0):
    """the one-launch forms (pool + excite gate; dL/dgate reduction + backward FC chain) against the separate kernels they
    replace, on an activation tensor: same pooled vector and gate bit for bit (identical arithmetic order), backward vectors to
    fp32 round-off (the cross-warp sum of d_r is partitioned by the CTA's warp count)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype)
    da = (0.1 * torch.randn(N, HW, C, device="cuda", generator=g)).to(dtype)
    scale, shift = _bn_params(C, g)
    Wr = torch.randn(Cse, C, device="cuda", generator=g) / math.sqrt(C)
    br = 0.1 * torch.randn(Cse, device="cuda", generator=g)
    We = torch.randn(C, Cse, device="cuda", generator=g) / math.sqrt(Cse)
    be = 0.1 * torch.randn(C, device="cuda", generator=g)
    d = DT[dtype]
    pooled_a, gate_a = torch.zeros(N, C, device="cuda"), torch.zeros(N, C, device="cuda")
    pooled_b, gate_b = torch.zeros(N, C, device="cuda"), torch.zeros(N, C, device="cuda")
    _lib.call("dfd_pool", P(y), P(scale), P(shift), P(pooled_a), N, HW, C, 1, d, None, 8, st())
    _lib.call("dfd_se_fc_fwd", P(pooled_a), P(Wr), P(br), P(We), P(be), P(gate_a), N, C, Cse, st())
    _lib.call("dfd_pool_se", P(y), P(scale), P(shift), P(pooled_b), P(Wr), P(br), P(We), P(be), P(gate_b), N, HW, C, Cse, 1, d, 8, st())
    torch.cuda.synchronize()
    ref_pool = (lambda u: u * torch.sigmoid(u))(y.float() * scale + shift).mean(1)
    out = dict(pool_equal=bool(torch.equal(pooled_a, pooled_b)), gate_equal=bool(torch.equal(gate_a, gate_b)),
               pool_rel=relerr(pooled_b, ref_pool))

    def zeros(*shape):
        return torch.zeros(*shape, device="cuda")

    va = dict(draw=zeros(N, C), d_e=zeros(N, C), r=zeros(N, Cse), drp=zeros(N, Cse), dpool=zeros(N, C),
              dWr=zeros(Cse, C), dbr=zeros(Cse), dWe=zeros(C, Cse), dbe=zeros(C))
    vb = {k: torch.zeros_like(v) for k, v in va.items()}
    _lib.call("dfd_se_bwd_reduce", P(da), P(y), P(scale), P(shift), P(va["draw"]), N, HW, C, d, st())
    _lib.call("dfd_se_fc_bwd", P(va["draw"]), P(pooled_a), P(Wr), P(br), P(We), P(be), P(va["d_e"]), P(va["r"]), P(va["drp"]),
              P(va["dpool"]), P(va["dWr"]), P(va["dbr"]), P(va["dWe"]), P(va["dbe"]), N, C, Cse, st())
    _lib.call("dfd_se_bwd_chain", P(da), P(y), P(scale), P(shift), P(vb["draw"]), P(pooled_a), P(Wr), P(br), P(We), P(be),
              P(vb["d_e"]), P(vb["r"]), P(vb["drp"]), P(vb["dpool"]), N, HW, C, Cse, d, st())
    _lib.call("dfd_se_fc_wgrad", P(vb["d_e"]), P(vb["r"]), P(vb["drp"]), P(pooled_a), P(vb["dWr"]), P(vb["dbr"]), P(vb["dWe"]),
              P(vb["dbe"]), N, C, Cse, st())
    torch.cuda.synchronize()
    out["draw_equal"] = bool(torch.equal(va["draw"], vb["draw"]))
    out["bwd_rel"] = max(relerr(vb[k], va[k]) for k in va)
    return out


def check_head(N, Fdim, smoothing=0.0, soft=False, seed=0, with_loss=True):
    """with_loss=False: the logits-only launch of Engine.head(False) (validate, test_img), with no target, loss, count or
    dlogits operand; only the logits are returned"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    pooled = torch.randn(N, Fdim, device="cuda", generator=g)
    W = (torch.randn(2, Fdim, device="cuda", generator=g) / math.sqrt(Fdim)).requires_grad_(True)
    b = (0.1 * torch.randn(2, device="cuda", generator=g)).requires_grad_(True)
    if not with_loss:
        logits = torch.full((N, 2), float("nan"), device="cuda")
        _lib.call("dfd_head_fwd", P(pooled), P(W), P(b), P(logits), N, Fdim, 2, None, None, 0.0, 1.0, None, None, None, None, st())
        torch.cuda.synchronize()
        ref = pooled.double() @ W.detach().double().t() + b.detach().double()
        return dict(logits_rel=relerr(logits, ref), nan=int(torch.isnan(logits).sum()))
    y = torch.randint(0, 2, (N,), device="cuda", generator=g)
    tf = torch.softmax(torch.randn(N, 2, device="cuda", generator=g), -1)
    logits = torch.zeros(N, 2, device="cuda")
    dlog = torch.zeros(N, 2, device="cuda")
    acc = torch.zeros(2, device="cuda")
    _lib.call("dfd_head_fwd", P(pooled), P(W), P(b), P(logits), N, Fdim, 2, None if soft else P(y), P(tf) if soft else None,
              smoothing, 1.0, None, P(acc), P(acc) + 4, P(dlog), st())
    pr = pooled.clone().requires_grad_(True)
    z = F.linear(pr, W, b)
    logp = F.log_softmax(z, -1)
    if soft:
        loss = torch.sum(-tf * logp, -1).mean()
        lab = tf.argmax(1)
    else:
        nll = -logp.gather(-1, y.unsqueeze(1)).squeeze(1)
        loss = ((1 - smoothing) * nll + smoothing * (-logp.mean(-1))).mean()
        lab = y
    z.retain_grad()
    loss.backward()
    dW, db, dpooled = torch.zeros_like(W), torch.zeros_like(b), torch.zeros(N, Fdim, device="cuda")
    _lib.call("dfd_head_bwd", P(dlog), P(pooled), P(W), P(dW), P(db), P(dpooled), N, Fdim, 2, st())
    torch.cuda.synchronize()
    correct = float((z.argmax(1) == lab).sum())
    return dict(logits_rel=relerr(logits, z.detach()), loss_rel=abs(float(acc[0]) - float(loss)) / abs(float(loss)),
                correct_diff=abs(float(acc[1]) - correct), dlogits_rel=relerr(dlog, z.grad), dW_rel=relerr(dW, W.grad),
                db_rel=relerr(db, b.grad), dpooled_rel=relerr(dpooled, pr.grad))


def _ulp32(x):
    """the fp32 ulp at each value of the fp64 tensor x (normal range)"""
    _, e = torch.frexp(x.abs())
    return torch.ldexp(torch.ones_like(x), e - 24)


def check_bn_finalize_eval(C, eps=1e-5, momentum=0.1, seed=0):
    """dfd_bn_finalize in eval form, as Engine.launch_args issues it (training = 0, no batch sums): the folded BatchNorm from
    the running statistics against fp64. Returns the errors in fp32 ulps of the fp64 values: rstd of 1/sqrt(rv + eps) (eps as
    the fp32 argument the kernel receives), scale of gamma * rstd, and shift over ulp(beta) + ulp(rm * scale) of
    beta - rm * scale; whether mean is the running mean exactly, and whether the running statistics and num_batches_tracked
    kept every bit. The running variances span 1e-4 .. 1e2 so that rsqrt meets many exponents."""
    import numpy as np
    g = torch.Generator(device="cuda").manual_seed(seed)
    gamma = 1.0 + 0.2 * torch.randn(C, device="cuda", generator=g)
    beta = 0.3 * torch.randn(C, device="cuda", generator=g)
    rm = 0.5 * torch.randn(C, device="cuda", generator=g)
    rv = 10.0 ** (6.0 * torch.rand(C, device="cuda", generator=g) - 4.0)
    nbt = torch.full((1,), 5, dtype=torch.int64, device="cuda")
    rm0, rv0 = rm.clone(), rv.clone()
    scale, shift, mean, rstd = (torch.full((C,), float("nan"), device="cuda") for _ in range(4))
    _lib.call("dfd_bn_finalize", None, None, 1000.0, P(gamma), P(beta), P(rm), P(rv), P(nbt), momentum, eps, 0, C, P(scale),
              P(shift), P(mean), P(rstd), st())
    torch.cuda.synchronize()
    r_ref = 1.0 / torch.sqrt(rv.double() + float(np.float32(eps)))
    sc_ref = gamma.double() * r_ref
    sh_ref = beta.double() - rm.double() * sc_ref
    return dict(rstd_ulp=float(((rstd.double() - r_ref).abs() / _ulp32(r_ref)).max()),
                scale_ulp=float(((scale.double() - sc_ref).abs() / _ulp32(sc_ref)).max()),
                shift_ulp=float(((shift.double() - sh_ref).abs() / (_ulp32(beta.double()) + _ulp32(rm.double() * sc_ref))).max()),
                mean_exact=bool(torch.equal(mean, rm0)),
                state_kept=bool(torch.equal(rm, rm0) and torch.equal(rv, rv0) and int(nbt) == 5),
                nan=int(sum(torch.isnan(t).sum() for t in (scale, shift, mean, rstd))))


def check_optimizer(kind, n=10007, steps=3, dtype=torch.bfloat16, seed=0):
    from oracle import train as OT
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.randn(n, device="cuda", generator=g)
    p_ref = {"w": p.cpu().clone().view(n, 1)}           # 2-D name without 'bias' -> weight decay applies
    lr, wd, mom, eps = 0.05, 1e-2, 0.9, 1e-3
    opt = OT.OptState(kind=kind, lr=lr, momentum=mom, weight_decay=wd, eps=eps)
    a = torch.ones(n, device="cuda") if kind == "rmsproptf" else torch.zeros(n, device="cuda")
    b = torch.zeros(n, device="cuda")
    p16 = torch.zeros(n, device="cuda", dtype=dtype)
    worst = 0.0
    for s in range(steps):
        gr = torch.randn(n, device="cuda", generator=g)
        OT.optimizer_step(opt, p_ref, {"w": gr.cpu().view(n, 1)})
        if kind == "sgd":
            _lib.call("dfd_sgd_step", P(p), P(gr), P(a), n, lr, mom, wd, 1, 1.0, None, None, P(p16), DT[dtype], None, st())
        elif kind in ("adam", "adamw"):
            _lib.call("dfd_adam_step", P(p), P(gr), P(a), P(b), n, lr, 0.9, 0.999, eps, wd, 1 if kind == "adamw" else 0, s + 1, 1.0,
                      None, None, P(p16), DT[dtype], None, None, st())
        else:
            _lib.call("dfd_rmsprop_tf_step", P(p), P(gr), P(a), P(b), n, lr, 0.9, eps, wd, mom, 1.0, None, None, P(p16), DT[dtype], None, st())
        torch.cuda.synchronize()
        worst = max(worst, relerr(p.cpu(), p_ref["w"].view(-1)))
    return dict(rel=worst, p16_rel=relerr(p16.float(), p.to(dtype).float()))


def check_transpose(dtype=torch.bfloat16):
    import struct
    shapes = [(96, 16), (24, 144), (1280, 320), (40, 240)]
    srcs = [torch.randn(o, i, device="cuda").to(dtype) for o, i in shapes]
    dsts = [torch.zeros(i, o, device="cuda", dtype=dtype) for o, i in shapes]
    raw = b"".join(struct.pack("<QQii", P(s), P(d), o, i) for s, d, (o, i) in zip(srcs, dsts, shapes))
    table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    _lib.call("dfd_transpose_weights", P(table), len(shapes), DT[dtype], st())
    torch.cuda.synchronize()
    return dict(mismatch=sum(int((d != s.t()).sum()) for s, d in zip(srcs, dsts)))


def check_conv_dense(N, H, W, Cin, Cout, k, s, dtype=torch.bfloat16, seed=0):
    """k x k dense conv = im2col + tensor-core GEMM; dgrad = GEMM + col2im; wgrad = mma GEMM on im2col + unpack, vs F.conv2d."""
    import struct
    g = torch.Generator(device="cuda").manual_seed(seed)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    M = N * Ho * Wo
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).to(dtype)
    w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / math.sqrt(Cin * k * k)).to(dtype)
    wp = torch.zeros(Cout * k * k * Cin, device="cuda", dtype=dtype)
    wpT = torch.zeros_like(wp)
    table = torch.frombuffer(bytearray(struct.pack("<QQQQiiii", P(w), P(wp), P(wpT), 0, Cout, Cin, k, 0)),
                             dtype=torch.uint8).cuda()
    d = DT[dtype]
    _lib.call("dfd_repack_weights", P(table), 1, d, st())
    cols = torch.full((M, k * k * Cin), float("nan"), device="cuda", dtype=dtype)
    y = torch.full((M, Cout), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_im2col", P(x), P(cols), N, H, W, Cin, k, s, pad, d, st())
    _lib.call("dfd_gemm_tn", P(cols), P(wp), P(y), M, Cout, k * k * Cin, d, None, None, None, st())
    torch.cuda.synchronize()
    xr = nchw(x.float()).requires_grad_(True)
    wr = w.float().clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, stride=s, padding=pad)
    res = dict(fwd_max=maxerr_scaled(nchw(y.view(N, Ho, Wo, Cout).float()), ref.detach()), nan=int(torch.isnan(y.float()).sum()))
    dy = (torch.randn(M, Cout, device="cuda", generator=g) * 0.1).to(dtype)
    ref.backward(nchw(dy.view(N, Ho, Wo, Cout).float()))
    dcols = torch.full((M, k * k * Cin), float("nan"), device="cuda", dtype=dtype)
    add = torch.randn(N, H, W, Cin, device="cuda", generator=g).to(dtype)
    dx = torch.full((N, H, W, Cin), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_gemm_tn", P(dy), P(wpT), P(dcols), M, k * k * Cin, Cout, d, None, None, None, st())
    _lib.call("dfd_col2im", P(dcols), P(add), P(dx), N, H, W, Cin, k, s, pad, d, st())
    gperm = torch.zeros(Cout, k * k * Cin, device="cuda")
    gw = torch.zeros(Cout, Cin, k, k, device="cuda")
    _lib.call("dfd_gemm_wgrad_mma", P(dy), P(cols), P(gperm), M, Cout, k * k * Cin, d, st())
    _lib.call("dfd_unpack_grad", P(gperm), P(gw), Cout, Cin, k, st())
    torch.cuda.synchronize()
    res["dgrad_rel"] = relerr(nchw(dx.float()), xr.grad + nchw(add.float()))
    res["wgrad_rel"] = relerr(gw, wr.grad)
    res["nan_b"] = int(torch.isnan(dx.float()).sum())
    return res


def check_conv_implicit(N, H, W, Cin, Cout, k=3, dtype=torch.bfloat16, seed=0, stride=1):
    """dfd_conv_tc (implicit GEMM, padding (k-1)/2, stride 1 or 2): forward + BatchNorm statistics, the input gradient (stride 1: the
    same kernel on dY with the tap-flipped weights) and the implicit weight gradient against fp64 F.conv2d / autograd; the forward
    also bit for bit against the im2col formulation."""
    import struct
    g = torch.Generator(device="cuda").manual_seed(seed)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).to(dtype)
    w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / math.sqrt(Cin * k * k)).to(dtype)
    wp = torch.zeros(Cout * k * k * Cin, device="cuda", dtype=dtype)
    wpT, wpD = torch.zeros_like(wp), torch.zeros_like(wp)
    table = torch.frombuffer(bytearray(struct.pack("<QQQQiiii", P(w), P(wp), P(wpT), P(wpD),
                                                   Cout, Cin, k, 0)), dtype=torch.uint8).cuda()
    d = DT[dtype]
    _lib.call("dfd_repack_weights", P(table), 1, d, st())
    y = torch.full((N, Ho, Wo, Cout), float("nan"), device="cuda", dtype=dtype)
    dsum, dsq = stat_buf(Cout), stat_buf(Cout)
    _lib.call("dfd_conv_tc", P(x), P(wp), P(y), N, H, W, Cin, Cout, k, stride, d, P(dsum), P(dsq), None, st())
    torch.cuda.synchronize()
    xr = nchw(x.double()).requires_grad_(True)      # fp64: cuDNN's fp32 algorithm choice (TF32 / Winograd / FFT) is not a reference
    wr = w.double().clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, stride=stride, padding=pad)
    yf = y.float()
    res = dict(fwd_max=maxerr_scaled(nchw(yf), ref.detach()), nan=int(torch.isnan(yf).sum()),
               fwd_max_bf16trip=maxerr_scaled(nchw(bf16_trip(y).float()), ref.detach()))
    # the statistics-free launch (the eval form, and the stride-1 input gradient) stores the same bits
    y_ns = torch.full_like(y, float("nan"))
    _lib.call("dfd_conv_tc", P(x), P(wp), P(y_ns), N, H, W, Cin, Cout, k, stride, d, None, None, None, st())
    torch.cuda.synchronize()
    res["nostats_mismatch"] = int((y_ns.view(torch.int16) != y.view(torch.int16)).sum())
    del y_ns
    # the statistics are those of the STORED (rounded) output
    s1, s2 = dsum.sum(0), dsq.sum(0)
    res["sum_rel"] = relerr(s1, yf.double().sum((0, 1, 2)))
    res["sq_rel"] = relerr(s2, (yf.double() ** 2).sum((0, 1, 2)))
    # the im2col formulation computes the same products in the same K order: bit-identical output
    cols = torch.zeros(N * Ho * Wo, k * k * Cin, device="cuda", dtype=dtype)
    y2 = torch.zeros_like(y)
    _lib.call("dfd_im2col", P(x), P(cols), N, H, W, Cin, k, stride, pad, d, st())
    _lib.call("dfd_gemm_tn", P(cols), P(wp), P(y2), N * Ho * Wo, Cout, k * k * Cin, d, None, None, None, st())
    torch.cuda.synchronize()
    res["vs_im2col_mismatch"] = int((y2.view(torch.int16) != y.view(torch.int16)).sum())
    dy = (torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g) * 0.1).to(dtype)
    ref.backward(nchw(dy.double()))
    res["dgrad_rel"], res["nan_b"] = 0.0, 0
    if stride == 2 and k == 3:
        dx = torch.full((N, H, W, Cin), float("nan"), device="cuda", dtype=dtype)      # every element must be written exactly once
        _lib.call("dfd_conv_dgrad_s2_tc", P(dy), P(wpD), P(dx), N, H, W, Cin, Cout, d, st())
        torch.cuda.synchronize()
        res["dgrad_rel"] = relerr(nchw(dx.float()), xr.grad)
        res["dgrad_max"], res["dgrad_max_bf16trip"] = _scaled_pair(dx, xr.grad)
        res["nan_b"] = int(torch.isnan(dx.float()).sum())
        # against the GEMM + col2im formulation (same products, different summation order inside a pixel: not bit-identical)
        dcols = torch.zeros(N * Ho * Wo, k * k * Cin, device="cuda", dtype=dtype)
        dx2 = torch.zeros_like(dx)
        _lib.call("dfd_gemm_tn", P(dy), P(wpT), P(dcols), N * Ho * Wo, k * k * Cin, Cout, d, None, None, None, st())
        _lib.call("dfd_col2im", P(dcols), None, P(dx2), N, H, W, Cin, k, 2, pad, d, st())
        torch.cuda.synchronize()
        res["dgrad_vs_col2im"] = relerr(dx.float(), dx2.float())
        res["col2im_dgrad_max"], res["col2im_dgrad_max_bf16trip"] = _scaled_pair(dx2, xr.grad)
    if stride == 1:
        dx = torch.full((N, H, W, Cin), float("nan"), device="cuda", dtype=dtype)
        _lib.call("dfd_conv_tc", P(dy), P(wpD), P(dx), N, H, W, Cout, Cin, k, 1, d, None, None, None, st())
        torch.cuda.synchronize()
        res["dgrad_rel"] = relerr(nchw(dx.float()), xr.grad)
        res["dgrad_max"], res["dgrad_max_bf16trip"] = _scaled_pair(dx, xr.grad)
        res["nan_b"] = int(torch.isnan(dx.float()).sum())
    # weight gradient (implicit too): packed [Cout][kh][kw][Cin] fp32 -> OIHW; atomic flush and workspace partials + ordered reduce
    Kw = k * k * Cin
    gperm = torch.zeros(Cout, Kw, device="cuda")
    _lib.call("dfd_conv_wgrad_tc", P(dy), P(x), P(gperm), N, H, W, Cin, Cout, k, stride, d, None, 0, st())
    gw = torch.zeros(Cout, Cin, k, k, device="cuda")
    _lib.call("dfd_unpack_grad", P(gperm), P(gw), Cout, Cin, k, st())
    splits = _lib.lib().cdll.dfd_conv_wgrad_splits(N, H, W, Cin, Cout, k, stride)
    ws = torch.full((splits, Cout, Kw), float("nan"), device="cuda")
    det = [torch.zeros(Cout, Kw, device="cuda"), torch.zeros(Cout, Kw, device="cuda")]
    for t in det:
        _lib.call("dfd_conv_wgrad_tc", P(dy), P(x), P(t), N, H, W, Cin, Cout, k, stride, d, P(ws), ws.numel() * 4, st())
        table = torch.frombuffer(bytearray(struct.pack("<QQqqii", P(ws), P(t), Cout * Kw, Cout * Kw, splits, 0)), dtype=torch.uint8).cuda()
        _lib.call("dfd_ordered_reduce", P(table), 1, P(t), min(1024, (Cout * Kw // 4 + 255) // 256), st())
        torch.cuda.synchronize()
    res["wgrad_rel"] = relerr(gw, wr.grad)
    res["wgrad_det_bitwise"] = bool(torch.equal(det[0], det[1]))
    res["wgrad_det_vs_atomic"] = relerr(det[0], gperm)
    res["wgrad_splits"] = splits
    return res


def check_conv1x1_dgrad_add(N, H, W, Cin, Cout, stride, dtype=torch.bfloat16, seed=0):
    """dfd_conv1x1_dgrad_add (TMA reduction store through a strided view) == dfd_gemm_tn + dfd_col2im(add) bit for bit"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    dy = (torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g) * 0.1).to(dtype)
    w = (torch.randn(Cout, Cin, device="cuda", generator=g) / math.sqrt(Cin)).to(dtype)
    wT = w.t().contiguous()                                      # [Cin][Cout]
    main = torch.randn(N, H, W, Cin, device="cuda", generator=g).to(dtype)
    d = DT[dtype]
    t2 = torch.zeros(N * Ho * Wo, Cin, device="cuda", dtype=dtype)
    ref = torch.full_like(main, float("nan"))
    _lib.call("dfd_gemm_tn", P(dy), P(wT), P(t2), N * Ho * Wo, Cin, Cout, d, None, None, None, st())
    _lib.call("dfd_col2im", P(t2), P(main), P(ref), N, H, W, Cin, 1, stride, 0, d, st())
    got = main.clone()
    _lib.call("dfd_conv1x1_dgrad_add", P(dy), P(wT), P(got), N, H, W, Cin, Cout, stride, d, st())
    torch.cuda.synchronize()
    exact = (dy.float().reshape(-1, Cout) @ w.float()).reshape(N, Ho, Wo, Cin)
    full = main.float().clone()
    full[:, ::stride, ::stride, :] += exact
    full64 = main.double()          # fp64: the scaled bound of the tensor-core contractions
    full64[:, ::stride, ::stride, :] += (dy.double().reshape(-1, Cout) @ w.double()).reshape(N, Ho, Wo, Cin)
    out_max, out_max_trip = _scaled_pair(got, full64, to_nchw=False)
    return dict(mismatch=int((got.view(torch.int16) != ref.view(torch.int16)).sum()), rel=relerr(got.float(), full),
                nan=int(torch.isnan(got.float()).sum()), out_max=out_max, out_max_bf16trip=out_max_trip)


def check_relu_bn_bwd_reduce(N, HW, C, dtype=torch.bfloat16, seed=0, two=False):
    """dfd_relu_bn_bwd_reduce == dfd_relu_bwd followed by dfd_bn_bwd_reduce: the masked gradient bit for bit, the sums to fp64 rounding"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    gy = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype)
    y = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype)
    out = torch.relu(torch.randn(N, HW, C, device="cuda", generator=g)).to(dtype)
    mean, rstd = torch.randn(C, device="cuda", generator=g) * 0.1, torch.rand(C, device="cuda", generator=g) + 0.5
    d = DT[dtype]
    gm_a, gm_b = torch.full_like(gy, float("nan")), torch.full_like(gy, float("nan"))
    a1, a2, b1, b2 = stat_buf(C), stat_buf(C), stat_buf(C), stat_buf(C)
    g2 = torch.randn(N, HW, C, device="cuda", generator=g).to(dtype) if two else None
    gsum = gy
    if two:                                     # the materialised residual add the fused kernel replaces
        gsum = gy.clone()
        _lib.call("dfd_add_inplace", P(gsum), P(g2), gsum.numel(), d, st())
    _lib.call("dfd_relu_bwd", P(gsum), P(out), P(gm_a), gy.numel(), d, st())
    _lib.call("dfd_bn_bwd_reduce", P(gm_a), P(y), None, P(mean), P(rstd), N, HW, C, d, P(a1), P(a2), None, st())
    _lib.call("dfd_relu_bn_bwd_reduce", P(gy), P(g2) if two else None, P(y), P(out), P(gm_b), P(mean), P(rstd), N, HW, C, d, P(b1), P(b2), st())
    torch.cuda.synchronize()
    gmf = gsum.float() * (out.float() > 0)
    xhat = (y.float() - mean) * rstd
    return dict(gm_mismatch=int((gm_a.view(torch.int16) != gm_b.view(torch.int16)).sum()), s1_rel=relerr(b1.sum(0), a1.sum(0)),
                s2_rel=relerr(b2.sum(0), a2.sum(0)), s1_ref=relerr(b1.sum(0), gmf.double().sum((0, 1))),
                s2_ref=relerr(b2.sum(0), (gmf * xhat).double().sum((0, 1))))


def check_maxpool_relu_pool(N, H, W, C, dtype=torch.bfloat16, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.relu(torch.randn(N, H, W, C, device="cuda", generator=g)).to(dtype)        # many exact ties at 0
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = torch.full((N, Ho, Wo, C), float("nan"), device="cuda", dtype=dtype)
    idx = torch.zeros(N * Ho * Wo * C, dtype=torch.uint8, device="cuda")
    d = DT[dtype]
    _lib.call("dfd_maxpool_fwd", P(x), P(out), P(idx), N, H, W, C, d, st())
    xr = nchw(x.float()).requires_grad_(True)
    ref = F.max_pool2d(xr, 3, 2, 1)
    gy = torch.randn(N, Ho, Wo, C, device="cuda", generator=g).to(dtype)
    ref.backward(nchw(gy.float()))
    gx = torch.full((N, H, W, C), float("nan"), device="cuda", dtype=dtype)
    _lib.call("dfd_maxpool_bwd", P(gy), P(idx), P(gx), N, H, W, C, d, st())
    gm = torch.zeros_like(gy)
    _lib.call("dfd_relu_bwd", P(gy), P(out), P(gm), gy.numel(), d, st())
    dp = torch.randn(N, C, device="cuda", generator=g)
    bro = torch.zeros(N, Ho * Wo, C, device="cuda", dtype=dtype)
    _lib.call("dfd_pool_bwd", P(dp), P(bro), N, Ho * Wo, C, d, st())
    torch.cuda.synchronize()
    bwd_ulp = maxpool_bwd_bound(gx, x, gy, lambda t: F.max_pool2d(t, 3, 2, 1), dtype)
    return dict(bwd_ulp=bwd_ulp[0], bwd_ulp_bf16trip=bwd_ulp[1],
                fwd_exact=int((nchw(out.float()) != ref.detach()).sum()), bwd_rel=relerr(nchw(gx.float()), xr.grad),
                relu_mismatch=int((gm.float() != gy.float() * (out.float() > 0)).sum()),
                pool_bwd_rel=relerr(bro.float(), (dp / (Ho * Wo)).to(dtype).float().unsqueeze(1).expand(N, Ho * Wo, C)))
