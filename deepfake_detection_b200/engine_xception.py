"""Kernel plan of Xception (`xception`) for `Engine` — host side only.

Reference graph: dfd/timm/models/xception.py. Stem conv1 3x3 s2 p0 -> BN -> ReLU -> conv2 3x3 p0 -> BN -> ReLU (:183-188);
twelve `Block`s (:72-124) of SeparableConv2d (depthwise 3x3 p1 straight into a 1x1 pointwise, no BN or activation between,
:58-69) each followed by a BatchNorm; conv3 / conv4 separable convolutions with bn3 / bn4 (:201-208); global pool, fc.

Plan:
  * conv1 runs through the stem im2col + GEMM, conv2 (Cin = 32) through the explicit im2col route (3x3, padding 0); both
    take their BatchNorm statistics in the GEMM epilogue. The stem output is materialised: block1's first depthwise
    convolution and its shortcut read it.
  * every separable convolution is a depthwise forward into a 16-bit buffer - its input's ReLU (and the preceding BN) applied
    at load, no statistics since no BN follows - then the pointwise GEMM with the statistics of the next BN. The ReLU
    outputs are never stored.
  * a strided block ends in `dfd_bn_maxpool_add`: BN of the last separable convolution, the 3x3 s2 p1 max-pool and the
    shortcut BN add in one pass (the pooled BN output is never stored). An identity block ends in `dfd_bn_act` with the
    block input as the residual, no activation: a block's output is stored before its ReLU, which the next block's first
    depthwise convolution applies (xception.py:107-108, the non-inplace rep[0]).
  * the shortcut 1x1 stride-2 convolutions run as implicit GEMMs where both channel counts are multiples of 64 (blocks 1, 2);
    blocks 3 and 12 (728 channels) gather the strided input with a k = 1 im2col and run a plain GEMM.
  * backward: the strided tail through `dfd_maxpool_bn_bwd_reduce` (pool gradient + BN-backward sums in one pass), the
    shortcut BN through `dfd_bn_bwd_reduce`; each pointwise dgrad feeds the fused depthwise backward in its ReLU mode,
    which masks by the staged 16-bit input and reduces the preceding BN's backward sums (or adds the identity gradient).
Dropout: the reference calls F.dropout and discards its result (xception.py:214-215); `drop_rate` changes nothing here.
"""
import torch

from .arch import xception_extents
from .engine import ACT_NONE, ACT_RELU, _ptr


def build_xception(e):
    spec, N, dev, dt = e.spec, e.N, e.device, e.dt
    fwd, bwd = [], []

    # ---- packed (kh, kw, ci) copy of conv2's weight (the im2col GEMM's B operand, its transpose and the dgrad layout) -------
    e._packed_weights(["conv2.weight"])
    e.gperm = torch.zeros(e.p_off["conv2.weight"][2], dtype=torch.float32, device=dev)

    P32, G32, P16, T16 = e._p32, e._g32, e._p16, e._t16

    # ---- shapes ------------------------------------------------------------------------------------------
    ext = xception_extents(e.H, e.W)
    if min(min(hw) for hw in ext) < 1:
        raise ValueError("input %dx%d is too small for Xception" % (e.H, e.W))
    (H1, W1), (H2, W2) = ext[0], ext[1]
    shapes = []
    h, w = H2, W2
    for b, (ho, wo) in zip(spec.blocks, ext[2:]):
        shapes.append((b, h, w, ho, wo))
        h, w = ho, wo
    Hf, Wf = h, w
    Mf = N * Hf * Wf

    # ---- BN arenas ---------------------------------------------------------------------------------------
    bn_specs = [("bn1", 32), ("bn2", 64)]
    for b in spec.blocks:
        if b.skip:
            bn_specs.append((b.name + ".skipbn", b.cout))
        bn_specs += [("%s.rep.%d" % (b.name, r + 1), co) for r, _, co in b.seps]
    bn_specs += [("bn3", 1536), ("bn4", spec.num_features)]
    e._alloc_bn(bn_specs)
    bns = e.bns
    gemm = lambda *a: e._gemm(*a, rowpack=False)        # every K is >= 32 and a multiple of 8; no row-packed GEMMs
    finalize, bwd_finalize = e._finalize, e._bwd_finalize
    implicit = e.gemm_impl == "tc"

    def dw_fwd(xin, scale, shift, name, out, h, w, C, act):
        return ("dfd_dwconv_fwd", (xin, scale, shift, P32(name), _ptr(out), N, h, w, C, 3, 1, act, dt, None, None, None))

    # ---- scratch -----------------------------------------------------------------------------------------
    max_act = max([N * H1 * W1 * 32, N * H2 * W2 * 64] + [N * hh * ww * max(b.cin, b.cout) for b, hh, ww, _, _ in shapes]
                  + [Mf * 2048])
    e.gbuf = [e._alloc16(max_act) for _ in range(6)]
    e.cols = e._alloc16(N * H2 * W2 * 9 * 32)
    COLS = _ptr(e.cols)

    # ---- forward: stem -------------------------------------------------------------------------------------
    bn1, bn2 = bns["bn1"], bns["bn2"]
    y1, a1 = e._alloc16(N, H1, W1, 32), e._alloc16(N, H1, W1, 32)
    y2, a2 = e._alloc16(N, H2, W2, 64), e._alloc16(N, H2, W2, 64)
    fwd += e._stem_gemm("conv1.weight", 32, 3, 2, 0, y1, N * H1 * W1, bn1, rowpack=False)
    fwd += finalize(bn1, N * H1 * W1)
    fwd.append(("dfd_bn_act", (_ptr(y1), bn1.scale, bn1.shift, None, None, _ptr(a1), N, H1 * W1, 32, ACT_RELU, 0, dt)))
    fwd.append(("dfd_im2col", (_ptr(a1), COLS, N, H1, W1, 32, 3, 1, 0, dt)))
    fwd.append(gemm(COLS, _ptr(e.wpack16), _ptr(y2), N * H2 * W2, 64, 9 * 32, bn2))
    fwd += finalize(bn2, N * H2 * W2)
    fwd.append(("dfd_bn_act", (_ptr(y2), bn2.scale, bn2.shift, None, None, _ptr(a2), N, H2 * W2, 64, ACT_RELU, 0, dt)))
    e.acts["stem.out"] = a2

    # ---- forward: blocks -------------------------------------------------------------------------------------
    x = a2
    recs = []
    for b, h, w, ho, wo in shapes:
        p = b.name
        M1, M2 = N * h * w, N * ho * wo
        rec = dict(b=b, h=h, w=w, ho=ho, wo=wo, x=x, seps=[])
        prev = None                     # (y, bn) of the previous separable convolution in the block
        for r, ci, co in b.seps:
            sp = "%s.rep.%d" % (p, r)
            bn = bns["%s.rep.%d" % (p, r + 1)]
            d = e._alloc16(N, h, w, ci)
            y = e._alloc16(N, h, w, co)
            if prev is None:            # rep[0]: ReLU of the block input, or the activated stem output as is (block1)
                fwd.append(dw_fwd(_ptr(x), None, None, sp + ".conv1.weight", d, h, w, ci,
                                  ACT_RELU if b.start_with_relu else ACT_NONE))
            else:
                fwd.append(dw_fwd(_ptr(prev[0]), prev[1].scale, prev[1].shift, sp + ".conv1.weight", d, h, w, ci, ACT_RELU))
            fwd.append(gemm(_ptr(d), P16(sp + ".pointwise.weight"), _ptr(y), M1, co, ci, bn))
            fwd += finalize(bn, M1)
            rec["seps"].append(dict(name=sp, ci=ci, co=co, d=d, y=y, bn=bn))
            prev = (y, bn)
        out = e._alloc16(N, ho, wo, b.cout)
        ylast, bnl = prev
        if b.skip:
            bnd = bns[p + ".skipbn"]
            yd = e._alloc16(N, ho, wo, b.cout)
            if implicit and b.cin % 64 == 0 and b.cout % 64 == 0:
                xs = None
                fwd.append(("dfd_conv_tc", (_ptr(x), P16(p + ".skip.weight"), _ptr(yd), N, h, w, b.cin, b.cout, 1, 2, dt)
                            + e._stats(bnd) + (None,)))
            else:
                xs = e._alloc16(N, ho, wo, b.cin)
                fwd.append(("dfd_im2col", (_ptr(x), _ptr(xs), N, h, w, b.cin, 1, 2, 0, dt)))
                fwd.append(gemm(_ptr(xs), P16(p + ".skip.weight"), _ptr(yd), M2, b.cout, b.cin, bnd))
            fwd += finalize(bnd, M2)
            idx = torch.zeros(N * ho * wo * b.cout, dtype=torch.uint8, device=dev)
            e._keep.append(idx)
            fwd.append(("dfd_bn_maxpool_add", (_ptr(ylast), bnl.scale, bnl.shift, _ptr(yd), bnd.scale, bnd.shift, _ptr(out),
                                               ("TRAIN_ONLY", _ptr(idx)), N, h, w, b.cout, dt)))
            rec.update(yd=yd, xs=xs, bnd=bnd, idx=idx)
        else:
            fwd.append(("dfd_bn_act", (_ptr(ylast), bnl.scale, bnl.shift, None, _ptr(x), _ptr(out), N, h * w, b.cout, ACT_NONE,
                                       1, dt)))
        e.acts[p + ".out"] = out
        rec["out"] = out
        recs.append(rec)
        x = out

    # ---- forward: conv3 / conv4 and the head -----------------------------------------------------------------
    bn3, bn4 = bns["bn3"], bns["bn4"]
    F = spec.num_features
    d3, y3 = e._alloc16(N, Hf, Wf, 1024), e._alloc16(N, Hf, Wf, 1536)
    d4, y4 = e._alloc16(N, Hf, Wf, 1536), e._alloc16(N, Hf, Wf, F)
    fwd.append(dw_fwd(_ptr(x), None, None, "conv3.conv1.weight", d3, Hf, Wf, 1024, ACT_NONE))
    fwd.append(gemm(_ptr(d3), P16("conv3.pointwise.weight"), _ptr(y3), Mf, 1536, 1024, bn3))
    fwd += finalize(bn3, Mf)
    fwd.append(dw_fwd(_ptr(y3), bn3.scale, bn3.shift, "conv4.conv1.weight", d4, Hf, Wf, 1536, ACT_RELU))
    fwd.append(gemm(_ptr(d4), P16("conv4.pointwise.weight"), _ptr(y4), Mf, F, 1536, bn4))
    fwd += finalize(bn4, Mf)
    e.acts["conv4"] = y4
    fwd += e._pool_head(y4, bn4, ACT_RELU, Hf * Wf, 0.0)         # no dropout: see the module docstring
    e.drop_masks = {}

    # ---- backward ----------------------------------------------------------------------------------------
    bufs = [_ptr(t) for t in e.gbuf]

    def free(*used):
        return [g for g in bufs if g not in used]

    def dw_bwd(gy, name, xin, bn_in, add, gx, h, w, C, mode):
        """fused depthwise backward: mode "bn_relu" (input relu(bn_in(xin)), bn_in's backward sums), "relu" (input relu(xin),
        + add) or "plain" (input xin, + add)"""
        if mode == "bn_relu":
            args = (gy, None, None, None, None, P32(name), _ptr(xin), bn_in.scale, bn_in.shift, bn_in.mean, bn_in.rstd, None,
                    gx, G32(name), N, h, w, C, 3, 1, dt, bn_in.bs1, bn_in.bs2)
        else:
            args = (gy, None, None, None, None, P32(name), _ptr(xin), None, None, None, None, add, gx, G32(name), N, h, w, C,
                    3, 1, dt, None, None)
        return e._dw_bwd(args, N, h, w, C, 3, 1, name="dfd_dwconv_bwd" if mode == "plain" else "dfd_dwconv_bwd_relu")

    def sep_bwd(gy, s, bn_in, xin, add, gx, h, w, mode, keep=()):
        """pointwise dgrad / wgrad of separable convolution `s` from gy (gradient of its pointwise output), then its depthwise
        backward into gx; `keep`: gradient buffers still live"""
        M = N * h * w
        gd = free(gy, gx, add, *keep)[0]
        return [gemm(gy, T16(s["name"] + ".pointwise.weight"), gd, M, s["ci"], s["co"]),
                e._wgrad(gy, _ptr(s["d"]), G32(s["name"] + ".pointwise.weight"), M, s["co"], s["ci"]),
                dw_bwd(gd, s["name"] + ".conv1.weight", xin, bn_in, add, gx, h, w, s["ci"], mode)]

    gA, gB, gC, gD = bufs[:4]
    bwd += e._pool_head_bwd(gA)
    bwd += bwd_finalize(bn4, Mf)
    bwd.append(e._bn_apply(gA, y4, bn4, gB, Hf * Wf, F))
    s4 = dict(name="conv4", ci=1536, co=F, d=d4)
    bwd += sep_bwd(gB, s4, bn3, y3, None, gC, Hf, Wf, "bn_relu")
    bwd += bwd_finalize(bn3, Mf)
    bwd.append(e._bn_apply(gC, y3, bn3, gB, Hf * Wf, 1536))
    s3 = dict(name="conv3", ci=1024, co=1536, d=d3)
    bwd += sep_bwd(gB, s3, None, x, None, gC, Hf, Wf, "plain")
    e._flush_reduce(bwd)
    dout = gC
    for rec in reversed(recs):
        b, h, w, ho, wo, xin = rec["b"], rec["h"], rec["w"], rec["ho"], rec["wo"], rec["x"]
        M1, M2 = N * h * w, N * ho * wo
        seps = rec["seps"]
        last = seps[-1]
        gbn, gy, gyd, gx, t = free(dout)[:5]
        if b.skip:
            bnd = rec["bnd"]
            bwd.append(("dfd_maxpool_bn_bwd_reduce", (dout, _ptr(rec["idx"]), _ptr(last["y"]), last["bn"].mean, last["bn"].rstd,
                                                      gbn, N, h, w, b.cout, dt, last["bn"].bs1, last["bn"].bs2)))
            bwd += bwd_finalize(last["bn"], M1)
            bwd.append(e._bn_apply(gbn, last["y"], last["bn"], gy, h * w, b.cout))
            bwd.append(("dfd_bn_bwd_reduce", (dout, _ptr(rec["yd"]), None, bnd.mean, bnd.rstd, N, ho * wo, b.cout, dt, bnd.bs1,
                                              bnd.bs2, None)))
            bwd += bwd_finalize(bnd, M2)
            bwd.append(e._bn_apply(dout, rec["yd"], bnd, gyd, ho * wo, b.cout))
        else:
            bwd.append(("dfd_bn_bwd_reduce", (dout, _ptr(last["y"]), None, last["bn"].mean, last["bn"].rstd, N, h * w, b.cout, dt,
                                              last["bn"].bs1, last["bn"].bs2, None)))
            bwd += bwd_finalize(last["bn"], M1)
            bwd.append(e._bn_apply(dout, last["y"], last["bn"], gy, h * w, b.cout))
            gyd = None
        # separable convolutions, last to first: gy is the gradient of the current pointwise output
        for j in range(len(seps) - 1, 0, -1):
            prev = seps[j - 1]
            gu = free(dout, gy, gyd)[0]
            bwd += sep_bwd(gy, seps[j], prev["bn"], prev["y"], None, gu, h, w, "bn_relu", keep=(dout, gyd))
            bwd += bwd_finalize(prev["bn"], M1)
            bwd.append(e._bn_apply(gu, prev["y"], prev["bn"], gy, h * w, prev["co"]))
        mode = "relu" if b.start_with_relu else "plain"
        gx = free(dout, gy, gyd)[0]
        bwd += sep_bwd(gy, seps[0], None, xin, None if b.skip else dout, gx, h, w, mode, keep=(gyd,))
        if b.skip:
            sw = b.name + ".skip.weight"
            if rec["xs"] is None:
                # the shortcut's input gradient is added into gx by the GEMM's epilogue (stride-2 pixel view of gx)
                bwd.append(("dfd_conv1x1_dgrad_add", (gyd, T16(sw), gx, N, h, w, b.cin, b.cout, 2, dt)))
                bwd.append(e._wgrad_conv(gyd, _ptr(xin), G32(sw), N, h, w, b.cin, b.cout, 1, 2))
            else:
                t, dst = free(gx, gyd)[:2]
                bwd.append(gemm(gyd, T16(sw), t, M2, b.cin, b.cout))
                bwd.append(e._wgrad(gyd, _ptr(rec["xs"]), G32(sw), M2, b.cout, b.cin))
                bwd.append(("dfd_col2im", (t, gx, dst, N, h, w, b.cin, 1, 2, 0, dt)))
                gx = dst
        e._flush_reduce(bwd)
        dout = gx

    # ---- backward: stem (dout = gradient of the activated stem output a2) ---------------------------------------------
    gu, gy = free(dout)[:2]
    bwd.append(("dfd_act_bwd", (dout, _ptr(y2), bn2.scale, bn2.shift, bn2.mean, bn2.rstd, None, None, gu, N, H2 * W2, 64,
                                ACT_RELU, dt, bn2.bs1, bn2.bs2, None)))
    bwd += bwd_finalize(bn2, N * H2 * W2)
    bwd.append(e._bn_apply(gu, y2, bn2, gy, H2 * W2, 64))
    ga1 = free(gy)[0]
    bwd.append(gemm(gy, _ptr(e.wpackT16), COLS, N * H2 * W2, 9 * 32, 64))
    bwd.append(("dfd_col2im", (COLS, None, ga1, N, H1, W1, 32, 3, 1, 0, dt)))
    bwd.append(("dfd_im2col", (_ptr(a1), COLS, N, H1, W1, 32, 3, 1, 0, dt)))
    bwd.append(("dfd_memset_async", (_ptr(e.gperm), 0, e.gperm.numel() * 4)))
    bwd.append(e._wgrad(gy, COLS, _ptr(e.gperm), N * H2 * W2, 64, 9 * 32))
    gu, gy1 = free(ga1)[:2]
    bwd.append(("dfd_act_bwd", (ga1, _ptr(y1), bn1.scale, bn1.shift, bn1.mean, bn1.rstd, None, None, gu, N, H1 * W1, 32,
                                ACT_RELU, dt, bn1.bs1, bn1.bs2, None)))
    bwd += bwd_finalize(bn1, N * H1 * W1)
    bwd.append(e._bn_apply(gu, y1, bn1, gy1, H1 * W1, 32))
    bwd += e._stem_wgrad(gy1)
    e._flush_reduce(bwd)
    bwd.append(("dfd_unpack_grad", (_ptr(e.gperm), G32("conv2.weight"), 64, 32, 3)))
    bwd.append(e._stem_unpad())
    e._finish_plan(fwd, bwd)
