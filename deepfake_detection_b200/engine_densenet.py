"""Kernel plan of DenseNet-121/161/169/201 (`densenet*`) for `Engine` — host side only.

Reference graph: dfd/timm/models/densenet.py. Stem conv0 7x7 s2 p3 -> norm0 -> ReLU -> max-pool 3x3 s2 p1 (:96-101); dense
blocks of `_DenseLayer`s (:37-56: norm1, ReLU, 1x1 conv1 to bn_size * k, norm2, ReLU, 3x3 conv2 to k, F.dropout, torch.cat);
`_Transition`s between the blocks (:62-70: norm, ReLU, 1x1 conv halving the width, AvgPool2d(2, 2)); norm5, F.relu, the
global pool, F.dropout and `classifier` (:124-140).

Plan:
  * one 16-bit NHWC buffer per dense block whose rows hold the block's final width. The stem pool or the transition output
    fills channels [0, C0); layer l writes its k channels at [C0 + l*k, C0 + (l+1)*k). Nothing is concatenated by copying.
  * the batch statistics of every channel are reduced ONCE, when the channel is produced, into one [slots][width] pair per
    block. Every BatchNorm that normalises a channel (each later norm1, the transition's norm, norm5) finalises its own
    scale / shift and running statistics from those sums (`dfd_bn_finalize_ld` over a channel prefix).
  * norm1 + ReLU is materialised per layer as a contiguous [M, C] operand (`dfd_bn_relu_ld`, a strided prefix read) for the
    conv1 GEMM, and kept for conv1's weight gradient; conv1 takes norm2's statistics in its epilogue.
  * conv2 (bn_size * k -> k, 3x3) runs as `dfd_conv3x3_narrow_tc`: the wgmma implicit GEMM with 32 / 48-wide tiles storing
    straight into the layer's channel slice of the block buffer, with the slice's statistics in the epilogue. With dropout it
    writes a contiguous scratch and `dfd_copy_ld` applies the mask, stores the slice and takes the statistics after the mask.
  * a transition is one pass of BN + ReLU + floor 2x2 average pool (`dfd_bn_relu_avgpool2`), then the 1x1 GEMM on the pooled
    tensor (pool-then-conv equals conv-then-pool: both are linear and the conv has no bias; a quarter of the FLOPs). The GEMM
    writes a contiguous [M', C/2] tensor that `dfd_copy_ld` stores into the next block's channel prefix with its statistics:
    one extra read and write of 2 * M' * C/2 bytes each.
  * backward, block by block in reverse layer order, with one 16-bit gradient buffer per block (same layout). norm5's backward
    or the transition's initialises it; each layer takes its now-complete k-channel slice into a contiguous buffer (applying
    the dropout mask), runs conv2's input gradient (`dfd_conv3x3_narrow_dgrad_tc`) and weight gradient (`dfd_conv_wgrad_tc`),
    relu2 / norm2, conv1's GEMMs, and norm1's backward, which ADDS into the gradient buffer's channel prefix
    (`dfd_relu_bn_bwd_reduce_ld` / `dfd_relu_bn_bwd_apply_add_ld`). The buffer accumulates in 16 bit, as the reference does
    under apex O1 (a float buffer would double its size: 822 MB for block 1 at batch 256, 224 x 224).
gemm_impl="mma" builds the same plan with conv2 as im2col + mma.sync GEMMs (the cross-check of the narrow kernels).
"""
import torch

from .arch import densenet_extents
from .engine import ACT_RELU, _ptr


def build_densenet(e):
    spec, N, dev, dt = e.spec, e.N, e.device, e.dt
    fwd, bwd = [], []
    k, K4, F = spec.growth, spec.bn_size * spec.growth, spec.num_features
    implicit = e.gemm_impl == "tc"
    P32, G32, P16, T16 = e._p32, e._g32, e._p16, e._t16
    S = e.L.stat_slots
    gemm = lambda *a: e._gemm(*a, rowpack=False)
    finalize, bwd_finalize = e._finalize, e._bwd_finalize

    ext = densenet_extents(e.H, e.W)
    if min(min(hw) for hw in ext) < 1:
        raise ValueError("input %dx%d is too small for %s" % (e.H, e.W, spec.arch))
    (H1, W1), (H2, W2) = ext[0], ext[1]
    widths = spec.block_widths
    nblocks = len(spec.block_config)

    def lname(b, l):
        return "features.denseblock%d.denselayer%d" % (b + 1, l + 1)

    # ---- packed (kh, kw, ci) copies of the 3x3 conv2 weights; one fp32 region for a layer's packed weight gradient ----------
    conv2 = [lname(b, l) + ".conv2.weight" for b in range(nblocks) for l in range(spec.block_config[b])]
    pk = e._packed_weights(conv2)
    e.gperm = torch.zeros(k * 9 * K4, dtype=torch.float32, device=dev)
    GPERM = _ptr(e.gperm)

    # ---- BN arenas: per-layer parameters / coefficients, and one statistics pair per block ---------------------------------
    c0 = spec.init_features
    bn_specs = [("features.norm0", c0)]
    for b, (cin, cend) in enumerate(widths):
        for l in range(spec.block_config[b]):
            bn_specs += [(lname(b, l) + ".norm1", cin + l * k), (lname(b, l) + ".norm2", K4)]
        bn_specs.append(("features.transition%d.norm" % (b + 1) if b + 1 < nblocks else "features.norm5", cend))
    base = e._alloc_bn(bn_specs, extra_stats=sum(2 * S * cend for _, cend in widths))
    bns = e.bns
    bstat, off = [], base
    for _, cend in widths:
        bstat.append((_ptr(e.stats, off), _ptr(e.stats, off + S * cend)))
        off += 2 * S * cend

    def fin_ld(bn, b, count):
        """finalise `bn` over the first bn.C channels of block b's statistics"""
        fs, fq = bstat[b]
        return ("dfd_bn_finalize_ld", [fs, fq, float(count), bn.gamma, bn.beta, bn.rm, bn.rv, bn.nbt, e.bn_momentum, e.bn_eps,
                                       "TRAINING", bn.C, widths[b][1], bn.scale, bn.shift, bn.mean, bn.rstd])

    def slice_stats(b, c):
        fs, fq = bstat[b]
        return ("TRAIN_ONLY", fs + 8 * c), ("TRAIN_ONLY", fq + 8 * c)

    # ---- buffers -----------------------------------------------------------------------------------------
    hw_b = ext[1:]
    Ms = [N * h * w for h, w in hw_b]
    X = [e._alloc16(N, h, w, cend) for (h, w), (_, cend) in zip(hw_b, widths)]
    GX = [e._alloc16(N, h, w, cend) for (h, w), (_, cend) in zip(hw_b, widths)]
    # scratch: T0-T2 the [M, bn_size * k] layer gradients (and the stem's), TB a prefix-wide gradient, TS a k-channel slice,
    # a transition's output gradient or the stem pool's
    mid = max([N * H1 * W1 * c0, Ms[-1] * F] + [M * K4 for M in Ms])
    big = max(M * cend for M, (_, cend) in zip(Ms, widths))
    small = max([Ms[0] * max(k, c0)] + [M * cin for M, (cin, _) in zip(Ms, widths)])
    e.gbuf = [e._alloc16(mid) for _ in range(3)] + [e._alloc16(big), e._alloc16(small)]
    T0, T1, T2, TB, TS = [_ptr(t) for t in e.gbuf]
    if not implicit:
        e.cols = e._alloc16(Ms[0] * 9 * K4)
    COLS = _ptr(e.cols) if not implicit else None

    # ---- dropout masks (drawn at the head of the training forward) -------------------------------------------------------
    drop = e.drop_rate
    e.drop_masks = {}
    if drop > 0.0:
        for b in range(nblocks):
            for l in range(spec.block_config[b]):
                m = torch.ones(Ms[b], k, dtype=torch.float32, device=dev)
                e.drop_masks[lname(b, l)] = m
                e._masks.append((m, Ms[b] * k, 1, 1.0 - drop))

    # ---- forward: stem -------------------------------------------------------------------------------------
    bn0 = bns["features.norm0"]
    y0, a0 = e._alloc16(N, H1, W1, c0), e._alloc16(N, H1, W1, c0)
    fwd += e._stem_gemm("features.conv0.weight", c0, 7, 2, 3, y0, N * H1 * W1, bn0, rowpack=False)
    fwd += finalize(bn0, N * H1 * W1)
    fwd.append(("dfd_bn_act", (_ptr(y0), bn0.scale, bn0.shift, None, None, _ptr(a0), N, H1 * W1, c0, ACT_RELU, 0, dt)))
    e.pool_idx = torch.zeros(N * H2 * W2 * c0, dtype=torch.uint8, device=dev)
    p0 = e._alloc16(N, H2, W2, c0)
    fwd.append(("dfd_maxpool_fwd", (_ptr(a0), _ptr(p0), _ptr(e.pool_idx), N, H1, W1, c0, dt)))
    fwd.append(("dfd_copy_ld", (_ptr(p0), c0, _ptr(X[0]), widths[0][1], None, Ms[0], c0, dt) + slice_stats(0, 0)
                + (widths[0][1],)))
    e.acts["stem.out"] = p0

    # ---- forward: dense blocks and transitions --------------------------------------------------------------------------
    recs, trans = [], []
    for b, ((h, w), (cin, Ct)) in enumerate(zip(hw_b, widths)):
        M, x = Ms[b], X[b]
        layers = []
        for l in range(spec.block_config[b]):
            p, C = lname(b, l), cin + l * k
            n1, n2 = bns[p + ".norm1"], bns[p + ".norm2"]
            a1, y1, a2 = e._alloc16(M, C), e._alloc16(M, K4), e._alloc16(M, K4)
            fwd.append(fin_ld(n1, b, M))
            fwd.append(("dfd_bn_relu_ld", (_ptr(x), Ct, n1.scale, n1.shift, _ptr(a1), M, C, dt)))
            fwd.append(gemm(_ptr(a1), P16(p + ".conv1.weight"), _ptr(y1), M, K4, C, n2))
            fwd += finalize(n2, M)
            fwd.append(("dfd_bn_act", (_ptr(y1), n2.scale, n2.shift, None, None, _ptr(a2), N, h * w, K4, ACT_RELU, 0, dt)))
            wp = _ptr(e.wpack16, pk[p + ".conv2.weight"])
            mask = e.drop_masks.get(p)
            if implicit and mask is None:
                fwd.append(("dfd_conv3x3_narrow_tc", (_ptr(a2), wp, _ptr(x, C), N, h, w, K4, k, Ct, dt) + slice_stats(b, C)
                            + (Ct,)))
            else:
                if implicit:
                    fwd.append(("dfd_conv3x3_narrow_tc", (_ptr(a2), wp, TS, N, h, w, K4, k, k, dt, None, None, 0)))
                else:
                    fwd += [("dfd_im2col", (_ptr(a2), COLS, N, h, w, K4, 3, 1, 1, dt)), gemm(COLS, wp, TS, M, k, 9 * K4)]
                fwd.append(("dfd_copy_ld", (TS, k, _ptr(x, C), Ct, None if mask is None else ("TRAIN_ONLY", _ptr(mask)), M, k,
                                            dt) + slice_stats(b, C) + (Ct,)))
            layers.append(dict(p=p, C=C, n1=n1, n2=n2, a1=a1, y1=y1, a2=a2, mask=mask))
        recs.append(layers)
        if b + 1 < nblocks:
            tn = bns["features.transition%d.norm" % (b + 1)]
            ho, wo = hw_b[b + 1]
            Mo, Cn = Ms[b + 1], Ct // 2
            pt, yt = e._alloc16(N, ho, wo, Ct), e._alloc16(Mo, Cn)
            fwd.append(fin_ld(tn, b, M))
            fwd.append(("dfd_bn_relu_avgpool2", (_ptr(x), tn.scale, tn.shift, _ptr(pt), N, h, w, Ct, dt)))
            fwd.append(gemm(_ptr(pt), P16("features.transition%d.conv.weight" % (b + 1)), _ptr(yt), Mo, Cn, Ct))
            fwd.append(("dfd_copy_ld", (_ptr(yt), Cn, _ptr(X[b + 1]), widths[b + 1][1], None, Mo, Cn, dt) + slice_stats(b + 1, 0)
                        + (widths[b + 1][1],)))
            trans.append(dict(tn=tn, pt=pt))
        e.acts["denseblock%d" % (b + 1)] = x

    # ---- forward: norm5, F.relu, pool, dropout (densenet.py:130-138) ---------------------------------------------------------
    n5 = bns["features.norm5"]
    (Hf, Wf), Mf = hw_b[-1], Ms[-1]
    fwd.append(fin_ld(n5, nblocks - 1, Mf))
    fwd += e._pool_head(X[-1], n5, ACT_RELU, Hf * Wf, drop)

    # ---- backward ----------------------------------------------------------------------------------------
    bwd += e._pool_head_bwd(T0)
    bwd += bwd_finalize(n5, Mf)
    bwd.append(e._bn_apply(T0, X[-1], n5, _ptr(GX[-1]), Hf * Wf, F))
    for b in range(nblocks - 1, -1, -1):
        (h, w), (cin, Ct), M, x, gx = hw_b[b], widths[b], Ms[b], X[b], GX[b]
        for r in reversed(recs[b]):
            p, C, n1, n2 = r["p"], r["C"], r["n1"], r["n2"]
            name2 = p + ".conv2.weight"
            bwd.append(("dfd_copy_ld", (_ptr(gx, C), Ct, TS, k, None if r["mask"] is None else _ptr(r["mask"]), M, k, dt, None,
                                        None, 0)))
            bwd.append(("dfd_memset_async", (GPERM, 0, k * 9 * K4 * 4)))
            if implicit:
                bwd.append(("dfd_conv3x3_narrow_dgrad_tc", (TS, _ptr(e.wpackD16, pk[name2]), T0, N, h, w, K4, k, dt)))
                bwd.append(e._wgrad_conv(TS, _ptr(r["a2"]), GPERM, N, h, w, K4, k, 3))
            else:
                bwd += [gemm(TS, _ptr(e.wpackT16, pk[name2]), COLS, M, 9 * K4, k),
                        ("dfd_col2im", (COLS, None, T0, N, h, w, K4, 3, 1, 1, dt)),
                        ("dfd_im2col", (_ptr(r["a2"]), COLS, N, h, w, K4, 3, 1, 1, dt)),
                        e._wgrad(TS, COLS, GPERM, M, k, 9 * K4)]
            bwd.append(("dfd_act_bwd", (T0, _ptr(r["y1"]), n2.scale, n2.shift, n2.mean, n2.rstd, None, None, T1, N, h * w, K4,
                                        ACT_RELU, dt, n2.bs1, n2.bs2, None)))
            bwd += bwd_finalize(n2, M)
            bwd.append(e._bn_apply(T1, r["y1"], n2, T2, h * w, K4))
            bwd.append(gemm(T2, T16(p + ".conv1.weight"), TB, M, C, K4))
            bwd.append(e._wgrad(T2, _ptr(r["a1"]), G32(p + ".conv1.weight"), M, K4, C))
            bwd.append(("dfd_relu_bn_bwd_reduce_ld", (TB, _ptr(r["a1"]), _ptr(x), Ct, n1.mean, n1.rstd, M, C, dt, n1.bs1,
                                                      n1.bs2)))
            bwd += bwd_finalize(n1, M)
            bwd.append(("dfd_relu_bn_bwd_apply_add_ld", (TB, _ptr(r["a1"]), _ptr(x), Ct, n1.cA, n1.cB, n1.cC, _ptr(gx), Ct, M, C,
                                                         dt)))
            e._flush_reduce(bwd)
            bwd.append(("dfd_unpack_grad", (GPERM, G32(name2), k, K4, 3)))
        if b > 0:
            # the transition in front of this block: its output gradient is this block's channel prefix
            t = trans[b - 1]
            (hp, wp_), (_, Cp), Mp = hw_b[b - 1], widths[b - 1], Ms[b - 1]
            tw = "features.transition%d.conv.weight" % b
            bwd.append(("dfd_copy_ld", (_ptr(gx), Ct, TS, cin, None, M, cin, dt, None, None, 0)))
            bwd.append(gemm(TS, T16(tw), TB, M, Cp, cin))
            bwd.append(e._wgrad(TS, _ptr(t["pt"]), G32(tw), M, cin, Cp))
            tn = t["tn"]
            bwd.append(("dfd_bn_relu_avgpool2_bwd_reduce", (TB, _ptr(X[b - 1]), tn.scale, tn.shift, tn.mean, tn.rstd, N, hp, wp_,
                                                            Cp, dt, tn.bs1, tn.bs2)))
            bwd += bwd_finalize(tn, Mp)
            bwd.append(("dfd_bn_relu_avgpool2_bwd_apply", (TB, _ptr(X[b - 1]), tn.scale, tn.shift, tn.cA, tn.cB, tn.cC,
                                                           _ptr(GX[b - 1]), N, hp, wp_, Cp, dt)))
            e._flush_reduce(bwd)

    # ---- backward: stem -----------------------------------------------------------------------------------------------
    bwd.append(("dfd_copy_ld", (_ptr(GX[0]), widths[0][1], TS, c0, None, Ms[0], c0, dt, None, None, 0)))
    bwd.append(("dfd_maxpool_bwd", (TS, _ptr(e.pool_idx), T0, N, H1, W1, c0, dt)))
    bwd.append(("dfd_act_bwd", (T0, _ptr(y0), bn0.scale, bn0.shift, bn0.mean, bn0.rstd, None, None, T1, N, H1 * W1, c0,
                                ACT_RELU, dt, bn0.bs1, bn0.bs2, None)))
    bwd += bwd_finalize(bn0, N * H1 * W1)
    bwd.append(e._bn_apply(T1, y0, bn0, T0, H1 * W1, c0))
    bwd += e._stem_wgrad(T0)
    e._flush_reduce(bwd)
    bwd.append(e._stem_unpad())
    e._finish_plan(fwd, bwd)
