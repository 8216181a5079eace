"""Kernel plan of the dense ResNet family (resnet18/26/34/50/101/152, tv_*, wide_*, resnet26d / resnet50d) for `Engine` — host
side only.

Reference graph: dfd/timm/models/resnet.py:450-468 (stem 7x7 s2 -> BN -> ReLU -> maxpool 3x3 s2 -> 4 stages -> GAP
-> fc), BasicBlock :150-175, Bottleneck :215-246 (stride on the 3x3, :195-197; width = planes * base_width / 64, :187),
downsample 1x1 conv + BN :249-260.

ResNet-D (resnet26d, resnet50d): the deep stem (3x3 s2 -> BN -> ReLU -> 3x3 -> BN -> ReLU -> 3x3, :365-377) runs its first
convolution through the stem im2col + GEMM and the two 32-channel 3x3 convolutions through the explicit im2col route below;
the average-pool shortcut (downsample_avg, :263-277) pools with `dfd_avgpool2_fwd` in front of a stride-1 1x1 GEMM, and its
backward adds the pooled gradient into the main-path gradient in one pass (`dfd_avgpool2_bwd_add`).

With gemm_impl="tc" every 3x3 convolution runs as an IMPLICIT GEMM on wgmma (`dfd_conv_tc`, csrc/gemm_tc.cu conv mode: the
TMA producer fetches the input box shifted by the tap through a 4-D tensor map, no im2col matrix in memory), and so does the
strided 1x1 downsample. Stride-2 convolutions use the same kernels with TMA element strides {1, 2, 2, 1}. The input gradient of
a stride-1 3x3 is the same kernel on dY with the tap-flipped [Cin][kh'][kw'][Cout] weights; that of a strided 3x3 is four
parity-class implicit GEMMs (`dfd_conv_dgrad_s2_tc`) storing through strided views of dx. The weight gradient of every 3x3 and
of the strided downsample is the MN-major wgmma wgrad GEMM, implicit too (`dfd_conv_wgrad_tc`: one pipeline stage = one patch of
<= 64 output pixels of dY and the input box shifted by the tap). The downsample's input gradient is added into the main-path
gradient by the GEMM's own epilogue (`dfd_conv1x1_dgrad_add`).

With gemm_impl="mma" (the mma.sync cross-check path) the convolutions keep the explicit formulation (csrc/conv_dense.cu):
materialised im2col -> GEMM (forward and weight gradient), GEMM -> col2im (input gradient), and the strided downsample reads
a gathered copy of its input.

1x1 convolutions are plain GEMMs on the NHWC tensors. BN + ReLU outputs are materialised (`dfd_bn_act`) because three
consumers read them.

SE-ResNets (seresnet18/34/50/101/152, senet.py): the stem pool is MaxPool2d(3, 2, ceil_mode=True) without padding
(`dfd_maxpool_ceil_fwd` / `_bwd`); the bottleneck's stride sits on its 1x1 conv1 (the strided implicit GEMM of the downsample,
whose input gradient is added by `dfd_conv1x1_dgrad_add` into the zeroed block-input gradient together with the downsample's);
every block ends in an SEModule on its last BN output (after a ReLU in the basic block, senet.py:213-215): `dfd_pool_se_relu`
pools it and computes the gate [N, C] (training and eval), and the tail `dfd_bn_act` (gate, residual, ReLU) applies it.
Backward: `dfd_relu_se_bwd_reduce` forms the masked gradient gm of the block output, dL/dgate and the SE chain in one pass;
`dfd_act_bwd` (gate and dpool) forms the last BN's input gradient (gm * gate + dpool / HW) * act' with its BN-backward sums;
`dfd_se_fc_wgrad` the SE parameter gradients.
"""
import struct
from collections import OrderedDict
from functools import partial

import torch

from .arch import stem_pool_out
from .engine import ACT_NONE, ACT_RELU, POOL_CHUNKS, _ptr


def conv_out(h, k, s, p):
    return (h + 2 * p - k) // s + 1


# DropBlock of the reference ResNet: DropBlock2d(rate, 7, gamma_scale) behind every main-branch BatchNorm of layer3 (gamma_scale
# 0.25) and layer4 (1.0), resnet.py:386-387,403-404
DROP_BLOCK_SIZE = 7
DROP_BLOCK_GAMMA_SCALE = {"layer3": 0.25, "layer4": 1.0}
DROP_BLOCK_STREAM0 = 1 << 20        # generator stream ids of the DropBlock sites (dfd_rng_masks' tables count from 0)


def drop_block_geometry(name, H, W, rate, gamma_scale):
    """(gamma, clipped block size) of drop_block_2d (layers/drop.py:36-42) on an H x W map, in the reference's double
    arithmetic. The shapes on which the reference fails are refused: (W - 6)(H - 6) == 0 divides by zero, and an even clipped
    block size makes the pooled mask one pixel larger than the map."""
    cb = min(DROP_BLOCK_SIZE, min(W, H))
    den = (W - DROP_BLOCK_SIZE + 1) * (H - DROP_BLOCK_SIZE + 1)
    if den == 0:
        raise ValueError("DropBlock at %s (%dx%d): (W - %d) * (H - %d) == 0, the reference divides by zero"
                         % (name, H, W, DROP_BLOCK_SIZE - 1, DROP_BLOCK_SIZE - 1))
    if cb % 2 == 0:
        raise ValueError("DropBlock at %s (%dx%d): even block size %d, the reference's pooled mask does not match the map"
                         % (name, H, W, cb))
    return gamma_scale * rate * (W * H) / cb ** 2 / den, cb


def drop_block_desc(mask, noise, kept, gamma, N, H, W, C, cb, stream):
    """one 64-byte entry of the dfd_drop_block_masks table (pointers as integers, noise may be None)"""
    return struct.pack("<QQQdiiiiiiii", mask, noise or 0, kept, gamma, N, H, W, C, cb, stream, 0, 0)


def ds_names(b):
    """(conv weight, BN prefix) of a block's downsample branch, relative to the block: downsample_conv is [conv, BN]; downsample_avg
    is [pool, conv, BN] (resnet.py:249-277)"""
    return (".downsample.1.weight", ".downsample.2") if b.avg_down else (".downsample.0.weight", ".downsample.1")


def build_resnet(e):
    spec, N, dev, dt = e.spec, e.N, e.device, e.dt
    fwd, bwd = [], []

    # ---- packed (kh, kw, ci) copies of every k x k weight but the stem-GEMM weights ----------------------------------------
    pk = e._packed_weights([n for n in e.param_names if len(e.p_off[n][1]) == 4 and e.p_off[n][1][2] > 1
                            and n not in (spec.stem_conv + ".weight", "conv1.0.weight")])
    # two regions: a BasicBlock has two 3x3 convolutions whose packed gradients wait for the block's single ordered reduce
    gperm_max = max([e.p_off[n][2] for n in pk] + [8])
    e.gperm = torch.zeros(2 * gperm_max, dtype=torch.float32, device=dev)

    P32, G32, P16, T16 = e._p32, e._g32, e._p16, e._t16

    deep = spec.stem_type == "deep"
    sw = spec.stem_width
    stem_w, stem_bn = spec.stem_conv + ".weight", spec.stem_bn
    se = spec.se_reduction > 0
    if se and (e.drop_path_rate > 0.0 or (e.drop_block_rate or 0.0) > 0.0):
        raise ValueError("%s: the SE-ResNet has no drop path or DropBlock (SENet takes neither, senet.py:226-230)" % spec.arch)

    # ---- shapes ------------------------------------------------------------------------------------------
    if deep:
        H1, W1 = conv_out(e.H, 3, 2, 1), conv_out(e.W, 3, 2, 1)
    else:
        H1, W1 = conv_out(e.H, 7, 2, 3), conv_out(e.W, 7, 2, 3)
    H2, W2 = stem_pool_out(H1, spec.stem_pool), stem_pool_out(W1, spec.stem_pool)
    shapes = []
    h, w = H2, W2
    for b in spec.blocks:
        ho, wo = conv_out(h, 3, b.stride, 1), conv_out(w, 3, b.stride, 1)
        shapes.append((b, h, w, ho, wo))
        h, w = ho, wo
    Hf, Wf = h, w

    # ---- BN arenas ---------------------------------------------------------------------------------------
    bn_specs = ([("conv1.1", sw), ("conv1.4", sw)] if deep else []) + [(stem_bn, 64)]
    for b in spec.blocks:
        if b.kind == "basic":
            bn_specs += [(b.name + ".bn1", b.planes), (b.name + ".bn2", b.cout)]
        else:
            bn_specs += [(b.name + ".bn1", b.width), (b.name + ".bn2", b.width), (b.name + ".bn3", b.cout)]
        if b.downsample:
            bn_specs.append((b.name + ds_names(b)[1], b.cout))
    e._alloc_bn(bn_specs)
    bns = e.bns

    # no row-packed GEMMs: every ResNet K is >= 64 except the stem's Kp = 56 at in_chans = 1, which keeps the plain GEMM
    gemm = partial(e._gemm, rowpack=False)
    finalize, bwd_finalize = e._finalize, e._bwd_finalize

    implicit = e.gemm_impl == "tc"

    def conv3x3(xin, name, y, h, w, cin, cout, stride, bn):
        """3x3 / padding 1 forward into y (+ BatchNorm statistics of y)"""
        if implicit and cin % 64 == 0 and cout % 64 == 0:
            return [("dfd_conv_tc", (xin, _ptr(e.wpack16, pk[name]), y, N, h, w, cin, cout, 3, stride, dt) + e._stats(bn)
                     + (None,))]
        ho, wo = conv_out(h, 3, stride, 1), conv_out(w, 3, stride, 1)
        return [("dfd_im2col", (xin, COLS, N, h, w, cin, 3, stride, 1, dt)),
                gemm(COLS, _ptr(e.wpack16, pk[name]), y, N * ho * wo, cout, 9 * cin, bn)]

    # ---- stochastic regularisation (training only): DropBlock sites, drop-path gates, classifier dropout ---------------
    dp_rate, db_rate = e.drop_path_rate, e.drop_block_rate
    sites = OrderedDict()           # "<block>.bn<i>" -> (H, W, C, gamma, cb)
    if db_rate > 0.0:
        for b, h, w, ho, wo in shapes:
            gs = DROP_BLOCK_GAMMA_SCALE.get(b.name.split(".")[0])
            if gs is None:
                continue
            if b.kind == "basic":
                dims = [("bn1", ho, wo, b.planes), ("bn2", ho, wo, b.cout)]
            else:       # the stride is on conv2: bn1 runs at the block's input resolution
                dims = [("bn1", h, w, b.width), ("bn2", ho, wo, b.width), ("bn3", ho, wo, b.cout)]
            for bn_name, hh, ww, C in dims:
                name = b.name + "." + bn_name
                sites[name] = (hh, ww, C) + drop_block_geometry(name, hh, ww, db_rate, gs)
    e.drop_block_masks = OrderedDict()      # site -> (uint8 mask [N, H, W, C], int64 kept count [1])
    if sites:
        e.drop_block_kept = torch.zeros(len(sites), dtype=torch.int64, device=dev)
        raw = b""
        for si, (name, (hh, ww, C, gamma, cb)) in enumerate(sites.items()):
            m = torch.zeros(N, hh, ww, C, dtype=torch.uint8, device=dev)
            e.drop_block_masks[name] = (m, e.drop_block_kept[si:si + 1])
            raw += drop_block_desc(_ptr(m), None, _ptr(e.drop_block_kept, si), gamma, N, hh, ww, C, cb, DROP_BLOCK_STREAM0 + si)
        e._drop_block_table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
    e.drop_block_sites = sites
    e.drop_masks = OrderedDict()            # block -> drop-path gate [N, cout] (0 or 1 / keep per sample)
    if dp_rate > 0.0:
        for b in spec.blocks:               # one DropPath(drop_path_rate) shared by every block, resnet.py:385
            gate = torch.ones(N, b.cout, dtype=torch.float32, device=dev)
            e.drop_masks[b.name] = gate
            e._masks.append((gate, N, b.cout, 1.0 - dp_rate))

    def site_args(name):
        """(mask, kept, numel) operands of a DropBlock site"""
        m, k = e.drop_block_masks[name]
        return _ptr(m), _ptr(k), m.numel()

    def bn_relu(y, bn, out, hw, C, site=None):
        if site in sites:
            m, k, numel = site_args(site)
            return ("dfd_bn_act_drop", [_ptr(y), bn.scale, bn.shift, ("TRAIN_ONLY", m), k, numel, None, None, _ptr(out), N, hw, C,
                                        0, dt])
        return ("dfd_bn_act", (_ptr(y), bn.scale, bn.shift, None, None, _ptr(out), N, hw, C, ACT_RELU, 0, dt))

    # ---- scratch -----------------------------------------------------------------------------------------
    max_act = max([N * H1 * W1 * 64] + [N * hh * ww * max(b.cin, b.width) for b, hh, ww, ho, wo in shapes] +
                  [N * ho * wo * b.cout for b, hh, ww, ho, wo in shapes])
    max_cols = max([N * ho * wo * 9 * (b.cin if b.kind == "basic" else b.width) for b, hh, ww, ho, wo in shapes] +
                   [N * ho * wo * 9 * b.width for b, hh, ww, ho, wo in shapes] + ([N * H1 * W1 * 9 * sw] if deep else []))
    e.gbuf = [e._alloc16(max_act) for _ in range(6)]
    e.cols = e._alloc16(max_cols)
    COLS = _ptr(e.cols)
    gA, gB, gC, gD, gE, gF = [_ptr(t) for t in e.gbuf]

    # ---- forward -----------------------------------------------------------------------------------------
    y0 = e._alloc16(N, H1, W1, 64)
    a0 = e._alloc16(N, H1, W1, 64)
    x0 = e._alloc16(N, H2, W2, 64)
    e.pool_idx = torch.zeros(N * H2 * W2 * 64, dtype=torch.uint8, device=dev)
    bn0 = bns[stem_bn]
    if deep:
        # conv1.0 (3x3 s2, in_chans -> sw) as im2col + GEMM, conv1.3 / conv1.6 (Cin = sw) through conv3x3's im2col route
        bs0, bs1 = bns["conv1.1"], bns["conv1.4"]
        ys0, as0 = e._alloc16(N, H1, W1, sw), e._alloc16(N, H1, W1, sw)
        ys1, as1 = e._alloc16(N, H1, W1, sw), e._alloc16(N, H1, W1, sw)
        fwd += e._stem_gemm("conv1.0.weight", sw, 3, 2, 1, ys0, N * H1 * W1, bs0, rowpack=False)
        fwd += finalize(bs0, N * H1 * W1)
        fwd.append(bn_relu(ys0, bs0, as0, H1 * W1, sw))
        fwd += conv3x3(_ptr(as0), "conv1.3.weight", _ptr(ys1), H1, W1, sw, sw, 1, bs1)
        fwd += finalize(bs1, N * H1 * W1)
        fwd.append(bn_relu(ys1, bs1, as1, H1 * W1, sw))
        fwd += conv3x3(_ptr(as1), "conv1.6.weight", _ptr(y0), H1, W1, sw, 64, 1, bn0)
    else:
        fwd += e._stem_gemm(stem_w, 64, 7, 2, 3, y0, N * H1 * W1, bn0, rowpack=False)
    fwd += finalize(bn0, N * H1 * W1)
    fwd.append(bn_relu(y0, bn0, a0, H1 * W1, 64))
    pool_op = "dfd_maxpool_ceil" if spec.stem_pool == "ceil" else "dfd_maxpool"
    fwd.append((pool_op + "_fwd", (_ptr(a0), _ptr(x0), _ptr(e.pool_idx), N, H1, W1, 64, dt)))
    e.acts["stem.out"] = x0
    x = x0
    recs = []
    if se:
        # per-image SE vectors of the backward, shared by the blocks (consumed within the block): dL/dgate, d_e, dpool [N, C];
        # r, d_rpre [N, Cse]
        cmax, rmax = max(b.cout for b in spec.blocks), max(b.cse for b in spec.blocks)
        e.se_tmp = torch.zeros(3 * N * cmax + 2 * N * rmax, dtype=torch.float32, device=dev)
        se_draw, se_de, se_dpool = [_ptr(e.se_tmp, i * N * cmax) for i in range(3)]
        se_r, se_drp = _ptr(e.se_tmp, 3 * N * cmax), _ptr(e.se_tmp, 3 * N * cmax + N * rmax)
    for b, h, w, ho, wo in shapes:
        p = b.name
        M1, M2 = N * h * w, N * ho * wo
        rec = dict(b=b, h=h, w=w, ho=ho, wo=wo, x=x)
        if b.kind == "basic":
            bn1, bn2 = bns[p + ".bn1"], bns[p + ".bn2"]
            y1 = e._alloc16(N, ho, wo, b.planes)
            a1 = e._alloc16(N, ho, wo, b.planes)
            y2 = e._alloc16(N, ho, wo, b.cout)
            fwd += conv3x3(_ptr(x), p + ".conv1.weight", _ptr(y1), h, w, b.cin, b.planes, b.stride, bn1)
            fwd += finalize(bn1, M2)
            fwd.append(bn_relu(y1, bn1, a1, ho * wo, b.planes, p + ".bn1"))
            fwd += conv3x3(_ptr(a1), p + ".conv2.weight", _ptr(y2), ho, wo, b.planes, b.cout, 1, bn2)
            fwd += finalize(bn2, M2)
            rec.update(y1=y1, a1=a1, ylast=y2, bnlast=bn2, site_last=p + ".bn2")
        else:
            bn1, bn2, bn3 = bns[p + ".bn1"], bns[p + ".bn2"], bns[p + ".bn3"]
            # SE-ResNet bottleneck: the stride on the 1x1 conv1, conv2 at stride 1 (senet.py:141-163)
            s1x1 = spec.stride_in_1x1 and b.stride != 1
            h1, w1 = (ho, wo) if s1x1 else (h, w)
            M1b = N * h1 * w1
            y1 = e._alloc16(N, h1, w1, b.width)
            a1 = e._alloc16(N, h1, w1, b.width)
            y2 = e._alloc16(N, ho, wo, b.width)
            a2 = e._alloc16(N, ho, wo, b.width)
            y3 = e._alloc16(N, ho, wo, b.cout)
            xs1 = None
            if not s1x1:
                fwd.append(gemm(_ptr(x), P16(p + ".conv1.weight"), _ptr(y1), M1, b.width, b.cin, bn1))
            elif implicit and b.cin % 64 == 0 and b.width % 64 == 0:
                # strided 1x1 straight from the block input, as the downsample below
                fwd.append(("dfd_conv_tc", (_ptr(x), P16(p + ".conv1.weight"), _ptr(y1), N, h, w, b.cin, b.width, 1, b.stride, dt)
                            + e._stats(bn1) + (None,)))
            else:
                xs1 = e._alloc16(N, ho, wo, b.cin)
                fwd.append(("dfd_im2col", (_ptr(x), _ptr(xs1), N, h, w, b.cin, 1, b.stride, 0, dt)))
                fwd.append(gemm(_ptr(xs1), P16(p + ".conv1.weight"), _ptr(y1), M2, b.width, b.cin, bn1))
            fwd += finalize(bn1, M1b)
            fwd.append(bn_relu(y1, bn1, a1, h1 * w1, b.width, p + ".bn1"))
            fwd += conv3x3(_ptr(a1), p + ".conv2.weight", _ptr(y2), h1, w1, b.width, b.width, 1 if s1x1 else b.stride, bn2)
            fwd += finalize(bn2, M2)
            fwd.append(bn_relu(y2, bn2, a2, ho * wo, b.width, p + ".bn2"))
            fwd.append(gemm(_ptr(a2), P16(p + ".conv3.weight"), _ptr(y3), M2, b.cout, b.width, bn3))
            fwd += finalize(bn3, M2)
            rec.update(y1=y1, a1=a1, y2=y2, a2=a2, ylast=y3, bnlast=bn3, site_last=p + ".bn3", s1x1=s1x1, xs1=xs1)
        res = x
        if b.downsample:
            dsw, dsbn = [p + n for n in ds_names(b)]
            bnd = bns[dsbn]
            yd = e._alloc16(N, ho, wo, b.cout)
            r = e._alloc16(N, ho, wo, b.cout)
            if b.stride == 1:
                xs = x
                fwd.append(gemm(_ptr(xs), P16(dsw), _ptr(yd), M2, b.cout, b.cin, bnd))
            elif b.avg_down:
                # ResNet-D: 2x2 average pool (ceil_mode, count_include_pad=False), then the stride-1 1x1 convolution; the pooled
                # input is kept for the weight gradient
                xs = e._alloc16(N, ho, wo, b.cin)
                fwd.append(("dfd_avgpool2_fwd", (_ptr(x), _ptr(xs), N, h, w, b.cin, dt)))
                fwd.append(gemm(_ptr(xs), P16(dsw), _ptr(yd), M2, b.cout, b.cin, bnd))
            elif implicit and b.cin % 64 == 0 and b.cout % 64 == 0:
                # strided 1x1 convolution straight from the block input (k = 1, stride 2 implicit GEMM): no gathered copy
                xs = None
                fwd.append(("dfd_conv_tc", (_ptr(x), P16(dsw), _ptr(yd), N, h, w, b.cin, b.cout, 1, b.stride, dt)
                            + e._stats(bnd) + (None,)))
            else:
                xs = e._alloc16(N, ho, wo, b.cin)
                fwd.append(("dfd_im2col", (_ptr(x), _ptr(xs), N, h, w, b.cin, 1, b.stride, 0, dt)))
                fwd.append(gemm(_ptr(xs), P16(dsw), _ptr(yd), M2, b.cout, b.cin, bnd))
            fwd += finalize(bnd, M2)
            fwd.append(("dfd_bn_act", (_ptr(yd), bnd.scale, bnd.shift, None, None, _ptr(r), N, ho * wo, b.cout, ACT_NONE, 0, dt)))
            rec.update(yd=yd, xs=xs, bnd=bnd, dsw=dsw)
            res = r
        out = e._alloc16(N, ho, wo, b.cout)
        bl = rec["bnlast"]
        gate = e.drop_masks.get(p)
        rec["gate"] = gate
        if b.cse:
            # SEModule on the last BN output: pooled [N, C] and the gate [N, C], in eval plans too
            sep = p + ".se_module."
            pooled = torch.zeros(N, b.cout, dtype=torch.float32, device=dev)
            sgate = torch.zeros(N, b.cout, dtype=torch.float32, device=dev)
            e._keep += [pooled, sgate]
            rec.update(se_pooled=pooled, se_gate=sgate, se_w=[sep + n for n in ("fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias")])
            # the SE input: the bare bn3 output of a bottleneck, ReLU(bn2) of a basic block (senet.py:94-114, 206-223)
            se_act = ACT_RELU if b.kind == "basic" else ACT_NONE
            rec["se_act"] = se_act
            fwd.append(("dfd_pool_se_relu", (_ptr(rec["ylast"]), bl.scale, bl.shift, _ptr(pooled))
                        + tuple(P32(n) for n in rec["se_w"]) + (_ptr(sgate), N, ho * wo, b.cout, b.cse, se_act, dt, POOL_CHUNKS)))
            fwd.append(("dfd_bn_act", (_ptr(rec["ylast"]), bl.scale, bl.shift, _ptr(sgate), _ptr(res), _ptr(out), N, ho * wo,
                                       b.cout, se_act, 2, dt)))
        elif rec["site_last"] in sites:
            m, k, numel = site_args(rec["site_last"])
            fwd.append(("dfd_bn_act_drop", [_ptr(rec["ylast"]), bl.scale, bl.shift, ("TRAIN_ONLY", m), k, numel,
                                            ("TRAIN_ONLY", _ptr(gate)) if gate is not None else None, _ptr(res), _ptr(out), N,
                                            ho * wo, b.cout, 2, dt]))
        elif gate is not None:
            fwd.append(("dfd_bn_act", [_ptr(rec["ylast"]), bl.scale, bl.shift, ("TRAIN_ONLY", _ptr(gate)), _ptr(res), _ptr(out),
                                       N, ho * wo, b.cout, ACT_NONE, 2, dt]))
        else:
            fwd.append(("dfd_bn_act", (_ptr(rec["ylast"]), bl.scale, bl.shift, None, _ptr(res), _ptr(out), N, ho * wo, b.cout,
                                       ACT_NONE, 2, dt)))
        e.acts[p + ".out"] = out
        rec["out"] = out
        recs.append(rec)
        x = out
    e.pool_partial = torch.zeros(8 * N * spec.num_features, dtype=torch.float32, device=dev)
    # global pool, then F.dropout on the pooled vector before fc (resnet.py:465-466)
    fwd += e._pool_head(x, None, ACT_NONE, Hf * Wf, e.drop_rate, partial=_ptr(e.pool_partial))

    # ---- backward ----------------------------------------------------------------------------------------
    pending_unpack = []         # (gperm region pointer, name, Cout, Cin): unpacked after the block's ordered reduce

    def zero_gperm(ptr, numel):
        return ("dfd_memset_async", (ptr, 0, numel * 4))

    def flush_block(ops):
        """ONE ordered reduce per block (every weight gradient of the block), then the packed 3x3 gradients -> OIHW arena"""
        e._flush_reduce(ops)
        for gp, name, Cout, Cin in pending_unpack:
            ops.append(("dfd_unpack_grad", (gp, G32(name), Cout, Cin, 3)))
        del pending_unpack[:]

    def conv3x3_bwd(name, dy, M_out, Cin, Cout, xin_t, n_h, n_w, stride, dx_out, dx_add=None):
        """dy [M_out, Cout] -> dx_out [N, n_h, n_w, Cin] (+dx_add) and the weight gradient of `name`"""
        if implicit and stride == 1 and dx_add is None and Cin % 64 == 0 and Cout % 64 == 0:
            # input gradient = the same implicit GEMM on dY with the tap-flipped [Cin][kh'][kw'][Cout] weights
            ops = [("dfd_conv_tc", (dy, _ptr(e.wpackD16, pk[name]), dx_out, N, n_h, n_w, Cout, Cin, 3, 1, dt, None, None, None))]
        elif implicit and stride == 2 and dx_add is None and Cin % 64 == 0 and Cout % 64 == 0:
            # strided input gradient: four parity-class implicit GEMMs storing through strided views of dx
            ops = [("dfd_conv_dgrad_s2_tc", (dy, _ptr(e.wpackD16, pk[name]), dx_out, N, n_h, n_w, Cin, Cout, dt))]
        else:
            ops = [gemm(dy, _ptr(e.wpackT16, pk[name]), COLS, M_out, 9 * Cin, Cout),
                   ("dfd_col2im", (COLS, dx_add, dx_out, N, n_h, n_w, Cin, 3, stride, 1, dt))]
        gp = _ptr(e.gperm, len(pending_unpack) * gperm_max)         # this block's next free region
        assert len(pending_unpack) < 2
        if implicit and Cin % 64 == 0:
            ops += [zero_gperm(gp, Cout * 9 * Cin),
                    e._wgrad_conv(dy, _ptr(xin_t), gp, N, n_h, n_w, Cin, Cout, 3, stride)]
        else:
            ops += [("dfd_im2col", (_ptr(xin_t), COLS, N, n_h, n_w, Cin, 3, stride, 1, dt)),
                    zero_gperm(gp, Cout * 9 * Cin),
                    e._wgrad(dy, COLS, gp, M_out, Cout, 9 * Cin)]
        pending_unpack.append((gp, name, Cout, Cin))     # complete after the block's ordered reduce (flush_block)
        return ops

    bwd += e._pool_head_bwd(gA)
    # The gradient entering a block is kept as up to TWO tensors (main-path dx + identity-path gm of the block above): the
    # fused ReLU / BN-backward reduction adds them on the fly (dfd_relu_bn_bwd_reduce), which removes the materialised
    # residual add of every block without a downsample branch.
    def relu_bwd(da, y, bn, gu, hw, C, site):
        """gradient through BN output -> (DropBlock) -> ReLU, plus the BN backward sums"""
        if site in sites:
            m, k, numel = site_args(site)
            return ("dfd_act_bwd_drop", (da, _ptr(y), bn.scale, bn.shift, bn.mean, bn.rstd, m, k, numel, gu, N, hw, C, dt,
                                         bn.bs1, bn.bs2))
        return ("dfd_act_bwd", (da, _ptr(y), bn.scale, bn.shift, bn.mean, bn.rstd, None, None, gu, N, hw, C, ACT_RELU, dt,
                                bn.bs1, bn.bs2, None))

    bufs = [gA, gB, gC, gD, gE, gF]
    dout, dout2 = gA, None
    for rec in reversed(recs):
        b, h, w, ho, wo, xin = rec["b"], rec["h"], rec["w"], rec["ho"], rec["wo"], rec["x"]
        p = b.name
        M1, M2 = N * h * w, N * ho * wo
        gm, t1, t2, t3 = [g for g in bufs if g not in (dout, dout2)][:4]
        bl = rec["bnlast"]
        if b.cse:
            # gm = (dout + dout2) * (out > 0) stored, dL/dgate and the SE backward chain in one pass; then the last BN's input
            # gradient (gm * gate + dpool / HW) * act' (with its BN-backward sums) in t2 and the SE parameter gradients
            Wr, br, We, be = rec["se_w"]
            bwd.append(("dfd_relu_se_bwd_reduce", (dout, dout2, _ptr(rec["ylast"]), _ptr(rec["out"]), bl.scale, bl.shift, gm, se_draw,
                                                   _ptr(rec["se_pooled"]), P32(Wr), P32(br), P32(We), P32(be), se_de, se_r, se_drp,
                                                   se_dpool, N, ho * wo, b.cout, b.cse, rec["se_act"], dt)))
            bwd.append(("dfd_act_bwd", (gm, _ptr(rec["ylast"]), bl.scale, bl.shift, bl.mean, bl.rstd, _ptr(rec["se_gate"]), se_dpool,
                                        t2, N, ho * wo, b.cout, rec["se_act"], dt, bl.bs1, bl.bs2, None)))
            bwd.append(("dfd_se_fc_wgrad", (se_de, se_r, se_drp, _ptr(rec["se_pooled"]), G32(Wr), G32(br), G32(We), G32(be), N,
                                            b.cout, b.cse)))
        elif rec["site_last"] in sites or rec["gate"] is not None:
            # gm goes unmasked to the identity / downsample path; the last BN sees gd = gm * (DropBlock) * (drop path) in t2
            m, k, numel = site_args(rec["site_last"]) if rec["site_last"] in sites else (None, None, 0)
            gate = _ptr(rec["gate"]) if rec["gate"] is not None else None
            bwd.append(("dfd_relu_bn_bwd_reduce_drop", (dout, dout2, _ptr(rec["ylast"]), _ptr(rec["out"]), gm, m, k, numel, gate, t2,
                                                        bl.mean, bl.rstd, N, ho * wo, b.cout, dt, bl.bs1, bl.bs2)))
        else:
            # gm = (dout + dout2) * (out > 0) is produced by the reduction itself (one pass over the block output instead of
            # the residual add, the ReLU backward and the reduction)
            bwd.append(("dfd_relu_bn_bwd_reduce", (dout, dout2, _ptr(rec["ylast"]), _ptr(rec["out"]), gm, bl.mean, bl.rstd, N, ho * wo,
                                                   b.cout, dt, bl.bs1, bl.bs2)))
        gd = t2 if (b.cse or rec["site_last"] in sites or rec["gate"] is not None) else gm
        bwd += bwd_finalize(bl, M2)
        bwd.append(e._bn_apply(gd, rec["ylast"], bl, t1, ho * wo, b.cout))
        if b.kind == "basic":
            bn1 = bns[p + ".bn1"]
            # conv2 (3x3 s1): dy2 = t1 -> da1 = t2
            bwd += conv3x3_bwd(p + ".conv2.weight", t1, M2, b.planes, b.cout, rec["a1"], ho, wo, 1, t2)
            bwd.append(relu_bwd(t2, rec["y1"], bn1, t1, ho * wo, b.planes, p + ".bn1"))
            bwd += bwd_finalize(bn1, M2)
            bwd.append(e._bn_apply(t1, rec["y1"], bn1, t2, ho * wo, b.planes))
            # conv1 (3x3 stride s): dy1 = t2 -> dx = t3 [M1, cin]
            bwd += conv3x3_bwd(p + ".conv1.weight", t2, M2, b.cin, b.planes, xin, h, w, b.stride, t3)
        else:
            bn1, bn2 = bns[p + ".bn1"], bns[p + ".bn2"]
            # conv3 (1x1): dy3 = t1 -> da2 = t2
            bwd.append(gemm(t1, T16(p + ".conv3.weight"), t2, M2, b.width, b.cout))
            bwd.append(e._wgrad(t1, _ptr(rec["a2"]), G32(p + ".conv3.weight"), M2, b.cout, b.width))
            bwd.append(relu_bwd(t2, rec["y2"], bn2, t1, ho * wo, b.width, p + ".bn2"))
            bwd += bwd_finalize(bn2, M2)
            bwd.append(e._bn_apply(t1, rec["y2"], bn2, t2, ho * wo, b.width))
            s1x1 = rec["s1x1"]
            h1, w1 = (ho, wo) if s1x1 else (h, w)
            M1b = N * h1 * w1
            # conv2 (3x3 stride s, or 1 when the stride is on conv1): dy2 = t2 -> da1 = t1 [M1b, width]
            bwd += conv3x3_bwd(p + ".conv2.weight", t2, M2, b.width, b.width, rec["a1"], h1, w1, 1 if s1x1 else b.stride, t1)
            bwd.append(relu_bwd(t1, rec["y1"], bn1, t2, h1 * w1, b.width, p + ".bn1"))
            bwd += bwd_finalize(bn1, M1b)
            bwd.append(e._bn_apply(t2, rec["y1"], bn1, t1, h1 * w1, b.width))
            c1 = p + ".conv1.weight"
            if not s1x1:
                # conv1 (1x1): dy1 = t1 -> dx = t3 [M1, cin]
                bwd.append(gemm(t1, T16(c1), t3, M1, b.cin, b.width))
                bwd.append(e._wgrad(t1, _ptr(xin), G32(c1), M1, b.width, b.cin))
            elif rec["xs1"] is None:
                # strided 1x1 conv1: its input gradient only reaches the stride-2 pixels, added into the zeroed t3 (the downsample's
                # gradient is added into the same buffer below)
                bwd.append(("dfd_memset_async", (t3, 0, M1 * b.cin * e.gbuf[0].element_size())))
                bwd.append(("dfd_conv1x1_dgrad_add", (t1, T16(c1), t3, N, h, w, b.cin, b.width, b.stride, dt)))
                bwd.append(e._wgrad_conv(t1, _ptr(xin), G32(c1), N, h, w, b.cin, b.width, 1, b.stride))
            else:
                # explicit formulation: the gradient of the gathered input, scattered onto the input grid (zeros elsewhere)
                bwd.append(gemm(t1, T16(c1), t2, M2, b.cin, b.width))
                bwd.append(("dfd_col2im", (t2, None, t3, N, h, w, b.cin, 1, b.stride, 0, dt)))
                bwd.append(e._wgrad(t1, _ptr(rec["xs1"]), G32(c1), M2, b.width, b.cin))
        # identity / downsample path: gradient gm flows to the block input too
        if b.downsample:
            bnd = rec["bnd"]
            bwd.append(("dfd_bn_bwd_reduce", (gm, _ptr(rec["yd"]), None, bnd.mean, bnd.rstd, N, ho * wo, b.cout, dt, bnd.bs1, bnd.bs2, None)))
            bwd += bwd_finalize(bnd, M2)
            bwd.append(e._bn_apply(gm, rec["yd"], bnd, t1, ho * wo, b.cout))
            pooled = b.avg_down and b.stride != 1
            ds_add = implicit and b.cin % 64 == 0 and b.cout % 64 == 0 and not pooled
            dsw = rec["dsw"]
            if ds_add:
                # the downsample input gradient is ADDED into t3 (main-path gradient) by the GEMM's own epilogue: a TMA reduction
                # store through the stride-s pixel view of t3 - no scratch tensor, no col2im scatter / add pass
                bwd.append(("dfd_conv1x1_dgrad_add", (t1, T16(dsw), t3, N, h, w, b.cin, b.cout, b.stride, dt)))
            else:
                bwd.append(gemm(t1, T16(dsw), t2, M2, b.cin, b.cout))
            if rec["xs"] is None:      # strided 1x1: implicit weight gradient on the block input itself
                bwd.append(e._wgrad_conv(t1, _ptr(xin), G32(dsw), N, h, w, b.cin, b.cout, 1, b.stride))
            else:
                bwd.append(e._wgrad(t1, _ptr(rec["xs"]), G32(dsw), M2, b.cout, b.cin))
            if ds_add:
                new_dout = (t3, None)
            elif b.stride == 1:
                bwd.append(("dfd_add_inplace", (t3, t2, M1 * b.cin, dt)))
                new_dout = (t3, None)
            elif pooled:
                # spread the pooled gradient over each 2x2 window (/ its in-image count) and add the main-path gradient, into the
                # old dout buffer (consumed by the reduction above)
                bwd.append(("dfd_avgpool2_bwd_add", (t2, t3, dout, N, h, w, b.cin, dt)))
                new_dout = (dout, None)
            else:
                # scatter the strided gradient back onto the input grid and add the main-path gradient (the old dout buffer
                # has been consumed by the reduction above: reused as the destination)
                bwd.append(("dfd_col2im", (t2, t3, dout, N, h, w, b.cin, 1, b.stride, 0, dt)))
                new_dout = (dout, None)
        else:
            new_dout = (t3, gm)             # the block below adds them while it masks and reduces
        flush_block(bwd)
        dout, dout2 = new_dout
    # stem: maxpool -> relu/bn1 -> conv1 wgrad
    if dout2 is not None:
        bwd.append(("dfd_add_inplace", (dout, dout2, N * H2 * W2 * 64, dt)))
    t1, t2 = [g for g in bufs if g != dout][:2]
    bwd.append((pool_op + "_bwd", (dout, _ptr(e.pool_idx), t1, N, H1, W1, 64, dt)))
    bwd.append(("dfd_act_bwd", (t1, _ptr(y0), bn0.scale, bn0.shift, bn0.mean, bn0.rstd, None, None, t2, N, H1 * W1, 64,
                                ACT_RELU, dt, bn0.bs1, bn0.bs2, None)))
    bwd += bwd_finalize(bn0, N * H1 * W1)
    bwd.append(e._bn_apply(t2, y0, bn0, t1, H1 * W1, 64))
    if deep:
        # conv1.6 and conv1.3 take the two packed-gradient regions; conv1.0's gradient goes through the padded stem buffer.
        M0 = N * H1 * W1
        bwd += conv3x3_bwd("conv1.6.weight", t1, M0, sw, 64, as1, H1, W1, 1, t2)
        bwd.append(relu_bwd(t2, ys1, bs1, t1, H1 * W1, sw, None))
        bwd += bwd_finalize(bs1, M0)
        bwd.append(e._bn_apply(t1, ys1, bs1, t2, H1 * W1, sw))
        bwd += conv3x3_bwd("conv1.3.weight", t2, M0, sw, sw, as0, H1, W1, 1, t1)
        bwd.append(relu_bwd(t1, ys0, bs0, t2, H1 * W1, sw, None))
        bwd += bwd_finalize(bs0, M0)
        bwd.append(e._bn_apply(t2, ys0, bs0, t1, H1 * W1, sw))
    bwd += e._stem_wgrad(t1)
    flush_block(bwd)            # one ordered reduce for the stem's weight gradients, then the unpack / unpad passes
    bwd.append(e._stem_unpad())
    e._finish_plan(fwd, bwd, len(sites))
