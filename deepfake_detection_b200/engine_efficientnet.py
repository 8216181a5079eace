"""Kernel plan of the EfficientNet family (efficientnet_b*, tf_efficientnet_b*, efficientnet_deepfake_v4) for `Engine` —
host side only.

Stem 3x3 s2 -> BN -> Swish -> MBConv blocks (depthwise-separable and inverted-residual, squeeze-excite, drop path) ->
1x1 head conv -> BN -> Swish -> global pool -> (dropout) -> classifier. Pointwise convolutions are tensor-core GEMMs on the
NHWC tensors, the depthwise convolutions and their fused backward are `dfd_dwconv_*`, and the BatchNorm + activation of
each conv output is folded into the kernel that consumes it, except where `dfd_bn_act` materialises it.
"""
from collections import OrderedDict

import torch

from . import _lib
from .arch import conv_pads
from .engine import ACT_NONE, ACT_SWISH, POOL_CHUNKS, _ptr


def build_efficientnet(e):
    spec, N, dev, dt = e.spec, e.N, e.device, e.dt
    e._keep = []
    e.acts = {}
    fwd, bwd = [], []

    # ---- pass 1: shapes --------------------------------------------------------------------
    Hs = (e.H + 2 - 3) // 2 + 1
    Ws = (e.W + 2 - 3) // 2 + 1
    blocks = []
    h, w = Hs, Ws
    for b in spec.blocks:
        ho = (h + 2 * b.pad - b.k) // b.stride + 1
        wo = (w + 2 * b.pad - b.k) // b.stride + 1
        blocks.append((b, h, w, ho, wo))
        h, w = ho, wo
    Hf, Wf = h, w
    # (top, left) pad of the stem and of every depthwise conv at this plan's extents. TF "SAME" padding (pad_type
    # 'same') is one short on the begin side of a stride-2 layer over an even extent; only such layers are planned
    # through the `_pad` kernels, every other layer issues exactly the launches of the symmetric models
    e.conv_pads = conv_pads(spec, e.H, e.W)
    pads = {name: (pt, pl) for name, k, s_, h_, w_, pt, pl, ho_, wo_ in e.conv_pads}
    asym = lambda name, k: pads[name] != ((k - 1) // 2, (k - 1) // 2)
    if asym("conv_stem", 3) and e.stem_impl != "gemm":
        raise ValueError("stem_impl=%r: TF 'SAME' padding of the stem is planned through dfd_stem_im2col_pad (stem_impl='gemm')"
                         % (e.stem_impl,))

    # ---- BN bookkeeping arenas ---------------------------------------------------------------
    bn_specs = [("bn1", spec.stem)]
    for b in spec.blocks:
        if b.kind == "ir":
            bn_specs += [(b.name + ".bn1", b.cmid), (b.name + ".bn2", b.cmid), (b.name + ".bn3", b.cout)]
        else:
            bn_specs += [(b.name + ".bn1", b.cmid), (b.name + ".bn2", b.cout)]
    bn_specs.append(("bn2", spec.num_features))
    e._alloc_bn(bn_specs)

    P32 = lambda n: _ptr(e.params32, e.p_off[n][0])
    G32 = lambda n: _ptr(e.grads32, e.p_off[n][0])
    P16 = lambda n: _ptr(e.params16, e.p_off[n][0])
    T16 = lambda n: _ptr(e.paramsT16, e.t_off[n][0])
    gemm, finalize, bwd_finalize = e._gemm, e._finalize, e._bwd_finalize

    # ---- scratch for backward ----------------------------------------------------------------
    mid_max = max([N * h * w * b.cmid for b, h, w, ho, wo in blocks if b.kind == "ir"] +
                  [N * ho * wo * b.cmid for b, h, w, ho, wo in blocks] + [N * Hf * Wf * spec.num_features] +
                  [N * Hs * Ws * spec.stem])
    small_max = max([N * h * w * b.cin for b, h, w, ho, wo in blocks] +
                    [N * ho * wo * b.cout for b, h, w, ho, wo in blocks])
    e.mid = [e._alloc16(mid_max) for _ in range(2)]
    e.small = [e._alloc16(small_max) for _ in range(3)]
    mid_a, mid_b = _ptr(e.mid[0]), _ptr(e.mid[1])
    sm = [_ptr(t) for t in e.small]
    se_max_c = max([b.cmid for b in spec.blocks if b.cse] + [8])
    se_max_r = max([b.cse for b in spec.blocks if b.cse] + [8])
    e.se_tmp = torch.zeros(3 * N * se_max_c + 2 * N * se_max_r, dtype=torch.float32, device=dev)
    se_draw = _ptr(e.se_tmp)
    e.pool_partial = torch.zeros(POOL_CHUNKS * N * max(se_max_c, spec.num_features), dtype=torch.float32, device=dev)
    se_de = _ptr(e.se_tmp, N * se_max_c)
    se_dpool = _ptr(e.se_tmp, 2 * N * se_max_c)
    se_r = _ptr(e.se_tmp, 3 * N * se_max_c)
    se_drp = _ptr(e.se_tmp, 3 * N * se_max_c + N * se_max_r)

    # ---- forward -----------------------------------------------------------------------------
    e.x_in = torch.zeros(N, spec.in_chans, e.H, e.W, dtype=e.tdtype, device=dev)
    y0 = e._alloc16(N, Hs, Ws, spec.stem)
    stem_out = e._alloc16(N, Hs, Ws, spec.stem)
    e.acts["conv_stem"] = y0
    e.acts["stem.out"] = stem_out
    bn = e.bns["bn1"]
    if e.stem_impl == "gemm":
        taps, Kp = e._stem_gemm_setup("conv_stem.weight", spec.stem, 3, N * Hs * Ws)
        if asym("conv_stem", 3):
            fwd.append(("dfd_stem_im2col_pad", (_ptr(e.x_in), _ptr(e.stem_cols), N, spec.in_chans, e.H, e.W, 3, 2)
                        + pads["conv_stem"] + (Kp, dt)))
        else:
            fwd.append(("dfd_stem_im2col", (_ptr(e.x_in), _ptr(e.stem_cols), N, spec.in_chans, e.H, e.W, 3, 2, 1, Kp, dt)))
        fwd.append(gemm(_ptr(e.stem_cols), _ptr(e.stem_wpad), _ptr(y0), N * Hs * Ws, spec.stem, Kp, bn))
    else:
        fwd.append(("dfd_stem_fwd", (_ptr(e.x_in), P32("conv_stem.weight"), _ptr(y0), N, spec.in_chans, e.H, e.W,
                                     spec.stem, 3, 2, 1, dt) + e._stats(bn)))
    fwd += finalize(bn, N * Hs * Ws)
    fwd.append(("dfd_bn_act", (_ptr(y0), bn.scale, bn.shift, None, None, _ptr(stem_out), N, Hs * Ws, spec.stem,
                               ACT_SWISH, 0, dt)))
    x = stem_out
    recs = []
    # stochastic regularisation (train mode only): per-sample drop-path scale of every residual block
    # (rate = drop_path_rate * block_idx / n_blocks, efficientnet_builder.py:228-230,343) and the classifier dropout mask;
    # the gates are [N, C] fp32 tensors (one draw per sample replicated over the channels) filled by ONE dfd_rng_masks
    # launch at the head of the forward plan, consumed through the GATE operand of dfd_bn_act
    masks = []               # (tensor, rows, width, keep_prob)
    n_blocks = len(blocks)
    for bi, (b, h, w, ho, wo) in enumerate(blocks):
        p = b.name
        M1, M2 = N * h * w, N * ho * wo
        rec = dict(b=b, h=h, w=w, ho=ho, wo=wo, x=x)
        if b.kind == "ir":
            bn1, bn2, bn3 = e.bns[p + ".bn1"], e.bns[p + ".bn2"], e.bns[p + ".bn3"]
            y1 = e._alloc16(N, h, w, b.cmid)
            e.acts[p + ".conv_pw"] = y1
            fwd.append(gemm(_ptr(x), P16(p + ".conv_pw.weight"), _ptr(y1), M1, b.cmid, b.cin, bn1))
            fwd += finalize(bn1, M1)
            dw_in, dw_bn, bn_mid, bn_out, pw_name = y1, bn1, bn2, bn3, ".conv_pwl"
            rec.update(y1=y1)
        else:
            dw_in, dw_bn, bn_mid, bn_out, pw_name = x, None, e.bns[p + ".bn1"], e.bns[p + ".bn2"], ".conv_pw"
        y2 = e._alloc16(N, ho, wo, b.cmid)
        e.acts[p + ".conv_dw"] = y2
        dw_pad = pads[p + ".conv_dw"] if asym(p + ".conv_dw", b.k) else ()
        fwd.append(("dfd_dwconv_fwd" + ("_pad" if dw_pad else ""),
                    (_ptr(dw_in), dw_bn.scale if dw_bn else None, dw_bn.shift if dw_bn else None,
                     P32(p + ".conv_dw.weight"), _ptr(y2), N, h, w, b.cmid, b.k, b.stride) + dw_pad +
                    (ACT_SWISH if dw_bn else ACT_NONE, dt) + e._stats(bn_mid) + (None,)))
        fwd += finalize(bn_mid, M2)
        gate_ptr = None
        if b.cse:
            pooled = torch.zeros(N, b.cmid, dtype=torch.float32, device=dev)
            gate = torch.zeros(N, b.cmid, dtype=torch.float32, device=dev)
            e._keep += [pooled, gate]
            rec.update(pooled=pooled, gate=gate)
            fwd.append(("dfd_pool", (_ptr(y2), bn_mid.scale, bn_mid.shift, _ptr(pooled), N, ho * wo, b.cmid, ACT_SWISH, dt,
                                     None, POOL_CHUNKS)))
            fwd.append(("dfd_se_fc_fwd", (_ptr(pooled), P32(p + ".se.conv_reduce.weight"), P32(p + ".se.conv_reduce.bias"),
                                          P32(p + ".se.conv_expand.weight"), P32(p + ".se.conv_expand.bias"),
                                          _ptr(gate), N, b.cmid, b.cse)))
            gate_ptr = _ptr(gate)
        a2 = e._alloc16(N, ho, wo, b.cmid)
        fwd.append(("dfd_bn_act", (_ptr(y2), bn_mid.scale, bn_mid.shift, gate_ptr, None, _ptr(a2), N, ho * wo, b.cmid,
                                   ACT_SWISH, 0, dt)))
        y3 = e._alloc16(N, ho, wo, b.cout)
        e.acts[p + pw_name] = y3
        fwd.append(gemm(_ptr(a2), P16(p + pw_name + ".weight"), _ptr(y3), M2, b.cout, b.cmid, bn_out))
        fwd += finalize(bn_out, M2)
        out = e._alloc16(N, ho, wo, b.cout)
        e.acts[p + ".out"] = out
        dp_rate = e.drop_path_rate * bi / n_blocks if b.has_residual else 0.0
        dp_gate = None
        if dp_rate > 0.0:
            dp_gate = torch.ones(N, b.cout, dtype=torch.float32, device=dev)
            e._keep.append(dp_gate)
            masks.append((dp_gate, N, b.cout, 1.0 - dp_rate))
        fwd.append(("dfd_bn_act", [_ptr(y3), bn_out.scale, bn_out.shift, ("TRAIN_ONLY", _ptr(dp_gate)) if dp_gate is not None else None,
                                   _ptr(x) if b.has_residual else None,
                                   _ptr(out), N, ho * wo, b.cout, ACT_NONE, 1 if b.has_residual else 0, dt]))
        rec.update(y2=y2, a2=a2, y3=y3, out=out, dw_bn=dw_bn, bn_mid=bn_mid, bn_out=bn_out, pw_name=pw_name, dp_gate=dp_gate,
                   dw_pad=dw_pad)
        recs.append(rec)
        x = out
    # head
    F = spec.num_features
    Mf = N * Hf * Wf
    bnh = e.bns["bn2"]
    yh = e._alloc16(N, Hf, Wf, F)
    e.acts["conv_head"] = yh
    fwd.append(gemm(_ptr(x), P16("conv_head.weight"), _ptr(yh), Mf, F, spec.head_in, bnh))
    fwd += finalize(bnh, Mf)
    P, pool_t = spec.pooled_features, _lib.POOL_TYPES[spec.global_pool]
    e.pooled = torch.zeros(N, P, dtype=torch.float32, device=dev)
    if pool_t == _lib.POOL_TYPES["avg"]:
        fwd.append(("dfd_pool", (_ptr(yh), bnh.scale, bnh.shift, _ptr(e.pooled), N, Hf * Wf, F, ACT_SWISH, dt,
                                 None, POOL_CHUNKS)))
    else:
        # max / avgmax / catavgmax: one pass gives the mean (dfd_pool's order), the max and its argmax for the backward
        e.pool_argmax = torch.zeros(N, F, dtype=torch.int32, device=dev)
        fwd.append(("dfd_global_pool", (_ptr(yh), bnh.scale, bnh.shift, _ptr(e.pooled), _ptr(e.pool_argmax), N,
                                        Hf * Wf, F, ACT_SWISH, pool_t, dt, POOL_CHUNKS)))
    e.drop_masks = OrderedDict()
    if e.drop_rate > 0.0:
        e.dropout_mask = torch.ones(N, P, dtype=torch.float32, device=dev)
        masks.append((e.dropout_mask, N * P, 1, 1.0 - e.drop_rate))
        fwd.append(("dfd_mul_f32_train", (_ptr(e.pooled), _ptr(e.dropout_mask), N * P)))
    for r_ in recs:
        if r_["dp_gate"] is not None:
            e.drop_masks[r_["b"].name] = r_["dp_gate"]
    fwd = e._mask_head(masks) + fwd
    if masks:
        cmax = max(t.shape[-1] for t, _, _, _ in masks)
        e._unit_affine = torch.cat([torch.ones(cmax, device=dev), torch.zeros(cmax, device=dev)]).float()
        e._keep.append(e._unit_affine)
    K = spec.num_classes
    e.logits = torch.zeros(N, K, dtype=torch.float32, device=dev)
    e.dlogits = torch.zeros(N, K, dtype=torch.float32, device=dev)
    e.dpooled = torch.zeros(N, P, dtype=torch.float32, device=dev)
    e.target_i = torch.zeros(N, dtype=torch.int64, device=dev)
    e.target_f = torch.zeros(N, K, dtype=torch.float32, device=dev)
    e._head_in = x

    # ---- backward ----------------------------------------------------------------------------
    bwd.append(("dfd_head_bwd", (_ptr(e.dlogits), _ptr(e.pooled), P32("classifier.weight"),
                                 G32("classifier.weight"), G32("classifier.bias"), _ptr(e.dpooled), N, P, K)))
    if e.drop_rate > 0.0:
        bwd.append(("dfd_mul_f32", (_ptr(e.dpooled), _ptr(e.dropout_mask), N * P)))
    if pool_t == _lib.POOL_TYPES["avg"]:
        bwd.append(("dfd_act_bwd", (None, _ptr(yh), bnh.scale, bnh.shift, bnh.mean, bnh.rstd, None, _ptr(e.dpooled),
                                    mid_a, N, Hf * Wf, F, ACT_SWISH, dt, bnh.bs1, bnh.bs2, None)))
    else:
        bwd.append(("dfd_act_bwd_gpool", (_ptr(yh), bnh.scale, bnh.shift, bnh.mean, bnh.rstd, _ptr(e.dpooled),
                                          _ptr(e.pool_argmax), mid_a, N, Hf * Wf, F, ACT_SWISH, pool_t, dt, bnh.bs1,
                                          bnh.bs2, None)))
    bwd += bwd_finalize(bnh, Mf)
    bwd.append(("dfd_bn_bwd_apply", (mid_a, _ptr(yh), None, bnh.cA, bnh.cB, bnh.cC, mid_b, N, Hf * Wf, F, dt)))
    cur = 0
    bwd.append(gemm(mid_b, T16("conv_head.weight"), sm[cur], Mf, spec.head_in, F))
    bwd.append(e._wgrad(mid_b, _ptr(e._head_in), G32("conv_head.weight"), Mf, F, spec.head_in))
    e._flush_reduce(bwd)
    for rec in reversed(recs):
        b, h, w, ho, wo, xin = rec["b"], rec["h"], rec["w"], rec["ho"], rec["wo"], rec["x"]
        p = b.name
        M1, M2 = N * h * w, N * ho * wo
        bn_out, bn_mid, dw_bn, pw_name = rec["bn_out"], rec["bn_mid"], rec["dw_bn"], rec["pw_name"]
        y2, a2, y3 = rec["y2"], rec["a2"], rec["y3"]
        dout = sm[cur]
        t1, t2 = sm[(cur + 1) % 3], sm[(cur + 2) % 3]
        gbn = dout
        if rec["dp_gate"] is not None:
            # drop path: the gradient reaching bn3 is dout * mask / keep (the identity branch keeps dout itself); one extra
            # pass through the gated streaming kernel with a unit affine, only in this regularised configuration
            cm = e._unit_affine.numel() // 2
            bwd.append(("dfd_bn_act", (dout, _ptr(e._unit_affine), _ptr(e._unit_affine, cm), _ptr(rec["dp_gate"]), None, t2,
                                       N, ho * wo, b.cout, ACT_NONE, 0, dt)))
            gbn = t2
        bwd.append(("dfd_bn_bwd_reduce", (gbn, _ptr(y3), None, bn_out.mean, bn_out.rstd, N, ho * wo, b.cout, dt,
                                          bn_out.bs1, bn_out.bs2, None)))
        bwd += bwd_finalize(bn_out, M2)
        bwd.append(("dfd_bn_bwd_apply", (gbn, _ptr(y3), None, bn_out.cA, bn_out.cB, bn_out.cC, t1, N, ho * wo, b.cout, dt)))
        bwd.append(gemm(t1, T16(p + pw_name + ".weight"), mid_a, M2, b.cmid, b.cout))
        bwd.append(e._wgrad(t1, _ptr(a2), G32(p + pw_name + ".weight"), M2, b.cout, b.cmid))
        gate_ptr = dpool_ptr = None
        if b.cse:
            gate_ptr, dpool_ptr = _ptr(rec["gate"]), se_dpool
            bwd.append(("dfd_se_bwd_reduce", (mid_a, _ptr(y2), bn_mid.scale, bn_mid.shift, se_draw, N, ho * wo, b.cmid, dt)))
            bwd.append(("dfd_se_fc_bwd", (se_draw, _ptr(rec["pooled"]), P32(p + ".se.conv_reduce.weight"),
                                          P32(p + ".se.conv_reduce.bias"), P32(p + ".se.conv_expand.weight"),
                                          P32(p + ".se.conv_expand.bias"), se_de, se_r, se_drp, se_dpool,
                                          G32(p + ".se.conv_reduce.weight"), G32(p + ".se.conv_reduce.bias"),
                                          G32(p + ".se.conv_expand.weight"), G32(p + ".se.conv_expand.bias"),
                                          N, b.cmid, b.cse)))
        bwd.append(("dfd_act_bwd", (mid_a, _ptr(y2), bn_mid.scale, bn_mid.shift, bn_mid.mean, bn_mid.rstd, gate_ptr,
                                    dpool_ptr, mid_b, N, ho * wo, b.cmid, ACT_SWISH, dt, bn_mid.bs1, bn_mid.bs2, None)))
        bwd += bwd_finalize(bn_mid, M2)
        if b.kind == "ir":
            y1 = rec["y1"]
            # input gradient (through bn1 + Swish) and weight gradient in one pass over the dy tile
            dw_pad = rec["dw_pad"]
            bwd.append(e._dw_bwd((mid_b, _ptr(y2), bn_mid.cA, bn_mid.cB, bn_mid.cC, P32(p + ".conv_dw.weight"),
                                  _ptr(y1), dw_bn.scale, dw_bn.shift, dw_bn.mean, dw_bn.rstd, None, mid_a,
                                  G32(p + ".conv_dw.weight"), N, h, w, b.cmid, b.k, b.stride) + dw_pad +
                                 (dt, dw_bn.bs1, dw_bn.bs2), N, h, w, b.cmid, b.k, b.stride,
                                 name="dfd_dwconv_bwd" + ("_pad" if dw_pad else "")))
            bwd += bwd_finalize(dw_bn, M1)
            bwd.append(("dfd_bn_bwd_apply", (mid_a, _ptr(y1), None, dw_bn.cA, dw_bn.cB, dw_bn.cC, mid_b, N, h * w, b.cmid, dt)))
            bwd.append(gemm(mid_b, T16(p + ".conv_pw.weight"), t2, M1, b.cin, b.cmid))
            if b.has_residual:
                bwd.append(("dfd_add_inplace", (t2, dout, M1 * b.cin, dt)))
            bwd.append(e._wgrad(mid_b, _ptr(xin), G32(p + ".conv_pw.weight"), M1, b.cmid, b.cin))
        else:
            # DS block: the depthwise conv reads the block input as is (mode 0 of the fused pass); stride 1 in every
            # EfficientNet, so its padding is symmetric under TF "SAME" too
            assert not rec["dw_pad"], p
            bwd.append(e._dw_bwd((mid_b, _ptr(y2), bn_mid.cA, bn_mid.cB, bn_mid.cC, P32(p + ".conv_dw.weight"),
                                  _ptr(xin), None, None, None, None, dout if b.has_residual else None, t2,
                                  G32(p + ".conv_dw.weight"), N, h, w, b.cmid, b.k, b.stride, dt, None, None),
                                 N, h, w, b.cmid, b.k, b.stride))
        e._flush_reduce(bwd)
        cur = (cur + 2) % 3
    # stem
    bn = e.bns["bn1"]
    bwd.append(("dfd_act_bwd", (sm[cur], _ptr(y0), bn.scale, bn.shift, bn.mean, bn.rstd, None, None, mid_a, N, Hs * Ws,
                                spec.stem, ACT_SWISH, dt, bn.bs1, bn.bs2, None)))
    bwd += bwd_finalize(bn, N * Hs * Ws)
    if e.stem_impl == "gemm":
        bwd.append(("dfd_bn_bwd_apply", (mid_a, _ptr(y0), None, bn.cA, bn.cB, bn.cC, mid_b, N, Hs * Ws, spec.stem, dt)))
        bwd.append(("dfd_memset_async", (_ptr(e.stem_gpad), 0, spec.stem * Kp * 4)))
        bwd.append(e._wgrad(mid_b, _ptr(e.stem_cols), _ptr(e.stem_gpad), N * Hs * Ws, spec.stem, Kp))
        e._flush_reduce(bwd)          # the padded gradient must be complete before it is un-padded into the arena
        bwd.append(("dfd_unpad_grad", (_ptr(e.stem_gpad), G32("conv_stem.weight"), spec.stem, taps, Kp)))
    else:
        bwd.append(("dfd_stem_wgrad", (_ptr(e.x_in), mid_a, _ptr(y0), bn.cA, bn.cB, bn.cC, G32("conv_stem.weight"), N,
                                       spec.in_chans, e.H, e.W, spec.stem, 3, 2, 1, dt)))
    e._finish_plan(fwd, bwd)
