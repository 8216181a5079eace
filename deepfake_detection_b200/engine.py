"""Native train / validate engine: lays the network out in HBM and drives the sm_90a kernels.

This is the host side of the hot path (dfd/runners/train.py:610-649): given an architecture spec it
  * owns the flat fp32 parameter / gradient arenas (reference tensor names, OIHW shapes) plus their 16-bit
    copies in the layouts the kernels read ([Cout,Cin] and transposed [Cin,Cout] for the 1x1 convs),
  * keeps every conv output NHWC in 16-bit (the only activation tensors that touch HBM),
  * builds, once, the ordered list of C-ABI calls ("plan") for forward, backward and the optimizer, and
  * replays the plan on the caller's current CUDA stream (optionally captured into a CUDA graph).

The family's plan builder (engine_efficientnet, engine_resnet, engine_xception, engine_densenet) lays out the activations
and lists the ops; the conventions every plan shares (BatchNorm statistics, finalisation and backward apply, the mask
generators, the deterministic weight-gradient reduce, the stem as im2col + GEMM, the pooled classifier head, the packed k x k
weights, validation against the ABI table) are the plan helpers of this class.

A plan op is (name, args). `base_name(name)` is the C-ABI entry point it calls: `<entry>_train` runs in training mode
only and `dfd_bn_finalize_sync` finalises the summed statistics of all ranks. In args, ("TRAIN_ONLY", ptr) is an operand
that is NULL in eval mode, "TRAINING" is the mode flag (1 / 0) and ("WS", off) a slot of the deterministic-reduce
workspace, resolved when the plan is finished.

PyTorch is used for device memory and streams only; there is no PyTorch compute on the hot path and no CPU
fallback: constructing an Engine without a CUDA device or without libdfd_b200.so raises.
"""
import struct
from collections import OrderedDict

import torch

from . import _lib
from .arch import get_spec, is_no_decay, param_entries, state_entries

ACT_NONE, ACT_SWISH, ACT_RELU = _lib.ACT_NONE, _lib.ACT_SWISH, _lib.ACT_RELU
POOL_CHUNKS = 8          # row chunks per image of the pooling kernels when the batch alone cannot fill the GPU


def _ptr(t, off_elems=0):
    return t.data_ptr() + off_elems * t.element_size()


def base_name(name):
    """the C-ABI entry point of the plan op `name`"""
    for suf in ("_train", "_sync"):
        if name.endswith(suf):
            return name[:-len(suf)]
    return name


class _BN:
    """Pointers of one BatchNorm layer (parameters, running stats, per-step statistics, bwd coefficients)."""
    __slots__ = ("name", "C", "gamma", "beta", "dgamma", "dbeta", "rm", "rv", "nbt", "scale", "shift", "mean",
                 "rstd", "cA", "cB", "cC", "fsum", "fsq", "bs1", "bs2", "stat_off")


class Engine:
    def __init__(self, arch, batch, height=None, width=None, num_classes=2, in_chans=3, dtype="bf16",
                 bn_momentum=0.1, bn_eps=1e-5, device=None, gemm_impl="tc", share_from=None, params_only=False,
                 drop_rate=0.0, drop_path_rate=0.0, sync_bn=False, global_pool="avg", drop_block_rate=0.0):
        # _plan_only: build the arenas and the call plan on the CPU for host-logic tests; nothing can be executed
        self._plan_only = device == "plan-only"
        if self._plan_only:
            device = "cpu"
        elif not torch.cuda.is_available():
            raise _lib.NativeError("deepfake_detection_b200.Engine needs a CUDA device (H100, sm_90a); "
                                   "there is no CPU path")
        self.L = _lib.lib()
        self.spec = spec = get_spec(arch, num_classes=num_classes, in_chans=in_chans, global_pool=global_pool)
        self.cls_name = "classifier" if spec.family in ("efficientnet", "densenet") else (
            spec.cls_name if spec.family == "resnet" else "fc")
        self.device = torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())
        self.N = int(batch)
        self.H = int(height or spec.input_size[1])
        self.W = int(width or spec.input_size[2])
        if dtype in ("bf16", "bfloat16", torch.bfloat16):
            self.dt, self.tdtype = _lib.DT_BF16, torch.bfloat16
        elif dtype in ("fp16", "float16", "half", torch.float16):
            self.dt, self.tdtype = _lib.DT_FP16, torch.float16
        else:
            raise ValueError("dtype %r: the native path computes in 'bf16' or 'fp16' (fp32 master weights)" % (dtype,))
        self.drop_rate = float(drop_rate)
        self.drop_path_rate = float(drop_path_rate)
        # DropBlock of the ResNet family (layer3 / layer4, resnet.py:386-387); the EfficientNet plan has no DropBlock sites
        self.drop_block_rate = float(drop_block_rate or 0.0)
        # synchronised BatchNorm (train.py:388-400 `convert_syncbn_model`): batch statistics and the BN-backward sums are
        # all-reduced over the process group between the kernel that produces them and the finalisation
        self.sync_bn = bool(sync_bn)
        self.sync_world = 1
        if self.sync_bn:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                self.sync_world = dist.get_world_size()
            self.sync_bn = self.sync_world > 1
        if self.sync_bn and spec.family in ("resnet", "xception", "densenet"):
            raise _lib.NativeError("sync_bn over %d ranks: the %s plan has no synchronised BatchNorm (only the "
                                   "EfficientNet plan all-reduces its batch statistics)"
                                   % (self.sync_world, {"resnet": "ResNet", "xception": "Xception",
                                                        "densenet": "DenseNet"}[spec.family]))
        self.bn_momentum = float(bn_momentum)
        self.bn_eps = float(bn_eps)
        # "tc": wgmma GEMMs and implicit convolutions; "mma": the mma.sync cross-check path (GEMMs over im2col columns)
        self.gemm_impl = gemm_impl
        self.training = True
        self.n_launch = {"fwd": 0, "bwd": 0, "opt": 0}
        self._shared_from = share_from
        if share_from is not None:
            # a second plan (other batch size / resolution, e.g. the validation loader) over the SAME weights,
            # gradients and running statistics
            if share_from.spec.arch != spec.arch or share_from.dt != self.dt or share_from.spec.global_pool != spec.global_pool:
                raise ValueError("share_from: architecture / dtype / global_pool mismatch")
            share_from = self._shared_from = share_from.arena
            for a in ("p_off", "n_decay", "n_params", "param_names", "params32", "grads32", "params16", "b_off", "bn_names",
                      "buffers32", "nbt", "t_off", "paramsT16", "_ttable", "_ttable_count", "loss_scale_state", "flags",
                      "rng_state"):
                setattr(self, a, getattr(share_from, a))
        else:
            self._layout_params()
            self.loss_scale_state = torch.ones(2, dtype=torch.float32, device=self.device)   # scale, 1/scale
            self.flags = torch.zeros(2, dtype=torch.int32, device=self.device)              # found_inf, good_steps
            # counter-based generator state of the dropout / drop-path masks: [seed, step]; the step advances on the device
            self.rng_state = torch.zeros(2, dtype=torch.int64, device=self.device)
            self.rng_state[0] = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF          # follows torch.manual_seed (train.py:299)
            self._derived_dirty = False
            # bumped whenever a plan registers a derived weight layout (block-diagonal copy, padded stem weight, packed k x k
            # weights): a CUDA graph captured around the optimizer's refresh holds the old table pointers and entry counts and
            # must be re-captured (Trainer._graph_signature)
            self.layout_gen = 0
            # bumped whenever weights or BN running statistics change (load, a training forward, EMA / distribute_bn): an
            # eval-mode plan recomputes its per-channel scale / shift vectors only when this moved (see forward)
            self.state_version = 0
        self._eval_version = -1
        self.params_only = bool(params_only)
        self._red_pending, self._ws_bytes = [], 0
        if self.params_only:
            # the owner of the parameter / gradient / running-statistic arenas without any activation plan: what
            # `NativeModel.engine`, the optimizer and the EMA need (a plan is built per (batch, H, W) that reaches forward)
            self.fwd_ops, self.bwd_ops = [], []
            return
        self._build()
        if not self._plan_only and self.arena._derived_dirty:
            # this plan registered new derived weight layouts with the owner: fill them now (never inside a graph capture)
            self.refresh_weight_layouts(torch.cuda.current_stream().cuda_stream)

    # ------------------------------------------------------------------------------------------
    # parameter / buffer arenas
    # ------------------------------------------------------------------------------------------
    def _layout_params(self):
        spec, dev = self.spec, self.device
        entries = param_entries(spec)
        decay = [(n, s) for n, s, _ in entries if not is_no_decay(n, s)]
        nodecay = [(n, s) for n, s, _ in entries if is_no_decay(n, s)]
        self.p_off = OrderedDict()
        off = 0
        for n, s in decay + nodecay:
            numel = 1
            for d in s:
                numel *= d
            self.p_off[n] = (off, tuple(s), numel)
            off += (numel + 3) // 4 * 4          # keep every tensor 16-byte aligned in fp32 and 8-byte in 16-bit
            if n == decay[-1][0]:
                off = (off + 7) // 8 * 8
                self.n_decay = off
        self.n_params = off
        self.param_names = [n for n, _, _ in entries]
        self.params32 = torch.zeros(off, dtype=torch.float32, device=dev)
        self.grads32 = torch.zeros(off, dtype=torch.float32, device=dev)
        self.params16 = torch.zeros(off, dtype=self.tdtype, device=dev)
        # buffers (running stats): flat fp32 + int64 counters
        self.b_off = OrderedDict()
        boff = 0
        self.bn_names = []
        for n, s, role in state_entries(spec):
            if role in ("bn_rm", "bn_rv"):
                self.b_off[n] = (boff, s[0])
                boff += (s[0] + 3) // 4 * 4
            elif role == "bn_nbt":
                self.bn_names.append(n[: -len(".num_batches_tracked")])
        self.buffers32 = torch.zeros(boff, dtype=torch.float32, device=dev)
        for n, (o, c) in self.b_off.items():
            if n.endswith("running_var"):
                self.buffers32[o:o + c] = 1.0
        self.nbt = torch.zeros(len(self.bn_names), dtype=torch.int64, device=dev)
        # transposed 16-bit copies of the 1x1 conv weights (dgrad B operand)
        self.t_off = OrderedDict()
        toff = 0
        for n, s, role in entries:
            if role == "conv_w" and s[2] == 1 and s[3] == 1:
                self.t_off[n] = (toff, s[0], s[1])
                toff += (s[0] * s[1] + 7) // 8 * 8
        self.paramsT16 = torch.zeros(max(toff, 8), dtype=self.tdtype, device=dev)
        raw = b"".join(struct.pack("<QQii", _ptr(self.params16, self.p_off[n][0]), _ptr(self.paramsT16, o), O, I)
                       for n, (o, O, I) in self.t_off.items())
        self._ttable = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
        self._ttable_count = len(self.t_off)

    @property
    def arena(self):
        """the engine that owns the weights, gradients, running statistics and derived weight layouts"""
        return self._shared_from if self._shared_from is not None else self

    def param_view(self, name):
        o, s, n = self.p_off[name]
        return self.params32[o:o + n].view(s)

    def grad_view(self, name):
        o, s, n = self.p_off[name]
        return self.grads32[o:o + n].view(s)

    def buffer_view(self, name):
        if name.endswith("num_batches_tracked"):
            return self.nbt[self.bn_names.index(name[: -len(".num_batches_tracked")])]
        o, c = self.b_off[name]
        return self.buffers32[o:o + c]

    def state_dict(self):
        """Reference-layout state dict (fp32 master weights, OIHW), a copy."""
        sd = OrderedDict()
        for n, s, role in state_entries(self.spec):
            if role in ("bn_rm", "bn_rv", "bn_nbt"):
                sd[n] = self.buffer_view(n).clone()
            else:
                sd[n] = self.param_view(n).clone()
        return sd

    def load_state_dict(self, sd, strict=True):
        missing = []
        with torch.no_grad():
            for n, s, role in state_entries(self.spec):
                if n not in sd:
                    missing.append(n)
                    continue
                src = sd[n].to(self.device)
                if role in ("bn_rm", "bn_rv"):
                    self.buffer_view(n).copy_(src.float())
                elif role == "bn_nbt":
                    self.nbt[self.bn_names.index(n[: -len(".num_batches_tracked")])] = int(src)
                else:
                    self.param_view(n).copy_(src.float().reshape(self.p_off[n][1]))
        if strict and missing:
            raise KeyError("missing keys in state_dict: %s" % missing[:5])
        self.sync_weights()
        return missing

    def sync_weights(self):
        """fp32 master -> 16-bit kernel copies (call after any out-of-band weight change)."""
        self.arena.state_version += 1
        st = torch.cuda.current_stream().cuda_stream
        _lib.call("dfd_cast_arena", _ptr(self.params32), _ptr(self.params16), self.n_params, self.dt, st)
        self.refresh_weight_layouts(st)

    # ------------------------------------------------------------------------------------------
    # plan construction
    # ------------------------------------------------------------------------------------------
    # ---- order-deterministic weight gradients ------------------------------------------------------------------
    # The tensor-core weight gradient and the fused depthwise backward run in WORKSPACE mode: every CTA stores its split partial
    # sum in a fixed slot of one workspace (plain stores, no atomics) and `dfd_ordered_reduce` - one table-driven launch per
    # block of the network, right behind that block's backward ops - adds the partials into the gradient arena in slot
    # order. Gradients (and with them every later step) therefore do not depend on the arrival order of CTAs; the reduce
    # launches are also the points at which a block's gradients become final for the DDP bucketing.
    def _wgrad(self, G, X, dW, M, Nw, Kw):
        if self.gemm_impl != "tc":
            return ("dfd_gemm_wgrad_mma", (G, X, dW, M, Nw, Kw, self.dt))
        splits = self.L.cdll.dfd_gemm_wgrad_splits(M, Nw, Kw)
        off, nbytes = self._ws_take(splits * Nw * Kw * 4)
        self._red_pending.append((off, dW, Nw * Kw, Nw * Kw, splits))
        return ("dfd_gemm_wgrad", [G, X, dW, M, Nw, Kw, self.dt, ("WS", off), nbytes])

    def _wgrad_conv(self, dY, X, dW, N, H, W, Cin, Cout, k, stride=1):
        """implicit-GEMM weight gradient of a dense k x k convolution (H, W = input extents) into the packed
        [Cout][kh][kw][Cin] fp32 buffer"""
        Kw = k * k * Cin
        splits = self.L.cdll.dfd_conv_wgrad_splits(N, H, W, Cin, Cout, k, stride)
        off, nbytes = self._ws_take(splits * Cout * Kw * 4)
        self._red_pending.append((off, dW, Cout * Kw, Cout * Kw, splits))
        return ("dfd_conv_wgrad_tc", [dY, X, dW, N, H, W, Cin, Cout, k, stride, self.dt, ("WS", off), nbytes])

    def _dw_bwd(self, args, N, H, W, C, k, stride, name="dfd_dwconv_bwd"):
        parts = self.L.cdll.dfd_dwconv_bwd_parts(N, H, W, C, k, stride)
        cw = self.L.cdll.dfd_dwconv_block_channels(C)          # channels per CTA: 64, or 32 / 16 for C = 32, 96 / 144
        cbs = (C + cw - 1) // cw
        off, nbytes = self._ws_take(cbs * parts * cw * k * k * 4)
        dW = args[13]
        for cb in range(cbs):
            n = min(cw, C - cw * cb) * k * k
            self._red_pending.append((off + cb * parts * cw * k * k * 4, dW + cb * cw * k * k * 4, n, cw * k * k, parts))
        return (name, list(args) + [("WS", off), nbytes, None])

    def _ws_take(self, nbytes):
        off = getattr(self, "_ws_bytes", 0)
        self._ws_bytes = off + (nbytes + 255) // 256 * 256
        return off, nbytes

    def _flush_reduce(self, ops):
        """emit the ordered-reduce launch for the partial sums produced since the last flush (call at block boundaries)"""
        pend = self.__dict__.setdefault("_red_pending", [])
        if pend:
            ops.append(("dfd_ordered_reduce", ["REDUCE", list(pend)]))
            del pend[:]

    def _patch_workspace(self, ops):
        self._flush_reduce(ops)
        total = getattr(self, "_ws_bytes", 0)
        if not total:
            return ops
        self.det_ws = torch.empty(total // 4, dtype=torch.float32, device=self.device)
        base = _ptr(self.det_ws)
        entries = [e for n, a in ops if n == "dfd_ordered_reduce" for e in a[1]]
        raw = b"".join(struct.pack("<QQqqii", base + off, dst, n, stride, parts, 0) for off, dst, n, stride, parts in entries)
        self._red_table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)
        out, pos = [], 0
        for n, a in ops:
            if n == "dfd_ordered_reduce":
                ents = a[1]
                bx = max((e[2] // 4 + 7) // 8 if e[4] > 64 else (e[2] // 4 + 255) // 256 for e in ents)
                a = (_ptr(self._red_table, pos * 40), len(ents), min(e[1] for e in ents), max(1, min(bx, 1024)))
                pos += len(ents)
            elif isinstance(a, list):
                a = [base + v[1] if isinstance(v, tuple) and v[0] == "WS" else v for v in a]
            out.append((n, a))
        return out

    def _alloc16(self, *shape):
        # the plan holds RAW pointers: every buffer must stay referenced for the engine's lifetime
        t = torch.empty(shape, dtype=self.tdtype, device=self.device)
        self._keep.append(t)
        return t

    # rows of A fused per TMA row for small-K pointwise convs (tools/gemm_time2.py times the choices): the factor makes
    # pack*K a multiple of the 64-element k-block where that keeps pack*N modest
    _ROW_PACK = {8: 8, 16: 4, 24: 8, 32: 4, 40: 2, 48: 4, 56: 2}

    @classmethod
    def _row_pack(cls, M, K):
        """rows of A read as one (dfd_gemm_tn_rowpack): keeps the TMA rows of small-K pointwise convs at >= 128 bytes"""
        pack = cls._ROW_PACK.get(K, 1)
        while pack > 1 and M % pack:
            pack //= 2
        return pack

    # Derived 16-bit weight layouts (block-diagonal small-K copies, the padded stem weight, the packed k x k weights of
    # the ResNet path) are registered with, owned by and refreshed through the ARENA engine, whichever plan asked for them:
    # the optimizer refreshes them once per step for every plan that shares the weights.
    def _blockdiag(self, B, Nn, K, pack):
        """block-diagonal [pack*Nn, pack*K] copy of the weight at B"""
        o = self.arena
        reg = o.__dict__.setdefault("_bd_reg", OrderedDict())
        key = (B, Nn, K, pack)
        if key not in reg:
            reg[key] = torch.zeros(pack * Nn * pack * K, dtype=self.tdtype, device=self.device)
            o._bd_table = None
            o._derived_dirty = True
            o.layout_gen += 1
        return _ptr(reg[key])

    def refresh_weight_layouts(self, stream):
        """derived 16-bit weight layouts (transposed 1x1, packed k x k, block-diagonal small-K) from the 16-bit arena"""
        o = self.arena
        _lib.call("dfd_transpose_weights", _ptr(o._ttable), o._ttable_count, o.dt, stream)
        reg = getattr(o, "_bd_reg", None)
        if reg and getattr(o, "_bd_table", None) is None:
            raw = b"".join(struct.pack("<QQiiii", B, _ptr(t), Nn, K, pack, 0) for (B, Nn, K, pack), t in reg.items())
            o._bd_table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(o.device)
        if getattr(o, "_rtable_count", 0):
            _lib.call("dfd_repack_weights", _ptr(o._rtable), o._rtable_count, o.dt, stream)
        for (name, O, taps, Kp), wpad in getattr(o, "_stem_reg", {}).items():
            _lib.call("dfd_pad_weight", _ptr(o.params16, o.p_off[name][0]), _ptr(wpad), O, taps, Kp, o.dt, stream)
        if reg:
            _lib.call("dfd_blockdiag_weights", _ptr(o._bd_table), len(reg), o.dt, stream)
        o._derived_dirty = False

    def _packed_weights(self, names):
        """the k x k weights `names` in the packed layouts of the dense convolutions: wpack16 [Cout][kh][kw][Cin] (forward),
        wpackT16 its transpose (input gradient over im2col columns) and wpackD16 the tap-flipped [Cin][kh][kw][Cout] (implicit
        input gradient). They depend on the parameter shapes only, so the arena engine registers them once; returns each
        weight's element offset into the three buffers"""
        offs, off = OrderedDict(), 0
        for n in names:
            offs[n] = off
            off += (self.p_off[n][2] + 7) // 8 * 8
        ar = self.arena
        if getattr(ar, "wpack16", None) is None:
            ar.wpack16, ar.wpackT16, ar.wpackD16 = [torch.zeros(max(off, 8), dtype=self.tdtype, device=self.device)
                                                    for _ in range(3)]
            raw = b"".join(struct.pack("<QQQQiiii", _ptr(self.params16, self.p_off[n][0]), _ptr(ar.wpack16, o),
                                       _ptr(ar.wpackT16, o), _ptr(ar.wpackD16, o), *self.p_off[n][1][:3], 0)
                           for n, o in offs.items())
            ar._rtable = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)
            ar._rtable_count = len(offs)
            ar._derived_dirty = True
            ar.layout_gen += 1
        self.wpack16, self.wpackT16, self.wpackD16 = ar.wpack16, ar.wpackT16, ar.wpackD16
        return offs

    def _stem_gemm(self, wname, Cout, k, stride, pad, y, M, bn, rowpack=True):
        """forward ops of the stem convolution of x_in as im2col + tensor-core GEMM into y [M, Cout], with the batch statistics
        of `bn`. The columns and a padded copy of the weight have K = Cin*k*k zero-padded to a multiple of 8. `pad` is the
        padding of every side, or the (top, left) padding of TF "SAME" (the bottom / right padding follows from the output
        extents)."""
        taps = self.spec.in_chans * k * k
        Kp = (taps + 7) // 8 * 8
        o = self.arena
        reg = o.__dict__.setdefault("_stem_reg", OrderedDict())
        key = (wname, Cout, taps, Kp)
        if key not in reg:
            reg[key] = torch.zeros(Cout * Kp, dtype=self.tdtype, device=self.device)
            o._derived_dirty = True
            o.layout_gen += 1
        self.stem_wpad = reg[key]
        self.stem_gpad = torch.zeros(Cout * Kp, dtype=torch.float32, device=self.device)
        self.stem_cols = self._alloc16(M, Kp)
        self._stem = (wname, Cout, M, taps, Kp)
        same = isinstance(pad, tuple)
        im2col = ("dfd_stem_im2col_pad" if same else "dfd_stem_im2col",
                  (_ptr(self.x_in), _ptr(self.stem_cols), self.N, self.spec.in_chans, self.H, self.W, k, stride)
                  + (pad if same else (pad,)) + (Kp, self.dt))
        return [im2col, self._gemm(_ptr(self.stem_cols), _ptr(self.stem_wpad), _ptr(y), M, Cout, Kp, bn, rowpack)]

    def _stem_wgrad(self, dy):
        """ops of the stem's weight gradient from dy [M, Cout] into the padded fp32 buffer. It is complete after the next
        ordered reduce; _stem_unpad then adds it into the gradient arena."""
        _, Cout, M, _, Kp = self._stem
        return [("dfd_memset_async", (_ptr(self.stem_gpad), 0, Cout * Kp * 4)),
                self._wgrad(dy, _ptr(self.stem_cols), _ptr(self.stem_gpad), M, Cout, Kp)]

    def _stem_unpad(self):
        wname, Cout, _, taps, Kp = self._stem
        return ("dfd_unpad_grad", (_ptr(self.stem_gpad), self._g32(wname), Cout, taps, Kp))

    def _alloc_bn(self, bn_specs, extra_stats=0):
        """per-BN pointers into the parameter / running-stat arenas + the per-step statistic and coefficient arenas.
        extra_stats: fp64 values appended to the statistics arena (zeroed with it every step) for statistics that several
        BatchNorms share; they start at element 4 * S * tot_c + 8, returned"""
        dev, S = self.device, self.L.stat_slots
        tot_c = sum((c + 3) // 4 * 4 for _, c in bn_specs)
        self.bnstate = torch.zeros(7 * tot_c, dtype=torch.float32, device=dev)      # scale shift mean rstd cA cB cC
        # fsum fsq bs1 bs2 (+ loss/correct)
        self.stats = torch.zeros(4 * S * tot_c + 8 + extra_stats, dtype=torch.float64, device=dev)
        self.bns = {}
        co = 0
        for name, c in bn_specs:
            bn = _BN()
            bn.name, bn.C = name, c
            bn.gamma = _ptr(self.params32, self.p_off[name + ".weight"][0])
            bn.beta = _ptr(self.params32, self.p_off[name + ".bias"][0])
            bn.dgamma = _ptr(self.grads32, self.p_off[name + ".weight"][0])
            bn.dbeta = _ptr(self.grads32, self.p_off[name + ".bias"][0])
            bn.rm = _ptr(self.buffers32, self.b_off[name + ".running_mean"][0])
            bn.rv = _ptr(self.buffers32, self.b_off[name + ".running_var"][0])
            bn.nbt = _ptr(self.nbt, self.bn_names.index(name))
            for i, f in enumerate(("scale", "shift", "mean", "rstd", "cA", "cB", "cC")):
                setattr(bn, f, _ptr(self.bnstate, i * tot_c + co))
            # per layer [fsum | fsq | bs1 | bs2], S slots x C doubles each: the forward pair and the backward pair are contiguous
            # (one collective each under synchronised BatchNorm)
            for i, f in enumerate(("fsum", "fsq", "bs1", "bs2")):
                setattr(bn, f, _ptr(self.stats, (4 * co + i * c) * S))
            bn.stat_off = 4 * co * S
            co += (c + 3) // 4 * 4
            self.bns[name] = bn
        self.scalars = torch.zeros(4, dtype=torch.float32, device=dev)     # loss_acc, correct_acc, (spare)
        return 4 * S * tot_c + 8


    def _build(self):
        from .engine_densenet import build_densenet
        from .engine_efficientnet import build_efficientnet
        from .engine_resnet import build_resnet
        from .engine_xception import build_xception
        self._keep, self.acts = [], {}
        self._masks = []            # dfd_rng_masks table: (tensor, rows, width, keep_prob), see _mask_head
        self.x_in = torch.zeros(self.N, self.spec.in_chans, self.H, self.W, dtype=self.tdtype, device=self.device)
        {"resnet": build_resnet, "xception": build_xception, "densenet": build_densenet}.get(self.spec.family, build_efficientnet)(self)

    # ---- plan helpers shared by the family builders ---------------------------------------------------------------------
    # pointers to a parameter's fp32 value and gradient, its 16-bit copy and the transposed 16-bit copy of a 1x1 weight
    def _p32(self, name):
        return _ptr(self.params32, self.p_off[name][0])

    def _g32(self, name):
        return _ptr(self.grads32, self.p_off[name][0])

    def _p16(self, name):
        return _ptr(self.params16, self.p_off[name][0])

    def _t16(self, name):
        return _ptr(self.paramsT16, self.t_off[name][0])

    def _stats(self, bn):
        """a forward producer's (sum, sum of squares) operands for `bn`, training-only (NULL in eval mode). Every producer
        passes NULL for its finalisation-descriptor operand: a finalise op of its own follows it."""
        if bn is None:
            return None, None
        return ("TRAIN_ONLY", bn.fsum), ("TRAIN_ONLY", bn.fsq)

    def _gemm(self, A, B, C, M, Nn, K, bn=None, rowpack=True):
        """C [M, Nn] = A [M, K] . B [Nn, K]^T (+ the batch statistics of `bn` over C)"""
        if self.gemm_impl != "tc":
            return ("dfd_gemm_tn_mma", (A, B, C, None, M, Nn, K, self.dt) + self._stats(bn))
        fs, fq = self._stats(bn)
        pack = self._row_pack(M, K) if rowpack else 1
        if pack > 1:
            return ("dfd_gemm_tn_rowpack", (A, self._blockdiag(B, Nn, K, pack), C, M, Nn, K, pack, self.dt, fs, fq, None))
        return ("dfd_gemm_tn", (A, B, C, M, Nn, K, self.dt, fs, fq, None))

    def _finalize(self, bn, count):
        """ops that finalise `bn` over `count` elements per rank: batch statistics -> scale / shift and the running
        statistics in training, running statistics -> scale / shift in eval (once per weight state, see forward).
        Synchronised BatchNorm finalises the SUM of every rank's statistics against the global count (torch SyncBatchNorm)."""
        args = [bn.fsum, bn.fsq, float(count), bn.gamma, bn.beta, bn.rm, bn.rv, bn.nbt, self.bn_momentum, self.bn_eps,
                "TRAINING", bn.C, bn.scale, bn.shift, bn.mean, bn.rstd]
        if self.sync_bn:
            return [("ALLREDUCE_train", (self.stats[bn.stat_off:bn.stat_off + 2 * self.L.stat_slots * bn.C], "sum")),
                    ("dfd_bn_finalize_sync", args)]
        return [("dfd_bn_finalize", args)]

    def _bwd_finalize(self, bn, count):
        """ops that turn the backward sums of `bn` into the coefficients of dy.
        Synchronised BatchNorm averages (sum g, sum g*xhat) over the ranks and keeps the LOCAL count: the coefficients then use
        the global means, and dgamma / dbeta receive global_sum / world - what the DDP gradient mean of the per-rank sums gives."""
        op = ("dfd_bn_bwd_finalize", (bn.bs1, bn.bs2, float(count), bn.gamma, bn.mean, bn.rstd, bn.dgamma, bn.dbeta,
                                      bn.cA, bn.cB, bn.cC, bn.C))
        if self.sync_bn:
            S = self.L.stat_slots
            return [("ALLREDUCE", (self.stats[bn.stat_off + 2 * S * bn.C:bn.stat_off + 4 * S * bn.C], "avg")), op]
        return [op]

    def _bn_apply(self, g, y, bn, out, hw, C):
        """out = the gradient of the input y of `bn` from the gradient g of its output (the coefficients of _bwd_finalize)"""
        return ("dfd_bn_bwd_apply", (g, _ptr(y), None, bn.cA, bn.cB, bn.cC, out, self.N, hw, C, self.dt))

    def _pool_head(self, feat, bn, act, hw, drop_rate, partial=None):
        """forward ops from the features feat [N, hw, F] to the classifier's input `pooled` [N, P]: the global pool (with `bn`,
        feat is that BatchNorm's input and the BatchNorm and `act` are applied on load), then dropout at `drop_rate` (a
        mask drawn at the head of the training forward). Allocates the head's tensors; `partial` goes to dfd_pool as is."""
        spec, N, dev = self.spec, self.N, self.device
        F, P, K = spec.num_features, spec.pooled_features, spec.num_classes
        pool_t = _lib.POOL_TYPES[spec.global_pool]
        scale, shift = (bn.scale, bn.shift) if bn is not None else (None, None)
        self._head = (feat, bn, act, hw)
        self.pooled = torch.zeros(N, P, dtype=torch.float32, device=dev)
        if pool_t == _lib.POOL_TYPES["avg"]:
            ops = [("dfd_pool", (_ptr(feat), scale, shift, _ptr(self.pooled), N, hw, F, act, self.dt, partial, POOL_CHUNKS))]
        else:
            # max / avgmax / catavgmax: one pass gives the mean (dfd_pool's order), the max and its argmax for the backward
            self.pool_argmax = torch.zeros(N, F, dtype=torch.int32, device=dev)
            ops = [("dfd_global_pool", (_ptr(feat), scale, shift, _ptr(self.pooled), _ptr(self.pool_argmax), N, hw, F, act,
                                        pool_t, self.dt, POOL_CHUNKS))]
        self.dropout_mask = None
        if drop_rate > 0.0:
            # F.dropout on the pooled vector, with a mask already divided by keep
            self.dropout_mask = torch.ones(N, P, dtype=torch.float32, device=dev)
            self._masks.append((self.dropout_mask, N * P, 1, 1.0 - drop_rate))
            ops.append(("dfd_mul_f32_train", (_ptr(self.pooled), _ptr(self.dropout_mask), N * P)))
        self.logits = torch.zeros(N, K, dtype=torch.float32, device=dev)
        self.dlogits = torch.zeros(N, K, dtype=torch.float32, device=dev)
        self.dpooled = torch.zeros(N, P, dtype=torch.float32, device=dev)
        self.target_i = torch.zeros(N, dtype=torch.int64, device=dev)
        self.target_f = torch.zeros(N, K, dtype=torch.float32, device=dev)
        return ops

    def _pool_head_bwd(self, gx):
        """backward ops of _pool_head from dlogits into gx [N, hw, F]: the classifier's gradients, the dropout mask, the pool.
        With a BatchNorm, gx is the gradient of the BatchNorm's output (through `act`), and its backward sums are reduced."""
        feat, bn, act, hw = self._head
        spec, N, dt = self.spec, self.N, self.dt
        F, P, K = spec.num_features, spec.pooled_features, spec.num_classes
        pool_t = _lib.POOL_TYPES[spec.global_pool]
        avg = pool_t == _lib.POOL_TYPES["avg"]
        ops = [("dfd_head_bwd", (_ptr(self.dlogits), _ptr(self.pooled), self._p32(self.cls_name + ".weight"),
                                 self._g32(self.cls_name + ".weight"), self._g32(self.cls_name + ".bias"), _ptr(self.dpooled),
                                 N, P, K))]
        if self.dropout_mask is not None:
            ops.append(("dfd_mul_f32", (_ptr(self.dpooled), _ptr(self.dropout_mask), N * P)))
        if bn is None and avg:
            ops.append(("dfd_pool_bwd", (_ptr(self.dpooled), gx, N, hw, F, dt)))
        elif bn is None:
            ops.append(("dfd_gpool_bwd", (_ptr(self.dpooled), _ptr(self.pool_argmax), gx, N, hw, F, pool_t, dt)))
        elif avg:
            ops.append(("dfd_act_bwd", (None, _ptr(feat), bn.scale, bn.shift, bn.mean, bn.rstd, None, _ptr(self.dpooled), gx,
                                        N, hw, F, act, dt, bn.bs1, bn.bs2, None)))
        else:
            ops.append(("dfd_act_bwd_gpool", (_ptr(feat), bn.scale, bn.shift, bn.mean, bn.rstd, _ptr(self.dpooled),
                                              _ptr(self.pool_argmax), gx, N, hw, F, act, pool_t, dt, bn.bs1, bn.bs2, None)))
        return ops

    def _mask_head(self, n_drop_block=0):
        """the ops at the head of the training forward that draw the step's masks: the DropBlock sites of
        self._drop_block_table, then the dropout / drop-path masks of self._masks; the generator's step then advances on the
        device"""
        head, masks = [], self._masks
        if n_drop_block:
            head.append(("dfd_memset_async_train", (_ptr(self.drop_block_kept), 0, 8 * n_drop_block)))
            head.append(("dfd_drop_block_masks_train", (_ptr(self._drop_block_table), n_drop_block, _ptr(self.rng_state))))
        if masks:
            raw = b"".join(struct.pack("<Qqifii", _ptr(t), rows, width, keep, si, 0) for si, (t, rows, width, keep) in enumerate(masks))
            self._mask_table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)
            head.append(("dfd_rng_masks_train", (_ptr(self._mask_table), len(masks), _ptr(self.rng_state))))
        if head:
            head.append(("dfd_rng_tick_train", (_ptr(self.rng_state),)))
        return head

    def _finish_plan(self, fwd, bwd, n_drop_block=0):
        """put the mask draws at the head of the forward, resolve the workspace, check every op against the ABI table and
        publish the plan as fwd_ops / bwd_ops: (function, name, args)"""
        fwd = self._mask_head(n_drop_block) + fwd
        bwd = self._patch_workspace(bwd)
        for n, a in fwd + bwd:
            if n.startswith("ALLREDUCE"):
                continue
            codes = _lib.SIGNATURES[base_name(n)]
            if len(a) != len(codes) - 1:
                raise AssertionError("%s: %d args for signature %r" % (n, len(a), codes))
            for v, c in zip(a, codes):
                if isinstance(v, tuple) and v[0] == "TRAIN_ONLY":
                    v = v[1]
                ok = (v is None or isinstance(v, int)) if c == "p" else (
                    isinstance(v, int) if c in "il" else isinstance(v, (int, float)))
                if not (ok or v == "TRAINING"):
                    raise AssertionError("%s: argument %r does not fit code %r" % (n, v, c))
        fn = lambda n: None if n.startswith("ALLREDUCE") else getattr(self.L, base_name(n))
        self.fwd_ops = [(fn(n), n, a) for n, a in fwd]
        self.bwd_ops = [(fn(n), n, tuple(a)) for n, a in bwd]
        self.n_launch["fwd"], self.n_launch["bwd"] = len(fwd), len(bwd)

    # ------------------------------------------------------------------------------------------
    # execution
    # ------------------------------------------------------------------------------------------
    def launch_args(self, name, args, training):
        """the C-ABI arguments (stream excluded) that the planned op `name` runs with in training or eval mode, or None when
        the op does not run in that mode. Eval mode: BatchNorm finalises from the running statistics (training = 0, no batch
        sums), producers write no batch statistics, `_train` ops and ("TRAIN_ONLY", ptr) operands drop out. Training: a
        synchronised BatchNorm counts every rank's elements."""
        if name == "dfd_bn_finalize_sync":
            args = list(args)
            if training:
                args[2] = args[2] * self.sync_world          # global element count behind the summed statistics
            name = "dfd_bn_finalize"
        if name in ("dfd_bn_finalize", "dfd_bn_finalize_ld"):
            args = tuple((1 if training else 0) if a == "TRAINING" else a for a in args)
            if not training:
                args = (None, None) + args[2:]
        elif name.endswith("_train"):
            if not training:
                return None
        elif any(isinstance(a, tuple) for a in args):
            args = tuple((a[1] if training else None) if isinstance(a, tuple) else a for a in args)
        return args

    def _run(self, ops, stream, training=None, skip_finalize=False):
        if self._plan_only:
            raise _lib.NativeError("plan-only engine cannot execute (no CUDA device)")
        L = self.L
        for fn, name, args in ops:
            if name.startswith("ALLREDUCE"):
                if training:
                    import torch.distributed as dist
                    dist.all_reduce(args[0], op=dist.ReduceOp.SUM if args[1] == "sum" else dist.ReduceOp.AVG)
                continue
            if skip_finalize and name.startswith("dfd_bn_finalize"):
                continue
            args = self.launch_args(name, args, training)
            if args is None:
                continue
            rc = fn(*args, stream)
            _lib.N_CALLS[0] += 1
            if rc != 0:
                raise _lib.NativeError("%s failed (%d): %s" % (name, rc, L.last_error()))

    def set_input(self, x):
        """x: [N, C, H, W] (NCHW, any float dtype / device)."""
        if tuple(x.shape) != tuple(self.x_in.shape):
            raise ValueError("input shape %s != engine shape %s" % (tuple(x.shape), tuple(self.x_in.shape)))
        self.x_in.copy_(x, non_blocking=True)

    def set_target(self, target):
        if target.dtype.is_floating_point:
            self.target_f.copy_(target, non_blocking=True)
            self._soft = True
        else:
            self.target_i.copy_(target, non_blocking=True)
            self._soft = False

    def zero_step_scratch(self, stream, grads=True):
        _lib.call("dfd_memset_async", _ptr(self.stats), 0, self.stats.numel() * 8, stream)
        _lib.call("dfd_memset_async", _ptr(self.scalars), 0, self.scalars.numel() * 4, stream)
        if grads:
            _lib.call("dfd_memset_async", _ptr(self.grads32), 0, self.grads32.numel() * 4, stream)

    def forward(self, training=True, stream=None):
        """Runs the network on self.x_in; logits land in self.logits ([N, num_classes] fp32)."""
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        ar = self.arena
        if training:
            ar.state_version += 1            # running statistics move
            self._run(self.fwd_ops, st, True)
        else:
            # inference: BN is an affine map with constants (running statistics). Its per-channel scale / shift - the
            # "folded" form every consumer kernel applies on load - is computed ONCE per weight state and kept, so a
            # steady-state eval forward launches no BN kernel at all (test_img, validate; dfd/runners/test.py:29-60)
            frozen = self._eval_version == ar.state_version
            self._run(self.fwd_ops, st, False, skip_finalize=frozen)
            self._eval_version = ar.state_version
        return self.logits

    def head(self, with_loss, smoothing=0.0, loss_scale=1.0, soft=False, stream=None, loss_scale_dev=None):
        """classifier (+ fused softmax-CE loss, top-1 count and dL/dlogits when with_loss; any num_classes)."""
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        spec = self.spec
        pw = _ptr(self.params32, self.p_off[self.cls_name + ".weight"][0])
        pb = _ptr(self.params32, self.p_off[self.cls_name + ".bias"][0])
        if with_loss:
            _lib.call("dfd_head_fwd", _ptr(self.pooled), pw, pb, _ptr(self.logits), self.N, spec.pooled_features,
                      spec.num_classes, None if soft else _ptr(self.target_i), _ptr(self.target_f) if soft else None,
                      float(smoothing), float(loss_scale), loss_scale_dev, _ptr(self.scalars), _ptr(self.scalars, 1),
                      _ptr(self.dlogits), st)
        else:
            _lib.call("dfd_head_fwd", _ptr(self.pooled), pw, pb, _ptr(self.logits), self.N, spec.pooled_features,
                      spec.num_classes, None, None, 0.0, 1.0, None, None, None, None, st)

    def backward(self, stream=None):
        """Back-propagates self.dlogits; gradients are ACCUMULATED into self.grads32 (zero it per step)."""
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        self._run(self.bwd_ops, st, True)

    @property
    def loss(self):
        return self.scalars[0]

    @property
    def correct(self):
        return self.scalars[1]
