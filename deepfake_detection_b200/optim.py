"""Flat-arena optimizers for the native engine (drop-in for the `torch.optim.Optimizer` protocol the runner uses).

Mirrors `dfd.timm.optim.create_optimizer` (dfd/timm/optim/optim_factory.py:26-100) for nine of its optimizers —
`sgd` (always nesterov, optim_factory.py:48-50), `adam`, `adamw`, `rmsproptf`, `radam` (radam.py), `adadelta` and
`rmsprop` (torch.optim, rho / alpha 0.9), `novograd` (novograd.py) and `nvnovograd` (nvnovograd.py) —
including its parameter-group split (`add_weight_decay`, optim_factory.py:11-23: 1-D tensors and biases get
weight_decay 0; group order is [no_decay, decay]; with `weight_decay == 0` or `filter_bias_and_bn=False` the
reference passes ONE group of `model.parameters()`, optim_factory.py:34-38, and so does this class) and the AdamW
weight-decay rescale, which the factory applies to `radam` too (optim_factory.py:29-33).  `nadam`, `lookahead_*`
(optim_factory.py:96-98) and the apex `fused*` names are not on the native path and are rejected by name instead of being
silently reduced to another optimizer.

NovoGrad and NvNovoGrad are layer-wise: each tensor's update depends on the L2 norm of its gradient.  Those norms come
from `dfd_tensor_sumsq` over a table of chunks built here at construction, and the per-tensor state (NovoGrad's `v` and
`grad_ema`, NvNovoGrad's `exp_avg_sq`) lives in small fp32 device arrays indexed by tensor.  NovoGrad takes its weight
decay, betas and eps from its constructor (novograd.py:20,41,69): the factory passes weight_decay 0 whenever it split the
groups, so with the default `filter_bias_and_bn=True` NovoGrad applies no decay at all, as the reference does.  Its first
applied step re-initialises every tensor's state (novograd.py:30-46), also after `load_state_dict`, because the reference's
`_momentum_initialized` is not part of its state_dict.  Unlike the reference, neither NovoGrad overwrites the gradients:
the gradient arena is left as backward wrote it.

`param_groups[i]['lr']` is re-read on every step because the schedulers mutate it
(dfd/timm/scheduler/scheduler.py:81-85).  The value travels to the device in a 1-block launch (`dfd_set_floats`,
`push_hyper`) and the update kernels read it from device memory, so a CUDA graph captured around `step()` stays
valid across every scheduler update; the step count lives on the device too (`dfd_opt_tick`) and does not
advance on an fp16-overflow-skipped step (apex semantics); a skipped step changes no state at all.

One kernel launch per arena range updates fp32 master weights, optimizer state and the 16-bit copies the conv
kernels read; further launches refresh the derived weight layouts.
"""
import struct
from collections import OrderedDict

import torch

from . import _lib
from .arch import is_no_decay
from .engine import _ptr

_KINDS = {"sgd": ("sgd", 1), "adam": ("adam", 0), "adamw": ("adamw", 0), "rmsproptf": ("rmsproptf", 0),
          "radam": ("radam", 0), "adadelta": ("adadelta", 0), "rmsprop": ("rmsprop", 0), "novograd": ("novograd", 0),
          "nvnovograd": ("nvnovograd", 0)}
SUPPORTED = ", ".join(_KINDS)
_LAYERWISE = ("novograd", "nvnovograd")
_TICKED = ("adam", "adamw", "radam", "adadelta", "rmsprop", "novograd", "nvnovograd")   # kinds with a `step` in their state
# betas where the factory leaves the class default (radam.py:12; novograd.py:13; nvnovograd.py:33)
_DEFAULT_BETAS = {"novograd": (0.95, 0.98), "nvnovograd": (0.95, 0.98)}
LW_CHUNK = 4096            # elements per chunk of the layer-wise table (a chunk never straddles a tensor)


class ArenaOptimizer:
    def __init__(self, engine, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, eps=1e-8, betas=None,
                 alpha=0.9, filter_bias_and_bn=True, rho=0.9):
        opt_lower = opt.lower()
        opt_split = opt_lower.split("_")
        if len(opt_split) > 1:
            # optim_factory.py:96-98 wraps the base optimizer in Lookahead for `lookahead_<name>`: a different algorithm
            raise ValueError("optimizer %r: Lookahead wrappers are not on the native hot path "
                             "(supported: %s)" % (opt, SUPPORTED))
        if opt_lower not in _KINDS:
            raise ValueError("optimizer %r is not on the native hot path (supported: %s)" % (opt, SUPPORTED))
        self.engine = e = getattr(engine, "arena", engine)      # the owner of the parameter / gradient arenas
        self.kind, self.nesterov = _KINDS[opt_lower]
        wd = float(weight_decay)
        if self.kind in ("adamw", "radam") and wd and lr:
            wd /= lr  # optim_factory.py:29-33
        if betas is None:
            betas = _DEFAULT_BETAS.get(self.kind, (0.9, 0.999))
        base = dict(lr=float(lr), momentum=float(momentum), eps=float(eps), betas=tuple(betas), alpha=float(alpha))
        if self.kind == "adadelta":
            base["rho"] = float(rho)
        elif self.kind == "nvnovograd":
            base.update(grad_averaging=False, amsgrad=False)        # nvnovograd.py:42-46 (the step reads both)
        split = bool(wd and filter_bias_and_bn)
        # NovoGrad's decay is its constructor's (novograd.py:20,41,69): the factory passes 0 there when it split the groups
        self.novograd_wd = 0.0 if split else wd
        if split:
            # ranges of the flat arena: decay tensors first, then no-decay tensors (engine._layout_params)
            names_nd = [n for n in e.param_names if is_no_decay(n, e.p_off[n][1])]
            names_d = [n for n in e.param_names if not is_no_decay(n, e.p_off[n][1])]
            self.param_groups = [
                dict(base, params=names_nd, weight_decay=0.0, _ranges=[(e.n_decay, e.n_params)]),
                dict(base, params=names_d, weight_decay=wd, _ranges=[(0, e.n_decay)]),
            ]
        else:
            # optim_factory.py:34-38: a single group over model.parameters() (named_parameters order)
            self.param_groups = [dict(base, params=list(e.param_names), weight_decay=wd,
                                      _ranges=[(0, e.n_decay), (e.n_decay, e.n_params)])]
        dev = e.device
        n = e.n_params
        self.state_a = torch.zeros(n, dtype=torch.float32, device=dev)          # momentum / exp_avg / square_avg
        has_b = self.kind not in ("sgd", "novograd", "nvnovograd") and not (self.kind == "rmsprop" and not momentum > 0)
        self.state_b = torch.zeros(n, dtype=torch.float32, device=dev) if has_b else None
        if self.kind == "rmsproptf":
            self.state_a.fill_(1.0)                                            # rmsprop_tf.py:80
        if self.kind in _LAYERWISE:
            self._build_layerwise()
        self.grad_scale = 1.0          # extra factor on the gradients (the DDP mean is taken by the reducer itself)
        self.skip_flag = None          # device int* (fp16 overflow)
        self.gscale_dev = None         # device float*: 1/loss_scale (fp16 dynamic loss scaling)
        # device-resident hyper-parameters: lr of every group, and the step counter of Adam's bias corrections
        self.hyper_dev = torch.zeros(8, dtype=torch.float32, device=dev)
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self._host_steps = 0           # launches of step(); the device counter is the authority (skips do not advance it)
        e.n_launch["opt"] = 5 if self.kind in _LAYERWISE else 3

    def _build_layerwise(self):
        """the chunk table of the layer-wise norms (tensors in arena order, decay range first), its scratch and the
        per-tensor state, all allocated here so that a captured step allocates nothing"""
        e = self.engine
        dev = e.device
        self.lw_names = list(e.p_off)                                  # tensor index -> parameter name (arena order)
        self.lw_index = {nm: t for t, nm in enumerate(self.lw_names)}
        rows, chunk0 = [], []
        for t, nm in enumerate(self.lw_names):
            o, _, k = e.p_off[nm]
            chunk0.append(len(rows))
            for c in range(0, k, LW_CHUNK):
                rows.append((o + c, min(LW_CHUNK, k - c), t))
        chunk0.append(len(rows))
        self.lw_nchunks = len(rows)
        # chunks of each arena range: tensors never cross n_decay
        nd = sum(1 for r in rows if r[0] < e.n_decay)
        self.lw_range_chunks = {(0, e.n_decay): (0, nd), (e.n_decay, e.n_params): (nd, len(rows) - nd)}
        raw = bytearray()
        for off, ln, t in rows:
            raw += struct.pack("<qii", off, ln, t)
        nt = len(self.lw_names)
        self.lw_table = torch.frombuffer(raw, dtype=torch.uint8).to(dev, copy=True)
        self.lw_chunk0 = torch.tensor(chunk0, dtype=torch.int32, device=dev)
        self.lw_partial = torch.zeros(len(rows), dtype=torch.float64, device=dev)
        self.lw_sumsq = torch.zeros(nt, dtype=torch.float32, device=dev)
        # novograd: v, grad_ema; nvnovograd: exp_avg_sq (and an unused row)
        self.lw_state = torch.zeros(2, nt, dtype=torch.float32, device=dev)
        self.lw_coef = torch.zeros(2 * nt, dtype=torch.float32, device=dev)
        self.lw_flags = torch.zeros(2, dtype=torch.int32, device=dev)    # NovoGrad: [initialised, this step initialised]

    # `step_count` mirrors the device counter (reads synchronise; used by state_dict / tests, not on the hot path)
    @property
    def step_count(self):
        if self.engine._plan_only:
            return self._host_steps
        return int(self.step_dev.item())

    @step_count.setter
    def step_count(self, v):
        self._host_steps = int(v)
        if not self.engine._plan_only:
            self.step_dev.fill_(int(v))

    def zero_grad(self, set_to_none=False):
        st = torch.cuda.current_stream().cuda_stream
        _lib.call("dfd_memset_async", _ptr(self.engine.grads32), 0, self.engine.grads32.numel() * 4, st)

    def hyper_signature(self):
        """everything EXCEPT lr that the captured launches bake in (a change re-captures the graph)"""
        sig = (self.kind, self.nesterov, self.grad_scale,
               tuple((g["momentum"], g["weight_decay"], g["eps"], g["betas"], g["alpha"]) for g in self.param_groups))
        if self.kind == "adadelta":
            sig += (tuple(g["rho"] for g in self.param_groups),)
        elif self.kind == "novograd":
            sig += (self.novograd_wd,)
        return sig

    def push_hyper(self, stream=None):
        """current param_groups[i]['lr'] -> device (one tiny launch; call it OUTSIDE a captured graph, before replay)"""
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        lrs = [float(g["lr"]) for g in self.param_groups]
        if len(lrs) > 8:
            raise ValueError("at most 8 parameter groups")
        lrs += [0.0] * (8 - len(lrs))
        _lib.call("dfd_set_floats", _ptr(self.hyper_dev), len(self.param_groups), *lrs, st)

    def step(self, closure=None, stream=None, push=True):
        e = self.engine
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        if push:
            self.push_hyper(st)
        self._host_steps += 1
        if self.kind in _TICKED:
            _lib.call("dfd_opt_tick", _ptr(self.step_dev), self.skip_flag, st)
        if self.kind in _LAYERWISE:
            self._layer_norms(st)
        for gi, g in enumerate(self.param_groups):
            lr_dev = _ptr(self.hyper_dev, gi)
            for lo, hi in g["_ranges"]:
                n = hi - lo
                if n <= 0:
                    continue
                p, gr, p16 = _ptr(e.params32, lo), _ptr(e.grads32, lo), _ptr(e.params16, lo)
                a = _ptr(self.state_a, lo)
                if self.kind == "sgd":
                    _lib.call("dfd_sgd_step", p, gr, a, n, g["lr"], g["momentum"], g["weight_decay"], self.nesterov,
                              self.grad_scale, self.gscale_dev, self.skip_flag, p16, e.dt, lr_dev, st)
                elif self.kind in ("adam", "adamw"):
                    _lib.call("dfd_adam_step", p, gr, a, _ptr(self.state_b, lo), n, g["lr"], g["betas"][0], g["betas"][1],
                              g["eps"], g["weight_decay"], 1 if self.kind == "adamw" else 0, self._host_steps,
                              self.grad_scale, self.gscale_dev, self.skip_flag, p16, e.dt, lr_dev, _ptr(self.step_dev), st)
                elif self.kind == "rmsproptf":
                    _lib.call("dfd_rmsprop_tf_step", p, gr, a, _ptr(self.state_b, lo), n, g["lr"], g["alpha"], g["eps"],
                              g["weight_decay"], g["momentum"], self.grad_scale, self.gscale_dev, self.skip_flag, p16, e.dt,
                              lr_dev, st)
                else:
                    self._step_ext(g, lo, hi, p, gr, p16, a, lr_dev, st)
        e.refresh_weight_layouts(st)

    def _layer_norms(self, st):
        """per-tensor ||g||^2 of the unscaled gradient, then the per-tensor state of the layer-wise kinds"""
        sk, b2, eps = self.skip_flag, self.param_groups[0]["betas"][1], self.param_groups[0]["eps"]
        nt = len(self.lw_names)
        _lib.call("dfd_tensor_sumsq", _ptr(self.engine.grads32), _ptr(self.lw_table), self.lw_nchunks, _ptr(self.lw_chunk0),
                  nt, _ptr(self.lw_partial), _ptr(self.lw_sumsq), self.grad_scale, self.gscale_dev, sk, st)
        if self.kind == "novograd":
            _lib.call("dfd_novograd_prepare", _ptr(self.lw_sumsq), _ptr(self.lw_state[0]), _ptr(self.lw_state[1]),
                      _ptr(self.lw_coef), _ptr(self.lw_flags), _ptr(self.step_dev), nt, b2, eps, sk, st)
        else:
            _lib.call("dfd_nvnovograd_prepare", _ptr(self.lw_sumsq), _ptr(self.lw_state[0]), _ptr(self.lw_coef), nt, b2, eps,
                      sk, st)

    def _step_ext(self, g, lo, hi, p, gr, p16, a, lr_dev, st):
        """one range of radam / adadelta / rmsprop / novograd / nvnovograd (csrc/optim_ext.cu)"""
        e, n, sk = self.engine, hi - lo, self.skip_flag
        b1, b2 = g["betas"]
        if self.kind == "radam":
            _lib.call("dfd_radam_step", p, gr, a, _ptr(self.state_b, lo), n, g["lr"], b1, b2, g["eps"], g["weight_decay"],
                      self.grad_scale, self.gscale_dev, sk, p16, e.dt, lr_dev, _ptr(self.hyper_dev, 0), _ptr(self.step_dev), st)
        elif self.kind == "adadelta":
            _lib.call("dfd_adadelta_step", p, gr, a, _ptr(self.state_b, lo), n, g["lr"], g["rho"], g["eps"], g["weight_decay"],
                      self.grad_scale, self.gscale_dev, sk, p16, e.dt, lr_dev, st)
        elif self.kind == "rmsprop":
            _lib.call("dfd_rmsprop_step", p, gr, a, _ptr(self.state_b, lo) if self.state_b is not None else None, n,
                      g["lr"], g["alpha"], g["eps"], g["weight_decay"], g["momentum"], self.grad_scale, self.gscale_dev, sk,
                      p16, e.dt, lr_dev, st)
        else:
            c0, nc = self.lw_range_chunks[(lo, hi)]
            tab = _ptr(self.lw_table) + 16 * c0
            if self.kind == "novograd":
                _lib.call("dfd_novograd_step", _ptr(e.params32), _ptr(e.grads32), _ptr(self.state_a), tab, nc,
                          _ptr(self.lw_coef), _ptr(self.lw_flags), g["lr"], b1, b2, self.novograd_wd, self.grad_scale,
                          self.gscale_dev, sk, _ptr(e.params16), e.dt, lr_dev, _ptr(self.step_dev), st)
            else:
                _lib.call("dfd_nvnovograd_step", _ptr(e.params32), _ptr(e.grads32), _ptr(self.state_a), tab, nc,
                          _ptr(self.lw_coef), g["lr"], b1, g["weight_decay"], self.grad_scale, self.gscale_dev, sk,
                          _ptr(e.params16), e.dt, lr_dev, st)

    # ---- torch-compatible (de)serialisation so `--resume` works across backends -----------------
    _KEYS = {"sgd": ("momentum_buffer", None), "adam": ("exp_avg", "exp_avg_sq"), "adamw": ("exp_avg", "exp_avg_sq"),
             "rmsproptf": ("square_avg", "momentum_buffer"), "radam": ("exp_avg", "exp_avg_sq"),
             "adadelta": ("square_avg", "acc_delta"), "rmsprop": ("square_avg", "momentum_buffer"), "novograd": ("m", None),
             "nvnovograd": ("exp_avg", None)}
    # per-tensor 0-d state of the layer-wise kinds -> row of lw_state
    _TENSOR_KEYS = {"novograd": ("v", "grad_ema"), "nvnovograd": ("exp_avg_sq",)}
    _TENSOR_STEP = ("adadelta", "rmsprop")        # torch.optim keeps `step` as a 0-d float tensor

    def _per_tensor(self):
        """host copy of the layer-wise per-tensor state, [rows, n_tensors] (one read)"""
        return self.lw_state.cpu() if self.kind in _LAYERWISE else None

    def state_dict(self):
        e = self.engine
        ka, kb = self._KEYS[self.kind]
        state = OrderedDict()
        groups = []
        idx = 0
        steps = self.step_count
        lw = self._per_tensor()
        for g in self.param_groups:
            ids = []
            for name in g["params"]:
                o, s, n = e.p_off[name]
                st = {ka: self.state_a[o:o + n].view(s).clone()}
                if kb is not None and self.state_b is not None:
                    st[kb] = self.state_b[o:o + n].view(s).clone()
                if self.kind != "sgd":
                    st["step"] = torch.tensor(float(steps)) if self.kind in self._TENSOR_STEP else steps
                for row, key in enumerate(self._TENSOR_KEYS.get(self.kind, ())):
                    st[key] = lw[row, self.lw_index[name]].clone().to(e.device)
                state[idx] = st
                ids.append(idx)
                idx += 1
            groups.append({k: v for k, v in g.items() if k not in ("params", "_ranges")} | {"params": ids})
        return {"state": state, "param_groups": groups, "step_count": steps}

    def load_state_dict(self, sd):
        e = self.engine
        ka, kb = self._KEYS[self.kind]
        idx = 0
        steps = None
        for g, gs in zip(self.param_groups, sd["param_groups"]):
            for k, v in gs.items():
                if k != "params":
                    g[k] = v
            for name in g["params"]:
                o, s, n = e.p_off[name]
                st = sd["state"].get(idx)
                if st is not None:
                    self.state_a[o:o + n].copy_(st[ka].reshape(-1))
                    if kb is not None and kb in st and self.state_b is not None:
                        self.state_b[o:o + n].copy_(st[kb].reshape(-1))
                    if "step" in st:
                        steps = int(st["step"])
                    for row, key in enumerate(self._TENSOR_KEYS.get(self.kind, ())):
                        if st.get(key) is not None:     # NovoGrad's grad_ema is None until its first step
                            self.lw_state[row, self.lw_index[name]] = float(st[key])
                idx += 1
        steps = sd.get("step_count", steps)
        if steps is not None:
            self.step_count = int(steps)


def create_optimizer(args, model, filter_bias_and_bn=True):
    """Same signature as dfd.timm.optim.create_optimizer (optim_factory.py:26); `model` is a NativeModel / NativeDDP /
    Engine."""
    model = getattr(model, "module", model)
    engine = getattr(model, "engine", model)
    return ArenaOptimizer(engine, opt=args.opt, lr=args.lr, momentum=getattr(args, "momentum", 0.9),
                          weight_decay=args.weight_decay, eps=getattr(args, "opt_eps", 1e-8),
                          filter_bias_and_bn=filter_bias_and_bn)
