"""One-call train / validate steps over the native engine — the public API `bench.py` and the runner mirror use.

A `Trainer` owns an Engine + ArenaOptimizer (+ the DDP gradient reducer when torch.distributed is initialised) and
executes the body of the reference's hot loop (dfd/runners/train.py:621-637):

    output = model(input); loss = loss_fn(output, target); prec1 = accuracy(output, target)
    optimizer.zero_grad(); loss.backward() [DDP all-reduce]; optimizer.step()

as one replayable sequence of kernel launches, optionally captured in a CUDA graph.  The per-step host
synchronisation + two `.item()` reads of the reference (train.py:639-645) are not part of the step: loss and the
correct-count stay on the device until the caller asks for them.
"""
import torch

from . import _lib
from .engine import Engine, _ptr
from .optim import ArenaOptimizer


class Trainer:
    def __init__(self, arch, batch, height=None, width=None, dtype="bf16", opt="sgd", lr=0.01, momentum=0.9,
                 weight_decay=1e-4, opt_eps=1e-8, smoothing=0.0, num_classes=2, in_chans=3, bn_momentum=0.1,
                 bn_eps=1e-5, use_graph=True, gemm_impl="tc", process_group=None, bucket_mb=4.0, loss_scale=None,
                 scale_window=2000, drop_rate=0.0, drop_path_rate=0.0, opt_alpha=0.9, global_pool="avg",
                 drop_block_rate=0.0):
        self.engine = Engine(arch, batch, height, width, num_classes=num_classes, in_chans=in_chans, dtype=dtype,
                             bn_momentum=bn_momentum, bn_eps=bn_eps, gemm_impl=gemm_impl, drop_rate=drop_rate,
                             drop_path_rate=drop_path_rate, global_pool=global_pool, drop_block_rate=drop_block_rate)
        self.optimizer = ArenaOptimizer(self.engine, opt=opt, lr=lr, momentum=momentum, weight_decay=weight_decay,
                                        eps=opt_eps, alpha=opt_alpha)
        self.smoothing = float(smoothing)
        # fp16: dynamic loss scaling with skip-on-overflow (apex AMP O1 semantics, train.py:353,632-634), entirely on the
        # device: scale / 1/scale / overflow flag / clean-step counter live in engine.loss_scale_state and engine.flags
        # (the engine resolved the dtype string: "float16" / "half" are fp16 too and get the same scaling)
        self.dynamic_scale = (self.engine.tdtype == torch.float16) if loss_scale is None else loss_scale == "dynamic"
        self.scale_window = int(scale_window)
        if self.dynamic_scale:
            e0 = self.engine
            e0.loss_scale_state.copy_(torch.tensor([65536.0, 1.0 / 65536.0]))
            self.optimizer.gscale_dev = _ptr(e0.loss_scale_state, 1)
            self.optimizer.skip_flag = _ptr(e0.flags, 0)
        # every optimizer is graph-captured: learning rates and Adam's step count are device-resident (optim.py)
        self.use_graph = bool(use_graph)
        self._graph = None
        self._graph_key = None
        self.n_captures = 0
        self.reducer = None
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1:
            from .ddp import GradReducer
            self.reducer = GradReducer(self.engine, process_group, bucket_mb=bucket_mb)     # takes the MEAN itself
            self.reducer.broadcast_parameters()
        # host-buffer (end-to-end) entry point: uint8 batches are uploaded on a copy stream into two recycled staging
        # buffers and normalised on the compute stream, so the upload of step i+1 overlaps the kernels of step i
        self._pin_out = torch.empty(4, dtype=torch.float32).pin_memory()
        self._h2d = None

    # ---- state ------------------------------------------------------------------------------------
    def state_dict(self):
        return self.engine.state_dict()

    def load_state_dict(self, sd, strict=True):
        return self.engine.load_state_dict(sd, strict=strict)

    # ---- the step ---------------------------------------------------------------------------------
    def _launch_step(self, soft, part=None):
        """part: None = the whole step; "back" = only the update phase that follows backward and the gradient mean"""
        e = self.engine
        st = torch.cuda.current_stream().cuda_stream
        if part != "back":
            e.zero_step_scratch(st, grads=True)
            e.forward(training=True, stream=st)
            e.head(True, smoothing=self.smoothing, soft=soft, stream=st,
                   loss_scale_dev=_ptr(e.loss_scale_state, 0) if self.dynamic_scale else None)
            if self.reducer is not None:
                self.reducer.backward_and_reduce(e)
            else:
                e.backward(stream=st)
        if self.dynamic_scale:
            _lib.call("dfd_check_finite", _ptr(e.grads32), e.n_params, _ptr(e.flags, 0), st)
        self.optimizer.step(stream=st, push=False)      # learning rates were pushed to the device before the launch / replay
        if self.dynamic_scale:
            _lib.call("dfd_update_loss_scale", _ptr(e.flags, 0), _ptr(e.loss_scale_state, 0), _ptr(e.flags, 1),
                      self.scale_window, _ptr(e.loss_scale_state, 1), st)

    def _graph_signature(self, soft):
        # the learning rate is NOT part of the key: it is read from device memory by the update kernels. The layout generation
        # is: a later plan over the same arena (another batch size) can register derived weight layouts, which replaces the
        # block-diagonal table the captured refresh points to and adds copies only a new capture refreshes
        return (soft, self.smoothing, self.optimizer.hyper_signature(), self.engine.arena.layout_gen)

    def step_resident(self, soft=False):
        """One full train step on the batch already resident in engine.x_in / target_i|target_f."""
        self.engine.arena.state_version += 1     # weights and running statistics move (a graph replay does not run Python)
        self.optimizer.push_hyper()          # param_groups[i]['lr'] of THIS step -> device (outside the captured graph)
        if not self.use_graph:
            self._launch_step(soft)
            return
        key = self._graph_signature(soft)
        if self._graph is None or key != self._graph_key:
            # warm-up launch outside capture (module loading, cudaFuncSetAttribute, tensor-map encoding paths)
            self._launch_step(soft)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._launch_step(soft)
            self._graph, self._graph_key = g, key
            self.n_captures += 1
            return
        self._graph.replay()

    def train_step(self, x, target):
        """x: [N,C,H,W] on any device; target: int64 [N] or float [N, num_classes]. Returns (loss, correct) DEVICE scalars."""
        e = self.engine
        e.set_input(x)
        e.set_target(target)
        self.step_resident(soft=target.dtype.is_floating_point)
        return e.loss, e.correct

    def _host_pipeline(self, mean, std):
        if self._h2d is None:
            from .data import InputNormalizer
            e = self.engine
            c = e.spec.in_chans
            self._h2d = dict(stream=torch.cuda.Stream(device=e.device), slot=0,
                             norm=InputNormalizer(mean, std, max(c // 3, 1), e.tdtype, device=e.device),
                             u8=[torch.empty(e.x_in.shape, dtype=torch.uint8, device=e.device) for _ in range(2)],
                             y=[torch.empty(e.N, dtype=torch.int64, device=e.device) for _ in range(2)],
                             ready=[torch.cuda.Event() for _ in range(2)], free=[torch.cuda.Event() for _ in range(2)])
            for ev in self._h2d["free"]:
                ev.record(torch.cuda.current_stream())
        return self._h2d

    def train_step_host(self, x_pinned, y_pinned, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
        """End-to-end entry: pinned HOST buffers in, loss/correct read back to the host (async: synchronise the current
        stream before reading the returned pinned tensor).

        x_pinned uint8 [N,C,H,W] (what the reference's fast_collate hands its prefetcher, loader.py:14-41): uploaded on a
        copy stream into one of two staging buffers (the upload of the NEXT call overlaps this call's kernels), then
        normalised by `dfd_input_normalize` (loader.py:250-253 as one kernel) straight into the engine's input buffer.
        A 16-bit / float x_pinned is taken as already normalised and copied on the compute stream."""
        e = self.engine
        main = torch.cuda.current_stream()
        if x_pinned.dtype == torch.uint8:
            h = self._host_pipeline(mean, std)
            b = h["slot"]
            h["slot"] ^= 1
            with torch.cuda.stream(h["stream"]):
                h["stream"].wait_event(h["free"][b])            # the step that last read this slot has consumed it
                h["u8"][b].copy_(x_pinned, non_blocking=True)
                h["y"][b].copy_(y_pinned, non_blocking=True)
                h["ready"][b].record(h["stream"])
            main.wait_event(h["ready"][b])
            h["norm"](h["u8"][b], out=e.x_in)
            e.target_i.copy_(h["y"][b], non_blocking=True)
            h["free"][b].record(main)
        else:
            e.x_in.copy_(x_pinned, non_blocking=True)
            e.target_i.copy_(y_pinned, non_blocking=True)
        self.step_resident(soft=False)
        self._pin_out.copy_(e.scalars, non_blocking=True)
        return self._pin_out

    @torch.no_grad()
    def validate_step(self, x, target=None):
        """Eval-mode forward (BN running statistics, no dropout): returns logits [N, num_classes] (device, fp32)
        and, when a target is given, fills engine.loss / engine.correct (train.py:719-731)."""
        e = self.engine
        st = torch.cuda.current_stream().cuda_stream
        e.set_input(x)
        e.zero_step_scratch(st, grads=False)
        e.forward(training=False, stream=st)
        if target is not None:
            e.set_target(target)
            e.head(True, smoothing=0.0, soft=target.dtype.is_floating_point, stream=st)
        else:
            e.head(False, stream=st)
        return e.logits
