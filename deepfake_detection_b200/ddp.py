"""Data-parallel wrapper and gradient reduction for the native engine (replaces the DDP wrapper at
dfd/runners/train.py:402,406, its unwrap convention dfd/timm/utils.py:25-33, and `reduce_tensor`,
dfd/timm/utils.py:256-260).

One process per GPU (`torch.distributed`, NCCL over NVLink/NVSwitch; gloo for the CPU-side tests).  The engine's
gradients live in ONE flat fp32 arena laid out in forward execution order, so:
  * the backward plan is cut into segments at block boundaries; after segment i the arena suffix that backward has
    finished writing is all-reduced on a side stream while segment i+1 computes — bucketed, overlapped all-reduce
    without per-tensor hooks;
  * the reduction is a MEAN (NCCL `ReduceOp.AVG`; SUM followed by a scale on gloo): after backward the `.grad`
    tensors hold the averaged gradients, exactly what the reference's DDP leaves behind for `optimizer.step()`;
  * BN running statistics stay rank-local (apex DDP semantics, SURVEY.md 8b); `distribute_bn` mirrors utils.py:263-274.

`NativeDDP` is the object the runner sees: `.module` unwraps, calling it runs the model, and the wrapped model's
backward (autograd bridge and fused step alike) goes through `GradReducer.backward_and_reduce`.
"""
import torch
import torch.distributed as dist
import torch.nn as nn

from . import _lib


def reduce_tensor(tensor, n, group=None):
    """dfd/timm/utils.py:256-260"""
    rt = tensor.clone()
    dist.all_reduce(rt, op=dist.ReduceOp.SUM, group=group)
    rt /= n
    return rt


def distribute_bn(model, world_size, reduce=False, group=None):
    """dfd/timm/utils.py:263-274 on the flat running-stat arena (one collective instead of 2 per BN layer).
    `model`: NativeDDP / NativeModel / Engine."""
    model = getattr(model, "module", model)
    engine = getattr(model, "engine", model)
    if reduce:
        dist.all_reduce(engine.buffers32, op=dist.ReduceOp.SUM, group=group)
        engine.buffers32 /= float(world_size)
    else:
        dist.broadcast(engine.buffers32, 0, group=group)
    engine.arena.state_version += 1          # eval plans re-derive their BN scale / shift from the new running statistics


def convert_syncbn_model(model):
    """apex.parallel.convert_syncbn_model / nn.SyncBatchNorm.convert_sync_batchnorm for a NativeModel (train.py:388-394):
    every BatchNorm of the plans built from now on all-reduces its batch statistics (forward) and its BN-backward sums over
    the default process group. Call it before DDP wrapping, as the reference does."""
    m = getattr(model, "module", model)
    if m.spec.family != "efficientnet":
        raise _lib.NativeError("synchronised BatchNorm is implemented for the EfficientNet family")
    m.sync_bn = True
    m._engines.clear()                      # plans built without the collectives are dropped
    m.__dict__.get("_trainers", {}).clear()
    return model


def plan_buckets(spans, bucket_elems):
    """spans: list of (lo, hi) arena ranges in the order backward completes them. Greedily merges consecutive spans
    into buckets of at least `bucket_elems` elements. Returns list of lists of (lo, hi)."""
    buckets, cur, size = [], [], 0
    for lo, hi in spans:
        if hi <= lo:
            continue
        cur.append((lo, hi))
        size += hi - lo
        if size >= bucket_elems:
            buckets.append(cur)
            cur, size = [], 0
    if cur:
        buckets.append(cur)
    return buckets


class GradReducer:
    """Bucketed, overlapped gradient MEAN over the process group.  The arena (weights / gradients) is shared by every
    execution plan of a model, but the cut points are positions in ONE plan's backward op list, so the bucket plan is
    computed (and cached) per engine: `backward_and_reduce(engine)` always replays the plan that ran the forward."""

    def __init__(self, engine, group=None, bucket_mb=4.0):
        # bucket_mb: the arena is cut greedily in backward order. Parameters concentrate in the LAST layers (EfficientNet-B0:
        # 11.6 of 16 MB sit in the head and stages 5-6), so 4 MB buckets start reducing early and leave ~2.6 MB (stages 1-4
        # and the stem) for the one collective that cannot overlap with anything - the final one. 1 MB buckets (12
        # collectives) were slower at 2 GPUs, NCCL CTAs competing with the memory-bound kernels (measured on the GPU this
        # code was first tuned on, not re-measured on the H100)
        self.engine = engine                      # default plan (Trainer) or the arena (NativeDDP)
        self.arena = engine.arena
        self.group = group
        self.world = dist.get_world_size(group)
        self.bucket_mb = float(bucket_mb)
        self.side = None if self.arena._plan_only else torch.cuda.Stream(device=self.arena.device)
        backend = dist.get_backend(group)
        self._avg = backend == "nccl"              # gloo has no AVG: SUM, then scale
        self._plans = {}
        self.n_reduce_calls = 0

    # ---- plan ---------------------------------------------------------------------------------------------
    @property
    def buckets(self):
        return self.plan_for(self.engine)

    def plan_for(self, e):
        key = id(e)
        if key not in self._plans:
            self._plans[key] = (e, self._make_plan(e))      # the engine reference keeps id() unique
        return self._plans[key][1]

    def _make_plan(self, e):
        # cut the backward plan where a block's last gradient has been produced: op index -> arena ranges done.
        # Arena layout = [decay tensors in exec order | no-decay tensors in exec order]; backward walks both from
        # the end towards the start, so after the ops of a block the suffixes starting at that block's first
        # tensors are final.
        from .arch import is_no_decay
        first_d, first_nd = {}, {}
        for n in e.param_names:
            o, s, k = e.p_off[n]
            key = self._owner(n)
            (first_nd if is_no_decay(n, s) else first_d).setdefault(key, o)
        owners = []
        for n in e.param_names:
            k = self._owner(n)
            if k not in owners:
                owners.append(k)
        off_index = sorted((o, o + k, self._owner(n)) for n, (o, s, k) in e.p_off.items())

        def owner_of_offset(off):
            for lo, hi, k in off_index:
                if lo <= off < hi:
                    return k
            return "stem"

        # map plan positions: find the last bwd op that writes into each owner (by gradient pointer range)
        last_op = {}
        g0 = e.grads32.data_ptr()
        g1 = g0 + e.grads32.numel() * 4
        for idx, (_, name, args) in enumerate(e.bwd_ops):
            for a in args:
                if isinstance(a, int) and g0 <= a < g1:
                    last_op[owner_of_offset((a - g0) // 4)] = idx
        n_ops = len(e.bwd_ops)
        prev_d, prev_nd = e.n_decay, e.n_params
        spans_by_op = []
        for k in reversed(owners):
            d_lo = first_d.get(k, prev_d)
            nd_lo = first_nd.get(k, prev_nd)
            spans_by_op.append((last_op.get(k, n_ops - 1), [(d_lo, prev_d), (nd_lo, prev_nd)]))
            prev_d, prev_nd = min(d_lo, prev_d), min(nd_lo, prev_nd)
        # ensure coverage of the arena heads (padding) by the final bucket
        spans_by_op.append((n_ops - 1, [(0, prev_d), (e.n_decay, prev_nd)]))
        # monotone op order, then bucket by size
        bucket_elems = int(self.bucket_mb * 1024 * 1024 / 4)
        buckets = []             # (op index, [(lo, hi), ...])
        cur, size, cur_op = [], 0, 0
        for op_idx, spans in spans_by_op:
            cur_op = max(cur_op, op_idx)
            for lo, hi in spans:
                if hi > lo:
                    cur.append((lo, hi))
                    size += hi - lo
            if size >= bucket_elems:
                buckets.append((cur_op, self._merge(cur)))
                cur, size = [], 0
        if cur:
            buckets.append((n_ops - 1, self._merge(cur)))
        if buckets:
            buckets[-1] = (n_ops - 1, buckets[-1][1])
        return buckets

    @staticmethod
    def _merge(spans):
        spans = sorted(spans)
        out = []
        for lo, hi in spans:
            if out and lo <= out[-1][1]:
                out[-1] = (out[-1][0], max(out[-1][1], hi))
            else:
                out.append((lo, hi))
        return out

    @staticmethod
    def _owner(name):
        parts = name.split(".")
        if parts[0] == "blocks":
            return ".".join(parts[:3])
        if parts[0].startswith("layer"):
            return ".".join(parts[:2])
        if parts[0] in ("conv_head", "bn2", "classifier", "fc"):
            return "head"
        return "stem"

    # ---- collectives ----------------------------------------------------------------------------------------
    def broadcast_parameters(self):
        """Rank-0 weights to every rank at wrap time (DDP constructor semantics, SURVEY.md C6)."""
        a = self.arena
        dist.broadcast(a.params32, 0, group=self.group)
        dist.broadcast(a.buffers32, 0, group=self.group)
        a.state_version += 1
        if not a._plan_only:
            a.sync_weights()

    def _mean(self, t):
        self.n_reduce_calls += 1
        if self._avg:
            dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
            t.mul_(1.0 / self.world)

    def backward_and_reduce(self, engine=None):
        """Runs `engine`'s backward plan (the one whose forward just ran) on the current stream, launching each bucket's
        mean all-reduce on the side stream as soon as the ops that produce it have been enqueued; joins at the end."""
        e = engine if engine is not None else self.engine
        if e.arena is not self.arena:
            raise _lib.NativeError("GradReducer: engine does not share this reducer's gradient arena")
        buckets = self.plan_for(e)
        g = self.arena.grads32
        if e._plan_only:        # host-logic tests (gloo on CPU): no kernels, only the bucketed collectives
            for _, spans in buckets:
                for lo, hi in spans:
                    self._mean(g[lo:hi])
            return
        main = torch.cuda.current_stream()
        st = main.cuda_stream
        start = 0
        for op_idx, spans in buckets:
            e._run(e.bwd_ops[start:op_idx + 1], st, True)
            start = op_idx + 1
            ev = torch.cuda.Event()
            ev.record(main)
            self.side.wait_event(ev)
            with torch.cuda.stream(self.side):
                for lo, hi in spans:
                    self._mean(g[lo:hi])
        if start < len(e.bwd_ops):
            e._run(e.bwd_ops[start:], st, True)
        main.wait_stream(self.side)


class NativeDDP(nn.Module):
    """The DDP object of the boundary (SURVEY.md 8b): `.module` unwraps (utils.py:25-33), calling it forwards to the
    model, parameters are broadcast from rank 0 at wrap time, and every backward of the wrapped NativeModel averages the
    gradients across the group before `optimizer.step()` (train.py:402-406: `DDP(model, delay_allreduce=True)` /
    `DDP(model, device_ids=[local_rank])`).  Extra keyword arguments of either constructor are accepted and ignored."""

    def __init__(self, module, process_group=None, bucket_mb=4.0, delay_allreduce=None, device_ids=None, **unused):
        super().__init__()
        if not (dist.is_available() and dist.is_initialized()):
            raise _lib.NativeError("NativeDDP needs an initialised torch.distributed process group")
        self.module = module
        self.reducer = GradReducer(module.engine, process_group, bucket_mb=bucket_mb)
        module._reducer = self.reducer
        self.reducer.broadcast_parameters()

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def train(self, mode=True):
        self.training = mode
        self.module.train(mode)
        return self

    def named_parameters(self, prefix="", recurse=True, remove_duplicate=True):
        for n, p in self.module.named_parameters():
            yield (prefix + ("." if prefix else "") + "module." + n, p)

    def parameters(self, recurse=True):
        return self.module.parameters()

    def state_dict(self, *args, **kwargs):
        from collections import OrderedDict
        return OrderedDict(("module." + k, v) for k, v in self.module.state_dict().items())

    def load_state_dict(self, state_dict, strict=True):
        sd = {(k[7:] if k.startswith("module.") else k): v for k, v in state_dict.items()}
        return self.module.load_state_dict(sd, strict=strict)
