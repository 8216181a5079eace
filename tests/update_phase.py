"""The update half of the training step: what `Trainer._launch_step` issues after backward (the finite check, the optimizer
kernels over the two arena ranges, Adam's step tick, the loss-scale update, the refresh of every derived weight layout) and the
EMA update behind it. Shared by tests/test_update_phase_cpu.py (which records the C-ABI calls of plan-only engines) and
tests/test_update_phase_gpu.py (which runs them), so that both wire the optimizer exactly as the Trainer does.
"""
import functools
import struct

import torch

import plan_launches as PL
from deepfake_detection_b200.engine import Engine, _ptr
from deepfake_detection_b200.optim import ArenaOptimizer

OPTS = ("sgd", "adam", "adamw", "rmsproptf")
DTYPES = ("bf16", "fp16")            # fp16 trains with dynamic loss scaling (Trainer's default for half precision)
# the batch each configuration runs at on the GPU: it registers the same derived layouts as the shipped batch
# (test_update_phase_cpu checks it); the arenas do not depend on the batch at all
GPU_BATCH = {"b0": 8, "b4": 8, "r50": 8, "r18": 8, "dfv4": 3}
LRS = (0.031, 0.0117)                # [no-decay group, decay group]: different, so a range updated with the other lr shows
HYPER = dict(momentum=0.9, weight_decay=1e-2, eps=1e-3, alpha=0.9)
# kernels of the update phase that no GPU case runs, and why
EXCLUDED = {"dfd_memset_async": "cudaMemsetAsync of the gradient arena (ArenaOptimizer.zero_grad); no kernel of ours"}


def config(tag):
    return next(c for c in PL.CONFIGS if c[0] == tag)


def engine(tag, dtype, batch=None, device=None, share_from=None):
    """the training plan of a configuration (plan-only on the CPU when device == "plan-only")"""
    _, arch, b, res, _, kw = config(tag)
    return Engine(arch, batch or b, res, res, dtype=dtype, device=device, share_from=share_from, **kw)


def arena(tag, dtype, device=None):
    """a parameter-only engine of the configuration: what NativeModel.engine and a ModelEma copy hold"""
    _, arch, _, _, _, kw = config(tag)
    return Engine(arch, 1, dtype=dtype, device=device, params_only=True, **kw)


def make_trainer(eng, opt, use_graph=False, lrs=LRS):
    """a Trainer over an existing plan, wired as Trainer.__init__ wires its own (and as the runner's _trainer_for does):
    fp16 -> dynamic loss scaling, the optimizer reading 1/scale and the skip flag from the device; one lr per group"""
    from deepfake_detection_b200.trainer import Trainer
    tr = Trainer.__new__(Trainer)
    tr.engine = eng
    tr.optimizer = ArenaOptimizer(eng, opt=opt, lr=lrs[0], **HYPER)
    assert len(tr.optimizer.param_groups) == 2
    for g, lr in zip(tr.optimizer.param_groups, lrs):
        g["lr"] = lr
    tr.smoothing = 0.0
    tr.dynamic_scale = eng.tdtype == torch.float16
    tr.scale_window = 2000
    if tr.dynamic_scale:
        a = eng.arena
        a.loss_scale_state.copy_(torch.tensor([65536.0, 1.0 / 65536.0]))
        tr.optimizer.gscale_dev = _ptr(a.loss_scale_state, 1)
        tr.optimizer.skip_flag = _ptr(a.flags, 0)
    tr.use_graph = use_graph
    tr._graph = tr._graph_key = None
    tr.n_captures = 0
    tr.reducer = None
    return tr


def ema_update(dst_arena, src_arena, decay):
    """ModelEma.update between two arenas (the EMA model's arena and the trained one)"""
    from types import SimpleNamespace
    from deepfake_detection_b200.ema import ModelEma
    ModelEma.update(SimpleNamespace(ema=SimpleNamespace(engine=dst_arena), decay=decay), SimpleNamespace(engine=src_arena))


# ---- derived weight layouts -------------------------------------------------------------------------------------------------
def _where(a, ptr):
    """(buffer, element offset) of a 16-bit pointer into the arena's own buffers"""
    for name in ("params16", "paramsT16"):
        t = getattr(a, name)
        if 0 <= ptr - _ptr(t) < t.numel() * t.element_size():
            return name, (ptr - _ptr(t)) // t.element_size()
    for key, wpad in getattr(a, "_stem_reg", {}).items():
        if ptr == _ptr(wpad):
            return "stem", key
    raise KeyError(ptr)


def repack_entries(a):
    """the packed k x k weights of the ResNet path: [(name, O, I, k, element offset)] decoded from the arena's repack table"""
    if not getattr(a, "_rtable_count", 0):
        return []
    raw = bytes(a._rtable.cpu().numpy())
    by_off = {o: n for n, (o, _, _) in a.p_off.items()}
    out = []
    for i in range(a._rtable_count):
        src, dst, dstT, dstD, O, I, k, _ = struct.unpack_from("<QQQQiiii", raw, i * 48)
        buf, off = _where(a, src)
        assert buf == "params16" and a.p_off[by_off[off]][1] == (O, I, k, k)
        d = (dst - _ptr(a.wpack16)) // 2
        assert (dstT - _ptr(a.wpackT16)) // 2 == d and (dstD - _ptr(a.wpackD16)) // 2 == d
        out.append((by_off[off], O, I, k, d))
    return out


def layout_keys(a):
    """the derived layouts an arena holds, without pointers: block-diagonal copies as (source, N, K, pack), the padded stem
    weights, the packed k x k weights"""
    bd = sorted((_where(a, B), Nn, K, pack) for (B, Nn, K, pack) in getattr(a, "_bd_reg", {}))
    stem = sorted(getattr(a, "_stem_reg", {}))
    return bd, stem, sorted(repack_entries(a))


@functools.lru_cache(maxsize=None)
def shipped_layout_keys(tag, dtype):
    return layout_keys(engine(tag, dtype, device="plan-only"))
