"""Guard bands around kernel operands: out-of-bounds stores and reads made visible.

`guard(t)` moves a tensor into the middle of a larger allocation, G bytes of a fixed bit pattern on either side, and
`verify()` reports every guard byte that changed. The caching allocator rounds each tensor up to 512 B and packs it next to
unrelated tensors, so without guards a store one row or channel past the end lands in slack or in a neighbour nobody reads
again, and a read past the end returns the neighbour's finite data. With guards:
  * a store into a guard changes its bytes. The 16-bit and fp32 guards are NaN patterns that no arithmetic produces: the
    H100's fp32 / fp16 / bf16 adds, atomic ones included, return the canonical NaN, so a stored NaN or an atomicAdd into
    such a guard is seen. The fp64 guard is not a NaN: the H100's fp64 atomic add returns a NaN operand bit for bit (a
    non-atomic fp64 add quiets it), so an fp64 atomic into a NaN guard would leave no trace. fp64 operands here are the
    BatchNorm statistics, accumulated by fp64 atomics, so their guard is a tiny normal number (about 1e-305) that any
    non-zero add replaces;
  * a read of a 16-bit or fp32 operand past its end returns NaN and poisons the result, which the checkers' NaN and error
    assertions then catch. A read past an fp64 operand returns the tiny guard value, close to zero, and is caught only
    through its effect on the result.

G is 64 KiB: more than any TMA box (128 rows x 128 B) or one CTA's manual store footprint, and a multiple of 1024 so the
payload keeps the allocator's 512 B alignment (the vectorised and TMA paths are chosen by alignment; a guarded run must
take the same paths as an unguarded one).

Two scopes put the guards in place:
  * guarded_checkers(): the pointer helper P of the kernel checkers (tests/gpu_checks.py and every module that takes P from
    it) guards each tensor the moment a checker takes its pointer, before any descriptor table is packed with that pointer,
    and every `_lib.call` is followed by a synchronise and verify(), so a violation names the entry point;
  * guarded_engine(): every tensor the engine modules allocate is guarded at allocation, before any view of it exists. The
    flat parameter / gradient arenas are guarded as wholes (the optimizer walks them flat; their internal layout is the
    reference state dict's).
"""
import contextlib
import os
import traceback
from collections import namedtuple

import torch

G = 64 * 1024
assert G % 1024 == 0

# per-dtype guard pattern. 16-bit and fp32: a NaN no arithmetic produces (the canonical NaNs are 0x7FC0 / 0x7E00 /
# 0x7FC00000; the H100 returns 0x7FFF / 0x7FFFFFFF). fp64: 0x00A5A5A5A5A5A5A5 = 1.2e-305, a normal number (not a NaN, which
# an fp64 atomic add leaves unchanged, nor a subnormal) below any statistic's ulp, so adding any value of magnitude above
# ~1e-290 changes its bits
_PATTERNS = {
    torch.bfloat16: (torch.int16, 0x7FA5),
    torch.float16: (torch.int16, 0x7DA5),
    torch.float32: (torch.int32, 0x7FA5A5A5),
    torch.float64: (torch.int64, 0x00A5A5A5A5A5A5A5),
}
_BYTE_PATTERN = (torch.uint8, 0xA5)         # integer, bool and uint8 operands

Violation = namedtuple("Violation", "operand side first last")
Violation.__doc__ = """a changed guard: the operand's description, "before" / "after", and the first and last changed byte as
offsets from the payload's first byte (negative before it, >= its size after it)"""


class _Guarded:
    __slots__ = ("big", "nbytes", "dtype", "shape", "where")

    def __init__(self, big, nbytes, dtype, shape, where):
        self.big, self.nbytes, self.dtype, self.shape, self.where = big, nbytes, dtype, shape, where

    @property
    def start(self):
        return self.big.data_ptr() + G

    @property
    def end(self):
        return self.start + self.nbytes

    def describe(self):
        name = str(self.dtype).replace("torch.", "")
        return "%s%s (%d B) allocated at %s" % (name, list(self.shape), self.nbytes, self.where)


_REGISTRY = []              # _Guarded, in guarding order
_BY_BASE = {}               # data_ptr of the whole allocation -> _Guarded
_REF = {}                   # (dtype, device) -> G bytes of the guard pattern


def pattern(dtype):
    """(integer dtype of the element's width, the guard's bit pattern)"""
    return _PATTERNS.get(dtype, _BYTE_PATTERN)


def _ref(dtype, device):
    key = (dtype, str(device))
    if key not in _REF:
        idt, bits = pattern(dtype)
        _REF[key] = torch.empty(G, dtype=torch.uint8, device=device).view(idt).fill_(bits).view(torch.uint8)
    return _REF[key]


def _call_site():
    """file:line (function) of the innermost frame outside this module"""
    for fr in reversed(traceback.extract_stack()[:-1]):
        if os.path.abspath(fr.filename) != os.path.abspath(__file__):
            return "%s:%d (%s)" % (os.path.basename(fr.filename), fr.lineno, fr.name)
    return "?"


def _new_guarded(shape, stride, dtype, device, where):
    """an empty payload of `shape` / `stride` in the middle of a guarded allocation, and its record"""
    shape, stride = tuple(shape), tuple(stride)
    esize = torch.empty(0, dtype=dtype).element_size()
    n = 1
    for s in shape:
        n *= s
    nbytes = n * esize
    big = torch.empty(2 * G + nbytes, dtype=torch.uint8, device=device)
    idt, bits = pattern(dtype)
    big[:G].view(idt).fill_(bits)
    big[G + nbytes:].view(idt).fill_(bits)
    t = torch.empty(0, dtype=dtype, device=device)
    t.set_(big.untyped_storage(), G // esize, shape, stride)
    rec = _Guarded(big, nbytes, dtype, shape, where)
    _REGISTRY.append(rec)
    _BY_BASE[big.data_ptr()] = rec
    return t, rec


def is_guarded(t):
    """t's storage is (part of) a guarded allocation"""
    return t.untyped_storage().data_ptr() in _BY_BASE


def guardable(t):
    """t owns its whole storage, densely: not a view, no offset, no slack (moving it cannot split it from a view)"""
    return (t._base is None and t.storage_offset() == 0 and t.is_contiguous()
            and t.untyped_storage().nbytes() == t.numel() * t.element_size())


def guard(t, where=None):
    """move `t` (which must own its whole storage) into the middle of a guarded allocation; every Python reference to t
    sees the moved storage. Returns t."""
    if is_guarded(t):
        raise ValueError("already guarded")
    if not guardable(t):
        raise ValueError("guard() takes a tensor that owns its whole storage, not a view or part of a storage "
                         "(moving a view's base would split it from the view)")
    moved, _ = _new_guarded(t.shape, t.stride(), t.dtype, t.device, where or _call_site())
    with torch.no_grad():               # a leaf that requires grad (an autograd reference input) moves as well
        moved.copy_(t)
        t.set_(moved.untyped_storage(), moved.storage_offset(), moved.size(), moved.stride())
    return t


def alloc(shape, dtype, device, fill=None, where=None):
    """a new guarded tensor, contiguous; fill None leaves the payload uninitialised (as torch.empty)"""
    shape = tuple(shape)
    stride, acc = [], 1
    for s in reversed(shape):
        stride.append(acc)
        acc *= max(s, 1)
    t, _ = _new_guarded(shape, tuple(reversed(stride)), dtype, device, where or _call_site())
    if fill is not None:
        t.fill_(fill)
    return t


def registered():
    return list(_REGISTRY)


def rearm():
    """write every guard's pattern again (after a reported violation, to locate it by a second run)"""
    for r in _REGISTRY:
        idt, bits = pattern(r.dtype)
        r.big[:G].view(idt).fill_(bits)
        r.big[G + r.nbytes:].view(idt).fill_(bits)


def reset():
    """forget every guard (the allocations are freed with their last reference)"""
    del _REGISTRY[:]
    _BY_BASE.clear()


class Spans:
    """lookup of the guarded payload holding an address"""

    def __init__(self, records=None):
        recs = sorted(_REGISTRY if records is None else records, key=lambda r: r.start)
        self.starts = [r.start for r in recs]
        self.recs = recs

    def find(self, ptr, nbytes=1):
        """the record whose payload holds bytes [ptr, ptr + nbytes), or None"""
        import bisect
        i = bisect.bisect_right(self.starts, ptr) - 1
        if i >= 0:
            r = self.recs[i]
            if r.start <= ptr and ptr + max(nbytes, 1) <= max(r.end, r.start + 1):
                return r
        return None


_VERIFY_CHUNK = 256         # guards compared per batched launch (2 x 256 x 64 KiB of scratch)


def verify(records=None):
    """list of Violation, one per changed guard side: every guard compared with its pattern on its device, the guards of
    up to _VERIFY_CHUNK tensors of one pattern per reduction"""
    records = _REGISTRY if records is None else records
    groups = {}
    for r in records:
        groups.setdefault((pattern(r.dtype), str(r.big.device)), []).append(r)
    flagged = []
    for recs in groups.values():
        ref = _ref(recs[0].dtype, recs[0].big.device)
        for i in range(0, len(recs), _VERIFY_CHUNK):
            part = recs[i:i + _VERIFY_CHUNK]
            lo = torch.stack([r.big[:G] for r in part])
            hi = torch.stack([r.big[G + r.nbytes:] for r in part])
            bad = torch.stack(((lo != ref).any(1), (hi != ref).any(1)), 1).tolist()
            flagged += [(r, b) for r, b in zip(part, bad) if b[0] or b[1]]
    out = []
    order = {id(r): i for i, r in enumerate(records)}
    for r, (lo, hi) in sorted(flagged, key=lambda x: order[id(x[0])]):
        ref = _ref(r.dtype, r.big.device)
        for side, bad, region, base in (("before", lo, r.big[:G], -G), ("after", hi, r.big[G + r.nbytes:], r.nbytes)):
            if bad:
                idx = (region != ref).nonzero().flatten()
                out.append(Violation(r.describe(), side, base + int(idx[0]), base + int(idx[-1])))
    return out


def format_violations(vs):
    return "; ".join("%s: %s the payload, bytes %d..%d" % (v.operand, v.side, v.first, v.last) for v in vs)


class GuardViolation(AssertionError):
    pass


# ---------------------------------------------------------------------------------------------------------------------------
# the kernel checkers
# ---------------------------------------------------------------------------------------------------------------------------
# every module that takes the pointer helper P from tests/gpu_checks.py binds it by name: each must be patched (the CPU test
# finds them with an AST scan and holds this tuple to it)
CHECKER_MODULES = ("gpu_checks", "family_checks", "tf_same_checks")

UNGUARDED = []          # pointer operands left unguarded: views P could not move, pointers packed raw into a table


def _guarding_P(t):
    if t is None:
        return None
    if not is_guarded(t):
        if guardable(t):
            guard(t)
        else:
            UNGUARDED.append("%s%s view at %s" % (str(t.dtype).replace("torch.", ""), list(t.shape), _call_site()))
    return t.data_ptr()


# entry points that read a host-packed table of pointers: name -> (struct format of one entry, offsets of its pointers).
# A checker that packs raw data_ptr()s instead of P()s would hand the kernel unguarded operands; the packed pointers are
# decoded before each launch and every one outside a guarded payload is recorded in UNGUARDED.
TABLES = {
    "dfd_transpose_weights": ("<QQii", (0, 1)),
    "dfd_repack_weights": ("<QQQQiiii", (0, 1, 2, 3)),
    "dfd_blockdiag_weights": ("<QQiiii", (0, 1)),
    "dfd_ordered_reduce": ("<QQqqii", (0, 1)),
}


def _check_table(name, args):
    if name not in TABLES:
        return
    import struct
    fmt, ptrs = TABLES[name]
    size = struct.calcsize(fmt)
    table, count = args[0], args[1]
    rec = Spans().find(table, size * count)
    if rec is None:
        UNGUARDED.append("%s: the table at %#x" % (name, table))
        return
    off = table - rec.start
    raw = rec.big[G + off:G + off + size * count].cpu().numpy().tobytes()
    spans = Spans()
    for i in range(count):
        entry = struct.unpack_from(fmt, raw, i * size)
        for j in ptrs:
            if entry[j] and spans.find(entry[j]) is None:
                UNGUARDED.append("%s: entry %d, pointer %d (%#x) outside every guarded payload" % (name, i, j, entry[j]))


@contextlib.contextmanager
def guarded_checkers():
    """inside: the checkers guard every tensor they take a pointer of, and each `_lib.call` is followed by a synchronise
    and a verify() that raises GuardViolation naming the entry point. On exit the guards are verified once more and
    forgotten."""
    import importlib

    from deepfake_detection_b200 import _lib
    mods = [importlib.import_module(m) for m in CHECKER_MODULES]
    saved_P = [m.P for m in mods]
    real_call = _lib.call

    def call(name, *args):
        _check_table(name, args)
        rc = real_call(name, *args)
        torch.cuda.synchronize()
        vs = verify()
        if vs:
            raise GuardViolation("%s: %s" % (name, format_violations(vs)))
        return rc

    reset()
    del UNGUARDED[:]
    for m in mods:
        m.P = _guarding_P
    _lib.call = call
    try:
        yield
        vs = verify()
        if vs:
            raise GuardViolation(format_violations(vs))
    finally:
        for m, p in zip(mods, saved_P):
            m.P = p
        _lib.call = real_call
        reset()


# ---------------------------------------------------------------------------------------------------------------------------
# whole plans
# ---------------------------------------------------------------------------------------------------------------------------
# the modules that allocate an engine's device tensors (and the optimizer's state over its arenas); each gets the torch
# stand-in below
ENGINE_MODULES = ("deepfake_detection_b200.engine", "deepfake_detection_b200.engine_efficientnet",
                  "deepfake_detection_b200.engine_resnet", "deepfake_detection_b200.engine_xception",
                  "deepfake_detection_b200.optim")


def _shape_of(size):
    return tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else tuple(size)


class _GuardedTorch:
    """`torch` for the engine modules: zeros / empty / full / ones (and their *_like) and cat allocate guarded; everything
    else is torch's own"""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def _new(shape, fill, dtype=None, device=None, **kw):
        dtype = dtype if dtype is not None else torch.get_default_dtype()
        return alloc(shape, dtype, torch.device(device) if device is not None else torch.device("cpu"), fill,
                     where=_call_site())

    def empty(self, *size, dtype=None, device=None, **kw):
        return self._new(_shape_of(size), None, dtype, device)

    def zeros(self, *size, dtype=None, device=None, **kw):
        return self._new(_shape_of(size), 0, dtype, device)

    def ones(self, *size, dtype=None, device=None, **kw):
        return self._new(_shape_of(size), 1, dtype, device)

    def full(self, size, fill_value, dtype=None, device=None, **kw):
        return self._new(_shape_of((size,)), fill_value, dtype, device)

    def _like(self, t, fill, dtype=None, device=None):
        return self._new(t.shape, fill, dtype or t.dtype, device or t.device)

    def empty_like(self, t, dtype=None, device=None, **kw):
        return self._like(t, None, dtype, device)

    def zeros_like(self, t, dtype=None, device=None, **kw):
        return self._like(t, 0, dtype, device)

    def ones_like(self, t, dtype=None, device=None, **kw):
        return self._like(t, 1, dtype, device)

    def full_like(self, t, fill_value, dtype=None, device=None, **kw):
        return self._like(t, fill_value, dtype, device)

    def cat(self, tensors, *args, **kw):
        out = torch.cat(tensors, *args, **kw)
        guard(out, where=_call_site())
        return out


@contextlib.contextmanager
def guarded_engine():
    """inside: every device tensor an Engine allocates is guarded at allocation (Engine._alloc16 and the engine modules'
    torch). The guards outlive the scope with the engine; verify() checks them until reset()."""
    import importlib

    from deepfake_detection_b200.engine import Engine
    mods = [importlib.import_module(m) for m in ENGINE_MODULES]
    saved = [m.torch for m in mods]
    real_alloc16 = Engine._alloc16

    def _alloc16(self, *shape):
        t = alloc(shape, self.tdtype, self.device, where=_call_site())
        self._keep.append(t)
        return t

    stand_in = _GuardedTorch()
    for m in mods:
        m.torch = stand_in
    Engine._alloc16 = _alloc16
    try:
        yield
    finally:
        for m, t in zip(mods, saved):
            m.torch = t
        Engine._alloc16 = real_alloc16
