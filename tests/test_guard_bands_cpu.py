"""The guard-band machinery of tests/guard_bands.py, without a GPU:
  * the helper on CPU tensors: values and alignment kept, a byte written just past either end (through the backing
    allocation) reported with its side and offset, a canonical NaN in a guard reported, a write inside the payload not,
    views refused;
  * coverage of the plans: every plan-only engine of the launch-geometry harvests (plan_launches.CONFIGS,
    family_launches.FAMILY_CONFIGS, their eval forms, the batch-1 fp16 test_img plans and the plan_variants plans), built
    under guarded_engine(), has every non-null pointer operand of every launch inside a guarded payload, except the
    host-built descriptor tables of ALLOWED_TABLES, whose packed pointers are decoded and held to the same rule; and the
    guarded plan is the unguarded plan launch for launch (kernels, non-pointer arguments, pointer masks);
  * checker coverage: guarded_checkers() patches exactly the modules that take P from tests/gpu_checks.py, and the guarded
    case list of tests/test_guard_bands_gpu.py is what pytest collects from the suites it runs under guards.
"""
import ast
import glob
import os
import struct
import subprocess
import sys
from collections import Counter, OrderedDict

import pytest
import torch

import family_launches as FL
import guard_bands as GB
import plan_launches as PL
import plan_variants as PV
from deepfake_detection_b200 import _lib

G = GB.G


@pytest.fixture(autouse=True)
def _forget_guards():
    GB.reset()
    yield
    GB.reset()


# ---------------------------------------------------------------------------------------------------------------------------
# the helper
# ---------------------------------------------------------------------------------------------------------------------------
DTYPES = [torch.bfloat16, torch.float16, torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8]


def _sample(dtype, shape=(37, 5)):
    g = torch.Generator().manual_seed(0)
    if dtype.is_floating_point:
        return torch.randn(shape, generator=g).to(dtype)
    return torch.randint(0, 100, shape, generator=g).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=[str(d).replace("torch.", "") for d in DTYPES])
def test_guard_keeps_values_and_alignment(dtype):
    t = _sample(dtype)
    keep = t.clone()
    alias = t
    GB.guard(t)
    rec = GB.registered()[-1]
    assert torch.equal(t, keep) and alias is t and GB.is_guarded(t)
    assert t.data_ptr() == rec.big.data_ptr() + G and G % 1024 == 0
    assert t.data_ptr() % 64 == 0 and t.is_contiguous() and tuple(t.shape) == (37, 5)
    assert rec.nbytes == t.numel() * t.element_size()
    assert GB.verify() == []
    # the guards hold the dtype's pattern
    idt, bits = GB.pattern(dtype)
    assert bool((rec.big[:G].view(idt) == bits).all()) and bool((rec.big[G + rec.nbytes:].view(idt) == bits).all())


@pytest.mark.parametrize("dtype", DTYPES, ids=[str(d).replace("torch.", "") for d in DTYPES])
def test_guard_reports_one_element_past_either_end(dtype):
    t = GB.guard(_sample(dtype))
    rec = GB.registered()[-1]
    es = t.element_size()
    rec.big[G + rec.nbytes: G + rec.nbytes + es] = 0xFF         # one element just past the end (every byte changed)
    vs = GB.verify()
    assert [(v.side, v.first, v.last) for v in vs] == [("after", rec.nbytes, rec.nbytes + es - 1)], vs
    assert "allocated at test_guard_bands_cpu.py" in vs[0].operand and str(list(t.shape)) in vs[0].operand
    GB.reset()
    t = GB.guard(_sample(dtype))
    rec = GB.registered()[-1]
    rec.big[G - es: G] = 0xFF                                    # one element just before the start
    vs = GB.verify()
    assert [(v.side, v.first, v.last) for v in vs] == [("before", -es, -1)], vs


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.float64],
                         ids=["bf16", "fp16", "fp32", "fp64"])
def test_guard_reports_a_canonical_nan(dtype):
    """arithmetic yields the canonical NaN, not the guard's pattern: a NaN stored into a guard is seen"""
    t = GB.guard(_sample(dtype))
    rec = GB.registered()[-1]
    es = t.element_size()
    tail = rec.big[G + rec.nbytes + 3 * es: G + rec.nbytes + 4 * es].view(dtype)
    tail.fill_(float("nan"))
    vs = GB.verify()
    # the bytes the canonical NaN differs in (bf16 0x7FC0 against 0x7FA5: the low byte only)
    assert len(vs) == 1 and vs[0].side == "after" and rec.nbytes + 3 * es <= vs[0].first <= vs[0].last < rec.nbytes + 4 * es, vs


def test_guard_ignores_writes_inside_the_payload():
    t = GB.guard(_sample(torch.float32))
    t[0, 0] = float("nan")
    t[-1, -1] = float("inf")
    t.view(-1)[-1] = 0.0
    assert GB.verify() == []


def test_guard_refuses_views():
    x = _sample(torch.float32)
    for v in (x[1:], x[:, 1], x.view(-1), x.t()):
        with pytest.raises(ValueError):
            GB.guard(v)
    with pytest.raises(ValueError):
        GB.guard(torch.empty(8).set_(torch.empty(16).untyped_storage(), 0, (8,), (1,)))     # part of a storage
    GB.guard(x)
    with pytest.raises(ValueError):
        GB.guard(x)                  # already guarded
    assert GB.verify() == []


def test_alloc_fills_and_guards():
    t = GB.alloc((3, 4), torch.float16, "cpu", 1)
    assert t.dtype == torch.float16 and tuple(t.shape) == (3, 4) and bool((t == 1).all()) and GB.is_guarded(t)
    assert GB.verify() == []


# ---------------------------------------------------------------------------------------------------------------------------
# coverage of the plans
# ---------------------------------------------------------------------------------------------------------------------------
# Host-built, read-only descriptor tables (torch.frombuffer(...).to(device) of packed structs): the only pointer operands a
# plan may have outside a guarded payload. The pointers packed inside them are decoded (_table_pointers) and must lie in
# guarded payloads like any other operand.
ALLOWED_TABLES = {
    "_red_table": "dfd_ordered_reduce entries <QQqqii (engine._patch_workspace)",
    "_mask_table": "dfd_rng_masks entries <Qqifii (engine._mask_head)",
    "_drop_block_table": "dfd_drop_block_masks site entries <QQQdiiiiiiii (engine_resnet.drop_block_desc)",
}

# workspace operands: kernel -> index of the pointer argument whose byte size is the next argument
_SIZED = {"dfd_gemm_wgrad": 7, "dfd_conv_wgrad_tc": 11, "dfd_dwconv_bwd": 23, "dfd_dwconv_bwd_pad": 25,
          "dfd_dwconv_bwd_relu": 23}


def _engines():
    """(table, tag, batch, dtype) of every plan-only engine, with the forms (training / eval) checked on it"""
    out = OrderedDict()

    def add(table, tag, batch, dtype, training):
        out.setdefault((table, tag, batch, dtype), set()).add(training)

    for tag, *_ in PL.CONFIGS:
        add("shipped", tag, None, None, True)
        add("shipped", tag, None, None, False)
    for tag in FL.tags():
        add("family", tag, None, None, True)
        add("family", tag, None, None, False)
        add("family", tag, FL.EVAL_BATCH, FL.EVAL_DTYPE, False)
    for p in PV.plans():
        add("shipped", p.tag, p.batch, p.dtype, p.training)
    return list(out.items())


_ENGINES = _engines()


def _engine(table, tag, batch, dtype):
    from deepfake_detection_b200.engine import Engine
    _, arch, b, res, dt, kw = next(c for c in PL.TABLES[table] if c[0] == tag)
    return Engine(arch, batch or b, res, res, device="plan-only", dtype=dtype or dt, **kw)


def _ops(eng, training, head=True):
    """(entry point, C-ABI arguments without the stream) of every launch of the plan in this form, then the head's (with
    the loss in training, logits only in eval)"""
    from deepfake_detection_b200.engine import base_name
    out = []
    for _, name, args in list(eng.fwd_ops) + (list(eng.bwd_ops) if training else []):
        if name.startswith("ALLREDUCE"):
            continue
        args = eng.launch_args(name, args, training)
        if args is not None:
            out.append((base_name(name), tuple(args)))
    if head:
        real = _lib.call
        _lib.call = lambda name, *args: out.append((name, args[:-1]))
        try:
            eng.head(training, stream=0)
        finally:
            _lib.call = real
    return out


def _launches(ops):
    out = OrderedDict()
    for name, args in ops:
        la = PL._split(name, args)
        out[la] = out.get(la, 0) + 1
    return out


def _table_of(eng, ptr):
    for name in ALLOWED_TABLES:
        for owner in (eng, eng.arena):
            t = getattr(owner, name, None)
            if t is not None and t.data_ptr() <= ptr < t.data_ptr() + t.numel():
                return name, t
    return None, None


def _table_pointers(name, t, ptr, count):
    """(pointer, byte extent, what) packed in `count` entries of table `name` from `ptr`"""
    raw = bytes(t.numpy().tobytes())
    off = ptr - t.data_ptr()
    out = []
    if name == "_red_table":
        for i in range(count):
            src, dst, n, stride, parts, _ = struct.unpack_from("<QQqqii", raw, off + 40 * i)
            out += [(src, ((parts - 1) * stride + n) * 4, "reduce partials"), (dst, n * 4, "reduce destination")]
    elif name == "_mask_table":
        for i in range(count):
            p, rows, width, _, _, _ = struct.unpack_from("<Qqifii", raw, off + 32 * i)
            out.append((p, rows * width * 4, "mask"))
    elif name == "_drop_block_table":
        for i in range(count):
            mask, noise, kept, _, N, H, W, C = struct.unpack_from("<QQQdiiii", raw, off + 64 * i)
            out += [(mask, N * H * W * C, "drop-block mask"), (kept, 8, "drop-block kept count")]
            if noise:
                out.append((noise, 1, "drop-block noise"))
    return out


def _derived_layout_pointers(eng):
    """(pointer, byte extent, what) of the derived weight layouts the arena refreshes: the transposed 1x1 table, the packed
    k x k table, the block-diagonal copies and the padded stem weights (sources in params16, destinations their own tensors)"""
    ar = eng.arena
    es = ar.params16.element_size()
    out = []
    raw = bytes(ar._ttable.numpy().tobytes())
    for i in range(ar._ttable_count):
        src, dst, O, I = struct.unpack_from("<QQii", raw, 24 * i)
        out += [(src, O * I * es, "transpose source"), (dst, O * I * es, "transpose destination")]
    if getattr(ar, "_rtable_count", 0):
        raw = bytes(ar._rtable.numpy().tobytes())
        for i in range(ar._rtable_count):
            src, a, b, c, O, I, k, _ = struct.unpack_from("<QQQQiiii", raw, 48 * i)
            out += [(p, O * I * k * k * es, "packed weights") for p in (src, a, b, c)]
    for (B, Nn, K, pack), t in getattr(ar, "_bd_reg", {}).items():
        out += [(B, Nn * K * es, "block-diagonal source"), (t.data_ptr(), pack * Nn * pack * K * es, "block-diagonal copy")]
    for (name, O, taps, Kp), wpad in getattr(ar, "_stem_reg", {}).items():
        out += [(ar.params16.data_ptr() + ar.p_off[name][0] * es, O * taps * es, "stem weight"),
                (wpad.data_ptr(), O * Kp * es, "padded stem weight")]
    return out


def _uncovered(eng, forms):
    """pointer operands outside every guarded payload and outside ALLOWED_TABLES, the table operands met, and the count of
    pointers checked"""
    spans = GB.Spans()
    bad, tables, n = [], set(), 0
    for training in sorted(forms, reverse=True):
        for name, args in _ops(eng, training):
            codes = _lib.SIGNATURES[name]
            for i, (v, c) in enumerate(zip(args, codes)):
                if c != "p" or v is None:
                    continue
                n += 1
                size = args[i + 1] if _SIZED.get(name) == i else (args[2] if name == "dfd_memset_async" else 1)
                if spans.find(v, size) is not None:
                    continue
                tname, t = _table_of(eng, v)
                if tname is None:
                    bad.append("%s arg %d (%s): %#x + %d B" % (name, i, "eval" if not training else "train", v, size))
                    continue
                tables.add(tname)
                for p, ext, what in _table_pointers(tname, t, v, args[i + 1]):
                    n += 1
                    if spans.find(p, ext) is None:
                        bad.append("%s: %s %#x + %d B in %s" % (name, what, p, ext, tname))
    for p, ext, what in _derived_layout_pointers(eng):
        n += 1
        if spans.find(p, ext) is None:
            bad.append("%s %#x + %d B" % (what, p, ext))
    return bad, tables, n


def _unguarded_launches(table, tag, batch, dtype, training):
    if table == "family":
        return FL.plan_launches(tag, batch, training, dtype)
    return PL.plan_launches(tag, batch, training, dtype)


@pytest.mark.parametrize("key,forms", _ENGINES,
                         ids=["%s-%s-N%s-%s-%s" % (k + ("+".join("train" if f else "eval" for f in sorted(fs, reverse=True)),))
                              for k, fs in _ENGINES])
def test_every_plan_operand_is_guarded(key, forms):
    table, tag, batch, dtype = key
    with GB.guarded_engine():
        eng = _engine(table, tag, batch, dtype)
    bad, tables, n = _uncovered(eng, forms)
    assert n > 0 and not bad, "%d of %d pointer operands outside a guarded payload: %s" % (len(bad), n, bad[:20])
    assert tables <= set(ALLOWED_TABLES), tables
    # the same plan as without guards, launch for launch (plan_launches lists the head in the eval form only)
    for training in forms:
        assert _launches(_ops(eng, training, head=not training)) == _unguarded_launches(table, tag, batch, dtype, training), training
    # building the plan wrote no guard byte
    assert GB.verify() == []


def test_guarded_engine_restores_the_modules():
    import importlib

    from deepfake_detection_b200.engine import Engine
    mods = [importlib.import_module(m) for m in GB.ENGINE_MODULES]
    alloc16 = Engine._alloc16
    with GB.guarded_engine():
        assert all(isinstance(m.torch, GB._GuardedTorch) for m in mods)
    assert all(m.torch is torch for m in mods) and Engine._alloc16 is alloc16


# ---------------------------------------------------------------------------------------------------------------------------
# checker coverage
# ---------------------------------------------------------------------------------------------------------------------------
def _modules_taking_P():
    here = os.path.dirname(os.path.abspath(__file__))
    found = set()
    for path in sorted(glob.glob(os.path.join(here, "*.py"))):
        with open(path) as f:
            tree = ast.parse(f.read(), path)
        name = os.path.splitext(os.path.basename(path))[0]
        for node in ast.walk(tree):
            if isinstance(node, ast.ImportFrom) and node.module == "gpu_checks" and any(a.name == "P" for a in node.names):
                found.add(name)
            if isinstance(node, ast.FunctionDef) and name == "gpu_checks" and node.name == "P":
                found.add(name)
    return found


def test_packed_table_pointers_outside_guards_are_recorded():
    """a table entry point whose packed pointers were taken with data_ptr() instead of P: each one is recorded in UNGUARDED"""
    src, dst, raw_dst = GB.alloc((4, 8), torch.bfloat16, "cpu", 0), GB.alloc((8, 4), torch.bfloat16, "cpu", 0), torch.zeros(8, 4)
    rows = [struct.pack("<QQii", src.data_ptr(), dst.data_ptr(), 4, 8), struct.pack("<QQii", src.data_ptr(), raw_dst.data_ptr(), 4, 8)]
    table = GB.guard(torch.frombuffer(bytearray(b"".join(rows)), dtype=torch.uint8).clone())
    del GB.UNGUARDED[:]
    GB._check_table("dfd_transpose_weights", (table.data_ptr(), 1, 0))
    assert GB.UNGUARDED == []
    GB._check_table("dfd_transpose_weights", (table.data_ptr(), 2, 0))
    assert len(GB.UNGUARDED) == 1 and "entry 1, pointer 1" in GB.UNGUARDED[0], GB.UNGUARDED
    del GB.UNGUARDED[:]


def test_guarded_checkers_patch_every_module_taking_P():
    import importlib
    found = _modules_taking_P()
    assert "gpu_checks" in found and "family_checks" in found and "tf_same_checks" in found, found
    assert found == set(GB.CHECKER_MODULES), found
    mods = [importlib.import_module(m) for m in GB.CHECKER_MODULES]
    saved = [m.P for m in mods]
    call = _lib.call
    with GB.guarded_checkers():
        assert all(m.P is GB._guarding_P for m in mods) and _lib.call is not call
    assert [m.P for m in mods] == saved and _lib.call is call


def test_guarded_cases_are_the_collected_suites():
    """the cases tests/test_guard_bands_gpu.py runs under guards, against pytest's own collection of the suites they come
    from: the same ids for the three launch-geometry tests, the same number of parameter sets per test_kernels_gpu test"""
    import test_guard_bands_gpu as TG
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    suites = {"plan": "tests/test_plan_launches_gpu.py::test_plan_launch",
              "variant": "tests/test_plan_variants_gpu.py::test_plan_variant",
              "family": "tests/test_family_launches_gpu.py::test_family_launch"}
    r = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        "tests/test_kernels_gpu.py"] + list(suites.values()), cwd=root, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    items = [ln for ln in r.stdout.splitlines() if "::" in ln]
    ours = [i for i, _ in TG._CASES]
    assert len(set(ours)) == len(ours)
    for prefix, node in suites.items():
        collected = {ln.split("[", 1)[1][:-1] for ln in items if ln.startswith(node + "[")}
        guarded = {i[len(prefix) + 1:] for i in ours if i.startswith(prefix + "-")}
        assert collected and guarded == collected, (prefix, len(guarded), len(collected))
    kernels = Counter(ln.split("::", 1)[1].split("[", 1)[0] for ln in items if ln.startswith("tests/test_kernels_gpu.py::"))
    guarded = Counter(i[len("kernels-"):].split("[", 1)[0] for i in ours if i.startswith("kernels-"))
    assert kernels and guarded == kernels, (guarded, kernels)
    assert len(ours) == len(items), (len(ours), len(items))
