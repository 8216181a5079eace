"""-m gpu: the kernel checkers and whole training steps with a guard band around every operand (tests/guard_bands.py).

  * Every launch-geometry case (plan_launches.gpu_cases(), plan_variants.variant_cases(), family_launches.gpu_cases()) and
    every parametrisation of tests/test_kernels_gpu.py, through its own checker and assertions, inside guarded_checkers():
    a case passes when its assertions hold and no guard byte changed. Tolerances are the existing tests' own.
  * Whole steps inside guarded_engine(): two captured training steps, a validation forward and a batch-1 fp16 test_img
    forward of each shipped configuration and each model family at the existing step tests' small batches, one ResNet with
    DropBlock, drop path and dropout. These cover what the per-kernel cases leave out (memsets, BatchNorm finalisation,
    the ordered reduce, the optimizer, the arena cast, the derived weight layouts, the loss-scale kernels) at the plans'
    real buffer adjacency. On a violation the step is run again without a graph, verifying after every launch, so the
    failure names the op.
  * Sensitivity: a real kernel writing one row, channel or partial past a deliberately short operand is reported, that
    operand and that side only, for each store style (TMA-stored GEMM epilogue, manual row stores, fp64 statistics atomics,
    split-K workspace). Each overrun is 8 bytes to 16 KiB, inside the 64 KiB guard this test allocated. And the reason the
    fp64 guard is not a NaN: an fp64 atomic add leaves a NaN operand's bits as they were, and changes the guard's.
  * tests/test_guard_bands_cpu.py holds the case list to the suites pytest collects.
"""
import math

import pytest
import torch

import family_launches as FL
import guard_bands as GB
import plan_launches as PL
import plan_variants as PV
import test_family_launches_gpu as TFL
import test_kernels_gpu as TK
import test_plan_launches_gpu as TPL
import test_plan_variants_gpu as TPV

pytestmark = pytest.mark.gpu


def _parametrisations(fn):
    """list of kwargs of every parameter set of a pytest function (its parametrize marks, crossed)"""
    sets = [{}]
    for m in reversed([m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]):
        names = m.args[0]
        names = [a.strip() for a in names.split(",")] if isinstance(names, str) else list(names)
        new = []
        for s in sets:
            for v in m.args[1]:
                v = v.values if type(v).__name__ == "ParameterSet" else ((v,) if len(names) == 1 else tuple(v))
                new.append(dict(s, **dict(zip(names, v))))
        sets = new
    return sets


def _kernel_cases():
    out = []
    for name, fn in vars(TK).items():
        if name.startswith("test_") and callable(fn):
            for kw in _parametrisations(fn):
                ident = "-".join(str(v).replace(" ", "") for v in kw.values())
                out.append(("kernels-%s[%s]" % (name, ident), (lambda fn=fn, kw=kw: fn(**kw))))
    return out


def _cases():
    out = [("plan-" + c.id, (lambda c=c: TPL.CHECKERS[c.check](c.kw, c.dtype))) for c in PL.gpu_cases()]
    out += [("variant-" + c.id, (lambda c=c: TPV.CHECKERS[c.check](c.kw, c.dtype))) for c in PV.variant_cases()]
    out += [("family-" + c.id, (lambda c=c: TFL.CHECKERS[c.check](c.kw, c.dtype))) for c in FL.gpu_cases()]
    return out + _kernel_cases()


_CASES = _cases()


@pytest.fixture(scope="module", autouse=True)
def _report_peak_memory():
    yield
    print("\nguard-band tests: peak device memory %.2f GiB" % (torch.cuda.max_memory_allocated() / 2 ** 30))


@pytest.fixture(autouse=True)
def _free_between_cases():
    GB.reset()
    yield
    GB.reset()
    torch.cuda.empty_cache()        # the GPU is shared: give back what the last (large) case held


@pytest.mark.parametrize("case", _CASES, ids=[i for i, _ in _CASES])
def test_case_under_guards(case):
    with GB.guarded_checkers():
        case[1]()
    assert not GB.UNGUARDED, "pointer operands the checker passed as views of unguarded tensors: %s" % GB.UNGUARDED


# ---------------------------------------------------------------------------------------------------------------------------
# whole steps
# ---------------------------------------------------------------------------------------------------------------------------
# (id, arch, batch, H, W, dtype, extra Trainer kwargs): the shipped configurations and the families at the existing step
# tests' small batches, one ResNet with every stochastic regulariser
STEPS = [
    ("b0", "efficientnet_b0", 8, 96, 96, "bf16", {}),
    ("b4", "efficientnet_b4", 8, 96, 96, "fp16", {}),          # dynamic loss scaling (the fp16 default)
    ("r50", "resnet50", 8, 96, 96, "bf16", {}),
    ("r18", "resnet18", 8, 96, 96, "bf16", {}),
    ("dfv4", "efficientnet_deepfake_v4", 2, 128, 128, "bf16", {"in_chans": 12}),
    ("r34", "resnet34", 8, 96, 96, "bf16", {}),
    ("r101", "resnet101", 8, 96, 96, "bf16", {}),
    ("wrn50", "wide_resnet50_2", 8, 96, 96, "bf16", {}),
    ("r50d", "resnet50d", 8, 96, 96, "bf16", {}),
    ("r26d", "resnet26d", 8, 104, 88, "bf16", {}),
    ("se50", "seresnet50", 8, 64, 64, "bf16", {}),
    ("se18", "seresnet18", 8, 70, 72, "fp16", {}),
    ("xc", "xception", 8, 96, 96, "bf16", {}),
    ("tfb0", "tf_efficientnet_b0", 8, 96, 96, "bf16", {}),
    ("tfb4", "tf_efficientnet_b4_ns", 8, 96, 96, "fp16", {}),
    ("r50d_drop", "resnet50d", 8, 160, 160, "bf16", {"drop_rate": 0.2, "drop_path_rate": 0.1, "drop_block_rate": 0.2}),
]


def _checked(fn, name):
    def run(*args):
        rc = fn(*args)
        torch.cuda.synchronize()
        vs = GB.verify()
        if vs:
            raise GB.GuardViolation("%s: %s" % (name, GB.format_violations(vs)))
        return rc
    return run


def _locate(tr, x, y):
    """the step once more without a graph, verifying after every launch: raises naming the first op that changed a guard"""
    from deepfake_detection_b200 import _lib
    GB.rearm()
    e = tr.engine
    e.fwd_ops = [(_checked(fn, n) if fn is not None else None, n, a) for fn, n, a in e.fwd_ops]
    e.bwd_ops = [(_checked(fn, n) if fn is not None else None, n, a) for fn, n, a in e.bwd_ops]
    real = _lib.call
    _lib.call = lambda name, *args: _checked(real, name)(name, *args)
    try:
        tr.use_graph = False
        tr.train_step(x, y)
    finally:
        _lib.call = real


@pytest.mark.parametrize("cfg", STEPS, ids=[s[0] for s in STEPS])
def test_whole_step_under_guards(cfg):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.trainer import Trainer
    from oracle.weights import synth_batch, synth_state
    _, arch, n, h, w, dtype, kw = cfg
    cin = kw.get("in_chans", 3)
    spec = get_spec(arch, in_chans=cin)
    sd = synth_state(spec, seed=7)
    if spec.family == "resnet":
        # damp the residual branches as engine_checks.run_parity(tame=True) does: with gamma ~ 1 in every block the deep
        # ResNets' activations overflow fp16 in the batch-1 forward, and NaN logits would hide a poisoned read
        for b in spec.blocks:
            k = b.name + (".bn2.weight" if b.kind == "basic" else ".bn3.weight")
            sd[k] = sd[k] * 0.2
    with GB.guarded_engine():
        tr = Trainer(arch, n, h, w, dtype=dtype, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, use_graph=True, **kw)
        img = Engine(arch, 1, h, w, dtype="fp16", in_chans=cin, global_pool="avg")       # test_img: batch 1, fp16, eval
    tr.load_state_dict(sd)
    img.load_state_dict(sd)
    x, y = synth_batch(n, cin, h, w, seed=1234)
    for _ in range(2):                      # the capture's warm-up launch, then a replay
        tr.train_step(x, y)
    tr.validate_step(x, y)
    img.set_input(x[:1])
    img.forward(training=False)
    img.head(False)
    torch.cuda.synchronize()
    vs = GB.verify()
    loss = float(tr.engine.loss)
    if vs:
        _locate(tr, x, y)
    assert not vs, GB.format_violations(vs)
    assert math.isfinite(loss) and bool(torch.isfinite(img.logits).all()), (loss, img.logits)
    print("%s: %d guarded tensors" % (cfg[0], len(GB.registered())))


# ---------------------------------------------------------------------------------------------------------------------------
# sensitivity: one operand deliberately short of what the launch writes
# ---------------------------------------------------------------------------------------------------------------------------
def _one_violation(short):
    torch.cuda.synchronize()
    vs = GB.verify()
    rec = next(r for r in GB.registered() if r.start == short.data_ptr())
    assert len(vs) == 1 and vs[0].operand == rec.describe() and vs[0].side == "after", vs
    assert vs[0].first >= rec.nbytes, vs
    return vs[0], rec


def test_sensitivity_tma_gemm_epilogue():
    """dfd_gemm_tn at M + 1 rows into a C of M rows: the TMA store of the tail tile writes exactly the missing row"""
    from deepfake_detection_b200 import _lib
    M, K, N = 1000, 64, 128
    g = torch.Generator(device="cuda").manual_seed(0)
    A = GB.guard((torch.randn(M + 1, K, device="cuda", generator=g)).to(torch.bfloat16))
    B = GB.guard((torch.randn(N, K, device="cuda", generator=g) / 8).to(torch.bfloat16))
    C = GB.alloc((M, N), torch.bfloat16, "cuda", 0)
    _lib.call("dfd_gemm_tn", A.data_ptr(), B.data_ptr(), C.data_ptr(), M + 1, N, K, 0, None, None, None,
              torch.cuda.current_stream().cuda_stream)
    v, rec = _one_violation(C)
    assert v.first == rec.nbytes and v.last < rec.nbytes + N * 2, v


def test_sensitivity_row_kernel_store():
    """dfd_bn_act over n * hw rows into an output one row short: the manual 16-byte stores of the last row are reported"""
    from deepfake_detection_b200 import _lib
    n, hw, C = 3, 77, 64
    g = torch.Generator(device="cuda").manual_seed(0)
    y = GB.guard(torch.randn(n * hw, C, device="cuda", generator=g).to(torch.bfloat16))
    scale = GB.guard(torch.ones(C, device="cuda"))
    shift = GB.guard(torch.zeros(C, device="cuda"))
    out = GB.alloc((n * hw - 1, C), torch.bfloat16, "cuda", 0)
    _lib.call("dfd_bn_act", y.data_ptr(), scale.data_ptr(), shift.data_ptr(), None, None, out.data_ptr(), n, hw, C, 1, 0, 0,
              torch.cuda.current_stream().cuda_stream)
    v, rec = _one_violation(out)
    assert v.first == rec.nbytes and v.last < rec.nbytes + C * 2, v


def test_sensitivity_fp64_statistics_atomics():
    """the GEMM's per-channel fp64 sums into a [slots, N] buffer one channel short: the atomics of the last slot's last
    channel (M = 4096 is 32 M tiles, so every slot bx % 8 is written, gemm_tc.cu:429 / common.cuh:128)"""
    from deepfake_detection_b200 import _lib
    M, K, N = 4096, 64, 64
    S = _lib.lib().stat_slots
    g = torch.Generator(device="cuda").manual_seed(0)
    A = GB.guard(torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16))
    B = GB.guard((torch.randn(N, K, device="cuda", generator=g) / 8).to(torch.bfloat16))
    C = GB.alloc((M, N), torch.bfloat16, "cuda", 0)
    s1 = GB.alloc((S * N - 1,), torch.float64, "cuda", 0)
    s2 = GB.alloc((S * N,), torch.float64, "cuda", 0)
    _lib.call("dfd_gemm_tn", A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, 0, s1.data_ptr(), s2.data_ptr(), None,
              torch.cuda.current_stream().cuda_stream)
    v, rec = _one_violation(s1)
    assert v.last == rec.nbytes + 7, v               # the one double past the end (its sign / exponent byte changed)


def test_fp64_atomic_add_changes_the_guard():
    """why the fp64 guard is a tiny normal number: an fp64 atomic add (index_add_ is atomicAdd(double)) returns a NaN operand
    bit for bit, so a NaN guard would hide the statistics atomics; the guard's own pattern is replaced by any such add"""
    idt, bits = GB.pattern(torch.float64)
    idx = torch.zeros(3, dtype=torch.long, device="cuda")
    vals = torch.tensor([1e-3, -2.5, 7.0], dtype=torch.float64, device="cuda")
    nan = torch.full((4,), 0x7FF4A5A5A5A5A5A5, dtype=torch.int64, device="cuda").view(torch.float64)
    nan.index_add_(0, idx, vals)
    assert int(nan.view(torch.int64)[0]) == 0x7FF4A5A5A5A5A5A5      # unchanged: the reason
    t = GB.alloc((5,), torch.float64, "cuda", 0)
    rec = GB.registered()[-1]
    tail = rec.big[GB.G + rec.nbytes:GB.G + rec.nbytes + 8].view(torch.float64)
    tail.index_add_(0, torch.zeros(1, dtype=torch.long, device="cuda"), vals[:1])
    v, _ = _one_violation(t)
    assert v.last == rec.nbytes + 7, v


def test_sensitivity_split_k_workspace():
    """dfd_gemm_wgrad in workspace mode with the workspace one split partial short of splits x Nw x Kw floats"""
    from deepfake_detection_b200 import _lib
    M, Nw, Kw = 50176, 64, 64
    splits = _lib.lib().cdll.dfd_gemm_wgrad_splits(M, Nw, Kw)
    assert splits >= 2 and Nw * Kw * 4 <= GB.G, splits
    g = torch.Generator(device="cuda").manual_seed(0)
    Gr = GB.guard((torch.randn(M, Nw, device="cuda", generator=g) * 0.3).to(torch.bfloat16))
    X = GB.guard(torch.randn(M, Kw, device="cuda", generator=g).to(torch.bfloat16))
    dW = GB.alloc((Nw, Kw), torch.float32, "cuda", 0)
    ws = GB.alloc(((splits - 1) * Nw * Kw,), torch.float32, "cuda", 0)
    _lib.call("dfd_gemm_wgrad", Gr.data_ptr(), X.data_ptr(), dW.data_ptr(), M, Nw, Kw, 0, ws.data_ptr(), splits * Nw * Kw * 4,
              torch.cuda.current_stream().cuda_stream)
    v, rec = _one_violation(ws)
    assert v.first >= rec.nbytes and v.last < rec.nbytes + Nw * Kw * 4, v
