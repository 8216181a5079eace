"""-m gpu: the dense ResNet family on the native path.

  * dfd_avgpool2_fwd / dfd_avgpool2_bwd_add against fp64 F.avg_pool2d(2, 2, ceil_mode=True, count_include_pad=False) and its
    autograd, and bit for bit against a torch emulation of their one-rounding formulas, at even and odd extents, bf16 / fp16;
  * resnet101 and resnet50d at batch 32, 224x224, from the reference init against the fp32 oracle; the runner's train_epoch
    over create_model("resnet101"); resnet50d with DropBlock, drop path and dropout;
  * checkpoints round-trip bit for bit, and two resnet50d engines agree bit for bit.
No test here reads the reference tree: the fixtures under tests/golden/ came from tools/mint_resnet_family_goldens.py.
Their train steps are held by tests/test_reference_steps_gpu.py.
"""
import io
import os
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
DT_CODE = {"bf16": 0, "fp16": 1}
EXTENTS = [(56, 56), (28, 28), (14, 14), (9, 11), (5, 6), (7, 7)]
CHANNELS = [64, 256, 1024, 2048]
N_POOL = 3          # not a multiple of 8


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _inv_count(H, W, device):
    """[Ho, Wo] 1 / (in-image elements of each 2x2 window)"""
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    ch = torch.tensor([2.0 if 2 * i + 1 < H else 1.0 for i in range(Ho)], device=device)
    cw = torch.tensor([2.0 if 2 * j + 1 < W else 1.0 for j in range(Wo)], device=device)
    return 1.0 / (ch[:, None] * cw[None, :])


def _emul_fwd(x, dt):
    """NHWC x -> round16(((x00 + x01) + x10) + x11) * (1 / count)) in fp32, out-of-image terms left out"""
    N, H, W, C = x.shape
    f = F.pad(x.float(), (0, 0, 0, W % 2, 0, H % 2))         # zeros: adding them is exact
    s = f[:, 0::2, 0::2] + f[:, 0::2, 1::2]
    s = s + f[:, 1::2, 0::2]
    s = s + f[:, 1::2, 1::2]
    return (s * _inv_count(H, W, x.device)[None, :, :, None]).to(dt)


def _emul_bwd(dy, add, H, W, dt):
    g = dy.float() * _inv_count(H, W, dy.device)[None, :, :, None]
    g = g.repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :H, :W]
    return (g if add is None else add.float() + g).to(dt)


def _call(name, *args):
    from deepfake_detection_b200 import _lib
    _lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("C", CHANNELS)
@pytest.mark.parametrize("H,W", EXTENTS)
def test_avgpool2_kernels(H, W, C, dtype):
    dt = TDT[dtype]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    g = torch.Generator(device="cuda").manual_seed(H * 1000 + W * 10 + C)
    x = torch.randn(N_POOL, H, W, C, device="cuda", generator=g).to(dt)
    dy = torch.randn(N_POOL, Ho, Wo, C, device="cuda", generator=g).to(dt)
    add = torch.randn(N_POOL, H, W, C, device="cuda", generator=g).to(dt)
    y = torch.full((N_POOL, Ho, Wo, C), float("nan"), device="cuda", dtype=dt)
    dx0 = torch.full_like(x, float("nan"))
    dx1 = torch.full_like(x, float("nan"))
    _call("dfd_avgpool2_fwd", x.data_ptr(), y.data_ptr(), N_POOL, H, W, C, DT_CODE[dtype])
    _call("dfd_avgpool2_bwd_add", dy.data_ptr(), None, dx0.data_ptr(), N_POOL, H, W, C, DT_CODE[dtype])
    _call("dfd_avgpool2_bwd_add", dy.data_ptr(), add.data_ptr(), dx1.data_ptr(), N_POOL, H, W, C, DT_CODE[dtype])
    torch.cuda.synchronize()
    # the one-rounding formulas, bit for bit
    assert torch.equal(y, _emul_fwd(x, dt))
    assert torch.equal(dx0, _emul_bwd(dy, None, H, W, dt))
    assert torch.equal(dx1, _emul_bwd(dy, add, H, W, dt))
    # fp64 torch: the forward and its autograd, within one 16-bit rounding of the result (the absolute floor covers the fp32
    # sum of a window whose terms cancel, and fp16 subnormals)
    x64 = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    y64 = F.avg_pool2d(x64, 2, 2, ceil_mode=True, count_include_pad=False)
    y64.backward(dy.permute(0, 3, 1, 2).double())
    eps, floor = (2.0 ** -8 if dtype == "bf16" else 2.0 ** -11), 1e-5
    ref = y64.detach().permute(0, 2, 3, 1)
    assert float(((y.double() - ref).abs() - eps * ref.abs()).max()) <= floor
    gref = x64.grad.permute(0, 2, 3, 1)
    assert float(((dx0.double() - gref).abs() - eps * gref.abs()).max()) <= floor
    sref = gref + add.double()
    assert float(((dx1.double() - sref).abs() - eps * sref.abs()).max()) <= floor


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_avgpool2_bwd_add_in_place(dtype):
    """add may be dx itself"""
    dt, H, W, C = TDT[dtype], 9, 11, 256
    g = torch.Generator(device="cuda").manual_seed(5)
    dy = torch.randn(N_POOL, 5, 6, C, device="cuda", generator=g).to(dt)
    acc = torch.randn(N_POOL, H, W, C, device="cuda", generator=g).to(dt)
    ref = _emul_bwd(dy, acc, H, W, dt)
    _call("dfd_avgpool2_bwd_add", dy.data_ptr(), acc.data_ptr(), acc.data_ptr(), N_POOL, H, W, C, DT_CODE[dtype])
    torch.cuda.synchronize()
    assert torch.equal(acc, ref)


# ---- realistic size -------------------------------------------------------------------------------------------------------
_ORACLE = {}


def _oracle_ref_init(arch, batch, res):
    """fp32 oracle step from the reference's own initialisers (cached: one CPU pass serves both dtypes)"""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.models import init_state_dict
    from oracle import train as OT
    from oracle.weights import synth_batch
    key = (arch, batch, res)
    if key not in _ORACLE:
        torch.set_num_threads(int(os.environ.get("DFD_ORACLE_THREADS", "32")))
        spec = get_spec(arch)
        sd = {k: v.clone() for k, v in init_state_dict(spec, seed=11).items()}
        x, y = synth_batch(batch, 3, res, res, seed=1234)
        out = OT.train_step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4))
        _ORACLE[key] = dict(spec=spec, sd=sd, x=x, y=y, logits=out["logits"], loss=float(out["loss"]),
                            pnames=[n for n, _, _ in param_entries(spec)])
    return _ORACLE[key]


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("arch", ["resnet101", "resnet50d"])
def test_batch32_224_reference_init(arch, dtype):
    """tests/test_parity_baseline_sizes.py::test_resnet50_config4_224_reference_init's statements: loss and updated weights
    within 1e-2 of the fp32 oracle, logits within 1e-2 (fp16) / 3e-2 (bf16)"""
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    o = _oracle_ref_init(arch, 32, 224)
    tr = Trainer(arch, 32, 224, 224, dtype=dtype, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, use_graph=False)
    eng = tr.engine
    for _ in range(8):
        # an overflowing fp16 step is skipped and the scale halves: parity is stated on the first applied step
        tr.load_state_dict(init_state_dict(o["spec"], seed=11))
        tr.train_step(o["x"].cuda(), o["y"].cuda())
        torch.cuda.synchronize()
        if not tr.dynamic_scale or int(eng.flags[1]) == 1:
            break
    else:
        raise AssertionError("no fp16 step was applied")
    w0 = init_state_dict(o["spec"], seed=11)
    live = [n for n in o["pnames"] if float(w0[n].abs().max()) > 0]
    worst = max((_rel(eng.param_view(n), o["sd"][n]), n) for n in live)
    glob = _rel(torch.cat([eng.param_view(n).flatten().cpu() for n in o["pnames"]]), torch.cat([o["sd"][n].flatten() for n in o["pnames"]]))
    loss_rel = abs(float(eng.loss) - o["loss"]) / abs(o["loss"])
    logits_rel = _rel(eng.logits, o["logits"])
    assert loss_rel < 1e-2 and worst[0] < 1e-2 and glob < 1e-2, (loss_rel, worst, glob)
    assert logits_rel < (1e-2 if dtype == "fp16" else 3e-2), logits_rel
    del eng, tr
    torch.cuda.empty_cache()


# ---- runner ----------------------------------------------------------------------------------------------------------------
def test_runner_train_epoch_resnet101_matches_oracle():
    """the runner's default model: train_epoch's loop body (train.py:610-649) over create_model("resnet101") and
    create_optimizer for two steps, against the oracle's two steps. Synthetic weights with the residual branches damped
    (engine_checks.run_parity(tame=True)); the weight updates are held to the yardstick of the oracle's own bf16 emulation."""
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from deepfake_detection_b200.runners.train import train_epoch
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state

    class _Loader(list):
        mixup_enabled = False

    args = SimpleNamespace(opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8, prefetcher=True, mixup=0.0,
                           mixup_off_epoch=0, num_classes=2, smoothing=0.0, distributed=False, world_size=1, local_rank=0,
                           log_interval=1, save_images=False, recovery_interval=0, tta=0, model="resnet101")
    spec = get_spec("resnet101")
    sd0 = synth_state(spec, seed=7)
    for b in spec.blocks:
        sd0[b.name + ".bn3.weight"] = sd0[b.name + ".bn3.weight"] * 0.2
    model = create_model("resnet101", num_classes=2)          # bf16, the factory's default: no loss scale, no skipped step
    model.load_state_dict(sd0)
    opt = create_optimizer(args, model)
    data = [synth_batch(16, 3, 96, 96, seed=1234 + i) for i in range(2)]
    m = train_epoch(0, model, _Loader((x.cuda(), y.cuda()) for x, y in data), opt, torch.nn.CrossEntropyLoss(), args)
    pn = [n for n, _, _ in param_entries(spec)]
    res = {}
    for key, adt in (("emul", torch.bfloat16), ("fp32", None)):
        sd = {k: v.clone() for k, v in sd0.items()}
        ost = OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
        losses = [float(OT.train_step(spec, sd, x, y, ost, act_dtype=adt)["loss"]) for x, y in data]
        res[key] = (sum(losses) / 2, torch.cat([(sd[n] - sd0[n]).flatten() for n in pn]))
    got = model.state_dict()
    dn = torch.cat([(got[n].cpu() - sd0[n]).flatten() for n in pn])
    assert abs(m["loss"] - res["fp32"][0]) < 2e-2 * max(1.0, res["fp32"][0]), (m, res["fp32"][0], res["emul"][0])
    yard = _rel(res["emul"][1], res["fp32"][1])
    assert _rel(dn, res["fp32"][1]) < 1.5 * yard + 3e-2, (_rel(dn, res["fp32"][1]), yard)


# ---- DropBlock + drop path + dropout ------------------------------------------------------------------------------------
def test_resnet50d_with_drop_matches_oracle():
    """one Trainer step of resnet50d at 160x160 with all three rates, against the oracle fed the engine's masks (emulation and
    fp32), with tests/test_resnet_drop_gpu.py's statements"""
    from engine_checks import engine_masks
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.trainer import Trainer
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    arch, batch, res, dtype = "resnet50d", 8, 160, "bf16"
    spec = get_spec(arch)
    sd0 = synth_state(spec, seed=7)
    for b in spec.blocks:                       # engine_checks.run_parity(tame=True): damp the residual branches
        sd0[b.name + ".bn3.weight"] = sd0[b.name + ".bn3.weight"] * 0.2
    tr = Trainer(arch, batch, res, res, dtype=dtype, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4, drop_rate=0.2,
                 drop_path_rate=0.1, drop_block_rate=0.2)
    eng = tr.engine
    eng.load_state_dict(sd0)
    x, y = synth_batch(batch, 3, res, res, seed=1234)
    tr.train_step(x.cuda(), y.cuda())
    torch.cuda.synchronize()
    db, dp, dm = engine_masks(eng)
    assert len(db) == 27 and len(dp) == len(spec.blocks) and dm is not None
    assert any(float(m.sum()) < m.numel() for m in db.values())
    pn = [n for n, _, _ in param_entries(spec)]
    rep = {}
    for key, adt in (("emul", TDT[dtype]), ("fp32", None)):
        sd = {k: v.clone() for k, v in sd0.items()}
        out = OT.train_step(spec, sd, x, y, None, act_dtype=adt, drop_block=db, drop_masks=dp, dropout_mask=dm)
        rep[key] = dict(logits=out["logits"], loss=float(out["loss"]), grads=torch.cat([out["grads"][n].flatten() for n in pn]))
    gn = torch.cat([eng.grad_view(n).flatten().cpu() for n in pn])
    em, fp = rep["emul"], rep["fp32"]
    yard_logits, yard_grads = _rel(em["logits"], fp["logits"]), _rel(em["grads"], fp["grads"])
    assert _rel(eng.logits, em["logits"]) < 6e-2
    assert abs(float(eng.loss) - em["loss"]) < 5e-3, (float(eng.loss), em["loss"])
    assert _rel(eng.logits, fp["logits"]) < 1.5 * yard_logits + 1e-2
    assert _rel(gn, fp["grads"]) < 1.5 * yard_grads + 3e-2, (_rel(gn, fp["grads"]), yard_grads)


# ---- checkpoints and determinism -------------------------------------------------------------------------------------------
def test_checkpoint_round_trip_is_bit_exact():
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import create_model
    from oracle.weights import synth_batch, synth_state
    spec = get_spec("resnet50d", num_classes=2)
    sd0 = synth_state(spec, seed=3)
    m1 = create_model("resnet50d", num_classes=2)
    m1.load_state_dict(sd0)
    m1.eval()
    x, _ = synth_batch(4, 3, 96, 112, seed=77)
    with torch.no_grad():
        l1 = m1(x.cuda())
    buf = io.BytesIO()
    torch.save(m1.state_dict(), buf)
    buf.seek(0)
    sd = torch.load(buf)
    assert list(sd) == list(sd0) and all(torch.equal(sd[k].cpu(), sd0[k]) for k in sd0)
    m2 = create_model("resnet50d", num_classes=2)
    m2.load_state_dict(sd)
    m2.eval()
    with torch.no_grad():
        l2 = m2(x.cuda())
    assert torch.equal(l1, l2)
    assert all(torch.equal(a, b) for a, b in zip(m1.state_dict().values(), m2.state_dict().values()))


def test_two_resnet50d_engines_agree_bit_for_bit():
    from deepfake_detection_b200.arch import get_spec
    from engine_checks import trainer_steps
    from oracle.weights import synth_state
    sd0 = synth_state(get_spec("resnet50d"), seed=7)
    runs = [trainer_steps("resnet50d", 8, 96, 96, "bf16", 2, sd0)[1] for _ in range(2)]
    for a, b in zip(*runs):
        assert a["loss"] == b["loss"]
        assert torch.equal(a["logits"], b["logits"]) and torch.equal(a["grads"], b["grads"]) and torch.equal(a["params"], b["params"])
