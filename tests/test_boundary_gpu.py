"""-m gpu: the rows either side of the step and the boundary objects added in round 2 — input normalisation + prefetch
loader (N1), arena ModelEma (N4), device-resident learning rate / Adam step under ONE captured graph, weight_decay = 0,
stochastic depth + dropout against the oracle with the SAME masks (H1f / H1g / N3), the 2-rank NativeDDP paths (H6, 8b).
Every comparison goes through the C-ABI; formulas are the ones pinned to the reference in
tests/test_oracle_vs_reference_goldens.py::test_aux_formulas_match_reference."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# N1: uint8 NCHW -> 16-bit, (x - mean*255) / (std*255)   (dfd/timm/data/loader.py:229-230,250-253)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,img_num,dtype", [((8, 3, 224, 224), 1, torch.bfloat16), ((3, 12, 40, 48), 4, torch.float16),
                                                 ((2, 3, 15, 7), 1, torch.bfloat16), ((2, 12, 5, 7), 4, torch.float16)])
def test_input_normalize_matches_loader_formula(shape, img_num, dtype):
    from deepfake_detection_b200.data import InputNormalizer
    from oracle.formulas import normalize_u8
    g = torch.Generator().manual_seed(3)
    x = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    norm = InputNormalizer(img_num=img_num, dtype=dtype)
    y = norm(x.cuda())
    torch.cuda.synchronize()
    ref = normalize_u8(x, (0.485, 0.456, 0.406), (0.229, 0.224, 0.225), img_num)       # fp32, the reference's expression
    # exact: fp32 subtraction and IEEE division, ONE rounding to the 16-bit type (tolerance stated: 0 ulp)
    assert torch.equal(y.cpu(), ref.to(dtype)), float((y.cpu().float() - ref).abs().max())
    # and within 1 ulp of the reference's fp16 flavour, which rounds mean, std, the difference and the quotient (loader.py:233-235,250)
    if dtype == torch.float16:
        c = shape[1]
        m = torch.tensor([v * 255 for v in (0.485, 0.456, 0.406)] * img_num).view(1, c, 1, 1).half()
        s = torch.tensor([v * 255 for v in (0.229, 0.224, 0.225)] * img_num).view(1, c, 1, 1).half()
        half_ref = x.half().sub_(m).div_(s).float()
        # (x - mean) computed in half carries up to 2^-5 absolute error at |x - mean| ~ 128, i.e. ~6e-4 after the division by
        # std ~ 58: the reference's own half flavour is that far from the exact value, this kernel is not
        assert float((y.cpu().float() - half_ref).abs().max()) <= 1.5e-3 + 2.0 ** -10 * float(half_ref.abs().max())


def test_prefetch_loader_yields_normalised_batches_in_order():
    from deepfake_detection_b200.data import NativePrefetchLoader
    from oracle.formulas import normalize_u8
    g = torch.Generator().manual_seed(5)
    batches = [(torch.randint(0, 256, (4, 12, 32, 32), generator=g, dtype=torch.uint8).pin_memory(),
                torch.randint(0, 2, (4,), generator=g)) for _ in range(5)]

    class L(list):
        sampler = None

    pl = NativePrefetchLoader(L(batches), fp16=True, img_num=4)
    assert len(pl) == 5
    seen = 0
    for (xin, tgt), (xu8, y) in zip(pl, batches):
        # the consumer reads the batch on the current stream, as train_epoch does
        got = xin.float().cpu()
        ref = normalize_u8(xu8, (0.485, 0.456, 0.406), (0.229, 0.224, 0.225), 4).half().float()
        assert torch.equal(got, ref) and torch.equal(tgt.cpu(), y)
        seen += 1
    assert seen == 5
    with pytest.raises(RuntimeError):
        NativePrefetchLoader(L(batches), re_prob=0.5)


def test_train_step_host_u8_equals_resident_step():
    """the end-to-end entry (uint8 pinned host batch -> copy stream -> normalise kernel -> step) trains on exactly the
    tensor the formula gives: same loss as a resident step on the pre-normalised batch"""
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.trainer import Trainer
    from oracle.formulas import normalize_u8
    from oracle.weights import synth_state
    sd = synth_state(get_spec("efficientnet_b0"), seed=7)
    g = torch.Generator().manual_seed(1)
    xu8 = torch.randint(0, 256, (8, 3, 96, 96), generator=g, dtype=torch.uint8).pin_memory()
    y = torch.randint(0, 2, (8,), generator=g).pin_memory()
    losses = []
    for mode in ("host", "resident"):
        tr = Trainer("efficientnet_b0", 8, 96, 96, dtype="bf16", lr=0.01)
        tr.load_state_dict(sd)
        if mode == "host":
            for _ in range(3):              # both staging slots and the captured graph get exercised
                out = tr.train_step_host(xu8, y)
            torch.cuda.synchronize()
            losses.append(float(out[0]))
        else:
            xn = normalize_u8(xu8, (0.485, 0.456, 0.406), (0.229, 0.224, 0.225), 1).to(torch.bfloat16)
            for _ in range(3):
                tr.train_step(xn.cuda(), y.cuda())
            torch.cuda.synchronize()
            losses.append(float(tr.engine.loss))
    assert abs(losses[0] - losses[1]) < 2e-3, losses


# ---------------------------------------------------------------------------------------------------------------------
# optimizer boundary: device-resident lr / step, one graph, weight_decay = 0, rejected names
# ---------------------------------------------------------------------------------------------------------------------
def test_one_graph_survives_lr_schedule_and_covers_adam():
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.trainer import Trainer
    from oracle.weights import synth_batch, synth_state
    sd = synth_state(get_spec("efficientnet_b0"), seed=7)
    x, y = synth_batch(8, 3, 96, 96, seed=1)
    for opt in ("sgd", "adam", "adamw", "rmsproptf"):
        tr = Trainer("efficientnet_b0", 8, 96, 96, dtype="fp16", opt=opt, lr=0.01, loss_scale="none")
        tr.load_state_dict(sd)
        snaps = []
        for lr in (0.01, 0.005, 0.0, 0.0):           # a per-update schedule (scheduler.py:81-85 mutates param_groups)
            for g in tr.optimizer.param_groups:
                g["lr"] = lr
            tr.train_step(x.cuda(), y.cuda())
            torch.cuda.synchronize()
            snaps.append(tr.engine.params32.clone())
        assert tr.n_captures == 1 and tr._graph is not None, (opt, tr.n_captures)     # no re-capture when lr changes
        assert not torch.equal(snaps[0], snaps[1])
        if opt in ("sgd", "adam", "rmsproptf"):
            # lr = 0 read from DEVICE memory by the replayed graph: the weights stop moving (adamw still decays: skip it;
            # rmsproptf keeps coasting on its lr-folded momentum buffer, so only the first two are exact)
            if opt != "rmsproptf":
                assert torch.equal(snaps[2], snaps[3]), opt
        if opt in ("adam", "adamw"):
            assert tr.optimizer.step_count == 4          # device step counter advanced inside the graph


def test_adam_kernel_device_step_matches_torch():
    """dfd_adam_step with the bias correction taken from the device counter == torch.optim.Adam over 3 steps"""
    from deepfake_detection_b200 import _lib
    g = torch.Generator().manual_seed(0)
    n = 4099
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) for _ in range(3)]
    ref = torch.nn.Parameter(p0.clone())
    o = torch.optim.Adam([ref], lr=1e-2, eps=1e-3, weight_decay=1e-2)
    p, m, v = p0.clone().cuda(), torch.zeros(n).cuda(), torch.zeros(n).cuda()
    step_dev = torch.zeros(1, dtype=torch.int32, device="cuda")
    lr_dev = torch.zeros(1, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for i, gr in enumerate(grads):
        lr = 1e-2 * (0.5 ** i)
        o.param_groups[0]["lr"] = lr
        ref.grad = gr.clone()
        o.step()
        _lib.call("dfd_set_floats", lr_dev.data_ptr(), 1, lr, 0, 0, 0, 0, 0, 0, 0, st)
        _lib.call("dfd_opt_tick", step_dev.data_ptr(), None, st)
        _lib.call("dfd_adam_step", p.data_ptr(), gr.cuda().data_ptr(), m.data_ptr(), v.data_ptr(), n, 123.0, 0.9, 0.999, 1e-3,
                  1e-2, 0, 999, 1.0, None, None, None, 0, lr_dev.data_ptr(), step_dev.data_ptr(), st)
    torch.cuda.synchronize()
    assert _rel(p, ref.detach()) < 2e-6 and int(step_dev) == 3


def test_weight_decay_zero_single_group_and_rejected_names():
    from types import SimpleNamespace
    from deepfake_detection_b200.models import create_model
    from deepfake_detection_b200.optim import create_optimizer
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    from deepfake_detection_b200.arch import get_spec
    spec = get_spec("efficientnet_b0")
    sd0 = synth_state(spec, seed=7)
    model = create_model("efficientnet_b0", num_classes=2, dtype="fp16")
    model.load_state_dict(sd0)
    args = SimpleNamespace(opt="sgd", lr=0.01, momentum=0.9, weight_decay=0.0, opt_eps=1e-8)
    opt = create_optimizer(args, model)
    assert len(opt.param_groups) == 1 and opt.param_groups[0]["weight_decay"] == 0.0          # optim_factory.py:34-38
    assert opt.param_groups[0]["params"] == [n for n, _ in model.named_parameters()]
    x, y = synth_batch(16, 3, 96, 96, seed=1234)
    model.train()
    out = model(x.cuda())
    loss = torch.nn.CrossEntropyLoss()(out, y.cuda())
    opt.zero_grad()
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    sd = {k: v.clone() for k, v in sd0.items()}
    OT.train_step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=0.0), act_dtype=torch.float16)
    got = model.state_dict()
    worst = max(_rel(got[k], sd[k]) for k in sd if sd[k].dtype.is_floating_point and sd[k].dim() > 1)
    assert worst < 2e-3, worst
    for bad in ("lookahead_sgd", "lookahead_adam", "nadam", "fusedsgd"):
        with pytest.raises(ValueError):
            create_optimizer(SimpleNamespace(opt=bad, lr=0.01, momentum=0.9, weight_decay=1e-4, opt_eps=1e-8), model)
    with pytest.raises(ValueError):
        create_model("efficientnet_b0", num_classes=2, dtype="float32").engine


# ---------------------------------------------------------------------------------------------------------------------
# N4: ModelEma as arena kernels (dfd/timm/utils.py:276-340)
# ---------------------------------------------------------------------------------------------------------------------
def test_model_ema_matches_reference_formula():
    from deepfake_detection_b200.ema import ModelEma
    from deepfake_detection_b200.models import create_model
    from oracle.formulas import ema_update
    from oracle.weights import synth_batch, synth_state
    from deepfake_detection_b200.arch import get_spec
    spec = get_spec("efficientnet_b0")
    model = create_model("efficientnet_b0", num_classes=2, dtype="fp16")
    model.load_state_dict(synth_state(spec, seed=7))
    ema = ModelEma(model, decay=0.9)
    expect = {k: v.cpu().clone() for k, v in model.state_dict().items()}
    assert all(torch.equal(expect[k], v.cpu()) for k, v in ema.ema.state_dict().items())       # deep copy, own arenas
    assert ema.ema.engine.params32.data_ptr() != model.engine.params32.data_ptr()
    for step in range(2):
        model.load_state_dict(synth_state(spec, seed=20 + step))        # "training" moved the weights
        model.engine.nbt.add_(3 + step)
        ema.update(model)
        torch.cuda.synchronize()
        msd = model.state_dict()
        for k in expect:
            expect[k] = ema_update(expect[k], msd[k].cpu(), 0.9)
    got = ema.ema.state_dict()
    for k in expect:
        if expect[k].dtype.is_floating_point:
            assert torch.allclose(got[k].cpu(), expect[k], rtol=1e-6, atol=1e-7), k
        else:
            assert torch.equal(got[k].cpu(), expect[k]), (k, got[k], expect[k])
    # validating the EMA weights (train.py:561-565) refreshes the 16-bit copies lazily and uses the averaged running stats
    x, y = synth_batch(8, 3, 96, 96, seed=3)
    ema.ema.eval()
    with torch.no_grad():
        lo = ema.ema(x.cuda())
    ref_model = create_model("efficientnet_b0", num_classes=2, dtype="fp16")
    ref_model.load_state_dict(got)
    ref_model.eval()
    with torch.no_grad():
        lr_ = ref_model(x.cuda())
    assert torch.allclose(lo, lr_, rtol=0, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# H1f / H1g / N3: stochastic depth + classifier dropout (layers/drop.py:84-100, efficientnet.py:346-347)
# ---------------------------------------------------------------------------------------------------------------------
def test_drop_path_and_dropout_against_oracle_with_the_same_masks():
    from deepfake_detection_b200.arch import get_spec, param_entries
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.optim import ArenaOptimizer
    from oracle import train as OT
    from oracle.weights import synth_batch, synth_state
    import engine_checks as EC
    torch.manual_seed(123)
    spec = get_spec("efficientnet_b0")
    sd0 = synth_state(spec, seed=7)
    N = 32
    eng = Engine("efficientnet_b0", N, 96, 96, dtype="fp16", drop_rate=0.35, drop_path_rate=0.2)
    eng.load_state_dict(sd0)
    opt = ArenaOptimizer(eng, opt="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4)
    x, y = synth_batch(N, 3, 96, 96, seed=1234)
    EC.engine_step(eng, opt, x.cuda(), y.cuda())
    # the masks the engine drew this step: binary / keep, rate = drop_path_rate * block_idx / n_blocks
    n_blocks = len(spec.blocks)
    masks = {}
    for i, b in enumerate(spec.blocks):
        if b.has_residual and i > 0:
            g = eng.drop_masks[b.name].cpu()
            keep = 1.0 - 0.2 * i / n_blocks
            assert bool((g == g[:, :1]).all()), b.name                         # one draw per sample, replicated over channels
            assert all(v == 0.0 or abs(v * keep - 1.0) < 1e-6 for v in torch.unique(g).tolist()), b.name        # binary / keep
            masks[b.name] = g[:, 0].clone()
    assert set(masks) == set(eng.drop_masks) and len(masks) == 9
    dmask = eng.dropout_mask.cpu().clone()
    assert abs(float((dmask > 0).float().mean()) - 0.65) < 0.02                  # keep rate of F.dropout(p=0.35)
    sd = {k: v.clone() for k, v in sd0.items()}
    out = OT.train_step(spec, sd, x, y, OT.OptState(kind="sgd", lr=0.01, momentum=0.9, weight_decay=1e-4), act_dtype=torch.float16,
                        drop_masks=masks, dropout_mask=dmask)
    assert abs(float(eng.loss) - float(out["loss"])) < 3e-3
    assert _rel(eng.logits, out["logits"]) < 2e-2
    pn = [n for n, _, _ in param_entries(spec)]
    gn = torch.cat([eng.grad_view(n).flatten().cpu() for n in pn])
    go = torch.cat([out["grads"][n].flatten() for n in pn])
    assert _rel(gn, go) < 5e-2
    assert max(_rel(eng.param_view(n), sd[n]) for n in pn if sd[n].dim() > 1) < 2e-3
    # a second step draws DIFFERENT masks (the generator's step counter advances on the device) ...
    first = torch.cat([m for m in masks.values()] + [dmask.flatten()])
    EC.engine_step(eng, opt, x.cuda(), y.cuda())
    second = torch.cat([eng.drop_masks[k][:, 0].cpu() for k in masks] + [eng.dropout_mask.cpu().flatten()])
    assert not torch.equal(first, second) and int(eng.rng_state[1]) == 2
    # ... eval mode applies none of them (drop.py:93, F.dropout(training=False)): same logits as an undropped engine
    ref = Engine("efficientnet_b0", N, 96, 96, dtype="fp16", share_from=eng)
    for e in (eng, ref):
        e.set_input(x.cuda())
        e.forward(training=False)
        e.head(False)
    torch.cuda.synchronize()
    assert torch.equal(eng.logits, ref.logits)


def test_drop_masks_keep_rate_statistics():
    """rate test of the counter-based generator: 200 draws of a [64]-sample drop-path mask at keep = 0.8"""
    import struct
    from deepfake_detection_b200 import _lib
    out = torch.zeros(64, 8, device="cuda")
    state = torch.tensor([12345, 0], dtype=torch.int64, device="cuda")
    table = torch.frombuffer(bytearray(struct.pack("<Qqifii", out.data_ptr(), 64, 8, 0.8, 0, 0)), dtype=torch.uint8).cuda()
    st = torch.cuda.current_stream().cuda_stream
    kept, cols = 0, []
    for _ in range(200):
        _lib.call("dfd_rng_masks", table.data_ptr(), 1, state.data_ptr(), st)
        _lib.call("dfd_rng_tick", state.data_ptr(), st)
        kept += int((out[:, 0] > 0).sum())
        cols.append((out[:, 0] > 0).float().cpu())
    rate = kept / (200 * 64)
    assert abs(rate - 0.8) < 0.015, rate                     # 3.5 sigma of Binomial(12800, 0.8)
    c = torch.stack(cols)
    # no sample is stuck: every one of the 64 positions is both kept and dropped over 200 steps, neighbours uncorrelated
    assert bool(((c.mean(0) > 0.6) & (c.mean(0) < 0.95)).all())
    assert abs(float(torch.corrcoef(torch.stack([c[:, 0], c[:, 1]]))[0, 1])) < 0.25


# ---------------------------------------------------------------------------------------------------------------------
# H6 / 8(b): NativeDDP over 2 ranks, protocol AND fused runner paths against the oracle with a gradient-mean hook
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_native_ddp_two_ranks_match_oracle(tmp_path):
    out = str(tmp_path / "ddp.json")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", DFD_DDP_OUT=out)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", str(29600 + os.getpid() % 300), os.path.join(ROOT, "tests", "ddp_worker.py")],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    rep = json.load(open(out))
    for flavour in ("protocol", "fused", "syncbn"):
        f = rep[flavour]
        assert f["weights_rel_worst"] < 2e-3, (flavour, f)          # post-step weights vs oracle with grad_hook mean
        assert f["ranks_identical"], flavour                        # replicas hold bit-identical weights after the epoch
        assert abs(f["loss"] - f["loss_oracle"]) < 5e-3, (flavour, f)
    assert rep["fused"]["plans"] >= 2                               # the smaller last batch ran on its own plan
    assert rep["raises_without_wrapper"]
