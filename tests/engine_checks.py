"""End-to-end parity of the native engine against the CPU oracle (which is pinned to the reference by
tests/test_oracle_vs_reference_goldens.py) on identical seeded weights and batches.

Two oracles are run beside the CUDA path:
  * `emul`: fp32 arithmetic with the activations rounded to the 16-bit type at the points where the native path
    stores them (tight: differences are accumulation order + the tanh-based sigmoid),
  * `fp32`: the plain reference arithmetic (the north_star tolerance: 1e-2 relative for bf16).
Per-layer taps localise the first diverging layer; per-parameter gradient errors localise a wrong backward kernel.
"""
import torch

from deepfake_detection_b200.arch import get_spec, param_entries
from deepfake_detection_b200.engine import Engine
from deepfake_detection_b200.optim import ArenaOptimizer
from deepfake_detection_b200.trainer import Trainer
from oracle import train as OT
from oracle.weights import synth_batch, synth_state, tame_state


def relerr(a, b, floor=0.0):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + floor + 1e-30))


def engine_step(eng, opt, x, y, smoothing=0.0):
    st = torch.cuda.current_stream().cuda_stream
    eng.set_input(x)
    eng.set_target(y)
    eng.zero_step_scratch(st, grads=True)
    eng.forward(training=True)
    eng.head(True, smoothing=smoothing, soft=y.dtype.is_floating_point)
    eng.backward()
    if opt is not None:
        opt.step()
    torch.cuda.synchronize()


def tap_to_nchw(t):
    return t.float().permute(0, 3, 1, 2).cpu()


def run_parity(arch, batch, H, W, dtype="bf16", steps=2, gemm_impl="tc", opt_kind="sgd", lr=0.01, smoothing=0.0,
               soft=False, verbose=False, tame=False):
    tdt = torch.bfloat16 if dtype == "bf16" else torch.float16
    spec = get_spec(arch)
    sd0 = synth_state(spec, seed=7)
    if tame and spec.family == "resnet":
        # damping the residual branches (both implementations see the same weights) keeps the comparison informative
        tame_state(spec, sd0)
    eng = Engine(arch, batch, H, W, dtype=dtype, gemm_impl=gemm_impl)
    eng.load_state_dict(sd0)
    wd = 1e-4
    opt = ArenaOptimizer(eng, opt=opt_kind, lr=lr, momentum=0.9, weight_decay=wd)
    oracles = {}
    for key, adt in (("emul", tdt), ("fp32", None)):
        sd = {k: v.clone() for k, v in sd0.items()}
        owd = wd / lr if opt_kind == "adamw" else wd
        oracles[key] = (sd, OT.OptState(kind=opt_kind, lr=lr, momentum=0.9, weight_decay=owd, eps=1e-8), adt)
    report = dict(arch=arch, batch=batch, H=H, W=W, dtype=dtype, gemm_impl=gemm_impl, steps=[])
    pnames = [n for n, _, _ in param_entries(spec)]
    for step in range(steps):
        x, y = synth_batch(batch, spec.in_chans, H, W, seed=1234 + step, soft=soft)
        engine_step(eng, opt, x.cuda(), y.cuda(), smoothing)
        rec = {}
        keep = {}
        for key, (sd, ost, adt) in oracles.items():
            taps = {} if (key == "emul" and step == 0) else None
            # capture the oracle gradients before the update changes the weights
            out = OT.train_step(spec, sd, x, y, ost, smoothing=smoothing, act_dtype=adt, taps=taps)
            r = dict(loss_native=float(eng.loss), loss_oracle=float(out["loss"]),
                     logits_rel=relerr(eng.logits, out["logits"]),
                     prec1_native=float(eng.correct) * 100.0 / batch, prec1_oracle=float(out["prec1"]))
            gmax = max(float(g.double().norm()) / max(g.numel(), 1) ** 0.5 for g in out["grads"].values())
            gerr = {n: relerr(eng.grad_view(n), out["grads"][n], floor=1e-3 * gmax * out["grads"][n].numel() ** 0.5) for n in pnames}
            worst = sorted(gerr.items(), key=lambda kv: -kv[1])[:6]
            r["grad_rel_worst"] = worst
            r["grad_rel_median"] = sorted(gerr.values())[len(gerr) // 2]
            tot_n = torch.cat([eng.grad_view(n).flatten().cpu() for n in pnames])
            tot_o = torch.cat([out["grads"][n].flatten() for n in pnames])
            r["grad_rel_total"] = relerr(tot_n, tot_o)
            keep[key] = (out["logits"].clone(), tot_o, float(out["loss"]))
            perr = {n: relerr(eng.param_view(n), sd[n]) for n in pnames}
            r["param_rel_worst"] = sorted(perr.items(), key=lambda kv: -kv[1])[:3]
            berr = {n: relerr(eng.buffer_view(n).float(), sd[n].float()) for n in sd if n not in pnames}
            r["buffer_rel_worst"] = sorted(berr.items(), key=lambda kv: -kv[1])[:3]
            if taps is not None:
                tl = []
                for name, t in taps.items():
                    if name in eng.acts:
                        tl.append((name, relerr(tap_to_nchw(eng.acts[name]), t.detach())))
                r["taps_first_bad"] = next(((n, e) for n, e in tl if e > 2e-2), None)
                r["taps_max"] = max(tl, key=lambda kv: kv[1]) if tl else None
                if verbose:
                    r["taps"] = tl
            rec[key] = r
        # the yardstick: how far the oracle's own 16-bit emulation is from the fp32 reference arithmetic. A perfect
        # 16-bit implementation cannot be closer to fp32 than this, so the bf16 tolerance is stated relative to it.
        rec["yard"] = dict(logits_rel=relerr(keep["emul"][0], keep["fp32"][0]), grad_rel_total=relerr(keep["emul"][1], keep["fp32"][1]),
                           loss_abs=abs(keep["emul"][2] - keep["fp32"][2]))
        report["steps"].append(rec)
    # eval-mode forward with the trained running statistics (validate path)
    x, y = synth_batch(batch, spec.in_chans, H, W, seed=999)
    eng.set_input(x.cuda())
    eng.forward(training=False)
    eng.head(False)
    torch.cuda.synchronize()
    sd = oracles["emul"][0]
    ev = OT.validate_step(spec, sd, x, y, act_dtype=tdt)
    report["eval_logits_rel"] = relerr(eng.logits, ev["logits"])
    return report


def trainer_steps(arch, batch, H, W, dtype, steps, sd0, loss_scale=1.0, **trainer_kw):
    """`steps` Trainer steps (graph-captured; SGD at lr 0.01, momentum 0.9, weight decay 1e-4 unless `trainer_kw` says
    otherwise) from the weights `sd0` on synth_batch(seed=1234 + i): per step the loss, the logits, the gradient arena with
    the loss scale it carries, and the updated parameters. The default static loss scale 1 leaves the fp16 gradients
    unscaled, as the oracle's fp16 emulation rounds them; a dynamically scaled first step can overflow and be skipped."""
    tr = Trainer(arch, batch, H, W, dtype=dtype, loss_scale=loss_scale, **trainer_kw)
    tr.engine.load_state_dict(sd0)
    out = []
    for i in range(steps):
        x, y = synth_batch(batch, 3, H, W, seed=1234 + i)
        e = tr.engine
        scale = float(e.loss_scale_state[0])
        loss, _ = tr.train_step(x.cuda(), y.cuda())
        torch.cuda.synchronize()
        out.append(dict(loss=float(loss), logits=e.logits.detach().cpu().clone(), scale=scale,
                        grads=e.grads32.detach().cpu().clone(), params=e.params32.detach().cpu().clone()))
    return tr, out


def engine_masks(eng):
    """the DropBlock, drop-path and dropout masks a native ResNet engine drew for its last training step, in the layout of
    oracle.train.train_step's `drop_block`, `drop_masks` and `dropout_mask` (CPU)"""
    db = {k: m.permute(0, 3, 1, 2).float().cpu() for k, (m, _) in eng.drop_block_masks.items()}
    dp = {k: g[:, 0].cpu().clone() for k, g in eng.drop_masks.items()}
    dm = eng.dropout_mask.cpu().clone() if eng.drop_rate > 0 else None
    return db, dp, dm
