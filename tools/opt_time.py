"""Cost of the optimizers: the update phase of every kind at the B0, B4 and R50 arenas, and the graph-replayed train step of
B0 and R50 with each new kind against sgd.

    python tools/opt_time.py [--iters 200] [--steps 20] [--rounds 3] [--kinds radam,...] [--out FILE]

1. Update phase: ArenaOptimizer.step() over the whole arena (lr push, tick, the layer-wise norms where the kind has them, one
   update launch per range, the derived-layout refresh), CUDA events around `--iters` phases after a warm-up; ms per phase.
   Every kind, sgd / adam / adamw / rmsproptf included, so the new ones read against the old.
2. Step: Trainer.step_resident (graph-replayed) of EfficientNet-B0 b256 and ResNet-50 b256, bf16, 224x224, each new kind
   alternated with sgd in one process (`--rounds` windows of `--steps` steps each); medians and the difference.
The GPU name, power limit and max SM clock are read in the same run. Needs a GPU; there is no fallback.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from head_time import gpu_info  # noqa: E402

ALL = ("sgd", "adam", "adamw", "rmsproptf", "radam", "adadelta", "rmsprop", "novograd", "nvnovograd")
NEW = ALL[4:]
ARENAS = {"b0": "efficientnet_b0", "b4": "efficientnet_b4", "r50": "resnet50"}


def time_update(arch, kinds, iters):
    from deepfake_detection_b200.engine import Engine
    from deepfake_detection_b200.optim import ArenaOptimizer
    a = Engine(arch, 1, dtype="bf16", params_only=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    a.params32.copy_(torch.randn(a.n_params, device="cuda", generator=g) * 0.05)
    a.grads32.copy_(torch.randn(a.n_params, device="cuda", generator=g) * 1e-3)
    out = dict(n_params=a.n_params)
    for kind in kinds:
        o = ArenaOptimizer(a, opt=kind, lr=1e-4, weight_decay=1e-5)
        for _ in range(10):
            o.step()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            o.step()
        t1.record()
        torch.cuda.synchronize()
        out[kind] = round(t0.elapsed_time(t1) / iters, 4)
        del o
    return out


def _trainer(arch, kind, batch, res):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    tr = Trainer(arch, batch, res, res, dtype="bf16", opt=kind, lr=1e-4, num_classes=2)
    tr.load_state_dict(init_state_dict(get_spec(arch, num_classes=2), seed=42))
    g = torch.Generator(device="cuda").manual_seed(1234)
    tr.engine.set_input(torch.randn(batch, 3, res, res, device="cuda", generator=g))
    tr.engine.set_target(torch.randint(0, 2, (batch,), device="cuda", generator=g))
    return tr


def time_steps(arch, kind, batch, steps, rounds):
    trs = {"sgd": _trainer(arch, "sgd", batch, 224), kind: _trainer(arch, kind, batch, 224)}
    for tr in trs.values():
        for _ in range(5):
            tr.step_resident()
    torch.cuda.synchronize()
    ms = {k: [] for k in trs}
    for _ in range(rounds):
        for k, tr in trs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                tr.step_resident()
            t1.record()
            torch.cuda.synchronize()
            ms[k].append(t0.elapsed_time(t1) / steps)
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    del trs
    torch.cuda.empty_cache()
    return dict(sgd=round(med["sgd"], 3), new=round(med[kind], 3), added_ms=round(med[kind] - med["sgd"], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--kinds", default=",".join(NEW))
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("opt_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    kinds = a.kinds.split(",")
    out = dict(info=gpu_info(), update_ms={}, step_ms={})
    for tag, arch in ARENAS.items():
        out["update_ms"][tag] = time_update(arch, list(ALL), a.iters)
        print("update phase %s (%d params): %s" % (tag, out["update_ms"][tag]["n_params"],
                                                   {k: v for k, v in out["update_ms"][tag].items() if k != "n_params"}))
    for tag in ("b0", "r50"):
        for kind in kinds:
            r = time_steps(ARENAS[tag], kind, a.batch, a.steps, a.rounds)
            out["step_ms"]["%s_%s" % (tag, kind)] = r
            print("%s b%d bf16 224 step: sgd %.3f ms, %s %.3f ms (%+.3f ms)" % (tag, a.batch, r["sgd"], kind, r["new"], r["added_ms"]))
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
