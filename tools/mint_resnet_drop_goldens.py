"""Mint the ResNet DropBlock / drop-path / dropout fixtures under tests/golden/ FROM THE UNMODIFIED REFERENCE (CPU only).

    python tools/mint_resnet_drop_goldens.py

drop_block_formulas.json: the reference's own drop_block_2d (layers/drop.py:24-63) on small tensors, with the uniform noise
it drew and its output: square 10x10 and 5x5 (positive gamma), 7x7, non-square 10x14 and 5x7 (negative gamma: nothing is
dropped), at gamma_scale 0.25 and 1.

Train steps of the reference's own `create_model(arch, drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.2)` with the
synthetic weights of oracle/weights.py, SGD (nesterov) and nn.CrossEntropyLoss, two steps each:

    step_resnet18_drop_160.json        ResNet-18, batch 4, 160 x 160
    step_resnet18_drop_160x224.json    ResNet-18, batch 4, 160 x 224
    step_resnet50_drop_160.json        ResNet-50, batch 2, 160 x 160

torch.rand, torch.rand_like, F.dropout and F.max_pool2d are wrapped only to RECORD what the reference drew (its code runs
unmodified): the drop-path draws, the dropout masks, and per DropBlock call the seed mask that enters the min-pool, stored
as the sparse indices of its zeros. Logits, loss, gradients and updated values use the compact summaries of
tools/mint_multiclass_goldens.py.
"""
import base64
import json
import os
import sys
import zlib

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))

from mint_multiclass_goldens import _pick, _summ  # noqa: E402
from deepfake_detection_b200.arch import get_spec  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle.mint_goldens import GOLDEN, _args  # noqa: E402
from oracle.weights import synth_batch, synth_state  # noqa: E402

RATES = dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.2)


def pack_f32(t):
    """exact float32 values, base64 of the little-endian bytes"""
    return base64.b64encode(t.detach().to(torch.float32).contiguous().numpy().astype("<f4").tobytes()).decode()


def pack_idx(idx):
    """ascending flat indices: base64 of the zlib-compressed int32 deltas"""
    t = torch.as_tensor(idx, dtype=torch.int64)
    d = torch.diff(t, prepend=torch.zeros(1, dtype=torch.int64)).to(torch.int32)
    return base64.b64encode(zlib.compress(d.numpy().astype("<i4").tobytes(), 9)).decode()


def mint_formulas():
    from dfd.timm.models.layers.drop import drop_block_2d
    cases = []
    real_rand_like = torch.rand_like
    for H, W in ((10, 10), (5, 5), (7, 7), (10, 14), (5, 7)):
        for gs in (0.25, 1.0):
            g = torch.Generator().manual_seed(H * 100 + W + int(gs * 4))
            x = torch.randn(1, 2, H, W, generator=g)
            drawn = []

            def rec_rand_like(t, *a, **k):
                u = real_rand_like(t, *a, **k)
                drawn.append(u.clone())
                return u

            torch.rand_like = rec_rand_like
            try:
                torch.manual_seed(H * W)
                out = drop_block_2d(x, 0.3, True, 7, gs)
            finally:
                torch.rand_like = real_rand_like
            cases.append(dict(H=H, W=W, drop_prob=0.3, block_size=7, gamma_scale=gs, x=pack_f32(x), noise=pack_f32(drawn[0]),
                              out=pack_f32(out)))
            print("drop_block_2d %dx%d gamma_scale %g: %d of %d zeroed" % (H, W, gs, int((out == 0).sum()), out.numel()))
    with open(os.path.join(GOLDEN, "drop_block_formulas.json"), "w") as f:
        json.dump(dict(shape=[1, 2], torch=torch.__version__, cases=cases), f)


def mint_drop_step(arch, batch, H, W, tag, n_steps=2):
    from dfd.timm.models import create_model
    from dfd.timm.optim import create_optimizer
    torch.manual_seed(0)
    spec = get_spec(arch)
    model = create_model(arch, num_classes=2, **RATES)
    model.load_state_dict(synth_state(spec, seed=7), strict=True)
    model.train()
    lr, wd = 0.01, 1e-4
    optimizer = create_optimizer(_args(opt="sgd", lr=lr, weight_decay=wd), model)
    params = dict(model.named_parameters())
    buffers = {k: b for k, b in model.named_buffers() if not k.endswith("num_batches_tracked")}
    pk, bk = _pick(list(params), 6), _pick([k for k in buffers if k.endswith("running_var")], 2)
    # DropBlock sites in call order: every main-branch BN of layer3 / layer4 (resnet.py:153-162,218-233)
    sites = []
    for b in spec.blocks:
        if b.name.split(".")[0] in ("layer3", "layer4"):
            sites += [b.name + "." + n for n in (("bn1", "bn2") if b.kind == "basic" else ("bn1", "bn2", "bn3"))]
    rec = dict(arch=arch, batch=batch, H=H, W=W, num_classes=2, weight_seed=7, opt="sgd", lr=lr, momentum=0.9,
               weight_decay=wd, smoothing=0.0, soft=False, torch=torch.__version__, sites=sites, steps=[], **RATES)
    real = (torch.rand, torch.rand_like, F.dropout, F.max_pool2d)
    for step in range(n_steps):
        x, y = synth_batch(batch, 3, H, W, seed=1234 + step)
        rands, seeds, drops = [], [], []

        def rec_rand(*a, **k):
            t = real[0](*a, **k)
            rands.append(t.clone())
            return t

        def rec_max_pool2d(inp, kernel_size, stride=None, padding=0, *a, **k):
            if stride == 1:             # DropBlock's min-pool of the seeds (the stem's max-pool has stride 2)
                seeds.append((-inp).clone())
            return real[3](inp, kernel_size, stride, padding, *a, **k)

        def rec_dropout(inp, p=0.5, training=True, inplace=False):
            out = real[2](inp, p, training, False)
            drops.append(((out != 0) | (inp == 0)).float() / (1.0 - p))
            return out

        torch.rand, torch.rand_like, F.dropout, F.max_pool2d = rec_rand, real[1], rec_dropout, rec_max_pool2d
        try:
            torch.manual_seed(5 + step)
            out = model(x)
        finally:
            torch.rand, torch.rand_like, F.dropout, F.max_pool2d = real
        loss = torch.nn.CrossEntropyLoss()(out, y)
        optimizer.zero_grad()
        loss.backward()
        grads = {k: _summ(params[k].grad) for k in pk}
        optimizer.step()
        # one torch.rand((N, 1, 1, 1)) per block (the shared DropPath), one seed mask per DropBlock call, in forward order
        assert len(rands) == len(spec.blocks) and len(seeds) == len(sites) and len(drops) == 1, (len(rands), len(seeds))
        keep = 1.0 - RATES["drop_path_rate"]
        drop_masks = {b.name: (torch.floor(keep + u) / keep).reshape(-1).tolist() for b, u in zip(spec.blocks, rands)}
        drop_block = {s: dict(shape=list(t.shape), zeros=pack_idx(torch.nonzero((t == 0).flatten()).flatten()))
                      for s, t in zip(sites, seeds)}
        dropout_zeros = pack_idx(torch.nonzero((drops[0] == 0).flatten()).flatten())
        rec["steps"].append(dict(logits=_summ(out, 32), loss=float(loss.detach()), grads=grads,
                                 params={k: _summ(params[k]) for k in pk},
                                 buffers={k: _summ(buffers[k].float()) for k in bk},
                                 drop_masks=drop_masks, dropout_shape=list(drops[0].shape),
                                 dropout_zeros=dropout_zeros, drop_block=drop_block))
    name = "step_%s_drop_%s.json" % (arch, tag)
    with open(os.path.join(GOLDEN, name), "w") as f:
        json.dump(rec, f)
    print(name, "loss", [s["loss"] for s in rec["steps"]])


def main():
    ref_shims.install()
    torch.set_num_threads(8)
    mint_formulas()
    mint_drop_step("resnet18", 4, 160, 160, "160")
    mint_drop_step("resnet18", 4, 160, 224, "160x224")
    mint_drop_step("resnet50", 2, 160, 160, "160")


if __name__ == "__main__":
    main()
