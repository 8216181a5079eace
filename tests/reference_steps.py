"""The reference-minted step fixtures (tests/golden/step_*.json) and what checks each one: the summary comparison every
fixture test uses, and the tables the CPU test (test_oracle_vs_reference_goldens.py::test_oracle_matches_reference_steps) and
the GPU test (test_reference_steps_gpu.py) parametrise over. A new model family adds rows here, not another loop.

Everything a step runs (arch, num_classes, global_pool, tame, opt, lr, weight_decay, soft, smoothing, batch, H, W) is
read from the fixture itself. Every CPU row is held to the same statements, so that table is a list of names; a GPU row is
(fixture name, overrides), the overrides holding the kind of run and where fixtures are held to different statements."""
import hashlib
import json
import os

import pytest
import torch

RTOL = 2e-4
# the optimizers whose factory hands the reference weight_decay / lr (optim_factory.py:29-33). The step fixtures cannot
# resolve this (their decay moves the weights by ~1e-4 relative); the optimizer fixtures (optimizers*.json) can
DECAY_PER_LR = ("adamw", "radam")


def check_summ(t, s, what, rtol=RTOL, floor=1e-7):
    """`t` against its recorded summary `s`: the norm within `rtol`, the sampled elements within 5 * rtol of the tensor's RMS
    plus rtol of their largest magnitude. `floor`: absolute slack for quantities that are mathematically zero (e.g. the
    gradient of a BN bias that feeds conv+BN), which are pure fp32 round-off in both implementations."""
    f = t.detach().reshape(-1).to(torch.float64)
    norm = float(f.norm())
    assert norm == pytest.approx(s["norm"], rel=rtol, abs=floor * max(f.numel(), 1) ** 0.5), what + " norm"
    got = f[torch.tensor(s["idx"])]
    ref = torch.tensor(s["samples"], dtype=torch.float64)
    scale = max(s["norm"] / max(f.numel(), 1) ** 0.5, 1e-8)
    assert float((got - ref).abs().max()) <= 5 * rtol * scale + rtol * float(ref.abs().max()) + floor, what + " samples"


def digest(entries):
    """sha256 of a state / parameter entry list, as the fixture scripts record it"""
    return hashlib.sha256(json.dumps(entries, separators=(",", ":")).encode()).hexdigest()


def load(golden_dir, name):
    with open(os.path.join(golden_dir, name + ".json")) as f:
        return json.load(f)


# every step fixture the CPU oracle (oracle.train) is held to, each once
CPU_STEPS = [
    # the BASELINE architectures: two-class head, average pool; label smoothing, soft targets, RMSpropTF and AdamW
    # (oracle/mint_goldens.py)
    "step_efficientnet_b0",
    "step_efficientnet_b4",
    "step_resnet18",
    "step_resnet50",
    "step_efficientnet_b0_ls",
    "step_efficientnet_b0_soft_rmsprop",
    "step_efficientnet_b0_adamw",
    # K-class heads (tools/mint_multiclass_goldens.py)
    "step_efficientnet_b0_k5_ls",
    "step_efficientnet_b0_k5_soft_rmsprop",
    "step_resnet18_k1000",
    # selectable global pool (tools/mint_gpool_goldens.py)
    "step_efficientnet_b0_gp_max",
    "step_efficientnet_b0_k5_gp_catavgmax_ls",
    "step_resnet18_gp_avgmax",
    # RAdam and NvNovoGrad (tools/mint_optimizer_goldens.py)
    "step_efficientnet_b0_radam",
    "step_resnet18_nvnovograd",
    # TF "SAME" padding, BatchNorm eps 1e-3 (tools/mint_tf_goldens.py)
    "step_tf_efficientnet_b0_64x96",
    "step_tf_efficientnet_b0_66x96",
    # dense ResNets, ResNet-D, Wide ResNet (tools/mint_resnet_family_goldens.py)
    "step_resnet26d_72x88",
    "step_resnet50d",
    "step_resnet34",
    "step_wide_resnet50_2",
    "step_resnet101",
    "step_resnet26d_tame_104x88",
    "step_resnet34_tame_96",
    "step_wide_resnet50_2_tame_96",
    "step_resnet101_tame_96",
    # SE-ResNets (tools/mint_senet_goldens.py)
    "step_seresnet18_70x72",
    "step_seresnet50_64x64",
    "step_seresnet101",
    "step_seresnet18_tame_70x72",
    "step_seresnet50_tame_64x64",
    "step_seresnet101_tame_64x64",
    # Xception (tools/mint_xception_goldens.py)
    "step_xception_64x80",
    "step_xception_299",
    "step_xception_tame_64x80",
]

# every step fixture the native path is held to. kind "engine": Engine + ArenaOptimizer steps from the untamed fixture in
# `dtypes`, the loss within 1e-2 at step 0 and `loss_after` later, the step-0 logits within 7e-2 (the whole tensor where the
# fixture stores it, else its samples), with `norm` also the logits' norm, with `step_count` the optimizer's step counter.
# kind "tamed": Trainer steps from a fixture with damped residual branches, held to the oracle's 16-bit emulation and to the
# reference in both 16-bit types.
_FP16 = ("fp16",)
_BOTH = ("bf16", "fp16")
GPU_STEPS = [
    ("step_efficientnet_b0", dict(kind="engine", dtypes=("bf16",))),
    # step 1 follows an update whose gradient depends on argmax choices that fp16 storage and the fp32 reference can resolve
    # differently
    ("step_efficientnet_b0_gp_max", dict(kind="engine", dtypes=_FP16, loss_after=8e-2, norm=True)),
    ("step_efficientnet_b0_k5_gp_catavgmax_ls", dict(kind="engine", dtypes=_FP16, loss_after=8e-2, norm=True)),
    ("step_resnet18_gp_avgmax", dict(kind="engine", dtypes=_FP16, loss_after=8e-2, norm=True)),
    ("step_efficientnet_b0_k5_ls", dict(kind="engine", dtypes=_FP16, norm=True)),
    ("step_efficientnet_b0_k5_soft_rmsprop", dict(kind="engine", dtypes=_FP16, norm=True)),
    ("step_resnet18_k1000", dict(kind="engine", dtypes=_FP16, norm=True)),
    ("step_efficientnet_b0_radam", dict(kind="engine", dtypes=_FP16, step_count=True)),
    ("step_resnet18_nvnovograd", dict(kind="engine", dtypes=_FP16, step_count=True)),
    ("step_resnet26d_tame_104x88", dict(kind="tamed", dtypes=_BOTH)),
    ("step_resnet34_tame_96", dict(kind="tamed", dtypes=_BOTH)),
    ("step_wide_resnet50_2_tame_96", dict(kind="tamed", dtypes=_BOTH)),
    ("step_resnet101_tame_96", dict(kind="tamed", dtypes=_BOTH)),
    ("step_seresnet18_tame_70x72", dict(kind="tamed", dtypes=_BOTH)),
    ("step_seresnet50_tame_64x64", dict(kind="tamed", dtypes=_BOTH)),
    ("step_seresnet101_tame_64x64", dict(kind="tamed", dtypes=_BOTH)),
    ("step_xception_tame_64x80", dict(kind="tamed", dtypes=_BOTH)),
]

# step fixtures held by a test of their own ("<module>::<test>"), with masks or a restatement the tables above do not run
ELSEWHERE = [
    # DenseNet: the torch-op restatement tests/densenet_ref.py, not oracle/
    ("step_densenet121_72x88", "test_densenet_cpu::test_restatement_matches_reference_steps"),
    ("step_densenet161_70x54", "test_densenet_cpu::test_restatement_matches_reference_steps"),
    ("step_densenet121_224", "test_densenet_cpu::test_restatement_matches_reference_steps"),
    ("step_densenet121_drop_48", "test_densenet_cpu::test_restatement_matches_reference_steps"),
    # DropBlock, drop path and dropout: the reference's masks rebuilt, at tolerances of their own
    ("step_resnet18_drop_160", "test_resnet_drop_cpu::test_drop_oracle_matches_reference_steps"),
    ("step_resnet18_drop_160x224", "test_resnet_drop_cpu::test_drop_oracle_matches_reference_steps"),
    ("step_resnet50_drop_160", "test_resnet_drop_cpu::test_drop_oracle_matches_reference_steps"),
    # stochastic depth and classifier dropout with the reference's masks
    ("step_efficientnet_b0_dropped", "test_oracle_vs_reference_goldens::test_dropped_step_matches_reference"),
]
