"""Canonical digest of the engine's call plans, for checking that a host-side change leaves the plans alone (CPU only).

For every configuration below a plan-only engine is built and written out as text: the training forward and backward and
the eval forward, each op as `Engine.launch_args` gives it (a skipped op is listed as such), then the descriptor tables the
engine uploads (ordered reduce, dropout / drop-path masks, DropBlock sites) and the derived weight layouts its arena
registers (block-diagonal copies, packed k x k weights, transposed 1x1 weights, padded stem weight). Every device pointer,
in the arguments and in the tables, is replaced by the index of its first appearance, so two builds of the same plan give
the same text.

    python tools/plan_digest.py OUT.txt              # every configuration
    python tools/plan_digest.py OUT.txt --quick      # the small configurations only

Run it on two commits and diff the outputs.
"""
import argparse
import os
import struct
import sys
from contextlib import contextmanager
from unittest import mock

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from deepfake_detection_b200 import _lib  # noqa: E402
from deepfake_detection_b200.engine import Engine  # noqa: E402

SUFFIXES = ("_train", "_sync")

# (arch, batch, H, W, Engine kwargs)
SMALL = [
    ("efficientnet_b0", 2, 64, 64, {}),
    ("efficientnet_b0", 2, 64, 64, dict(drop_rate=0.2, drop_path_rate=0.2)),
    ("efficientnet_b0", 2, 64, 64, dict(sync_bn=True)),
    ("efficientnet_b0", 2, 64, 64, dict(gemm_impl="mma")),
    ("efficientnet_b0", 3, 64, 64, dict(drop_rate=0.2, drop_path_rate=0.2, sync_bn=True)),
    ("efficientnet_b4", 1, 76, 76, {}),
    ("efficientnet_b0", 4, 224, 224, {}),
    ("efficientnet_deepfake_v4", 1, 96, 96, dict(in_chans=12)),
    ("tf_efficientnet_b0", 2, 66, 96, {}),
    ("tf_efficientnet_b0", 2, 64, 96, {}),
    ("tf_efficientnet_b0", 2, 66, 96, dict(drop_rate=0.2, drop_path_rate=0.2)),
    ("resnet18", 2, 64, 64, {}),
    ("resnet18", 2, 64, 64, dict(gemm_impl="mma")),
    ("resnet18", 2, 64, 64, dict(in_chans=1)),
    ("resnet18", 2, 160, 224, dict(drop_block_rate=0.1)),
    ("resnet18", 2, 160, 160, dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.1)),
    ("resnet34", 2, 64, 64, dict(global_pool="avgmax")),
    ("resnet50", 2, 160, 160, dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.1)),
    ("resnet50", 2, 160, 160, dict(drop_path_rate=0.1)),
    ("resnet50", 3, 96, 96, {}),
    ("wide_resnet50_2", 2, 64, 64, {}),
    ("resnet26d", 2, 72, 88, {}),
    ("resnet50d", 2, 160, 160, dict(drop_rate=0.2, drop_path_rate=0.1, drop_block_rate=0.1)),
    ("resnet50d", 2, 64, 64, dict(gemm_impl="mma")),
    ("seresnet18", 2, 70, 72, {}),
    ("seresnet50", 2, 64, 64, dict(drop_rate=0.2)),
    ("seresnet50", 2, 64, 64, dict(gemm_impl="mma")),
    ("xception", 2, 64, 80, {}),
    ("xception", 2, 64, 80, dict(gemm_impl="mma")),
    ("xception", 2, 64, 80, dict(global_pool="catavgmax")),
] + [(a, 2, 64, 64, dict(global_pool=g)) for a in ("efficientnet_b0", "resnet18") for g in ("max", "avgmax", "catavgmax")]


def shipped_configs():
    from plan_launches import CONFIGS
    return [(arch, b, res, res, dict(kw, dtype=dt)) for _, arch, b, res, dt, kw in CONFIGS]


@contextmanager
def world_size(world):
    """a process group of `world` ranks, as a synchronised BatchNorm plan sees it"""
    if world == 1:
        yield
        return
    with mock.patch("torch.distributed.is_available", return_value=True), \
            mock.patch("torch.distributed.is_initialized", return_value=True), \
            mock.patch("torch.distributed.get_world_size", return_value=world):
        yield


class Pointers:
    """device pointer -> index of its first appearance"""

    def __init__(self):
        self.ids = {}

    def __call__(self, p):
        if not p:
            return "NULL"
        return "P%d" % self.ids.setdefault(p, len(self.ids))


def base_name(name):
    for suf in SUFFIXES:
        if name.endswith(suf):
            return name[:-len(suf)]
    return name


def op_line(ptr, name, args):
    if name.startswith("ALLREDUCE"):
        t, red = args
        return "%s(%s, %d, %s)" % (name, ptr(t.data_ptr()), t.numel(), red)
    codes = _lib.SIGNATURES[base_name(name)]
    out = []
    for v, c in zip(args, codes):
        if isinstance(v, tuple):
            out.append("%s:%s" % (v[0], ptr(v[1]) if c == "p" else repr(v[1])))
        elif c == "p" and v != "MIN_DST":
            out.append(ptr(v))
        else:
            out.append(repr(v))
    return "%s(%s)" % (name, ", ".join(out))


def table(ptr, raw, fmt, n_ptr):
    """decode a packed descriptor table: the first n_ptr fields of each entry are pointers"""
    size = struct.calcsize(fmt)
    rows = []
    for i in range(len(raw) // size):
        f = struct.unpack_from(fmt, raw, i * size)
        rows.append(", ".join([ptr(x) for x in f[:n_ptr]] + [repr(x) for x in f[n_ptr:]]))
    return rows


def as_bytes(t):
    return t.cpu().contiguous().view(torch.uint8).numpy().tobytes()


def digest(e):
    ptr, lines = Pointers(), []
    for part, ops, training in (("fwd", e.fwd_ops, True), ("bwd", e.bwd_ops, True), ("eval", e.fwd_ops, False)):
        for i, (_, name, args) in enumerate(ops):
            if name.startswith("ALLREDUCE"):
                lines.append("%s[%d] %s" % (part, i, op_line(ptr, name, args)))
                continue
            a = e.launch_args(name, args, training)
            if name == "dfd_ordered_reduce":
                # first_dst is the lowest destination address of the op's table entries: which entry that is depends on
                # where the host allocator put the arenas, so it is checked here and written as a symbol
                tab = as_bytes(e._red_table)
                off = a[0] - e._red_table.data_ptr()
                dsts = [struct.unpack_from("<QQ", tab, off + 40 * j)[1] for j in range(a[1])]
                assert a[2] == min(dsts), (part, i)
                a = (a[0], a[1], "MIN_DST", a[3])
            lines.append("%s[%d] %s" % (part, i, "%s SKIPPED" % name if a is None else op_line(ptr, name, a)))
    lines.append("n_launch %r" % sorted(e.n_launch.items()))
    if getattr(e, "_red_table", None) is not None:
        lines += ["reduce " + r for r in table(ptr, as_bytes(e._red_table), "<QQqqii", 2)]
    if getattr(e, "_mask_table", None) is not None:
        lines += ["mask " + r for r in table(ptr, as_bytes(e._mask_table), "<Qqifii", 1)]
    if getattr(e, "_drop_block_table", None) is not None:
        lines += ["dropblock " + r for r in table(ptr, as_bytes(e._drop_block_table), "<QQQdiiiiiiii", 3)]
    ar = e.arena
    for (B, Nn, K, pack), t in getattr(ar, "_bd_reg", {}).items():
        lines.append("blockdiag %s, %s, %d, %d, %d" % (ptr(B), ptr(t.data_ptr()), Nn, K, pack))
    if getattr(ar, "_rtable_count", 0):
        lines += ["repack " + r for r in table(ptr, as_bytes(ar._rtable)[:48 * ar._rtable_count], "<QQQQiiii", 4)]
    lines += ["transpose " + r for r in table(ptr, as_bytes(ar._ttable)[:24 * ar._ttable_count], "<QQii", 2)]
    for (name, O, taps, Kp), t in getattr(ar, "_stem_reg", {}).items():
        lines.append("stem_pad %s, %s, %d, %d, %d" % (name, ptr(t.data_ptr()), O, taps, Kp))
    return lines


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("out")
    ap.add_argument("--quick", action="store_true", help="the small configurations only")
    args = ap.parse_args()
    configs = SMALL + ([] if args.quick else shipped_configs())
    with open(args.out, "w") as f:
        for arch, batch, H, W, kw in configs:
            kw = dict(kw)
            head = "=== %s n=%d %dx%d %r" % (arch, batch, H, W, sorted(kw.items()))
            with world_size(2 if kw.get("sync_bn") else 1):
                try:
                    e = Engine(arch, batch, H, W, device="plan-only", **kw)
                except (ValueError, _lib.NativeError) as err:
                    f.write("%s\nREFUSED %s: %s\n" % (head, type(err).__name__, err))
                    continue
                f.write("\n".join([head] + digest(e)) + "\n")
                e = None
            print(arch, batch, H, W, kw, flush=True)


if __name__ == "__main__":
    main()
