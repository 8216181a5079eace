"""CPU ORACLE — TEST INFRASTRUCTURE (see oracle/model.py header).

Plain torch restatements of the small formulas around the step, pinned to the reference by tests/golden/aux_formulas.json
(tests/test_oracle_vs_reference_goldens.py::test_aux_formulas_match_reference):

  drop_path_mask : dfd/timm/models/layers/drop.py:94-99   mask = floor(keep + u) / keep, one u per sample
  normalize_u8   : dfd/timm/data/loader.py:229-230,250-253  uint8 -> float, (x - mean*255) / (std*255), per-frame repeat
  ema_update     : dfd/timm/utils.py:329-340             ema*decay + (1-decay)*model, copy_() back into the buffer's dtype

and the DropBlock formulas of drop_block_2d (dfd/timm/models/layers/drop.py:24-61), pinned by tests/golden/drop_block_formulas.json
(tests/test_resnet_drop_cpu.py::test_drop_block_formulas_reproduced_exactly).
"""
import torch
import torch.nn.functional as F


def drop_path_mask(u, drop_prob):
    keep = 1.0 - drop_prob
    return torch.floor(keep + u) / keep


def drop_block_gamma(H, W, rate, gamma_scale, block_size=7):
    """(gamma, clipped block size) exactly as drop_block_2d computes them (drop.py:36-42)"""
    cb = min(block_size, min(W, H))
    return gamma_scale * rate * (W * H) / cb ** 2 / ((W - block_size + 1) * (H - block_size + 1)), cb


def valid_block(H, W, cb):
    """drop.py:45-48: built on a [W, H] meshgrid and reshaped to [H, W] (scrambled for non-square maps)"""
    w_i, h_i = torch.meshgrid(torch.arange(W), torch.arange(H), indexing="ij")
    v = ((w_i >= cb // 2) & (w_i < W - (cb - 1) // 2)) & ((h_i >= cb // 2) & (h_i < H - (cb - 1) // 2))
    return torch.reshape(v, (1, 1, H, W)).float()


def seeds_from_noise(u, gamma, cb):
    """[N, C, H, W] 0/1 seed-keep mask from the uniform draws, in the reference's fp32 order (drop.py:51)"""
    H, W = u.shape[-2:]
    return ((2 - gamma - valid_block(H, W, cb) + u) >= 1).float()


def block_from_seeds(seeds, cb):
    """drop.py:52-56: min-pool of the seeds (the -inf padding of max_pool2d is ignored)"""
    return -F.max_pool2d(-seeds, kernel_size=cb, stride=1, padding=cb // 2)


def drop_block_apply(x, m):
    """drop.py:60-61"""
    return x * m * (m.numel() / (torch.sum(m) + 1e-7))


def normalize_u8(x_u8, mean, std, img_num):
    c = 3 * img_num
    m = torch.tensor([[v * 255 for v in mean] for _ in range(img_num)]).view(1, c, 1, 1)
    s = torch.tensor([[v * 255 for v in std] for _ in range(img_num)]).view(1, c, 1, 1)
    return x_u8.float().sub_(m).div_(s)


def ema_update(ema_v, model_v, decay):
    out = ema_v.clone()
    out.copy_(ema_v * decay + (1.0 - decay) * model_v)
    return out
