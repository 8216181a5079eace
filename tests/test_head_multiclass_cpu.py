"""The oracle's loss for class counts other than 2, against torch's own. The K-class fixtures under tests/golden/ were produced
by the UNMODIFIED reference (tools/mint_multiclass_goldens.py) and are held by tests/reference_steps.py's tables."""
import torch

from oracle import model as OM


def test_oracle_cross_entropy_is_k_general():
    """oracle/model.py::cross_entropy against torch's own losses at K = 5 and 1000 (hard, smoothed, soft targets)."""
    g = torch.Generator().manual_seed(0)
    for K in (5, 1000):
        z = torch.randn(16, K, generator=g, dtype=torch.float64) * 3
        y = torch.randint(0, K, (16,), generator=g)
        assert torch.allclose(OM.cross_entropy(z, y), torch.nn.functional.cross_entropy(z, y))
        assert torch.allclose(OM.cross_entropy(z, y, 0.1), torch.nn.functional.cross_entropy(z, y, label_smoothing=0.1))
        t = torch.softmax(torch.randn(16, K, generator=g, dtype=torch.float64), -1)
        assert torch.allclose(OM.cross_entropy(z, t), torch.nn.functional.cross_entropy(z, t))
