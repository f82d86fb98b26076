import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs.pt")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


@pytest.fixture(scope="session")
def golden():
    """What the original federated-pytorch-test code computed for the cases below (written by oracle/make_golden.py)."""
    import torch

    return torch.load(GOLDEN, weights_only=False)


def fill_state(net, seed=0):
    """Deterministic weights for comparisons with the golden outputs: N(0, 0.05^2) everywhere, running variances in
    [0.5, 1.5).  Every floating-point state-dict entry is drawn in state-dict order from one seeded generator."""
    import torch

    g = torch.Generator().manual_seed(seed)
    new = {}
    for k, v in net.state_dict().items():
        if not v.is_floating_point():
            new[k] = v
        elif k.endswith("running_var"):
            new[k] = torch.rand(v.shape, generator=g) + 0.5
        else:
            new[k] = torch.randn(v.shape, generator=g) * 0.05
    net.load_state_dict(new)
    return net


def sample_index(n, size=1024):
    """The fixed, seeded sample of positions of an n-element vector that the golden file stores."""
    import torch

    return torch.randperm(n, generator=torch.Generator().manual_seed(7))[:size].sort().values


def assert_matches_sample(vec, ref, rtol=0.0, atol=0.0):
    """``vec`` against the stored seeded sample (``values`` at ``sample_index``) and float64 sum of the original's vector."""
    import torch

    vec = vec.detach().reshape(-1)
    assert vec.numel() == ref["n"]
    torch.testing.assert_close(vec[sample_index(vec.numel())], ref["values"], rtol=rtol, atol=atol)
    s = float(vec.double().sum())
    assert s == pytest.approx(ref["sum"], rel=max(rtol, 1e-12), abs=atol * ref["n"] ** 0.5 + 1e-12)


@pytest.fixture(scope="session")
def fill():
    return fill_state


@pytest.fixture(scope="session")
def matches_sample():
    return assert_matches_sample
