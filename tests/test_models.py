"""Model zoo: shapes, parameter/block inventory (SURVEY §2.2) and forward parity with the original models (stored
outputs of the original code on the same seeded weights and inputs: tests/golden, oracle/make_golden.py)."""
import pytest
import torch

from federated_pytorch_test_b200 import models
from federated_pytorch_test_b200.ops import functional as FX

SPEC = [  # (factory, #tensors, #params)
    (models.Net, 10, 62006), (models.Net1, 12, 890410), (models.Net2, 18, 2513418),
    (models.ResNet18, 62, 11173962), (models.ResNet9, 38, 4903242),
    (models.AutoEncoderCNN, 24, 205679), (lambda: models.AutoEncoderCNNCL(10, 32), 42, 350744),
    (lambda: models.EncoderCNN(256), 16, 701928), (lambda: models.ContextgenCNN(256), 4, 98304),
    (lambda: models.PredictorCNN(256, 32), 2, 16384),
]


@pytest.mark.parametrize("factory,ntensors,nparams", SPEC)
def test_inventory(factory, ntensors, nparams):
    net = factory()
    ps = list(net.parameters())
    assert len(ps) == ntensors
    assert sum(p.numel() for p in ps) == nparams
    covered = []
    for lo, hi in net.train_order_block_ids():
        covered += list(range(lo, hi + 1))
    assert sorted(covered) == list(range(ntensors)), "blocks must cover every parameter index exactly once"


def test_resnet18_block_sizes():
    net = models.ResNet18()
    sizes = [net.block_numel(i) for i in range(10)]
    assert sizes == [1856, 73984, 73984, 230144, 295424, 919040, 1180672, 3673088, 4720640, 5130]
    assert [models.Net().block_numel(i) for i in range(5)] == [48120, 456, 2416, 10164, 850]


def test_protocol_methods():
    net = models.Net()
    assert net.linear_layer_ids() == [4, 6, 8]
    assert net.train_order_block_ids() == [[4, 5], [0, 1], [2, 3], [6, 7], [8, 9]]
    assert net.linear_layer_parameters().numel() == 48120 + 10164 + 850
    assert models.ResNet18().linear_layer_ids() == []


PAIRS = [("Net", lambda m: m.Net(), (4, 3, 32, 32)), ("Net1", lambda m: m.Net1(), (4, 3, 32, 32)),
         ("Net2", lambda m: m.Net2(), (4, 3, 32, 32)), ("ResNet18", lambda m: m.ResNet18(), (4, 3, 32, 32)),
         ("ResNet9", lambda m: m.ResNet9(), (4, 3, 32, 32)),
         ("ContextgenCNN", lambda m: m.ContextgenCNN(32), (2, 32, 3, 3))]


@pytest.mark.parametrize("name,make,shape", PAIRS)
def test_forward_matches_reference(golden, fill, name, make, shape):
    """Same state_dict keys, and the original's outputs for the same weights and input, in train mode (BatchNorm on batch
    statistics) and in eval mode (running statistics)."""
    FX.set_fast_path(False)
    ref = golden["forward"][name]
    mine = fill(make(models))
    assert list(mine.state_dict().keys()) == ref["keys"]
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        torch.testing.assert_close(mine.train()(x), ref["y_train"], rtol=1e-5, atol=1e-5)
        fill(mine)
        torch.testing.assert_close(mine.eval()(x), ref["y"], rtol=1e-5, atol=1e-5)


def test_encoder_predictor_match_reference(golden, fill):
    ref = golden["encoder_predictor"]
    with torch.no_grad():
        mine = fill(models.EncoderCNN(64)).eval()
        x = torch.randn(6, 8, 32, 32, generator=torch.Generator().manual_seed(2))
        torch.testing.assert_close(mine(x), ref["enc"], rtol=1e-5, atol=1e-5)
        mp = fill(models.PredictorCNN(64, 8)).eval()
        a = torch.randn(2, 64, 3, 3, generator=torch.Generator().manual_seed(3))
        b = torch.randn(2, 64, 3, 3, generator=torch.Generator().manual_seed(4))
        for u, v in zip(mp(a, b), ref["pred"]):
            torch.testing.assert_close(u, v)


def test_vae_deterministic_parts_match_reference(golden, fill):
    ref = golden["vae"]
    with torch.no_grad():
        mine = fill(models.AutoEncoderCNN()).eval()
        x = torch.rand(3, 3, 32, 32, generator=torch.Generator().manual_seed(5))
        for u, v in zip(mine.encode(x), ref["encode"]):
            torch.testing.assert_close(u, v, rtol=1e-5, atol=1e-6)
        z = torch.randn(3, 10, generator=torch.Generator().manual_seed(6))
        torch.testing.assert_close(mine.decode(z), ref["decode"], rtol=1e-5, atol=1e-6)


def test_vae_cl_batched_equals_loop(golden, fill):
    ref = golden["vae_cl"]
    a = fill(models.AutoEncoderCNNCL(K=4, L=8, batched_clusters=True)).eval()
    b = models.AutoEncoderCNNCL(K=4, L=8, batched_clusters=False).eval()
    b.load_state_dict(a.state_dict())
    a.force_disable_repr()
    b.force_disable_repr()
    x = torch.rand(5, 3, 32, 32, generator=torch.Generator().manual_seed(8))
    with torch.no_grad():
        torch.testing.assert_close(a.encodeclus(x), ref["encodeclus"], rtol=1e-5, atol=1e-6)
        oa, ob = a(x), b(x)
        torch.testing.assert_close(oa[0], ob[0])
        for da, db in zip(oa[1:], ob[1:]):
            for k in range(4):
                torch.testing.assert_close(da[k], db[k], rtol=1e-5, atol=1e-6)
        # deterministic heads against the original, cluster by cluster
        ek = torch.zeros(5, 4)
        ek[:, 2] = 1
        for u, v in zip(a.encode(x, ek), ref["encode"]):
            torch.testing.assert_close(u, v, rtol=1e-5, atol=1e-6)
        z = torch.randn(5, 8, generator=torch.Generator().manual_seed(9))
        for u, v in zip(a.decode(ek, z), ref["decode"]):
            torch.testing.assert_close(u, v, rtol=1e-5, atol=1e-6)


def test_disable_repr_quirk_preserved():
    net = models.AutoEncoderCNNCL(2, 4)
    net.disable_repr()
    assert net.repr_flag is True  # SURVEY Q11
    net.force_disable_repr()
    assert net.repr_flag is False
