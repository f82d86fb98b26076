"""Record what the original federated-pytorch-test code computes, as small golden fixtures for the test suite.

    python oracle/make_golden.py /path/to/federated-pytorch-test/src

writes ``tests/golden/reference_outputs.pt``.  The tests that compare this package with the original project read that
file, so they run without the original sources.  Weights come from ``fill_state`` (tests/conftest.py): a seeded fill of
every floating-point state-dict entry in order, identical for both implementations, so only the math is compared.
Large vectors (initialised weights, packed blocks) are stored as a fixed seeded sample plus their float64 sum.
"""
import importlib.util
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import fill_state, sample_index  # noqa: E402  (the tests fill weights and sample the same way)


def load(src, name):
    spec = importlib.util.spec_from_file_location("_orig_" + name, os.path.join(src, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def sample(v):
    v = v.detach().reshape(-1)
    return {"n": v.numel(), "values": v[sample_index(v.numel())].clone(), "sum": float(v.double().sum())}


def main(src):
    warnings.filterwarnings("ignore")
    rm, rl, ru = load(src, "simple_models"), load(src, "lbfgsnew"), load(src, "simple_utils")
    out = {}

    # ---- model forwards (test_models.py)
    pairs = {"Net": (lambda m: m.Net(), (4, 3, 32, 32)), "Net1": (lambda m: m.Net1(), (4, 3, 32, 32)),
             "Net2": (lambda m: m.Net2(), (4, 3, 32, 32)), "ResNet18": (lambda m: m.ResNet18(), (4, 3, 32, 32)),
             "ResNet9": (lambda m: m.ResNet9(), (4, 3, 32, 32)), "ContextgenCNN": (lambda m: m.ContextgenCNN(32), (2, 32, 3, 3))}
    fw = {}
    for name, (make, shape) in pairs.items():
        net = fill_state(make(rm))
        x = torch.randn(*shape, generator=torch.Generator().manual_seed(1))
        with torch.no_grad():
            y_train = net.train()(x)               # batch statistics, as in training
            fill_state(net)                        # the train-mode pass updated the running statistics
            fw[name] = {"keys": list(net.state_dict().keys()), "y_train": y_train, "y": net.eval()(x)}
    out["forward"] = fw
    with torch.no_grad():
        enc = fill_state(rm.EncoderCNN(64)).eval()
        x = torch.randn(6, 8, 32, 32, generator=torch.Generator().manual_seed(2))
        pred = fill_state(rm.PredictorCNN(64, 8)).eval()
        a = torch.randn(2, 64, 3, 3, generator=torch.Generator().manual_seed(3))
        b = torch.randn(2, 64, 3, 3, generator=torch.Generator().manual_seed(4))
        out["encoder_predictor"] = {"enc": enc(x), "pred": [t.clone() for t in pred(a, b)]}
        vae = fill_state(rm.AutoEncoderCNN()).eval()
        x = torch.rand(3, 3, 32, 32, generator=torch.Generator().manual_seed(5))
        z = torch.randn(3, 10, generator=torch.Generator().manual_seed(6))
        out["vae"] = {"encode": [t.clone() for t in vae.encode(x)], "decode": vae.decode(z)}
        cl = fill_state(rm.AutoEncoderCNNCL(K=4, L=8)).eval()
        x = torch.rand(5, 3, 32, 32, generator=torch.Generator().manual_seed(8))
        ek = torch.zeros(5, 4)
        ek[:, 2] = 1
        z = torch.randn(5, 8, generator=torch.Generator().manual_seed(9))
        out["vae_cl"] = {"encodeclus": cl.encodeclus(x), "encode": [t.clone() for t in cl.encode(x, ek)],
                         "decode": [t.clone() for t in cl.decode(ek, z)]}

    # ---- packing and initialisation (test_utils_flat.py)
    net = fill_state(rm.Net(), seed=1)
    packs = []
    for blk in range(5):
        ru.unfreeze_one_block(net, blk)
        packs.append(sample(ru.get_trainable_values(net)))
    out["pack"] = packs
    r9 = rm.ResNet9()
    torch.manual_seed(0)
    r9.apply(ru.init_weights)
    out["init_weights"] = {k: sample(v) for k, v in r9.state_dict().items() if v.is_floating_point()}

    # ---- L-BFGS (test_lbfgs.py)
    import test_lbfgs as tl
    x, calls, iters, evals = tl._rosenbrock(rl.LBFGSNew)
    log, vec, opt = tl._stochastic(rl.LBFGSNew)
    out["lbfgs"] = {"rosenbrock": (x, calls, iters, evals), "stochastic_counts": [e[1:] for e in log],
                    "stochastic_vec": vec.detach().clone(), "state_keys": sorted(opt.state_dict()["state"][0].keys())}

    # ---- one ADMM block visit in the original recipe (test_engine.py)
    import test_engine as te
    out["block_visit"] = te.reference_style_block_visit(rm, ru)

    # ---- checkpoint interop (test_config_ckpt_logs.py): the original's state-dict layout of Net
    out["net_state_layout"] = [(k, tuple(v.shape)) for k, v in rm.Net().state_dict().items()]

    dst = os.path.join(ROOT, "tests", "golden", "reference_outputs.pt")
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    torch.save(out, dst)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("FEDERATED_PYTORCH_TEST_SRC", "src"))
