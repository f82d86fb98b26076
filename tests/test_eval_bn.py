"""``eval_bn``: evaluation of the classifier drivers with train-mode BatchNorm (the reference's behaviour, SURVEY Q4) or
with eval-mode BatchNorm on the running statistics (``--eval_bn running``)."""
import pytest
import torch

from federated_pytorch_test_b200.api import common, federated_multi
from federated_pytorch_test_b200.config import CommonConfig, FederatedConfig, parse_config


def test_eval_bn_default_and_parsing():
    assert CommonConfig().eval_bn == "batch"
    assert FederatedConfig().eval_bn == "batch"
    assert parse_config(FederatedConfig, ["--eval_bn", "running"]).eval_bn == "running"
    assert parse_config(FederatedConfig, []).eval_bn == "batch"


def test_unknown_eval_bn_is_rejected():
    cfg = FederatedConfig(K=2, model="ResNet9", use_cuda=False, distributed=False, eval_bn="train")
    topo, _ = common.setup_runtime(cfg)
    with pytest.raises(ValueError, match="'batch' or 'running'"):
        common.ClassifierTask(cfg, topo)


def _bn_buffers(net):
    return {k: v.detach().clone() for k, v in net.named_buffers()
            if k.endswith(("running_mean", "running_var", "num_batches_tracked"))}


def _run_and_watch_evaluate(monkeypatch, eval_bn):
    """A tiny CPU run of federated_multi with ResNet9; every ``ClassifierTask.evaluate`` call is recorded with the BatchNorm
    buffers before and after it, the training flags afterwards, the reported accuracies and, in eval mode, a hand-written
    ``net.eval()`` + argmax loop over the same test loader."""
    calls = []
    original = common.ClassifierTask.evaluate

    def watched(self, reps, engine):
        before = [_bn_buffers(r.nets["net"]) for r in reps]
        accs = original(self, reps, engine)
        after = [_bn_buffers(r.nets["net"]) for r in reps]
        training = [all(m.training for m in r.nets["net"].modules()) for r in reps]
        manual = []
        if eval_bn == "running":
            with torch.no_grad():
                for r in reps:
                    net = r.nets["net"]
                    net.eval()
                    correct = total = 0
                    for x, y in self.test_loader(r.ck):
                        correct += int((net(x).argmax(dim=1) == y).sum())
                        total += y.shape[0]
                    net.train()
                    manual.append(100.0 * correct / total)
        calls.append(dict(before=before, after=after, training=training, accs=accs, manual=manual))
        return accs

    monkeypatch.setattr(common.ClassifierTask, "evaluate", watched)
    cfg = federated_multi.Config(K=2, model="ResNet9", Nloop=1, Nadmm=1, max_minibatches=1, check_results=True, save_model=False,
                                 train_size=128, test_size=48, default_batch=16, use_cuda=False, distributed=False,
                                 collective="torch", eval_bn=eval_bn)
    federated_multi.run(cfg, log=lambda s: None)
    assert calls, "evaluate was never called"
    return calls


def test_running_eval_leaves_batchnorm_buffers_and_mode_unchanged(monkeypatch):
    calls = _run_and_watch_evaluate(monkeypatch, "running")
    for c in calls:
        assert all(c["training"]), "networks must be back in training mode after evaluation"
        for before, after in zip(c["before"], c["after"]):
            assert before.keys() == after.keys() and before
            for k in before:
                assert torch.equal(before[k], after[k]), k
        assert c["accs"] == c["manual"]


def test_batch_eval_updates_running_statistics(monkeypatch):
    """The default keeps the reference's behaviour (Q4): evaluation runs BatchNorm in training mode, so the test batches
    move the running statistics."""
    calls = _run_and_watch_evaluate(monkeypatch, "batch")
    for c in calls:
        assert all(c["training"])
        for before, after in zip(c["before"], c["after"]):
            assert any(not torch.equal(before[k], after[k]) for k in before if k.endswith("running_mean"))
            assert any(int(after[k]) > int(before[k]) for k in before if k.endswith("num_batches_tracked"))
