"""Training through the cost volume, without a GPU: the fp64 restatement (oracle/train.py) reproduces the reference's own
training step stored in the fixtures, install_training keeps a reference-constructed model's parameters, and it refuses
the configurations it does not implement."""
import copy

import pytest
import torch

from oracle import reference
from tests import train_common as T


@pytest.mark.parametrize("name", T.CASES)
def test_restatement_reproduces_reference_step(name):
    g, _, _ = T.fixture(name)
    r = T.restated_step(g)
    assert T.rel(r["volume"], g["volume_mean"]) < T.FIXTURE_TOL
    assert T.rel(r["features_grad"], g["features_grad"]) < T.FIXTURE_TOL
    assert sorted(r["grads"]) == sorted(k[len("grad."):] for k in g if k.startswith("grad."))
    for k, v in r["grads"].items():
        assert T.rel(v, g["grad." + k]) < T.FIXTURE_TOL, k
    for k, v in r["running"].items():
        assert T.rel(v, g["after." + k]) < T.FIXTURE_TOL, k


def _reference_model():
    if reference.root("models", reference.CONFIG) is None:
        pytest.skip("the reference's sources are not available")
    reference.import_models()
    from models.networks.DINOv2_mvsformer_model import DINOv2MVSNet
    cfg = reference.config()
    cfg["vit_path"] = ""
    torch.manual_seed(0)
    return DINOv2MVSNet(cfg), cfg


def test_install_training_keeps_parameters():
    from mvsformerplusplus_b200 import install_training
    model, _ = _reference_model()
    params = {k: p for k, p in model.named_parameters()}
    keys = list(model.state_dict().keys())
    modules = {k: m for k, m in model.named_modules()}
    assert install_training(model) is model
    assert {k: p for k, p in model.named_parameters()}.keys() == params.keys()
    assert all(p is params[k] for k, p in model.named_parameters())
    assert list(model.state_dict().keys()) == keys
    assert all(m is modules[k] for k, m in model.named_modules())
    for stage in model.fusions:
        assert stage.forward.__func__.__module__ == "mvsformerplusplus_b200.training"


@pytest.mark.parametrize("field,value", [("fusion_type", "pcd"), ("depth_type", "reg"), ("base_ch", 4)])
def test_install_training_refuses_unimplemented(field, value):
    from mvsformerplusplus_b200 import install_training
    model, _ = _reference_model()
    stage = model.fusions[2]
    if field == "base_ch":
        stage.args = copy.deepcopy(stage.args)
        stage.args["base_ch"] = [8, 8, value, 8]
    else:
        setattr(stage, field, value)
    forwards = [s.forward for s in model.fusions]
    with pytest.raises(NotImplementedError):
        install_training(model)
    assert [s.forward for s in model.fusions] == forwards   # nothing was rebound


def test_install_training_refuses_package_stagenet():
    from mvsformerplusplus_b200 import HotPathNet, default_args, install_training
    with pytest.raises(NotImplementedError, match="parameter container"):
        install_training(HotPathNet(default_args()))
