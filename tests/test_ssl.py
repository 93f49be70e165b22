"""CPU: the self-supervised models (SimCLR, BYOL, MemoryBank), make_multilayer_perceptron, the NaiveSyncBatchNorm
classes and SoftTargetCrossEntropyLoss - module trees and state_dict keys against tests/golden/ssl.pt (written by
oracle/gen_golden_ssl.py from the reference), host RNG draws bit for bit, argument errors, and dry-run lowerings of the
embedding plans."""
import os
import types

import pytest
import torch
import torch.nn as nn

from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine.lower import lower_only
from pytorchvideo_b200.layers import (NaiveSyncBatchNorm1d, NaiveSyncBatchNorm2d, NaiveSyncBatchNorm3d,
                                      make_multilayer_perceptron)
from pytorchvideo_b200.losses import SoftTargetCrossEntropyLoss
from pytorchvideo_b200.models.byol import BYOL
from pytorchvideo_b200.models.embedding import EmbeddingChain
from pytorchvideo_b200.models.memory_bank import MemoryBank
from pytorchvideo_b200.models.resnet import create_resnet
from pytorchvideo_b200.models.simclr import SimCLR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ssl.pt")
NS = types.SimpleNamespace(SimCLR=SimCLR, BYOL=BYOL, MemoryBank=MemoryBank, create_resnet=create_resnet,
                           make_multilayer_perceptron=make_multilayer_perceptron)


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.mark.parametrize("name", TS.SSL_CASES)
def test_tree_and_state_dict_match_reference(gold, name):
    m, _ = TS.build_ssl_case(name, NS)
    assert TS.tree_digests(m) == gold["cases"][name]["tree"]
    fresh, _ = TS.build_ssl_case(name, NS, seed=5)
    fresh.load_state_dict(m.state_dict(), strict=True)
    for (k, a), (k2, b) in zip(m.state_dict().items(), fresh.state_dict().items()):
        assert k == k2 and torch.equal(a, b)


@pytest.mark.parametrize("dims,kw", [([8, 4, 2], {}), ([2048, 2048, 128], {"norm": nn.BatchNorm1d}),
                                     ([16, 0, 4], {"dropout_rate": 0.5, "final_activation": None})])
def test_mlp_matches_reference(gold, dims, kw):
    mlp, od = make_multilayer_perceptron(dims, **kw)
    g = gold["mlp"][str(dims)]
    assert repr(mlp) == g["repr"] and list(mlp.state_dict()) == g["keys"] and od == g["output_dim"]


def test_mlp_asserts():
    for bad in ([8], (8, 4), [8, 4.0], [8, -1], [8, True]):
        with pytest.raises(AssertionError):
            make_multilayer_perceptron(bad)


def test_naive_sync_bn_constructors():
    for cls in (NaiveSyncBatchNorm1d, NaiveSyncBatchNorm2d, NaiveSyncBatchNorm3d):
        bn = cls(num_features=6)
        assert bn.global_sync and bn.num_features == 6 and list(bn.state_dict()) == list(
            nn.BatchNorm1d(6).state_dict())
        local = cls(num_sync_devices=0, global_sync=False, num_features=4)
        assert local.num_sync_devices == 1 and local.num_groups == 1
        with pytest.raises(ValueError):
            cls(num_sync_devices=2, num_features=4)
        with pytest.raises(ValueError):
            cls(global_sync=False, num_features=4)
        with pytest.raises(RuntimeError):
            bn.eval()(torch.zeros(2, 6))


def test_memory_bank_host_draws_match_reference(gold):
    m, (x, x_ind) = TS.build_ssl_case("memory_bank_video", NS)
    g = gold["cases"]["memory_bank_video"]
    assert TS.tensor_checksum(m.memory) == g["memory"]
    torch.manual_seed(77)
    assert torch.equal(m.draw_indices(x.shape[0], x_ind, "cpu"), g["indices"])
    m, (x, x_ind) = TS.build_ssl_case("memory_bank_unit", NS)
    torch.manual_seed(77)
    assert torch.equal(m.draw_indices(x.shape[0], x_ind, "cpu"), gold["cases"]["memory_bank_unit"]["indices"])


@pytest.mark.parametrize("dt", ["f16", "f32"])
@pytest.mark.parametrize("width", [2, 4, 8])
def test_lower_only_narrow_rows(dt, width):
    mlp, _ = make_multilayer_perceptron([width, 16, width], norm=nn.BatchNorm1d, dropout_rate=0.1)
    plan, shape = lower_only(EmbeddingChain(nn.Linear(width, width), mlp.eval()), torch.zeros(3, width), dtype=dt)
    names = [m["name"] for m in plan.meta]
    assert shape == (3, width)
    # Linear, Linear+BN+ReLU, Linear: three GEMM launches (the BatchNorm folds away); Dropout is the identity and the
    # final ReLU after it, with no Linear right before it, is its own activation launch
    assert [n for n in names if n.startswith("seq.")] == ["seq.0", "seq.1.0", "seq.1.3", "seq.1.5"]


def test_lower_only_headless_trunk_and_projector():
    trunk = TS._slow_r50_trunk(NS)
    mlp, _ = make_multilayer_perceptron([2048, 2048, 128], norm=lambda d: NaiveSyncBatchNorm1d(num_features=d))
    plan, shape = lower_only(EmbeddingChain(trunk.eval(), mlp.eval()), torch.zeros(2, 3, 8, 224, 224))
    names = [m["name"] for m in plan.meta]
    assert shape == (2, 128)
    assert names[-3:] == ["seq.1.0", "seq.1.3", "output.to_tokens"]
    assert "seq.0.blocks.5.pool" in names and not any("proj" in n for n in names)


def test_lower_only_byol_default_predictor():
    byol = BYOL(backbone=nn.Linear(16, 8), feature_dim=8, predictor_inner=32).eval()   # nn.SyncBatchNorm
    plan, shape = lower_only(EmbeddingChain(byol.backbone, byol.predictor), torch.zeros(4, 16))
    assert shape == (4, 8)
    assert [m["name"] for m in plan.meta if m["name"].startswith("seq.")] == ["seq.0", "seq.1.0", "seq.1.3"]
    plan, shape = lower_only(EmbeddingChain(byol.backbone_mmt), torch.zeros(4, 16))
    assert shape == (4, 8)


def test_bn_without_running_stats_refused():
    seq = nn.Sequential(nn.Linear(8, 8), nn.BatchNorm1d(8, track_running_stats=False))
    with pytest.raises(NotImplementedError):
        lower_only(EmbeddingChain(seq.eval()), torch.zeros(2, 8))


def test_wrappers_refuse_cpu_and_training():
    for name in ("simclr_unit", "byol_unit", "memory_bank_unit"):
        m, args = TS.build_ssl_case(name, NS)
        with pytest.raises(RuntimeError):
            m(*args)
        m.train()
        with pytest.raises(RuntimeError):
            m(*args)


def test_byol_mmt_accessors():
    byol = BYOL(backbone=nn.Linear(8, 4), projector=nn.Linear(4, 4), feature_dim=4, norm=nn.BatchNorm1d)
    assert byol.get_mmt() == 0.99
    byol.update_mmt(0.5)
    assert byol.get_mmt() == 0.5
    assert all(not p.requires_grad for p in byol.backbone_mmt.parameters())


def test_soft_target_ce_argument_errors():
    with pytest.raises(NotImplementedError):
        SoftTargetCrossEntropyLoss(reduction="sum")
    with pytest.raises(AssertionError):
        SoftTargetCrossEntropyLoss(normalize_targets=1)
    loss = SoftTargetCrossEntropyLoss()
    with pytest.raises(AssertionError):
        loss(torch.zeros(3, 4), torch.zeros(3, 5))
    with pytest.raises(AssertionError):
        loss(torch.zeros(3, 4), torch.zeros(2, dtype=torch.long))
    # the reference reads the misspelt self.ignore_idx for an ignore_index inside [0, C)
    with pytest.raises(AttributeError):
        SoftTargetCrossEntropyLoss(ignore_index=2)(torch.zeros(3, 4), torch.zeros(3, 4))
    with pytest.raises(RuntimeError):           # no CPU path
        SoftTargetCrossEntropyLoss(ignore_index=4)(torch.zeros(3, 4), torch.zeros(3, 4))
